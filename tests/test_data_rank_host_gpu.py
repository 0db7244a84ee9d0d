"""GPU: the native pipeline with a data rank WITHOUT a GPU outside the stage pipeline (`runtime.py -d cpu -D 0 -r 1,...`).
The data rank's process hides every GPU before anything touches CUDA and never creates a context: it publishes its
micro-batches into a ring in shared memory, which the first stage copies out of with its copy engine, and reads the
results the last stage's send kernel stores into a second ring. Results bit for bit against the same shards and
QuantPipe hooks run locally (which the pipelines with the data rank inside and with a GPU feeder outside match bit for
bit, `test_pipeline_gpu.py` / `test_data_rank_native_gpu.py`); every stage rank shares one GPU."""
import faulthandler
import os
import subprocess
import sys
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _multirank as mr  # noqa: E402
SEQS = (32, 16)   # BERT: the sequence length alternates between micro-batches (two graph shapes)


def _input(spec, i, n_ubatch, ubatch):
    from pipeedge_b200.synth import synth_input
    return synth_input(spec, mr.ragged(i, n_ubatch, ubatch), seed=10 + i, seq_len=SEQS[i % 2])


def _rank_main(rank, worker, world, port, args, env, out_q):
    if rank == 0:
        os.environ['CUDA_VISIBLE_DEVICES'] = ''   # the data rank: before anything touches CUDA
    faulthandler.enable()
    faulthandler.dump_traceback_later(400, exit=True)   # a hung rank shows where, and ends
    sys.path.insert(0, mr.ROOT)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), PIPEEDGE_LINK_TIMEOUT_S='60', **env)
    if rank > 0:
        torch.cuda.set_device(0)
    out_q.put((rank, worker(rank, world, *args)))
    faulthandler.cancel_dump_traceback_later()
    out_q.close()
    out_q.join_thread()


def _spawn(worker, world, args, env):
    """As `_multirank.spawn`, with the GPUs hidden from rank 0."""
    ctx = torch.multiprocessing.get_context('spawn')
    out_q = ctx.Queue()
    port = mr.free_port()
    procs = [ctx.Process(target=_rank_main, args=(r, worker, world, port, args, env, out_q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    try:
        for _ in range(world):
            rank, result = out_q.get(timeout=600)
            got[rank] = result
    finally:
        for p in procs:
            p.join(180)
            if p.is_alive():
                p.kill()
                p.join(10)
    for r, p in enumerate(procs):
        assert p.exitcode == 0, f"rank {r} exited with {p.exitcode}"
    return got


def _worker(rank, world, name, cuts, qbits, n_ubatch, ubatch, hooked):
    import threading
    import model_cfg
    from pipeedge_b200.comm.p2p import DistP2pContext
    from pipeedge_b200.synth import MODEL_SPECS
    spec = MODEL_SPECS[name]
    stage_ranks = list(range(1, world))
    s = rank - 1 if rank > 0 else None
    shard = mr.make_shard(name, cuts, s, qbits[s]) if s is not None else None
    stop = threading.Event()
    results, done, sends = [], threading.Event(), []

    def results_cb(t):
        results.append(t.numpy())
        if len(results) == n_ubatch:
            done.set()

    out = {}
    with DistP2pContext(('gloo',), {'world_size': world, 'rank': rank}, lambda c, t: stop.set() if c == 0 else None) as ctx:
        with model_cfg.dist_p2p_pipeline_stage_factory(stage_ranks, 0, rank, s, shard, results_cb) as stage:
            native = stage.native
            assert native is not None, "the native pipeline was not selected"
            if rank == 0:
                assert type(native).__name__ == 'NativeHostFeeder'
                if hooked:
                    stage.register_send_timing_hook(lambda mbits, sec: sends.append((mbits, sec)), ())
                for i in range(n_ubatch):
                    stage.enqueue_tensor(_input(spec, i, n_ubatch, ubatch))
                assert done.wait(300), "results did not arrive"
                stage.check_workers()
                ctx.cmd_broadcast(0)
            else:
                assert stop.wait(420)
                stage.check_workers()
    if rank == 0:
        out.update(results=results, sends=sends, geometry=native.input_geometry,
                   cuda_initialized=torch.cuda.is_initialized(), shm=[f for f in os.listdir('/dev/shm')
                                                                      if f.startswith('pipeedge_b200_')])
    return out


@pytest.mark.parametrize('name,cuts,qbits,slots,hooked', [
    ('test/vit-tiny', (6, 12), (0, 0), 4, True),         # raw hop; send-timing hook on the data rank
    ('test/vit-tiny', (5, 12), (8, 0), 2, False),        # tuple payload (ctx, skip), fused 8-bit send; 2-slot rings
    ('test/bert-tiny', (7, 12), (4, 0), 4, False),       # int64 token ids of two sequence lengths, 4-bit
    ('test/deit-tiny', (4, 6, 8), (8, 6, 0), 4, False),  # three stages: fused 8-bit and staged 6-bit hops
    ('test/vit-tiny', (12,), (0,), 4, False),            # one stage: both of its hops go to the data rank
])
def test_host_data_rank_is_bit_identical_and_never_opens_a_context(name, cuts, qbits, slots, hooked):
    """18 micro-batches (not a multiple of the ring's slots), the last one ragged, through the shared-memory rings:
    results in FIFO order, bit-identical to the local shards and hooks; the data rank never initialised CUDA and left
    no segment behind; a send-timing hook on it fires once per micro-batch with the input's Mbit."""
    from pipeedge_b200.synth import MODEL_SPECS
    spec = MODEL_SPECS[name]
    n_ubatch, ubatch = 18, 3
    got = _spawn(_worker, len(cuts) + 1, (name, cuts, qbits, n_ubatch, ubatch, hooked),
                 {'PIPEEDGE_NATIVE': '1', 'PIPEEDGE_LINK_SLOTS': str(slots)})
    out = got[0]
    assert out['cuda_initialized'] is False
    assert out['shm'] == []
    nbytes, dtype, ndim = out['geometry']
    assert (dtype, ndim) == ((torch.int64, 2) if 'bert' in name else (torch.float32, 4))
    inputs = [_input(spec, i, n_ubatch, ubatch) for i in range(n_ubatch)]
    local = mr.run_local([mr.make_shard(name, cuts, s, qbits[s]) for s in range(len(cuts))], inputs)
    assert len(out['results']) == n_ubatch
    for i, (logits, want) in enumerate(zip(out['results'], local)):
        assert logits.shape == want.shape, i
        np.testing.assert_array_equal(logits, want, err_msg=f"micro-batch {i}")
    if hooked:
        assert len(out['sends']) == n_ubatch
        for i, (mbits, seconds) in enumerate(out['sends']):
            assert mbits == pytest.approx(inputs[i].numel() * inputs[i].element_size() * 8e-6, rel=1e-12), i
            assert seconds > 0, i


def test_runtime_with_a_cpu_data_rank_outside(tmp_path):
    """`runtime.py -pt 1,24,25,48 -r 1,2 -D 0` on 3 processes, rank 0 with `-d cpu`, MONITORING=1: the data rank runs
    as the host feeder, every result arrives, the data rank reports its send and output heartbeats and the first stage
    its send heartbeats, and every rank exits with 0."""
    env = dict(os.environ, PYTHONUNBUFFERED='1', PIPEEDGE_LINK_TIMEOUT_S='60', MONITORING='1')
    port = mr.free_port()
    procs = {}
    for rank in reversed(range(3)):
        argv = [sys.executable, os.path.join(mr.ROOT, 'runtime.py'), str(rank), '3', '--port', str(port),
                *mr.RUNTIME_MODEL, '-q', '0,0', '-r', '1,2', '-D', '0'] + (['-d', 'cpu'] if rank == 0 else [])
        procs[rank] = subprocess.Popen(argv, cwd=str(tmp_path), env=dict(env, LOCAL_RANK=str(rank)),
                                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    outs = {}
    for rank, p in procs.items():
        try:
            outs[rank], _ = p.communicate(timeout=600)
        except subprocess.TimeoutExpired:
            p.kill()
            outs[rank], _ = p.communicate()
    for rank, p in procs.items():
        assert p.returncode == 0, outs[rank][-3000:]
    assert 'Data rank: native (host)' in outs[0], outs[0][-3000:]
    assert 'Device: cpu' in outs[0], outs[0][-3000:]
    assert 'throughput is' in outs[0], outs[0][-3000:]
    for key in ('send', 'output'):
        assert f'{key}: Global Time' in outs[0], outs[0][-3000:]
    assert 'send: Global Time' in outs[1], outs[1][-3000:]
    for rank in (1, 2):
        assert 'Pipeline stage: native' in outs[rank], outs[rank][-3000:]
