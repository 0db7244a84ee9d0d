"""GPU: replicas of the stage pipeline fed by one data rank outside them (`runtime.py --replicas R`). The data rank holds
one feeder per replica (`NativeFeeder` with a GPU, `NativeHostFeeder` without), sends micro-batch i to replica i mod R
and hands the results on in enqueue order. Per micro-batch, the logits are bit for bit those of the same shards and
QuantPipe hooks run locally; `runtime.py --replicas 2` end to end, with and without MONITORING=1. Every rank shares one
GPU (cudaIpc between processes of the same device), like `test_data_rank_native_gpu.py`."""
import faulthandler
import os
import re
import sys
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _multirank as mr  # noqa: E402
SEQ = 32   # BERT sequence length of every micro-batch
N_UBATCH, UBATCH = 11, 3   # not a multiple of 2 or 3 replicas; the last micro-batch is one short

CASES = [
    ('test/vit-tiny', (6, 12), (0, 0), 2),      # 1 + 2x2: raw hops
    ('test/vit-tiny', (5, 12), (8, 0), 2),      # 1 + 2x2: tuple payload (ctx, skip), fused 8-bit send
    ('test/bert-tiny', (7, 12), (4, 0), 2),     # 1 + 2x2: int64 token ids in, 4-bit
    ('test/vit-tiny', (12,), (0,), 3),          # 1 + 3x1: both hops of every stage go to the data rank
]


def _input(spec, i):
    from pipeedge_b200.synth import synth_input
    return synth_input(spec, mr.ragged(i, N_UBATCH, UBATCH), seed=10 + i, seq_len=SEQ)


def _replica_ranks(cuts, replicas):
    n = len(cuts)
    return [list(range(1 + k * n, 1 + (k + 1) * n)) for k in range(replicas)]


def _worker(rank, world, name, cuts, qbits, replicas):
    import threading
    import model_cfg
    from pipeedge_b200.comm.p2p import DistP2pContext
    from pipeedge_b200.synth import MODEL_SPECS
    spec = MODEL_SPECS[name]
    ranks = _replica_ranks(cuts, replicas)
    replica, s, _, _ = model_cfg.replica_neighbours(ranks, 0, rank)
    shard = mr.make_shard(name, cuts, s, qbits[s]) if s is not None else None
    stop = threading.Event()
    results, done = [], threading.Event()

    def results_cb(t):
        results.append(t.cpu().numpy())
        if len(results) == N_UBATCH:
            done.set()

    out = {}
    with DistP2pContext(('gloo',), {'world_size': world, 'rank': rank}, lambda c, t: stop.set() if c == 0 else None) as ctx:
        with model_cfg.dist_p2p_pipeline_stage_factory(ranks, 0, rank, s, shard, results_cb) as stage:
            native = stage.native
            assert native is not None, "the native pipeline was not selected"
            if rank == 0:
                out['feeders'] = [type(f).__name__ for f in native.feeders]
                for i in range(N_UBATCH):
                    stage.enqueue_tensor(_input(spec, i))
                assert done.wait(300), "results did not arrive"
                stage.check_workers()
                ctx.cmd_broadcast(0)
            else:
                assert stop.wait(420)
                stage.check_workers()
                out['replica'], out['stage'] = replica, s
                out['shapes'] = sorted(native.graph_kernels)
    if rank == 0:
        out.update(results=results, geometry=native.input_geometry, delivered=native.delivered,
                   cuda_initialized=torch.cuda.is_initialized())
    return out


def _host_rank_main(rank, worker, world, port, args, env, out_q):
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


def _spawn_host(world, args, env):
    """As `_multirank.spawn`, with the GPUs hidden from rank 0; every process is joined."""
    ctx = torch.multiprocessing.get_context('spawn')
    out_q = ctx.Queue()
    port = mr.free_port()
    procs = [ctx.Process(target=_host_rank_main, args=(r, _worker, world, port, args, env, out_q)) for r in range(world)]
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


def _check(name, cuts, qbits, replicas, got):
    """Results in enqueue order, each bit-identical to the same shards + hooks back to back in this process; every
    replica's first stage captured the shapes of its own micro-batches only."""
    from pipeedge_b200.synth import MODEL_SPECS
    spec = MODEL_SPECS[name]
    inputs = [_input(spec, i) for i in range(N_UBATCH)]
    data = got[0]
    assert data['delivered'] == N_UBATCH
    assert len(data['results']) == N_UBATCH
    local = mr.run_local([mr.make_shard(name, cuts, s, qbits[s]) for s in range(len(cuts))], inputs)
    for i, (logits, want) in enumerate(zip(data['results'], local)):
        assert logits.shape == want.shape, i
        np.testing.assert_array_equal(logits, want, err_msg=f"micro-batch {i}")
    dim1 = SEQ if spec.family == 'bert' else 0
    for rank, out in got.items():
        if rank == 0 or out['stage'] != 0:
            continue
        mine = {(mr.ragged(i, N_UBATCH, UBATCH), dim1) for i in range(out['replica'], N_UBATCH, replicas)}
        assert set(out['shapes']) == mine, rank
    nbytes, dtype, ndim = data['geometry']
    assert (dtype, ndim) == ((torch.int64, 2) if 'bert' in name else (torch.float32, 4))


@pytest.mark.parametrize('name,cuts,qbits,replicas', CASES)
def test_replicas_are_bit_identical_to_local_shards_in_enqueue_order(name, cuts, qbits, replicas):
    world = 1 + replicas * len(cuts)
    got = mr.spawn(_worker, world, (name, cuts, qbits, replicas), env={'PIPEEDGE_NATIVE': '1'}, hang_dump=300)
    assert got[0]['feeders'] == ['NativeFeeder'] * replicas
    _check(name, cuts, qbits, replicas, got)


@pytest.mark.parametrize('name,cuts,qbits,replicas', CASES)
def test_host_data_rank_feeds_replicas_bit_identically_and_never_opens_a_context(name, cuts, qbits, replicas):
    world = 1 + replicas * len(cuts)
    got = _spawn_host(world, (name, cuts, qbits, replicas), {'PIPEEDGE_NATIVE': '1'})
    assert got[0]['feeders'] == ['NativeHostFeeder'] * replicas
    assert got[0]['cuda_initialized'] is False
    _check(name, cuts, qbits, replicas, got)


@pytest.mark.parametrize('monitor', [False, True])
def test_runtime_with_two_replicas(monitor, tmp_path):
    """`runtime.py -pt 1,24,25,48 --replicas 2` on 5 processes sharing one GPU (rank 0 the data rank, replicas on ranks
    1,2 and 3,4): every rank runs the native pipeline and names its replica and stage, every result arrives. With
    MONITORING=1 every stage rank reports its own heartbeats, and the data rank's output series counts the items of
    every micro-batch after the first, which opens the series (as on one pipeline)."""
    env = dict(os.environ, PYTHONUNBUFFERED='1', PIPEEDGE_LINK_TIMEOUT_S='60', MONITORING='1' if monitor else '0')
    outs = mr.run_runtime(tmp_path, 5, ['-q', '8,0', '--replicas', '2'], env)
    assert 'Data rank: native (replicas 2)' in outs[0], outs[0][-3000:]
    assert 'throughput is' in outs[0], outs[0][-3000:]
    for rank, (replica, stage) in {1: (0, 0), 2: (0, 1), 3: (1, 0), 4: (1, 1)}.items():
        assert f'Pipeline stage: native (replica {replica}, stage {stage})' in outs[rank], outs[rank][-3000:]
        if monitor:
            for key in ('shard', 'send'):
                assert f'{key}: Global Time' in outs[rank], outs[rank][-3000:]
    if monitor:
        assert 'send: Global Time' in outs[0], outs[0][-3000:]
        work = re.search(r'output: Global Time: .*Work: ([0-9.]+) classifications', outs[0])
        assert work is not None, outs[0][-3000:]
        assert float(work.group(1)) == 64 - 8   # -b 64 -u 8: 8 micro-batches, the first one opens the series
