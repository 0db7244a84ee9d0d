"""GPU: the native pipeline with the data rank outside the stage pipeline (`runtime.py -D 0 -r 1,...`). The data rank
is a feeder without a shard: one relay kernel per micro-batch moves its input, bytes unchanged, into the first stage's
ring; the first stage receives it as a raw payload from a peer link. Results bit for bit against the same shards and
QuantPipe hooks run locally, the inputs the feeder takes, the kernel counts of both ends, the send-timing hook on the
feeder and `runtime.py` with this topology. Ranks share one GPU (cudaIpc between processes of the same device), like
`test_pipeline_gpu.py`."""
import os
import socket
import subprocess
import sys
import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEQ = 32   # BERT sequence length of every micro-batch


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _n_items(i, n_ubatch, ubatch):
    return ubatch - 1 if i == n_ubatch - 1 else ubatch   # the last micro-batch is ragged


def _make_shard(name, cuts, qbits, s, weights=None):
    """Stage `s` of the pipeline cut after `cuts`, with the QuantPipe hooks `runtime.py` gives it."""
    sys.path.insert(0, ROOT)
    import runtime as rt
    from pipeedge_b200.models import ModuleShardConfig
    from pipeedge_b200.models.transformers import bert, deit, vit
    from pipeedge_b200.synth import MODEL_SPECS, hf_config, synth_weights
    spec = MODEL_SPECS[name]
    classes = {'vit': vit.ViTShardForImageClassification, 'deit': deit.DeiTShardForImageClassification,
               'bert': bert.BertShardForSequenceClassification}
    lo = 1 if s == 0 else cuts[s - 1] + 1
    cfg = ModuleShardConfig(layer_start=lo, layer_end=cuts[s], is_first=lo == 1, is_last=cuts[s] == spec.layers)
    shard = classes[spec.family](hf_config(spec), cfg, weights if weights is not None else synth_weights(spec, seed=0))
    shard.register_buffer('quant_bit', torch.tensor(qbits[s]), persistent=False)
    if s != len(cuts) - 1:
        shard.register_forward_hook(rt.forward_hook_quant_encode)
    if s != 0:
        shard.register_forward_pre_hook(rt.forward_pre_hook_quant_decode)
    return shard


def _input(spec, i, n_ubatch, ubatch, mixed):
    """Micro-batch i. `mixed`: a host tensor, a device tensor, or a host tensor of a dtype the feeder converts (float64
    images / int32 token ids, both converted exactly), in turn."""
    from pipeedge_b200.synth import synth_input
    x = synth_input(spec, _n_items(i, n_ubatch, ubatch), seed=10 + i, seq_len=SEQ)
    if mixed and i % 3 == 1:
        return x.cuda()
    if mixed and i % 3 == 2:
        return x.double() if x.is_floating_point() else x.int()
    return x


def _inside_kernels(name, cuts, qbits, ubatch, dim1):
    """graph_kernels of the first stage when the data rank owns it (a world of one: host-fed input, loop-back output),
    for the full and the ragged micro-batch."""
    from pipeedge_b200.comm.p2p._native import NativeStage
    stage = NativeStage(None, None, _make_shard(name, cuts, qbits, 0), lambda _t: None)
    stage.init(None, None)
    try:
        stage.prepare(ubatch, dim1)
        stage.prepare(ubatch - 1, dim1)
        return dict(stage.graph_kernels)
    finally:
        stage.shutdown()


def _worker(rank, world, port, name, cuts, qbits, n_ubatch, ubatch, mixed, hooked, out_q):
    import faulthandler
    import threading
    faulthandler.enable()   # a native crash prints every thread's Python stack into the test log
    faulthandler.dump_traceback_later(300, exit=True)   # a hung rank shows where, and ends
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), PIPEEDGE_NATIVE='1')
    os.environ.setdefault('PIPEEDGE_LINK_TIMEOUT_S', '60')   # ranks sharing one GPU are time-sliced
    if mixed:
        os.environ['PIPEEDGE_LINK_SLOTS'] = '2'   # the feeder outruns the first stage sooner: back-pressure
    torch.cuda.set_device(rank % torch.cuda.device_count())
    import model_cfg
    from pipeedge_b200.comm.p2p import DistP2pContext
    from pipeedge_b200.synth import MODEL_SPECS
    spec = MODEL_SPECS[name]
    stage_ranks = list(range(1, world))
    s = rank - 1 if rank > 0 else None
    shard = _make_shard(name, cuts, qbits, s) if s is not None else None
    stop = threading.Event()
    results, done, sends = [], threading.Event(), []

    def results_cb(t):
        results.append(t.cpu().numpy())
        if len(results) == n_ubatch:
            done.set()

    out = {}
    with DistP2pContext(('gloo',), {'world_size': world, 'rank': rank}, lambda c, t: stop.set() if c == 0 else None) as ctx:
        with model_cfg.dist_p2p_pipeline_stage_factory(stage_ranks, 0, rank, s, shard, results_cb) as stage:
            native = stage.native
            assert native is not None, "the native pipeline was not selected"
            if rank == 0:
                assert type(native).__name__ == 'NativeFeeder'
                if hooked:
                    stage.register_send_timing_hook(lambda mbits, sec: sends.append((mbits, sec)), ())
                for i in range(n_ubatch):
                    stage.enqueue_tensor(_input(spec, i, n_ubatch, ubatch, mixed))
                assert done.wait(300), "results did not arrive"
                stage.check_workers()
                ctx.cmd_broadcast(0)
            else:
                assert stop.wait(420)
                stage.check_workers()
        out['graph_kernels'] = dict(native.graph_kernels)
    if rank == 0:
        out.update(results=results, sends=sends, geometry=native.input_geometry)
    if rank == 1:
        out['inside_kernels'] = _inside_kernels(name, cuts, qbits, ubatch, SEQ if spec.family == 'bert' else 0)
    faulthandler.cancel_dump_traceback_later()
    out_q.put((rank, out))
    out_q.close()
    out_q.join_thread()


def _run(name, cuts, qbits, n_ubatch, ubatch, mixed=False, hooked=False):
    world = len(cuts) + 1
    ctx = mp.get_context('spawn')
    out_q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, name, cuts, qbits, n_ubatch, ubatch, mixed, hooked,
                                               out_q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    try:
        for _ in range(world):
            rank, out = out_q.get(timeout=600)
            got[rank] = out
    finally:
        for p in procs:
            p.join(180)
            if p.is_alive():
                p.kill()
                p.join(10)
    for r, p in enumerate(procs):
        assert p.exitcode == 0, f"rank {r} exited with {p.exitcode}"
    return got


def _local_reference(name, cuts, qbits, n_ubatch, ubatch):
    """The same shards + QuantPipe hooks back to back in this process."""
    from pipeedge_b200.synth import MODEL_SPECS, synth_weights
    spec = MODEL_SPECS[name]
    weights = synth_weights(spec, seed=0)
    shards = [_make_shard(name, cuts, qbits, s, weights) for s in range(len(cuts))]
    outs = []
    for i in range(n_ubatch):
        x = _input(spec, i, n_ubatch, ubatch, False)
        for shard in shards:
            x = shard(x)
        outs.append(x.cpu().numpy())
    return outs


def _check(name, cuts, qbits, n_ubatch, ubatch, got):
    from pipeedge_b200.synth import MODEL_SPECS, synth_weights
    results = got[0]['results']
    assert len(results) == n_ubatch
    for i, (logits, want) in enumerate(zip(results, _local_reference(name, cuts, qbits, n_ubatch, ubatch))):
        assert logits.shape == want.shape, i
        np.testing.assert_array_equal(logits, want, err_msg=f"micro-batch {i}")
    if not any(qbits):
        sys.path.insert(0, ROOT)
        from oracle import shards as osh
        spec = MODEL_SPECS[name]
        w = synth_weights(spec, seed=0)
        for i, logits in enumerate(results):
            want = osh.shard_forward(spec, w, 1, spec.layers, _input(spec, i, n_ubatch, ubatch, False)).numpy()
            assert np.abs(logits - want).max() <= 4e-3 * np.abs(want).max(), f"micro-batch {i}"


def _shapes(name, ubatch):
    from pipeedge_b200.synth import MODEL_SPECS
    dim1 = SEQ if MODEL_SPECS[name].family == 'bert' else 0
    return {(ubatch, dim1), (ubatch - 1, dim1)}


@pytest.mark.parametrize('name,cuts,qbits', [
    ('test/vit-tiny', (6, 12), (0, 0)),            # mid-block cut after an output projection
    ('test/vit-tiny', (5, 12), (8, 0)),            # tuple payload (ctx, skip), fused 8-bit send
    ('test/bert-tiny', (7, 12), (4, 0)),           # int64 token ids in, tuple payload out, 4-bit
    ('test/deit-tiny', (4, 6, 8), (8, 6, 0)),      # three stages: fused 8-bit and staged 6-bit hops
    ('test/vit-tiny', (12,), (0,)),                # one stage: both of its hops go to the data rank
])
def test_outside_data_rank_is_bit_identical_to_local_shards(name, cuts, qbits):
    """18 micro-batches through 4-slot rings, the last one ragged: results in FIFO order, bit-identical to the local
    shards and hooks (and within the oracle's bound for raw hops). The first stage's graphs have the kernels of the
    same stage owned by the data rank; the feeder's relay graph is one kernel."""
    n_ubatch, ubatch = 18, 3
    got = _run(name, cuts, qbits, n_ubatch, ubatch)
    _check(name, cuts, qbits, n_ubatch, ubatch, got)
    assert got[0]['graph_kernels'] == {shape: 1 for shape in _shapes(name, ubatch)}
    assert set(got[1]['graph_kernels']) == _shapes(name, ubatch)
    assert got[1]['graph_kernels'] == got[1]['inside_kernels']
    nbytes, dtype, ndim = got[0]['geometry']
    assert (dtype, ndim) == ((torch.int64, 2) if 'bert' in name else (torch.float32, 4))


@pytest.mark.parametrize('name,cuts,qbits', [
    ('test/vit-tiny', (6, 12), (8, 0)),
    ('test/bert-tiny', (7, 12), (0, 0)),
])
def test_feeder_inputs_back_pressure_and_send_timing(name, cuts, qbits):
    """Host, device and converted-dtype inputs in turn through 2-slot rings, enqueued as fast as the feeder takes them:
    nothing is dropped or reordered. A send-timing hook on the feeder is called once per micro-batch with the input's
    Mbit (bytes * 8e-6, as the thread path reports a raw tensor) and a positive device time; its relay graph then
    carries two stamp kernels."""
    from pipeedge_b200.synth import MODEL_SPECS
    n_ubatch, ubatch = 18, 3
    got = _run(name, cuts, qbits, n_ubatch, ubatch, mixed=True, hooked=True)
    _check(name, cuts, qbits, n_ubatch, ubatch, got)
    spec = MODEL_SPECS[name]
    sends = got[0]['sends']
    assert len(sends) == n_ubatch
    for i, (mbits, seconds) in enumerate(sends):
        x = _input(spec, i, n_ubatch, ubatch, False)
        assert mbits == pytest.approx(x.numel() * x.element_size() * 8e-6, rel=1e-12), i
        assert seconds > 0, i
    assert got[0]['graph_kernels'] == {shape: 3 for shape in _shapes(name, ubatch)}


def test_relay_capture_refuses_oversized_inputs_before_launching():
    """The host refuses a relay of more bytes than the rings' slots hold, and a pipe whose input is not host-fed."""
    import ctypes
    from pipeedge_b200._lib import LIB, PipeEdgeB200Error, check
    torch.cuda.set_device(0)
    link_in, loop, pipe, other = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
    kernels = ctypes.c_int()
    check(LIB.pe_link_open_host(4096, 2, ctypes.byref(link_in)))
    check(LIB.pe_link_open_local(4096, 2, 0, ctypes.byref(loop)))
    try:
        check(LIB.pe_pipe_create(link_in, loop, loop, ctypes.byref(pipe)))
        room = LIB.pe_link_slot_bytes(link_in)
        with pytest.raises(PipeEdgeB200Error, match='exceed'):
            check(LIB.pe_pipe_capture_relay(pipe, 1, 0, room + 1, ctypes.byref(kernels)))
        assert LIB.pe_pipe_has_graph(pipe, 1, 0) == 0
        check(LIB.pe_pipe_create(loop, loop, None, ctypes.byref(other)))
        with pytest.raises(PipeEdgeB200Error, match='not host-fed'):
            check(LIB.pe_pipe_capture_relay(other, 1, 0, 64, ctypes.byref(kernels)))
    finally:
        LIB.pe_pipe_destroy(other)
        LIB.pe_pipe_destroy(pipe)
        LIB.pe_link_close(loop)
        LIB.pe_link_close(link_in)


def test_relay_moves_the_bytes_unchanged_through_a_loop_back_link():
    """The relay graph and a first stage's raw receive in one process: a host-fed ring relayed into a loop-back link and
    received from it with its header checked - fp32 and int64 payloads of several sizes (not all multiples of 16 bytes),
    more payloads than slots."""
    import ctypes
    from pipeedge_b200._lib import LIB, check
    torch.cuda.set_device(0)
    link_in, loop, pipe = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
    check(LIB.pe_link_open_host(1 << 20, 2, ctypes.byref(link_in)))
    check(LIB.pe_link_open_local(1 << 20, 2, 0, ctypes.byref(loop)))
    kernels = ctypes.c_int()
    try:
        check(LIB.pe_pipe_create(link_in, loop, None, ctypes.byref(pipe)))
        gen = torch.Generator().manual_seed(7)
        srcs = [torch.randn(3, 3, 64, 64, generator=gen), torch.randint(-2**62, 2**62, (5, 32), generator=gen),
                torch.randn(1, 37, generator=gen), torch.randn(3, 3, 64, 64, generator=gen)]
        for src in srcs:
            items, nbytes = src.shape[0], src.numel() * src.element_size()
            if not LIB.pe_pipe_has_graph(pipe, items, nbytes):
                check(LIB.pe_pipe_capture_relay(pipe, items, nbytes, nbytes, ctypes.byref(kernels)))
                assert kernels.value == 1
            src = src.pin_memory()
            check(LIB.pe_pipe_submit(pipe, src.data_ptr(), nbytes, 1, items, nbytes))
            check(LIB.pe_pipe_sync(pipe))
            buf = torch.empty(max(nbytes, 64), dtype=torch.uint8, device='cuda')
            _raw_receive(loop, buf, nbytes, items)
            assert torch.equal(buf[:nbytes].cpu(), src.view(-1).view(torch.uint8))
        check(LIB.pe_pipe_sync(pipe))
        assert LIB.pe_link_check(loop) == 0
    finally:
        LIB.pe_pipe_destroy(pipe)
        LIB.pe_link_close(loop)
        LIB.pe_link_close(link_in)


def _raw_receive(link, buf, nbytes, items):
    """What a first stage fed by a relay starts its graph with (pe_pipe_capture_begin with raw_bytes: the raw receive,
    its header checked against the bytes and items), run once through a stage loop that reads the relay's ticket."""
    import ctypes
    from pipeedge_b200._lib import LIB, check
    # a consumer pipe on the loop-back link: the raw receive, no stage kernels, a 16-value send into a sink
    sink_in, sink = ctypes.c_void_p(), ctypes.c_void_p()
    check(LIB.pe_link_open_local(4096, 2, 0, ctypes.byref(sink_in)))
    try:
        check(LIB.pe_pipe_create(link, sink_in, None, ctypes.byref(sink)))
        kernels = ctypes.c_int()
        check(LIB.pe_pipe_capture_begin(sink, items, 0, 0, buf.data_ptr(), None, 0, 0, nbytes))
        check(LIB.pe_pipe_capture_end(sink, buf.data_ptr(), None, 16, None, None, 0, 1, 0, 0, 0, ctypes.byref(kernels)))
        need = (ctypes.c_longlong * 2)()
        ticket = (ctypes.c_longlong * 2)()
        check(LIB.pe_link_ticket_recv(link, ticket))   # the relay's ticket (items, dim1)
        assert ticket[0] == items
        check(LIB.pe_link_ticket_send(link, items, 0))   # hand it to the stage loop under the key it was captured for
        check(LIB.pe_link_ticket_send(link, -1, 0))
        assert LIB.pe_pipe_run(sink, need) == 1
        check(LIB.pe_pipe_sync(sink))
    finally:
        LIB.pe_pipe_destroy(sink)
        LIB.pe_link_close(sink_in)


@pytest.mark.parametrize('env,expect', [
    ({}, 'throughput'),
    ({'MONITORING': '1'}, 'heartbeats'),
    ({'ADAPTIVE_QUANT': 'CONTROLLER', 'SEND_CONSTRAINT': '1e9', 'WINDOW_SIZE': '2'}, 'policy'),
])
def test_runtime_with_the_data_rank_outside(env, expect, tmp_path):
    """`runtime.py -pt 1,24,25,48 -r 1,2 -D 0` on 3 processes sharing one GPU: every rank runs the native pipeline
    (rank 0 as the feeder), every result arrives; with MONITORING=1 the data rank reports its send and output
    heartbeats; with a send-rate constraint no hop can meet, the controller on the first stage's rank moves the
    bit-width off 'no quantization'."""
    import re
    port = _free_port()
    base = dict(os.environ, PYTHONUNBUFFERED='1', PIPEEDGE_LINK_TIMEOUT_S='60', MONITORING='0')
    base.update(env)
    cmd = [sys.executable, os.path.join(ROOT, 'runtime.py'), None, '3', '--port', str(port), '-m',
           'facebook/deit-tiny-distilled-patch16-224', '-b', '64', '-u', '8', '-pt', '1,24,25,48', '-q', '0,0',
           '-r', '1,2', '-D', '0']
    procs = []
    for rank in (2, 1, 0):
        argv = list(cmd)
        argv[2] = str(rank)
        procs.append(subprocess.Popen(argv, cwd=str(tmp_path), env=dict(base, LOCAL_RANK=str(rank)),
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    for p in procs:
        try:
            out, _ = p.communicate(timeout=600)
        except subprocess.TimeoutExpired:
            p.kill()
            out, _ = p.communicate()
        outs.append(out)
    for p, out in zip(procs, outs):
        assert p.returncode == 0, out[-3000:]
    rank2, rank1, rank0 = outs
    assert 'Data rank: native' in rank0, rank0[-3000:]
    assert 'throughput is' in rank0, rank0[-3000:]
    for out in (rank1, rank2):
        assert 'Pipeline stage: native' in out, out[-3000:]
    if expect == 'heartbeats':
        for key in ('send', 'output'):
            assert f'{key}: Global Time' in rank0, rank0[-3000:]
    if expect == 'policy':
        bits = [int(b) for b in re.findall(r'Adaptive quantization \(controller\): bitwidth1=(\d+)', rank1)]
        assert any(0 < b < 32 for b in bits), rank1[-3000:]
