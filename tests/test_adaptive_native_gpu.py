"""GPU: stages that switch their QuantPipe bit-width between micro-batches on the native pipeline, by picking one of the
graph variants captured per (shape, bit-width) - results bit for bit against the local shards run at the bit-widths the
records report, the C-ABI's variant selection, and `runtime.py`'s adaptive policies on the native pipeline. Ranks share
one GPU (cudaIpc between processes of the same device), like `test_pipeline_gpu.py`."""
import ctypes
import os
import socket
import sys
import threading
import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# every bit-width the adaptive policies use: raw, the fused 2 / 4 / 8 / 16-bit send and the staged 3 / 5 / 6 / 10-bit one
BITS = (0, 2, 3, 4, 5, 6, 8, 10, 16)
# the data rank's bit-width per micro-batch: every member of BITS, back-to-back changes, repeats, 0 in the middle
DATA_SCHEDULE = (0, 2, 3, 4, 5, 6, 8, 10, 16, 16, 0, 8, 8, 3, 0, 10, 2, 6, 5, 4)
# the middle rank's scripted policy: after record i it sends with MID_SCHEDULE[(i + 1) % len]
MID_SCHEDULE = (8, 16, 2, 10, 0, 0, 5, 3, 4, 6, 8, 2, 16)


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _n_items(i, n_ubatch, ubatch):
    return ubatch - 1 if i == n_ubatch - 1 else ubatch   # the last micro-batch is ragged


def _make_shard(name, cuts, rank, weights=None):
    from pipeedge_b200.models import ModuleShardConfig
    from pipeedge_b200.models.transformers import deit, vit
    from pipeedge_b200.synth import MODEL_SPECS, hf_config, synth_weights
    spec = MODEL_SPECS[name]
    classes = {'vit': vit.ViTShardForImageClassification, 'deit': deit.DeiTShardForImageClassification}
    lo = 1 if rank == 0 else cuts[rank - 1] + 1
    cfg = ModuleShardConfig(layer_start=lo, layer_end=cuts[rank], is_first=lo == 1, is_last=cuts[rank] == spec.layers)
    return classes[spec.family](hf_config(spec), cfg, weights if weights is not None else synth_weights(spec, seed=0))


def _worker(rank, world, port, name, cuts, n_ubatch, ubatch, overlap, out_q):
    import faulthandler
    faulthandler.enable()
    faulthandler.dump_traceback_later(300, exit=True)
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), PIPEEDGE_NATIVE='1',
                      PIPEEDGE_OVERLAP_SEND=str(overlap))
    os.environ.setdefault('PIPEEDGE_LINK_TIMEOUT_S', '60')
    # slots sized for exactly this micro-batch: its raw payload fills them, and every bit-width must still be accepted
    os.environ['PIPEEDGE_MAX_UBATCH'] = str(ubatch)
    torch.cuda.set_device(rank % torch.cuda.device_count())
    import runtime as rt
    from pipeedge_b200.comm.p2p import DistP2pContext, DistP2pPipelineStage
    from pipeedge_b200.synth import MODEL_SPECS, synth_input
    spec = MODEL_SPECS[name]
    shard = _make_shard(name, cuts, rank)
    first_bit = DATA_SCHEDULE[0] if rank == 0 else MID_SCHEDULE[0]
    shard.register_buffer('quant_bit', torch.tensor(first_bit if rank < world - 1 else 0), persistent=False)
    records = []

    def collect(rec):
        records.append(tuple(rec))
        if 0 < rank < world - 1:   # the middle rank's policy: the next micro-batch's bit-width from its script
            shard.quant_bit = torch.tensor(MID_SCHEDULE[(rec.index + 1) % len(MID_SCHEDULE)])

    policy = lambda *_: None   # noqa: E731  (on the thread path it would set quant_bit in the forward)
    policy._pe_native = True
    policy._pe_records = lambda _shard: collect
    if rank < world - 1:
        policy._pe_send_bits = BITS
    shard.register_forward_hook(policy)
    if rank != world - 1:
        shard.register_forward_hook(rt.forward_hook_quant_encode)
    if rank != 0:
        shard.register_forward_pre_hook(rt.forward_pre_hook_quant_decode)
    stop = threading.Event()
    results, done = [], threading.Event()

    def results_cb(t):
        results.append(t.cpu().numpy())
        if len(results) == n_ubatch:
            done.set()

    captures_after_first = {}
    with DistP2pContext(('gloo',), {'world_size': world, 'rank': rank}, lambda c, t: stop.set() if c == 0 else None) as ctx:
        src = world - 1 if rank == 0 else rank - 1
        dst = 0 if rank == world - 1 else rank + 1
        with DistP2pPipelineStage(src, dst, shard, results_cb if rank == 0 else None) as stage:
            native = stage.native
            assert native is not None, "the native pipeline was not selected"
            assert native.adaptive == (rank < world - 1) and native.send_bits == (list(BITS) if rank < world - 1 else [0])
            if rank == 0:
                for i in range(n_ubatch):
                    shard.quant_bit = torch.tensor(DATA_SCHEDULE[i % len(DATA_SCHEDULE)])
                    stage.enqueue_tensor(synth_input(spec, _n_items(i, n_ubatch, ubatch), seed=10 + i))
                    captures_after_first.setdefault(_n_items(i, n_ubatch, ubatch), native.captures)
                assert done.wait(300), "results did not arrive"
                stage.check_workers()
                ctx.cmd_broadcast(0)
            else:
                assert stop.wait(420)
                stage.check_workers()
            stats = {'captures': native.captures, 'variants': native.variants,
                     'variant_kernels': dict(native.variant_kernels), 'graph_kernels': dict(native.graph_kernels)}
    faulthandler.cancel_dump_traceback_later()
    out_q.put((rank, results, records, stats, captures_after_first))
    out_q.close()
    out_q.join_thread()


def _local_reference(name, cuts, n_ubatch, ubatch, bits):
    """The same shards + QuantPipe hooks back to back in this process, micro-batch i quantised at bits[i][rank]."""
    sys.path.insert(0, ROOT)
    import runtime as rt
    from pipeedge_b200.synth import MODEL_SPECS, synth_input, synth_weights
    spec = MODEL_SPECS[name]
    weights = synth_weights(spec, seed=0)
    world = len(cuts)
    shards = [_make_shard(name, cuts, r, weights) for r in range(world)]
    for r, shard in enumerate(shards):
        shard.register_buffer('quant_bit', torch.tensor(0), persistent=False)
        if r != world - 1:
            shard.register_forward_hook(rt.forward_hook_quant_encode)
        if r != 0:
            shard.register_forward_pre_hook(rt.forward_pre_hook_quant_decode)
    outs = []
    for i in range(n_ubatch):
        x = synth_input(spec, _n_items(i, n_ubatch, ubatch), seed=10 + i)
        for r, shard in enumerate(shards):
            shard.quant_bit = torch.tensor(bits[i][r] if r < world - 1 else 0)
            x = shard(x)
        outs.append(x.cpu().numpy())
    return outs


@pytest.mark.parametrize('overlap', [1, 0])
@pytest.mark.parametrize('name,cuts', [
    ('test/vit-tiny', (5, 12)),       # 2 ranks: (ctx, skip) tuple payload
    ('test/deit-tiny', (4, 6, 8)),    # 3 ranks: the middle rank runs a scripted policy through the record protocol
])
def test_switching_bit_widths_is_bit_identical(name, cuts, overlap):
    """The data rank changes `quant_bit` before every enqueue (every bit-width, back-to-back changes), a middle rank from
    its record consumer. Every micro-batch's logits equal the local shards run at the bit-widths the producers' records
    report; every consumer received what its producer sent; no capture after each shape's first micro-batch."""
    from pipeedge_b200.comm.p2p._native import StampRecord
    world = len(cuts)
    n_ubatch, ubatch = 22, 3
    ctx = mp.get_context('spawn')
    out_q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, name, cuts, n_ubatch, ubatch, overlap, out_q))
             for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    try:
        for _ in range(world):
            rank, results, records, stats, first = out_q.get(timeout=600)
            got[rank] = (results, [StampRecord(*r) for r in records], stats, first)
    finally:
        for p in procs:
            p.join(180)
            if p.is_alive():
                p.kill()
                p.join(10)
    for r, p in enumerate(procs):
        assert p.exitcode == 0, f"rank {r} exited with {p.exitcode}"
    for rank in range(world):
        recs = got[rank][1]
        assert [r.index for r in recs] == list(range(n_ubatch)), rank
        assert [r.items for r in recs] == [_n_items(i, n_ubatch, ubatch) for i in range(n_ubatch)]
    bits = [[got[r][1][i].bit_out for r in range(world)] for i in range(n_ubatch)]
    assert [b[0] for b in bits] == [DATA_SCHEDULE[i % len(DATA_SCHEDULE)] for i in range(n_ubatch)]
    if world > 2:
        # the middle rank's policy decides after each drained record, for the next launch: it switched variants
        assert len(set(b[1] for b in bits)) > 2 and set(b[1] for b in bits) <= set(BITS), bits
    for rank in range(1, world):
        for i in range(n_ubatch):
            assert got[rank][1][i].bit_in == got[rank - 1][1][i].bit_out, (rank, i)
    local = _local_reference(name, cuts, n_ubatch, ubatch, bits)
    for i, (logits, want) in enumerate(zip(got[0][0], local)):
        np.testing.assert_array_equal(logits, want, err_msg=f"micro-batch {i} at bit-widths {bits[i]}")
    shapes = 2   # the full and the ragged micro-batch size
    for rank in range(world):
        stats = got[rank][2]
        per_shape = len(BITS) if rank < world - 1 else 1
        assert stats['captures'] == stats['variants'] == shapes * per_shape, (rank, stats)
        assert set(stats['graph_kernels']) == {(ubatch, 0), (ubatch - 1, 0)}
    # data rank: each shape's variants were all captured at its first micro-batch
    assert got[0][3] == {ubatch: len(BITS), ubatch - 1: 2 * len(BITS)}


def _pipe_fixture(items, n):
    """A host-fed pipe whose sends go into a loop-back link it also drains its results from (raw receive, no stage
    kernels), and a capture helper."""
    from pipeedge_b200._lib import LIB, check
    nbytes = items * n * 4
    link_in, loop, pipe = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
    check(LIB.pe_link_open_host(nbytes, 4, ctypes.byref(link_in)))
    check(LIB.pe_link_open_local(nbytes + 65536, 4, 8, ctypes.byref(loop)))
    check(LIB.pe_pipe_create(link_in, loop, loop, ctypes.byref(pipe)))
    check(LIB.pe_pipe_set_out_dim(pipe, n))
    buf = torch.zeros(items * n, dtype=torch.float32, device='cuda')

    def capture(bit):
        kernels = ctypes.c_int()
        check(LIB.pe_pipe_capture_begin(pipe, items, 0, 0, buf.data_ptr(), None, 0, 0, nbytes))
        check(LIB.pe_pipe_capture_end(pipe, buf.data_ptr(), None, n, None, None, 0, items, bit, 1 if bit else 0, 0,
                                      ctypes.byref(kernels)))
        return kernels.value

    def close():
        LIB.pe_pipe_destroy(pipe)
        LIB.pe_link_close(loop)
        LIB.pe_link_close(link_in)
    return pipe, buf, capture, close


def _submit_and_drain(pipe, src, items, n):
    from pipeedge_b200._lib import LIB, check
    check(LIB.pe_pipe_submit(pipe, src.data_ptr(), src.numel() * 4, 1, items, 0))
    ptr, got_items, got_n = ctypes.c_void_p(), ctypes.c_int(), ctypes.c_size_t()
    check(LIB.pe_pipe_next_result(pipe, ctypes.byref(ptr), ctypes.byref(got_items), ctypes.byref(got_n)))
    return np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_float)), shape=(items * n,)).copy()


def test_c_abi_variant_selection():
    """Without pe_pipe_set_send_bit a capture replaces the shape's graph of another bit-width, as before, with the
    kernel counts of a pipe that only ever held that graph. With a bit-width set, captures of other bit-widths are kept
    side by side and each launches its own variant; a bit-width without a graph is reported missing and refused instead
    of launching another variant."""
    from pipeedge_b200._lib import LIB, PipeEdgeB200Error, check
    sys.path.insert(0, ROOT)
    from oracle import quant as oq
    torch.cuda.set_device(0)
    items, n = 2, 4096
    src = torch.randn(items * n, generator=torch.Generator().manual_seed(3)).pin_memory()
    want8 = oq.hook_decode(oq.hook_encode(src.view(items, n), 8)).numpy().reshape(-1)
    fresh, _, fresh_capture, fresh_close = _pipe_fixture(items, n)
    pipe, _, capture, close = _pipe_fixture(items, n)
    try:
        only8 = fresh_capture(8)
        raw = capture(0)
        assert raw > 0 and capture(8) == only8   # a second capture of the shape at another bit-width
        assert LIB.pe_pipe_has_graph(pipe, items, 0) == 1
        assert LIB.pe_pipe_has_variant(pipe, items, 0, 8) == 1
        assert LIB.pe_pipe_has_variant(pipe, items, 0, 0) == 0   # replaced, as before
        np.testing.assert_array_equal(_submit_and_drain(pipe, src, items, n), want8)   # the latest capture, as before
        check(LIB.pe_pipe_set_send_bit(pipe, 0))
        assert LIB.pe_pipe_has_graph(pipe, items, 0) == 0
        assert capture(0) == raw                                   # kept beside the 8-bit graph now
        assert LIB.pe_pipe_has_variant(pipe, items, 0, 8) == 1 and LIB.pe_pipe_has_variant(pipe, items, 0, 0) == 1
        np.testing.assert_array_equal(_submit_and_drain(pipe, src, items, n), src.numpy())
        check(LIB.pe_pipe_set_send_bit(pipe, 8))
        np.testing.assert_array_equal(_submit_and_drain(pipe, src, items, n), want8)
        check(LIB.pe_pipe_set_send_bit(pipe, 4))
        assert LIB.pe_pipe_has_graph(pipe, items, 0) == 0
        with pytest.raises(PipeEdgeB200Error, match='no graph captured'):
            check(LIB.pe_pipe_submit(pipe, src.data_ptr(), src.numel() * 4, 1, items, 0))
        check(LIB.pe_pipe_set_send_bit(pipe, -1))
        np.testing.assert_array_equal(_submit_and_drain(pipe, src, items, n), src.numpy())   # the latest: 0 bits
        assert LIB.pe_pipe_set_send_bit(pipe, 17) != 0
        check(LIB.pe_pipe_sync(pipe))
    finally:
        close()
        fresh_close()


def test_pipe_run_asks_for_the_missing_variant():
    """A stage loop (pe_pipe_run) whose bit-width has no graph for the payload's shape returns 'graph needed' and keeps
    the ticket; once the variant exists it launches it."""
    from pipeedge_b200._lib import LIB, check
    sys.path.insert(0, ROOT)
    from oracle import quant as oq
    torch.cuda.set_device(0)
    items, n = 2, 4096
    nbytes = items * n * 4
    src = torch.randn(items * n, generator=torch.Generator().manual_seed(5)).pin_memory()
    link_in, hop, back = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
    head, stage = ctypes.c_void_p(), ctypes.c_void_p()
    check(LIB.pe_link_open_host(nbytes, 4, ctypes.byref(link_in)))
    check(LIB.pe_link_open_local(nbytes + 65536, 4, 0, ctypes.byref(hop)))
    check(LIB.pe_link_open_local(nbytes + 65536, 4, 8, ctypes.byref(back)))
    check(LIB.pe_pipe_create(link_in, hop, back, ctypes.byref(head)))       # data rank: input -> hop, results <- back
    check(LIB.pe_pipe_create(hop, back, None, ctypes.byref(stage)))        # next stage: hop -> back
    buf_head = torch.zeros(items * n, dtype=torch.float32, device='cuda')
    buf_stage = torch.zeros(items * n, dtype=torch.float32, device='cuda')
    kernels = ctypes.c_int()
    need = (ctypes.c_longlong * 2)()
    try:
        check(LIB.pe_pipe_set_out_dim(stage, n))
        check(LIB.pe_pipe_capture_begin(head, items, 0, 0, buf_head.data_ptr(), None, 0, 0, nbytes))
        check(LIB.pe_pipe_capture_end(head, buf_head.data_ptr(), None, n, None, None, 0, items, 0, 0, 0, ctypes.byref(kernels)))
        check(LIB.pe_pipe_capture_begin(stage, items, 0, 0, buf_stage.data_ptr(), None, n, 0, 0))
        check(LIB.pe_pipe_capture_end(stage, buf_stage.data_ptr(), None, n, None, None, 0, items, 0, 0, 0, ctypes.byref(kernels)))
        check(LIB.pe_pipe_set_send_bit(stage, 8))
        check(LIB.pe_pipe_submit(head, src.data_ptr(), nbytes, 1, items, 0))
        rc = []
        runner = threading.Thread(target=lambda: rc.append(LIB.pe_pipe_run(stage, need)), daemon=True)
        runner.start()
        runner.join(60)
        assert rc == [2] and list(need) == [items, 0]   # no 8-bit graph: asked for one, launched nothing
        check(LIB.pe_pipe_capture_begin(stage, items, 0, 0, buf_stage.data_ptr(), None, n, 0, 0))
        check(LIB.pe_pipe_capture_end(stage, buf_stage.data_ptr(), None, n, None, None, 0, items, 8, 1, 0, ctypes.byref(kernels)))
        check(LIB.pe_pipe_close_input(head))
        runner = threading.Thread(target=lambda: rc.append(LIB.pe_pipe_run(stage, need)), daemon=True)
        runner.start()
        ptr, got_items, got_n = ctypes.c_void_p(), ctypes.c_int(), ctypes.c_size_t()
        check(LIB.pe_pipe_next_result(head, ctypes.byref(ptr), ctypes.byref(got_items), ctypes.byref(got_n)))
        got = np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_float)), shape=(items * n,)).copy()
        runner.join(60)
        assert rc == [2, 1]   # served the kept ticket with the 8-bit variant, then the close
        want8 = oq.hook_decode(oq.hook_encode(src.view(items, n), 8)).numpy().reshape(-1)
        np.testing.assert_array_equal(got, want8)
        assert LIB.pe_pipe_next_result(head, ctypes.byref(ptr), ctypes.byref(got_items), ctypes.byref(got_n)) == 1
    finally:
        LIB.pe_pipe_sync(stage)
        LIB.pe_pipe_sync(head)
        LIB.pe_pipe_destroy(stage)
        LIB.pe_pipe_destroy(head)
        for link in (back, hop, link_in):
            LIB.pe_link_close(link)


@pytest.mark.parametrize('policy,monitored', [('HEURISTIC', False), ('HEURISTIC2', False), ('CONTROLLER', False),
                                              ('CONTROLLER', True)])
def test_runtime_adaptive_quant_on_the_native_pipeline(policy, monitored, tmp_path):
    """`runtime.py` on 2 ranks sharing one GPU with an adaptive policy and a send-rate constraint no hop can meet: both
    ranks run the native pipeline, the policy moves the bit-width off 'no quantization', every result arrives."""
    import re
    import subprocess
    port = _free_port()
    env = dict(os.environ, ADAPTIVE_QUANT=policy, SEND_CONSTRAINT='1e9', WINDOW_SIZE='2', PYTHONUNBUFFERED='1',
               MONITORING='1' if monitored else '0', PIPEEDGE_LINK_TIMEOUT_S='60')
    cmd = [sys.executable, os.path.join(ROOT, 'runtime.py'), None, '2', '--port', str(port), '-m',
           'facebook/deit-tiny-distilled-patch16-224', '-b', '64', '-u', '8', '-pt', '1,24,25,48', '-q', '0,0']
    procs = []
    for rank in (1, 0):
        argv = list(cmd)
        argv[2] = str(rank)
        procs.append(subprocess.Popen(argv, cwd=str(tmp_path), env=dict(env, LOCAL_RANK=str(rank)), stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True))
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
    rank1, rank0 = outs
    assert 'throughput is' in rank0, rank0[-3000:]
    for out in (rank0, rank1):
        assert 'Pipeline stage: native' in out, out[-3000:]
    bits = [int(b) for b in re.findall(r'Adaptive quantization \(\w+\): bitwidth1?=(\d+)', rank0)]
    assert any(0 < b < 32 for b in bits), rank0[-3000:]
    if monitored:
        for key in ('shard', 'quant_encode', 'output', 'send'):
            assert f'{key}: Global Time' in rank0, rank0[-3000:]
