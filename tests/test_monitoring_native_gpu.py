"""GPU: per-micro-batch device timestamps on the native pipeline (`pe_pipe_enable_stamps`), the MONITORING=1 heartbeats
and the send-timing hook fed from them. Multi-rank pipelines share one GPU (cudaIpc between processes of the same
device), like `test_pipeline_gpu.py`."""
import ctypes
import os
import socket
import sys
import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ('shard', 'quant_encode', 'quant_decode', 'send')
# stamp kernels per micro-batch: Start, Got, Stage(+SendStart), SendEnd with the send in the main graph; a separate
# SendStart in the send graph when it overlaps; one more (Encoded) on a staged send
STAMPS_IN_GRAPH, STAMPS_OVERLAPPED, STAMPS_STAGED = 4, 5, 1
# Σ of the main graphs' timestamped durations may exceed the CUDA-event phase by at most this (the two clocks are read
# at slightly different points of the first and last graph) plus one %globaltimer step per record
SLACK_MS = 0.1


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _shard(spec, rank, cuts, qbits, world, rt, extra_hooks=()):
    from pipeedge_b200.models import ModuleShardConfig
    from pipeedge_b200.models.transformers import deit, vit
    from pipeedge_b200.synth import hf_config, synth_weights
    classes = {'vit': vit.ViTShardForImageClassification, 'deit': deit.DeiTShardForImageClassification}
    lo = 1 if rank == 0 else cuts[rank - 1] + 1
    cfg = ModuleShardConfig(layer_start=lo, layer_end=cuts[rank], is_first=lo == 1, is_last=cuts[rank] == spec.layers)
    shard = classes[spec.family](hf_config(spec), cfg, synth_weights(spec, seed=0))
    shard.register_buffer('quant_bit', torch.tensor(qbits[rank]), persistent=False)
    for hook in extra_hooks:
        shard.register_forward_hook(hook)
    shard.register_forward_hook(rt.forward_hook_monitor)
    if rank != world - 1:
        shard.register_forward_hook(rt.forward_hook_quant_encode)
    if rank != 0:
        shard.register_forward_pre_hook(rt.forward_pre_hook_quant_decode)
    shard.register_forward_pre_hook(rt.forward_pre_hook_monitor)
    return shard


def _inputs(spec, n_ubatch, ubatch):
    from pipeedge_b200.synth import synth_input
    return [synth_input(spec, ubatch - 1 if i == n_ubatch - 1 else ubatch, seed=10 + i) for i in range(n_ubatch)]


def _worker(rank, world, port, name, cuts, qbits, n_ubatch, ubatch, overlap, out_q):
    import faulthandler
    import threading
    faulthandler.enable()
    faulthandler.dump_traceback_later(300, exit=True)
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), PIPEEDGE_NATIVE='1',
                      PIPEEDGE_OVERLAP_SEND=str(overlap))
    os.environ.setdefault('PIPEEDGE_LINK_TIMEOUT_S', '60')
    torch.cuda.set_device(rank % torch.cuda.device_count())
    import monitoring
    import runtime as rt
    from pipeedge_b200.comm.p2p import DistP2pContext, DistP2pPipelineStage
    from pipeedge_b200.synth import MODEL_SPECS
    spec = MODEL_SPECS[name]
    phase_done = [threading.Event(), threading.Event()]
    src = world - 1 if rank == 0 else rank - 1
    dst = 0 if rank == world - 1 else rank + 1

    def run(ctx, phase, monitored):
        records, calls = [], {'before': [], 'after': []}
        marker = lambda *_: None   # noqa: E731  (a no-op hook that collects the stage's records)
        marker._pe_native = True
        marker._pe_records = lambda _shard: records.append
        shard = _shard(spec, rank, cuts, qbits, world, rt, extra_hooks=(marker,) if monitored else ())
        results, done = [], threading.Event()

        def results_cb(t):
            results.append(t.cpu().numpy())
            if len(results) == n_ubatch:
                done.set()

        stage = DistP2pPipelineStage(src, dst, shard, results_cb if rank == 0 else None)
        if monitored:
            stage.register_send_timing_hook(lambda mb, s: calls['before'].append((mb, s)), ())
        stage.init()
        assert stage.native is not None, "the native pipeline was not selected"
        if monitored:
            stage.register_send_timing_hook(rt.hop_timing_hook_monitor, (rt.MONITORING_KEY_SEND,))
            stage.register_send_timing_hook(lambda mb, s: calls['after'].append((mb, s)), ())
        if rank == 0:
            for x in _inputs(spec, n_ubatch, ubatch):
                stage.enqueue_tensor(x)
            assert done.wait(300), "results did not arrive"
            ctx.cmd_broadcast(phase)
        else:
            assert phase_done[phase].wait(420)
        stage.check_workers()
        timing = stage.native.timing()
        kernels = dict(stage.native.graph_kernels)
        native = stage.native
        stage.shutdown()
        return {'results': results, 'kernels': kernels, 'timing': timing, 'records': [tuple(r) for r in records],
                'dropped': native.records_dropped, 'calls': calls}

    with DistP2pContext(('gloo',), {'world_size': world, 'rank': rank},
                        lambda c, t: phase_done[c].set() if c < 2 else None) as ctx:
        off = run(ctx, 0, False)
        monitoring.init(rt.MONITORING_KEY_SEND, 1000, work_type='Mbits')
        rt.enable_monitoring()
        on = run(ctx, 1, True)
        rt.disable_monitoring()
        with monitoring.get_locked_context(rt.MONITORING_KEY_SEND) as mctx:
            on['tags'] = {k: mctx.get_tag(key=k) for k in KEYS}
        monitoring.finish()
    faulthandler.cancel_dump_traceback_later()
    out_q.put((rank, off, on))
    out_q.close()
    out_q.join_thread()


def _local(name, cuts, qbits, n_ubatch, ubatch):
    """The same shards + QuantPipe hooks back to back in this process; also the bytes the thread path would send per
    stage and micro-batch (its CUDA tensors: the activation, or codes + scale + shift)."""
    sys.path.insert(0, ROOT)
    import runtime as rt
    from pipeedge_b200 import _lib
    from pipeedge_b200.synth import MODEL_SPECS
    spec = MODEL_SPECS[name]
    world = len(cuts)
    sent = [[] for _ in range(world)]

    def sizer(r):
        def hook(_m, _i, out):
            outs = (out,) if isinstance(out, torch.Tensor) else out
            items = outs[0].shape[0]
            sent[r].append(sum(_lib.LIB.pe_link_payload_bytes(items, t.numel() // items, qbits[r] if r < world - 1 else 0, 0)
                               for t in outs))
        return hook

    shards = [_shard(spec, r, cuts, qbits, world, rt, extra_hooks=(sizer(r),)) for r in range(world)]
    logits = []
    for x in _inputs(spec, n_ubatch, ubatch):
        for shard in shards:
            x = shard(x)
        logits.append(x.cpu().numpy())
    return logits, sent


def _run(name, cuts, qbits, n_ubatch, ubatch, overlap):
    world = len(cuts)
    ctx = mp.get_context('spawn')
    out_q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, name, cuts, qbits, n_ubatch, ubatch, overlap, out_q))
             for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    try:
        for _ in range(world):
            rank, off, on = out_q.get(timeout=600)
            got[rank] = (off, on)
    finally:
        for p in procs:
            p.join(180)
            if p.is_alive():
                p.kill()
                p.join(10)
    for r, p in enumerate(procs):
        assert p.exitcode == 0, f"rank {r} exited with {p.exitcode}"
    return got


@pytest.mark.parametrize('overlap', [1, 0])
@pytest.mark.parametrize('name,cuts,qbits', [
    ('test/vit-tiny', (5, 12), (8, 0)),          # 2 ranks: (ctx, skip) payload through the fused 8-bit send
    ('test/deit-tiny', (4, 6, 8), (8, 6, 0)),    # 3 ranks: a fused 8-bit hop, then a staged 6-bit hop
])
def test_monitoring_on_the_native_pipeline(name, cuts, qbits, overlap):
    """MONITORING=1 keeps the native pipeline, leaves its results bit-identical, and gives on every rank one record and
    one heartbeat per key per micro-batch, with ordered timestamps that fit in the rank's CUDA-event phase time."""
    from pipeedge_b200._lib import PE_STAMP_FUSED, PE_STAMP_OVERLAPPED, PE_STAMP_STAGED
    from pipeedge_b200.comm.p2p._native import StampRecord
    n_ubatch, ubatch = 12, 3
    world = len(cuts)
    got = _run(name, cuts, qbits, n_ubatch, ubatch, overlap)
    local, sent = _local(name, cuts, qbits, n_ubatch, ubatch)
    off, on = got[0]
    assert len(on['results']) == n_ubatch
    for i, (a, b, want) in enumerate(zip(off['results'], on['results'], local)):
        np.testing.assert_array_equal(b, a, err_msg=f"micro-batch {i}: monitoring changed the logits")
        np.testing.assert_array_equal(b, want, err_msg=f"micro-batch {i}: differs from the local shards")
    for rank in range(world):
        off, on = got[rank]
        bit_out = qbits[rank] if rank < world - 1 else 0
        staged = bit_out not in (0, 2, 4, 8, 16)
        recs = [StampRecord(*r) for r in on['records']]
        assert [r.index for r in recs] == list(range(n_ubatch)) and on['dropped'] == 0, rank
        want_tags = {'shard': n_ubatch, 'send': n_ubatch, 'quant_encode': n_ubatch if rank < world - 1 else 0,
                     'quant_decode': n_ubatch if rank > 0 else 0}
        assert on['tags'] == want_tags, (rank, on['tags'])
        # graphs: today's kernels without stamps, plus the stamp kernels with them
        extra = (STAMPS_OVERLAPPED if overlap else STAMPS_IN_GRAPH) + (STAMPS_STAGED if staged else 0)
        assert set(on['kernels']) == set(off['kernels'])
        # graph_kernels counts the library's launches during the capture, process-wide: on the data rank the ragged
        # graph is captured mid-stream while its results thread launches receive kernels, so only its first graph
        # (captured before any traffic) has an exact count there
        keys = list(off['kernels']) if rank > 0 else [(ubatch, 0)]
        assert all(on['kernels'][k] == off['kernels'][k] + extra for k in keys), (rank, off['kernels'], on['kernels'])
        steps = []
        for i, r in enumerate(recs):
            assert r.items == (ubatch - 1 if i == n_ubatch - 1 else ubatch)
            assert r.bit_out == bit_out and r.bit_in == (qbits[rank - 1] if rank > 0 else -1), (rank, r)
            assert r.bytes_out == sent[rank][i], (rank, i, r.bytes_out, sent[rank][i])
            assert bool(r.flags & PE_STAMP_OVERLAPPED) == bool(overlap)
            assert bool(r.flags & PE_STAMP_STAGED) == staged
            assert bool(r.flags & PE_STAMP_FUSED) == (bit_out > 0 and not staged)
            seq = [r.t_start, r.t_got, r.t_stage, r.t_send_start] + ([r.t_encoded] if staged else []) + [r.t_send_end]
            assert seq == sorted(seq), (rank, r)
            assert r.t_encoded == 0 or staged
            if not overlap:
                assert r.t_send_start == r.t_stage
            steps += [b - a for a, b in zip(seq, seq[1:]) if b > a]
        tick_ms = max(min(steps), 1000) * 1e-6   # the smallest step seen: an upper bound of the timer's granularity
        main_ms = sum(((r.t_stage if overlap else r.t_send_end) - r.t_start) * 1e-6 for r in recs)
        phase_ms = on['timing']['compute_ms']
        assert main_ms <= phase_ms + SLACK_MS + n_ubatch * tick_ms, (rank, main_ms, phase_ms)
        # the send-timing hook, registered before and after init(): once per payload, positive, the thread path's Mbit
        for when in ('before', 'after'):
            calls = on['calls'][when]
            assert len(calls) == n_ubatch, (rank, when)
            assert all(s > 0 for _, s in calls)
            assert [mb for mb, _ in calls] == pytest.approx([b * 8e-6 for b in sent[rank]], rel=1e-12)
        print(f"rank {rank}: {n_ubatch} records, main graphs {main_ms:.3f} ms of a {phase_ms:.3f} ms phase, "
              f"kernels {off['kernels']} -> {on['kernels']}")


def test_stamp_ring_recapture_and_dropped_records():
    """One pipe driven through the C-ABI (host-fed input -> raw receive -> send into a loop-back link): turning stamps on
    makes the graph captured without them count as missing; the new graph has 4 more kernels; a reader that lets the
    ring wrap gets the newest PE_PIPE_STAMP_DEPTH records in order and the count of the others."""
    from pipeedge_b200 import _lib
    from pipeedge_b200._lib import LIB, check
    torch.cuda.set_device(0)
    items, n = 2, 256
    nbytes = items * n * 4
    link_in, loop, pipe = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
    check(LIB.pe_link_open_host(nbytes, 4, ctypes.byref(link_in)))
    check(LIB.pe_link_open_local(nbytes, 4, 0, ctypes.byref(loop)))
    check(LIB.pe_pipe_create(link_in, loop, loop, ctypes.byref(pipe)))
    buf = torch.zeros(items * n, dtype=torch.float32, device='cuda')
    src = torch.arange(items * n, dtype=torch.float32).pin_memory()
    try:
        check(LIB.pe_pipe_set_out_dim(pipe, n))

        def capture():
            kernels = ctypes.c_int()
            check(LIB.pe_pipe_capture_begin(pipe, items, 0, 0, buf.data_ptr(), None, 0, 0, nbytes))
            check(LIB.pe_pipe_capture_end(pipe, buf.data_ptr(), None, n, None, None, 0, items, 0, 0, 0,
                                          ctypes.byref(kernels)))
            return kernels.value

        plain = capture()
        assert LIB.pe_pipe_has_graph(pipe, items, 0) == 1
        check(LIB.pe_pipe_enable_stamps(pipe, 1))
        assert LIB.pe_pipe_has_graph(pipe, items, 0) == 0
        assert capture() == plain + STAMPS_IN_GRAPH
        depth, total = _lib.PE_PIPE_STAMP_DEPTH, _lib.PE_PIPE_STAMP_DEPTH + 44
        ptr, got_items, got_n = ctypes.c_void_p(), ctypes.c_int(), ctypes.c_size_t()
        for _ in range(total):
            check(LIB.pe_pipe_submit(pipe, src.data_ptr(), nbytes, 1, items, 0))
            check(LIB.pe_pipe_next_result(pipe, ctypes.byref(ptr), ctypes.byref(got_items), ctypes.byref(got_n)))
            out = np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_float)), shape=(items * n,))
            assert np.array_equal(out, src.numpy())
        check(LIB.pe_pipe_sync(pipe))
        recs = (_lib.PipeRecord * (2 * depth))()
        count, dropped = ctypes.c_int(), ctypes.c_ulonglong()
        check(LIB.pe_pipe_drain_stamps(pipe, recs, len(recs), ctypes.byref(count), ctypes.byref(dropped)))
        assert dropped.value == total - depth and count.value == depth
        assert [recs[i].index for i in range(depth)] == list(range(total - depth, total))
        for i in range(depth):
            r = recs[i]
            assert r.items == items and r.bit_out == 0 and r.bit_in == -1 and r.bytes_out == nbytes and r.flags == 0
            assert r.t_start <= r.t_got <= r.t_stage == r.t_send_start <= r.t_send_end and r.t_encoded == 0
        check(LIB.pe_pipe_drain_stamps(pipe, recs, len(recs), ctypes.byref(count), ctypes.byref(dropped)))
        assert count.value == 0 and dropped.value == total - depth
        # stamps off again: the stamped graph counts as missing, and the plain capture is what it was
        check(LIB.pe_pipe_enable_stamps(pipe, 0))
        assert LIB.pe_pipe_has_graph(pipe, items, 0) == 0
        assert capture() == plain
    finally:
        LIB.pe_pipe_destroy(pipe)
        LIB.pe_link_close(loop)
        LIB.pe_link_close(link_in)


def test_runtime_monitoring_on_the_native_pipeline(tmp_path):
    """`runtime.py` on 2 ranks sharing one GPU with MONITORING=1 and no adaptive policy: it runs on the native pipeline
    and prints the monitored keys' global figures."""
    import subprocess
    port = _free_port()
    env = dict(os.environ, MONITORING='1', PYTHONUNBUFFERED='1', PIPEEDGE_LINK_TIMEOUT_S='60')
    env.pop('ADAPTIVE_QUANT', None)
    cmd = [sys.executable, os.path.join(ROOT, 'runtime.py'), None, '2', '--port', str(port), '-m',
           'facebook/deit-tiny-distilled-patch16-224', '-b', '64', '-u', '8', '-pt', '1,24,25,48', '-q', '8,0']
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
    for key in ('shard', 'quant_encode', 'send', 'output'):
        assert f'{key}: Global Time' in rank0, rank0[-3000:]
    for key in ('shard', 'quant_decode', 'send'):
        assert f'{key}: Global Time' in rank1, rank1[-3000:]
