"""GPU: per-micro-batch device timestamps on the native pipeline (`pe_pipe_enable_stamps`), the MONITORING=1 heartbeats
and the send-timing hook fed from them. Multi-rank pipelines share one GPU (cudaIpc between processes of the same
device), like `test_pipeline_gpu.py`."""
import ctypes
import os
import sys
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _multirank as mr  # noqa: E402
KEYS = ('shard', 'quant_encode', 'quant_decode', 'send')
# stamp kernels per micro-batch: Start, Got, Stage(+SendStart), SendEnd with the send in the main graph; a separate
# SendStart in the send graph when it overlaps; one more (Encoded) on a staged send
STAMPS_IN_GRAPH, STAMPS_OVERLAPPED, STAMPS_STAGED = 4, 5, 1
# Σ of the main graphs' timestamped durations may exceed the CUDA-event phase by at most this (the two clocks are read
# at slightly different points of the first and last graph) plus one %globaltimer step per record
SLACK_MS = 0.1


def _inputs(spec, n_ubatch, ubatch):
    from pipeedge_b200.synth import synth_input
    return [synth_input(spec, mr.ragged(i, n_ubatch, ubatch), seed=10 + i) for i in range(n_ubatch)]


def _worker(rank, world, name, cuts, qbits, n_ubatch, ubatch):
    import threading
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
        shard = mr.make_shard(name, cuts, rank, qbits[rank], hooks=(marker,) if monitored else (), monitor=True)
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
    return off, on


def _local(name, cuts, qbits, n_ubatch, ubatch):
    """The same shards + QuantPipe hooks back to back in this process; also the bytes the thread path would send per
    stage and micro-batch (its CUDA tensors: the activation, or codes + scale + shift)."""
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

    shards = [mr.make_shard(name, cuts, r, qbits[r], hooks=(sizer(r),), monitor=True) for r in range(world)]
    return mr.run_local(shards, _inputs(spec, n_ubatch, ubatch)), sent


def _run(name, cuts, qbits, n_ubatch, ubatch, overlap):
    env = {'PIPEEDGE_NATIVE': '1', 'PIPEEDGE_OVERLAP_SEND': str(overlap)}
    return mr.spawn(_worker, len(cuts), (name, cuts, qbits, n_ubatch, ubatch), env=env, hang_dump=300)


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
    src = torch.arange(items * n, dtype=torch.float32).pin_memory()
    with mr.LoopbackPipe(nbytes, nbytes) as lp:
        pipe = lp.pipe
        plain = lp.capture(items, n, 0, nbytes)
        assert LIB.pe_pipe_has_graph(pipe, items, 0) == 1
        check(LIB.pe_pipe_enable_stamps(pipe, 1))
        assert LIB.pe_pipe_has_graph(pipe, items, 0) == 0
        assert lp.capture(items, n, 0, nbytes) == plain + STAMPS_IN_GRAPH
        depth, total = _lib.PE_PIPE_STAMP_DEPTH, _lib.PE_PIPE_STAMP_DEPTH + 44
        for _ in range(total):
            out = lp.submit_and_drain(src, items, n)
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
        assert lp.capture(items, n, 0, nbytes) == plain


def test_runtime_monitoring_on_the_native_pipeline(tmp_path):
    """`runtime.py` on 2 ranks sharing one GPU with MONITORING=1 and no adaptive policy: it runs on the native pipeline
    and prints the monitored keys' global figures."""
    env = dict(os.environ, MONITORING='1', PYTHONUNBUFFERED='1', PIPEEDGE_LINK_TIMEOUT_S='60')
    env.pop('ADAPTIVE_QUANT', None)
    outs = mr.run_runtime(tmp_path, 2, ['-q', '8,0'], env)
    rank1, rank0 = outs[1], outs[0]
    assert 'throughput is' in rank0, rank0[-3000:]
    for out in (rank0, rank1):
        assert 'Pipeline stage: native' in out, out[-3000:]
    for key in ('shard', 'quant_encode', 'send', 'output'):
        assert f'{key}: Global Time' in rank0, rank0[-3000:]
    for key in ('shard', 'quant_decode', 'send'):
        assert f'{key}: Global Time' in rank1, rank1[-3000:]
