"""CPU: the native pipeline's per-micro-batch timestamp records -> the thread path's monitoring heartbeats and
send-timing hook values, on synthetic records (no GPU needed)."""
import ctypes
import os
import subprocess
import sys
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from pipeedge_b200 import _lib   # noqa: E402
from pipeedge_b200.comm.p2p import _native   # noqa: E402


def _rec(index=0, items=3, bit_out=8, bit_in=8, flags=_lib.PE_STAMP_FUSED, t0=1_000_000, got=2_000, stage=30_000,
         send=5_000, encoded=0, overlapped_gap=0, bytes_out=1234):
    """A record whose phases last `got` / `stage` / `send` ns; `encoded` > 0: a staged send whose encode took that long;
    `overlapped_gap` > 0: the send graph started that long after the main graph ended."""
    t_got = t0 + got
    t_stage = t_got + stage
    t_send_start = t_stage + overlapped_gap
    return _native.StampRecord(index=index, items=items, bit_out=bit_out, bit_in=bit_in, bytes_out=bytes_out,
                               flags=flags | (_lib.PE_STAMP_OVERLAPPED if overlapped_gap else 0), t_start=t0,
                               t_got=t_got, t_stage=t_stage, t_send_start=t_send_start,
                               t_encoded=t_send_start + encoded if encoded else 0, t_send_end=t_send_start + send)


def _beats(rec, encode=True, decode=True, layers=4):
    import runtime as rt
    return {key: (seconds, work, acc) for key, seconds, work, acc in rt.native_heartbeats(rec, layers, encode, decode)}


def test_in_graph_fused_send():
    """Send inside the main graph (t_send_start == t_stage), fused 8-bit: encode = the send kernel's duration."""
    beats = _beats(_rec())
    assert beats['shard'] == pytest.approx((30e-6, 3, 4))
    assert beats['quant_decode'] == pytest.approx((2e-6, 3, 8))   # the receive kernel, from the graph's start
    assert beats['quant_encode'] == pytest.approx((5e-6, 3, 8))   # the whole fused send kernel


def test_overlapped_send_measures_the_send_graph_only():
    """Overlapped send: the gap between the main graph's end and the send graph's start is in neither key."""
    beats = _beats(_rec(overlapped_gap=7_000))
    assert beats['shard'][0] == pytest.approx(30e-6)
    assert beats['quant_encode'][0] == pytest.approx(5e-6)
    rec = _rec(overlapped_gap=7_000)
    assert rec.send_seconds == pytest.approx(5e-6)


def test_staged_hop_reports_the_encode_kernels():
    """Staged 6-bit send: encode = send start -> the stand-alone encode kernels done; the shipping kernel is not in it."""
    rec = _rec(bit_out=6, bit_in=8, flags=_lib.PE_STAMP_STAGED, send=9_000, encoded=4_000)
    beats = _beats(rec)
    assert beats['quant_encode'] == pytest.approx((4e-6, 3, 6))
    assert beats['quant_decode'] == pytest.approx((2e-6, 3, 8))
    assert rec.send_seconds == pytest.approx(9e-6)   # the send-timing hook: the whole send


def test_ragged_last_micro_batch():
    """The ragged micro-batch's record carries its own item count (its graph was captured for that size)."""
    beats = _beats(_rec(items=2))
    assert beats['shard'][1] == 2 and beats['quant_encode'][1] == 2 and beats['quant_decode'][1] == 2


def test_bit_zero_does_no_quantisation_work():
    """bit 0 on either side: work 0, accuracy 0, no time (the thread path's hooks pass the payload through)."""
    beats = _beats(_rec(bit_out=0, bit_in=0, flags=0))
    assert beats['quant_encode'] == (0.0, 0, 0)
    assert beats['quant_decode'] == (0.0, 0, 0)
    assert beats['shard'][1] == 3


def test_keys_follow_the_registered_hooks():
    """First stage: no decode key; last stage: no encode key - as the thread path registers its hooks."""
    assert set(_beats(_rec(bit_in=-1), decode=False)) == {'shard', 'quant_encode'}
    assert set(_beats(_rec(bit_out=0), encode=False)) == {'shard', 'quant_decode'}


def test_record_consumer_gives_one_heartbeat_per_key(monkeypatch):
    """`forward_hook_monitor._pe_records` with MONITORING=1: each record -> one heartbeat of each key the shard's
    hooks cover; without MONITORING it asks for no records at all."""
    import monitoring
    import runtime as rt
    from pipeedge_b200.models import ModuleShardConfig

    class FakeShard:
        shard_config = ModuleShardConfig(layer_start=3, layer_end=6, is_first=False, is_last=False)
        _forward_hooks = {0: rt.forward_hook_monitor, 1: rt.forward_hook_quant_encode}
        _forward_pre_hooks = {0: rt.forward_pre_hook_monitor, 1: rt.forward_pre_hook_quant_decode}

    assert _native.hook_is_native(rt.forward_hook_monitor) and _native.hook_is_native(rt.forward_pre_hook_monitor)
    assert not _native.record_consumers(FakeShard())
    monitoring.init(rt.MONITORING_KEY_SEND, 4, work_type='Mbits')
    try:
        monkeypatch.setattr(rt, '_device_iters', object())
        for key in (rt.MONITORING_KEY_MODEL, rt.MONITORING_KEY_QUANT_ENCODE, rt.MONITORING_KEY_QUANT_DECODE):
            monitoring.add_key(key)
        assert _native.hook_is_native(rt.forward_hook_monitor) and _native.hook_is_native(rt.forward_pre_hook_monitor)
        consumers = _native.record_consumers(FakeShard())
        assert len(consumers) == 1
        for i in range(5):
            consumers[0](_rec(index=i, items=3 if i < 4 else 2))
        with monitoring.get_locked_context(rt.MONITORING_KEY_MODEL) as ctx:
            assert ctx.get_tag(key='shard') == 5 and ctx.get_global_work(key='shard') == 14
            assert ctx.get_global_accuracy(key='shard') == 5 * 4
            assert ctx.get_tag(key='quant_encode') == 5 and ctx.get_tag(key='quant_decode') == 5
            assert ctx.get_global_time_s(key='shard') == pytest.approx(5 * 30e-6)
            assert ctx.get_tag(key='send') == 0   # fed by the send-timing hook, not by the record consumer
    finally:
        monitoring.finish()


class _FakeRing:
    """pe_pipe_drain_stamps over a list of published record indices, with a ring of `depth` records and gaps where the
    writer lapped the reader (the same accounting as the C function)."""

    def __init__(self, depth):
        self.depth = depth
        self.written = 0
        self.next = 0

    def __call__(self, buf, max_n, n, dropped):
        n = n._obj
        dropped = dropped._obj
        oldest = max(0, self.written - self.depth)
        if self.next < oldest:
            dropped.value += oldest - self.next
            self.next = oldest
        k = 0
        while k < max_n and self.next < self.written:
            buf[k].index = self.next
            buf[k].items = 1
            k += 1
            self.next += 1
        n.value = k
        return 0


def test_drain_counts_dropped_records_and_delivers_the_rest_in_order():
    ring = _FakeRing(depth=16)
    got = []
    drain = _native.RecordDrain(ring, got.append, batch=5)
    ring.written = 12
    assert drain.poll() == 12 and drain.dropped == 0
    ring.written = 12 + 40          # the reader fell 24 records more than a whole ring behind
    assert drain.poll() == 16 and drain.dropped == 24
    assert [r.index for r in got] == list(range(12)) + list(range(36, 52))
    assert drain.records == 28
    assert drain.poll() == 0


def test_record_struct_matches_the_header():
    """`pe_pipe_record` is 8 u64 + 4 int; the Python mirror has every field of the NamedTuple."""
    assert ctypes.sizeof(_lib.PipeRecord) == 80
    names = {f[0] for f in _lib.PipeRecord._fields_}
    assert set(_native.StampRecord._fields) == names
    with open(os.path.join(ROOT, 'include', 'pipeedge_b200.h'), encoding='utf-8') as fh:
        header = fh.read()
    assert f'#define PE_PIPE_STAMP_DEPTH {_lib.PE_PIPE_STAMP_DEPTH}' in header
    for name in names:
        assert f' {name};' in header, name


def _thread_path_mbits(items, n, bit):
    """What `TensorSendThread` reports for one tensor of a payload: its CUDA tensors' bytes * 8e-6. bit 0: the f32
    activation itself; bit > 0: the codes [items, 4 * words] u8, scale and shift f32 [items] of
    `tensor_encode_outerdim` (shape and bit-width travel as CPU tensors)."""
    if bit == 0:
        cuda = [torch.empty((items, n), dtype=torch.float32)]
    else:
        words = _lib.LIB.pe_quant_words(n, bit)
        cuda = [torch.empty((items, 4 * words), dtype=torch.uint8), torch.empty(items), torch.empty(items)]
    return sum(t.numel() * t.element_size() for t in cuda) * 8e-6


@pytest.mark.parametrize('items', [1, 3, 8, 64])
@pytest.mark.parametrize('n,bit', [(197 * 192, 0), (197 * 192, 8), (197 * 192, 6), (197 * 768, 4), (50 * 1000, 2),
                                   (10, 6), (33, 16), (1000, 0), (1000, 3), (768, 12)])
def test_mbits_equal_the_thread_paths(items, n, bit):
    native = _lib.LIB.pe_link_payload_bytes(items, n, bit, 0)
    rec = _rec(items=items, bit_out=bit, bytes_out=native)
    assert rec.send_mbits == pytest.approx(_thread_path_mbits(items, n, bit), rel=1e-12)


def test_two_tensor_payload_mbits_add_up():
    """A (ctx, skip) payload: the record's bytes are the sum over its tensors, like the thread path's sum."""
    total = sum(_lib.LIB.pe_link_payload_bytes(3, n, 8, 0) for n in (197 * 192, 197 * 768))
    assert _rec(bytes_out=total).send_mbits == pytest.approx(_thread_path_mbits(3, 197 * 192, 8) +
                                                             _thread_path_mbits(3, 197 * 768, 8))
    assert _lib.LIB.pe_link_payload_bytes(3, 100, 0, 1) == 3 * 100 * 2    # fp16 wire: half the bytes actually move
    assert _lib.LIB.pe_link_payload_bytes(0, 100, 8, 0) == 0 and _lib.LIB.pe_link_payload_bytes(3, 100, 17, 0) == 0


def test_package_imports_neither_runtime_nor_monitoring():
    code = ("import sys; import pipeedge_b200.comm.p2p, pipeedge_b200.comm.p2p._native; "
            "bad = [m for m in ('runtime', 'monitoring') if m in sys.modules]; assert not bad, bad")
    subprocess.run([sys.executable, '-c', code], cwd=ROOT, check=True)
