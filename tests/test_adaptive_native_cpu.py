"""CPU: the adaptive QuantPipe policies on the native pipeline - their record consumers against the thread-path hooks on
the same window history, the bit-width sets they declare, the record -> payload shape mapping and the native vote."""
import itertools
import os
import sys
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from pipeedge_b200 import _lib   # noqa: E402
from pipeedge_b200.comm.p2p import _native   # noqa: E402

POLICIES = ('forward_hook_set_quant_bandwidth_heuristic', 'forward_hook_set_quant_bandwidth_heuristic_2',
            'forward_hook_set_quant_controller')
SETS = {'forward_hook_set_quant_bandwidth_heuristic': 'QUANT_BITS_HEURISTIC',
        'forward_hook_set_quant_bandwidth_heuristic_2': 'QUANT_BITS_HEURISTIC2',
        'forward_hook_set_quant_controller': 'QUANT_BITS_CONTROLLER'}


class _Shard(torch.nn.Module):
    """The attributes the policies and their record consumers read; `shapes`: the payloads its graphs were captured for."""

    def __init__(self, quant_bit=0, rate=0.0, shapes=()):
        super().__init__()
        self.register_buffer('quant_bit', torch.tensor(quant_bit), persistent=False)
        self.register_buffer('rate_constraint', torch.tensor(float(rate)), persistent=False)
        self._shapes = set(shapes)

    def native_payload_shapes(self):
        return set(self._shapes)


def _payload_bytes(items, elems, bit):
    return sum(_lib.LIB.pe_link_payload_bytes(items, n, bit, 0) for n in elems)


def _record(index, items, elems, bit):
    return _native.StampRecord(index=index, items=items, bit_out=bit, bit_in=-1, bytes_out=_payload_bytes(items, elems, bit),
                               flags=0, t_start=0, t_got=0, t_stage=0, t_send_start=0, t_encoded=0, t_send_end=1000)


@pytest.fixture
def send_monitor():
    import monitoring
    import runtime
    monitoring.init(runtime.MONITORING_KEY_SEND, 4, work_type='Mbits')
    yield monitoring, runtime
    monitoring.finish()


# BERT-like micro-batches: (items, tokens) with a ragged one and a second sequence length; tuple (inter, hidden) payloads
HIDDEN, INTER = 128, 512
SCHEDULE = [(8, 32), (8, 32), (8, 48), (5, 32), (8, 32), (8, 48), (8, 48), (5, 48)] * 4


@pytest.mark.parametrize('policy', POLICIES)
@pytest.mark.parametrize('rate', [0.0, 2e4, 2e5, 2e6])
def test_record_consumer_follows_the_thread_path_hook(send_monitor, policy, rate):
    """Per micro-batch: the thread path calls the hook with the real output tensors, the native pipeline calls the
    hook's record consumer with the record of the micro-batch sent at the stage's bit-width; both see the same send
    heartbeats before them. The two stages must walk through the same `quant_bit` sequence."""
    monitoring, rt = send_monitor
    hook = getattr(rt, policy)
    shapes = {(items, (tokens * INTER, tokens * HIDDEN)) for items, tokens in SCHEDULE}
    threaded = _Shard(0, rate)
    native = _Shard(0, rate, shapes)
    consumer = hook._pe_records(native)   # pylint: disable=protected-access
    seen_threaded, seen_native = [], []
    for i, (items, tokens) in enumerate(SCHEDULE):
        outputs = (torch.zeros(items, tokens, INTER), torch.zeros(items, tokens, HIDDEN))
        hook(threaded, None, outputs)
        bit = int(native.quant_bit)   # what the graph launched for this micro-batch sends with
        consumer(_record(i, items, (tokens * INTER, tokens * HIDDEN), bit))
        seen_threaded.append(int(threaded.quant_bit))
        seen_native.append(int(native.quant_bit))
        # the micro-batch's send: its payload at the bit-width chosen for it, in a scripted time
        sent = _payload_bytes(items, (tokens * INTER, tokens * HIDDEN), seen_threaded[-1]) * 8e-6
        monitoring.iteration(rt.MONITORING_KEY_SEND, work=sent, seconds=(1 + (7 * i) % 5) * 1e-4)
    assert seen_native == seen_threaded
    if rate >= 2e5:
        assert len(set(seen_native)) > 1, seen_native   # the policy did move


def _run_policy(monitoring, rt, policy, rate, mbits_per_send, seconds, start_bit, windows=3):
    """The bit-widths a policy sets over `windows` windows of identical sends."""
    hook = getattr(rt, policy)
    shard = _Shard(start_bit, rate)
    out = torch.zeros(8, 4, 4)
    bits = []
    for _ in range(4 * windows):
        monitoring.iteration(rt.MONITORING_KEY_SEND, work=mbits_per_send, seconds=seconds)
        hook(shard, None, out)
        bits.append(int(shard.quant_bit))
    return bits


@pytest.mark.parametrize('policy', POLICIES)
def test_declared_sets_cover_every_returned_bit_width(policy):
    """Each policy's `_pe_send_bits` contains every value it set over a grid of rate constraints, bandwidths and start
    bit-widths; the sets are the ones the policies are documented to use."""
    import monitoring
    import runtime as rt
    declared = getattr(rt, policy)._pe_send_bits   # pylint: disable=protected-access
    assert declared == getattr(rt, SETS[policy])
    assert sorted(rt.QUANT_BITS_HEURISTIC) == [0, 2, 4, 6, 8, 16]
    assert sorted(rt.QUANT_BITS_HEURISTIC2) == sorted(rt.QUANT_BITS_CONTROLLER) == [0, 2, 3, 4, 5, 6, 8, 10, 16]
    seen = set()
    for rate, mbits, seconds, start in itertools.product((0.0, 1e2, 1e3, 5e3, 2e4, 1e5, 1e7),
                                                         (0.01, 1.0, 38.7, 400.0), (1e-5, 1e-3, 1e-1),
                                                         (0, 2, 4, 6, 8, 16)):
        monitoring.init(rt.MONITORING_KEY_SEND, 4, work_type='Mbits')
        try:
            seen.update(_run_policy(monitoring, rt, policy, rate, mbits, seconds, start))
        finally:
            monitoring.finish()
            rt._MODULE_QUANT_CONTROLLERS.clear()   # pylint: disable=protected-access
    assert seen <= declared, seen - declared
    assert len(seen) > 2, seen


@pytest.mark.parametrize('name', ['test/bert-tiny', 'textattack/bert-base-uncased-CoLA'])
def test_record_maps_to_a_unique_bert_payload_shape(name):
    """Payloads of several sequence lengths (and item counts, and single / tuple cuts) captured side by side: the record
    of each, at every bit-width a policy may use, maps back to exactly its own shape."""
    import runtime as rt
    from pipeedge_b200.synth import MODEL_SPECS
    spec = MODEL_SPECS[name]
    bits = sorted(rt.QUANT_BITS_HEURISTIC | rt.QUANT_BITS_CONTROLLER)
    for cut in ('single', 'ctx_skip', 'inter_data'):
        shapes = set()
        for items, seq in itertools.product((1, 3, 7, 8), (8, 9, 16, 31, 32, 48, 64)):
            per_token = {'single': (spec.hidden,), 'ctx_skip': (spec.hidden, spec.hidden),
                         'inter_data': (spec.inter, spec.hidden)}[cut]
            shapes.add((items, tuple(seq * w for w in per_token)))
        for (items, elems), bit in itertools.product(sorted(shapes), bits):
            assert _native.record_payload_elems(_record(0, items, elems, bit), shapes) == elems, (cut, items, elems, bit)
    with pytest.raises(LookupError):
        _native.record_payload_elems(_record(0, 2, (100,), 8), {(2, (64,))})


def test_a_shard_with_a_policy_hook_wins_the_native_vote(monkeypatch):
    """The policy hooks carry the protocol (`_pe_native`, `_pe_records`, `_pe_send_bits`): a native shard with one
    votes for the native pipeline; PIPEEDGE_NATIVE=0 still selects the thread path; a hook without the protocol does."""
    import runtime as rt
    from pipeedge_b200.comm.p2p import DistP2pPipelineStage
    from pipeedge_b200.models import ModuleShardConfig
    from pipeedge_b200.models.transformers._shard import GpuTransformerShard

    class FakeShard(GpuTransformerShard):
        def __init__(self):   # pylint: disable=super-init-not-called
            torch.nn.Module.__init__(self)   # pylint: disable=non-parent-init-called
            self.shard_config = ModuleShardConfig(layer_start=1, layer_end=4, is_first=True, is_last=False)

    for policy in POLICIES:
        shard = FakeShard()
        shard.register_forward_hook(getattr(rt, policy))
        shard.register_forward_hook(rt.forward_hook_quant_encode)
        assert _native.shard_is_native(shard)
        assert _native.declared_send_bits(shard) == set(getattr(rt, SETS[policy]))
        assert len(_native.record_consumers(shard)) == 1
        stage = DistP2pPipelineStage(1, 1, shard, lambda _: None)   # data rank of a two-rank ring
        monkeypatch.setattr(torch.cuda, 'is_available', lambda: True)
        monkeypatch.setenv('PIPEEDGE_NATIVE', '1')
        assert stage._native_capable()   # pylint: disable=protected-access
        monkeypatch.setenv('PIPEEDGE_NATIVE', '0')
        assert not stage._native_capable()   # pylint: disable=protected-access
        monkeypatch.undo()
    shard = FakeShard()
    shard.register_forward_hook(lambda *_: None)
    assert not _native.shard_is_native(shard)


@pytest.mark.parametrize('per_item', [(197 * 768,), (197 * 768, 197 * 768), (197 * 3072, 197 * 768), (128 * 768,)])
@pytest.mark.parametrize('items', [1, 8, 64])
def test_every_bit_width_fits_slots_sized_for_the_raw_payload(per_item, items):
    """A link's slots are sized for the largest raw payload (`native_out_bytes`): at exactly that micro-batch size every
    bit-width fits, placed as the send kernel places it; a slot a byte short of the raw payload rejects bit 0 only."""
    import runtime as rt
    raw = sum(n * 4 for n in per_item) * items
    header = _lib.PE_LINK_HEADER_BYTES
    slot = (header + raw + 8192 + 4095) // 4096 * 4096           # pe_link_open's rounding of native_out_bytes
    room = slot - header                                          # pe_link_slot_bytes
    bits = sorted(rt.QUANT_BITS_HEURISTIC | rt.QUANT_BITS_CONTROLLER)
    assert all(_native.payload_fits(room, items, per_item, bit, 0) for bit in bits)
    sizes = [items * n * 4 for n in per_item]
    tight = sum((b + 255) // 256 * 256 for b in sizes[:-1]) + sizes[-1] - 1   # the raw payload's extent, less a byte
    assert not _native.payload_fits(tight, items, per_item, 0, 0)
    assert all(_native.payload_fits(tight, items, per_item, bit, 0) for bit in bits if bit > 0)


def test_a_record_without_a_payload_shape_fails_the_stage():
    """A record consumer that cannot map a record to a captured shape (a policy would stop adapting) makes the stage's
    next check() raise; other consumer failures are only logged."""
    stage = _native.NativeStage.__new__(_native.NativeStage)
    calls = []

    def lost(rec):
        calls.append(rec.index)
        _native.record_payload_elems(rec, set())

    stage._record_cbs = [lost, lambda rec: 1 / 0]   # pylint: disable=protected-access
    stage._send_hooks, stage._rank_dst, stage._is_data = [], None, True   # pylint: disable=protected-access
    stage.adaptive, stage.exception, stage._record_error = False, None, None   # pylint: disable=protected-access
    for i in range(3):
        stage._dispatch(_record(i, 2, (64,), 8))   # pylint: disable=protected-access
    assert calls == [0, 1, 2]
    with pytest.raises(RuntimeError, match='matched no captured payload shape'):
        stage.check()
