"""CPU: the oracle restatement vs fixtures produced by executing the reference (oracle/make_goldens.py)."""
import os
import numpy as np
import pytest
import torch

from oracle import quant as oq
from oracle import shards as osh
from pipeedge_b200.synth import MODEL_SPECS, synth_weights

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')


def _load(name):
    return np.load(os.path.join(GOLDEN, f"shards_{name.replace('/', '_')}.npz"))


def _tup(g, key):
    if key in g:
        return torch.from_numpy(g[key])
    return (torch.from_numpy(g[key + '_0']), torch.from_numpy(g[key + '_1']))


@pytest.mark.parametrize('name', ['test/vit-tiny', 'test/deit-tiny', 'test/bert-tiny', 'test/vit-huge-tiny'])
def test_tiny_every_sublayer_boundary(name):
    """Oracle reproduces the reference after EVERY sub-layer, incl. the tuple payloads (A2)."""
    spec = MODEL_SPECS[name]
    g = _load(name)
    w = synth_weights(spec, seed=0)
    data = torch.from_numpy(g['input'])
    for layer in range(1, spec.layers + 1):
        data = osh.shard_forward(spec, w, layer, layer, data)
        want = _tup(g, f"after_{layer}")
        got = data if isinstance(data, tuple) else (data,)
        want = want if isinstance(want, tuple) else (want,)
        assert len(got) == len(want)
        for a, b in zip(got, want):
            torch.testing.assert_close(a, b, rtol=2e-5, atol=2e-5)
    whole = osh.shard_forward(spec, w, 1, spec.layers, torch.from_numpy(g['input']))
    torch.testing.assert_close(whole, torch.from_numpy(g['logits_whole']), rtol=2e-5, atol=2e-5)


@pytest.mark.parametrize('name', ['google/vit-base-patch16-224', 'google/vit-large-patch16-224',
                                  'facebook/deit-base-distilled-patch16-224',
                                  'textattack/bert-base-uncased-CoLA'])
def test_full_size_models(name):
    """Full-size registry models: sampled hidden states at the cuts and the logits."""
    from pipeedge_b200.synth import synth_input
    spec = MODEL_SPECS[name]
    g = _load(name)
    w = synth_weights(spec, seed=0)
    data = synth_input(spec, int(g['ubatch']), seed=1, seq_len=int(g['seq_len']))
    start = 1
    stride = int(g['stride'])
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    for cut in g['cuts'].tolist():
        data = osh.shard_forward(spec, w, start, cut, data)
        start = cut + 1
        if cut == spec.layers:
            torch.testing.assert_close(data, torch.from_numpy(g['logits']), rtol=1e-4, atol=1e-4)
        else:
            got = data.reshape(-1)[::stride]
            torch.testing.assert_close(got, torch.from_numpy(g[f"after_{cut}_sample"]), rtol=1e-4, atol=1e-4)


def test_sublayer_ranges():
    assert osh.sublayer_ranges(1, 48)[0] == (0, 0, 3) and len(osh.sublayer_ranges(1, 48)) == 12
    assert osh.sublayer_ranges(7, 12) == [(1, 2, 3), (2, 0, 3)]
    assert osh.sublayer_ranges(2, 3) == [(0, 1, 2)]
    assert osh.sublayer_ranges(4, 5) == [(0, 3, 3), (1, 0, 0)]


QG = np.load(os.path.join(GOLDEN, 'quant.npz'))


@pytest.mark.parametrize('tag', ['a', 'b', 'c'])
@pytest.mark.parametrize('bit', [2, 3, 4, 5, 6, 8, 10, 16])
def test_quant_encode_decode_bit_exact(tag, bit):
    x = torch.from_numpy(QG[f"x_{tag}"])
    enc = oq.hook_encode(x, bit)
    for nm, t in zip(('comm', 'shape', 'scale', 'shift', 'bit'), enc):
        want = QG[f"{nm}_{tag}_{bit}"]
        assert t.numpy().dtype == want.dtype, nm
        np.testing.assert_array_equal(t.numpy(), want, err_msg=nm)
    dec = oq.hook_decode(enc)
    np.testing.assert_array_equal(dec.numpy(), QG[f"dec_{tag}_{bit}"])
    alpha, kind = oq.clamp_alpha(x, bit)
    assert kind == 'laplace'
    if x.abs().max() > alpha:
        assert alpha == QG[f"alpha_{tag}_{bit}"]


@pytest.mark.parametrize('bit', [4, 8])
def test_quant_gelu_branch(bit):
    x = torch.from_numpy(QG['x_g'])
    alpha, kind = oq.clamp_alpha(x, bit)
    assert kind == 'gelu'
    enc = oq.hook_encode(x, bit)
    for nm, t in zip(('comm', 'shape', 'scale', 'shift', 'bit'), enc):
        np.testing.assert_array_equal(t.numpy(), QG[f"{nm}_g_{bit}"], err_msg=nm)
    np.testing.assert_array_equal(oq.hook_decode(enc).numpy(), QG[f"dec_g_{bit}"])


def test_quant_bit0_passthrough():
    x = torch.from_numpy(QG['x_g'])
    enc = oq.hook_encode(x, 0)
    for nm, t in zip(('comm', 'shape', 'scale', 'shift', 'bit'), enc):
        want = QG[f"{nm}_g_0"]
        assert t.numpy().dtype == want.dtype, nm
        np.testing.assert_array_equal(t.numpy(), want, err_msg=nm)
    assert oq.hook_decode(enc) is enc[0]


def test_reference_roundtrip_property():
    """The reference's own unit test (test/quant/test_quant.py:7-30), against the oracle functions."""
    for shape in ([8, 10, 10], [1, 100, 100], [8, 197, 786]):
        for bit in (1, 2, 3, 4, 5, 6, 8, 16):
            x = torch.rand(*shape).numpy()
            levels = (1 << bit) - 1
            res = np.around(levels * x)
            codes = res.astype(np.uint32)
            back = oq.unpack_codes(oq.pack_codes(codes, bit), codes.size, bit).reshape(shape)
            np.testing.assert_array_equal(back, codes)
            assert np.all((back / levels).astype(np.float32) - (res / levels) < 1e-6)


def test_gelu_clamp_threshold_of_the_reference_is_not_a_single_number():
    """`clamp_banner2019_gelu` (`clamp_op.py:16`) sums fp32 squares with torch's CPU reduction, whose order - and hence
    last bits - depends on how many threads split the tensor: the reference's own threshold for ONE input varies by a
    few ulp with `torch.get_num_threads()`. "Bit-exact codes" on that branch is therefore only defined up to this
    spread; the CUDA path (fp64 accumulation of the fp32-rounded squares) is held to 2 ulp of the oracle
    (`tests/test_quant_gpu.py::test_gelu_clamp_branch`) and must land inside the reference's own range here.
    (The Laplace branch, the one activations with negative values take, uses `torch.var` and is bit-exact.)"""
    gen = torch.Generator().manual_seed(0)
    x = torch.rand(32, 198, 768, generator=gen) + 0.2          # BASELINE config 5's hop shape, all values >= 0.2
    keep = torch.get_num_threads()
    sums = []
    try:
        for n in (1, 2, 3, 4, 8):
            torch.set_num_threads(n)
            sums.append(float(torch.pow(x, 2).sum()))
    finally:
        torch.set_num_threads(keep)
    exact = float((x.double() ** 2).sum())
    lo, hi = min(sums), max(sums)
    ulp = float(np.spacing(np.float32(exact)))
    assert hi - lo <= 8 * ulp                                    # a handful of ulp, but ...
    if (os.cpu_count() or 1) >= 4:
        assert hi > lo, "expected the fp32 sum to depend on the thread count on a multi-core host"
    # what the CUDA kernel computes: the fp64 sum of fp32-rounded squares, rounded to fp32
    ours = float(np.float32((x * x).double().sum()))
    assert lo - 2 * ulp <= ours <= hi + 2 * ulp


QB = np.load(os.path.join(GOLDEN, 'quant_bits.npz'))


@pytest.mark.parametrize('kind', ['normal', 'outliers', 'ties', 'ramp'])
@pytest.mark.parametrize('bit', [1, 7, 9, 11, 12, 13, 14, 15])
def test_quant_remaining_bit_widths_bit_exact(kind, bit):
    """The bit-widths `quant.npz` leaves out, made by the reference's `basic_op` + `clamp_op`: the oracle reproduces
    every wire byte, scale, shift and decoded value, and the clamp threshold wherever the clamp bites."""
    key = f"{kind}_{bit}"
    x = torch.from_numpy(QB[f"x_{key}"])
    enc = oq.hook_encode(x, bit)
    for nm, t in zip(('comm', 'shape', 'scale', 'shift', 'bit'), enc):
        want = QB[f"{nm}_{key}"]
        assert t.numpy().dtype == want.dtype, nm
        np.testing.assert_array_equal(t.numpy(), want, err_msg=nm)
    np.testing.assert_array_equal(oq.hook_decode(enc).numpy(), QB[f"dec_{key}"])
    alpha, kind_ = oq.clamp_alpha(x, bit)
    assert kind_ == 'laplace'
    if x.abs().max() > alpha:
        assert alpha == QB[f"alpha_{key}"]
    if kind == 'ramp':
        codes = oq.unpack_codes(enc[0][0].numpy().view(np.uint32), x.shape[1], bit)
        assert set(codes.tolist()) == set(range(1 << bit))
