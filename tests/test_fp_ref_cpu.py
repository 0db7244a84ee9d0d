"""CPU: the conformance checkers of `_fp_ref.py` reject plausible wrong kernels (emulated here in fp64 / fp32 torch) and
accept a correct one, and the GEMM case list reaches every path it claims (host-only tile planner)."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _fp_ref as R  # noqa: E402


# ----------------------------------------------------------------------------------------------- fp16 helpers
def test_f16_rounding_helpers_match_numpy():
    import numpy as np
    gen = torch.Generator().manual_seed(0)
    x = torch.cat([torch.randn(20000, generator=gen, dtype=torch.float64) * 10.0 ** torch.randint(-9, 5, (20000,), generator=gen),
                   torch.tensor([0.0, -0.0, 65504.0, 65519.99, 65520.0, 1e6, -1e6, 2.0 ** -25, 3 * 2.0 ** -25, 2.0 ** -26],
                                dtype=torch.float64)])
    with np.errstate(over='ignore'):   # numpy rounds double -> half directly
        want = torch.from_numpy(x.numpy().astype(np.float16).astype(np.float64))
    assert torch.equal(R.f16_nearest(x), want)
    lo, hi = R.f16_down(x), R.f16_up(x)
    assert bool(((lo <= x) & (x <= hi)).all())
    assert bool(((lo == x) == (hi == x)).all())
    assert bool((R._step16(lo.half(), up=True).double() >= hi).all())


# ------------------------------------------------------------------------------------------------- GEMM checks
def _small_gemm(m=64, n=48, k=72, seed=1):
    gen = torch.Generator().manual_seed(seed)
    a = torch.randn(m, k, generator=gen).half()
    w = (torch.randn(n, k, generator=gen) * 0.3).half()
    bias = torch.randn(n, generator=gen)
    resid = torch.randn(m, n, generator=gen)
    acc32 = a.float() @ w.float().t()            # an honest fp32 accumulation
    return a, w, bias, resid, acc32


def _fp32_gelu_like_kernel(x32):
    """x Phi(x) evaluated in fp64 and rounded to fp32: what an accurate fp32 epilogue produces."""
    return R.gelu64(x32.double()).float()


def test_gemm_checker_accepts_correct_epilogues():
    a, w, bias, resid, acc = _small_gemm()
    x = acc + bias
    assert R.check_gemm('F32', x, a, w, bias).passed
    assert R.check_gemm('RESID_F32', x + resid, a, w, bias, resid).passed
    assert R.check_gemm('TANH_F32', torch.tanh(x.double()).float(), a, w, bias).passed
    assert R.check_gemm('F16', x.half(), a, w, bias).passed
    assert R.check_gemm('GELU_F16', _fp32_gelu_like_kernel(x).half(), a, w, bias).passed
    assert R.check_gemm('F16', acc.half(), a, w, None).passed


def test_gemm_checker_rejects_tanh_form_gelu():
    a, w, bias, _, acc = _small_gemm()
    wrong = R.gelu_tanh64((acc + bias).double()).half()
    assert not R.check_gemm('GELU_F16', wrong, a, w, bias).passed
    h, b = R.scan_inputs()
    x = R.scan_preact(h, b)
    assert R.check_gelu_scan(R.f16_nearest(R.gelu64(x)).half(), x).passed
    assert not R.check_gelu_scan(R.gelu_tanh64(x).half(), x).passed


def test_gemm_checker_rejects_double_rounding():
    """GELU applied to an fp16-rounded pre-activation, then rounded again."""
    a, w, bias, _, acc = _small_gemm()
    wrong = R.gelu64((acc + bias).half().double()).half()
    assert not R.check_gemm('GELU_F16', wrong, a, w, bias).passed


def test_gemm_checker_rejects_bias_after_rounding():
    a, w, bias, _, acc = _small_gemm()
    wrong = (acc.half().float() + bias).half()
    assert not R.check_gemm('F16', wrong, a, w, bias).passed
    assert not R.check_gemm('F32', acc.half().float() + bias, a, w, bias).passed


def test_gemm_checker_rejects_missing_bias_or_residual_and_bad_tanh():
    a, w, bias, resid, acc = _small_gemm()
    assert not R.check_gemm('F16', acc.half(), a, w, bias).passed
    assert not R.check_gemm('RESID_F32', acc + bias, a, w, bias, resid).passed
    h, b = R.scan_inputs(-3, 3)
    xs = R.scan_preact(h, b)
    assert R.check_tanh_scan(torch.tanh(xs).float(), xs).passed
    assert not R.check_tanh_scan((torch.tanh(xs) + 4 * R.ulp32(torch.tanh(xs))).float(), xs).passed


def test_gelu_scan_covers_the_edges():
    h, b = R.scan_inputs()
    x = R.scan_preact(h, b)
    assert float(x.min()) <= -12.0 and float(x.max()) >= 12.0
    assert bool(((x.abs() > 5.9) & (x.abs() < 6.0)).any()) and bool(((x.abs() > 6.0) & (x.abs() < 6.1)).any())
    g = R.gelu64(x)
    sub = (g < 0) & (g.abs() < 2.0 ** -14) & (g.abs() > 2.0 ** -25)     # negative GELU in fp16's subnormal range
    assert int(sub.sum()) > 1000
    tiny = x[(x != 0) & (x.abs() < 1e-20)]
    assert bool((tiny > 0).any()) and bool((tiny < 0).any()) and bool((tiny.abs() < 1.2e-38).any())


LONG_K_STAGES = 4     # ring depth of the stale-stage kernel: BN 160 / 224 plans run 4 stages


def _kblock_gemm(a, w, bias, mutate=None, j=None):
    """fp32 emulation of the wgmma main loop: k-blocks of 64 summed in fp32, in order, onto an fp32 accumulator, then
    + bias. `mutate` plants one wrong k-block `j`: 'drop' (never added), 'twice' (added twice), 'stale' (the operands
    of block j - LONG_K_STAGES, what a ring slot still holds when its refill was not waited for), 'f16' (the block's
    64 products summed in fp16)."""
    kb = a.shape[1] // 64
    acc = torch.zeros(a.shape[0], w.shape[0])
    for b in range(kb):
        src = b - LONG_K_STAGES if (mutate == 'stale' and b == j) else b
        sl = slice(64 * src, 64 * src + 64)
        if mutate == 'f16' and b == j:
            part = torch.zeros_like(acc).half()
            for i in range(sl.start, sl.stop):   # fp16 x fp16 products are exact in fp32; the running sum is not
                part = (part.float() + a[:, i, None].float() * w[None, :, i].float()).half()
            blk = part.float()
        else:
            blk = a[:, sl].float() @ w[:, sl].float().t()
        if not (mutate == 'drop' and b == j):
            acc = acc + blk
        if mutate == 'twice' and b == j:
            acc = acc + blk
    return acc + bias


@pytest.mark.parametrize('k', [3072, 4096])
def test_gemm_bound_at_long_k(k):
    """At the K of the product's FC2 GEMMs (3072, 4096) the GEMM bound accepts an fp32 kernel that sums k-blocks of 64
    in order, and rejects one wrong k-block out of 48 / 64: dropped, counted twice, taken from a stale ring slot, or
    summed in fp16. Operands at model scale: A ~ N(0, 1), W ~ N(0, 0.03^2)."""
    gen = torch.Generator().manual_seed(k)
    m, n = 16, 24
    a = torch.randn(m, k, generator=gen).half()
    w = (torch.randn(n, k, generator=gen) * 0.03).half()
    bias = torch.randn(n, generator=gen) * 0.05
    right = _kblock_gemm(a, w, bias)
    rep = R.check_gemm('F32', right, a, w, bias)
    assert rep.passed, rep.describe(right, R.gemm_ref(a, w, bias, None)[0])
    for j in (LONG_K_STAGES, k // 128, k // 64 - 1):
        for mutate in ('drop', 'twice', 'stale', 'f16'):
            wrong = _kblock_gemm(a, w, bias, mutate, j)
            assert not R.check_gemm('F32', wrong, a, w, bias).passed, (mutate, j)


def _truncating_gemm(a, w):
    """An fp32 accumulator that adds each K_STEP products exactly and then rounds toward zero (the tensor cores'
    accumulation, as far as the bound is concerned)."""
    acc = torch.zeros(a.shape[0], w.shape[0], dtype=torch.float64)
    for k0 in range(0, a.shape[1], R.K_STEP):
        s = acc + a[:, k0:k0 + R.K_STEP].double() @ w[:, k0:k0 + R.K_STEP].double().t()   # exact: 16 products of fp16
        f = s.float()
        toward_zero = torch.nextafter(f, torch.zeros_like(f))
        acc = torch.where(f.double().abs() > s.abs(), toward_zero, f).double()
    return acc.float()


def test_gemm_bound_covers_a_truncating_accumulator():
    """Where every partial sum has the same sign (here: all operands positive) the truncation errors of the
    accumulator add up with the number of k-steps: at K = 4096 they exceed C_GEMM u sum|a w|, the bound at K <= 776.
    The partial-sum term of the bound (2 u per k-step) holds them, and the four wrong k-blocks stay rejected."""
    gen = torch.Generator().manual_seed(5)
    m, n, k = 16, 24, 4096
    a = torch.rand(m, k, generator=gen).half()
    w = (torch.rand(n, k, generator=gen) * 0.03).half()
    got = _truncating_gemm(a, w)
    x, mag = R.gemm_ref(a, w, None, None)
    assert not R.check_f32(got, x, R.C_GEMM * R.U32 * mag).passed
    rep = R.check_gemm('F32', got, a, w)
    assert rep.passed, rep.describe(got, x)
    for mutate in ('drop', 'twice', 'stale', 'f16'):
        assert not R.check_gemm('F32', _kblock_gemm(a, w, 0.0, mutate, k // 128), a, w).passed, mutate


# -------------------------------------------------------------------------------------------- attention checks
def _attn(q, k, v):
    """fp64 attention of [B, H, S, d] tensors -> merged [B*S, H*d]."""
    b, h, s, d = q.shape
    p = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(d), dim=-1)
    return (p @ v).permute(0, 2, 1, 3).reshape(b * s, h * d)


def _online_attention(qkv, batch, tokens, heads, d, chunk=64, l_corr=True, o_corr=True):
    """Flash-style chunked softmax with P rounded to fp16, optionally missing one of its two rescales."""
    q, k, v = R._split_qkv(qkv, batch, tokens, heads, d)
    s = q @ k.transpose(-1, -2) / math.sqrt(d)
    m = torch.full(s.shape[:-1] + (1,), -math.inf, dtype=torch.float64)
    l = torch.zeros_like(m)
    o = torch.zeros(s.shape[:-1] + (d,), dtype=torch.float64)
    for c0 in range(0, tokens, chunk):
        sc = s[..., c0:c0 + chunk]
        m_new = torch.maximum(m, sc.max(-1, keepdim=True).values)
        corr = torch.exp(m - m_new)
        p = torch.exp(sc - m_new)
        l = (l * corr if l_corr else l) + p.sum(-1, keepdim=True)
        o = (o * corr if o_corr else o) + R.f16_nearest(p) @ v[..., c0:c0 + chunk, :]
        m = m_new
    return (o / l).permute(0, 2, 1, 3).reshape(batch * tokens, heads * d).half()


def test_attention_checker_accepts_a_correct_online_kernel():
    for kind, tokens in (('rescale_last', 100), ('rescale_first', 100), ('mask', 33), ('large', 70), ('uniform', 65)):
        qkv = R.attention_case(kind, 1, tokens, 2, 64, seed=tokens)
        got = _online_attention(qkv, 1, tokens, 2, 64)
        rep = R.check_attention(got, qkv, 1, tokens, 2, 64, kind)
        assert rep.passed, rep.describe(got, R.attention_ref(qkv, 1, tokens, 2, 64)[0])


def test_attention_checker_rejects_unmasked_padding():
    batch, tokens, heads, d = 1, 33, 2, 64
    qkv = R.attention_case('mask', batch, tokens, heads, d, seed=3)
    q, k, v = R._split_qkv(qkv, batch, tokens, heads, d)
    pad = 64 - tokens                                  # zero-filled keys (logit 0) and values
    k = torch.cat([k, torch.zeros(batch, heads, pad, d, dtype=torch.float64)], dim=2)
    v = torch.cat([v, torch.zeros(batch, heads, pad, d, dtype=torch.float64)], dim=2)
    wrong = _attn(q, k, v).half()
    assert not R.check_attention(wrong, qkv, batch, tokens, heads, d).passed


@pytest.mark.parametrize('missing', ['l', 'o'])
def test_attention_checker_rejects_a_missing_online_rescale(missing):
    batch, tokens, heads, d = 1, 100, 2, 64
    qkv = R.attention_case('rescale_last', batch, tokens, heads, d, seed=4)
    wrong = _online_attention(qkv, batch, tokens, heads, d, l_corr=missing != 'l', o_corr=missing != 'o')
    assert not R.check_attention(wrong, qkv, batch, tokens, heads, d).passed


def test_attention_readout_rejects_p_kept_in_fp32():
    batch, tokens, heads, d = 2, 48, 2, 64
    qkv = R.attention_case('readout', batch, tokens, heads, d, seed=5)
    q, k, _ = R._split_qkv(qkv, batch, tokens, heads, d)
    t = q @ k.transpose(-1, -2) / math.sqrt(d)
    p = torch.exp(t - t.max(-1, keepdim=True).values)
    l32 = p.float().sum(-1, keepdim=True)

    def out(x):
        x = torch.cat([x, torch.zeros(batch, heads, tokens, d - tokens, dtype=x.dtype)], dim=-1)
        return x.permute(0, 2, 1, 3).reshape(batch * tokens, heads * d).half()

    right = out(R.f16_nearest(p).float() * (1.0 / l32))      # P rounded to fp16 before P.V, as the kernels do
    assert R.check_attention_readout(right, qkv, batch, tokens, heads, d).passed
    wrong = out(p.float() * (1.0 / l32))                       # P kept in fp32
    assert not R.check_attention_readout(wrong, qkv, batch, tokens, heads, d).passed
    assert R.check_attention(wrong, qkv, batch, tokens, heads, d).passed   # the general bound cannot tell them apart


@pytest.mark.parametrize('tokens', [65, 197, 300, 512])
def test_attention_uniform_check_pins_the_row_sum(tokens):
    """The uniform-weights check holds the output to a faithful rounding of the exact mean of V: a kernel whose row sum
    l counts one key too many or too few (the output off by S / (S +- 1)) is rejected at every S, up to 512."""
    batch, heads, d = 1, 2, 64
    qkv = R.attention_case('uniform', batch, tokens, heads, d, seed=tokens)
    _, _, v = R._split_qkv(qkv, batch, tokens, heads, d)
    mean = v.mean(-2, keepdim=True).expand(batch, heads, tokens, d)

    def out(x):
        return x.permute(0, 2, 1, 3).reshape(batch * tokens, heads * d).half()

    sums = v.sum(-2, keepdim=True).float().expand(batch, heads, tokens, d)     # exact: V is a multiple of 1/64
    right = out((sums * (1.0 / torch.tensor(float(tokens), dtype=torch.float32))).double())
    assert R.check_attention_uniform(right, qkv, batch, tokens, heads, d).passed
    assert R.check_attention(right, qkv, batch, tokens, heads, d).passed
    for miscount in (tokens - 1, tokens + 1):
        wrong = out(mean * tokens / miscount)
        assert not R.check_attention_uniform(wrong, qkv, batch, tokens, heads, d).passed, miscount


# -------------------------------------------------------------------------------------------- LayerNorm checks
def _ln_fp32(x, g, b, eps, single_pass=False, bessel=False):
    n = x.shape[-1]
    mean = x.sum(-1, keepdim=True) / n
    if single_pass:
        var = (x * x).sum(-1, keepdim=True) / n - mean * mean
    else:
        var = ((x - mean) ** 2).sum(-1, keepdim=True) / (n - 1 if bessel else n)
    return (x - mean) * torch.rsqrt(var.clamp_min(0) + eps) * g + b


@pytest.mark.parametrize('kind', R.LN_KINDS)
def test_layernorm_checker(kind):
    """An fp32 two-pass LayerNorm passes. Rejected: a Bessel-corrected variance (rows N(0.5, 2)), a one-pass variance
    (offset rows, where it cancels) and an output of just beta (wherever the bound is informative, i.e. not on the
    1e4 + N(0, 1e-2) rows)."""
    x, g, b = R.layernorm_case(13, 768, kind, seed=2)
    eps = 1e-12
    ref, bound = R.layernorm_ref(x.double(), g, b, eps)
    assert R.check_f32(_ln_fp32(x, g, b, eps), ref, bound).passed
    wrong = {'normal': ('bessel', 'beta'), 'offset': ('single', 'beta'), 'offset_1e4': ('single',)}[kind]
    if 'bessel' in wrong:
        assert not R.check_f32(_ln_fp32(x, g, b, eps, bessel=True), ref, bound).passed
    if 'single' in wrong:
        assert not R.check_f32(_ln_fp32(x, g, b, eps, single_pass=True), ref, bound).passed
    if 'beta' in wrong:
        assert not R.check_f32(b.expand_as(x), ref, bound).passed


@pytest.mark.parametrize('offset', [0.0, 1e3])
def test_linear_ln_checker(offset):
    """The fused projection + residual + LayerNorm check: an fp32 kernel (accumulate, + bias, + resid, two-pass
    LayerNorm) passes with either fp32 output. Rejected: a LayerNorm of v without the residual, and (on rows offset by
    1e3, where it cancels) a one-pass variance."""
    m, n, k = 70, 192, 256
    gen = torch.Generator().manual_seed(11)
    a = (torch.randn(m, k, generator=gen) * 0.7).half()
    w = (torch.randn(n, k, generator=gen) * (1.0 / math.sqrt(k))).half()
    bias = torch.randn(n, generator=gen) * 0.1
    resid = offset + torch.randn(m, n, generator=gen)
    g = 1 + 0.1 * torch.randn(n, generator=gen)
    b = 0.1 * torch.randn(n, generator=gen)
    eps = 1e-12
    x = a.float() @ w.float().t() + bias
    v = x + resid
    ln = _ln_fp32(v, g, b, eps)

    def passes(got32, got16, f32_is_ln):
        r32, r16 = R.check_linear_ln(got32, got16, a, w, bias, resid, g, b, eps, f32_is_ln)
        return r32.passed and r16.passed

    assert passes(v, ln.half(), False) and passes(ln, ln.half(), True)
    no_resid = _ln_fp32(x, g, b, eps)
    assert not passes(v, no_resid.half(), False) and not passes(no_resid, ln.half(), True)
    if offset:
        one_pass = _ln_fp32(v, g, b, eps, single_pass=True)
        assert not passes(v, one_pass.half(), False) and not passes(one_pass, ln.half(), True)


# ------------------------------------------------------------------------------------ GEMM case list coverage
def _plan(case):
    from pipeedge_b200 import _lib
    return R.query_plan(_lib, case)


def test_epilogue_ids_match_the_library():
    from pipeedge_b200 import _lib
    for name, value in R.EPI.items():
        assert getattr(_lib, 'PE_EPI_' + name) == value


def test_gemm_cases_reach_every_path():
    """Each case's plan has the properties its name claims, and together the cases run every epilogue on the scalar
    (n % 8 != 0) path with and without bias, on n % 8 in {odd, 4, 0}, k < 64, ragged K and M, under several rounds per
    CTA, under clusters along M and along N, and on partly empty clusters along both."""
    seen = {epi: set() for epi in R.EPI}
    for case in R.RAGGED_CASES + R.SCHEDULE_CASES:
        geom = _plan(case)
        bad = R.expectation_failures(case, geom)
        assert not bad, (case.name, bad)
        tags = seen[case.epi]
        tags.add(('n%8', 'odd' if case.n % 2 else case.n % 8))
        if geom['scalar']:
            tags.add('scalar-bias' if case.bias else 'scalar-nobias')
        if case.k < 64:
            tags.add('k<64')
        if case.k % 64:
            tags.add('ragged-k')
        if case.m < 128:
            tags.add('m<128')
        if case.m > 128 and case.m % 128:
            tags.add('ragged-m')
        if geom['rounds'] > 1:
            tags.add('multi-round')
            if geom['cm'] * geom['cn'] > 1:
                tags.add('multi-round-cluster')
        if geom['cm'] > 1:
            tags.add('cluster-m')
        if geom['cn'] > 1:
            tags.add('cluster-n')
        if geom['partial_m']:
            tags.add('partial-m')
        if geom['partial_n']:
            tags.add('partial-n')
        if case.inplace:
            tags.add('inplace')
    need = {('n%8', 'odd'), ('n%8', 4), ('n%8', 0), 'scalar-bias', 'scalar-nobias', 'k<64', 'ragged-k', 'm<128',
            'ragged-m', 'multi-round', 'multi-round-cluster', 'cluster-m', 'cluster-n', 'partial-m', 'partial-n'}
    for epi, tags in seen.items():
        missing = need - tags
        assert not missing, (epi, missing)
    assert 'inplace' in seen['RESID_F32']
