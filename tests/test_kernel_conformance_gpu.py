"""GPU: the wgmma GEMM (every epilogue, every schedule), both attention kernels, the patch / BERT embeddings, the casts and
LayerNorm against fp64 restatements of the same operation on the same operands, element by element, at the shapes,
tiles, paddings and values where such kernels go wrong. References, bounds and case lists live in `_fp_ref.py` (the CPU
tests in `test_fp_ref_cpu.py` show that each checker rejects a plausible wrong kernel).

Run with `-s` to see, per kernel family, the largest err / bound and the fraction of fp16 outputs that are correctly
rounded (not merely faithful)."""
import json
import os
import subprocess
import sys
import zlib

import pytest
import torch
import torch.nn.functional as F

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
sys.path.insert(0, TESTS)
import _fp_ref as R  # noqa: E402
import _gemm_census as G  # noqa: E402

gpu = pytest.mark.gpu
pytestmark = gpu

_STATS = {}


def _record(family, rep):
    s = _STATS.setdefault(family, {'max_ratio': 0.0, 'min_cr': 1.0, 'cr_sum': 0.0, 'checks': 0})
    s['max_ratio'] = max(s['max_ratio'], rep.max_ratio)
    s['checks'] += 1
    if rep.correctly_rounded is not None:
        s['min_cr'] = min(s['min_cr'], rep.correctly_rounded)
        s['cr_sum'] += rep.correctly_rounded


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    for family, s in sorted(_STATS.items()):
        print(f"\nCONFORMANCE {json.dumps({'family': family, **s})}")


def _assert(rep, got, ref, family):
    _record(family, rep)
    assert rep.passed, rep.describe(got, ref)


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from pipeedge_b200 import ops as _ops
    return _ops


def _lib():
    from pipeedge_b200 import _lib
    return _lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------------- GEMM
def _run_gemm_case(ops, case, seed):
    lib = _lib()
    geom = R.query_plan(lib, case)
    bad = R.expectation_failures(case, geom)
    assert not bad, f"{case.name}: the planner no longer gives this case its path: {bad}"
    a, w, bias, resid = (None if t is None else t.cuda() for t in R.gemm_operands(case, seed))
    epi = R.EPI[case.epi]
    resid_before = resid.clone()
    if case.inplace:
        got = ops.linear(a, w, bias, epi, resid=resid, out=resid)
        assert got.data_ptr() == resid.data_ptr()
    else:
        got = ops.linear(a, w, bias, epi, resid=resid if case.epi == 'RESID_F32' else None)
    torch.cuda.synchronize()
    rep = R.check_gemm(case.epi, got, a, w, bias, resid_before, where=case.name)
    family = 'gemm-' + case.epi
    _record(family, rep)
    if not rep.passed:
        x, _ = R.gemm_ref(a, w, bias, None)
        ref = {'RESID_F32': x + resid_before.double(), 'TANH_F32': torch.tanh(x), 'GELU_F16': R.gelu64(x)}.get(case.epi, x)
        pytest.fail(rep.describe(got, ref) + f"\n  plan {geom}")


@pytest.mark.parametrize('case', R.RAGGED_CASES, ids=lambda c: c.name)
def test_gemm_ragged_grid(ops, case):
    """Every epilogue with and without bias on n % 8 in {odd, 4, 0} (the scalar epilogue path), k < 64, ragged K and a
    ragged last M tile."""
    _run_gemm_case(ops, case, seed=case.m * 7 + case.n * 3 + case.k)


@pytest.mark.parametrize('case', R.SCHEDULE_CASES, ids=lambda c: c.name)
def test_gemm_schedules(ops, case, monkeypatch):
    """Every epilogue (RESID_F32 in place) under the natural one-round and multi-round plans and the forced plans:
    several tiles per CTA, clusters along M and N with TMA multicast, and partly empty clusters along both."""
    if case.force:
        monkeypatch.setenv('PE_GEMM_FORCE', case.force)
    _run_gemm_case(ops, case, seed=17)


@pytest.mark.parametrize('n', [8, 5])
def test_gemm_activation_scan(ops, n):
    """a[:, 0] = every fp16 h in [-12, 12], w[:, 0] = 1, the rest 0: the pre-activation is exactly fl32(h + b). GELU_F16
    must be a faithful fp16 rounding of x Phi(x) (both sides of the polynomial's clamp at |x| = 6, the fp16-subnormal
    tail of negative GELU, 0 and +-tiny); TANH_F32 within 2 ulp of fp32. n = 5 runs the scalar epilogue path."""
    lib = _lib()
    h, b = R.scan_inputs()
    b = b[:n]
    m, k = h.numel(), 8
    a = torch.zeros(m, k, dtype=torch.float16)
    a[:, 0] = h
    w = torch.zeros(n, k, dtype=torch.float16)
    w[:, 0] = 1
    x = R.scan_preact(h, b)
    g16 = ops.linear(a.cuda(), w.cuda(), b.cuda(), lib.PE_EPI_GELU_F16).cpu()
    t32 = ops.linear(a.cuda(), w.cuda(), b.cuda(), lib.PE_EPI_TANH_F32).cpu()
    _assert(R.check_gelu_scan(g16, x), g16, R.gelu64(x), 'gelu-scan')
    _assert(R.check_tanh_scan(t32, x), t32, torch.tanh(x), 'tanh-scan')


PRODUCT_CASES = G.census(_lib())
W_STD, BIAS_STD = 0.03, 0.05    # model-scale weights and biases (the synthetic checkpoints use 0.02)


def _product_feeder(ops, case, k, gen):
    """-> a function that launches the kernel that writes A [m, k] fp16 just before `case` in the product (on the
    current stream, inputs already on the device) and returns A. The operands come out roughly N(0, 1), FC2's A is
    the GELU output of an FC1 run as the stage runs it."""
    m = case.m
    if case.feeder == 'layernorm':
        x = (torch.randn(m, k, generator=gen) * 1.5 + 0.3).cuda()
        g = (1 + 0.1 * torch.randn(k, generator=gen)).cuda()
        b = (0.1 * torch.randn(k, generator=gen)).cuda()
        return lambda: ops.layernorm(x, g, b, 1e-6, want_f32=False, want_f16=True)[1]
    if case.feeder == 'cast':
        x = torch.randn(m, k, generator=gen).cuda()
        a = torch.empty(m, k, dtype=torch.float16, device='cuda')
        return lambda: (_cast(_lib().LIB.pe_cast_f32_to_f16, x, a, m * k), a)[1]
    if case.feeder == 'attention':
        spec = G.MODEL_SPECS[case.model]
        qkv = torch.randn(m, 3 * k, generator=gen)
        qkv[:, 2 * k:] *= (case.tokens / 3) ** 0.5       # the context (a weighted mean of V rows) comes out ~N(0, 1)
        qkv = qkv.half().cuda()
        return lambda: ops.attention(qkv, case.ub, case.tokens, spec.heads)
    if case.feeder == 'fc1':
        h = case.n                                        # FC2 [m, H] reads FC1's GELU output [m, I]
        a0 = torch.randn(m, h, generator=gen).half().cuda()
        w1 = (torch.randn(k, h, generator=gen) * W_STD).half().cuda()
        b1 = (torch.randn(k, generator=gen) * BIAS_STD).cuda()
        return lambda: ops.linear(a0, w1, b1, _lib().PE_EPI_GELU_F16, static_w=True)
    raise ValueError(case.feeder)


def _product_patch_embed(case, gen):
    """The patch embedding as the first ViT / DeiT stage runs it (im2col, prefix rows, then the GEMM's row-remapped
    RESID_F32 epilogue adding the position rows) -> (got [B * patches, H], A, W, bias, resid) for check_gemm."""
    spec = G.MODEL_SPECS[case.model]
    n_prefix = 2 if spec.family == 'deit' else 1
    hidden, kpad, batch = case.n, case.k, case.ub
    kdim = spec.channels * spec.patch ** 2
    pixels = torch.randn(batch, spec.channels, spec.image_size, spec.image_size, generator=gen).cuda()
    w16 = torch.zeros(hidden, kpad, dtype=torch.float16)
    w16[:, :kdim] = (torch.randn(hidden, kdim, generator=gen) * W_STD).half()
    w16 = w16.cuda()
    bias = (torch.randn(hidden, generator=gen) * BIAS_STD).cuda()
    pos = torch.randn(case.tokens, hidden, generator=gen).cuda()
    prefix = torch.randn(n_prefix, hidden, generator=gen).cuda()
    lib = _lib()
    n_patches = case.tokens - n_prefix
    out = torch.empty((batch, case.tokens, hidden), dtype=torch.float32, device='cuda')
    work = torch.empty((batch * n_patches, kpad), dtype=torch.float16, device='cuda')
    torch.cuda.synchronize()
    lib.check(lib.LIB.pe_patch_embed(pixels.data_ptr(), w16.data_ptr(), bias.data_ptr(), pos.data_ptr(), prefix.data_ptr(),
                                     out.data_ptr(), work.data_ptr(), batch, spec.channels, spec.image_size, spec.patch,
                                     hidden, n_prefix, _stream()))
    torch.cuda.synchronize()
    assert torch.equal(out[:, :n_prefix], prefix.expand(batch, n_prefix, hidden))
    resid = pos[n_prefix:].repeat(batch, 1)
    return out[:, n_prefix:].reshape(batch * n_patches, hidden), work, w16, bias, resid


@pytest.mark.parametrize('case', PRODUCT_CASES, ids=lambda c: c.name)
def test_gemm_product_plans(ops, case):
    """Every plan the supported models run (`_gemm_census`: one case per (epilogue, static_w, plan, ring depth, one
    or several tiles per CTA, K loop against the ring, partly empty clusters, scalar epilogue), at its smallest
    product shape, plus the benchmark's 16 GEMMs), run the way the product runs it: A written on the same stream, with
    nothing synchronised in between, by the kernel that writes it in the product (LayerNorm, cast, attention, FC1's
    GELU epilogue, im2col), stage GEMMs with static_w (W streamed before that kernel has finished), model-scale
    operands. Every element against fp64 on the A actually produced."""
    lib = _lib()
    geom = R.query_plan(lib, case)
    bad = R.expectation_failures(case, geom)
    assert not bad, f"{case.name}: the planner no longer gives this call the plan of its census key: {bad}"
    gen = torch.Generator().manual_seed(zlib.crc32(case.name.encode()))
    if case.feeder == 'im2col':
        got, a, w, bias, resid = _product_patch_embed(case, gen)
    else:
        w = (torch.randn(case.n, case.k, generator=gen) * W_STD).half().cuda()
        bias = (torch.randn(case.n, generator=gen) * BIAS_STD).cuda()
        resid = None
        feed = _product_feeder(ops, case, case.k, gen)
        torch.cuda.synchronize()
        a = feed()
        got = ops.linear(a, w, bias, R.EPI[case.epi], static_w=bool(case.static_w))
        torch.cuda.synchronize()
    rep = R.check_gemm(case.epi, got, a, w, bias, resid, where=case.name)
    _record('gemm-product-' + case.epi, rep)
    if case.k >= 3072:
        _record('gemm-product-k>=3072-' + case.epi, rep)
    if not rep.passed:
        x, _ = R.gemm_ref(a, w, bias, None)
        ref = {'RESID_F32': x + (0 if resid is None else resid.double()), 'TANH_F32': torch.tanh(x),
               'GELU_F16': R.gelu64(x)}.get(case.epi, x)
        pytest.fail(rep.describe(got, ref) + f"\n  plan {geom}")


def test_gemm_dependent_chain_under_pdl(ops):
    """F16 -> GELU_F16 (static_w) -> RESID_F32 (static_w, in place), each consuming the previous output with nothing
    synchronising in between: bit-identical to the same chain with a device synchronisation after every step."""
    lib = _lib()
    gen = torch.Generator().manual_seed(8)
    m, h, inter = 1576, 768, 3072
    x = torch.randn(m, h, generator=gen).half().cuda()
    w1 = (torch.randn(h, h, generator=gen) * 0.04).half().cuda()
    w2 = (torch.randn(inter, h, generator=gen) * 0.04).half().cuda()
    w3 = (torch.randn(h, inter, generator=gen) * 0.02).half().cuda()
    b1, b2, b3 = (torch.randn(n, generator=gen).cuda() for n in (h, inter, h))
    r0 = torch.randn(m, h, generator=gen).cuda()

    def chain(sync):
        r = r0.clone()
        torch.cuda.synchronize()
        y1 = ops.linear(x, w1, b1, lib.PE_EPI_F16)
        if sync:
            torch.cuda.synchronize()
        y2 = ops.linear(y1, w2, b2, lib.PE_EPI_GELU_F16, static_w=True)
        if sync:
            torch.cuda.synchronize()
        ops.linear(y2, w3, b3, lib.PE_EPI_RESID_F32, resid=r, out=r, static_w=True)
        torch.cuda.synchronize()
        return y1, y2, r

    for got, want in zip(chain(False), chain(True)):
        assert torch.equal(got, want)


# ----------------------------------------------------------------------------------------------- patch embedding
def patch_embed(pixels, w16, bias, pos, prefix, patch, n_prefix):
    """`pe_patch_embed` as vit.py calls it: pixels f32 [B, C, img, img], w f16 [H, kpad], bias f32 [H], pos f32
    [tokens, H], prefix f32 [n_prefix, H] -> f32 [B, tokens, H]."""
    lib = _lib()
    batch, channels, img, _ = pixels.shape
    hidden, kpad = w16.shape
    n_patches = (img // patch) ** 2
    out = torch.empty((batch, n_patches + n_prefix, hidden), dtype=torch.float32, device=pixels.device)
    work = torch.empty((batch * n_patches, kpad), dtype=torch.float16, device=pixels.device)
    lib.check(lib.LIB.pe_patch_embed(pixels.data_ptr(), w16.data_ptr(), bias.data_ptr(), pos.data_ptr(), prefix.data_ptr(),
                                     out.data_ptr(), work.data_ptr(), batch, channels, img, patch, hidden, n_prefix, _stream()))
    return out


@pytest.mark.parametrize('batch', [1, 3])
@pytest.mark.parametrize('name,patch,hidden,n_prefix', [('vit-b', 16, 768, 1), ('deit', 16, 768, 2), ('vit-huge', 14, 1280, 1)])
def test_patch_embed(ops, name, patch, hidden, n_prefix, batch):
    """The GEMM's row-remap epilogue (rows_per_item, out_row_offset, resid_per_item) against fp64 conv2d on the
    fp16-rounded pixels and weights, + bias + position rows; 196 / 256 patches per item so that 128-row tiles straddle
    items; ViT-Huge's K = 588 padded to 592. Prefix rows are copied bit for bit."""
    gen = torch.Generator().manual_seed(hidden + patch + batch)
    channels, img = 3, 224
    kdim = channels * patch * patch
    kpad = (kdim + 7) // 8 * 8
    n_patches = (img // patch) ** 2
    tokens = n_patches + n_prefix
    pixels = torch.randn(batch, channels, img, img, generator=gen)
    conv = torch.randn(hidden, channels, patch, patch, generator=gen) * (1.5 / kdim ** 0.5)
    w16 = torch.zeros(hidden, kpad, dtype=torch.float16)
    w16[:, :kdim] = conv.reshape(hidden, kdim).half()
    bias = torch.randn(hidden, generator=gen) * 0.1
    pos = torch.randn(tokens, hidden, generator=gen) * 0.5
    prefix = torch.randn(n_prefix, hidden, generator=gen)
    got = patch_embed(pixels.cuda(), w16.cuda(), bias.cuda(), pos.cuda(), prefix.cuda(), patch, n_prefix)
    torch.cuda.synchronize()
    got = got.cpu()
    assert torch.equal(got[:, :n_prefix], prefix.expand(batch, n_prefix, hidden))
    p64 = pixels.half().double()
    w64 = w16[:, :kdim].double().reshape(hidden, channels, patch, patch)
    conv64 = F.conv2d(p64, w64, stride=patch).flatten(2).transpose(1, 2)              # [B, patches, H]
    mag = F.conv2d(p64.abs(), w64.abs(), stride=patch).flatten(2).transpose(1, 2)
    ref = conv64 + bias.double() + pos[n_prefix:].double()
    mag = mag + bias.double().abs() + pos[n_prefix:].double().abs()
    rep = R.check_f32(got[:, n_prefix:], ref, R.C_GEMM * R.U32 * mag, f'patch-embed {name} batch {batch}')
    _assert(rep, got[:, n_prefix:], ref, 'patch-embed')


# ----------------------------------------------------------------------------------------------------- attention
ATTN_BATCH, ATTN_HEADS = 2, 2


def attention_cases(head_dim):
    return [(kind, tokens) for tokens in R.ATTN_TOKENS for kind in R.ATTN_KINDS
            if R.attention_kind_applies(kind, tokens, head_dim)]


def run_attention_case(ops, kind, tokens, head_dim):
    """-> (report, got, ref) for one case."""
    seed = tokens * 13 + head_dim + R.ATTN_KINDS.index(kind)
    qkv = R.attention_case(kind, ATTN_BATCH, tokens, ATTN_HEADS, head_dim, seed)
    got = ops.attention(qkv.cuda(), ATTN_BATCH, tokens, ATTN_HEADS, head_dim=head_dim)
    torch.cuda.synchronize()
    got = got.cpu()
    where = f'attention d={head_dim} {kind} S={tokens}'
    ref = R.attention_ref(qkv, ATTN_BATCH, tokens, ATTN_HEADS, head_dim)[0]
    if kind == 'uniform':
        rep = R.check_attention_uniform(got, qkv, ATTN_BATCH, tokens, ATTN_HEADS, head_dim, where=where)
    elif kind == 'readout':
        rep = R.check_attention_readout(got, qkv, ATTN_BATCH, tokens, ATTN_HEADS, head_dim, where=where)
    else:
        rep = R.check_attention(got, qkv, ATTN_BATCH, tokens, ATTN_HEADS, head_dim, where=where)
    if kind == 'large':
        assert bool(torch.isfinite(got).all()), where
    return rep, got, ref


@pytest.mark.parametrize('head_dim', [64, 80])
@pytest.mark.parametrize('kind,tokens', attention_cases(64), ids=lambda v: str(v))
def test_attention(ops, kind, tokens, head_dim):
    """Default kernel selection: wgmma for head_dim 64 and S <= 256, mma.sync otherwise (head_dim 80 always)."""
    if not R.attention_kind_applies(kind, tokens, head_dim):
        pytest.skip('case does not apply')
    rep, got, ref = run_attention_case(ops, kind, tokens, head_dim)
    family = 'attention-wgmma' if head_dim == 64 and tokens <= 256 else 'attention-mma.sync'
    _assert(rep, got, ref, family)


_CHILD = """
import json, os, sys
sys.path[:0] = [sys.argv[1], os.path.join(sys.argv[1], 'tests')]
import test_kernel_conformance_gpu as T
from pipeedge_b200 import ops
sys.exit(T.child_main(ops, sys.argv[2]))
"""


def child_main(ops, what):
    """Entry point of the child processes (the library reads PE_ATTN_WGMMA / PE_FUSE_LN once per process)."""
    failures = []
    if what == 'attention':
        for kind, tokens in attention_cases(64):
            rep, got, ref = run_attention_case(ops, kind, tokens, 64)
            _record('attention-mma.sync', rep)
            if not rep.passed:
                failures.append(rep.describe(got, ref))
    elif what == 'layernorm':
        for args in LN_CASES:
            failures += run_layernorm_case(ops, *args, family='layernorm-fuse-ln')
    for family, s in sorted(_STATS.items()):
        print(f"CONFORMANCE {json.dumps({'family': family, **s})}", flush=True)
    print('\n'.join(failures) if failures else 'all ok', flush=True)
    return 1 if failures else 0


def _child(what, env):
    res = subprocess.run([sys.executable, '-c', _CHILD, ROOT, what], capture_output=True, text=True, timeout=900,
                         env={**os.environ, **env})
    for line in res.stdout.splitlines():
        if line.startswith('CONFORMANCE '):
            print('\n' + line)
    assert res.returncode == 0 and 'all ok' in res.stdout, res.stdout[-4000:] + res.stderr[-4000:]


def test_attention_mma_sync_kernel(ops):
    """Every attention case on the mma.sync kernel (PE_ATTN_WGMMA=0, child process): 16-key groups, 64-key chunks and
    the online-softmax rescale across chunks."""
    _child('attention', {'PE_ATTN_WGMMA': '0'})


def test_attention_rejections(ops):
    """More than 512 tokens, or head_dim other than 64 / 80, fail on the host before anything is launched."""
    lib = _lib()
    for tokens, heads, head_dim in ((513, 2, 64), (600, 1, 80), (16, 2, 32), (16, 1, 128), (16, 2, 96), (300, 2, 48)):
        qkv = torch.zeros(tokens, 3 * heads * head_dim, dtype=torch.float16, device='cuda')
        before = ops.launch_count()
        with pytest.raises(lib.PipeEdgeB200Error):
            ops.attention(qkv, 1, tokens, heads, head_dim=head_dim)
        assert ops.launch_count() == before, (tokens, head_dim)


# ---------------------------------------------------------------------------------------------------------- casts
def _cast(fn, src, dst, n):
    _lib().check(fn(src.data_ptr(), dst.data_ptr(), n, _stream()))


def _same_bits_or_nan(got, want):
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan)
    assert torch.equal(got[~nan].view(torch.int16 if got.dtype == torch.float16 else torch.int32),
                       want[~nan].view(torch.int16 if want.dtype == torch.float16 else torch.int32))


def test_cast_f16_to_f32_exhaustive(ops):
    """All 65 536 fp16 bit patterns, bit-exact (NaN as NaN); lengths of every remainder modulo 4."""
    lib = _lib()
    bits = torch.arange(0, 0x10000, dtype=torch.int32)
    h = torch.where(bits >= 0x8000, bits - 0x10000, bits).to(torch.int16).view(torch.float16)
    want = h.float()
    src = h.cuda()
    for n in (65536, 65535, 65534, 65533, 1, 2, 3):
        dst = torch.full((n,), 7.0, device='cuda')
        _cast(lib.LIB.pe_cast_f16_to_f32, src, dst, n)
        torch.cuda.synchronize()
        _same_bits_or_nan(dst.cpu(), want[:n])
    with pytest.raises(lib.PipeEdgeB200Error):
        _cast(lib.LIB.pe_cast_f16_to_f32, src[1:], torch.empty(8, device='cuda'), 8)         # src not 4-byte aligned
    with pytest.raises(lib.PipeEdgeB200Error):
        _cast(lib.LIB.pe_cast_f16_to_f32, src, torch.empty(9, device='cuda')[1:], 8)         # dst not 8-byte aligned


def test_cast_f32_to_f16_edges(ops):
    """Round-to-nearest-even against torch's .half() on +-0, fp16 subnormals and their rounding boundaries, the top of
    the range (65504, 65519.99 -> 65504, 65520 -> inf), +-inf and NaN; lengths of every remainder modulo 4."""
    lib = _lib()
    sub = [k * 2.0 ** -25 for k in range(0, 12)] + [2.0 ** -14, 2.0 ** -14 - 2.0 ** -25, 2.0 ** -24]
    vals = torch.tensor(sub + [65504.0, 65519.99, 65520.0, 65519.0, 1e5, float('inf'), float('nan'), 1.0, 1.0 + 2.0 ** -11,
                               1.0 + 3 * 2.0 ** -11, 2049.0, 2051.0], dtype=torch.float32)
    near = torch.cat([vals, torch.nextafter(vals, torch.full_like(vals, float('inf'))),
                      torch.nextafter(vals, torch.full_like(vals, -float('inf')))])
    gen = torch.Generator().manual_seed(1)
    rnd = torch.randn(4000, generator=gen) * 10.0 ** torch.randint(-9, 6, (4000,), generator=gen).float()
    x = torch.cat([near, -near, rnd])
    src = x.cuda()
    for n in (x.numel(), x.numel() - 1, x.numel() - 2, x.numel() - 3, 1, 2, 3, 5):
        dst = torch.zeros(n, dtype=torch.float16, device='cuda')
        _cast(lib.LIB.pe_cast_f32_to_f16, src, dst, n)
        torch.cuda.synchronize()
        _same_bits_or_nan(dst.cpu(), x[:n].half())
    with pytest.raises(lib.PipeEdgeB200Error):
        _cast(lib.LIB.pe_cast_f32_to_f16, src[1:], torch.empty(8, dtype=torch.float16, device='cuda'), 8)   # src 16 B
    with pytest.raises(lib.PipeEdgeB200Error):
        _cast(lib.LIB.pe_cast_f32_to_f16, src, torch.empty(9, dtype=torch.float16, device='cuda')[1:], 8)   # dst 8 B


# --------------------------------------------------------------------------------------------- BERT embedding
@pytest.mark.parametrize('hidden', [128, 768])
@pytest.mark.parametrize('batch,seq', [(3, 7), (2, 33)])
def test_bert_embed(ops, batch, seq, hidden):
    """LayerNorm(word[id] + type0 + pos[pos_id]) against fp64: ids 0 and V - 1, permuted position ids, row counts not
    divisible by 4."""
    lib = _lib()
    vocab, max_pos = 50, 64
    gen = torch.Generator().manual_seed(batch * seq + hidden)
    word = torch.randn(vocab, hidden, generator=gen)
    type0 = torch.randn(hidden, generator=gen) * 0.5
    pos = torch.randn(max_pos, hidden, generator=gen) * 0.5
    gamma = 1 + 0.1 * torch.randn(hidden, generator=gen)
    beta = 0.1 * torch.randn(hidden, generator=gen)
    ids = torch.randint(0, vocab, (batch, seq), generator=gen)
    ids[0, 0], ids[-1, -1] = 0, vocab - 1
    pos_ids = torch.randperm(max_pos, generator=gen)[:seq]
    eps = 1e-12
    out = torch.empty(batch, seq, hidden, device='cuda')
    dev = [t.cuda() for t in (ids, pos_ids, word, type0, pos, gamma, beta)]
    lib.check(lib.LIB.pe_bert_embed(*(t.data_ptr() for t in dev), eps, out.data_ptr(), batch, seq, hidden, _stream()))
    torch.cuda.synchronize()
    parts = (word[ids].double(), type0.double(), pos[pos_ids].double())
    x = parts[0] + parts[1] + parts[2]
    in_err = 2 * R.U32 * (parts[0].abs() + parts[1].abs() + parts[2].abs())    # (word + type) + pos in fp32
    ref, bound = R.layernorm_ref(x, gamma, beta, eps, in_err)
    got = out.cpu()
    _assert(R.check_f32(got, ref, bound, f'bert-embed {batch}x{seq}x{hidden}'), got, ref, 'bert-embed')


# --------------------------------------------------------------------------------------------------- LayerNorm
LN_CASES = [(rows, hidden, kind) for hidden in (4, 128, 768, 1024, 1536)
            for rows, kind in ((7, 'normal'), (13, 'offset'), (11, 'offset_1e4'), (394, 'normal'))]


def run_layernorm_case(ops, rows, hidden, kind, family='layernorm'):
    """pe_layernorm (f32 + f16) and pe_residual_layernorm with sum_out aliasing resid; returns failure messages.
    Statistics go to `family`-{f32, f16, residual}; the 1e4-offset rows, whose bound is of the order of the output,
    to a family of their own."""
    lib = _lib()
    if kind == 'offset_1e4':
        family += '-offset1e4'
    x, g, b = R.layernorm_case(rows, hidden, kind, seed=rows * 5 + hidden)
    eps = 1e-12
    failures = []
    o32, o16 = ops.layernorm(x.cuda(), g.cuda(), b.cuda(), eps, want_f32=True, want_f16=True)
    ref, bound = R.layernorm_ref(x.double(), g, b, eps)
    where = f'layernorm {rows}x{hidden} {kind}'
    for rep, got, out in ((R.check_f32(o32.cpu(), ref, bound, where + ' f32'), o32.cpu(), 'f32'),
                          (R.check_f16(o16.cpu(), ref, ref - bound, ref + bound, where + ' f16'), o16.cpu(), 'f16')):
        _record(f'{family}-{out}', rep)
        if not rep.passed:
            failures.append(rep.describe(got, ref))
    # residual form, the updated stream written over resid itself
    gen = torch.Generator().manual_seed(rows + hidden)
    y = torch.randn(rows, hidden, generator=gen) * 0.5
    r = x.cuda().clone()
    o32 = torch.empty(rows, hidden, device='cuda')
    yd, gd, bd = y.cuda(), g.cuda(), b.cuda()      # held: a temporary's block would be handed to the next one
    lib.check(lib.LIB.pe_residual_layernorm(yd.data_ptr(), r.data_ptr(), gd.data_ptr(), bd.data_ptr(), eps, r.data_ptr(),
                                            o32.data_ptr(), None, rows, hidden, _stream()))
    torch.cuda.synchronize()
    t32 = y + x                                               # the fp32 sum the kernel must write back
    if not torch.equal(r.cpu(), t32):
        failures.append(f'{where}: sum_out aliasing resid is not y + resid')
    ref, bound = R.layernorm_ref(t32.double(), g, b, eps)
    rep = R.check_f32(o32.cpu(), ref, bound, where + ' residual')
    _record(f'{family}-residual', rep)
    if not rep.passed:
        failures.append(rep.describe(o32.cpu(), ref))
    return failures


@pytest.mark.parametrize('rows,hidden,kind', LN_CASES)
def test_layernorm(ops, rows, hidden, kind):
    """Hidden 4 .. 1536 (the stand-alone limit), row counts not divisible by 4, rows with a large common offset
    (1e3 + N(0, 1); and 1e4 + N(0, 1e-2), which only catches a one-pass variance), and the residual form updating the
    stream in place."""
    failures = run_layernorm_case(ops, rows, hidden, kind)
    assert not failures, '\n'.join(failures)


def test_layernorm_rejects_too_wide_rows(ops):
    lib = _lib()
    x = torch.zeros(4, 1540, device='cuda')
    g = torch.ones(1540, device='cuda')
    with pytest.raises(lib.PipeEdgeB200Error):
        ops.layernorm(x, g, g, 1e-12)


# ------------------------------------------------------------------------- projection + residual + LayerNorm (fused)
LINEAR_LN_CASES = [
    # m, n, k, rows, cluster: 1 to 3 row tiles of 128 with ragged last ones, several tiles per cluster (4096 rows)
    (128, 768, 768, 'normal', 8),
    (300, 768, 3072, 'offset', 8),
    (256, 1024, 4096, 'normal', 8),
    (384, 384, 1536, 'offset', 4),
    (70, 192, 768, 'normal', 2),
    (200, 96, 512, 'offset', 1),
    (4096, 768, 768, 'offset', 8),
]


@pytest.mark.parametrize('f32_is_ln', [False, True], ids=['f32=v', 'f32=ln'])
@pytest.mark.parametrize('m,n,k,rows,cluster', LINEAR_LN_CASES, ids=lambda v: str(v))
def test_linear_residual_layernorm(ops, m, n, k, rows, cluster, f32_is_ln):
    """The fused epilogue (clusters of 8, 4, 2 and 1 CTAs exchanging row statistics) against fp64, its fp32 output
    written over the residual in place as the stage does: LayerNorm(v) within the LayerNorm bound fed by the GEMM's
    error, the fp16 output a faithful rounding of it, and v itself (f32_is_ln off) within the GEMM bound. 'offset'
    rows sit at 1e3 + N(0, 1) (a one-pass variance cancels there)."""
    assert _lib().LIB.pe_linear_ln_cluster(n) == cluster
    gen = torch.Generator().manual_seed(m + n + k)
    a = (torch.randn(m, k, generator=gen) * 0.7).half()
    w = (torch.randn(n, k, generator=gen) * (1.0 / k ** 0.5)).half()
    bias = torch.randn(n, generator=gen) * 0.1
    resid = (1e3 if rows == 'offset' else 0.2) + torch.randn(m, n, generator=gen) * 1.3
    gamma = 1.0 + 0.1 * torch.randn(n, generator=gen)
    beta = 0.1 * torch.randn(n, generator=gen)
    eps = 1e-12
    dev = [t.cuda() for t in (a, w, bias, resid, gamma, beta)]
    r_dev = dev[3]
    o32, o16 = ops.linear_residual_layernorm(dev[0], dev[1], dev[2], r_dev, dev[4], dev[5], eps, f32_is_ln=f32_is_ln,
                                             out_f32=r_dev)
    torch.cuda.synchronize()
    assert o32.data_ptr() == r_dev.data_ptr()
    where = f'linear+ln {m}x{n}x{k} {rows} cluster {cluster}'
    rep32, rep16 = R.check_linear_ln(o32, o16, dev[0], dev[1], dev[2], resid.cuda(), dev[4], dev[5], eps, f32_is_ln,
                                     where=where)
    v, _, ln, _ = R.linear_ln_ref(dev[0], dev[1], dev[2], resid.cuda(), dev[4], dev[5], eps)
    _assert(rep32, o32, ln if f32_is_ln else v, 'linear-ln-f32-' + ('ln' if f32_is_ln else 'v'))
    _assert(rep16, o16, ln, 'linear-ln-f16')


def test_layernorm_fused_mirror(ops):
    """The same cases with PE_FUSE_LN=1 (child process): the chunked stand-alone kernel for the widths the fused
    projection supports, the two-pass kernel for the others."""
    _child('layernorm', {'PE_FUSE_LN': '1'})
