"""fp64 references, error-bound checkers and case lists for the kernel conformance tests.

No GPU needed: everything here is plain torch maths that runs on whatever device its tensors live on. The GPU tests
(`test_kernel_conformance_gpu.py`) compare each kernel with a restatement of the same operation in fp64 on the same
fp16 / fp32 operands, element by element, against an error bound derived from the operation rather than a flat
tolerance. The CPU tests (`test_fp_ref_cpu.py`) show that each checker rejects plausible wrong kernels.

Bounds (u = 2^-24, the fp32 unit roundoff):
  * fp32 GEMM outputs: |got - ref| <= C u (sum_k |a_ik w_jk| + |b_j| + |resid_ij|) + 2 u sum_s |S_ij(s)|, S(s) the exact
    partial sum after k-step s of K_STEP products (`gemm_ref`).
  * tanh epilogue: the same, propagated through tanh, plus 2 ulp of fp32 (CUDA's documented tanhf accuracy).
  * fp16 outputs: `got` is one of the two fp16 neighbours of some exact value within the fp32 bound ("faithful").
"""
import collections
import ctypes
import math
import os

import torch

U32 = 2.0 ** -24
# One constant for every GEMM shape, plan and epilogue: the error of summing one wgmma instruction's products into the
# accumulator plus the epilogue's few roundings, in units of u * sum |a w|. Calibrated on an H100 (see the commit that
# introduced it) at K <= 776.
C_GEMM = 16.0
# k per wgmma instruction. The tensor cores add each instruction's 16 products to the fp32 accumulator with one
# rounding that is not to nearest (it truncates): its errors do not cancel, they pile up with the number of
# instructions, each at most 2 u of the partial sum it produces. With operands whose dot products drift one way (FC2
# reads GELU outputs, which are mostly positive) that term grows about linearly in K: measured on an H100 SXM (700 W),
# ViT-L's FC2 (K = 4096) reached 1.05 x the C u sum|a w| bound on 2 of 3.2 million outputs; with this term no
# product GEMM of K >= 3072 comes above 0.30 x the bound.
K_STEP = 16

# epilogue ids, in the order of PE_EPI_* in include/pipeedge_b200.h (asserted by the tests)
EPI = {'F16': 0, 'GELU_F16': 1, 'RESID_F32': 2, 'F32': 3, 'TANH_F32': 4}
HALF_OUT = ('F16', 'GELU_F16')


# --------------------------------------------------------------------------------------------------- fp16 rounding
def _step16(h: torch.Tensor, up: bool) -> torch.Tensor:
    """The fp16 value next to `h` (fp16) towards +inf (`up`) or -inf; +-inf and NaN stay."""
    bits = h.view(torch.int16).to(torch.int32) & 0xFFFF
    sign, mag = bits & 0x8000, bits & 0x7FFF
    away = (sign == 0) if up else (sign != 0)          # moving away from zero grows the magnitude
    new_mag = torch.where(away, mag + 1, mag - 1)
    new_sign = sign
    zero = mag == 0
    new_mag = torch.where(zero, torch.ones_like(mag), new_mag)
    new_sign = torch.where(zero, torch.zeros_like(sign) if up else torch.full_like(sign, 0x8000), new_sign)
    keep = (mag >= 0x7C00) & (away | (mag > 0x7C00))   # +inf up, -inf down, NaN
    out = torch.where(keep, bits, new_sign | new_mag)
    return torch.where(out >= 0x8000, out - 0x10000, out).to(torch.int16).view(torch.float16)


def f16_down(x: torch.Tensor) -> torch.Tensor:
    """Largest fp16 <= x (x float64), as float64 (-inf below -65504)."""
    h = x.to(torch.float16)          # may round twice (via fp32), but always lands on one of x's two fp16 neighbours
    return torch.where(h.double() > x, _step16(h, up=False), h).double()


def f16_up(x: torch.Tensor) -> torch.Tensor:
    """Smallest fp16 >= x (x float64), as float64."""
    h = x.to(torch.float16)
    return torch.where(h.double() < x, _step16(h, up=True), h).double()


def f16_nearest(x: torch.Tensor) -> torch.Tensor:
    """x (float64) correctly rounded to fp16 (ties to even), as float64: no double rounding through fp32."""
    lo, hi = f16_down(x), f16_up(x)
    dlo, dhi = x - lo, hi - x
    lo_even = (lo.to(torch.float16).view(torch.int16) & 1) == 0
    pick_lo = (dlo < dhi) | ((dlo == dhi) & lo_even)
    out = torch.where(pick_lo, lo, hi)
    return torch.where(x.abs() >= 65520.0, torch.copysign(torch.full_like(x, math.inf), x), out)   # overflow


def ulp16(x: torch.Tensor) -> torch.Tensor:
    """Spacing of fp16 above |x| (x float64), as float64 (inf beyond 65504)."""
    a = f16_down(x.abs())
    return _step16(a.to(torch.float16), up=True).double() - a


def ulp32(y: torch.Tensor) -> torch.Tensor:
    """Spacing of fp32 above |y| (float64 in, float64 out)."""
    a = y.abs().float()
    return (torch.nextafter(a, torch.full_like(a, math.inf)) - a).double()


# ------------------------------------------------------------------------------------------------------ reports
class Report:
    """Outcome of one element-wise check: which elements passed, how close the worst came to its bound (`ratio`) and,
    for fp16 outputs, the fraction that is the correctly rounded value of the fp64 reference.

    fp32 outputs: ratio = |got - ref| / bound (<= 1 passes). fp16 outputs: ratio = |got - ref| / (widest distance from
    ref to the edge of the exact interval + one fp16 ulp at ref); a faithful result stays <= 1, a correctly rounded one
    with an exact interval <= 0.5. Pass / fail for fp16 is faithfulness itself (`check_f16`)."""

    def __init__(self, ok, ratio, correctly_rounded=None, where=''):
        self.ok = ok
        self.ratio = ratio
        self.correctly_rounded = correctly_rounded
        self.where = where

    @property
    def passed(self) -> bool:
        return bool(self.ok.all())

    @property
    def max_ratio(self) -> float:
        r = self.ratio[torch.isfinite(self.ratio)]
        return float(r.max()) if r.numel() else 0.0

    def describe(self, got, ref, limit=6) -> str:
        bad = (~self.ok).nonzero()
        lines = [f"{self.where}: {bad.shape[0]} of {self.ok.numel()} elements outside the bound "
                 f"(max err/bound {self.max_ratio:.3g})"]
        for idx in bad[:limit].tolist():
            idx = tuple(idx)
            lines.append(f"  at {idx}: got {float(got[idx])!r} ref {float(ref[idx])!r}")
        return '\n'.join(lines)


def _ratio16(got, ref, lo, hi):
    """|got - ref| in units of (interval half-width + one fp16 ulp at ref); lo <= ref <= hi."""
    err = (got - ref).abs()
    scale = torch.maximum(ref - lo, hi - ref) + ulp16(ref)
    return torch.where(err == 0, torch.zeros_like(err), err / scale.clamp_min(1e-300))


def check_f32(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, where='') -> Report:
    """fp32 output: |got - ref| <= bound, NaN never passes, +-inf only where ref is the same inf."""
    g = got.double()
    err = (g - ref).abs()
    ok = (err <= bound) | ((g == ref) & torch.isinf(ref))
    ok &= ~torch.isnan(g)
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound.clamp_min(1e-300))
    return Report(ok, ratio, None, where)


def check_f16(got: torch.Tensor, ref: torch.Tensor, lo: torch.Tensor, hi: torch.Tensor, where='') -> Report:
    """fp16 output faithful to some exact value in [lo, hi] (float64): f16_down(lo) <= got <= f16_up(hi).
    `ref` (inside [lo, hi]) is the fp64 value the correctly-rounded fraction refers to."""
    g = got.double()
    elo, ehi = f16_down(lo), f16_up(hi)
    ok = (g >= elo) & (g <= ehi) & ~torch.isnan(g)
    cr = float((g == f16_nearest(ref)).double().mean()) if g.numel() else 1.0
    return Report(ok, _ratio16(g, ref, lo, hi), cr, where)


# ------------------------------------------------------------------------------------------ GEMM + epilogues
def gelu64(x: torch.Tensor) -> torch.Tensor:
    """x Phi(x) in fp64 (erfc form: accurate on the negative tail)."""
    return 0.5 * x * torch.special.erfc(-x / math.sqrt(2.0))


def gelu_tanh64(x: torch.Tensor) -> torch.Tensor:
    """The tanh approximation of GELU (what a kernel must NOT compute for nn.GELU())."""
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


_GELU_XMIN = -0.7517915246  # argmin of x Phi(x)


def _gelu_range(lo, hi):
    """min / max of x Phi(x) over [lo, hi] (GELU is decreasing below _GELU_XMIN, increasing above)."""
    glo, ghi = gelu64(lo), gelu64(hi)
    inside = (lo <= _GELU_XMIN) & (hi >= _GELU_XMIN)
    gmin = torch.where(inside, torch.full_like(lo, float(gelu64(torch.tensor(_GELU_XMIN, dtype=torch.float64)))),
                       torch.minimum(glo, ghi))
    return gmin, torch.maximum(glo, ghi)


def partial_sums_magnitude(ad, wd, step=K_STEP):
    """sum over the k-steps s of |S(s)|, S(s) = the exact a w^T over k < step * (s + 1) (float64 operands)."""
    s = torch.zeros(ad.shape[0], wd.shape[0], dtype=torch.float64, device=ad.device)
    total = torch.zeros_like(s)
    for k0 in range(0, ad.shape[1], step):
        s += ad[:, k0:k0 + step] @ wd[:, k0:k0 + step].t()
        total += s.abs()
    return total


def gemm_ref(a16, w16, bias, resid):
    """(pre-activation x = a w^T + bias in fp64, magnitude sum|a w| + |bias| + |resid|) on the operands' device."""
    ad, wd = a16.double(), w16.double()
    x = ad @ wd.t()
    mag = ad.abs() @ wd.abs().t()
    if bias is not None:
        x = x + bias.double()
        mag = mag + bias.double().abs()
    if resid is not None:
        mag = mag + resid.double().abs()
    return x, mag


def gemm_bound(a16, w16, mag, c=C_GEMM):
    """The fp32 error bound of a GEMM output: C u per unit of `mag` (from gemm_ref) plus the truncating accumulation
    of one wgmma instruction after the other (2 u of every partial sum, see K_STEP)."""
    return c * U32 * mag + 2 * U32 * partial_sums_magnitude(a16.double(), w16.double())


def check_gemm(epi: str, got, a16, w16, bias=None, resid=None, c=C_GEMM, where='') -> Report:
    """Check one pe_linear output. `resid` is the residual as it was BEFORE the call (for in-place RESID_F32)."""
    x, mag = gemm_ref(a16, w16, bias, resid if epi == 'RESID_F32' else None)
    bound = gemm_bound(a16, w16, mag, c)
    if epi == 'F32':
        return check_f32(got, x, bound, where)
    if epi == 'RESID_F32':
        return check_f32(got, x + resid.double(), bound, where)
    if epi == 'TANH_F32':
        ref = torch.tanh(x)
        lo, hi = torch.tanh(x - bound), torch.tanh(x + bound)
        slack = 2 * ulp32(ref)
        width = torch.maximum(ref - lo, hi - ref) + slack
        return check_f32(got, ref, width, where)
    if epi == 'F16':
        return check_f16(got, x, x - bound, x + bound, where)
    if epi == 'GELU_F16':
        lo, hi = _gelu_range(x - bound, x + bound)
        return check_f16(got, gelu64(x), lo, hi, where)
    raise ValueError(epi)


# exhaustive-ish scan of the activations: a[:, 0] = h, w[:, 0] = 1, all else 0 -> pre-activation exactly fl32(h + b)
SCAN_BIAS = [0.0, 1e-40, -1e-40, 1e-30, -1e-30, 0.3337, -0.1234567, 2.0 ** -20 * 0.37]


def scan_inputs(lo=-12.0, hi=12.0):
    """Every fp16 value in [lo, hi] (both zeros included) as the column h, and the SCAN_BIAS row."""
    bits = torch.arange(0, 0x10000, dtype=torch.int32)
    h = torch.where(bits >= 0x8000, bits - 0x10000, bits).to(torch.int16).view(torch.float16)
    h = h[torch.isfinite(h) & (h.float() >= lo) & (h.float() <= hi)]
    return h, torch.tensor(SCAN_BIAS, dtype=torch.float32)


def scan_preact(h16, bias32):
    """fl32(h + b) as float64, [len(h), len(b)]."""
    return (h16.double()[:, None] + bias32.double()[None, :]).float().double()


def check_gelu_scan(got16, x) -> Report:
    """GELU_F16 on exact pre-activations: faithful fp16 rounding of x Phi(x)."""
    g = gelu64(x)
    return check_f16(got16, g, g, g, 'gelu scan')


def check_tanh_scan(got32, x) -> Report:
    ref = torch.tanh(x)
    return check_f32(got32, ref, 2 * ulp32(ref), 'tanh scan')


# ------------------------------------------------------------------------------------------------ GEMM cases
GemmCase = collections.namedtuple('GemmCase', 'name m n k epi bias force inplace expect')

RAGGED_M = (1, 63, 64, 65, 127, 128, 129, 1000)
RAGGED_N = (1, 3, 12, 31, 33, 100, 257, 1000)
RAGGED_K = (8, 24, 72, 776)
FORCED_PLANS = ('1,1,32', '1,1,160', '2,1,64', '1,2,128', '2,2,128', '1,4,64', '4,1,128', '1,8,32')
SCHED_SHAPE = (1100, 1080, 776)      # 9 M blocks (odd), ragged K; N blocks odd for BN 128, not a multiple of 4 / 8 for 64 / 32


def plan_geometry(plan6, m, n, k):
    """pe_debug_gemm_plan's {cm, cn, block_n, stages, tiles, ctas} -> what decides the kernel's path: the cluster and
    tile shape, the tiles of the busiest CTA (`rounds`; more than one puts the epilogue staging behind the ring instead
    of aliasing it), partly empty clusters, the scalar epilogue, the ring depth, a K loop shorter than the ring
    (`kb_lt_stages`) and whether every tile starts on ring slot 0 with the same barrier phase (`ring_repeats`:
    k-blocks a multiple of the depth; otherwise a CTA's later tiles start mid-ring, or on the other phase)."""
    cm, cn, bn, stages, tiles, ctas = plan6
    mb, nb = -(-m // 128), -(-n // bn)
    kb = -(-k // 64)
    supers = -(-mb // cm) * -(-nb // cn)
    clusters = ctas // (cm * cn)
    rounds = -(-supers // clusters)
    return {'cm': cm, 'cn': cn, 'bn': bn, 'rounds': rounds, 'partial_m': mb % cm != 0,
            'partial_n': nb % cn != 0, 'scalar': n % 8 != 0, 'tiles': tiles, 'stages': stages, 'kb': kb,
            'multi_round': rounds > 1, 'kb_lt_stages': kb < stages, 'ring_repeats': kb % stages == 0}


def _ragged_cases():
    cases = []
    for epi, e in EPI.items():
        for with_bias in (True, False):
            b = int(with_bias)
            for i, m in enumerate(RAGGED_M):
                n = RAGGED_N[(i + 3 * e + b) % len(RAGGED_N)]
                k = RAGGED_K[(i + e + 2 * b) % len(RAGGED_K)]
                expect = {'scalar': n % 8 != 0, 'rounds': 1, 'cm': 1, 'cn': 1}
                cases.append(GemmCase(f"ragged-{epi}-{'bias' if with_bias else 'nobias'}-{m}x{n}x{k}", m, n, k, epi,
                                      with_bias, None, False, expect))
    return cases


def _schedule_cases():
    cases = []
    m, n, k = SCHED_SHAPE
    for epi in EPI:
        inplace = epi == 'RESID_F32'
        cases.append(GemmCase(f'natural-one-round-{epi}', m, n, k, epi, True, None, inplace,
                              {'rounds': 1, 'cm': 1, 'cn': 1, 'scalar': False}))
        cases.append(GemmCase(f'natural-multi-round-{epi}', 4096, 3072, 768, epi, True, None, inplace,
                              {'rounds_gt': 1, 'cm': 1, 'cn': 1, 'scalar': False}))
        for plan in FORCED_PLANS:
            cm, cn, bn = (int(v) for v in plan.split(','))
            expect = {'cm': cm, 'cn': cn, 'bn': bn, 'scalar': False,
                      'partial_m': cm > 1 and -(-m // 128) % cm != 0, 'partial_n': cn > 1 and -(-n // bn) % cn != 0}
            cases.append(GemmCase(f'forced-{plan}-{epi}', m, n, k, epi, True, plan, inplace, expect))
    return cases


RAGGED_CASES = _ragged_cases()
SCHEDULE_CASES = _schedule_cases()


def query_geometry(lib, m, n, k, epi, force=None) -> dict:
    """The plan geometry pe_debug_gemm_plan (host-only) reports for one shape, under PE_GEMM_FORCE = `force` (if any)."""
    out = (ctypes.c_int * 6)()
    old = os.environ.pop('PE_GEMM_FORCE', None)
    try:
        if force:
            os.environ['PE_GEMM_FORCE'] = force
        lib.check(lib.LIB.pe_debug_gemm_plan(m, n, k, EPI[epi], out))
    finally:
        os.environ.pop('PE_GEMM_FORCE', None)
        if old is not None:
            os.environ['PE_GEMM_FORCE'] = old
    return plan_geometry(list(out), m, n, k)


def query_plan(lib, case) -> dict:
    """The plan geometry of `case` (a GemmCase, or anything with m, n, k, epi, force), under its PE_GEMM_FORCE."""
    return query_geometry(lib, case.m, case.n, case.k, case.epi, case.force)


def expectation_failures(case: GemmCase, geom: dict):
    """The properties a case's name claims that its plan does not have (empty list = the case runs its path)."""
    bad = []
    for key, want in case.expect.items():
        if key == 'rounds_gt':
            if not geom['rounds'] > want:
                bad.append(f"rounds {geom['rounds']} not > {want}")
        elif geom[key] != want:
            bad.append(f"{key} {geom[key]} != {want}")
    return bad


def gemm_operands(case: GemmCase, seed: int):
    gen = torch.Generator().manual_seed(seed)
    a = torch.randn(case.m, case.k, generator=gen).half()
    w = (torch.randn(case.n, case.k, generator=gen) * (2.0 / math.sqrt(case.k))).half()
    bias = torch.randn(case.n, generator=gen) if case.bias else None
    resid = torch.randn(case.m, case.n, generator=gen) * 2
    return a, w, bias, resid


# ------------------------------------------------------------------------------------------------- attention
ATTN_TOKENS = (1, 17, 31, 32, 33, 63, 64, 65, 128, 197, 198, 223, 225, 255, 256, 257, 300, 511, 512)
ATTN_KINDS = ('mask', 'rescale_first', 'rescale_last', 'uniform', 'readout', 'large')


def attention_kind_applies(kind: str, tokens: int, head_dim: int) -> bool:
    if kind == 'readout':
        return tokens <= 64 and tokens <= head_dim
    if kind == 'rescale_first':
        return tokens > 1
    return True


def attention_case(kind: str, batch: int, tokens: int, heads: int, head_dim: int, seed: int) -> torch.Tensor:
    """qkv fp16 [batch*tokens, 3*heads*head_dim] for one of ATTN_KINDS."""
    gen = torch.Generator().manual_seed(seed)
    bh = (batch, heads)
    sq = math.sqrt(head_dim)

    def unit():
        u = torch.randn(*bh, 1, head_dim, generator=gen, dtype=torch.float64)
        return u / u.norm(dim=-1, keepdim=True)

    def noise(scale):
        return scale * torch.randn(*bh, tokens, head_dim, generator=gen, dtype=torch.float64)

    v = torch.randn(*bh, tokens, head_dim, generator=gen, dtype=torch.float64)
    if kind == 'mask':
        # every real logit ~ -30 (q ~ a u, k ~ -a u): an unmasked zero-padded key (logit 0) would take all the weight
        u = unit()
        a = math.sqrt(30.0 * sq)
        q = a * u + noise(0.05)
        k = -a * u + noise(0.05)
    elif kind in ('rescale_first', 'rescale_last'):
        # one key per row >= 30 above the rest; in the first key chunk, or in the last (partial) one
        u = unit()
        q = 7.0 * u + noise(0.1)
        k = noise(0.1)
        hot = 0 if kind == 'rescale_first' else tokens - 1
        k[:, :, hot] = 40.0 * u[:, :, 0]        # logit ~ 7 * 40 / 8 = 35 against ~0
    elif kind == 'uniform':
        # identical K rows: every weight exactly 1 / S; V exactly representable -> O = mean of V per head, pinning
        # 1 / l and that every real key, and only those, reaches P V (check_attention_uniform)
        q = torch.randn(*bh, tokens, head_dim, generator=gen, dtype=torch.float64)
        k = torch.randn(*bh, 1, head_dim, generator=gen, dtype=torch.float64).expand(*bh, tokens, head_dim).clone()
        j = torch.arange(tokens, dtype=torch.float64)[:, None]
        d = torch.arange(head_dim, dtype=torch.float64)[None, :]
        v = (((7 * j + 13 * d) % 64) / 64 - 0.5).expand(*bh, tokens, head_dim).clone()
    elif kind == 'readout':
        # V = identity (tokens <= head_dim): O = P
        q = 1.5 * torch.randn(*bh, tokens, head_dim, generator=gen, dtype=torch.float64)
        k = 1.5 * torch.randn(*bh, tokens, head_dim, generator=gen, dtype=torch.float64)
        v = torch.zeros(*bh, tokens, head_dim, dtype=torch.float64)
        v[:, :, torch.arange(tokens), torch.arange(tokens)] = 1.0
    elif kind == 'large':
        # |q|, |k| up to 60: q = 40 sigma + U(-20, 20), k_j = c_j 40 sigma + U(-20, 20) with a shared sign pattern sigma
        # and c_j in [-1, 1], so q.k ~ c_j * 1600 d and the logits reach ~1e4 (fp32 logit ulp ~1e-3, above half an
        # fp16 ulp of P)
        sigma = torch.where(torch.rand(*bh, 1, head_dim, generator=gen) < 0.5, -1.0, 1.0).double()
        c = 2 * torch.rand(*bh, tokens, 1, generator=gen, dtype=torch.float64) - 1
        q = 40.0 * sigma + 20.0 * (2 * torch.rand(*bh, tokens, head_dim, generator=gen, dtype=torch.float64) - 1)
        k = 40.0 * c * sigma + 20.0 * (2 * torch.rand(*bh, tokens, head_dim, generator=gen, dtype=torch.float64) - 1)
    else:
        raise ValueError(kind)
    hidden = heads * head_dim
    parts = [t.permute(0, 2, 1, 3).reshape(batch * tokens, hidden) for t in (q, k, v)]
    return torch.cat(parts, dim=1).half()


def _split_qkv(qkv16, batch, tokens, heads, head_dim):
    hidden = heads * head_dim
    return [t.double().reshape(batch, tokens, heads, head_dim).permute(0, 2, 1, 3)
            for t in qkv16.split(hidden, dim=1)]


def attention_ref(qkv16, batch, tokens, heads, head_dim, c=C_GEMM):
    """fp64 softmax(Q K^T / sqrt(d)) V and the per-element bound of an fp32 flash-style kernel that rounds P to fp16.

    Error sources, per query row i and output column d:
      logits: S in fp32 (C u sum_d |q k|), times the fp32 scale, exp2f                -> factor e^(2 delta_i) - 1
      P rounded to fp16 (relative 2^-11, absolute 2^-25 below the normal range)       -> 2^-11 sum_j P_ij |V_jd| + ...
      P V accumulated in fp32, row sum l in fp32, 1 / l and the product              -> (2C + 4) u sum_j P_ij |V_jd|
    Returns (ref [B*S, H], lo, hi) in float64; the fp16 output must be faithful to a value in [lo, hi]."""
    q, k, v = _split_qkv(qkv16, batch, tokens, heads, head_dim)
    scale = 1.0 / math.sqrt(head_dim)
    s = q @ k.transpose(-1, -2)
    t = s * scale
    smag = q.abs() @ k.abs().transpose(-1, -2)
    tmax = t.max(dim=-1, keepdim=True).values
    dt = (c * U32 * smag + 4 * U32 * t.abs()) * scale + 4 * U32 * (t.abs() + tmax.abs())
    delta = (dt + dt.gather(-1, t.argmax(dim=-1, keepdim=True))).max(dim=-1, keepdim=True).values
    p = torch.exp(t - tmax)
    l = p.sum(dim=-1, keepdim=True)
    pn = p / l
    o = pn @ v
    pv = pn @ v.abs()
    err = (torch.expm1(2 * delta) + 2.0 ** -11 + (2 * c + 4) * U32) * pv + 2.0 ** -25 / l * v.abs().sum(-2, keepdim=True)

    def merge(x):
        return x.permute(0, 2, 1, 3).reshape(batch * tokens, heads * head_dim)

    return merge(o), merge(o - err), merge(o + err)


def check_attention(got16, qkv16, batch, tokens, heads, head_dim, where='') -> Report:
    ref, lo, hi = attention_ref(qkv16, batch, tokens, heads, head_dim)
    return check_f16(got16, ref, lo, hi, where)


def check_attention_uniform(got16, qkv16, batch, tokens, heads, head_dim, where='') -> Report:
    """Identical K rows: every logit of a row is the same fp32 value, so every p is exp2 of at most the rounding
    residual of the scaled logit (1 within a few fp32 ulps, exactly 1 in fp16) and l = S up to fp32 summation. V is a
    multiple of 1/64, so P V sums exactly. The output must be a faithful fp16 rounding of the exact fp64 mean of V,
    widened only by that fp32 slack: (S + 4 max|logit| + 8) u relative. A row sum that miscounts one key is 1/S off."""
    q, k, v = _split_qkv(qkv16, batch, tokens, heads, head_dim)
    assert bool((k == k[:, :, :1]).all()), 'not a uniform-weights case'
    t = (q @ k.transpose(-1, -2)) / math.sqrt(head_dim)
    mean = v.mean(-2, keepdim=True).expand(batch, heads, tokens, head_dim)
    rel = (tokens + 4 * t.abs().amax(-1, keepdim=True) * math.log2(math.e) + 8) * U32
    err = mean.abs() * rel

    def merge(x):
        return x.permute(0, 2, 1, 3).reshape(batch * tokens, heads * head_dim)

    return check_f16(got16, merge(mean), merge(mean - err), merge(mean + err), where)


def check_attention_readout(got16, qkv16, batch, tokens, heads, head_dim, c=C_GEMM, where='') -> Report:
    """V = identity: output column d < S is the weight of key d, which the kernel computes as fl16(fl32(p_d / l)) with
    p_d = fl16(exp(t_d - max)) rounded to fp16 BEFORE the product with V. The admissible set holds exactly the values
    that rounding can give for p_d anywhere in its logit-error interval: a kernel keeping P in fp32 falls outside."""
    q, k, _ = _split_qkv(qkv16, batch, tokens, heads, head_dim)
    scale = 1.0 / math.sqrt(head_dim)
    t = (q @ k.transpose(-1, -2)) * scale
    smag = q.abs() @ k.abs().transpose(-1, -2)
    tmax = t.max(dim=-1, keepdim=True).values
    dt = (c * U32 * smag + 4 * U32 * t.abs()) * scale + 4 * U32 * (t.abs() + tmax.abs()) + 4 * U32
    dmax = dt.gather(-1, t.argmax(dim=-1, keepdim=True))
    p = torch.exp(t - tmax)
    p_lo, p_hi = p * torch.exp(-(dt + dmax)), (p * torch.exp(dt + dmax)).clamp_max(1.0)
    l = p.sum(-1, keepdim=True)
    l_lo = (p_lo.sum(-1, keepdim=True)) * (1 - tokens * U32)
    l_hi = (p_hi.sum(-1, keepdim=True)) * (1 + tokens * U32)
    h_lo, h_hi = f16_nearest(p_lo), f16_nearest(p_hi)
    lo = h_lo / l_hi * (1 - 3 * U32)
    hi = h_hi / l_lo * (1 + 3 * U32)
    ref = p / l
    pad = torch.zeros(batch, heads, tokens, head_dim - tokens, dtype=torch.float64)

    def merge(x):
        x = torch.cat([x, pad], dim=-1)
        return x.permute(0, 2, 1, 3).reshape(batch * tokens, heads * head_dim)

    return check_f16(got16, merge(ref), merge(lo), merge(hi), where)


# ------------------------------------------------------------------------------------------------- LayerNorm
LN_SUM_DEPTH = 64   # additions any one input passes through in the kernels' mean / variance reductions (upper bound)


def layernorm_ref(x64, gamma, beta, eps, in_err=None, depth=LN_SUM_DEPTH):
    """fp64 LayerNorm over the last dim and a per-element bound for an fp32 kernel that computes the mean and then the
    variance about it (two passes or Chan merges). `in_err` bounds the error of the kernel's own fp32 inputs (e.g. a
    residual add or an embedding sum done in fp32). Returns (ref, bound)."""
    g, b = gamma.double(), beta.double()
    mu = x64.mean(-1, keepdim=True)
    xc = x64 - mu
    var = (xc * xc).mean(-1, keepdim=True)
    r = 1.0 / torch.sqrt(var + eps)
    ein = torch.zeros_like(x64) if in_err is None else in_err
    dmu = depth * U32 * x64.abs().mean(-1, keepdim=True) + ein.mean(-1, keepdim=True)
    dvar = dmu ** 2 + (depth + 3) * U32 * (var + dmu ** 2) + 2 * (xc.abs() * ein).mean(-1, keepdim=True) + U32 * eps
    rel_r = 0.5 * dvar / (var + eps) + 4 * U32
    ec = dmu + ein + U32 * (x64.abs() + mu.abs())
    y = xc * r * g + b
    bound = g.abs() * r * (ec + xc.abs() * rel_r) * (1 + 1e-6) + 3 * U32 * (xc.abs() * r * g.abs() + b.abs())
    return y, bound


def linear_ln_ref(a16, w16, bias, resid, gamma, beta, eps, c=C_GEMM):
    """The fused projection + residual + LayerNorm epilogue (PE_EPI_RESID_LN): v = a w^T + bias + resid in fp64 with the
    bound of the kernel's fp32 v (the GEMM's, the residual counted in the magnitude), and LayerNorm(v) with a bound that
    takes that error as the LayerNorm's input error, plus the rounding of v itself. Returns (v, v_bound, ln, ln_bound)."""
    x, mag = gemm_ref(a16, w16, bias, resid)
    v = x + resid.double()
    v_bound = gemm_bound(a16, w16, mag, c)
    ln, ln_bound = layernorm_ref(v, gamma, beta, eps, in_err=v_bound + U32 * v.abs())
    return v, v_bound, ln, ln_bound


def check_linear_ln(got32, got16, a16, w16, bias, resid, gamma, beta, eps, f32_is_ln, c=C_GEMM, where=''):
    """-> (report of the fp32 output, report of the fp16 output). The fp32 output is LayerNorm(v) when `f32_is_ln`, else
    v held to the GEMM bound; the fp16 output must be a faithful rounding of LayerNorm(v). `resid` is the residual as it
    was BEFORE the call (the kernel may write its fp32 output over it)."""
    v, v_bound, ln, ln_bound = linear_ln_ref(a16, w16, bias, resid, gamma, beta, eps, c)
    if f32_is_ln:
        rep32 = check_f32(got32, ln, ln_bound, where + ' f32 = LayerNorm(v)')
    else:
        rep32 = check_f32(got32, v, v_bound, where + ' f32 = v')
    return rep32, check_f16(got16, ln, ln - ln_bound, ln + ln_bound, where + ' f16')


LN_KINDS = ('normal', 'offset', 'offset_1e4')


def layernorm_case(rows, hidden, kind, seed):
    """'offset': rows 1e3 + N(0, 1), where the fp32 mean keeps enough digits for the bound to mean something (~4e-3
    on outputs of std 1). 'offset_1e4': 1e4 + N(0, 1e-2), where the fp32 mean itself loses most of its digits: the
    bound is then of the order of the output and this kind only catches a variance taken in one pass (E x^2 - mean^2),
    which cancels catastrophically there."""
    gen = torch.Generator().manual_seed(seed)
    if kind == 'offset':
        x = 1e3 + torch.randn(rows, hidden, generator=gen)
    elif kind == 'offset_1e4':
        x = 1e4 + 1e-2 * torch.randn(rows, hidden, generator=gen)
    else:
        x = torch.randn(rows, hidden, generator=gen) * 2.0 + 0.5
    g = 1 + 0.1 * torch.randn(hidden, generator=gen)
    b = 0.1 * torch.randn(hidden, generator=gen)
    return x, g, b
