"""QuantPipe conformance: case lists, expected outputs and NumPy mutants for the encode / send / decode kernels.

No GPU needed. The expected outputs come from `oracle/quant.py` (the NumPy restatement of the reference, itself pinned
to the reference by `tests/golden/quant*.npz`). The GPU tests (`test_quant_conformance_gpu.py`) hold the stand-alone
kernels (`pe_quant_encode` / `pe_quant_alpha` / `pe_quant_decode`) and a loop-back link (`pe_link_put` /
`pe_link_get`) to those outputs bit for bit. The CPU tests (`test_quant_ref_cpu.py`) show that the cases reach every
bit-width, rounding tie, code value and send path, and that each mutant - a plausible wrong kernel restated in NumPy -
differs from the oracle on at least one case.
"""
import collections
import ctypes
import functools
import math

import numpy as np
import torch

from oracle import quant as oq

BITS = tuple(range(1, 17))
PACK16 = (2, 4, 8, 16)          # widths with a 16-value pack kernel and a fused send kernel
CLAMP = {'none': 0, 'auto': 1, 'laplace': 2, 'gelu': 3}   # PE_CLAMP_*
QUANT_CACHE_BYTES = 160 * 1024  # shared memory a CTA of the fused send kernel may keep its fp32 slice in
MAX_CHUNKS = 64                 # segments per item of the fused send kernel (kQMaxChunks)
MAX_ITEMS = 512                 # items a link slot header has room for
HDR = 16384                     # PE_LINK_HEADER_BYTES
F32_02 = np.float32(0.2)        # the Laplace / GeLU switch of the runtime hook: min(x) < 0.2


def ratio(bit):
    """Codes per uint32 word."""
    return 32 // bit


def levels(bit):
    return (1 << bit) - 1


# --------------------------------------------------------------------------------------------------- value kinds
@functools.lru_cache(maxsize=None)
def tie_values(bit):
    """fp32 values v in (0, S) for which levels * (v / S), evaluated in fp32 as the kernels do, is exactly k + 1/2,
    for S in {levels, 1, 3.7} and k among the lowest 512 and highest 128 codes. Returns [(S, [(v, k), ...]), ...]:
    both parities of k wherever both exist."""
    out = []
    lv = np.float32(levels(bit))
    ks = sorted(set(range(min(levels(bit), 512))) | set(range(max(0, levels(bit) - 128), levels(bit))))
    for s in (np.float32(levels(bit)), np.float32(1.0), np.float32(3.7)):
        found = []
        for k in ks:
            want = k + 0.5
            v0 = np.float32(want * float(s) / float(lv))
            for v in (v0, np.nextafter(v0, np.float32(0)), np.nextafter(v0, np.float32(np.inf))):
                if 0 < v < s and float(lv * np.float32(v / s)) == want:
                    found.append((np.float32(v), k))
                    break
        out.append((s, found))
    return out


def ramp_values(bit):
    """0, 1, ..., levels as fp32: with shift 0 and scale levels, value c quantises to code c."""
    return np.arange(levels(bit) + 1, dtype=np.float32)


def _fill(vals, n, rng):
    """`vals` (which must keep their min and max) repeated / permuted to exactly n values."""
    vals = np.asarray(vals, dtype=np.float32)
    reps = np.resize(vals, max(n, len(vals)))[:n]
    return rng.permutation(reps).astype(np.float32)


def _guard_item(n, big, rng):
    """An item of +-big: it sets a Laplace threshold well above the other items' range, so that they are not clamped."""
    return (np.where(rng.random(n) < 0.5, -big, big)).astype(np.float32)


Case = collections.namedtuple('Case', 'bit kind items n offset clamp seed')


def case_id(c):
    return f"b{c.bit}-{c.kind}-i{c.items}-n{c.n}-o{c.offset}-{c.clamp}"


def make_input(c):
    """The case's fp32 input [items, n]."""
    rng = np.random.default_rng(c.seed)
    shape = (c.items, c.n)
    if c.kind in ('normal', 'outliers', 'constant_item', 'subnormal'):
        x = (rng.standard_normal(shape) * 1.3 + 0.1).astype(np.float32)
        if c.kind == 'outliers':
            x[0, :3] = np.array([40.0, -35.0, 12.0], np.float32)[:c.n]
        elif c.kind == 'constant_item':
            x[1] = np.float32(0.75)
        elif c.kind == 'subnormal':
            x[1] = (rng.random(c.n) * 1e-38).astype(np.float32)     # differences of a few ulp of the subnormal range
            x[1, 0], x[1, -1] = np.float32(0.0), np.float32(1e-38)
        return x
    if c.kind == 'clamped_item':
        # item 0 entirely above the Laplace threshold: it clamps to the constant +alpha (scale 0); its weight
        # 1 / items in the variance keeps alpha below it at every bit-width
        x = (rng.standard_normal(shape) * 1.3 + 0.1).astype(np.float32)
        x[0] = np.float32(1000.0) + rng.random(c.n).astype(np.float32)
        return x
    if c.kind in ('branch_gelu', 'branch_laplace'):
        x = (rng.random(shape) * 3 + 0.25).astype(np.float32)
        x[0, 0] = F32_02 if c.kind == 'branch_gelu' else np.nextafter(F32_02, np.float32(0))
        return x
    if c.kind in ('ties', 'ramp'):
        if c.kind == 'ties':
            s, found = tie_values(c.bit)[c.seed % 3]
            vals = [np.float32(0.0), s] + [v for v, _ in found]
        else:
            s = np.float32(levels(c.bit))
            vals = ramp_values(c.bit)
        x = np.empty(shape, np.float32)
        x[0] = _fill(vals, c.n, rng)
        for i in range(1, c.items):
            x[i] = _guard_item(c.n, np.float32(100.0) * s, rng)
        return x
    raise ValueError(c.kind)


# --------------------------------------------------------------------------------------------------- expected output
Expected = collections.namedtuple('Expected', 'codes scale shift alpha dec kind')


def oracle_alpha(x: np.ndarray, bit: int, clamp: str):
    """(alpha, branch) the oracle's clamp picks for mode `clamp` (alpha = +inf, branch None without a clamp)."""
    if clamp == 'none':
        return np.float32(np.inf), None
    return oq.clamp_alpha(torch.from_numpy(x), bit, None if clamp == 'auto' else clamp)


def ieee_alpha(x: np.ndarray, bit: int, clamp: str):
    """The oracle's Laplace threshold with the same fp32 variance, but its sqrt correctly rounded (IEEE, as the kernels'
    __fsqrt_rn). torch's CPU sqrt of an fp32 scalar is occasionally one ulp off; where it is, the kernels and the
    oracle differ by that ulp and by nothing else."""
    xt = torch.from_numpy(x)
    var = np.float32(torch.var(xt, unbiased=False).item())
    factor = oq.clamp_factor_laplace(bit)
    return np.float32(factor * np.sqrt(np.float32(np.float32(0.5) * var)))


def torch_sqrt_misrounds(v) -> bool:
    """torch's CPU fp32 sqrt of v differs from the correctly rounded one."""
    v = np.float32(v)
    return np.float32(torch.sqrt(torch.tensor(v)).item()) != np.sqrt(v)


def expected(x: np.ndarray, bit: int, alpha) -> Expected:
    """Oracle codes (u8 [items, 4 * words]), scale, shift and decoded values for x clamped at `alpha`."""
    enc = oq.encode_given_alpha(torch.from_numpy(x), bit, alpha)
    dec = oq.tensor_decode_outerdim(enc).numpy()
    return Expected(enc[0].numpy(), enc[2].numpy(), enc[3].numpy(), np.float32(alpha), dec, None)


# --------------------------------------------------------------------------------------------------- case lists
def standalone_shapes(bit):
    """(n, offset) per bit: n mod ratio in {0, 1, ratio - 1}, n < ratio, n % 16 != 0 with whole words for the pack16
    widths, and a base pointer 1-3 floats past 16-byte alignment."""
    r = ratio(bit)
    base = 32 * r                       # a multiple of 16 and of the ratio
    ns = [base, base + 1, base + r - 1, max(1, r - 1), 1]
    if bit in PACK16 and r < 16:
        ns.append(base + 8)             # whole words, but not whole 16-value groups
    out, seen = [], set()
    for n in ns:
        if n not in seen:
            seen.add(n)
            out.append((n, 0))
    out.append((base, 1 + bit % 3))
    return out


def standalone_cases():
    cases = []
    for bit in BITS:
        for j, (n, off) in enumerate(standalone_shapes(bit)):
            for kind in ('normal', 'outliers'):
                clamp = ('auto', 'none', 'laplace', 'gelu')[(j + (kind == 'outliers')) % 4]
                cases.append(Case(bit, kind, 3, n, off, clamp, 1000 * bit + 10 * j + (kind == 'outliers')))
        base = 32 * ratio(bit)
        cases.append(Case(bit, 'outliers', 16, max(base, 256), 0, 'auto', 1000 * bit + 99))   # enough values to clamp
        for seed in range(3):                                  # the three scales S of tie_values
            cases.append(Case(bit, 'ties', 2, max(64, 4 * len(tie_values(bit)[seed][1]) + 3), 0, 'auto', seed))
        cases.append(Case(bit, 'ramp', 2, levels(bit) + 1 + (bit % 3), 0, 'auto', 7))
        cases.append(Case(bit, 'constant_item', 3, base + 1, 0, 'auto', 11))
        cases.append(Case(bit, 'clamped_item', 320, 32, 0, 'auto', 12))
        cases.append(Case(bit, 'subnormal', 3, base, 0, 'auto', 13))
        cases.append(Case(bit, 'subnormal', 3, base, 0, 'none', 14))
        cases.append(Case(bit, 'branch_gelu', 2, base, 0, 'auto', 15))
        cases.append(Case(bit, 'branch_laplace', 2, base, 0, 'auto', 16))
    return cases


# --------------------------------------------------------------------------------------------------- link plans
LinkPlan = collections.namedtuple('LinkPlan', 'path grid chunks per cache')
PATHS = {0: 'copy', 1: 'fused', 2: 'staged'}   # PE_LINK_PATH_*


def link_plan(lib, items, n, bit, aligned=True):
    """pe_debug_link_put_plan: how pe_link_put ships one tensor on this device (132 SMs without one)."""
    out = (ctypes.c_int * 5)()
    lib.check(lib.LIB.pe_debug_link_put_plan(items, n, bit, 1 if aligned else 0, out))
    return LinkPlan(PATHS[out[0]], *out[1:])


def plan_kind(p, items):
    """What a plan exercises: 'copy', 'staged', 'fused-cached-1seg', 'fused-cached-multiseg', 'fused-stream', plus
    '-cap' when the chunks of an item hit MAX_CHUNKS."""
    if p.path != 'fused':
        return p.path
    segs_per_cta = -(-items * p.chunks // p.grid)
    kind = 'fused-stream' if not p.cache else ('fused-cached-1seg' if segs_per_cta == 1 else 'fused-cached-multiseg')
    return kind + ('-cap' if p.chunks == MAX_CHUNKS else '')


def get_fast_path(bit, n):
    """link_get_kernel decodes 4 words per thread when whole 4-word groups cover every item (else word by word)."""
    r = ratio(bit)
    return r % 4 == 0 and n % r == 0 and (-(-n // r)) % 4 == 0


def link_shapes(lib):
    """(role, items, n, bit) for the fused send kernel's plans, derived from the plan query so that every SM count
    reaches them: slice cached with one and with several segments per CTA, slice streamed from HBM, the 64-chunk cap,
    items in {1, max_ctas, max_ctas + 1, 512}."""
    max_ctas = link_plan(lib, MAX_ITEMS, 16, 8).grid           # one segment per item, as many CTAs as the kernel uses
    stream_n = 16 * (QUANT_CACHE_BYTES // (2 * 4 * 16) + 1)    # two such segments per CTA overflow the cache
    cap_n = 4096 * MAX_CHUNKS + 4096 + 16                       # one item needs more than 64 chunks of 4096
    return [('cached-1seg', 4, 8 * 4096, 8),
            ('items-1', 1, 4 * 4096, 4),
            ('items-maxctas', max_ctas, 64, 2),
            ('items-maxctas+1', max_ctas + 1, 64, 16),
            ('items-512', MAX_ITEMS, 64, 8),
            ('stream', max_ctas + 1, stream_n, 8),
            ('chunk-cap', 1, cap_n, 4),
            ('baseline-c5', 32, 198 * 768, 8)]


# --------------------------------------------------------------------------------------------------- mutants
def model(x: np.ndarray, bit: int, alpha, *, rounding='half_even', pack='lsb', tail='zero', decode='two_roundings',
          alpha_scope='tensor', lv='reference', unit='divide'):
    """An independent NumPy restatement of encode + decode with the kernels' plausible mistakes as switches; with the
    defaults it equals the oracle (asserted by the CPU tests). Returns (codes u8 [items, 4 * words], scale, shift,
    decoded)."""
    items, n = x.shape
    r = ratio(bit)
    words = -(-n // r)
    codes_out = np.zeros((items, words), np.uint32)
    scales = np.zeros(items, np.float32)
    shifts = np.zeros(items, np.float32)
    dec = np.zeros_like(x)
    for i in range(items):
        a = alpha
        if alpha_scope == 'item' and not math.isinf(float(alpha)):
            a, _ = oq.clamp_alpha(torch.from_numpy(x[i:i + 1].copy()), bit)
        a = np.float32(a)
        xc = np.minimum(np.maximum(x[i], -a), a)
        shift = xc.min()
        scale = np.float32(xc.max() - shift)
        if lv == 'reference':
            L = np.float32(levels(bit))
        else:                              # the reference's unused 'modified' mode: 2^bit levels, floor, clip
            L = np.float32(1 << bit)
        with np.errstate(invalid='ignore', divide='ignore'):
            v = L * ((xc - shift) / scale)
        v = np.nan_to_num(v, nan=0.0)      # scale 0: zero codes
        if lv != 'reference':
            q = np.clip(np.floor(v), 0, (1 << bit) - 1)
        elif rounding == 'half_even':
            q = np.rint(v)
        else:
            q = np.floor(v.astype(np.float64) + 0.5)
        q = q.astype(np.uint32)
        padded = np.zeros(words * r, np.uint32)
        padded[:n] = q
        if tail == 'garbage':
            padded[n:] = levels(bit)
        g = padded.reshape(words, r)
        pos = np.arange(r, dtype=np.uint32) if pack == 'lsb' else np.arange(r - 1, -1, -1, dtype=np.uint32)
        codes_out[i] = np.bitwise_or.reduce(np.left_shift(g, pos * np.uint32(bit)), axis=1)
        div = float(levels(bit)) if lv == 'reference' else float(1 << bit)
        if unit == 'divide':
            u = (q / div).astype(np.float32)
        else:                              # an fp32 reciprocal, as a kernel that avoids the divide would compute it
            u = q.astype(np.float32) * (np.float32(1) / np.float32(div))
        if decode == 'two_roundings':
            dec[i] = u * scale + shift
        else:
            dec[i] = (u.astype(np.float64) * np.float64(scale) + np.float64(shift)).astype(np.float32)
        scales[i], shifts[i] = scale, shift
    return codes_out.view(np.uint8).reshape(items, 4 * words), scales, shifts, dec


MUTANTS = {
    'round_half_away': dict(rounding='half_away'),
    'pack_msb_first': dict(pack='msb'),
    'tail_garbage': dict(tail='garbage'),
    'decode_one_fma': dict(decode='fma'),
    'alpha_per_item': dict(alpha_scope='item'),
    'levels_2pow_bit': dict(lv='modified'),
    'unit_times_reciprocal': dict(unit='reciprocal'),
}


def differs(exp: Expected, got) -> bool:
    codes, scale, shift, dec = got
    return not (np.array_equal(codes, exp.codes) and np.array_equal(scale, exp.scale) and
                np.array_equal(shift, exp.shift) and np.array_equal(dec.view(np.uint32), exp.dec.view(np.uint32)))
