"""GPU: the QuantPipe kernels bit for bit against the NumPy oracle at every bit-width 1-16, send path and rounding edge.

Stand-alone (`pe_quant_encode`, `pe_quant_alpha`, `pe_quant_decode`, called through the C-ABI so that base pointers can
be misaligned and the clamp forced) and through a loop-back link (`pe_link_put` -> the bytes in the consumer's slot ->
`pe_link_get`): code bytes including the zero padding of the tail word, scale, shift, the clamp threshold alpha and
the decoded fp32 values must equal the oracle's. On the GeLU branch the threshold is only defined up to torch's fp32
summation order, so alpha is held to 2 ulp and the codes to the oracle evaluated at the kernel's own alpha. Each link
case asserts the send plan it runs first (`pe_debug_link_put_plan`). Cases and expected outputs: `_quant_ref.py`.

Run with `-s` to see one summary line per (implementation, path, bit)."""
import collections
import ctypes
import json
import os
import sys

import numpy as np
import pytest
import torch

TESTS = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, TESTS)
import _quant_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = R.standalone_cases()
ROLES = ('cached-1seg', 'items-1', 'items-maxctas', 'items-maxctas+1', 'items-512', 'stream', 'chunk-cap', 'baseline-c5')
ROLE_KIND = {'cached-1seg': 'fused-cached-1seg', 'items-1': 'fused-cached-1seg', 'items-maxctas': 'fused-cached-1seg',
             'items-maxctas+1': 'fused-cached-multiseg', 'items-512': 'fused-cached-multiseg', 'stream': 'fused-stream',
             'chunk-cap': 'fused-cached-1seg-cap'}
_RAN = collections.Counter()


@pytest.fixture(scope='module', autouse=True)
def _summary():
    yield
    for (impl, path, bit), cases in sorted(_RAN.items()):
        print(f"\nQUANT {json.dumps({'impl': impl, 'path': path, 'bit': bit, 'cases': cases})}", end='')
    print()


@pytest.fixture(scope='module')
def lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from pipeedge_b200 import _lib
    return _lib


class Loop:
    """A loop-back link (both ends in this process) and the number of payloads sent through it so far."""

    def __init__(self, lib, payload_bytes):
        self.lib = lib
        self.h = ctypes.c_void_p()
        lib.check(lib.LIB.pe_link_open_local(payload_bytes, 2, 8, ctypes.byref(self.h)))
        self.seq = 0

    def put(self, tensors, items, bit, clamp):
        """tensors: [(a_ptr, b_ptr or None, n)] (one or two)."""
        (a0, b0, n0), (a1, b1, n1) = (tensors + [(None, None, 0)])[:2]
        self.lib.check(self.lib.LIB.pe_link_put(self.h, a0, b0, n0, a1, b1, n1, items, bit, clamp,
                                                torch.cuda.current_stream().cuda_stream))

    def read(self, offset, nbytes, dtype=np.uint8):
        """Bytes of the slot of the payload received last (it stays there until the ring comes round to it again)."""
        buf = (ctypes.c_uint8 * nbytes)()
        self.lib.check(self.lib.LIB.pe_link_debug_read(self.h, self.seq - 1, offset, buf, nbytes))
        return np.frombuffer(buf, dtype=np.uint8).copy().view(dtype)

    def get(self, items, n0, n1=0):
        d0 = torch.empty(items * n0, dtype=torch.float32, device='cuda')
        d1 = torch.empty(items * n1, dtype=torch.float32, device='cuda') if n1 else None
        self.lib.check(self.lib.LIB.pe_link_get(self.h, d0.data_ptr(), None if d1 is None else d1.data_ptr(), items,
                                                n0, n1, torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        self.lib.check(self.lib.LIB.pe_link_check(self.h))
        self.seq += 1
        return d0.cpu().numpy().reshape(items, n0), None if d1 is None else d1.cpu().numpy().reshape(items, n1)


@pytest.fixture(scope='module')
def link(lib):
    lk = Loop(lib, 16 << 20)
    yield lk
    lib.LIB.pe_link_close(lk.h)


def _device(x, offset):
    """x on the GPU starting `offset` floats past a 256-byte aligned allocation; returns (keep-alive, pointer)."""
    buf = torch.zeros(x.size + offset + 4, dtype=torch.float32, device='cuda')
    buf[offset:offset + x.size] = torch.from_numpy(np.ascontiguousarray(x).reshape(-1)).cuda()
    return buf, buf.data_ptr() + 4 * offset


def _kernel_alpha(got, x, bit, clamp):
    """The kernel's threshold against the oracle's: equal on the Laplace branch, within 2 ulp on the GeLU branch."""
    got = np.float32(got)
    want, branch = R.oracle_alpha(x, bit, clamp)
    if clamp == 'none':
        assert np.isposinf(got)
    elif branch == 'laplace':
        if got != want:   # only where torch's fp32 sqrt (in the oracle, as in the reference) misrounds
            half_var = np.float32(0.5) * np.float32(torch.var(torch.from_numpy(x), unbiased=False).item())
            assert R.torch_sqrt_misrounds(half_var) and got == R.ieee_alpha(x, bit, clamp), (float(got), float(want))
    else:
        assert abs(float(got) - float(want)) <= 2 * float(np.spacing(want)), (float(got), float(want))
    return got


def _same(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, what
    if got.dtype == np.float32:
        got, want = got.view(np.uint32), want.view(np.uint32)   # bit patterns: -0.0 != 0.0
    bad = np.flatnonzero(got.reshape(-1) != want.reshape(-1))
    assert bad.size == 0, f"{what}: {bad.size} of {got.size} differ, first at {bad[:5].tolist()}"


def _quant_standalone(lib, ptr, items, n, bit, clamp):
    words = lib.LIB.pe_quant_words(n, bit)
    codes = torch.empty(items * 4 * words, dtype=torch.uint8, device='cuda')
    scale, shift = torch.empty(items, device='cuda'), torch.empty(items, device='cuda')
    alpha = torch.empty(1, device='cuda')
    work = torch.empty(lib.LIB.pe_quant_workspace_bytes(items, n), dtype=torch.uint8, device='cuda')
    stream = torch.cuda.current_stream().cuda_stream
    lib.check(lib.LIB.pe_quant_encode(ptr, items, n, bit, R.CLAMP[clamp], codes.data_ptr(), scale.data_ptr(),
                                      shift.data_ptr(), alpha.data_ptr(), work.data_ptr(), stream))
    scale2, shift2 = torch.empty(items, device='cuda'), torch.empty(items, device='cuda')
    alpha2 = torch.empty(1, device='cuda')
    lib.check(lib.LIB.pe_quant_alpha(ptr, items, n, bit, R.CLAMP[clamp], scale2.data_ptr(), shift2.data_ptr(),
                                     alpha2.data_ptr(), work.data_ptr(), stream))
    out = torch.empty(items * n, device='cuda')
    lib.check(lib.LIB.pe_quant_decode(codes.data_ptr(), items, n, bit, scale.data_ptr(), shift.data_ptr(),
                                      out.data_ptr(), stream))
    torch.cuda.synchronize()
    return (codes.cpu().numpy().reshape(items, 4 * words), scale.cpu().numpy(), shift.cpu().numpy(),
            alpha.cpu().numpy()[0], out.cpu().numpy().reshape(items, n),
            (scale2.cpu().numpy(), shift2.cpu().numpy(), alpha2.cpu().numpy()[0]))


@pytest.mark.parametrize('case', CASES, ids=R.case_id)
def test_standalone_kernels(lib, case):
    c = case
    x = R.make_input(c)
    keep, ptr = _device(x, c.offset)
    codes, scale, shift, alpha, dec, by_alpha = _quant_standalone(lib, ptr, c.items, c.n, c.bit, c.clamp)
    del keep
    a = _kernel_alpha(alpha, x, c.bit, c.clamp)
    exp = R.expected(x, c.bit, a)
    _same(codes, exp.codes, 'codes')
    _same(scale, exp.scale, 'scale')
    _same(shift, exp.shift, 'shift')
    _same(dec, exp.dec, 'decoded')
    _same(by_alpha[0], scale, 'pe_quant_alpha scale')           # the threshold-only entry point agrees
    _same(by_alpha[1], shift, 'pe_quant_alpha shift')
    _same(np.float32(by_alpha[2]), np.float32(alpha), 'pe_quant_alpha alpha')
    pack16 = c.bit in R.PACK16 and c.n % 16 == 0 and c.offset == 0
    _RAN[('standalone', 'pack16' if pack16 else 'generic', c.bit)] += 1


QB = np.load(os.path.join(TESTS, 'golden', 'quant_bits.npz'))


@pytest.mark.parametrize('kind', ['normal', 'outliers', 'ties', 'ramp'])
@pytest.mark.parametrize('bit', [1, 7, 9, 11, 12, 13, 14, 15])
def test_standalone_kernels_vs_reference_goldens(lib, kind, bit):
    """The bytes and values the reference itself produced (`oracle/make_goldens.py quant_bits`) at the widths
    `quant.npz` leaves out."""
    key = f"{kind}_{bit}"
    x = QB[f"x_{key}"]
    items = x.shape[0]
    n = x.size // items
    keep, ptr = _device(x, 0)
    codes, scale, shift, alpha, dec, _ = _quant_standalone(lib, ptr, items, n, bit, 'auto')
    del keep
    _same(codes, QB[f"comm_{key}"], 'codes')
    _same(scale, QB[f"scale_{key}"], 'scale')
    _same(shift, QB[f"shift_{key}"], 'shift')
    _same(dec, QB[f"dec_{key}"].reshape(items, n), 'decoded')
    if np.abs(x).max() > alpha:
        assert np.float32(alpha) == QB[f"alpha_{key}"]


def _check_link_tensor(link, ti, x, bit, clamp, items):
    """Header fields, scale / shift and codes of tensor `ti` of the payload in the current slot vs the oracle."""
    base = 16 + 32 * ti                                        # LinkHeader.t[ti]
    assert link.read(base, 4, np.uint32)[0] == bit
    n = x.shape[1]
    assert link.read(base + 8, 8, np.uint64)[0] == n
    data_off = int(link.read(base + 16, 8, np.uint64)[0])
    a = _kernel_alpha(link.read(base + 24, 4, np.float32)[0], x, bit, clamp)
    exp = R.expected(x, bit, a)
    _same(link.read(256 + 4096 * ti, 4 * items, np.float32), exp.scale, 'slot scale')
    _same(link.read(256 + 4096 * ti + 2048, 4 * items, np.float32), exp.shift, 'slot shift')
    _same(link.read(data_off, exp.codes.size).reshape(exp.codes.shape), exp.codes, 'slot codes')
    return exp


def _send_one(lib, link, x, bit, clamp, offset=0, b=None):
    """x (or the deferred sum x + b) through the link as one quantised tensor; returns the plan it ran."""
    items, n = x.shape
    keep_a, pa = _device(x, offset)
    keep_b, pb = _device(b, offset) if b is not None else (None, None)
    plan = R.link_plan(lib, items, n, bit, aligned=offset == 0)
    want_path = 'fused' if (bit in R.PACK16 and n % 16 == 0 and offset == 0) else 'staged'
    assert plan.path == want_path
    link.put([(pa, pb, n)], items, bit, R.CLAMP[clamp])
    dec, _ = link.get(items, n)   # received before anything is checked: every put is matched by its get
    del keep_a, keep_b
    payload = x if b is None else (x + b).astype(np.float32)   # fp32 add, as the send kernels do
    assert link.read(0, 4, np.uint32)[0] == 0x4b4c4550          # magic
    assert tuple(link.read(4, 8, np.uint32)) == (1, items)
    exp = _check_link_tensor(link, 0, payload, bit, clamp, items)
    _same(dec, exp.dec, 'link decoded')
    return plan


@pytest.mark.parametrize('case', CASES, ids=R.case_id)
def test_link_send_and_receive(lib, link, case):
    c = case
    x = R.make_input(c)
    plan = _send_one(lib, link, x, c.bit, c.clamp, c.offset)
    kind = R.plan_kind(plan, c.items)
    get = 'get-fast' if R.get_fast_path(c.bit, c.n) else 'get-word'
    _RAN[('link', f"{kind}/{get}", c.bit)] += 1
    if c.kind in ('normal', 'outliers') and (c.items * c.n) % 4 == 0:
        # the deferred residual add: the payload is a + b, summed while the send reads it
        b = (np.random.default_rng(c.seed + 1).standard_normal(x.shape) * 0.3).astype(np.float32)
        _send_one(lib, link, x, c.bit, c.clamp, c.offset, b)
        _RAN[('link', f"{kind}/a+b", c.bit)] += 1


@pytest.mark.parametrize('role', ROLES)
def test_link_fused_send_plans(lib, link, role):
    """The fused send kernel's plans, shaped from the plan query for this GPU's SM count: the slice cached with one or
    several segments per CTA, streamed from HBM in pass 2, one item split into the maximum 64 chunks, items in
    {1, max_ctas, max_ctas + 1, 512}, and BASELINE config 5's hop. Both x and the deferred sum a + b."""
    _, items, n, bit = next(s for s in R.link_shapes(lib) if s[0] == role)
    plan = R.link_plan(lib, items, n, bit)
    kind = R.plan_kind(plan, items)
    if role in ROLE_KIND:
        assert kind == ROLE_KIND[role], (role, plan)
    rng = np.random.default_rng(ROLES.index(role))
    x = (rng.standard_normal((items, n)) * 1.7 + 0.1).astype(np.float32)
    x[0, :2] = np.array([60.0, -45.0], np.float32)              # outliers: the clamp bites
    _send_one(lib, link, x, bit, 'auto')
    b = (rng.standard_normal((items, n)) * 0.3).astype(np.float32)
    _send_one(lib, link, x, bit, 'auto', b=b)
    _RAN[('link', f"{kind}/{role}", bit)] += 2


@pytest.mark.parametrize('order', ['fused+staged', 'staged+fused'])
@pytest.mark.parametrize('deferred', [False, True])
def test_link_two_quantised_tensors(lib, link, order, deferred):
    """A mid-block cut's (data, skip) payload, both quantised: one tensor on the fused kernel (n % 16 == 0), the other
    on the staged path (n % 16 != 0); each has its own threshold, scale / shift block and codes."""
    rng = np.random.default_rng(41 + deferred)
    items, bit = 3, 8
    ns = (1024, 1000) if order == 'fused+staged' else (1000, 1024)
    xs = [(rng.standard_normal((items, n)) * s + 0.1).astype(np.float32) for n, s in zip(ns, (1.3, 2.1))]
    bs = [(rng.standard_normal((items, n)) * 0.3).astype(np.float32) for n in ns] if deferred else [None, None]
    keep, tensors = [], []
    for x, b in zip(xs, bs):
        ka, pa = _device(x, 0)
        kb, pb = _device(b, 0) if b is not None else (None, None)
        keep += [ka, kb]
        tensors.append((pa, pb, x.shape[1]))
    paths = [R.link_plan(lib, items, n, bit).path for n in ns]
    assert paths == order.split('+')
    link.put(tensors, items, bit, R.CLAMP['auto'])
    d0, d1 = link.get(items, ns[0], ns[1])
    assert tuple(link.read(4, 8, np.uint32)) == (2, items)
    payloads = [x if b is None else (x + b).astype(np.float32) for x, b in zip(xs, bs)]
    exps = [_check_link_tensor(link, ti, p, bit, 'auto', items) for ti, p in enumerate(payloads)]
    _same(d0, exps[0].dec, 'tensor 0 decoded')
    _same(d1, exps[1].dec, 'tensor 1 decoded')
    _RAN[('link', 'two-tensors/' + order, bit)] += 1


def test_link_rejects_bad_width_and_too_many_items_on_the_host(lib, link):
    from pipeedge_b200._lib import PipeEdgeB200Error
    x = torch.randn(513 * 64, device='cuda')
    torch.cuda.synchronize()
    before = lib.LIB.pe_launch_count()
    for items, bit in ((4, 17), (513, 8)):
        with pytest.raises(PipeEdgeB200Error):
            link.put([(x.data_ptr(), None, 64)], items, bit, R.CLAMP['auto'])
    assert lib.LIB.pe_launch_count() == before
