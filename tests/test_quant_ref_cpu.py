"""CPU: the QuantPipe conformance cases of `_quant_ref.py` are strong enough to catch a wrong kernel.

Every bit-width gets rounding ties (of both parities where both exist) and every code value; the stand-alone cases and
the link shapes together reach every send plan of `pe_debug_link_put_plan` (host-only: the library's default of 132
SMs without a GPU); each NumPy mutant differs from the oracle on at least one case; and the mutant model with no
mutation is the oracle."""
import os
import sys

import numpy as np
import pytest
import torch

TESTS = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, TESTS)
import _quant_ref as R  # noqa: E402
from oracle import quant as oq  # noqa: E402

CASES = R.standalone_cases()


def _expected(c):
    x = R.make_input(c)
    alpha, _ = R.oracle_alpha(x, c.bit, c.clamp)
    return x, alpha, R.expected(x, c.bit, alpha)


@pytest.fixture(scope='module')
def oracle_out():
    return [(c, *_expected(c)) for c in CASES]


def test_every_bit_has_ties_of_both_parities():
    for bit in R.BITS:
        ks = {k for _, found in R.tie_values(bit) for _, k in found}
        assert ks, bit
        assert {k % 2 for k in ks} == ({0} if bit == 1 else {0, 1}), bit


def test_ties_round_half_to_even(oracle_out):
    """The ties item really quantises ties: its codes are the even neighbours of k + 1/2."""
    for c, x, _, exp in oracle_out:
        if c.kind != 'ties':
            continue
        s, found = R.tie_values(c.bit)[c.seed % 3]
        assert exp.scale[0] == s and exp.shift[0] == 0, R.case_id(c)   # item 0 is not clamped
        codes = oq.unpack_codes(exp.codes[0].view(np.uint32), c.n, c.bit)
        by_value = dict(found)
        for v, q in zip(x[0], codes):
            if v in by_value:
                k = by_value[v]
                assert q == (k if k % 2 == 0 else k + 1), (R.case_id(c), float(v), k, int(q))


def test_every_ramp_produces_every_code(oracle_out):
    seen = set()
    for c, _, _, exp in oracle_out:
        if c.kind != 'ramp':
            continue
        codes = oq.unpack_codes(exp.codes[0].view(np.uint32), c.n, c.bit)
        assert set(codes.tolist()) == set(range(R.levels(c.bit) + 1)), R.case_id(c)
        seen.add(c.bit)
    assert seen == set(R.BITS)


def test_special_items_are_what_they_claim(oracle_out):
    kinds, bites = {}, set()
    for c, x, alpha, exp in oracle_out:
        kinds.setdefault(c.kind, set()).add(c.bit)
        if c.kind == 'constant_item':
            assert exp.scale[1] == 0 and exp.shift[1] == np.float32(0.75) and np.all(exp.dec[1] == np.float32(0.75))
            assert not exp.codes[1].any()
        elif c.kind == 'clamped_item':
            assert alpha < x[0].min(), R.case_id(c)                      # the whole item lies beyond alpha
            assert exp.scale[0] == 0 and exp.shift[0] == alpha and np.all(exp.dec[0] == alpha)
        elif c.kind == 'subnormal':
            assert 0 < exp.scale[1] < np.finfo(np.float32).tiny               # the item's scale is itself subnormal
            assert np.count_nonzero(exp.dec[1]) > c.n // 2
        elif c.kind in ('branch_gelu', 'branch_laplace') and c.clamp == 'auto':
            _, branch = R.oracle_alpha(x, c.bit, 'auto')
            assert branch == ('gelu' if c.kind == 'branch_gelu' else 'laplace')
            assert x.min() == R.F32_02 or x.min() == np.nextafter(R.F32_02, np.float32(0))
        elif c.kind == 'outliers' and np.abs(x).max() > alpha:
            bites.add(c.bit)                                                  # the clamp bites
    for kind in ('normal', 'outliers', 'ties', 'ramp', 'constant_item', 'clamped_item', 'subnormal', 'branch_gelu',
                 'branch_laplace'):
        assert kinds[kind] == set(R.BITS), kind
    assert bites == set(R.BITS)


def test_shapes_per_bit():
    for bit in R.BITS:
        r = R.ratio(bit)
        shapes = R.standalone_shapes(bit)
        mods = {n % r for n, _ in shapes if n >= r}
        assert {0, 1 % r, (r - 1) % r} <= mods, bit
        assert any(n < r for n, _ in shapes) or r == 1, bit
        assert any(off in (1, 2, 3) for _, off in shapes), bit
        if bit in R.PACK16:
            assert any(n % 16 == 0 and off == 0 for n, off in shapes), bit   # the pack16 kernel
            assert any(n % 16 != 0 for n, _ in shapes), bit                  # the generic kernel at a pack16 width
    clamps = {c.clamp for c in CASES}
    assert clamps == set(R.CLAMP)


def test_mutant_model_without_mutation_is_the_oracle(oracle_out):
    for c, x, alpha, exp in oracle_out:
        assert not R.differs(exp, R.model(x, c.bit, alpha)), R.case_id(c)


@pytest.mark.parametrize('mutant', sorted(R.MUTANTS))
def test_every_mutant_is_rejected(oracle_out, mutant):
    caught = [R.case_id(c) for c, x, alpha, exp in oracle_out
              if R.differs(exp, R.model(x, c.bit, alpha, **R.MUTANTS[mutant]))]
    assert caught, f"no case tells the mutant {mutant} from the oracle"


def test_reciprocal_unit_differs_where_expected():
    """code * (1 / levels) in fp32 vs fp32(code / levels) with an fp64 divide: the number of codes whose unit differs."""
    def n_diff(bit):
        c = np.arange(R.levels(bit) + 1)
        want = (c / R.levels(bit)).astype(np.float32)
        got = c.astype(np.float32) * (np.float32(1) / np.float32(R.levels(bit)))
        return int(np.count_nonzero(want != got))
    assert (n_diff(3), n_diff(8), n_diff(16)) == (2, 126, 512)


def _plan_lib():
    from pipeedge_b200 import _lib
    return _lib


def test_link_cases_reach_every_send_plan():
    """At the library's default SM count (no GPU here): the link shapes and the stand-alone cases sent through a link
    reach the fused kernel with its slice cached (one and several segments per CTA), streamed from HBM, at the 64-chunk
    cap, the staged path, items in {1, max_ctas, max_ctas + 1, 512}, and both decode paths of the get kernel."""
    if torch.cuda.is_available():
        pytest.skip("checks the host-only plan at the default SM count; a GPU is present")
    lib = _plan_lib()
    max_ctas = R.link_plan(lib, R.MAX_ITEMS, 16, 8).grid
    assert max_ctas == 132 - 8
    kinds, items, get_paths = set(), set(), set()
    for role, it, n, bit in R.link_shapes(lib):
        p = R.link_plan(lib, it, n, bit)
        kinds.add(R.plan_kind(p, it))
        items.add(it)
        get_paths.add(R.get_fast_path(bit, n))
    for c in CASES:
        p = R.link_plan(lib, c.items, c.n, c.bit, aligned=c.offset == 0)
        kinds.add(R.plan_kind(p, c.items))
        get_paths.add(R.get_fast_path(c.bit, c.n))
    assert {'staged', 'fused-cached-1seg', 'fused-cached-multiseg', 'fused-stream', 'fused-cached-1seg-cap'} <= kinds
    assert {1, max_ctas, max_ctas + 1, R.MAX_ITEMS} <= items
    assert get_paths == {True, False}
    assert R.plan_kind(R.link_plan(lib, 32, 198 * 768, 8), 32) == 'fused-stream'   # BASELINE config 5's hop
    for bit in R.BITS:
        assert any(R.get_fast_path(bit, c.n) for c in CASES if c.bit == bit) == (R.ratio(bit) % 4 == 0), bit


def test_link_plan_follows_the_rules():
    """The plan query's rules, independent of the SM count: fused only for the pack16 widths with whole 16-value groups
    and aligned inputs; chunks of 16-multiple length covering the item; the slice cached iff it fits in 160 KiB."""
    lib = _plan_lib()
    for items in (1, 3, 64, 200, 512):
        for n in (16, 100, 4096, 50_000, 300_000):
            for bit in (1, 2, 3, 8, 16):
                for aligned in (True, False):
                    p = R.link_plan(lib, items, n, bit, aligned)
                    fused = bit in R.PACK16 and n % 16 == 0 and aligned
                    assert p.path == ('fused' if fused else 'staged')
                    if fused:
                        assert p.per % 16 == 0 and p.per * p.chunks >= n and 1 <= p.chunks <= R.MAX_CHUNKS
                        segs_per_cta = -(-items * p.chunks // p.grid)
                        slice_bytes = -(-segs_per_cta * p.per * 4 // 128) * 128
                        assert p.cache == (slice_bytes <= R.QUANT_CACHE_BYTES)
    assert R.link_plan(lib, 4, 64, 0).path == 'copy'
    from pipeedge_b200._lib import PipeEdgeB200Error
    import ctypes
    out = (ctypes.c_int * 5)()
    for args in ((513, 64, 8, 1), (4, 64, 17, 1), (0, 64, 8, 1)):
        with pytest.raises(PipeEdgeB200Error):
            lib.check(lib.LIB.pe_debug_link_put_plan(*args, out))
