"""CPU: the stage sub-layer program of `_stage_ref.py` states the model, not the executor.

With the exact fp64 backend it equals the fp64 CPU oracle (`oracle.shards`, the restatement of the reference's shard
forward) at every cut of a 3-block model of each family, fused or not; its kernel-kind sequence is the one written out
by hand below for a handful of cuts; and plausible executor bugs planted in it (swapped LayerNorms, the previous block's
LayerNorm, a wrong eps, the residual add on the wrong side of a LayerNorm) make the fp64 comparison fail. The GPU test
`test_stage_composition_gpu.py` then holds the stage executor to this program bit for bit."""
import dataclasses
import os
import sys

import numpy as np
import pytest
import torch

TESTS = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, TESTS)
import _stage_ref as SR  # noqa: E402
from oracle import shards as osh  # noqa: E402
from pipeedge_b200.synth import MODEL_SPECS, synth_weights  # noqa: E402

SPECS = {
    'vit': dataclasses.replace(MODEL_SPECS['test/vit-tiny'], blocks=3),
    'deit': dataclasses.replace(MODEL_SPECS['test/deit-tiny'], blocks=3),
    'bert': dataclasses.replace(MODEL_SPECS['test/bert-tiny'], blocks=3, classify=False),
}
BATCH, BERT_TOKENS = 2, 9
EXACT = 1e-12     # fp64 restatements of the same maths in a different op order
WRONG = 1e3 * EXACT   # what a planted bug must exceed (eps 1e-6 on rows of unit variance: ~5e-7)


def all_cuts(layers):
    return [(ls, le) for ls in range(1, layers + 1) for le in range(ls, layers + 1)]


@pytest.fixture(scope='module')
def weights():
    return {fam: synth_weights(spec, seed=3) for fam, spec in SPECS.items()}


@pytest.fixture
def oracle64(monkeypatch):
    """The oracle's shard forward with its weights converted to float64 instead of float32."""
    monkeypatch.setattr(osh, '_t', lambda arr: torch.from_numpy(np.ascontiguousarray(arr)).double())

    def run(spec, w, ls, le, data):
        shard = osh.PreparedShard(spec, w, ls, le)
        shard.is_first = shard.is_last = False    # the encoder sub-layers only: no embeddings, no head
        return shard.forward(data)
    return run


def stage_input(spec, ls, seed):
    gen = torch.Generator().manual_seed(seed)
    tokens = BERT_TOKENS if spec.family == 'bert' else spec.tokens
    first_sub = (ls - 1) % 4
    rnd = lambda width: torch.randn(BATCH, tokens, width, generator=gen, dtype=torch.float64)  # noqa: E731
    if first_sub in (1, 3):
        return (rnd(spec.inter if first_sub == 3 else spec.hidden), rnd(spec.hidden))
    return rnd(spec.hidden)


def program(spec, w, ls, le, data, **kw):
    ranges = osh.sublayer_ranges(ls, le)
    params = [SR.Fp64Backend.weights(osh.block_params(spec.family, w, block, spec.hidden)) for block, _, _ in ranges]
    return SR.stage_program(spec.family, ranges, params, data, SR.Fp64Backend(), spec.heads, spec.eps, **kw)


def rel_err(got, want):
    got = got if isinstance(got, tuple) else (got,)
    want = want if isinstance(want, tuple) else (want,)
    assert len(got) == len(want)
    err = 0.0
    for g, r in zip(got, want):
        assert g.shape == r.shape
        err = max(err, float((g - r).abs().max() / r.abs().max()))
    return err


@pytest.mark.parametrize('family', sorted(SPECS))
def test_program_equals_fp64_oracle_at_every_cut(family, weights, oracle64):
    """All 78 (layer_start, layer_end) of a 3-block model, with and without the fused epilogue, and the deferred add."""
    spec, w = SPECS[family], weights[family]
    for ls, le in all_cuts(spec.layers):
        data = stage_input(spec, ls, seed=ls * 100 + le)
        want = oracle64(spec, w, ls, le, data)
        for fuse in (False, True):
            res = program(spec, w, ls, le, data, fuse=fuse)
            assert res.deferred is None
            err = rel_err(res.out, want)
            assert err <= EXACT, (family, ls, le, fuse, err)
        res = program(spec, w, ls, le, data, defer_add=True)
        if res.deferred is not None:
            assert family != 'bert' and (le - 1) % 4 in (1, 3)
            assert rel_err(res.deferred[0] + res.deferred[1], want) <= EXACT, (family, ls, le)
        else:
            assert family == 'bert' or (le - 1) % 4 in (0, 2)


L, Q, A, O, F1, F2, C = 'layernorm', 'gemm_qkv', 'attention', 'gemm_out', 'gemm_fc1', 'gemm_fc2', 'cast'
KIND_CASES = [
    # family, layer_start, layer_end, fused, deferred add, kernel kinds
    ('vit', 1, 4, False, False, [L, Q, A, O, L, F1, F2, C]),
    ('vit', 1, 4, True, False, [L, Q, A, O, F1, F2, C]),            # LN2 in the out-proj; the last FC2 has no next LN
    ('vit', 1, 4, False, True, [L, Q, A, O, L, F1, F2]),            # the final add left to the consumer
    ('vit', 1, 5, False, False, [L, Q, A, O, L, F1, F2, L, Q, A, C]),   # tuple out: ctx widened to fp32
    ('vit', 1, 5, True, False, [L, Q, A, O, F1, F2, Q, A, C]),      # block 1's LN1 in block 0's FC2
    ('vit', 2, 3, False, False, [C, O, L, F1, C]),                  # tuple in and out
    ('vit', 2, 3, True, False, [C, O, F1, C]),
    ('vit', 4, 4, True, False, [C, F2, C]),
    ('deit', 3, 8, False, False, [L, F1, F2, L, Q, A, O, L, F1, F2, C]),
    ('deit', 3, 8, True, False, [L, F1, F2, Q, A, O, F1, F2, C]),
    ('bert', 3, 6, False, False, [C, F1, F2, L, Q, A, O, L]),        # starts at sub-layer 2
    ('bert', 3, 6, True, False, [C, F1, F2, Q, A, O]),
    ('bert', 5, 8, False, False, [C, Q, A, O, L, F1, F2, L]),        # starts at sub-layer 0 of block 1
    ('bert', 4, 5, False, False, [C, F2, L, Q, A, C]),               # starts at sub-layer 3, ends at 0
    ('bert', 4, 5, True, False, [C, F2, Q, A, C]),
    ('bert', 2, 4, False, True, [C, O, L, F1, F2, L]),               # post-LN: nothing to defer
    ('bert', 1, 1, False, False, [C, Q, A, C]),
]


@pytest.mark.parametrize('family,ls,le,fuse,defer,kinds', KIND_CASES,
                         ids=[f'{c[0]}-{c[1]}-{c[2]}{"-fused" if c[3] else ""}{"-defer" if c[4] else ""}' for c in KIND_CASES])
def test_kernel_kind_sequence(family, ls, le, fuse, defer, kinds, weights):
    spec = SPECS[family]
    res = program(spec, weights[family], ls, le, stage_input(spec, ls, seed=1), fuse=fuse, defer_add=defer)
    assert res.kinds == kinds
    assert set(res.kinds) <= set(SR.KINDS)
    assert (res.deferred is not None) == (defer and family != 'bert')


MUTATION_CASES = [(family, m) for family in sorted(SPECS) for m in SR.MUTATIONS
                  if not (m == 'stale_ln' and family == 'bert')]   # BERT's LayerNorms follow their own block's projections


@pytest.mark.parametrize('family,mutation', MUTATION_CASES)
def test_planted_executor_bugs_are_rejected(family, mutation, weights, oracle64):
    """Each planted bug moves the fp64 result far outside EXACT, fused or not, on a cut crossing two block boundaries
    (and the unmutated program stays inside it)."""
    spec, w = SPECS[family], weights[family]
    for ls, le in ((1, 12), (3, 10)):
        data = stage_input(spec, ls, seed=7)
        want = oracle64(spec, w, ls, le, data)
        for fuse in (False, True):
            assert rel_err(program(spec, w, ls, le, data, fuse=fuse).out, want) <= EXACT
            err = rel_err(program(spec, w, ls, le, data, fuse=fuse, mutate=mutation).out, want)
            assert err > WRONG, (family, mutation, ls, le, fuse, err)
