"""CPU: the census of the product's GEMM calls (`_gemm_census.py`) covers the plans the planner gives the supported
models, and each census case still takes the plan of the key it stands for (host-only tile planner). The GPU test
`test_kernel_conformance_gpu.py::test_gemm_product_plans` runs every case against fp64."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _fp_ref as R  # noqa: E402
import _gemm_census as G  # noqa: E402


def _lib():
    from pipeedge_b200 import _lib as lib
    return lib


def _find(cases, **want):
    return [c for c in cases if all(getattr(c, f) == v for f, v in want.items() if f in c._fields) and
            all(c.expect[f] == v for f, v in want.items() if f not in c._fields)]


def test_census_holds_the_planners_headline_choices():
    lib = _lib()
    cases = G.census(lib)
    keys = G.census_keys(lib)
    new = [k for k in keys if k not in G.conformance_keys(lib)]
    print(f"\nGEMM census: {len(G.product_calls())} product calls, {len(keys)} plan keys ({len(new)} not reached by "
          f"the shape-driven cases), {len(cases)} cases")
    assert len(keys) > 0 and len(cases) >= len(keys)
    # ViT-B FC2 at micro-batch 8: a 1 x 2 cluster multicasting A, BN 96
    vit_b = G.MODEL_SPECS['google/vit-base-patch16-224']
    assert G.call_key(lib, G.Call(vit_b.name, 8, 197, 'fc2', 8 * 197, 768, 3072, 'F32', 1, 'fc1'))[1]['cn'] == 2
    assert _find(cases, site='fc2', epi='F32', static_w=1, cm=1, cn=2, bn=96)
    # BERT-base FC2 on BN 192, ViT-L FC2 on BN 224 (single CTAs), ViT-L QKV on BN 224 over several tiles per CTA
    assert _find(cases, site='fc2', k=3072, cm=1, cn=1, bn=192)
    assert _find(cases, site='fc2', k=4096, cm=1, cn=1, bn=224)
    assert _find(cases, site='qkv', n=3072, k=1024, bn=224, multi_round=True)
    # the benchmark's 16 GEMMs are all run, as cases of their own or as the representative of their key
    baseline = {(c.m, c.n, c.k, c.epi) for c in G.baseline_calls()}
    assert len(baseline) == 16
    assert baseline <= {(c.m, c.n, c.k, c.epi) for c in cases}


def test_census_has_every_tile_width_the_product_runs():
    lib = _lib()
    planned = {G.call_key(lib, c)[1]['bn'] for c in G.product_calls()}
    assert planned == {c.expect['bn'] for c in G.census(lib)}
    assert {192, 224} <= planned


def test_census_keys_are_distinct_and_cover_every_call():
    lib = _lib()
    keys = G.census_keys(lib)
    assert len(set(keys)) == len(keys)
    assert {G.call_key(lib, c)[0] for c in G.product_calls()} == set(keys)
    reps = [c for c in G.census(lib) if not c.baseline]
    assert len(reps) == len(keys)
    assert sorted(G.call_key(lib, c)[0] for c in reps) == sorted(keys)


def test_census_cases_take_the_plan_they_claim():
    """Each case's plan has the key it stands for (a planner change that moves a product call onto another plan shows
    here first, and the census then picks up the new key)."""
    lib = _lib()
    for case in G.census(lib):
        bad = R.expectation_failures(case, R.query_plan(lib, case))
        assert not bad, (case.name, bad)
        assert case.static_w == (0 if case.site in ('patch', 'head', 'pooler') else 1), case.name
        assert case.feeder in ('layernorm', 'cast', 'attention', 'fc1', 'im2col'), case.name


def test_census_records_the_kernel_that_writes_a():
    """The recording backend sees the stage's own data flow: a whole-block pre-LN stage feeds QKV and FC1 from a
    LayerNorm, the output projection from attention and FC2 from FC1; BERT's first QKV reads the cast of the stage's
    input; stages cut at the output projection or at FC2 read a cast."""
    vit = G.MODEL_SPECS['google/vit-base-patch16-224']
    bert = G.MODEL_SPECS['bert-base-uncased']
    flow = [(c.site, c.feeder) for c in G.stage_calls(vit, 2, vit.tokens, (1, 4))]
    assert flow == [('qkv', 'layernorm'), ('out', 'attention'), ('fc1', 'layernorm'), ('fc2', 'fc1')]
    flow = [(c.site, c.feeder) for c in G.stage_calls(bert, 2, 128, (1, 8))]
    assert flow[0] == ('qkv', 'cast') and flow[4] == ('qkv', 'layernorm')
    assert [(c.site, c.feeder) for c in G.stage_calls(vit, 2, vit.tokens, (4, 5))] == [('fc2', 'cast'), ('qkv', 'layernorm')]
    assert G.stage_calls(vit, 2, vit.tokens, (2, 3))[0][3:] == ('out', 2 * 197, 768, 768, 'F32', 1, 'cast')
