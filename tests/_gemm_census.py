"""The GEMM calls the supported models make, and the kernel paths they take.

`pe_linear` picks a plan from the shape (`plan_gemm`, gemm_wgmma.cu): the tile width BN, single CTAs or a 1 x 2
multicast cluster, the ring depth, one tile per CTA (epilogue staging aliases the ring) or several. Each combination is
its own code path, so the fp64 conformance suite has to run every combination the product runs, not only the shapes
someone thought of. This module lists them:

  * `product_calls()`: every pe_linear call of every `synth.MODEL_SPECS` model at micro-batches 1-64 (BERT at sequence
    lengths 32, 128 and 512, capped at the model's position table). The encoder-stage GEMMs come from running
    `_stage_ref.stage_program` (the stage's sub-layer program) over a recording backend whose ops return `meta` tensors
    of the right shape, on a stage of two whole blocks and on stages starting at the output projection and at FC2;
    each call also records the library kernel that writes its A operand. The edge GEMMs are added with the arguments
    that `edges.cu` and the shard classes pass: the patch embedding (RESID_F32 over the im2col'ed patches, W read after
    the predecessor), the classifier (F32) and BERT's pooler (TANH_F32).
  * `census(lib)`: the calls keyed by the plan `pe_debug_gemm_plan` (host-only) returns for them, through
    `_fp_ref.plan_geometry`; per key the smallest call is kept, and the 16 GEMMs of the four benchmark configurations
    besides. Each kept case claims its key in `expect` (checked with `_fp_ref.expectation_failures`).

No GPU is needed: the plan query runs on the host.
"""
import collections
import functools

import torch

import _fp_ref as R
import _stage_ref as SR
from oracle import shards as osh
from pipeedge_b200.synth import MODEL_SPECS

MICRO_BATCHES = range(1, 65)
BERT_SEQ = (32, 128, 512)
# (layer_start, layer_end): two whole blocks (every A operand written by a LayerNorm, by attention or by FC1 - and for
# BERT by the cast of the stage's input and by the LayerNorms inside); a stage that starts at the output projection and
# ends mid-block, and one that starts at FC2 (A written by the cast of the incoming fp32 payload)
CUTS = ((1, 8), (2, 7), (4, 5))
# the benchmark's four fp16 pipeline configurations: (model, micro-batch, BERT sequence length)
BASELINE = (('google/vit-base-patch16-224', 8, None), ('google/vit-large-patch16-224', 16, None),
            ('textattack/bert-base-uncased-CoLA', 32, 128), ('facebook/deit-base-distilled-patch16-224', 32, None))
# the plan properties a key is made of (see _fp_ref.plan_geometry)
KEY_FIELDS = ('cm', 'cn', 'bn', 'stages', 'multi_round', 'kb_lt_stages', 'ring_repeats', 'partial_m', 'partial_n',
              'scalar')

# One pe_linear call. site: qkv | out | fc1 | fc2 | patch | head | pooler. feeder: the kernel that writes A just
# before the call (layernorm | cast | attention | fc1 (the GELU output) | im2col). static_w: the call lets the weight
# warp read W before the predecessor kernel has finished (every stage GEMM does).
Call = collections.namedtuple('Call', 'model ub tokens site m n k epi static_w feeder')
# A census case: the call plus its name, the key it claims (`expect`) and `force` (always None: the natural plan).
ProductCase = collections.namedtuple('ProductCase', Call._fields + ('name', 'expect', 'force', 'baseline'))


def _short(model):
    return model.split('/')[-1]


def _tokens(spec):
    """Sequence lengths the model runs at."""
    if spec.family == 'bert':
        return sorted({min(s, spec.max_pos) for s in BERT_SEQ})
    return [spec.tokens]


class _Recorder:
    """A `_stage_ref` backend that computes nothing: every op returns `meta` tensors of the right shape and dtype,
    remembers which op produced them, and `linear` records the call."""

    _F16, _F32 = torch.float16, torch.float32

    def __init__(self, spec, ub, tokens, params):
        self.spec, self.ub, self.tokens = spec, ub, tokens
        self.sites = {id(params['w_qkv']): 'qkv', id(params['w_o']): 'out', id(params['w_fc1']): 'fc1',
                      id(params['w_fc2']): 'fc2'}
        self.calls = []
        self._producer = {}
        self._keep = []          # the tensors stay alive, so that their ids stay unique

    def _new(self, shape, dtype, producer):
        t = torch.empty(tuple(shape), dtype=dtype, device='meta')
        self._producer[id(t)] = producer
        self._keep.append(t)
        return t

    def input(self, shape):
        return self._new(shape, self._F32, 'input')

    def done(self):
        pass

    def to_f16(self, x):
        return self._new(x.shape, self._F16, 'cast')

    def to_f32(self, x):
        return self._new(x.shape, self._F32, 'cast')

    def layernorm(self, x, g, b, eps):
        return self._new(x.shape, self._F16, 'layernorm')

    def layernorm_f32(self, x, g, b, eps):
        return self._new(x.shape, self._F32, 'layernorm')

    def add_layernorm(self, t, skip, g, b, eps):
        return self._new(t.shape, self._F32, 'layernorm'), self._new(t.shape, self._F16, 'layernorm')

    add_layernorm_post = add_layernorm

    def linear(self, a, w, b, act):
        m, k = a.shape
        n = w.shape[0]
        epi = {'f16': 'F16', 'gelu_f16': 'GELU_F16', 'f32': 'F32'}[act]
        self.calls.append(Call(self.spec.name, self.ub, self.tokens, self.sites[id(w)], m, n, k, epi, 1,
                               self._producer[id(a)]))
        return self._new((m, n), self._F32 if act == 'f32' else self._F16, 'fc1' if act == 'gelu_f16' else 'gemm')

    def attention(self, qkv, batch, tokens, heads):
        return self._new((qkv.shape[0], qkv.shape[1] // 3), self._F16, 'attention')

    def add(self, t, skip):
        return self._new(t.shape, self._F32, 'add')

    def linear_add_layernorm(self, *args):
        raise NotImplementedError('the fused projection + LayerNorm epilogue is not part of the census')


def _block_params(spec):
    h, i = spec.hidden, spec.inter

    def meta(*shape):
        return torch.empty(shape, device='meta')

    return {'w_qkv': meta(3 * h, h), 'b_qkv': meta(3 * h), 'w_o': meta(h, h), 'b_o': meta(h), 'w_fc1': meta(i, h),
            'b_fc1': meta(i), 'w_fc2': meta(h, i), 'b_fc2': meta(h), 'ln1_w': meta(h), 'ln1_b': meta(h),
            'ln2_w': meta(h), 'ln2_b': meta(h)}


def stage_calls(spec, ub, tokens, cut):
    """The GEMM calls of one stage [layer_start, layer_end] = `cut` at `ub` items of `tokens` tokens."""
    ranges = osh.sublayer_ranges(*cut)
    params = _block_params(spec)
    be = _Recorder(spec, ub, tokens, params)
    first_sub = ranges[0][1]
    shape = (ub, tokens, spec.hidden)
    if first_sub in (1, 3):
        data = (be.input((ub, tokens, spec.inter if first_sub == 3 else spec.hidden)), be.input(shape))
    else:
        data = be.input(shape)
    SR.stage_program(spec.family, ranges, [params] * len(ranges), data, be, spec.heads, spec.eps)
    return be.calls


def edge_calls(spec, ub, tokens):
    """The GEMMs around the encoder: patch embedding (first stage of ViT / DeiT), classifier and BERT pooler (last
    stage). None of them passes static_w."""
    h = spec.hidden
    calls = []
    if spec.family == 'bert':
        # BertModelShard: tanh(dense(x[:, 0])) on the [CLS] rows copied to fp16; the classification shard then
        # classifies the pooled rows cast to fp16
        calls.append(Call(spec.name, ub, tokens, 'pooler', ub, h, h, 'TANH_F32', 0, 'cast'))
        if spec.classify:
            calls.append(Call(spec.name, ub, tokens, 'head', ub, spec.num_labels, h, 'F32', 0, 'cast'))
    else:
        n_patches = (spec.image_size // spec.patch) ** 2
        kpad = (spec.channels * spec.patch ** 2 + 7) // 8 * 8
        calls.append(Call(spec.name, ub, tokens, 'patch', ub * n_patches, h, kpad, 'RESID_F32', 0, 'im2col'))
        # the classifier reads the final LayerNorm's fp16 output of the [CLS] rows
        calls.append(Call(spec.name, ub, tokens, 'head', ub, spec.num_labels, h, 'F32', 0, 'layernorm'))
    return calls


@functools.lru_cache(maxsize=None)
def product_calls():
    """Every distinct call (first occurrence kept: model order, micro-batch, sequence length, cut, program order)."""
    seen = {}
    for spec in MODEL_SPECS.values():
        for tokens in _tokens(spec):
            for ub in MICRO_BATCHES:
                calls = [c for cut in CUTS for c in stage_calls(spec, ub, tokens, cut)] + edge_calls(spec, ub, tokens)
                for c in calls:
                    seen.setdefault(c, None)
    return list(seen)


def baseline_calls():
    """The 16 encoder-stage GEMMs of the benchmark's four configurations (a whole block each)."""
    out = []
    for model, ub, seq in BASELINE:
        spec = MODEL_SPECS[model]
        out += stage_calls(spec, ub, seq or spec.tokens, (1, 4))
    return out


def call_key(lib, call):
    """(epilogue, static_w) + the plan properties of KEY_FIELDS, as a tuple and as the dict a case claims."""
    geom = R.query_geometry(lib, call.m, call.n, call.k, call.epi)
    expect = {f: geom[f] for f in KEY_FIELDS}
    return (call.epi, call.static_w) + tuple(expect[f] for f in KEY_FIELDS), expect


def _case(call, expect, baseline):
    name = (f"{'baseline-' if baseline else ''}{_short(call.model)}-ub{call.ub}-S{call.tokens}-{call.site}-"
            f"{call.m}x{call.n}x{call.k}-{call.epi}")
    return ProductCase(*call, name=name, expect=expect, force=None, baseline=baseline)


@functools.lru_cache(maxsize=None)
def _census(lib):
    groups = {}
    for call in product_calls():
        key, expect = call_key(lib, call)
        best = groups.get(key)
        if best is None or call.m * call.n * call.k < best[0].m * best[0].n * best[0].k:
            groups[key] = (call, expect)
    reps = [_case(call, expect, False) for call, expect in groups.values()]
    have = {(c.m, c.n, c.k, c.epi, c.static_w) for c in reps}
    for call in baseline_calls():
        if (call.m, call.n, call.k, call.epi, call.static_w) not in have:
            reps.append(_case(call, call_key(lib, call)[1], True))
    return tuple(reps), tuple(groups)


def census(lib):
    """The census cases: one per plan key (its smallest product call), then the benchmark's GEMMs not among them."""
    return list(_census(lib)[0])


def census_keys(lib):
    return list(_census(lib)[1])


def conformance_keys(lib):
    """The keys of the shape-driven GEMM cases of `_fp_ref` (ragged grid and schedules, none with static_w)."""
    keys = set()
    for case in R.RAGGED_CASES + R.SCHEDULE_CASES:
        geom = R.query_plan(lib, case)
        keys.add((case.epi, 0) + tuple(geom[f] for f in KEY_FIELDS))
    return keys
