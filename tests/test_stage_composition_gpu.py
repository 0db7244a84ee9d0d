"""GPU: the stage executor composes its kernels exactly.

The executor (`csrc/stage.cu` behind `EncoderStage` and the shard classes) decides which kernel runs on which buffer with
which weights: pre- vs post-LN, the deferred residual add, mid-block (data, skip) tuples, the next block's LayerNorm
inside a fused projection, workspace aliasing, CUDA graphs keyed by pointers, PDL chains. Every kernel is deterministic
for its shape, so a stage must be `torch.equal` to the sub-layer program of `_stage_ref.py` (written from the model's
semantics and checked against the fp64 oracle on the CPU) run over the library's stand-alone ops, each of which the
conformance suite pins to fp64. Checked here, bit for bit, on both outputs of a tuple:

  * 3-block ViT-B (S 197), DeiT-B (198), BERT-base (128 and 33), ViT-L (197) and a head_dim-80 model (320 wide, S 257:
    mma.sync attention, no fused-LayerNorm width), at every cut of the 768-wide ViT and BERT and every
    (first, last sub-layer) pair over 1, 2 and 3 blocks elsewhere, at micro-batches 3 and 1 of a stage sized for 3;
  * launch paths: eager; the graph path's warm-up, capture and replay; a replay after the inputs change in place;
    `pe_stage_profile` (kinds = the program's, count = kernel_count()); the deferred final add (a + b = the output,
    one kernel fewer);
  * the graph cache cycled through more than 64 buffer sets with nothing synchronised, then revisited. Evicting a graph
    that may still be queued is allowed: cuGraphExecDestroy documents that an in-flight executable graph "will not be
    terminated, but rather freed asynchronously on completion";
  * the shard classes: embedding op, program, head ops; and the shards' graph mode fed distinct pinned, pageable and
    device inputs through the staging and output rings;
  * the same with PE_FUSE_LN=1 against the fused program, and PE_NO_PDL=1 giving the bits of the PDL chain (child
    processes: the library reads both once per process).
"""
import ctypes
import dataclasses
import hashlib
import os
import subprocess
import sys
import time

import pytest
import torch

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
sys.path.insert(0, TESTS)
import _stage_ref as SR  # noqa: E402
from oracle import shards as osh  # noqa: E402
from pipeedge_b200.synth import MODEL_SPECS, ModelSpec, hf_config, synth_input, synth_weights  # noqa: E402

pytestmark = pytest.mark.gpu

MAX_UBATCH = 3
UBATCHES = (3, 1)


def _spec3(name, **kw):
    return dataclasses.replace(MODEL_SPECS[name], blocks=3, **kw)


SHAPES = {
    # name: (3-block spec, tokens, every cut)
    'vit-b': (_spec3('google/vit-base-patch16-224'), 197, True),
    'deit-b': (_spec3('facebook/deit-base-distilled-patch16-224'), 198, False),
    'bert-128': (_spec3('bert-base-uncased'), 128, True),
    'bert-33': (_spec3('bert-base-uncased'), 33, True),
    'vit-l': (_spec3('google/vit-large-patch16-224'), 197, False),
    'hd80': (ModelSpec('test/vit-hd80', 'vit', 320, 3, 4, 1280, 10, patch=14), 257, False),
}
NO_PDL_SHAPES = ('vit-b', 'bert-33', 'hd80')


def cuts(every, layers=12):
    if every:
        return [(ls, le) for ls in range(1, layers + 1) for le in range(ls, layers + 1)]
    out = []
    for blocks in (1, 2, 3):
        for first in range(4):
            for last in range(4):
                ls, le = first + 1, 4 * (blocks - 1) + last + 1
                if le >= ls:
                    out.append((ls, le))
    return out


def _libs():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from pipeedge_b200 import _lib, ops   # pylint: disable=import-outside-toplevel
    return _lib, ops


# --------------------------------------------------------------------------------------------------------- helpers
class Model:
    """One shape's weights (reference npz layout) and the program's device weights per block."""
    _cache = {}

    def __init__(self, shape):
        self.shape = shape
        self.spec, self.tokens, self.every = SHAPES[shape]
        key = (self.spec.name, self.spec.hidden)
        if key not in Model._cache:
            Model._cache.clear()    # one model's weights at a time
            w = synth_weights(self.spec, seed=0)
            be = SR.GpuBackend()
            params = [be.weights(osh.block_params(self.spec.family, w, b, self.spec.hidden)) for b in range(3)]
            Model._cache[key] = (w, params)
        self.weights, self.params = Model._cache[key]
        self.be = SR.GpuBackend()
        self.fuse = self.be.fusable(self.spec.hidden)

    def stage(self, ls, le):
        from pipeedge_b200.models.transformers._stage import EncoderStage   # pylint: disable=import-outside-toplevel
        return EncoderStage(self.spec.family, hf_config(self.spec), ls, le, self.weights, self.tokens, MAX_UBATCH)

    def program(self, ls, le, data, defer_add=False):
        ranges = osh.sublayer_ranges(ls, le)
        return SR.stage_program(self.spec.family, ranges, [self.params[b] for b, _, _ in ranges], data, self.be,
                                self.spec.heads, self.spec.eps, fuse=self.fuse, defer_add=defer_add)

    def stage_input(self, ls, ubatch, seed):
        gen = torch.Generator().manual_seed(seed)
        first_sub = (ls - 1) % 4
        rnd = lambda width: torch.randn(ubatch, self.tokens, width, generator=gen).cuda()  # noqa: E731
        if first_sub in (1, 3):
            return (rnd(self.spec.inter if first_sub == 3 else self.spec.hidden), rnd(self.spec.hidden))
        return rnd(self.spec.hidden)


def _tuple(x):
    return x if isinstance(x, tuple) else (x,)


def same(got, want):
    got, want = _tuple(got), _tuple(want)
    return len(got) == len(want) and all(g.shape == w.shape and torch.equal(g, w) for g, w in zip(got, want))


def digest(x):
    h = hashlib.sha256()
    for t in _tuple(x):
        h.update(t.detach().cpu().contiguous().numpy().tobytes())
    return h.hexdigest()[:16]


def clone(x):
    return tuple(t.clone() for t in x) if isinstance(x, tuple) else x.clone()


def out_buffers(stage, ubatch):
    s0, s1 = stage.out_shapes(ubatch)
    return (torch.empty(s0, device='cuda'), None if s1 is None else torch.empty(s1, device='cuda'))


def profile(stage, data, out):
    """pe_stage_profile into caller-owned output buffers: (kernel kinds, outputs)."""
    lib, _ = _libs()
    in0, in1 = data if stage.in_is_tuple else (data, None)
    cap = 16 * len(stage.ranges) + 8
    ms, kinds, n = (ctypes.c_float * cap)(), (ctypes.c_int * cap)(), ctypes.c_int(0)
    lib.check(lib.LIB.pe_stage_profile(stage._handle, in0.data_ptr(), None if in1 is None else in1.data_ptr(),   # pylint: disable=protected-access
                                       out[0].data_ptr(), None if out[1] is None else out[1].data_ptr(), in0.shape[0],
                                       torch.cuda.current_stream().cuda_stream, ms, kinds, cap, ctypes.byref(n)))
    got = out if stage.out_is_tuple else out[0]
    return [stage.KERNEL_KINDS[kinds[i]] for i in range(n.value)], got


class _DeviceArray:
    """fp32 device memory at a raw address, for torch.as_tensor."""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {'shape': tuple(shape), 'typestr': '<f4', 'data': (ptr, False), 'version': 3,
                                         'strides': None}


def _fail(failures, tag, what):
    failures.append(f'{tag}: {what}')


# ------------------------------------------------------------------------------------------------ stage-level runs
def check_cut(model, ls, le, failures, digests=None):
    """Every launch path of stage [ls, le] at every micro-batch against the program."""
    stage = model.stage(ls, le)
    for ubatch in UBATCHES:
        tag = f'{model.shape} [{ls},{le}] ubatch {ubatch}{" fused" if model.fuse else ""}'
        data = model.stage_input(ls, ubatch, seed=1000 * ls + 10 * le + ubatch)
        data2 = model.stage_input(ls, ubatch, seed=1000 * ls + 10 * le + ubatch + 5)
        want, want2 = model.program(ls, le, data), model.program(ls, le, data2)
        n_kinds = len(want.kinds)
        got = stage.forward(data)
        if digests is not None:
            digests[tag.replace(' fused', '')] = digest(got)
        if not same(got, want.out):
            _fail(failures, tag, 'eager output differs from the program')
        if stage.kernel_count() != n_kinds:
            _fail(failures, tag, f'eager kernel_count {stage.kernel_count()} != program {n_kinds}')
        # graph path over persistent input / output buffers: warm-up, capture, replay, replay on new contents
        ins, out = clone(data), out_buffers(stage, ubatch)
        for call in ('graph warm-up', 'graph capture', 'graph replay'):
            got = stage.forward(ins, out=out, use_graph=True)
            if not same(got, want.out):
                _fail(failures, tag, f'{call} output differs from the program')
            if stage.kernel_count() != n_kinds:
                _fail(failures, tag, f'{call} kernel_count {stage.kernel_count()} != program {n_kinds}')
        for dst, src in zip(_tuple(ins), _tuple(data2)):
            dst.copy_(src)
        if not same(stage.forward(ins, out=out, use_graph=True), want2.out):
            _fail(failures, tag, 'graph replay after the inputs changed in place differs from the program')
        kinds, got = profile(stage, data, out_buffers(stage, ubatch))
        if kinds != want.kinds:
            _fail(failures, tag, f'profile kinds {kinds} != program {want.kinds}')
        if len(kinds) != stage.kernel_count():
            _fail(failures, tag, f'profile ran {len(kinds)} kernels, kernel_count() says {stage.kernel_count()}')
        if not same(got, want.out):
            _fail(failures, tag, 'profile output differs from the program')
        if stage.out_is_tuple:
            continue
        # the final residual add left to the consumer
        defer = model.program(ls, le, data, defer_add=True)
        got = stage.forward(data, defer_add=True)
        addrs = stage.deferred()
        if defer.deferred is None:
            if addrs is not None or not same(got, want.out) or stage.kernel_count() != n_kinds:
                _fail(failures, tag, 'a stage with no pending add deferred one or changed its output')
            continue
        if addrs is None:
            _fail(failures, tag, 'defer_add left no deferred add')
            continue
        shape = (ubatch, model.tokens, model.spec.hidden)
        a = torch.as_tensor(_DeviceArray(addrs[0], shape), device='cuda')
        b = torch.as_tensor(_DeviceArray(addrs[1], shape), device='cuda')
        if not same(a + b, want.out):
            _fail(failures, tag, 'deferred a + b differs from the program output')
        if stage.kernel_count() != n_kinds - 1 or len(defer.kinds) != n_kinds - 1:
            _fail(failures, tag, f'deferred forward ran {stage.kernel_count()} kernels, not {n_kinds} - 1')
    stage.close()


def check_shape(shape, failures, digests=None):
    model = Model(shape)
    for ls, le in cuts(model.every):
        check_cut(model, ls, le, failures, digests)


def check_graph_cache(failures, n_sets=70, revisit=10):
    """One stage cycled through n_sets > 64 (in, out) buffer sets - warm-up then capture for each, nothing
    synchronised, so the capture that overflows the cache evicts graphs still queued - then the first sets again
    (warm-up, capture, replay). Every output of every call is kept and compared at the end."""
    model = Model('vit-b')
    ls, le, ubatch = 2, 6, 1          # tuple input, ends on the output projection
    stage = model.stage(ls, le)
    sets = []
    for i in range(n_sets):
        data = model.stage_input(ls, ubatch, seed=50_000 + i)
        sets.append((data, out_buffers(stage, ubatch), model.program(ls, le, data).out))
    calls = [i for i in range(n_sets) for _ in range(2)] + [i for i in range(revisit) for _ in range(3)]
    torch.cuda.synchronize()
    kept = []
    for i in calls:
        data, out, _ = sets[i]
        kept.append((i, clone(stage.forward(data, out=out, use_graph=True))))
    torch.cuda.synchronize()
    bad = sorted({i for i, got in kept if not same(got, sets[i][2])})
    if bad:
        _fail(failures, f'graph cache{" fused" if model.fuse else ""}', f'buffer sets {bad} gave outputs that differ')
    stage.close()


# ------------------------------------------------------------------------------------------------ shard-level runs
SHARD_MODELS = {
    'vit': (_spec3('google/vit-base-patch16-224'), 'vit'),
    'deit': (_spec3('facebook/deit-base-distilled-patch16-224'), 'deit'),
    'bert': (_spec3('textattack/bert-base-uncased-CoLA'), 'bert'),
}
SHARD_CUTS = ((1, 5), (6, 12), (1, 12))
BERT_SEQ = 33


def make_shard(spec, weights, ls, le):
    from pipeedge_b200.models import ModuleShardConfig   # pylint: disable=import-outside-toplevel
    from pipeedge_b200.models.transformers import bert, deit, vit   # pylint: disable=import-outside-toplevel
    cls = {'vit': vit.ViTShardForImageClassification, 'deit': deit.DeiTShardForImageClassification,
           'bert': bert.BertShardForSequenceClassification}[spec.family]
    cfg = ModuleShardConfig(layer_start=ls, layer_end=le, is_first=ls == 1, is_last=le == spec.layers)
    return cls(hf_config(spec), cfg, weights)


def embed_op(spec, prep, data):
    """The stage-0 edge kernel on weights taken from the oracle's embedding parameters."""
    lib, _ = _libs()
    e = prep.embed_weights
    stream = torch.cuda.current_stream().cuda_stream
    hidden = spec.hidden
    if spec.family == 'bert':
        batch, seq = data.shape
        out = torch.empty(batch, seq, hidden, device='cuda')
        dev = [data.cuda(), e['pos_ids'].reshape(-1).cuda(), e['word'].cuda(), e['type'][0].contiguous().cuda(),
               e['pos'].cuda(), e['ln_w'].cuda(), e['ln_b'].cuda()]
        lib.check(lib.LIB.pe_bert_embed(*(t.data_ptr() for t in dev), spec.eps, out.data_ptr(), batch, seq, hidden,
                                        stream))
        return out
    batch = data.shape[0]
    kdim = spec.channels * spec.patch ** 2
    kpad = (kdim + 7) // 8 * 8
    w16 = torch.zeros(hidden, kpad, dtype=torch.float16)
    w16[:, :kdim] = e['conv_w'].reshape(hidden, kdim).half()
    pos = e['pos'][0]
    n_prefix = 1 if spec.family == 'vit' else 2
    prefix = torch.cat([e['cls'][0] + pos[:1], pos[1:n_prefix]], 0)     # DeiT: the zero distillation token + its position
    n_patches = (spec.image_size // spec.patch) ** 2
    out = torch.empty(batch, n_patches + n_prefix, hidden, device='cuda')
    work = torch.empty(batch * n_patches, kpad, dtype=torch.float16, device='cuda')
    dev = [data.cuda(), w16.cuda(), e['conv_b'].cuda(), pos.contiguous().cuda(), prefix.contiguous().cuda()]
    lib.check(lib.LIB.pe_patch_embed(*(t.data_ptr() for t in dev), out.data_ptr(), work.data_ptr(), batch,
                                     spec.channels, spec.image_size, spec.patch, hidden, n_prefix, stream))
    return out


def head_ops(spec, prep, x):
    """ViT / DeiT: final LayerNorm of the [CLS] rows (fp16) and the classifier; BERT: pooler (tanh) and classifier."""
    lib, ops = _libs()
    cls_rows = x[:, 0, :].contiguous()
    if spec.family == 'bert':
        pool_w, pool_b, cls_w, cls_b = (t.cuda() for t in prep.head)
        pooled = ops.linear(cls_rows.half(), pool_w.half(), pool_b, lib.PE_EPI_TANH_F32)
        return ops.linear(pooled.half(), cls_w.half(), cls_b, lib.PE_EPI_F32)
    ln_w, ln_b, head_w, head_b = (t.cuda() for t in prep.head)
    a16 = ops.layernorm(cls_rows, ln_w, ln_b, spec.eps, want_f32=False, want_f16=True)[1]
    return ops.linear(a16, head_w.half(), head_b, lib.PE_EPI_F32)


def shard_reference(spec, weights, ls, le, data, be, fuse):
    prep = osh.PreparedShard(spec, weights, ls, le)
    x = embed_op(spec, prep, data) if prep.is_first else data
    ranges = osh.sublayer_ranges(ls, le)
    x = SR.stage_program(spec.family, ranges, [be.weights(prep.params[b]) for b, _, _ in ranges], x, be, spec.heads,
                         spec.eps, fuse=fuse).out
    return head_ops(spec, prep, x) if prep.is_last else x


def shard_input(spec, ls, le, batch, seed):
    if ls == 1:
        return synth_input(spec, batch, seed=seed, seq_len=BERT_SEQ)
    tokens = BERT_SEQ if spec.family == 'bert' else spec.tokens
    gen = torch.Generator().manual_seed(seed)
    first_sub = (ls - 1) % 4
    rnd = lambda width: torch.randn(batch, tokens, width, generator=gen).cuda()  # noqa: E731
    if first_sub in (1, 3):
        return (rnd(spec.inter if first_sub == 3 else spec.hidden), rnd(spec.hidden))
    return rnd(spec.hidden)


def check_shards(family, failures):
    """First, last and whole-model shards through the real classes = edge op, program, head op; then the shards'
    graph mode on distinct pinned / pageable / device inputs (H2D staging ring, output slot ring)."""
    spec, _ = SHARD_MODELS[family]
    weights = synth_weights(spec, seed=0)
    be = SR.GpuBackend()
    fuse = be.fusable(spec.hidden)
    for ls, le in SHARD_CUTS:
        tag = f'{family} shard [{ls},{le}]{" fused" if fuse else ""}'
        data = shard_input(spec, ls, le, 3, seed=ls + le)
        got = make_shard(spec, weights, ls, le)(data)
        if not same(got, shard_reference(spec, weights, ls, le, data, be, fuse)):
            _fail(failures, tag, 'output differs from edge op + program + head op')
    ls, le = (1, 7) if family == 'bert' else (1, 6)       # a first stage: host inputs go through the staging ring
    shard = make_shard(spec, weights, ls, le)
    inputs = []
    for i in range(3 * shard.num_slots):
        x = synth_input(spec, 2, seed=100 + i, seq_len=BERT_SEQ)
        inputs.append(x.pin_memory() if i % 3 == 0 else (x if i % 3 == 1 else x.cuda()))
    eager = [clone(shard(x)) for x in inputs]
    shard.use_cuda_graph = True
    outs = [shard(x) for x in inputs]      # warm-up, capture and replays of every slot, nothing synchronised
    torch.cuda.synchronize()
    for i in range(len(inputs) - shard.num_slots, len(inputs)):
        if not same(outs[i], eager[i]):
            _fail(failures, f'{family} shard [{ls},{le}] graph mode', f'input {i} ({["pinned", "pageable", "device"][i % 3]}) '
                  'differs from its eager result')


# ---------------------------------------------------------------------------------------------------------- tests
def _assert_ok(failures):
    assert not failures, f'{len(failures)} failures:\n' + '\n'.join(failures[:40])


def test_fused_widths():
    """The widths the fused epilogue takes (768 and 1024 in clusters of 8) and one it does not (320)."""
    lib, _ = _libs()
    assert [lib.LIB.pe_linear_ln_cluster(n) for n in (768, 1024, 320)] == [8, 8, 0]


@pytest.mark.parametrize('shape', list(SHAPES))
def test_stage_equals_program(shape):
    _libs()
    failures = []
    check_shape(shape, failures)
    _assert_ok(failures)


def test_graph_cache_eviction():
    _libs()
    failures = []
    check_graph_cache(failures)
    _assert_ok(failures)


@pytest.mark.parametrize('family', list(SHARD_MODELS))
def test_shards_equal_edges_program_head(family):
    _libs()
    failures = []
    check_shards(family, failures)
    _assert_ok(failures)


_CHILD = """
import os, sys
sys.path[:0] = [sys.argv[1], os.path.join(sys.argv[1], 'tests')]
import test_stage_composition_gpu as T
sys.exit(T.child_main(sys.argv[2]))
"""


def child_main(what):
    """Entry point of the child processes (the library reads PE_FUSE_LN / PE_NO_PDL once per process)."""
    failures, digests = [], {}
    t0 = time.time()
    if what == 'fuse':
        for shape in SHAPES:
            check_shape(shape, failures)
        check_graph_cache(failures)
        for family in SHARD_MODELS:
            check_shards(family, failures)
    elif what == 'nopdl':
        for shape in NO_PDL_SHAPES:
            check_shape(shape, failures, digests)
    for tag, d in sorted(digests.items()):
        print(f'DIGEST {tag}|{d}', flush=True)
    print(f'child {what}: {time.time() - t0:.1f} s', flush=True)
    print('\n'.join(failures) if failures else 'all ok', flush=True)
    return 1 if failures else 0


def _child(what, env):
    res = subprocess.run([sys.executable, '-c', _CHILD, ROOT, what], capture_output=True, text=True, timeout=1800,
                         env={**os.environ, **env})
    assert res.returncode == 0 and 'all ok' in res.stdout, res.stdout[-6000:] + res.stderr[-4000:]
    return res.stdout


def test_fused_layernorm_executor():
    """PE_FUSE_LN=1 (child process): every shape, cut, micro-batch and launch path, the graph cache and the shards
    against the fused program (the head_dim-80 model has no fused width and must run unfused)."""
    _libs()
    _child('fuse', {'PE_FUSE_LN': '1'})


def test_no_pdl_gives_the_same_bits():
    """PE_NO_PDL=1 (child process): the stage equals the program there too, and its eager outputs carry the same bits
    as the PDL chain's in this process."""
    _libs()
    failures, digests = [], {}
    for shape in NO_PDL_SHAPES:
        model = Model(shape)
        for ls, le in cuts(model.every):
            stage = model.stage(ls, le)
            for ubatch in UBATCHES:
                data = model.stage_input(ls, ubatch, seed=1000 * ls + 10 * le + ubatch)
                digests[f'{shape} [{ls},{le}] ubatch {ubatch}'] = digest(stage.forward(data))
            stage.close()
    out = _child('nopdl', {'PE_NO_PDL': '1'})
    child = dict(line[len('DIGEST '):].split('|') for line in out.splitlines() if line.startswith('DIGEST '))
    assert set(child) == set(digests)
    for tag, d in sorted(digests.items()):
        if child[tag] != d:
            _fail(failures, tag, 'PE_NO_PDL=1 output differs from the PDL chain')
    _assert_ok(failures)
