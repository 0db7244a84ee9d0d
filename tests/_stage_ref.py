"""The sub-layer program of one encoder stage, over an exchangeable op backend.

`stage_program` runs sub-layers `[layer_start, layer_end]` of a ViT / DeiT / BERT stage as a sequence of ops, written
from the model's semantics (`oracle/shards.py::block_sublayers`, `sublayer_ranges`):

  pre-LN (ViT, DeiT)  0: (attention(LN1(x)), x)   1: out-proj(ctx) + skip   2: (GELU(FC1(LN2(x))), x)   3: FC2(inter) + skip
  post-LN (BERT)      0: (attention(x), x)        1: LN1(out-proj(ctx) + skip)  2: (GELU(FC1(x)), x)   3: LN2(FC2(inter) + skip)

and records the kernel kind of every op (the names of `EncoderStage.KERNEL_KINDS`). Where the rounding points are
concerned it states what a kernel library that keeps GEMM operands in fp16 must do: a LayerNorm (or, for BERT, the stream
itself) becomes the fp16 A operand of the next GEMM; a pre-LN residual add is summed in fp32 by the LayerNorm that reads
it (or by an add where the stage ends on it); with the fused projection + residual + LayerNorm epilogue the LayerNorm
that follows a projection moves into it wherever that LayerNorm belongs to the same stage.

Backends:
  `Fp64Backend`  exact torch ops on CPU, no rounding: the program must equal the fp64 oracle (test_stage_ref_cpu.py).
  `GpuBackend`   the library's stand-alone ops (`pipeedge_b200.ops`), each pinned to fp64 by the conformance suite, with
                 the kernels' rounding points: the stage executor must equal it bit for bit
                 (test_stage_composition_gpu.py).

No GPU is needed to import this module.
"""
import collections
import math
import os

import torch
import torch.nn.functional as F

KINDS = ('cast', 'layernorm', 'gemm_qkv', 'attention', 'gemm_out', 'gemm_fc1', 'gemm_fc2')
MUTATIONS = ('swap_ln', 'stale_ln', 'eps', 'add_after_ln')

Result = collections.namedtuple('Result', 'out kinds deferred')


def sublayer_steps(ranges):
    """[(range index, sub-layer)] in execution order for `oracle.shards.sublayer_ranges` triples."""
    return [(i, sub) for i, (_, s0, s1) in enumerate(ranges) for sub in range(s0, s1 + 1)]


def stage_program(family, ranges, params, data, be, heads, eps, fuse=False, defer_add=False, mutate=None):
    """Run the sub-layers `ranges` (`oracle.shards.sublayer_ranges` triples) with `params[i]` the backend weights of
    range i's block (`be.weights(oracle.shards.block_params(...))`). `data` is [B, S, H] or the (data, skip) tuple of a
    mid-block cut. `fuse`: the fused projection + residual + LayerNorm epilogue is available for this width.
    `defer_add`: a pre-LN stage ending on a projection leaves its last residual add to the consumer.
    `mutate` (one of MUTATIONS, fp64 checks only) plants a plausible executor bug.

    Returns Result(out, kinds, deferred): `out` shaped like the oracle's (tuple for a stage ending mid-block), or None
    with `deferred` = (a, b) [B, S, H] whose sum is the output."""
    post = family == 'bert'
    if mutate == 'eps':
        eps = 1e-6
    steps = sublayer_steps(ranges)
    kinds = []

    def op(kind, name, *args):
        kinds.append(kind)
        out = getattr(be, name)(*args)
        be.done()
        return out

    def ln_of(i, sub):
        """LayerNorm parameters of the step (range i, sub): pre-LN before sub 0 / 2, post-LN after sub 1 / 3."""
        first_half = sub in (0, 1)
        if mutate == 'swap_ln':
            first_half = not first_half
        p = params[i]
        if mutate == 'stale_ln' and sub == 0 and i > 0:
            p = params[i - 1]              # the previous block's LayerNorm where this block's belongs
        return (p['ln1_w'], p['ln1_b']) if first_half else (p['ln2_w'], p['ln2_b'])

    in0 = data[0] if isinstance(data, tuple) else data
    batch, tokens = in0.shape[0], in0.shape[1]
    flat = lambda t: t.reshape(batch * tokens, t.shape[-1])  # noqa: E731
    x = skip = t = opnd = a16 = None
    # x: the residual stream (fp32); t: a projection output whose residual add (t + skip) is still pending (pre-LN);
    # opnd: the fp16 context / GELU output a projection reads; a16: the fp16 A operand the next QKV / FC1 reads, when
    # a fused projection (or BERT's LayerNorm) already produced it
    if isinstance(data, tuple):
        opnd, skip = op('cast', 'to_f16', flat(data[0])), flat(data[1])
    else:
        x = flat(data)
    for n, (i, sub) in enumerate(steps):
        p = params[i]
        if sub in (0, 2):
            if a16 is not None:
                a = a16
            elif post:
                a = op('cast', 'to_f16', x)
            elif t is not None:
                g, b = ln_of(i, sub)
                if mutate == 'add_after_ln':
                    a = op('layernorm', 'layernorm', t, g, b, eps)
                    x = be.add(t, skip)
                else:
                    x, a = op('layernorm', 'add_layernorm', t, skip, g, b, eps)
                t = None
            else:
                a = op('layernorm', 'layernorm', x, *ln_of(i, sub), eps)
            a16 = None
            if sub == 0:
                qkv = op('gemm_qkv', 'linear', a, p['w_qkv'], p['b_qkv'], 'f16')
                opnd = op('attention', 'attention', qkv, batch, tokens, heads)
            else:
                opnd = op('gemm_fc1', 'linear', a, p['w_fc1'], p['b_fc1'], 'gelu_f16')
            skip, x = x, None
            continue
        kind = 'gemm_out' if sub == 1 else 'gemm_fc2'
        w, b = (p['w_o'], p['b_o']) if sub == 1 else (p['w_fc2'], p['b_fc2'])
        if post:
            g, beta = ln_of(i, sub)
            if mutate == 'add_after_ln':
                t = op(kind, 'linear', opnd, w, b, 'f32')
                x, a16, t = be.add(be.layernorm_f32(t, g, beta, eps), skip), None, None
            elif fuse:
                x, a16 = op(kind, 'linear_add_layernorm', opnd, w, b, skip, g, beta, eps, True)
            else:
                t = op(kind, 'linear', opnd, w, b, 'f32')
                x, a16 = op('layernorm', 'add_layernorm_post', t, skip, g, beta, eps)
                t = None
            skip = None
        elif fuse and n + 1 < len(steps) and mutate != 'add_after_ln':
            # the LayerNorm of the next sub-layer belongs to this stage: it moves into the projection's epilogue
            g, beta = ln_of(*steps[n + 1])
            x, a16 = op(kind, 'linear_add_layernorm', opnd, w, b, skip, g, beta, eps, False)
            skip = None
        else:
            t = op(kind, 'linear', opnd, w, b, 'f32')
    shape = lambda v: v.reshape(batch, tokens, v.shape[-1])  # noqa: E731
    if t is not None:
        if defer_add and steps[-1][1] in (1, 3):
            return Result(None, kinds, (shape(t), shape(skip)))
        x = op('cast', 'add', t, skip)     # the stage's add kernel is counted as a cast-class kernel
    if steps[-1][1] in (0, 2):
        return Result((shape(op('cast', 'to_f32', opnd)), shape(skip)), kinds, None)
    return Result(shape(x), kinds, None)


# --------------------------------------------------------------------------------------------------------- backends
def _qkv(p):
    return torch.cat([p['wq'], p['wk'], p['wv']], 0), torch.cat([p['bq'], p['bk'], p['bv']], 0)


class Fp64Backend:
    """Exact ops in float64 on CPU: no rounding point at all."""

    @staticmethod
    def weights(p):
        w_qkv, b_qkv = _qkv(p)
        out = {'w_qkv': w_qkv, 'b_qkv': b_qkv, 'w_o': p['wo'], 'b_o': p['bo'], 'w_fc1': p['w1'], 'b_fc1': p['b1'],
               'w_fc2': p['w2'], 'b_fc2': p['b2'], 'ln1_w': p['ln1_w'], 'ln1_b': p['ln1_b'], 'ln2_w': p['ln2_w'],
               'ln2_b': p['ln2_b']}
        return {k: v.double() for k, v in out.items()}

    def done(self):
        pass

    @staticmethod
    def to_f16(x):
        return x

    @staticmethod
    def to_f32(x):
        return x

    @staticmethod
    def _ln(x, g, b, eps):
        return F.layer_norm(x, (x.shape[-1],), g, b, eps)

    def layernorm(self, x, g, b, eps):
        return self._ln(x, g, b, eps)

    def layernorm_f32(self, x, g, b, eps):
        return self._ln(x, g, b, eps)

    def add_layernorm(self, t, skip, g, b, eps):
        x = t + skip
        return x, self._ln(x, g, b, eps)

    def add_layernorm_post(self, t, skip, g, b, eps):
        y = self._ln(t + skip, g, b, eps)
        return y, y

    @staticmethod
    def linear(a, w, b, act):
        y = F.linear(a, w, b)
        return F.gelu(y) if act == 'gelu_f16' else y

    @staticmethod
    def attention(qkv, batch, tokens, heads):
        h = qkv.shape[-1] // 3
        d = h // heads
        q, k, v = (u.reshape(batch, tokens, heads, d).transpose(1, 2) for u in qkv.split(h, dim=-1))
        probs = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(d), dim=-1)
        return (probs @ v).transpose(1, 2).reshape(batch * tokens, h)

    @staticmethod
    def add(t, skip):
        return t + skip

    def linear_add_layernorm(self, a, w, b, skip, g, beta, eps, ln_is_stream):
        v = F.linear(a, w, b) + skip
        y = self._ln(v, g, beta, eps)
        return (y if ln_is_stream else v), y


class GpuBackend:
    """The library's stand-alone ops with the kernels' rounding points: LayerNorm -> fp16 operand; QKV with an fp16
    epilogue, FC1 with GELU -> fp16, output projection and FC2 fp32; the pre-LN residual add folded into the next
    LayerNorm (`residual_layernorm`), or an fp32 add where the stage ends on it; `.half()` / `.float()` at a tuple's
    edges. With `fuse`, the program calls `linear_residual_layernorm` (and the library's LayerNorms take their chunked
    mirror by themselves, as the library reads PE_FUSE_LN once per process). Every op is followed by a device
    synchronisation, so that no op overlaps the next (the executor chains its kernels with programmatic dependent
    launches and nothing in between)."""

    def __init__(self):
        from pipeedge_b200 import _lib, ops   # pylint: disable=import-outside-toplevel
        self.ops, self.lib = ops, _lib
        self.epi = {'f16': _lib.PE_EPI_F16, 'gelu_f16': _lib.PE_EPI_GELU_F16, 'f32': _lib.PE_EPI_F32}

    @staticmethod
    def done():
        torch.cuda.synchronize()

    def fusable(self, hidden):
        """Whether the executor fuses projections at this width in this process: PE_FUSE_LN=1 (read once by the library)
        and a width the fused epilogue supports."""
        return os.environ.get('PE_FUSE_LN', '').startswith('1') and self.lib.LIB.pe_linear_ln_cluster(hidden) > 0

    @staticmethod
    def weights(p, device='cuda'):
        w_qkv, b_qkv = _qkv(p)
        half = {'w_qkv': w_qkv, 'w_o': p['wo'], 'w_fc1': p['w1'], 'w_fc2': p['w2']}
        full = {'b_qkv': b_qkv, 'b_o': p['bo'], 'b_fc1': p['b1'], 'b_fc2': p['b2'], 'ln1_w': p['ln1_w'],
                'ln1_b': p['ln1_b'], 'ln2_w': p['ln2_w'], 'ln2_b': p['ln2_b']}
        out = {k: v.to(device=device, dtype=torch.float16).contiguous() for k, v in half.items()}
        out.update({k: v.to(device=device, dtype=torch.float32).contiguous() for k, v in full.items()})
        return out

    @staticmethod
    def to_f16(x):
        return x.half()

    @staticmethod
    def to_f32(x):
        return x.float()

    def layernorm(self, x, g, b, eps):
        return self.ops.layernorm(x, g, b, eps, want_f32=False, want_f16=True)[1]

    def layernorm_f32(self, x, g, b, eps):
        return self.ops.layernorm(x, g, b, eps)[0]

    def add_layernorm(self, t, skip, g, b, eps):
        x, _, a16 = self.ops.residual_layernorm(t, skip, g, b, eps, want_sum=True, want_f32=False, want_f16=True)
        return x, a16

    def add_layernorm_post(self, t, skip, g, b, eps):
        _, y, a16 = self.ops.residual_layernorm(t, skip, g, b, eps, want_sum=False, want_f32=True, want_f16=True)
        return y, a16

    def linear(self, a, w, b, act):
        return self.ops.linear(a, w, b, self.epi[act], static_w=True)

    def attention(self, qkv, batch, tokens, heads):
        return self.ops.attention(qkv, batch, tokens, heads)

    @staticmethod
    def add(t, skip):
        return t + skip

    def linear_add_layernorm(self, a, w, b, skip, g, beta, eps, ln_is_stream):
        return self.ops.linear_residual_layernorm(a, w, b, skip, g, beta, eps, f32_is_ln=ln_is_stream)
