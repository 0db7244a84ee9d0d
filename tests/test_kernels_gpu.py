"""GPU: each kernel of libpipeedge_b200.so, called through the C-ABI, against a plain fp32 restatement.

LayerNorm / GEMM / attention are floating point: compared with torch fp32 maths on the same (fp16-rounded)
operands, tolerances written in each test. The wgmma GEMM is additionally compared with the library's own
CUDA-core debug GEMM to localise failures.
"""
import math
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from pipeedge_b200 import ops as _ops
    return _ops


def _lib():
    from pipeedge_b200 import _lib
    return _lib


@pytest.mark.parametrize('rows,hidden', [(394, 768), (197, 1024), (34, 128), (7, 192), (64, 1280), (1, 384)])
def test_layernorm(ops, rows, hidden):
    gen = torch.Generator().manual_seed(rows * 31 + hidden)
    x = (torch.randn(rows, hidden, generator=gen) * 2.0 + 0.5)
    g = 1 + 0.1 * torch.randn(hidden, generator=gen)
    b = 0.1 * torch.randn(hidden, generator=gen)
    want = F.layer_norm(x, (hidden,), g, b, 1e-12)
    o32, o16 = ops.layernorm(x.cuda(), g.cuda(), b.cuda(), 1e-12, want_f32=True, want_f16=True)
    torch.testing.assert_close(o32.cpu(), want, rtol=2e-5, atol=2e-5)
    torch.testing.assert_close(o16.cpu().float(), want, rtol=1e-3, atol=1e-3)   # one fp16 rounding


def test_residual_layernorm(ops):
    """t = y + resid (returned as the new residual stream) and LayerNorm(t) in one pass."""
    gen = torch.Generator().manual_seed(5)
    y, r = torch.randn(394, 768, generator=gen), torch.randn(394, 768, generator=gen) * 2
    g, b = 1 + 0.1 * torch.randn(768, generator=gen), 0.1 * torch.randn(768, generator=gen)
    tsum, o32, o16 = ops.residual_layernorm(y.cuda(), r.cuda(), g.cuda(), b.cuda(), 1e-12, want_f32=True)
    assert torch.equal(tsum.cpu(), y + r)
    want = F.layer_norm(y + r, (768,), g, b, 1e-12)
    torch.testing.assert_close(o32.cpu(), want, rtol=2e-5, atol=2e-5)
    torch.testing.assert_close(o16.cpu().float(), want, rtol=1e-3, atol=1e-3)


def _gemm_case(m, n, k, seed):
    gen = torch.Generator().manual_seed(seed)
    a = torch.randn(m, k, generator=gen).half()
    w = (torch.randn(n, k, generator=gen) * 0.05).half()
    bias = torch.randn(n, generator=gen)
    resid = torch.randn(m, n, generator=gen)
    return a, w, bias, resid


def _gemm_ref(a, w, bias, resid, epi):
    lib = _lib()
    acc = a.double() @ w.double().t() + bias.double()
    if epi == lib.PE_EPI_GELU_F16:
        acc = F.gelu(acc)
    elif epi == lib.PE_EPI_TANH_F32:
        acc = torch.tanh(acc)
    elif epi == lib.PE_EPI_RESID_F32:
        acc = acc + resid.double()
    return acc.float()


GEMM_SHAPES = [(128, 256, 64), (128, 128, 128), (256, 512, 768), (1576, 2304, 768), (1576, 768, 3072),
               (197, 3072, 768), (200, 1000, 768), (2, 2, 768), (300, 776, 136), (4096, 768, 768), (33, 40, 72)]


@pytest.mark.parametrize('epi_name', ['PE_EPI_F16', 'PE_EPI_GELU_F16', 'PE_EPI_RESID_F32', 'PE_EPI_F32', 'PE_EPI_TANH_F32'])
def test_linear_simt_debug_kernel(ops, epi_name):
    """The CUDA-core debug GEMM itself is right (it is the comparator for the wgmma kernel)."""
    epi = getattr(_lib(), epi_name)
    a, w, bias, resid = _gemm_case(77, 200, 136, 5)
    want = _gemm_ref(a, w, bias, resid, epi)
    got = ops.linear(a.cuda(), w.cuda(), bias.cuda(), epi, resid=resid.cuda(), debug_simt=True)
    tol = 2e-3 if 'F16' in epi_name else 2e-5
    torch.testing.assert_close(got.cpu().float(), want, rtol=tol, atol=tol)


@pytest.mark.parametrize('m,n,k', GEMM_SHAPES)
def test_linear_tcgen05_f32(ops, m, n, k):
    """fp32-out epilogue: only accumulation order differs from the fp64 reference -> tight tolerance."""
    lib = _lib()
    a, w, bias, resid = _gemm_case(m, n, k, m + n + k)
    want = _gemm_ref(a, w, bias, resid, lib.PE_EPI_F32)
    got = ops.linear(a.cuda(), w.cuda(), bias.cuda(), lib.PE_EPI_F32)
    torch.cuda.synchronize()
    scale = want.abs().max().item()
    err = (got.cpu() - want).abs().max().item()
    assert err <= 2e-5 * max(1.0, scale) * math.sqrt(k / 64), f"max abs err {err} (scale {scale})"


@pytest.mark.parametrize('epi_name', ['PE_EPI_F16', 'PE_EPI_GELU_F16', 'PE_EPI_RESID_F32', 'PE_EPI_TANH_F32'])
@pytest.mark.parametrize('m,n,k', [(1576, 768, 768), (394, 3072, 768), (200, 1000, 136)])
def test_linear_tcgen05_epilogues(ops, epi_name, m, n, k):
    epi = getattr(_lib(), epi_name)
    a, w, bias, resid = _gemm_case(m, n, k, 11 + m)
    want = _gemm_ref(a, w, bias, resid, epi)
    got = ops.linear(a.cuda(), w.cuda(), bias.cuda(), epi, resid=resid.cuda())
    simt = ops.linear(a.cuda(), w.cuda(), bias.cuda(), epi, resid=resid.cuda(), debug_simt=True)
    tol = 2e-3 if 'F16' in epi_name else 5e-5
    torch.testing.assert_close(got.cpu().float(), want, rtol=tol, atol=tol)
    torch.testing.assert_close(got.cpu().float(), simt.cpu().float(), rtol=tol, atol=tol)


def test_linear_resid_in_place(ops):
    """`out` may alias `resid` (the residual stream is updated in place inside a stage)."""
    lib = _lib()
    a, w, bias, resid = _gemm_case(500, 768, 768, 3)
    want = _gemm_ref(a, w, bias, resid, lib.PE_EPI_RESID_F32)
    buf = resid.cuda().clone()
    ops.linear(a.cuda(), w.cuda(), bias.cuda(), lib.PE_EPI_RESID_F32, resid=buf, out=buf)
    torch.testing.assert_close(buf.cpu(), want, rtol=5e-5, atol=5e-5)


def test_linear_static_weight_flag(ops):
    """PE_EPI_STATIC_W (weights fetched ahead of the programmatic dependency) changes timing, not results; back-to-back
    launches exercise the overlap with a predecessor that is still running."""
    lib = _lib()
    a, w, bias, resid = _gemm_case(1576, 3072, 768, 21)
    want = _gemm_ref(a, w, bias, resid, lib.PE_EPI_GELU_F16)
    ad, wd, bd = a.cuda(), w.cuda(), bias.cuda()
    torch.cuda.synchronize()
    outs = [ops.linear(ad, wd, bd, lib.PE_EPI_GELU_F16, static_w=True) for _ in range(4)]
    plain = ops.linear(ad, wd, bd, lib.PE_EPI_GELU_F16)
    for o in outs:
        assert torch.equal(o, plain)
    torch.testing.assert_close(plain.cpu().float(), want, rtol=2e-3, atol=2e-3)


def test_linear_rejects_bad_arguments(ops):
    lib = _lib()
    a, w, bias, _ = _gemm_case(16, 16, 12, 1)     # k % 8 != 0
    with pytest.raises(lib.PipeEdgeB200Error):
        ops.linear(a.cuda(), w.cuda(), bias.cuda(), lib.PE_EPI_F32)
    with pytest.raises(ValueError):
        ops.linear(a, w, bias, lib.PE_EPI_F32)    # CPU tensors: there is no CPU path


@pytest.mark.parametrize('batch,tokens,heads', [(2, 197, 12), (1, 128, 2), (3, 17, 2), (1, 64, 1), (1, 65, 1),
                                                (2, 198, 12), (1, 1, 1), (1, 512, 2), (2, 257, 16), (1, 256, 2),
                                                (8, 197, 12), (4, 240, 3), (32, 128, 12), (16, 197, 16)])
@pytest.mark.parametrize('head_dim', [64, 80])
def test_attention(ops, batch, tokens, heads, head_dim):
    """head_dim 64 (ViT-B/L, DeiT, BERT) and 80 (ViT-Huge)."""
    gen = torch.Generator().manual_seed(tokens + heads)
    hidden = heads * head_dim
    qkv = (torch.randn(batch * tokens, 3 * hidden, generator=gen) * 1.5).half()
    q, k, v = [t.float().view(batch, tokens, heads, head_dim).transpose(1, 2) for t in qkv.split(hidden, dim=1)]
    probs = F.softmax(torch.matmul(q, k.transpose(2, 3)) * head_dim ** -0.5, dim=-1)
    want = torch.matmul(probs, v).transpose(1, 2).reshape(batch * tokens, hidden)
    got = ops.attention(qkv.cuda(), batch, tokens, heads, head_dim=head_dim)
    # P is rounded to fp16 before P.V and the output is fp16: 2e-3 absolute on O(1) values
    torch.testing.assert_close(got.cpu().float(), want, rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize('plan', ['1,1,224', '1,1,96', '2,2,128', '1,1,64'])
def test_linear_forced_tile_plans(ops, plan, monkeypatch):
    """Tile plans the heuristic may not pick (BN not a power of two, BN wider than the heuristic's, clusters with TMA
    multicast) stay correct."""
    lib = _lib()
    monkeypatch.setenv('PE_GEMM_FORCE', plan)
    for epi_name in ('PE_EPI_F16', 'PE_EPI_F32'):
        epi = getattr(lib, epi_name)
        a, w, bias, resid = _gemm_case(1576, 2304, 768, 9)
        want = _gemm_ref(a, w, bias, resid, epi)
        got = ops.linear(a.cuda(), w.cuda(), bias.cuda(), epi)
        tol = 2e-3 if 'F16' in epi_name else 5e-5
        torch.testing.assert_close(got.cpu().float(), want, rtol=tol, atol=tol)


_TCGEN05_ATTENTION_CHECK = """
import os, sys, torch
import torch.nn.functional as F
sys.path.insert(0, sys.argv[1])
os.environ['PE_ATTN_WGMMA'] = sys.argv[2]
from pipeedge_b200 import ops
for batch, tokens, heads in [(2, 197, 12), (1, 128, 2), (3, 17, 2), (1, 64, 1), (1, 65, 1), (2, 198, 12), (1, 1, 1),
                             (1, 256, 2), (8, 197, 12), (4, 240, 3), (32, 128, 12), (16, 197, 16)]:
    gen = torch.Generator().manual_seed(tokens + heads)
    hidden = heads * 64
    qkv = (torch.randn(batch * tokens, 3 * hidden, generator=gen) * 1.5).half()
    q, k, v = [t.float().view(batch, tokens, heads, 64).transpose(1, 2) for t in qkv.split(hidden, dim=1)]
    probs = F.softmax(torch.matmul(q, k.transpose(2, 3)) * 0.125, dim=-1)
    want = torch.matmul(probs, v).transpose(1, 2).reshape(batch * tokens, hidden)
    got = ops.attention(qkv.cuda(), batch, tokens, heads)
    torch.cuda.synchronize()
    torch.testing.assert_close(got.cpu().float(), want, rtol=2e-3, atol=2e-3, msg=lambda m: f"{(batch, tokens, heads)}: {m}")
    print('shape ok', batch, tokens, heads, flush=True)
print('all ok')
"""


@pytest.mark.parametrize('mode', ['1', '0'])
def test_attention_tcgen05(ops, mode):
    """Both attention kernels - wgmma (S in registers, P fed back from registers as the A operand, V read MN-major from
    the TMA image; the default for head_dim 64, S <= 256) and mma.sync (PE_ATTN_WGMMA=0; also the fall-back for other
    shapes) - against fp32 maths over S in {1 .. 256} incl. the ViT / DeiT / BERT shapes. The library reads its selector
    once per process, so each mode runs in a child process."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, '-c', _TCGEN05_ATTENTION_CHECK, root, mode], capture_output=True, text=True,
                         timeout=600)
    assert res.returncode == 0 and 'all ok' in res.stdout, res.stdout[-2000:] + res.stderr[-4000:]


@pytest.mark.parametrize('m,n,k', [(1576, 768, 768), (1576, 768, 3072), (3152, 1024, 4096), (130, 128, 512), (300, 192, 768),
                                   (70, 384, 1536), (4096, 768, 768)])
@pytest.mark.parametrize('post_ln', [False, True])
def test_linear_residual_layernorm_fused(ops, m, n, k, post_ln):
    """Projection + residual add + LayerNorm in one kernel (cluster of the row's column slices exchanging (mean, M2)
    through distributed shared memory) against fp32 maths on the same fp16 operands: clusters of 8 (768, 1024), 4, 2
    and 1 CTAs, several row tiles per cluster (4096 rows), a ragged last row tile, and the in-place residual update."""
    gen = torch.Generator().manual_seed(m + n + k)
    a = (torch.randn(m, k, generator=gen) * 0.7).half()
    w = (torch.randn(n, k, generator=gen) * 0.05).half()
    bias = torch.randn(n, generator=gen) * 0.1
    resid = torch.randn(m, n, generator=gen) * 1.3 + 0.2
    gamma = 1.0 + 0.1 * torch.randn(n, generator=gen)
    beta = 0.1 * torch.randn(n, generator=gen)
    v = a.float() @ w.float().t() + bias + resid
    ln = F.layer_norm(v, (n,), gamma, beta, 1e-12)
    r_dev = resid.cuda()
    o32, o16 = ops.linear_residual_layernorm(a.cuda(), w.cuda(), bias.cuda(), r_dev, gamma.cuda(), beta.cuda(), 1e-12,
                                             f32_is_ln=post_ln, out_f32=r_dev)      # in place, as the stage uses it
    torch.cuda.synchronize()
    assert o32.data_ptr() == r_dev.data_ptr()
    torch.testing.assert_close(o32.cpu(), ln if post_ln else v, rtol=2e-4, atol=2e-4)
    torch.testing.assert_close(o16.cpu().float(), ln, rtol=2e-3, atol=2e-3)


_FUSED_LN_CHECK = """
import os, sys, torch
sys.path.insert(0, sys.argv[1])
os.environ['PE_FUSE_LN'] = '1'
from pipeedge_b200 import _lib, ops
from pipeedge_b200.models import ModuleShardConfig
from pipeedge_b200.models.transformers import bert, vit
from pipeedge_b200.synth import MODEL_SPECS, hf_config, synth_input, synth_weights
# 1. fused kernel == GEMM (fp32 out) + the stand-alone LayerNorm that mirrors its statistics, bit for bit
for m, n, k in ((1576, 768, 768), (1576, 768, 3072), (600, 1024, 1024), (130, 128, 512), (300, 192, 768), (4096, 768, 768)):
    gen = torch.Generator().manual_seed(m + n)
    a = (torch.randn(m, k, generator=gen) * 0.7).half().cuda()
    w = (torch.randn(n, k, generator=gen) * 0.05).half().cuda()
    bias, resid = (torch.randn(n, generator=gen) * 0.1).cuda(), (torch.randn(m, n, generator=gen) * 1.3).cuda()
    gamma, beta = (1.0 + 0.1 * torch.randn(n, generator=gen)).cuda(), (0.1 * torch.randn(n, generator=gen)).cuda()
    f32, f16 = ops.linear_residual_layernorm(a, w, bias, resid, gamma, beta, 1e-12)
    t = ops.linear(a, w, bias, _lib.PE_EPI_F32)
    s32, l32, l16 = ops.residual_layernorm(t, resid, gamma, beta, 1e-12, want_sum=True, want_f32=True, want_f16=True)
    p32, _ = ops.linear_residual_layernorm(a, w, bias, resid, gamma, beta, 1e-12, f32_is_ln=True, want_f16=False)
    torch.cuda.synchronize()
    assert torch.equal(f32, s32.view(m, n)) and torch.equal(f16, l16.view(m, n)) and torch.equal(p32, l32.view(m, n)), (m, n, k)
    print('kernel ok', m, n, k, flush=True)
# 2. a pipeline's result does not depend on where it is cut (fused inside a stage, stand-alone at its edges)
for name, cls, cuts_list in (('test/vit-tiny', vit.ViTShardForImageClassification, ((12,), (5, 12), (2, 4, 6, 8, 10, 12))),
                             ('test/bert-tiny', bert.BertShardForSequenceClassification, ((12,), (7, 12), (2, 6, 12)))):
    spec = MODEL_SPECS[name]
    weights = synth_weights(spec, seed=0)
    x = synth_input(spec, 3, seed=5, seq_len=32)
    outs = []
    for cuts in cuts_list:
        data, lo = x, 1
        for hi in cuts:
            cfg = ModuleShardConfig(layer_start=lo, layer_end=hi, is_first=lo == 1, is_last=hi == spec.layers)
            data = cls(hf_config(spec), cfg, weights)(data)
            lo = hi + 1
        outs.append(data.cpu())
    for o in outs[1:]:
        assert torch.equal(o, outs[0]), name
    print('partition ok', name, flush=True)
print('all ok')
"""


def test_fused_layernorm_is_bit_identical_to_its_standalone_mirror(ops):
    """PE_FUSE_LN=1 (child process): the cluster epilogue and the chunked stand-alone LayerNorm share ln_dev.cuh, so the
    fused kernel equals GEMM + LayerNorm bit for bit, and a model's logits are the same for every partition."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, '-c', _FUSED_LN_CHECK, root], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and 'all ok' in res.stdout, res.stdout[-3000:] + res.stderr[-4000:]
