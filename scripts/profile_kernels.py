"""One launch of every kernel on the hot path at BASELINE shapes, bracketed by cudaProfilerStart/Stop, for

    ncu --set full --clock-control none --import-source on --profile-from-start off -o kernels \
        python scripts/profile_kernels.py

ViT-B micro-batch 8 (M = 1576): LayerNorm (+ residual), the four wgmma GEMMs, attention, patch embedding (im2col + GEMM +
prefix rows); BASELINE config 5's hop [32, 198, 768] at 8 bits: the three stand-alone quant kernels, decode, the fused
quantise-and-send and the receive kernel of a link, the raw send / receive; BERT embedding [32, 128]."""
import ctypes
import os
import sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pipeedge_b200 import _lib, ops  # noqa: E402
from pipeedge_b200._lib import LIB, check  # noqa: E402

dev = torch.device('cuda', 0)
torch.cuda.set_device(dev)
g = torch.Generator(device=dev).manual_seed(0)
B, S, H, I, NH = 8, 197, 768, 3072, 12
M = B * S
x = torch.randn(M, H, device=dev, generator=g)
r = torch.randn(M, H, device=dev, generator=g)
gam, bet = torch.ones(H, device=dev), torch.zeros(H, device=dev)
a16 = torch.randn(M, H, device=dev, generator=g).half()
i16 = torch.randn(M, I, device=dev, generator=g).half()
w_qkv = (torch.randn(3 * H, H, device=dev, generator=g) * 0.02).half()
w_o = (torch.randn(H, H, device=dev, generator=g) * 0.02).half()
w_fc1 = (torch.randn(I, H, device=dev, generator=g) * 0.02).half()
w_fc2 = (torch.randn(H, I, device=dev, generator=g) * 0.02).half()
b3, b1, bi = torch.zeros(3 * H, device=dev), torch.zeros(H, device=dev), torch.zeros(I, device=dev)
qkv = (torch.randn(M, 3 * H, device=dev, generator=g) * 1.5).half()
hop = torch.randn(32, 198, 768, device=dev, generator=g) * 1.7
skip = torch.randn(32, 198, 768, device=dev, generator=g) * 0.3
act8 = torch.randn(8, 197, 768, device=dev, generator=g)
ids = torch.randint(0, 30522, (32, 128), device=dev)

loop = ctypes.c_void_p()
check(LIB.pe_link_open_local(hop.numel() * 4 + 4096, 4, 8, ctypes.byref(loop)))
dst = torch.empty_like(hop)
dst8 = torch.empty_like(act8)
stream = torch.cuda.current_stream().cuda_stream


def once():
    ops.residual_layernorm(x, r, gam, bet, 1e-12)                               # layernorm_kernel (+ residual, f16 out)
    ops.layernorm(x, gam, bet, 1e-12, want_f32=False, want_f16=True)           # layernorm_kernel (plain)
    ops.linear(a16, w_qkv, b3, _lib.PE_EPI_F16, static_w=True)                 # gemm<F16>      QKV
    ops.attention(qkv, B, S, NH)                                               # attention
    ops.linear(a16, w_o, b1, _lib.PE_EPI_F32, static_w=True)                   # gemm<F32>      out-proj
    ops.linear(a16, w_fc1, bi, _lib.PE_EPI_GELU_F16, static_w=True)            # gemm<GELU_F16> FC1
    ops.linear(i16, w_fc2, b1, _lib.PE_EPI_F32, static_w=True)                 # gemm<F32>      FC2
    c, sc, sh, _ = ops.quant_encode(hop, 8, True)                              # quant_stats / finalize / pack16
    ops.quant_decode(c, hop.shape[1:], 8, sc, sh)                              # quant_decode
    check(LIB.pe_link_put(loop, hop.data_ptr(), skip.data_ptr(), 198 * 768, None, None, 0, 32, 8, _lib.PE_CLAMP_AUTO, stream))
    check(LIB.pe_link_get(loop, dst.data_ptr(), None, 32, 198 * 768, 0, stream))                       # fused send + receive
    check(LIB.pe_link_put(loop, act8.data_ptr(), None, 197 * 768, None, None, 0, 8, 0, 0, stream))
    check(LIB.pe_link_get(loop, dst8.data_ptr(), None, 8, 197 * 768, 0, stream))                       # raw send + receive
    torch.cuda.synchronize()


from pipeedge_b200.models import ModuleShardConfig  # noqa: E402
from pipeedge_b200.models.transformers import bert, vit  # noqa: E402
from pipeedge_b200.synth import MODEL_SPECS, hf_config, synth_input, synth_weights  # noqa: E402
vspec = MODEL_SPECS['google/vit-base-patch16-224']
vshard = vit.ViTShardForImageClassification(hf_config(vspec), ModuleShardConfig(layer_start=1, layer_end=2, is_first=True,
                                                                               is_last=False), synth_weights(vspec, seed=0))
bspec = MODEL_SPECS['textattack/bert-base-uncased-CoLA']
bshard = bert.BertShardForSequenceClassification(hf_config(bspec), ModuleShardConfig(layer_start=1, layer_end=2, is_first=True,
                                                                                    is_last=False), synth_weights(bspec, seed=0))
pix = synth_input(vspec, 8, seed=1).to(dev)

once()
vshard.vit._embed(pix)
bshard.bert._embed(ids)
torch.cuda.synchronize()
torch.cuda.profiler.start()
once()
vshard.vit._embed(pix)      # im2col_patches_kernel + gemm<RESID_F32> + prefix_rows_kernel
bshard.bert._embed(ids)     # bert_embed_kernel
torch.cuda.synchronize()
torch.cuda.profiler.stop()
LIB.pe_link_close(loop)
print('profiled')
