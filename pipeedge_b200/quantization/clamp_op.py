"""Banner-2019 clamps on the device - drop-in for `pipeedge.quantization.clamp_op` (reference `clamp_op.py`).

The pipeline never calls these directly on the native path (the clamp is fused into the encode kernels, see
`basic_op.tensor_encode_outerdim(clamp=True)`); they exist for API parity and tests. The threshold comes
from the library's statistics kernels; only the final elementwise min/max uses torch."""
import torch
from .. import _lib
from .._lib import LIB, check


def _alpha(tensor: torch.Tensor, bit: int, kind: int) -> torch.Tensor:
    if not tensor.is_cuda or tensor.dtype != torch.float32:
        raise ValueError("clamp: expected an fp32 CUDA tensor")
    x = tensor.contiguous()
    items = x.shape[0] if x.dim() > 1 else 1
    n = x.numel() // items
    dev = x.device
    scale = torch.empty(items, dtype=torch.float32, device=dev)
    shift = torch.empty(items, dtype=torch.float32, device=dev)
    alpha = torch.empty(1, dtype=torch.float32, device=dev)
    work = torch.empty(LIB.pe_quant_workspace_bytes(items, n), dtype=torch.uint8, device=dev)
    check(LIB.pe_quant_alpha(x.data_ptr(), items, n, int(bit), kind, scale.data_ptr(), shift.data_ptr(),
                             alpha.data_ptr(), work.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return alpha


def clamp_banner2019_laplace(tensor: torch.Tensor, bit: int) -> torch.Tensor:
    """Clamp to +-W(3*4^bit)*sqrt(var/2) (`clamp_op.py:27-33`)."""
    alpha = _alpha(tensor, bit, _lib.PE_CLAMP_LAPLACE)
    return torch.minimum(torch.maximum(tensor, -alpha), alpha)


def clamp_banner2019_gelu(tensor: torch.Tensor, bit: int) -> torch.Tensor:
    """Like the Laplace clamp but for a GeLU output's half bell curve (`clamp_op.py:11-19`)."""
    alpha = _alpha(tensor, bit, _lib.PE_CLAMP_GELU)
    return torch.minimum(torch.maximum(tensor, -alpha), alpha)
