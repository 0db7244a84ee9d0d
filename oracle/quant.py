"""CPU oracle: QuantPipe clamp / quantise / bit-pack - TEST INFRASTRUCTURE (see oracle/__init__.py).

NumPy restatement of `pipeedge/quantization/basic_op.py` and `clamp_op.py`, plus the two runtime
hooks that drive them (`runtime.py:73-119`). Integer codes, scales and shifts produced here are
the bit-exact target for the CUDA path.
"""
import math
from typing import List, Optional, Sequence, Tuple
import numpy as np
import torch
from scipy.special import lambertw


def clamp_factor_laplace(bit: int) -> np.float32:
    """`_clamp_factor_laplace` (`clamp_op.py:22-24`): W(3*4^bit), float64 -> float32 via `.to(tensor)`."""
    return np.float32(lambertw(3.0 * 4.0 ** bit).real)


def clamp_factor_gelu(bit: int) -> np.float32:
    """`_clamp_factor_gelu` (`clamp_op.py:6-8`): W(3*4^(bit+1))."""
    return np.float32(lambertw(3.0 * 4.0 ** (bit + 1)).real)


def clamp_alpha(tensor: torch.Tensor, bit: int, kind: Optional[str] = None) -> Tuple[np.float32, str]:
    """Clamp threshold chosen by `forward_hook_quant_encode` (`runtime.py:84`) for a micro-batch.

    Laplace (`clamp_op.py:27-33`): alpha = W * sqrt(0.5 * var(x, biased)); GeLU (`:11-19`):
    var ~= 2 * sum(x^2) / n. All in fp32 after torch's own reductions. `kind` = 'laplace' / 'gelu' calls that clamp
    function directly (PE_CLAMP_LAPLACE / PE_CLAMP_GELU) instead of choosing by min(x) < 0.2.
    """
    if kind == 'laplace' or (kind is None and tensor.min() < 0.2):
        variance = torch.var(tensor, unbiased=False)
        factor, kind = clamp_factor_laplace(bit), 'laplace'
    else:
        variance = 2 * torch.pow(tensor, 2).sum() / torch.numel(tensor)
        factor, kind = clamp_factor_gelu(bit), 'gelu'
    dist = torch.sqrt(0.5 * variance)
    alpha = torch.tensor(factor, dtype=torch.float32) * dist
    return np.float32(alpha.item()), kind


def clamp(tensor: torch.Tensor, bit: int) -> torch.Tensor:
    """`clamp_banner2019_{laplace,gelu}` selected as in `runtime.py:84-85`."""
    alpha, _ = clamp_alpha(tensor, bit)
    return tensor.clamp(min=-float(alpha), max=float(alpha))


def enc_ratio(bit: int) -> int:
    """Codes per uint32 word (`basic_op.py:43`)."""
    return int(32 / bit)


def packed_words(n: int, bit: int) -> int:
    """uint32 words needed for `n` codes (`basic_op.py:48-50`)."""
    r = enc_ratio(bit)
    return (n + r - 1) // r


def quant_codes(item: np.ndarray, bit: int) -> Tuple[np.ndarray, np.float32, np.float32]:
    """Per-item affine quantisation (`tensor_encode`, `basic_op.py:124-132`, + `_quant_op`, `:17-21`).

    shift = min; scale = max(x - shift); code = around((x - shift) / scale * (2^bit - 1)), all fp32,
    round-half-even. Returns (uint32 codes, scale, shift).
    """
    item = np.asarray(item, dtype=np.float32)
    shift = item.min()
    centred = item - shift
    scale = centred.max()
    if scale == 0:
        return constant_item_codes(item)
    rescale = centred / scale
    assert np.all(rescale >= 0) and np.all(rescale <= 1)   # `_quant_op` asserts (NaN if scale == 0)
    levels = (1 << bit) - 1
    codes = np.around(levels * rescale).astype(np.uint32)
    return codes, np.float32(scale), np.float32(shift)


def constant_item_codes(item: np.ndarray) -> Tuple[np.ndarray, np.float32, np.float32]:
    """A constant item (scale 0; also an item the clamp maps entirely onto +-alpha): zero codes, scale 0, shift = the
    value, so that decoding (0 * 0 + shift) gives the value back. The reference trips its NaN assert here
    (`basic_op.py:12-13`); this is the deliberate deviation of DESIGN.md section 2, restated for the tests."""
    item = np.asarray(item, dtype=np.float32)
    return np.zeros(item.shape, dtype=np.uint32), np.float32(0.0), np.float32(item.min())


def pack_codes(codes: np.ndarray, bit: int) -> np.ndarray:
    """`_intmap_encode` (`basic_op.py:38-55`): LSB-first, floor(32/bit) codes per uint32, zero tail."""
    codes = codes.flatten()
    r = enc_ratio(bit)
    pad = (r - len(codes) % r) % r
    ext = np.append(codes, np.zeros(pad, dtype=np.uint32)).reshape(-1, r)
    shifts = np.array([(i % r) * bit for i in range(r)], dtype=np.uint32)
    return np.bitwise_or.reduce(np.left_shift(ext, shifts), axis=1, dtype=np.uint32)


def unpack_codes(words: np.ndarray, n: int, bit: int) -> np.ndarray:
    """`_intmap_decode` (`basic_op.py:58-90`) without the final reshape."""
    r = enc_ratio(bit)
    shifts = np.array([(i % r) * bit for i in range(r)], dtype=np.uint32)
    exploded = np.right_shift(np.repeat(words, r).reshape(-1, r), shifts).flatten()
    return np.bitwise_and(exploded, np.uint32(2 ** bit - 1))[:n]


def tensor_encode_outerdim(batched: torch.Tensor, bit: int) -> List[torch.Tensor]:
    """`tensor_encode_outerdim` (`basic_op.py:166-170`): the 5-tensor wire format per input tensor."""
    if bit == 0:
        b = batched.shape[0]
        return [batched, torch.tensor(batched.shape[1:]).expand(b, -1).clone(), torch.ones(b), torch.zeros(b),
                torch.zeros(b, dtype=torch.int8)]
    comm, scales, shifts = [], [], []
    for item in batched.numpy():
        codes, scale, shift = quant_codes(item, bit)
        comm.append(pack_codes(codes, bit).view(np.uint8))
        scales.append(scale)
        shifts.append(shift)
    b = batched.shape[0]
    return [torch.from_numpy(np.stack(comm, 0)),
            torch.tensor(batched.shape[1:], dtype=torch.int32).expand(b, -1).clone(),
            torch.tensor(np.array(scales, dtype=np.float32)),
            torch.tensor(np.array(shifts, dtype=np.float32)),
            torch.full((b,), bit, dtype=torch.int8)]


def tensor_decode_outerdim(enc: Sequence[torch.Tensor]) -> torch.Tensor:
    """`tensor_decode_outerdim` (`basic_op.py:173-176`, `tensor_decode` `:146-163`).

    value = float32(code / (2^bit - 1)) (float64 divide, then cast: `_intmap2float`, `:93-96`),
    then `* scale + shift` as two fp32 roundings.
    """
    comm, shape, scale, shift, bits = enc
    bit = int(bits[0])
    if bit == 0:
        return comm
    out = []
    for i in range(comm.shape[0]):
        dims = shape[i].tolist()
        words = comm[i].numpy().view(np.uint32)
        codes = unpack_codes(words, int(np.prod(dims)), bit)
        val = (codes / ((1 << bit) - 1)).astype(np.float32)
        val = (val * np.float32(scale[i].item()) + np.float32(shift[i].item())).astype(np.float32)
        out.append(torch.from_numpy(val.reshape(dims)))
    return torch.stack(out, 0)


def hook_encode(output, bit: int) -> tuple:
    """`forward_hook_quant_encode` (`runtime.py:73-91`) minus monitoring: clamp then encode each tensor."""
    if isinstance(output, torch.Tensor):
        output = (output,)
    comm = []
    for tensor in output:
        if bit > 0:
            tensor = clamp(tensor, bit)
        comm += tensor_encode_outerdim(tensor, bit)
    return tuple(comm)


def encode_given_alpha(x: torch.Tensor, bit: int, alpha) -> tuple:
    """`hook_encode` of one tensor with the clamp threshold given instead of computed: x clamped to [-alpha, alpha]
    (no clamp when alpha is +inf), then `tensor_encode_outerdim`. The GeLU branch's threshold depends in its last bits
    on the fp32 summation order (`clamp_alpha`), so a kernel's codes are held to the oracle at the kernel's own alpha."""
    a = float(np.float32(alpha))
    if not math.isinf(a):
        x = x.clamp(min=-a, max=a)
    return tuple(tensor_encode_outerdim(x, bit))


def hook_decode(tensors: tuple):
    """`forward_pre_hook_quant_decode` (`runtime.py:93-119`) minus monitoring."""
    assert len(tensors) % 5 == 0 and len(tensors) >= 5
    out = [tensor_decode_outerdim(tensors[i * 5:i * 5 + 5]) for i in range(len(tensors) // 5)]
    return out[0] if len(out) == 1 else tuple(out)
