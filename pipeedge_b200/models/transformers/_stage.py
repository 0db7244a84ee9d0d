"""Device-resident stage behind the ViT / DeiT / BERT shard classes.

Takes the reference's npz key layouts (`vit.py:120-159`, `deit.py:119-156`, `bert.py:104-140`), packs the
sub-layers this shard owns into an fp16/fp32 device arena laid out for the kernels (fused `[3H, H]` QKV
weight in `nn.Linear` = K-major order, fp32 biases and LayerNorm parameters), creates a `pe_stage` and
drives the stage-0 / last-stage edges through the same C-ABI.
"""
import ctypes
import math
from typing import List, Mapping, Optional, Tuple, Union
import numpy as np
import torch
from ... import _lib
from ..._lib import LIB, BlockWeights, StageDesc, check

ShardData = Union[torch.Tensor, Tuple[torch.Tensor, torch.Tensor]]


def sublayer_ranges(layer_start: int, layer_end: int) -> List[Tuple[int, int, int]]:
    """(block id, first sub-layer, last sub-layer) triples covered by 1-based `[layer_start, layer_end]`."""
    out = []
    cur = layer_start
    last_block = math.ceil(layer_end / 4) - 1
    while cur <= layer_end:
        block = math.ceil(cur / 4) - 1
        s0 = (cur - 1) % 4
        s1 = (layer_end - 1) % 4 if block == last_block else 3
        out.append((block, s0, s1))
        cur += s1 - s0 + 1
    return out


def _dev(arr, dtype: torch.dtype, device) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(arr)).to(device=device, dtype=dtype).contiguous()


# ---------------------------------------------------------------------------------------------------
# Family-specific readers: npz layout -> canonical numpy arrays in nn.Linear ([out, in]) orientation.
# ---------------------------------------------------------------------------------------------------
def _vit_block(w: Mapping, i: int, hidden: int, subs) -> dict:
    root = f"Transformer/encoderblock_{i}/"
    att = root + "MultiHeadDotProductAttention_1/"
    p = {}
    if 0 in subs:
        p['ln1_w'], p['ln1_b'] = w[root + "LayerNorm_0/scale"], w[root + "LayerNorm_0/bias"]
        # JAX kernels are [in, heads, d]: flatten heads and transpose to [out, in]
        p['w_qkv'] = np.concatenate([np.asarray(w[att + n + "/kernel"]).reshape(hidden, hidden).T
                                     for n in ("query", "key", "value")], axis=0)
        p['b_qkv'] = np.concatenate([np.asarray(w[att + n + "/bias"]).reshape(-1) for n in ("query", "key", "value")])
    if 1 in subs:
        p['w_o'] = np.asarray(w[att + "out/kernel"]).reshape(hidden, hidden).T
        p['b_o'] = np.asarray(w[att + "out/bias"]).reshape(-1)
    if 2 in subs:
        p['ln2_w'], p['ln2_b'] = w[root + "LayerNorm_2/scale"], w[root + "LayerNorm_2/bias"]
        p['w_fc1'] = np.asarray(w[root + "MlpBlock_3/Dense_0/kernel"]).T
        p['b_fc1'] = w[root + "MlpBlock_3/Dense_0/bias"]
    if 3 in subs:
        p['w_fc2'] = np.asarray(w[root + "MlpBlock_3/Dense_1/kernel"]).T
        p['b_fc2'] = w[root + "MlpBlock_3/Dense_1/bias"]
    return p


def _deit_block(w: Mapping, i: int, hidden: int, subs) -> dict:
    del hidden
    root = f"blocks.{i}."
    p = {}
    if 0 in subs:
        p['ln1_w'], p['ln1_b'] = w[root + "norm1.weight"], w[root + "norm1.bias"]
        p['w_qkv'], p['b_qkv'] = w[root + "attn.qkv.weight"], w[root + "attn.qkv.bias"]  # already [Wq; Wk; Wv]
    if 1 in subs:
        p['w_o'], p['b_o'] = w[root + "attn.proj.weight"], w[root + "attn.proj.bias"]
    if 2 in subs:
        p['ln2_w'], p['ln2_b'] = w[root + "norm2.weight"], w[root + "norm2.bias"]
        p['w_fc1'], p['b_fc1'] = w[root + "mlp.fc1.weight"], w[root + "mlp.fc1.bias"]
    if 3 in subs:
        p['w_fc2'], p['b_fc2'] = w[root + "mlp.fc2.weight"], w[root + "mlp.fc2.bias"]
    return p


def _bert_block(w: Mapping, i: int, hidden: int, subs) -> dict:
    del hidden
    root = f"encoder.layer.{i}."
    p = {}
    if 0 in subs:
        p['w_qkv'] = np.concatenate([w[root + f"attention.self.{n}.weight"] for n in ("query", "key", "value")], axis=0)
        p['b_qkv'] = np.concatenate([w[root + f"attention.self.{n}.bias"] for n in ("query", "key", "value")])
    if 1 in subs:
        p['w_o'], p['b_o'] = w[root + "attention.output.dense.weight"], w[root + "attention.output.dense.bias"]
        p['ln1_w'], p['ln1_b'] = w[root + "attention.output.LayerNorm.weight"], w[root + "attention.output.LayerNorm.bias"]
    if 2 in subs:
        p['w_fc1'], p['b_fc1'] = w[root + "intermediate.dense.weight"], w[root + "intermediate.dense.bias"]
    if 3 in subs:
        p['w_fc2'], p['b_fc2'] = w[root + "output.dense.weight"], w[root + "output.dense.bias"]
        p['ln2_w'], p['ln2_b'] = w[root + "output.LayerNorm.weight"], w[root + "output.LayerNorm.bias"]
    return p


_BLOCK_READERS = {'vit': _vit_block, 'deit': _deit_block, 'bert': _bert_block}
_F16_KEYS = ('w_qkv', 'w_o', 'w_fc1', 'w_fc2')


class EncoderStage:
    """The encoder blocks `[layer_start, layer_end]` of one shard on the current CUDA device."""

    def __init__(self, family: str, config, layer_start: int, layer_end: int, weights: Mapping, tokens: int,
                 max_ubatch: int = 64):
        if not torch.cuda.is_available():
            raise RuntimeError("pipeedge_b200 shards need a CUDA (sm_90a) device: there is no CPU fallback")
        self.family = family
        self.hidden = int(config.hidden_size)
        self.heads = int(config.num_attention_heads)
        self.inter = int(config.intermediate_size)
        self.eps = float(config.layer_norm_eps)
        self.tokens = int(tokens)
        self.layer_start, self.layer_end = int(layer_start), int(layer_end)
        self.max_ubatch = int(max_ubatch)
        self.device = torch.device('cuda', torch.cuda.current_device())
        self.ranges = sublayer_ranges(self.layer_start, self.layer_end)
        self.first_sub, self.last_sub = self.ranges[0][1], self.ranges[-1][2]
        self._tensors = []   # keeps the device arena alive
        blocks = (BlockWeights * len(self.ranges))()
        for idx, (block, s0, s1) in enumerate(self.ranges):
            packed = _BLOCK_READERS[family](weights, block, self.hidden, range(s0, s1 + 1))
            for key, arr in packed.items():
                t = _dev(arr, torch.float16 if key in _F16_KEYS else torch.float32, self.device)
                self._tensors.append(t)
                setattr(blocks[idx], key, t.data_ptr())
        self._blocks = blocks
        self._stamps = None   # (stamps, row_ctr, col0) of set_stamps
        self._handle = ctypes.c_void_p()
        self._create()

    def _create(self) -> None:
        desc = StageDesc(_lib.PE_FAMILY[self.family], self.hidden, self.heads, self.inter, self.tokens, self.eps,
                         self.layer_start, self.layer_end, self.max_ubatch)
        check(LIB.pe_stage_create(ctypes.byref(desc), self._blocks, len(self.ranges), ctypes.byref(self._handle)))
        if self._stamps is not None:
            self.set_stamps(*self._stamps)

    @staticmethod
    def _check_stamp_table(stamps: torch.Tensor, row_ctr: torch.Tensor) -> None:
        if not (stamps.is_cuda and stamps.dtype == torch.int64 and stamps.dim() == 2 and stamps.is_contiguous()):
            raise ValueError("stamps must be a contiguous int64 CUDA tensor [rows, cols]")
        if not (row_ctr.is_cuda and row_ctr.dtype == torch.int64 and row_ctr.numel() >= 1):
            raise ValueError("row_ctr must be an int64 CUDA tensor of one element")

    def set_stamps(self, stamps: Optional[torch.Tensor], row_ctr: Optional[torch.Tensor] = None, col0: int = 0) -> None:
        """Timestamp every later forward after each sub-layer k of the stage: %globaltimer (ns) into
        `stamps[row_ctr[0], col0 + k]`; the stamp in the last column advances `row_ctr[0]` (pe_stage_set_stamps).
        `stamps` is an int64 CUDA tensor [rows, cols], `row_ctr` an int64 CUDA tensor holding the next row; the stage
        keeps references to both. None turns stamps off."""
        if stamps is None:
            self._stamps = None
            check(LIB.pe_stage_set_stamps(self._handle, None, None, 0, 0, 0))
            return
        self._check_stamp_table(stamps, row_ctr)
        check(LIB.pe_stage_set_stamps(self._handle, stamps.data_ptr(), row_ctr.data_ptr(), stamps.shape[0],
                                      stamps.shape[1], int(col0)))
        self._stamps = (stamps, row_ctr, int(col0))

    @staticmethod
    def stamp(stamps: torch.Tensor, row_ctr: torch.Tensor, col: int, bump_row: bool = False) -> None:
        """One stand-alone stamp on the current stream into `stamps[row_ctr[0], col]`, then advance the row if
        `bump_row` (pe_stamp): what a shard charges to its first / last sub-layer outside the stage (embeddings, head)."""
        EncoderStage._check_stamp_table(stamps, row_ctr)
        check(LIB.pe_stamp(stamps.data_ptr(), row_ctr.data_ptr(), stamps.shape[0], stamps.shape[1], int(col),
                           1 if bump_row else 0, torch.cuda.current_stream().cuda_stream))

    def resize(self, tokens: int, max_ubatch: int) -> None:
        """Re-create the workspace for a different sequence length / micro-batch bound (BERT inputs vary)."""
        self.close()
        self.tokens, self.max_ubatch = int(tokens), int(max_ubatch)
        self._handle = ctypes.c_void_p()
        self._create()

    def needs_resize(self, ubatch: int, tokens: int) -> bool:
        """Whether a payload of `ubatch` items of `tokens` tokens would re-create the workspace (which invalidates
        every CUDA graph captured over it)."""
        return tokens != self.tokens or ubatch > self.max_ubatch

    def ensure_shape(self, in0: torch.Tensor) -> None:
        """Adopt the payload's sequence length / micro-batch (callers must do this BEFORE sizing output buffers)."""
        if in0.shape[1] != self.tokens or in0.shape[0] > self.max_ubatch:
            self.resize(in0.shape[1], max(in0.shape[0], self.max_ubatch))

    def close(self) -> None:
        """Release the library-owned workspace."""
        if getattr(self, '_handle', None) is not None and self._handle.value:
            LIB.pe_stage_destroy(self._handle)
            self._handle = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:  # pylint: disable=broad-except
            pass

    @property
    def in_is_tuple(self) -> bool:
        """Whether the stage starts mid-block and consumes a (data, skip) tuple."""
        return self.first_sub in (1, 3)

    @property
    def out_is_tuple(self) -> bool:
        """Whether the stage ends mid-block and produces a (data, skip) tuple."""
        return self.last_sub in (0, 2)

    def out_shapes(self, ubatch: int):
        """Shapes of (out0, out1 or None) for `ubatch` items."""
        skip = (ubatch, self.tokens, self.hidden)
        if self.last_sub == 0:
            return skip, skip
        if self.last_sub == 2:
            return (ubatch, self.tokens, self.inter), skip
        return skip, None

    def deferred(self) -> Optional[Tuple[int, int]]:
        """Device addresses (a, b) when the last forward left its final residual add to the consumer (output =
        a + b, see PE_STAGE_DEFER_ADD), else None."""
        a, b = ctypes.c_void_p(), ctypes.c_void_p()
        check(LIB.pe_stage_deferred(self._handle, ctypes.byref(a), ctypes.byref(b)))
        return (a.value, b.value) if a.value else None

    def forward(self, data: ShardData, out: Optional[Tuple[torch.Tensor, Optional[torch.Tensor]]] = None,
                use_graph: bool = False, defer_add: bool = False) -> ShardData:
        """Run the blocks on fp32 CUDA payload(s); `out` supplies persistent output buffers (graph replay).
        `defer_add` (eager launches only): a stage ending on a projection skips its last residual add - read the two
        addends with `deferred()` (the link's send kernel adds while it reads)."""
        if self.in_is_tuple:
            in0, in1 = data
        else:
            in0, in1 = data, None
        ubatch = in0.shape[0]
        self.ensure_shape(in0)
        for t in (in0, in1):
            if t is not None and (not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous()):
                raise ValueError("EncoderStage.forward: payloads must be contiguous fp32 CUDA tensors")
        if out is None:
            s0, s1 = self.out_shapes(ubatch)
            out = (torch.empty(s0, dtype=torch.float32, device=self.device),
                   None if s1 is None else torch.empty(s1, dtype=torch.float32, device=self.device))
        out0, out1 = out
        check(LIB.pe_stage_forward(self._handle, in0.data_ptr(), None if in1 is None else in1.data_ptr(),
                                   out0.data_ptr(), None if out1 is None else out1.data_ptr(), ubatch,
                                   1 if use_graph else (_lib.PE_STAGE_DEFER_ADD if defer_add else 0),
                                   torch.cuda.current_stream().cuda_stream))
        return (out0, out1) if self.out_is_tuple else out0

    KERNEL_KINDS = ('cast', 'layernorm', 'gemm_qkv', 'attention', 'gemm_out', 'gemm_fc1', 'gemm_fc2')

    def profile(self, data: ShardData):
        """One eager forward with a CUDA event after every kernel: list of (kind, milliseconds)."""
        in0, in1 = data if self.in_is_tuple else (data, None)
        ubatch = in0.shape[0]
        s0, s1 = self.out_shapes(ubatch)
        out0 = torch.empty(s0, dtype=torch.float32, device=self.device)
        out1 = None if s1 is None else torch.empty(s1, dtype=torch.float32, device=self.device)
        cap = 16 * len(self.ranges) + 8
        ms = (ctypes.c_float * cap)()
        kinds = (ctypes.c_int * cap)()
        n = ctypes.c_int(0)
        check(LIB.pe_stage_profile(self._handle, in0.data_ptr(), None if in1 is None else in1.data_ptr(),
                                   out0.data_ptr(), None if out1 is None else out1.data_ptr(), ubatch,
                                   torch.cuda.current_stream().cuda_stream, ms, kinds, cap, ctypes.byref(n)))
        return [(self.KERNEL_KINDS[kinds[i]], float(ms[i])) for i in range(min(n.value, cap))]

    def kernel_count(self) -> int:
        """Kernels enqueued by the last forward."""
        return int(LIB.pe_stage_kernel_count(self._handle))
