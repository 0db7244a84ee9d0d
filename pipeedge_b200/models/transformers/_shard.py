"""Common machinery of the ViT / DeiT / BERT shard classes: weight-file handling, payload staging on the
device, output-buffer rings for CUDA-graph replay, and the last-stage heads."""
from collections.abc import Mapping
from typing import Optional, Tuple, Union
import numpy as np
import torch
from ... import _lib, ops
from ..._lib import LIB, check
from .. import ModuleShard, ModuleShardConfig
from . import TransformerShardData
from ._stage import EncoderStage, _dev


class GpuTransformerShard(ModuleShard):
    """A shard whose encoder blocks (and edges) run through `libpipeedge_b200.so` on the current device.

    Constructor contract = the reference's (`vit.py:192-204`): `(config, shard_config, model_weights)` with
    `model_weights` an `.npz` path or an already-loaded mapping. `forward` takes/returns a tensor or the
    `(data, skip)` tuple of a mid-block cut (SURVEY.md 8a-A2); outputs are fp32 CUDA tensors.

    Attributes that tune the device path (not part of the reference API):
      use_cuda_graph  replay the stage's kernel sequence as one CUDA graph (needs stable buffers)
      num_slots       ring of persistent output buffers used when `use_cuda_graph` is on; an output is
                      overwritten `num_slots` forwards later, which matches the reference's pipeline depth of
                      queued + in-flight payloads (`p2p/__init__.py:374-376`)
    """
    FAMILY = ''

    def __init__(self, config, shard_config: ModuleShardConfig, model_weights: Union[str, Mapping]):
        super().__init__(config, shard_config)
        self.use_cuda_graph = False
        self.num_slots = 4
        self._static = False       # native pipeline capture: persistent buffers, eager launches
        self._static_parity = 0    # ... which of the two buffer sets (overlapped send: micro-batch index mod 2)
        self._static_defer = True  # ... leave a final residual add to the link's send kernel
        self._deferred = None      # (a, b) device addresses when the last static forward deferred its final add
        self._slot = 0
        self._slot_sent = {}       # ring slot -> CUDA event recorded once the hop has SENT what the slot held
        self._last_slot = None
        self._rings = {}
        self._copy_stream = None
        self._h2d_rings = {}
        self._h2d_count = {}
        self._pending_h2d = []
        if isinstance(model_weights, str):
            with np.load(model_weights) as weights:
                self._build_shard(weights)
        else:
            self._build_shard(model_weights)

    # ------------------------------------------------------------------ construction
    def _build_shard(self, weights: Mapping) -> None:
        raise NotImplementedError

    def _make_stage(self, weights: Mapping, tokens: int, max_ubatch: int = 64) -> EncoderStage:
        return EncoderStage(self.FAMILY, self.config, self.shard_config.layer_start, self.shard_config.layer_end,
                            weights, tokens, max_ubatch)

    @staticmethod
    def _f16(arr, device) -> torch.Tensor:
        return _dev(arr, torch.float16, device)

    @staticmethod
    def _f32(arr, device) -> torch.Tensor:
        return _dev(arr, torch.float32, device)

    # ------------------------------------------------------------------ payload staging
    def _to_device(self, data: TransformerShardData, dtype=torch.float32) -> TransformerShardData:
        if isinstance(data, torch.Tensor):
            return self._one_to_device(data, dtype, 0)
        return tuple(self._one_to_device(t, dtype, i) for i, t in enumerate(data))

    def _one_to_device(self, t: torch.Tensor, dtype, pos: int) -> torch.Tensor:
        dev = self.stage.device
        if t.is_cuda:
            return t.to(device=dev, dtype=dtype).contiguous()
        # Host input (the data rank's images / token ids): copy on a side stream into a small ring of device
        # buffers so that the H2D of micro-batch i+1 overlaps the kernels of micro-batch i. Replaces
        # `devices.forward_pre_hook_to_device` (`devices.py:8-16`); pinned host memory makes it truly async.
        if self._copy_stream is None:
            self._copy_stream = torch.cuda.Stream(device=dev)
        key = ('h2d', pos, tuple(t.shape), dtype)
        ring = self._h2d_rings.setdefault(key, [])
        idx = self._h2d_count.get(key, 0)
        self._h2d_count[key] = idx + 1
        if len(ring) < 4:
            ring.append([torch.empty(t.shape, dtype=dtype, device=dev), None])
        slot = ring[idx % 4]
        buf, last_use = slot
        compute = torch.cuda.current_stream()
        with torch.cuda.stream(self._copy_stream):
            if last_use is not None:
                self._copy_stream.wait_event(last_use)   # kernels that read this buffer 4 forwards ago are done
            buf.copy_(t if t.dtype == dtype else t.to(dtype), non_blocking=True)
            done = torch.cuda.Event()
            done.record(self._copy_stream)
        compute.wait_event(done)
        self._pending_h2d.append(slot)
        return buf

    def _mark_inputs_consumed(self) -> None:
        """Record, on the compute stream, that the kernels reading the current host-staged inputs were enqueued."""
        if self._pending_h2d:
            evt = torch.cuda.Event()
            evt.record(torch.cuda.current_stream())
            for slot in self._pending_h2d:
                slot[1] = evt
            self._pending_h2d.clear()

    def _ring(self, name: str, shape, dtype=torch.float32) -> torch.Tensor:
        """Persistent buffer `name` of the current slot (allocated on first use per shape)."""
        key = (name, tuple(shape), dtype, ('static', self._static_parity) if self._static else self._slot)
        buf = self._rings.get(key)
        if buf is None:
            buf = torch.empty(tuple(shape), dtype=dtype, device=self.stage.device)
            self._rings[key] = buf
        return buf

    @property
    def persistent(self) -> bool:
        """Whether forward outputs live in persistent buffers (either graph mode)."""
        return self.use_cuda_graph or self._static

    def _tmp(self, name: str, shape, dtype=torch.float32) -> torch.Tensor:
        """A small edge / head buffer: persistent while the native pipeline captures (`_static`), fresh otherwise (the
        per-call graph mode hands results to queues that may still hold them `num_slots` forwards later)."""
        if self._static:
            return self._ring(name, shape, dtype)
        return torch.empty(tuple(shape), dtype=dtype, device=self.stage.device)

    def _stage_out(self, ubatch: int) -> Optional[Tuple[torch.Tensor, Optional[torch.Tensor]]]:
        if not self.persistent:
            return None
        s0, s1 = self.stage.out_shapes(ubatch)
        return self._ring('out0', s0), (None if s1 is None else self._ring('out1', s1))

    def _run_blocks(self, data: TransformerShardData) -> TransformerShardData:
        in0 = data[0] if isinstance(data, tuple) else data
        self.stage.ensure_shape(in0)   # BERT: the sequence length is the input's; output rings are sized after this
        out = self._stage_out(in0.shape[0])
        if self._static:
            # captured by the native pipeline: plain launches; a non-final stage that ends on a projection leaves its
            # last residual add to the link's send kernel
            res = self.stage.forward(data, out=out, defer_add=self._static_defer and not self.shard_config.is_last)
            self._deferred = self.stage.deferred()
            return res
        if self.use_cuda_graph:
            sent = self._slot_sent.pop(self._slot, None)
            if sent is not None:    # the hop may still be sending what this slot held num_slots forwards ago
                torch.cuda.current_stream().wait_event(sent)
        res = self.stage.forward(data, out=out, use_graph=self.use_cuda_graph)
        self._mark_inputs_consumed()
        if self.use_cuda_graph:
            self._last_slot = self._slot
            self._slot = (self._slot + 1) % max(1, self.num_slots)
        return res

    def output_guard(self):
        """Called by the stage's work thread after a forward: returns `on_sent(event)` through which the send thread
        reports when the hop has finished with the forward's output buffers (None when outputs are not ring buffers)."""
        inner = self._inner()
        if not inner.use_cuda_graph or inner._last_slot is None:   # pylint: disable=protected-access
            return None
        slot = inner._last_slot                                    # pylint: disable=protected-access

        def on_sent(event, slot=slot, inner=inner):
            if event is not None:
                inner._slot_sent[slot] = event                     # pylint: disable=protected-access
        return on_sent

    # ------------------------------------------------------------------ native pipeline (comm/p2p/_native.py)
    def _inner(self) -> 'GpuTransformerShard':
        """The shard that owns the stage (classification shards wrap a model shard)."""
        return self

    def native_input_spec(self, ubatch: int, dim1: int):
        """[(shape, dtype)] of the persistent input buffer(s) for micro-batches of `ubatch` items."""
        stage = self.stage
        if self.shard_config.is_first:
            return [self._first_input_spec(ubatch, dim1)]
        tokens = dim1 or stage.tokens
        spec = [((ubatch, tokens, stage.inter if stage.first_sub == 3 else stage.hidden), torch.float32)]
        if stage.in_is_tuple:
            spec.append(((ubatch, tokens, stage.hidden), torch.float32))
        return spec

    def _first_input_spec(self, ubatch: int, dim1: int):
        raise NotImplementedError

    def native_out_bytes(self, max_ubatch: int, max_tokens: int) -> int:
        """Upper bound of this shard's output payload (fp32 on the wire) for sizing the downstream link's slots."""
        stage = self.stage
        if self.shard_config.is_last:
            n = 1
            for d in self.native_result_item_shape():
                n *= d
            return max_ubatch * n * 4 + 4096
        widths = {0: 2 * stage.hidden, 2: stage.inter + stage.hidden}.get(stage.last_sub, stage.hidden)
        return max_ubatch * max_tokens * widths * 4 + 8192

    def native_payload_shapes(self):
        """{(items, (elements per item of each output tensor))} for every input shape `native_forward` has run: the
        payloads the stage's graphs send (the record consumers of the native pipeline map a record back to one)."""
        keep = list(getattr(self, '_native_keep', {}).values())   # one C-level copy: a capture may add to it meanwhile
        return {(outs[0].shape[0], tuple(t.numel() // outs[0].shape[0] for t in outs)) for outs in keep}

    def native_max_tokens(self) -> int:
        """Largest sequence length a payload can have."""
        return self.stage.tokens

    def native_result_item_shape(self):
        """Per-item shape of the LAST stage's output for this model (known on every rank from the config)."""
        raise NotImplementedError

    def native_needs_resize(self, ubatch: int, dim1: int) -> bool:
        return self.stage.needs_resize(ubatch, dim1 or self.stage.tokens)

    def native_forward(self, inputs, parity: int = 0, defer: bool = True):
        """One forward on persistent buffers for graph capture (no hooks, no allocation after the first call per
        shape and parity): returns [(a, b or None, elements per item)] device addresses of the output payload (a + b).
        `parity` picks one of two output buffer sets (a send that overlaps the next micro-batch reads set i mod 2 while
        the stage writes the other); `defer` leaves a final residual add to the send kernel (needs the single set)."""
        inner = self._inner()
        prev = (self._static, inner._static)
        self._static = inner._static = True
        self._static_parity = inner._static_parity = parity
        self._static_defer = inner._static_defer = defer
        inner._deferred = None
        try:
            data = inputs[0] if len(inputs) == 1 else tuple(inputs)
            out = self.forward(data)
            outs = out if isinstance(out, tuple) else (out,)
            ubatch = inputs[0].shape[0]
            self._native_keep = getattr(self, '_native_keep', {})
            self._native_keep[(tuple(inputs[0].shape), parity)] = outs   # the graphs write into these for as long as they live
            if inner._deferred is not None and len(outs) == 1:
                a, b = inner._deferred
                return [(a, b, outs[0].numel() // ubatch)]
            for t in outs:
                if t.dtype != torch.float32 or not t.is_contiguous():
                    raise RuntimeError("native pipeline: stage outputs must be contiguous fp32 tensors")
            return [(t.data_ptr(), None, t.numel() // ubatch) for t in outs]
        finally:
            self._static, inner._static = prev

    # ------------------------------------------------------------------ heads
    def _cls_rows(self, data: torch.Tensor, dtype=torch.float32, name: str = 'cls_rows') -> torch.Tensor:
        """Row 0 of every item ([CLS]), gathered (and cast) into a contiguous buffer."""
        buf = self._tmp(name, (data.shape[0], data.shape[2]), dtype)
        buf.copy_(data[:, 0, :])
        return buf

    def _classify(self, a16: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
        out = self._tmp('logits', (a16.shape[0], weight.shape[0]))
        return ops.linear(a16, weight, bias, _lib.PE_EPI_F32, out=out)
