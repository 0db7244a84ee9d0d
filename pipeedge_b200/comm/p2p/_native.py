"""Native pipeline stage: the body of `DistP2pPipelineStage` when every rank drives a native shard.

The reference's stage is three Python threads handing each micro-batch through queues (`p2p/__init__.py:261-295,
373-394`). Here a stage's micro-batch is ONE CUDA graph (link get -> shard kernels -> link put, `csrc/pipe.cu`) and the
per-micro-batch host work runs in C with the GIL released:

* data rank: `enqueue_tensor` -> `pe_pipe_submit` (copy into the host-fed input ring on a side stream, graph launch,
  ticket to the next rank); a results thread blocks in `pe_pipe_next_result` and calls `results_cb` with each result;
* other ranks: one thread sits in `pe_pipe_run` (ticket in -> graph launch -> ticket out) until the pipeline closes.

Activations cross hops as peer-memory stores synchronised by device-polled flags (`csrc/link.cu`); QuantPipe
quantisation (`-q`, the shard's `quant_bit` buffer) is fused into the send kernel and undone by the receive kernel, so
the Python quantisation hooks (`runtime.py:73-119`) are represented by those kernels rather than called. Python runs
once per (micro-batch size, sequence length): to capture the graph.
"""
import collections
import ctypes
import logging
import os
import threading
from typing import Callable, Optional
import torch
import torch.distributed as dist
from ... import _lib
from ..._lib import LIB, check

logger = logging.getLogger(__name__)


def max_ubatch() -> int:
    """Largest micro-batch the links' slots are sized for (`PIPEEDGE_MAX_UBATCH`, default 64)."""
    return max(1, int(os.environ.get('PIPEEDGE_MAX_UBATCH', '64')))


def link_slots() -> int:
    """Slots per link ring (`PIPEEDGE_LINK_SLOTS`, default 4): payloads a producer may run ahead of its consumer."""
    return min(8, max(2, int(os.environ.get('PIPEEDGE_LINK_SLOTS', '4'))))


def drain_barrier(seconds: float = 120.0) -> None:
    """Barrier over the control plane that gives up (instead of hanging) when a rank has died."""
    import datetime   # pylint: disable=import-outside-toplevel
    try:
        dist.monitored_barrier(timeout=datetime.timedelta(seconds=seconds))
    except RuntimeError:
        logger.exception("native pipeline: a rank did not reach the drain barrier")


def overlap_send() -> bool:
    """Whether a stage's send runs on its own stream and overlaps the next micro-batch (`PIPEEDGE_OVERLAP_SEND`, default
    on): the stage then alternates between two output buffer sets and always materialises its output (no residual add
    left to the send kernel)."""
    return os.environ.get('PIPEEDGE_OVERLAP_SEND', '1') != '0'


def hook_is_native(hook) -> bool:
    """Whether a module hook is represented by the native pipeline's kernels (quantisation encode / decode) or is a
    no-op there (device placement, disabled monitoring): marked by `_pe_native` (a bool or a callable)."""
    flag = getattr(hook, '_pe_native', None)
    return bool(flag() if callable(flag) else flag)


def shard_is_native(shard) -> bool:
    """A native shard whose registered hooks the native pipeline accounts for."""
    from ...models.transformers._shard import GpuTransformerShard   # pylint: disable=import-outside-toplevel
    if not isinstance(shard, GpuTransformerShard):
        return False
    hooks = list(getattr(shard, '_forward_hooks', {}).values()) + list(getattr(shard, '_forward_pre_hooks', {}).values())
    return all(hook_is_native(h) for h in hooks)


class NativeStage:
    """One rank's stage on the native pipeline. `rank_src` / `rank_dst` as `DistP2pPipelineStage`; the data rank is the
    one with a `results_cb` (it must own the first shard)."""

    def __init__(self, rank_src: Optional[int], rank_dst: Optional[int], shard, results_cb: Optional[Callable]):
        self._rank_src, self._rank_dst = rank_src, rank_dst
        self._shard = shard
        self._results_cb = results_cb
        self._is_data = results_cb is not None
        self._device = torch.cuda.current_device()
        self._pipe = ctypes.c_void_p()
        self._links = []                      # every pe_link this rank opened (closed at shutdown)
        self._link_in = self._link_out = self._link_res = None
        self._socks = []
        self._inputs = {}                     # (ubatch, dim1) -> persistent input tensors
        self._keep = collections.deque(maxlen=link_slots() + 2)   # sources of in-flight input copies
        self._threads = []
        self._closed = False
        self._capture_lock = threading.Lock()
        self.exception: Optional[BaseException] = None
        self.graph_kernels = {}               # (ubatch, dim1) -> kernels per micro-batch
        self._result_shape = None
        self._captured_bit = None             # the QuantPipe bit-width the captured graphs send with
        self._quant_key, self._quant_val = None, 0
        self._stream = None
        self._copy_stream = None

    # ------------------------------------------------------------------ set-up
    def _open_link(self, sock, is_producer: bool, payload_bytes: int) -> ctypes.c_void_p:
        handle = ctypes.c_void_p()
        check(LIB.pe_link_open(sock.fileno(), 1 if is_producer else 0, payload_bytes if is_producer else 0,
                               link_slots() if is_producer else 0, self._quant()[0] if is_producer else 0,
                               ctypes.byref(handle)))
        self._links.append(handle)
        return handle

    def init(self, connect_to: Callable, accept_from: Callable) -> None:
        """Open this rank's links (hops in ascending order of the SENDER's rank, like the NCCL hops: opening blocks
        until the peer joins, a global order rules out circular waits), build the pipe, start the threads."""
        shard = self._shard
        ub, tokens = max_ubatch(), shard.native_max_tokens()
        out_bytes = shard.native_out_bytes(ub, tokens)
        rank = dist.get_rank() if dist.is_initialized() else 0
        hops = []
        if self._rank_dst is not None:
            hops.append((rank, 'send'))
        if self._rank_src is not None:
            hops.append((self._rank_src, 'recv'))
        peer_in = peer_out = None
        for _, kind in sorted(hops):
            if kind == 'send':
                sock = connect_to(self._rank_dst)
                self._socks.append(sock)
                peer_out = self._open_link(sock, True, out_bytes)
            else:
                sock = accept_from(self._rank_src)
                self._socks.append(sock)
                peer_in = self._open_link(sock, False, 0)
        if self._is_data:
            # inputs arrive from the host; results come back on the hop from the last stage (or a loop-back link)
            spec_shape, spec_dtype = shard.native_input_spec(ub, tokens)[0]
            in_bytes = torch.empty((), dtype=spec_dtype).element_size()
            for d in spec_shape:
                in_bytes *= int(d)
            handle = ctypes.c_void_p()
            check(LIB.pe_link_open_host(in_bytes, link_slots(), ctypes.byref(handle)))
            self._links.append(handle)
            self._link_in = handle
            if peer_out is None:
                loop = ctypes.c_void_p()
                check(LIB.pe_link_open_local(out_bytes, link_slots(), 0, ctypes.byref(loop)))
                self._links.append(loop)
                self._link_out = self._link_res = loop
            else:
                self._link_out, self._link_res = peer_out, peer_in
        else:
            self._link_in, self._link_out = peer_in, peer_out
        check(LIB.pe_pipe_create(self._link_in, self._link_out, self._link_res, ctypes.byref(self._pipe)))
        self._stream = torch.cuda.ExternalStream(LIB.pe_pipe_stream(self._pipe), device=self._device)
        self._copy_stream = torch.cuda.ExternalStream(LIB.pe_pipe_copy_stream(self._pipe), device=self._device)
        if shard.shard_config.is_last:
            n = 1
            for d in shard.native_result_item_shape():
                n *= int(d)
            check(LIB.pe_pipe_set_out_dim(self._pipe, n))
        if self._is_data:
            self._result_shape = tuple(int(d) for d in shard.native_result_item_shape())
            thr = threading.Thread(target=self._guard, args=(self._results_loop,), daemon=True, name='pe-results')
        else:
            thr = threading.Thread(target=self._guard, args=(self._run_loop,), daemon=True, name='pe-stage')
        self._threads.append(thr)
        thr.start()

    def _guard(self, fn) -> None:
        try:
            torch.cuda.set_device(self._device)
            fn()
        except BaseException as exc:   # pylint: disable=broad-except
            self.exception = exc       # re-raised on the owner by check_workers()
            logger.exception("native pipeline thread failed")

    # ------------------------------------------------------------------ graph capture
    def _quant(self):
        """(bit-width, clamp mode) this stage sends with: the shard's `quant_bit` buffer (`runtime.py:79`), 0 on the
        last stage. The tensor is converted once per object / in-place version, never per micro-batch (a CUDA-resident
        buffer would cost a device synchronisation each time)."""
        shard = self._shard
        if shard.shard_config.is_last or not hasattr(shard, 'quant_bit'):
            return 0, _lib.PE_CLAMP_NONE
        qb = shard.quant_bit
        key = (id(qb), getattr(qb, '_version', 0))
        if key != self._quant_key:
            self._quant_key, self._quant_val = key, int(qb)
        bit = self._quant_val
        return bit, (_lib.PE_CLAMP_AUTO if bit > 0 else _lib.PE_CLAMP_NONE)

    def invalidate(self) -> None:
        """Forget the captured graphs (they bake in the shard's `quant_bit` and buffer addresses): the next payload of
        each shape captures again. For callers that change a stage's bit-width between micro-batches by hand - the
        adaptive policies do it from forward hooks, which select the Python-thread path in the first place."""
        with self._capture_lock:
            check(LIB.pe_pipe_invalidate(self._pipe))
            self.graph_kernels.clear()

    def prepare(self, ubatch: int, dim1: int = 0) -> None:
        """Capture the graph for micro-batches of `ubatch` items (`dim1`: sequence length for BERT) ahead of the first
        payload, so that micro-batch 1 is already a replay."""
        if not LIB.pe_pipe_has_graph(self._pipe, ubatch, dim1):
            self._capture(ubatch, dim1)

    def _capture(self, ubatch: int, dim1: int) -> None:
        shard = self._shard
        with self._capture_lock:
            if LIB.pe_pipe_has_graph(self._pipe, ubatch, dim1):
                return
            if ubatch > max_ubatch():
                raise ValueError(f"micro-batch of {ubatch} items exceeds PIPEEDGE_MAX_UBATCH={max_ubatch()}")
            if shard.native_needs_resize(ubatch, dim1) and self.graph_kernels:
                check(LIB.pe_pipe_invalidate(self._pipe))   # the stage's workspace is about to be re-created
                self.graph_kernels.clear()
            bit, clamp = self._quant()
            overlap = overlap_send()
            with torch.cuda.stream(self._stream):
                ins = self._inputs.get((ubatch, dim1))
                if ins is None:     # zero-filled (valid token ids / finite activations for the eager run below)
                    ins = [torch.zeros(shape, dtype=dtype, device=torch.device('cuda', self._device))
                           for shape, dtype in shard.native_input_spec(ubatch, dim1)]
                    self._inputs[(ubatch, dim1)] = ins
                kernels = ctypes.c_int(0)
                for parity in range(2 if overlap else 1):
                    # eager run on the same buffers first: sizes every persistent buffer and does all first-use work
                    # (module loads, function attributes, tensor-map driver entry points) outside the capture
                    shard.native_forward(ins, parity, defer=not overlap)
                    self._stream.synchronize()
                    if self._is_data:
                        raw = ins[0].numel() * ins[0].element_size()
                        check(LIB.pe_pipe_capture_begin(self._pipe, ubatch, dim1, parity, ins[0].data_ptr(), None, 0, 0, raw))
                    else:
                        n0 = ins[0].numel() // ubatch
                        n1 = ins[1].numel() // ubatch if len(ins) > 1 else 0
                        check(LIB.pe_pipe_capture_begin(self._pipe, ubatch, dim1, parity, ins[0].data_ptr(),
                                                        ins[1].data_ptr() if len(ins) > 1 else None, n0, n1, 0))
                    try:
                        parts = shard.native_forward(ins, parity, defer=not overlap)
                    except BaseException:
                        LIB.pe_pipe_capture_abort(self._pipe)
                        raise
                    a0, b0, m0 = parts[0]
                    a1, b1, m1 = parts[1] if len(parts) > 1 else (None, None, 0)
                    check(LIB.pe_pipe_capture_end(self._pipe, a0, b0, m0, a1, b1, m1, ubatch, bit, clamp,
                                                  1 if overlap else 0, ctypes.byref(kernels)))
            self.graph_kernels[(ubatch, dim1)] = kernels.value
            self._captured_bit = bit

    # ------------------------------------------------------------------ data rank
    def enqueue(self, tensor: torch.Tensor) -> None:
        """Insert one micro-batch (host or device tensor); blocks while the input ring is full."""
        self.check()
        shape, dtype = self._shard.native_input_spec(tensor.shape[0], 0)[0]
        dim1 = int(tensor.shape[1]) if len(shape) == 2 else 0          # BERT: the sequence length is the payload's
        ubatch = int(tensor.shape[0])
        if self._captured_bit is not None and self._quant()[0] != self._captured_bit:
            self.invalidate()     # the data rank's own bit-width was changed since its graphs were captured
        if not LIB.pe_pipe_has_graph(self._pipe, ubatch, dim1):
            self._capture(ubatch, dim1)
        if tensor.dtype != dtype or not tensor.is_contiguous():
            tensor = tensor.to(dtype).contiguous()
        if tensor.is_cuda:
            # the copy runs on the pipe's side stream: order it behind whatever produced the tensor
            self._copy_stream.wait_event(torch.cuda.current_stream().record_event())
        self._keep.append(tensor)
        check(LIB.pe_pipe_submit(self._pipe, tensor.data_ptr(), tensor.numel() * tensor.element_size(),
                                 0 if tensor.is_cuda else 1, ubatch, dim1))

    def _results_loop(self) -> None:
        ptr, items, n = ctypes.c_void_p(), ctypes.c_int(), ctypes.c_size_t()
        while True:
            rc = LIB.pe_pipe_next_result(self._pipe, ctypes.byref(ptr), ctypes.byref(items), ctypes.byref(n))
            if rc == 1:
                return
            check(rc)
            count = items.value * n.value
            buf = (ctypes.c_float * count).from_address(ptr.value)
            out = torch.frombuffer(buf, dtype=torch.float32, count=count).clone()
            shape = self._result_shape
            prod = 1
            for d in shape:
                prod *= d
            out = out.view(items.value, *shape) if prod == n.value else out.view(items.value, n.value)
            self._results_cb(out)

    # ------------------------------------------------------------------ other ranks
    def _run_loop(self) -> None:
        need = (ctypes.c_longlong * 2)()
        while True:
            rc = LIB.pe_pipe_run(self._pipe, need)
            if rc == 1:
                return
            if rc == 2:
                self._capture(int(need[0]), int(need[1]))
                continue
            check(rc)

    # ------------------------------------------------------------------ common
    def check(self) -> None:
        """Re-raise what killed a native thread."""
        if self.exception is not None:
            raise RuntimeError("a native pipeline thread failed") from self.exception

    def timing_reset(self) -> None:
        """The next micro-batch starts a new device-timed phase."""
        check(LIB.pe_pipe_timing_reset(self._pipe))

    def timing(self) -> dict:
        """Device time of the current phase on this rank (after it has drained)."""
        c, r = ctypes.c_float(), ctypes.c_float()
        launches, kernels = ctypes.c_ulonglong(), ctypes.c_ulonglong()
        check(LIB.pe_pipe_timing(self._pipe, ctypes.byref(c), ctypes.byref(r), ctypes.byref(launches),
                                 ctypes.byref(kernels)))
        return {'compute_ms': c.value, 'results_ms': r.value, 'graph_launches': launches.value,
                'kernels': kernels.value}

    def sync(self) -> None:
        """Wait for everything this rank has enqueued on the device."""
        check(LIB.pe_pipe_sync(self._pipe))

    def shutdown(self, timeout: float = 120.0) -> None:
        """Data rank: close the input (the closing ticket travels down the pipeline and back); everyone: wait for the
        stage thread, then - after ALL ranks have drained (barrier) - unmap the peers' memory and free this rank's."""
        if self._closed:
            return
        self._closed = True
        failure = self.exception
        if self._is_data and self._pipe:
            LIB.pe_pipe_close_input(self._pipe)
        for thr in self._threads:
            thr.join(timeout)
        if self._pipe:
            LIB.pe_pipe_sync(self._pipe)
        if dist.is_initialized() and dist.get_world_size() > 1 and failure is None and self.exception is None:
            drain_barrier()   # no rank frees its ring while a neighbour's kernel may still store into it
        if self._pipe:
            LIB.pe_pipe_destroy(self._pipe)
            self._pipe = ctypes.c_void_p()
        for handle in self._links:
            LIB.pe_link_close(handle)
        self._links.clear()
        for sock in self._socks:
            try:
                sock.close()
            except OSError:
                pass
        self._socks.clear()
        self._inputs.clear()
