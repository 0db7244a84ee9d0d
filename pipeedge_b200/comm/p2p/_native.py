"""Native pipeline stage: the body of `DistP2pPipelineStage` when every rank drives a native shard.

The reference's stage is three Python threads handing each micro-batch through queues (`p2p/__init__.py:261-295,
373-394`). Here a stage's micro-batch is ONE CUDA graph (link get -> shard kernels -> link put, `csrc/pipe.cu`) and the
per-micro-batch host work runs in C with the GIL released:

* data rank: `enqueue_tensor` -> `pe_pipe_submit` (copy into the host-fed input ring on a side stream, graph launch,
  ticket to the next rank); a results thread blocks in `pe_pipe_next_result` and calls `results_cb` with each result;
* other ranks: one thread sits in `pe_pipe_run` (ticket in -> graph launch -> ticket out) until the pipeline closes;
* a data rank outside the stage pipeline (`NativeFeeder`) owns no shard: its graph is one relay kernel that moves each
  input micro-batch, bytes unchanged, from its host-fed ring into the first stage's ring (`pe_pipe_capture_relay`);
  the first stage receives it as a raw payload from a peer link. The first stage tells the feeder its input geometry
  over their hop's socket before the link opens (`send_input_geometry`);
* such a data rank without a CUDA device (`NativeHostFeeder`) never touches CUDA: its hops are rings in shared memory
  (`pe_hostring_*`). The last stage's send kernel stores results into one (its `pe_link_open` learns from the
  handshake that the peer is such a ring); the first stage feeds inputs out of the other into a host-fed ring, as a
  data rank that owns it does (`NativeStage._shm_loop`).

Activations cross hops as peer-memory stores synchronised by device-polled flags (`csrc/link.cu`); QuantPipe
quantisation (`-q`, the shard's `quant_bit` buffer) is fused into the send kernel and undone by the receive kernel, so
the Python quantisation hooks (`runtime.py:73-119`) are represented by those kernels rather than called. Python runs
once per (micro-batch size, sequence length): to capture the graph.

Per-micro-batch timing: with stamps on (a shard hook that asks for records, or a send-timing hook), the graphs also
write device timestamps into a ring of records in host memory (`pe_pipe_enable_stamps`); a drain thread turns each
completed record into calls of the stage's record consumers and send-timing hooks, off the graph-launch path.

Adaptive bit-widths: a shard hook may declare the bit-widths it sets `quant_bit` to (`_pe_send_bits`). A stage whose
set S = {initial bit-width} | declared sets has more than one member captures one graph per bit-width in S for every
shape, all at once, and picks the variant per micro-batch (`pe_pipe_set_send_bit`): after each record's consumers (a
policy hook's record consumer decides the next bit-width there) and, on the data rank, at every `enqueue`. No kernel and
no graph changes; switching never captures while payloads are in flight.
"""
import collections
import ctypes
import logging
import os
import struct
import threading
import time
from typing import Callable, Iterable, List, NamedTuple, Optional, Set, Tuple
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


def _clamp(bit: int) -> int:
    return _lib.PE_CLAMP_AUTO if bit > 0 else _lib.PE_CLAMP_NONE


def hook_is_native(hook) -> bool:
    """Whether a module hook is represented by the native pipeline's kernels (quantisation encode / decode) or is a
    no-op there (device placement, disabled monitoring): marked by `_pe_native` (a bool or a callable)."""
    flag = getattr(hook, '_pe_native', None)
    return bool(flag() if callable(flag) else flag)


def _shard_hooks(shard) -> list:
    return list(getattr(shard, '_forward_hooks', {}).values()) + list(getattr(shard, '_forward_pre_hooks', {}).values())


def shard_is_native(shard) -> bool:
    """A native shard whose registered hooks the native pipeline accounts for."""
    from ...models.transformers._shard import GpuTransformerShard   # pylint: disable=import-outside-toplevel
    if not isinstance(shard, GpuTransformerShard):
        return False
    return all(hook_is_native(h) for h in _shard_hooks(shard))


def record_consumers(shard) -> List[Callable]:
    """The per-micro-batch record consumers the shard's hooks ask for: a hook may carry `_pe_records`, a callable
    `(shard) -> Optional[consumer]`; each consumer is called with every `StampRecord` of the stage."""
    consumers = []
    for hook in _shard_hooks(shard):
        factory = getattr(hook, '_pe_records', None)
        consumer = factory(shard) if factory is not None else None
        if consumer is not None:
            consumers.append(consumer)
    return consumers


def declared_send_bits(shard) -> Set[int]:
    """The bit-widths the shard's hooks may set its `quant_bit` to: the union of the hooks' `_pe_send_bits` (an iterable
    of ints, or a callable returning one)."""
    bits = set()
    for hook in _shard_hooks(shard):
        declared = getattr(hook, '_pe_send_bits', None)
        if declared is not None:
            bits.update(int(b) for b in (declared() if callable(declared) else declared))
    return bits


def wire_f16() -> bool:
    """Whether links put raw payloads on the wire as fp16 (`PIPEEDGE_WIRE_F16=1`; read by the links at open)."""
    return os.environ.get('PIPEEDGE_WIRE_F16', '0')[:1] == '1'


def payload_fits(room: int, items: int, elems: Iterable[int], bit: int, wire: int) -> bool:
    """Whether a payload of tensors [items, n] (n in `elems`) at `bit` bits fits `room` bytes of slot payload
    (`pe_link_slot_bytes`), placed as `pe_link_put` places it: each tensor's wire bytes (the values, or the packed codes -
    per-item scale and shift live in the slot header) at an offset rounded up to 256 bytes."""
    off = 0
    for n in elems:
        wire_bytes = LIB.pe_link_payload_bytes(items, n, bit, wire) - (8 * items if bit > 0 else 0)
        if off + wire_bytes > room:
            return False
        off += (wire_bytes + 255) // 256 * 256
    return True


# Input geometry the first stage announces to a data rank outside the stage pipeline, on their hop's socket before the
# link opens: magic | the largest input micro-batch in bytes | dtype name (NUL-padded) | tensor rank.
_GEOMETRY = struct.Struct('<4sQ16sI')
_GEOMETRY_MAGIC = b'PEIN'
_INPUT_DTYPES = {'float32': torch.float32, 'int64': torch.int64}   # images, token ids


def max_input_geometry(shard) -> Tuple[int, torch.dtype, int]:
    """(bytes, dtype, tensor rank) of the largest input micro-batch a first-stage shard takes: `PIPEEDGE_MAX_UBATCH`
    items of its longest sequence."""
    shape, dtype = shard.native_input_spec(max_ubatch(), shard.native_max_tokens())[0]
    nbytes = torch.empty((), dtype=dtype).element_size()
    for d in shape:
        nbytes *= int(d)
    return nbytes, dtype, len(shape)


def send_input_geometry(sock, nbytes: int, dtype: torch.dtype, ndim: int) -> None:
    """First stage -> data rank outside the stage pipeline: what its input micro-batches look like."""
    name = str(dtype).split('.')[-1]
    if _INPUT_DTYPES.get(name) != dtype:
        raise ValueError(f"native pipeline: input dtype {dtype} cannot be announced to the data rank")
    sock.sendall(_GEOMETRY.pack(_GEOMETRY_MAGIC, nbytes, name.encode(), ndim))


def recv_input_geometry(sock) -> Tuple[int, torch.dtype, int]:
    """The data rank's side of `send_input_geometry`: (largest input in bytes, dtype, tensor rank)."""
    buf = b''
    while len(buf) < _GEOMETRY.size:
        chunk = sock.recv(_GEOMETRY.size - len(buf))
        if not chunk:
            raise ConnectionError("native pipeline: the first stage closed its hop before announcing its input")
        buf += chunk
    magic, nbytes, name, ndim = _GEOMETRY.unpack(buf)
    dtype = _INPUT_DTYPES.get(name.rstrip(b'\0').decode(errors='replace'))
    if magic != _GEOMETRY_MAGIC or dtype is None or nbytes == 0 or ndim == 0:
        raise ConnectionError("native pipeline: malformed input geometry from the first stage")
    return nbytes, dtype, ndim


class RecordShapeError(LookupError):
    """A timestamp record matches no payload shape the stage has captured (or more than one)."""


def record_payload_elems(rec, shapes: Iterable[Tuple[int, Tuple[int, ...]]]) -> Tuple[int, ...]:
    """Elements per item of each tensor of the payload a record's micro-batch sent. `shapes`: (items, elements per item
    of each tensor) of the payloads the stage has captured graphs for; the match is the one whose payload at the record's
    bit-width has the record's size. It is unique: payloads of one item count differ by at least one row of the stage's
    output (a BERT sequence length more or less), and every row adds bytes at every bit-width."""
    wire = 1 if wire_f16() else 0
    found = {elems for items, elems in shapes
             if items == rec.items and sum(LIB.pe_link_payload_bytes(items, n, rec.bit_out, wire) for n in elems)
             == rec.bytes_out}
    if len(found) != 1:
        raise RecordShapeError(f"native pipeline: {len(found)} captured payload shapes match the record of micro-batch "
                          f"{rec.index} ({rec.items} items, {rec.bit_out} bits, {rec.bytes_out} bytes)")
    return found.pop()


class StampRecord(NamedTuple):
    """One micro-batch of a stage on the native pipeline, as its graph timestamped it (`pe_pipe_record`; times are
    device %globaltimer nanoseconds). `t_send_start == t_stage` when the send runs inside the main graph; `t_encoded`
    is 0 unless the send took the staged path (stand-alone encode kernels, then a shipping kernel). `bit_in` is -1 on
    the data rank (its input is fed by the host)."""
    index: int
    items: int
    bit_out: int
    bit_in: int
    bytes_out: int
    flags: int
    t_start: int
    t_got: int
    t_stage: int
    t_send_start: int
    t_encoded: int
    t_send_end: int

    @classmethod
    def from_c(cls, rec: _lib.PipeRecord) -> 'StampRecord':
        """Copy a `pe_pipe_record`."""
        return cls(**{name: getattr(rec, name) for name in cls._fields})

    @property
    def send_mbits(self) -> float:
        """The payload in Mbit, as the Python-thread path's send-timing hook reports it (bytes * 8e-6)."""
        return self.bytes_out * 8e-6

    @property
    def send_seconds(self) -> float:
        """Device time of the send: send start -> the payload published to the consumer."""
        return (self.t_send_end - self.t_send_start) * 1e-9


class RecordDrain:
    """Reader side of a pipe's timestamp ring: `poll()` drains what has completed (non-blocking) and hands each record to
    `dispatch`; `dropped` counts records overwritten before they were read. `drain_fn(buf, max, n, dropped)` is
    `pe_pipe_drain_stamps` bound to one pipe (injectable for tests)."""

    def __init__(self, drain_fn: Callable, dispatch: Callable[[StampRecord], None], batch: int = 64):
        self._drain_fn = drain_fn
        self._dispatch = dispatch
        self._buf = (_lib.PipeRecord * batch)()
        self.dropped = 0
        self.records = 0

    def poll(self) -> int:
        """Dispatch every completed record; returns how many."""
        total = 0
        n, dropped = ctypes.c_int(), ctypes.c_ulonglong()
        while True:
            dropped.value = 0
            check(self._drain_fn(self._buf, len(self._buf), ctypes.byref(n), ctypes.byref(dropped)))
            if dropped.value:
                self.dropped += dropped.value
                logger.warning("native pipeline: %d timestamp records were overwritten before they were read",
                               dropped.value)
            for i in range(n.value):
                self._dispatch(StampRecord.from_c(self._buf[i]))
            total += n.value
            self.records += n.value
            if n.value < len(self._buf):
                return total


class NativeStage:
    """One rank's stage on the native pipeline. `rank_src` / `rank_dst` as `DistP2pPipelineStage`; the data rank is the
    one with a `results_cb` (here it owns the first shard; `NativeFeeder` is a data rank that owns none). A first stage
    that is not the data rank receives its input relayed from a `NativeFeeder`."""

    def __init__(self, rank_src: Optional[int], rank_dst: Optional[int], shard, results_cb: Optional[Callable]):
        self._rank_src, self._rank_dst = rank_src, rank_dst
        self._shard = shard
        self._results_cb = results_cb
        self._is_data = results_cb is not None
        # fed by a data rank outside the stage pipeline: a raw input payload arrives on the peer link
        self._raw_in = shard is not None and shard.shard_config.is_first and not self._is_data and rank_src is not None
        self._device = torch.cuda.current_device()
        self._pipe = ctypes.c_void_p()
        self._links = []                      # every pe_link this rank opened (closed at shutdown)
        self._link_in = self._link_out = self._link_res = None
        self._shm_in = None                   # first stage fed by a data rank without a GPU: its shared-memory ring
        self._socks = []
        self._inputs = {}                     # (ubatch, dim1) -> persistent input tensors
        self._keep = collections.deque(maxlen=link_slots() + 2)   # sources of in-flight input copies
        self._threads = []
        self._closed = False
        self._capture_lock = threading.Lock()
        self.exception: Optional[BaseException] = None
        self.graph_kernels = {}               # (ubatch, dim1) -> kernels per micro-batch
        self.variant_kernels = {}             # (ubatch, dim1, bit) -> kernels per micro-batch of that variant
        self.captures = 0                     # graph variants captured so far (every parity of one counts once)
        self._result_shape = None
        self._captured_bit = None             # the QuantPipe bit-width the captured graphs send with
        self._quant_cache = (None, 0, 0)      # (quant_bit tensor, its in-place version, its value)
        # Adaptive bit-widths: S = the initial bit-width | every set the shard's hooks declare; one graph per member
        bit0 = self._quant()[0]
        declared = set() if shard is None or shard.shard_config.is_last else declared_send_bits(shard)
        self._send_bits = sorted(declared | {bit0})
        self.adaptive = len(self._send_bits) > 1
        self._pushed_bit = None               # the last pe_pipe_set_send_bit (by one thread: enqueue's or the drain's)
        self._stream = None
        self._copy_stream = None
        self._record_cbs = record_consumers(shard)   # per-micro-batch record consumers (from the shard's hooks)
        self._send_hooks = []                          # (hook, args): hook(mbits, seconds, *args) per payload sent
        self._drain = None                             # RecordDrain once stamps are on
        self._drain_stop = threading.Event()
        self._drain_thread = None
        self._record_error: Optional[BaseException] = None   # a record no captured payload shape matched

    # ------------------------------------------------------------------ set-up
    def _open_link(self, sock, is_producer: bool, payload_bytes: int) -> ctypes.c_void_p:
        handle = ctypes.c_void_p()
        # an adaptive producer announces a quantised payload even if it starts raw (it only sizes the receive grid)
        hint = max(self._send_bits) if self.adaptive else self._quant()[0]
        check(LIB.pe_link_open(sock.fileno(), 1 if is_producer else 0, payload_bytes if is_producer else 0,
                               link_slots() if is_producer else 0, hint if is_producer else 0,
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
                if self._raw_in:   # the feeder owns no shard: it sizes the link from this
                    send_input_geometry(sock, *max_input_geometry(shard))
                peer_in = self._open_link(sock, False, 0)
        # fed by a data rank without a GPU: its inputs wait in a shared-memory ring, and this rank feeds them to a
        # host-fed ring as a data rank that owns the first stage does (`_shm_loop`)
        self._shm_in = peer_in if self._raw_in and LIB.pe_link_is_shm(peer_in) else None
        if self._is_data or self._shm_in is not None:
            # inputs arrive from the host; results come back on the hop from the last stage (or a loop-back link)
            in_bytes = max_input_geometry(shard)[0]
            handle = ctypes.c_void_p()
            check(LIB.pe_link_open_host(in_bytes, link_slots(), ctypes.byref(handle)))
            self._links.append(handle)
            self._link_in = handle
            if not self._is_data:
                self._link_out = peer_out
            elif peer_out is None:
                loop = ctypes.c_void_p()
                check(LIB.pe_link_open_local(out_bytes, link_slots(), 0, ctypes.byref(loop)))
                self._links.append(loop)
                self._link_out = self._link_res = loop
            else:
                self._link_out, self._link_res = peer_out, peer_in
        else:
            self._link_in, self._link_out = peer_in, peer_out
        check(LIB.pe_pipe_create(self._link_in, self._link_out, self._link_res, ctypes.byref(self._pipe)))
        if self.adaptive:
            self._push_bit()
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
        elif self._shm_in is not None:
            thr = threading.Thread(target=self._guard, args=(self._shm_loop,), daemon=True, name='pe-shm-feed')
        else:
            thr = threading.Thread(target=self._guard, args=(self._run_loop,), daemon=True, name='pe-stage')
        if self._record_cbs or self._send_hooks:
            self._start_stamps()   # before the first capture, so that every micro-batch has a record
        self._threads.append(thr)
        thr.start()

    # ------------------------------------------------------------------ per-micro-batch timestamps
    def add_send_timing_hook(self, hook: Callable[..., None], args: tuple) -> None:
        """`hook(mbits, seconds, *args)` once per payload this stage sends to the next rank, from its device timestamps
        (before or after `init()`; graphs captured without stamps are captured again). A stage without a next rank
        (a world of one) sends nothing and never calls it, as on the Python-thread path."""
        self._send_hooks.append((hook, args))
        if self._pipe:
            self._start_stamps()

    def _start_stamps(self) -> None:
        if self._drain_thread is not None:
            return
        check(LIB.pe_pipe_enable_stamps(self._pipe, 1))
        pipe = self._pipe
        self._drain = RecordDrain(lambda *a: LIB.pe_pipe_drain_stamps(pipe, *a), self._dispatch)
        self._drain_thread = threading.Thread(target=self._drain_loop, daemon=True, name='pe-stamps')
        self._drain_thread.start()

    def _dispatch(self, rec: StampRecord) -> None:
        calls = [(consumer, (rec,)) for consumer in self._record_cbs]
        if self._rank_dst is not None:
            calls += [(hook, (rec.send_mbits, rec.send_seconds, *args)) for hook, args in self._send_hooks]
        for fn, args in calls:
            try:
                fn(*args)
            except RecordShapeError as exc:
                # a consumer could not tell which micro-batch the record is (a policy would stop adapting): the stage
                # fails at its owner's next check()
                if self._record_error is None:
                    self._record_error = exc
                    logger.exception("native pipeline: a timestamp record matches no captured payload shape")
            except Exception:   # pylint: disable=broad-except
                logger.exception("native pipeline: a timestamp record consumer failed")
        if self.adaptive and not self._is_data:
            # a policy among the consumers may have changed `quant_bit`: the stage loop launches that variant from its
            # next micro-batch on. The data rank instead selects at every enqueue, on the thread that launches.
            self._push_bit()

    def _push_bit(self) -> None:
        """The bit-width in `quant_bit` selects the graph variant from the next launch on."""
        bit = self._quant()[0]
        if bit != self._pushed_bit:
            check(LIB.pe_pipe_set_send_bit(self._pipe, bit))
            self._pushed_bit = bit

    def _drain_loop(self) -> None:
        """Poll the ring (each C call releases the GIL and never waits on the device); a last pass after the stop."""
        while True:
            stopping = self._drain_stop.is_set()
            got = self._drain.poll()
            if stopping:
                return
            if got == 0:
                self._drain_stop.wait(0.001)

    @property
    def records(self) -> int:
        """Timestamp records dispatched so far (0 without stamps)."""
        return self._drain.records if self._drain is not None else 0

    @property
    def records_dropped(self) -> int:
        """Timestamp records overwritten before the drain thread read them."""
        return self._drain.dropped if self._drain is not None else 0

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
        if shard is None or shard.shard_config.is_last or not hasattr(shard, 'quant_bit'):
            return 0, _lib.PE_CLAMP_NONE
        qb = shard.quant_bit
        version = getattr(qb, '_version', 0)
        cached, cached_version, bit = self._quant_cache   # one tuple: the drain thread may call this concurrently
        if qb is not cached or version != cached_version:
            bit = int(qb)
            self._quant_cache = (qb, version, bit)        # holds the tensor, so that its id cannot be reused
        return bit, _clamp(bit)

    @property
    def send_bits(self) -> List[int]:
        """The bit-widths this stage keeps a graph variant of per shape (one member: a fixed-bit stage)."""
        return list(self._send_bits)

    @property
    def variants(self) -> int:
        """Graph variants captured and held now, over every shape and bit-width."""
        return len(self.variant_kernels)

    def invalidate(self) -> None:
        """Forget the captured graphs (they bake in the shard's `quant_bit` and buffer addresses): the next payload of
        each shape captures again. For callers that change a fixed-bit stage's bit-width between micro-batches by hand;
        a stage whose hooks declare their bit-widths (`_pe_send_bits`) switches between captured variants instead."""
        with self._capture_lock:
            self._invalidate_locked()

    def _invalidate_locked(self) -> None:
        check(LIB.pe_pipe_invalidate(self._pipe))
        self.graph_kernels.clear()
        self.variant_kernels.clear()

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
                self._invalidate_locked()   # the stage's workspace is about to be re-created
            bit = self._quant()[0]
            if self.adaptive and bit not in self._send_bits:
                self._send_bits = sorted(set(self._send_bits) | {bit})   # a bit-width no hook declared
            # a fixed-bit stage: the one bit-width it sends with; an adaptive stage: every variant of this shape it does
            # not hold yet, at once
            bits = [b for b in self._send_bits if not LIB.pe_pipe_has_variant(self._pipe, ubatch, dim1, b)] \
                if self.adaptive else [bit]
            overlap = overlap_send()
            with torch.cuda.stream(self._stream):
                ins = self._inputs.get((ubatch, dim1))
                if ins is None:     # zero-filled (valid token ids / finite activations for the eager run below)
                    ins = [torch.zeros(shape, dtype=dtype, device=torch.device('cuda', self._device))
                           for shape, dtype in shard.native_input_spec(ubatch, dim1)]
                    self._inputs[(ubatch, dim1)] = ins
                for variant_bit in bits:
                    kernels = self._capture_variant(ins, ubatch, dim1, variant_bit, overlap,
                                                    check_slots=self.adaptive and variant_bit == bits[0])
                    self.variant_kernels[(ubatch, dim1, variant_bit)] = kernels
                    self.captures += 1
                    if variant_bit == bit:
                        self.graph_kernels[(ubatch, dim1)] = kernels
            self._captured_bit = bit

    def _check_slot_fits(self, parts, ubatch: int) -> None:
        """Every bit-width of an adaptive stage's set fits the downstream link's slots (sized for the raw payload)."""
        room = LIB.pe_link_slot_bytes(self._link_out)
        elems = [m for _, _, m in parts]
        for bit in self._send_bits:
            if not payload_fits(room, ubatch, elems, bit, 1 if wire_f16() else 0):
                raise ValueError(f"native pipeline: a {bit}-bit payload of {ubatch} items x {elems} elements does not "
                                 f"fit the link's {room}-byte slots (bit-widths of this stage: {self._send_bits})")

    def _capture_variant(self, ins, ubatch: int, dim1: int, bit: int, overlap: bool, check_slots: bool) -> int:
        """Capture the graph(s) of one (shape, send bit-width): both buffer parities with an overlapped send."""
        shard = self._shard
        kernels = ctypes.c_int(0)
        for parity in range(2 if overlap else 1):
            # eager run on the same buffers first: sizes every persistent buffer and does all first-use work
            # (module loads, function attributes, tensor-map driver entry points) outside the capture
            parts = shard.native_forward(ins, parity, defer=not overlap)
            self._stream.synchronize()
            if check_slots and parity == 0:
                self._check_slot_fits(parts, ubatch)
            if self._is_data or self._raw_in:   # host-fed, or relayed unchanged by a data rank outside the pipeline
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
            check(LIB.pe_pipe_capture_end(self._pipe, a0, b0, m0, a1, b1, m1, ubatch, bit, _clamp(bit),
                                          1 if overlap else 0, ctypes.byref(kernels)))
        return kernels.value

    # ------------------------------------------------------------------ data rank
    def enqueue(self, tensor: torch.Tensor) -> None:
        """Insert one micro-batch (host or device tensor); blocks while the input ring is full."""
        self.check()
        shape, dtype = self._shard.native_input_spec(tensor.shape[0], 0)[0]
        dim1 = int(tensor.shape[1]) if len(shape) == 2 else 0          # BERT: the sequence length is the payload's
        ubatch = int(tensor.shape[0])
        bit = self._quant()[0]
        if self.adaptive:
            if bit not in self._send_bits:
                self.invalidate()     # a bit-width outside the declared set: captured again, with the set
            self._push_bit()
        elif self._captured_bit is not None and bit != self._captured_bit:
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
            for d in shape or ():
                prod *= d
            out = out.view(items.value, *shape) if shape is not None and prod == n.value \
                else out.view(items.value, n.value)
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

    def _shm_loop(self) -> None:
        """First stage fed by a data rank without a GPU: per ticket, wait for the input in the shared-memory ring, copy
        it into the host-fed ring and launch the graph (`pe_pipe_submit`, the registered slot as a pinned source), then
        hand the slot back behind that copy on the copy stream. The data rank's close travels on downstream."""
        ticket = (ctypes.c_longlong * 2)()
        src = ctypes.c_void_p()
        copy_stream = LIB.pe_pipe_copy_stream(self._pipe)
        while True:
            rc = LIB.pe_link_ticket_recv(self._shm_in, ticket)
            if rc == 1 or (rc == 0 and ticket[0] < 0):
                check(LIB.pe_pipe_close_input(self._pipe))
                return
            check(rc)
            ubatch, dim1 = int(ticket[0]), int(ticket[1])
            if not LIB.pe_pipe_has_graph(self._pipe, ubatch, dim1):
                self._capture(ubatch, dim1)
            x = self._inputs[(ubatch, dim1)][0]   # the graph's input buffer: the size of this shape's inputs
            nbytes = x.numel() * x.element_size()
            check(LIB.pe_link_shm_wait(self._shm_in, ubatch, nbytes, ctypes.byref(src)))
            check(LIB.pe_pipe_submit(self._pipe, src, nbytes, 1, ubatch, dim1))
            check(LIB.pe_link_shm_release(self._shm_in, copy_stream))

    # ------------------------------------------------------------------ common
    def check(self) -> None:
        """Re-raise what killed a native thread."""
        if self.exception is not None:
            raise RuntimeError("a native pipeline thread failed") from self.exception
        if self._record_error is not None:
            raise RuntimeError("a timestamp record of the native pipeline matched no captured payload shape") \
                from self._record_error

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
        if self._drain_thread is not None:
            self._drain_stop.set()      # every graph has completed: the drain thread's last pass reads every record
            self._drain_thread.join(timeout)
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


class NativeFeeder(NativeStage):
    """A data rank outside the stage pipeline (`runtime.py -D <rank>` with the rank not in `-r`) on the native
    pipeline: a stage without a shard. `enqueue` feeds its host-fed ring and launches its graph, ONE relay kernel that
    moves the input micro-batch, bytes unchanged, into the first stage's ring; a results thread drains the last stage's
    results as on a data rank that owns the first stage. `rank_dst`: the first stage; `rank_src`: the last stage."""

    def __init__(self, rank_src: int, rank_dst: int, results_cb: Callable):
        super().__init__(rank_src, rank_dst, None, results_cb)
        self._geometry = None       # (largest input micro-batch in bytes, dtype, tensor rank) from the first stage
        self._relay_bytes = {}      # (ubatch, dim1) -> input bytes its relay graph moves

    def init(self, connect_to: Callable, accept_from: Callable) -> None:
        """Open the hop to the first stage (reading its input geometry first) and the hop from the last one, in
        ascending order of the sender's rank like every stage, then the host-fed ring; build the pipe."""
        rank = dist.get_rank() if dist.is_initialized() else 0
        peer_in = peer_out = None
        for _, kind in sorted([(rank, 'send'), (self._rank_src, 'recv')]):
            if kind == 'send':
                sock = connect_to(self._rank_dst)
                self._socks.append(sock)
                self._geometry = recv_input_geometry(sock)
                peer_out = self._open_link(sock, True, self._geometry[0])
            else:
                sock = accept_from(self._rank_src)
                self._socks.append(sock)
                peer_in = self._open_link(sock, False, 0)
        handle = ctypes.c_void_p()
        check(LIB.pe_link_open_host(self._geometry[0], link_slots(), ctypes.byref(handle)))
        self._links.append(handle)
        self._link_in, self._link_out, self._link_res = handle, peer_out, peer_in
        check(LIB.pe_pipe_create(self._link_in, self._link_out, self._link_res, ctypes.byref(self._pipe)))
        self._stream = torch.cuda.ExternalStream(LIB.pe_pipe_stream(self._pipe), device=self._device)
        self._copy_stream = torch.cuda.ExternalStream(LIB.pe_pipe_copy_stream(self._pipe), device=self._device)
        thr = threading.Thread(target=self._guard, args=(self._results_loop,), daemon=True, name='pe-results')
        if self._send_hooks:
            self._start_stamps()
        self._threads.append(thr)
        thr.start()

    @property
    def input_geometry(self) -> Optional[Tuple[int, torch.dtype, int]]:
        """(largest input micro-batch in bytes, dtype, tensor rank) the first stage announced (after `init()`)."""
        return self._geometry

    def prepare(self, ubatch: int, dim1: int = 0) -> None:
        """No-op: a relay graph is captured at a shape's first `enqueue` (its size comes from the tensor)."""

    def enqueue(self, tensor: torch.Tensor) -> None:
        """Insert one micro-batch (host or device tensor, converted to the first stage's input dtype); blocks while the
        input ring is full."""
        self.check()
        max_bytes, dtype, ndim = self._geometry
        if tensor.dim() != ndim:
            raise ValueError(f"native pipeline: a {tensor.dim()}-D input where the first stage takes {ndim}-D ones")
        ubatch = int(tensor.shape[0])
        dim1 = int(tensor.shape[1]) if ndim == 2 else 0      # BERT: the sequence length is the payload's
        if tensor.dtype != dtype or not tensor.is_contiguous():
            tensor = tensor.to(dtype).contiguous()
        nbytes = tensor.numel() * tensor.element_size()
        if not LIB.pe_pipe_has_graph(self._pipe, ubatch, dim1):
            self._capture_relay(ubatch, dim1, nbytes, max_bytes)
        elif self._relay_bytes.get((ubatch, dim1)) != nbytes:
            raise ValueError(f"native pipeline: an input of {nbytes} bytes where micro-batches of {ubatch} items "
                             f"(dim {dim1}) had {self._relay_bytes.get((ubatch, dim1))}")
        if tensor.is_cuda:
            # the copy runs on the pipe's side stream: order it behind whatever produced the tensor
            self._copy_stream.wait_event(torch.cuda.current_stream().record_event())
        self._keep.append(tensor)
        check(LIB.pe_pipe_submit(self._pipe, tensor.data_ptr(), nbytes, 0 if tensor.is_cuda else 1, ubatch, dim1))

    def _capture_relay(self, ubatch: int, dim1: int, nbytes: int, max_bytes: int) -> None:
        if ubatch > max_ubatch():
            raise ValueError(f"micro-batch of {ubatch} items exceeds PIPEEDGE_MAX_UBATCH={max_ubatch()}")
        if nbytes > max_bytes:
            raise ValueError(f"native pipeline: an input of {nbytes} bytes exceeds the first stage's largest "
                             f"({max_bytes} bytes)")
        kernels = ctypes.c_int(0)
        with self._capture_lock:
            check(LIB.pe_pipe_capture_relay(self._pipe, ubatch, dim1, nbytes, ctypes.byref(kernels)))
            self._relay_bytes[(ubatch, dim1)] = nbytes
            self.graph_kernels[(ubatch, dim1)] = kernels.value
            self.variant_kernels[(ubatch, dim1, 0)] = kernels.value
            self.captures += 1


def shm_name(src: int, dst: int) -> str:
    """Name of the shared-memory ring of the hop `src` -> `dst` of a data rank without a GPU (ranks share a node;
    MASTER_PORT keeps concurrent jobs apart, as `DistP2pContext.sock_path` does)."""
    return f"/pipeedge_b200_{os.environ.get('MASTER_PORT', '0')}_{src}_{dst}"


class NativeHostFeeder:
    """A data rank outside the stage pipeline WITHOUT a CUDA device (`runtime.py -d cpu`, or no visible GPU) on the
    native pipeline. It never touches CUDA. Both of its hops are rings in shared memory that it creates
    (`pe_hostring_create`): `enqueue` converts each micro-batch on the CPU to the first stage's input dtype and publishes
    it into the input ring, which the first stage copies out of with its copy engine; the last stage's send kernel
    stores the results into the other ring, and a results thread hands them to `results_cb` in order, as [items, n]
    fp32 CPU tensors. `rank_dst`: the first stage; `rank_src`: the last stage."""

    def __init__(self, rank_src: int, rank_dst: int, results_cb: Callable):
        self._rank_src, self._rank_dst = rank_src, rank_dst
        self._results_cb = results_cb
        self._ring_in = self._ring_res = None
        self._socks = []
        self._geometry = None       # (largest input micro-batch in bytes, dtype, tensor rank) from the first stage
        self._send_hooks = []       # (hook, args): hook(mbits, seconds, *args) per micro-batch published
        self._thread = None
        self._closed = False
        self.exception: Optional[BaseException] = None

    def init(self, connect_to: Callable, accept_from: Callable) -> None:
        """Open the hop to the first stage (reading its input geometry first) and the hop from the last one, in
        ascending order of the sender's rank like every stage; start the results thread."""
        rank = dist.get_rank() if dist.is_initialized() else 0
        for _, kind in sorted([(rank, 'send'), (self._rank_src, 'recv')]):
            handle = ctypes.c_void_p()
            if kind == 'send':
                sock = connect_to(self._rank_dst)
                self._socks.append(sock)
                self._geometry = recv_input_geometry(sock)
                check(LIB.pe_hostring_create(sock.fileno(), shm_name(rank, self._rank_dst).encode(), 1,
                                             self._geometry[0], link_slots(), ctypes.byref(handle)))
                self._ring_in = handle
            else:
                sock = accept_from(self._rank_src)
                self._socks.append(sock)
                check(LIB.pe_hostring_create(sock.fileno(), shm_name(self._rank_src, rank).encode(), 0, 0, 0,
                                             ctypes.byref(handle)))
                self._ring_res = handle
        self._thread = threading.Thread(target=self._guard, daemon=True, name='pe-host-results')
        self._thread.start()

    @property
    def input_geometry(self) -> Optional[Tuple[int, torch.dtype, int]]:
        """(largest input micro-batch in bytes, dtype, tensor rank) the first stage announced (after `init()`)."""
        return self._geometry

    def add_send_timing_hook(self, hook: Callable[..., None], args: tuple) -> None:
        """`hook(mbits, seconds, *args)` once per micro-batch: the payload in Mbit and the host-clock time its publication
        took (waiting for a free slot included, as a device send includes waiting for the receiver)."""
        self._send_hooks.append((hook, args))

    def prepare(self, ubatch: int, dim1: int = 0) -> None:
        """No-op: this rank captures no graph."""

    def enqueue(self, tensor: torch.Tensor) -> None:
        """Insert one micro-batch (converted to the first stage's input dtype); blocks while the input ring is full."""
        self.check()
        max_bytes, dtype, ndim = self._geometry
        if tensor.dim() != ndim:
            raise ValueError(f"native pipeline: a {tensor.dim()}-D input where the first stage takes {ndim}-D ones")
        ubatch = int(tensor.shape[0])
        dim1 = int(tensor.shape[1]) if ndim == 2 else 0      # BERT: the sequence length is the payload's
        if ubatch > max_ubatch():
            raise ValueError(f"micro-batch of {ubatch} items exceeds PIPEEDGE_MAX_UBATCH={max_ubatch()}")
        tensor = tensor.detach().to(dtype).contiguous()
        nbytes = tensor.numel() * tensor.element_size()
        if nbytes > max_bytes:
            raise ValueError(f"native pipeline: an input of {nbytes} bytes exceeds the first stage's largest "
                             f"({max_bytes} bytes)")
        t0 = time.perf_counter()
        check(LIB.pe_hostring_publish(self._ring_in, tensor.data_ptr(), nbytes, ubatch, dim1))
        seconds = time.perf_counter() - t0
        for hook, args in self._send_hooks:
            hook(nbytes * 8e-6, seconds, *args)

    def _guard(self) -> None:
        try:
            self._results_loop()
        except BaseException as exc:   # pylint: disable=broad-except
            self.exception = exc       # re-raised on the owner by check()
            logger.exception("native pipeline results thread failed")

    def _results_loop(self) -> None:
        ticket = (ctypes.c_longlong * 2)()
        data = ctypes.c_void_p()
        while True:
            rc = LIB.pe_hostring_next(self._ring_res, ticket)
            if rc == 1:
                return
            check(rc)
            items, n = int(ticket[0]), int(ticket[1])
            check(LIB.pe_hostring_wait(self._ring_res, items, items * n * 4, ctypes.byref(data)))
            buf = (ctypes.c_float * (items * n)).from_address(data.value)
            out = torch.frombuffer(buf, dtype=torch.float32, count=items * n).clone().view(items, n)
            check(LIB.pe_hostring_release(self._ring_res))
            self._results_cb(out)

    def check(self) -> None:
        """Re-raise what killed the results thread."""
        if self.exception is not None:
            raise RuntimeError("the native pipeline's results thread failed") from self.exception

    def shutdown(self, timeout: float = 120.0) -> None:
        """Close the input (the closing ticket travels down the pipeline and back), wait for the results thread, then -
        after ALL ranks have drained (barrier) - unmap the rings."""
        if self._closed:
            return
        self._closed = True
        failure = self.exception
        if self._ring_in:
            LIB.pe_hostring_close_input(self._ring_in)
        if self._thread is not None:
            self._thread.join(timeout)
        if dist.is_initialized() and dist.get_world_size() > 1 and failure is None and self.exception is None:
            drain_barrier()   # no rank unmaps a ring while a neighbour may still use it
        for handle in (self._ring_in, self._ring_res):
            if handle:
                LIB.pe_hostring_close(handle)
        self._ring_in = self._ring_res = None
        for sock in self._socks:
            try:
                sock.close()
            except OSError:
                pass
        self._socks.clear()
