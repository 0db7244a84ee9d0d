"""Peer-to-peer pipeline communication - drop-in for `pipeedge.comm.p2p` (reference `p2p/__init__.py`).

Same classes and call contract (`DistP2pContext`, `DistP2pPipelineStage` with `enqueue_tensor`, the four
`register_*_hook`s, `work_cb` / `results_cb`, FIFO per hop, back-pressure through size-1 queues), rebuilt
for one rank per GPU:

* Per-payload control data (the payload description, only when it changes, and any CPU tensors) goes over one
  Unix-domain socket per hop: a Gloo message costs ~170 us of host time (measured), a local socket ~10 us, and at
  8 stages a micro-batch of 8 images is only ~150 us of GPU work per stage. Single node only, as is the target.
* The DEVICE of a tensor picks its plane. CUDA tensors (activations, int8 codes, per-item scales) travel
  over a dedicated 2-rank NCCL communicator per hop direction on a side stream, ordered against the compute
  stream with CUDA events, so the hop of micro-batch i overlaps the compute of micro-batch i+1 without the
  host ever waiting on the GPU. CPU tensors and the (cached) payload header travel over the hop's socket,
  where the reference sends every message over Gloo (`p2p/__init__.py:96-121`).
* One NCCL communicator per ordered rank pair: the reference's send and receive threads run concurrently
  (`p2p/__init__.py:155-258`) and NCCL serialises a communicator's operations on one internal stream, so a
  shared communicator could deadlock when two ranks send to each other (stage 0 <-> last stage on 2 ranks).
* The command channel (`cmd_broadcast`, `CommandThread`; `p2p/__init__.py:75-85,298-331`) stays on Gloo:
  NCCL has neither tags nor any-source receive.

Without CUDA (the CPU test-suite) payloads ride the hop sockets alone and the classes behave like the reference's.
With CUDA, a process that cannot load libnccl.so.2 refuses to open a hop; there is no second data plane.
"""
import collections
import logging
import os
import pickle
import queue
import socket
import struct
import threading
import time
from typing import Any, Callable, List, Optional, Tuple
import ctypes
import torch
import torch.distributed as dist
from .. import DistCmdHandler, DistContext

logger = logging.getLogger(__name__)

# Gloo message tags
TAG_CMD = 10          # [cmd, n_tensors, sender rank]
_CMD_EXIT = -1        # internal: unblocks the receiver's CommandThread at shutdown
TAG_CMD_META = 11     # per command tensor: [n_bytes] then pickled (dtype, shape)
TAG_CMD_DATA = 12

# Envelope on the hop's socket: int64 meta_len | int64 cpu_len | pickled payload description | CPU tensor bytes.
# meta_len == 0: same description as the previous payload of this hop (shapes are static per schedule);
# meta_len == -1: the hop is closing. cpu_len == -1: the payload's CPU tensors are the very same objects as the
# previous payload's (the constant shape / scale / bit-width tensors of the QuantPipe wire format), so the receiver
# reuses its copies. Every Python-level operation here costs a GIL hand-off between the stage's threads, which
# measured at tens of microseconds each - the steady-state path is therefore two comparisons and a 16-byte write.
_ENV_HEAD = struct.Struct('<qq')
_POLL_SEC = 0.0002


def queue_depth() -> int:
    """Capacity of the stage's in / out / res queues. The reference uses 1 (`p2p/__init__.py:374-376`); a thread
    hand-off costs a wake-up of ~0.1 ms on a busy host, so with capacity 1 producer and consumer run in lock-step.
    `PIPEEDGE_QUEUE_DEPTH` > 1 lets hand-offs overlap at the price of that many more micro-batches in flight."""
    return max(1, int(os.environ.get('PIPEEDGE_QUEUE_DEPTH', '1')))


def ring_slots() -> int:
    """Device buffers per ring: queued + in transfer + being produced + being consumed."""
    return queue_depth() + 3


def _native_lib():
    """`libpipeedge_b200.so` when this process drives a GPU (its hops carry CUDA payloads over NCCL), else None."""
    if not torch.cuda.is_available():
        return None
    from ..._lib import LIB   # pylint: disable=import-outside-toplevel
    if not LIB.pe_hop_available():
        raise RuntimeError("libnccl.so.2 cannot be loaded in this process; the hops' CUDA payloads travel over NCCL "
                           "(a CUDA build of PyTorch ships and loads it)")
    return LIB


_NCCL_HOPS_OPENED = 0


def nccl_hops_opened() -> int:
    """How many per-hop NCCL communicators this process has created (the Python-thread path; the native pipeline creates
    none). Entry points use it to decide whether the process may leave through the normal interpreter exit."""
    return _NCCL_HOPS_OPENED


class _NativeHop:
    """`pe_hop_*`: one C call per payload and side moves the device tensors over the hop's NCCL communicator."""

    def __init__(self, lib, sock: socket.socket, is_sender: bool):
        global _NCCL_HOPS_OPENED   # pylint: disable=global-statement
        from ..._lib import check   # pylint: disable=import-outside-toplevel
        self._lib, self._check = lib, check
        self._handle = ctypes.c_void_p()
        check(lib.pe_hop_open(sock.fileno(), 1 if is_sender else 0, ctypes.byref(self._handle)))
        _NCCL_HOPS_OPENED += 1

    def close(self) -> None:
        if self._handle:
            self._lib.pe_hop_close(self._handle)
            self._handle = ctypes.c_void_p()

    @staticmethod
    def _arrays(tensors):
        for t in tensors:
            if not t.is_contiguous():   # data_ptr + numel * element_size below describes contiguous memory only
                raise ValueError("hop payloads must be contiguous tensors (as the reference's Gloo send requires)")
        n = len(tensors)
        ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t in tensors])
        sizes = (ctypes.c_size_t * n)(*[t.numel() * t.element_size() for t in tensors])
        return ptrs, sizes, n

    def send(self, tensors, ready, stream, done, write_envelope: bool) -> None:
        ptrs, sizes, n = self._arrays(tensors)
        self._check(self._lib.pe_hop_send(self._handle, ptrs, sizes, n, None if ready is None else ready.cuda_event,
                                          stream.cuda_stream, done.cuda_event, 1 if write_envelope else 0))

    def wait_envelope(self):
        head = (ctypes.c_longlong * 2)()
        rc = self._lib.pe_hop_wait_envelope(self._handle, head)   # blocks with the GIL released
        if rc == 1:
            return None
        self._check(rc)
        return int(head[0]), int(head[1])

    def recv(self, slots, stream, ready) -> None:
        ptrs, sizes, n = self._arrays([slot[0] for slot in slots])
        guards = (ctypes.c_void_p * n)(*[None if slot[1] is None else slot[1].cuda_event for slot in slots])
        self._check(self._lib.pe_hop_recv(self._handle, ptrs, sizes, guards, n, stream.cuda_stream, ready.cuda_event))


def _fresh_event(stream) -> 'torch.cuda.Event':
    """An event whose CUDA handle exists (torch creates it lazily on the first record)."""
    evt = torch.cuda.Event()
    evt.record(stream)
    return evt


class ConditionQueue(queue.Queue):
    """A Queue with a public `condition: threading.Condition` for synchronization (`p2p/__init__.py:88-93`)."""

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        self.condition = threading.Condition()


class _Payload:
    """What the internal queues carry: the user-visible data plus device-side ordering information."""
    __slots__ = ('data', 'ready', 'on_consumed')

    def __init__(self, data: Any, ready: Optional['torch.cuda.Event'] = None,
                 on_consumed: Optional[Callable[['torch.cuda.Event'], None]] = None):
        self.data = data                # Tensor | Tuple[Tensor | object, ...]
        self.ready = ready              # recorded when the producing stream has written `data`
        self.on_consumed = on_consumed  # given an event recorded after the consumer's reads


def _cuda_tensors(data) -> List[torch.Tensor]:
    objs = data if isinstance(data, tuple) else (data,)
    return [o for o in objs if isinstance(o, torch.Tensor) and o.is_cuda]


class DistP2pContext(DistContext):
    """The singleton distributed P2P context manager (`p2p/__init__.py:41-85`).

    Parameters are the reference's: `ipg_args` / `ipg_kwargs` for `torch.distributed.init_process_group()`
    (the default group is the Gloo control plane) and the command handler `cmd_cb`. The data plane is not a process
    group: each hop's exchange threads open its socket and, with CUDA, its NCCL communicator (`_NativeHop`).
    """
    _instance: Optional['DistP2pContext'] = None

    def __init__(self, ipg_args: tuple, ipg_kwargs: dict, cmd_cb: DistCmdHandler):
        super().__init__(ipg_args, ipg_kwargs)
        self._thread_cmd = CommandThread(cmd_cb)
        self._listener = None
        self._sock_path = None
        self._inbound = {}                      # src rank -> accepted connection
        self._inbound_cond = threading.Condition()

    def init(self) -> None:
        """Initialize the distributed context and threads."""
        super().init()
        dist.init_process_group(*self._init_args, **self._init_kwargs)
        if self._world_size > 1:
            self._sock_path = self.sock_path(self._rank)
            if os.path.exists(self._sock_path):
                os.unlink(self._sock_path)
            self._listener = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
            self._listener.bind(self._sock_path)
            self._listener.listen(self._world_size)
            threading.Thread(target=self._accept_loop, daemon=True).start()
        DistP2pContext._instance = self
        if self._world_size > 1:   # nobody can send a command to a world of one
            self._thread_cmd.start()

    def shutdown(self) -> None:
        """Shutdown threads and the distributed context."""
        super().shutdown()
        if self._world_size > 1:
            # each rank releases its successor's any-source receive, so no request is left pending
            self._thread_cmd.stop()
            dist.send(torch.tensor([_CMD_EXIT, 0, self._rank], dtype=torch.int), dst=(self._rank + 1) % self._world_size,
                      tag=TAG_CMD)
            self._thread_cmd.join(timeout=_STOP_GRACE_SEC + 5)
            dist.barrier()
        DistP2pContext._instance = None
        if self._listener is not None:
            try:
                self._listener.close()
                os.unlink(self._sock_path)
            except OSError:
                pass
            self._listener = None
        dist.destroy_process_group()

    @staticmethod
    def sock_path(rank: int) -> str:
        """Path of `rank`'s hop listener (ranks share a node; MASTER_PORT keeps concurrent jobs apart)."""
        return f"/tmp/pipeedge_b200_{os.environ.get('MASTER_PORT', '0')}_{rank}.sock"

    def _accept_loop(self) -> None:
        while True:
            try:
                conn, _ = self._listener.accept()
            except OSError:
                return   # listener closed at shutdown
            src = struct.unpack('<i', _recv_exact(conn, 4))[0]
            with self._inbound_cond:
                self._inbound[src] = conn
                self._inbound_cond.notify_all()

    @classmethod
    def accept_from(cls, src: int, timeout: float = 120.0) -> socket.socket:
        """The inbound hop connection from rank `src` (waits for it to connect)."""
        inst = cls._instance
        assert inst is not None, "DistP2pContext is not initialised"
        with inst._inbound_cond:   # pylint: disable=protected-access
            if not inst._inbound_cond.wait_for(lambda: src in inst._inbound, timeout):
                raise TimeoutError(f"rank {src} never opened its hop to this rank")
            return inst._inbound.pop(src)

    @classmethod
    def connect_to(cls, dst: int, timeout: float = 120.0) -> socket.socket:
        """Open the outbound hop connection to rank `dst` (retries until its listener is up)."""
        inst = cls._instance
        assert inst is not None, "DistP2pContext is not initialised"
        deadline = time.monotonic() + timeout
        while True:
            sock = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
            try:
                sock.connect(cls.sock_path(dst))
                sock.sendall(struct.pack('<i', inst._rank))   # pylint: disable=protected-access
                return sock
            except OSError:
                sock.close()
                if time.monotonic() > deadline:
                    raise
                time.sleep(0.01)

    def cmd_broadcast(self, cmd: int, tensors: Optional[Tuple[torch.Tensor, ...]] = None) -> None:
        """Broadcast a command with optional (CPU) tensors to every other rank (`p2p/__init__.py:72-85`)."""
        assert self._initialized
        tensors = () if tensors is None else tuple(tensors)
        head = torch.tensor([cmd, len(tensors), self._rank], dtype=torch.int)
        reqs = []
        keep = []
        for dst in range(self._world_size):
            if dst == self._rank:
                continue
            reqs.append(dist.isend(head, dst=dst, tag=TAG_CMD))
            for tensor in tensors:
                tensor = tensor.detach().cpu().contiguous()
                meta = torch.frombuffer(bytearray(pickle.dumps((tensor.dtype, tuple(tensor.shape)))), dtype=torch.uint8)
                size = torch.tensor([meta.numel()], dtype=torch.int64)
                keep += [meta, size, tensor]
                reqs.append(dist.isend(size, dst=dst, tag=TAG_CMD_META))
                reqs.append(dist.isend(meta, dst=dst, tag=TAG_CMD_META))
                if tensor.numel() > 0:
                    reqs.append(dist.isend(tensor.view(-1), dst=dst, tag=TAG_CMD_DATA))
        for req in reqs:
            req.wait()


def _recv_exact(conn: socket.socket, n: int) -> bytes:
    """Read exactly n bytes (b'' on EOF)."""
    chunks = []
    while n > 0:
        chunk = conn.recv(min(n, 1 << 20))
        if not chunk:
            return b''
        chunks.append(chunk)
        n -= len(chunk)
    return b''.join(chunks)


class _RequestWaiter(threading.Thread):
    """Blocks in `req.wait()` on a daemon thread so that the owner can poll and still stop cleanly:
    `is_completed()` never turns true for a Gloo irecv and `wait()` cannot be interrupted (the reference works
    around the same PyTorch behaviour, `p2p/util.py:8-24`)."""

    def __init__(self, req):
        super().__init__(daemon=True)
        self._req = req
        self.done = threading.Event()
        self.error: Optional[BaseException] = None

    def run(self):
        try:
            self._req.wait()
        except BaseException as exc:   # pylint: disable=broad-except
            self.error = exc           # e.g. the process group was destroyed under us at shutdown
        self.done.set()


_STOP_GRACE_SEC = 10.0


def _poll(req, stop_evt: threading.Event) -> bool:  # noqa: C901
    """Wait for a distributed request. Once `stop_evt` is set the peer is expected to unblock us with its
    closing message; only after a grace period is the request abandoned (False). Abandoning leaves a daemon
    thread inside `wait()`, which PyTorch turns into an abort at process exit - the reference's teardown race
    (SURVEY.md section 5) - hence the explicit closing handshake instead."""
    waiter = _RequestWaiter(req)
    waiter.start()
    deadline = None
    while not waiter.done.wait(_POLL_SEC * 5):
        if stop_evt.is_set():
            if deadline is None:
                deadline = time.monotonic() + _STOP_GRACE_SEC
            elif time.monotonic() > deadline:
                return False
    return waiter.error is None


class AbstractTensorExchangeThread(threading.Thread):
    """Abstract tensor exchange thread with pre/post hooks (`p2p/__init__.py:124-152`)."""

    def __init__(self):
        super().__init__(daemon=True)
        self._pre_hooks = []
        self._post_hooks = []
        self.stats = {'wait_s': 0.0, 'busy_s': 0.0, 'n': 0}   # time blocked on the queue / peer vs. doing work
        self._evt_stop_thread = threading.Event()
        self._device = torch.cuda.current_device() if torch.cuda.is_available() else None
        self._stream = None

    def register_pre_hook(self, hook: Callable[..., None], args: tuple) -> None:
        """Register hook with signature: `hook(*args)`."""
        self._pre_hooks.append((hook, args))

    def register_post_hook(self, hook: Callable[..., None], args: tuple) -> None:
        """Register hook with signature: `hook(tensors, *args)`."""
        self._post_hooks.append((hook, args))

    def _call_pre_hooks(self):
        for hook, args in self._pre_hooks:
            hook(*args)

    def _call_post_hooks(self, tensors):
        for hook, args in self._post_hooks:
            hook(tensors, *args)

    def _enter_device(self):
        if self._device is not None:
            torch.cuda.set_device(self._device)
            self._stream = torch.cuda.Stream(device=self._device)


def _signature(objs: tuple, is_tuple: bool):
    """Cheap hashable description of a payload's structure; only pickled when it changes."""
    sig = [is_tuple]
    for obj in objs:
        if isinstance(obj, torch.Tensor):
            sig.append(('cuda' if obj.is_cuda else 'cpu', obj.dtype, tuple(obj.shape)))
        else:
            sig.append(('obj', pickle.dumps(obj), None))   # non-tensor objects ride in the description (util.py:28-38)
    return tuple(sig)


class TensorSendThread(AbstractTensorExchangeThread):
    """Thread for sending payloads to `dst_rank` (`p2p/__init__.py:155-204`)."""

    def __init__(self, queue_out: ConditionQueue, dst_rank: int):
        super().__init__()
        self._queue_out = queue_out
        self._dst_rank = dst_rank
        self._last_sig = None
        self._last_cpu: List[torch.Tensor] = []
        self._last_cpu_versions: List[int] = []
        self._sock = None
        self._hop = None
        self._inflight = collections.deque()
        self._timing_hooks: List[Tuple[Callable[..., None], tuple]] = []
        self._timed = collections.deque()     # (start event, done event, Mbits) of sends not yet reported

    def register_timing_hook(self, hook: Callable[..., None], args: tuple) -> None:
        """`hook(mbits, seconds, *args)` is called on this thread once a payload's device-side transfer has finished:
        `seconds` is the time between the CUDA events around its NCCL sends on the hop stream (it includes waiting
        for the receiver to post its buffers, like the reference's blocking send), `mbits` the bytes moved * 8e-6."""
        self._timing_hooks.append((hook, args))

    def _report_timed(self, drain: bool = False) -> None:
        while self._timed and (drain or self._timed[0][1].query()):
            start, done, mbits = self._timed.popleft()
            done.synchronize()
            seconds = start.elapsed_time(done) * 1e-3
            for hook, args in self._timing_hooks:
                hook(mbits, seconds, *args)

    def stop(self) -> None:
        """Direct the thread to stop."""
        with self._queue_out.condition:
            self._evt_stop_thread.set()
            self._queue_out.condition.notify_all()

    def run(self):
        """Dequeue payloads and send them."""
        self._enter_device()
        if self._sock is None:
            self.open_hop()
        try:
            self._run()
        finally:
            if self._hop is not None and self._inflight:
                self._inflight[-1].synchronize()     # every send has left: the peer's matching receives complete too
            try:
                self._report_timed(drain=True)
            except Exception:   # pylint: disable=broad-except
                logger.exception("hop timing hook failed during shutdown")
            if self._sock is not None:   # (None when open_hop itself failed)
                try:   # tell the receiver this hop is closing, so that its blocking receive returns
                    self._sock.sendall(_ENV_HEAD.pack(-1, 0))
                except OSError:
                    pass
            if self._hop is not None:
                self._hop.close()                    # both ends now destroy the hop's communicator at about the same time
            if self._sock is not None:
                try:
                    self._sock.close()
                except OSError:
                    pass

    def open_hop(self) -> None:
        """Connect to the receiver and, on a GPU, join the hop's NCCL communicator (blocks until the peer does)."""
        self._sock = DistP2pContext.connect_to(self._dst_rank)
        lib = _native_lib()
        self._hop = _NativeHop(lib, self._sock, True) if lib is not None else None

    def _send_envelope(self, sig, cpu: List[torch.Tensor], defer_fast: bool = False) -> bool:
        """Write the payload's envelope; returns True if it was (or, with `defer_fast`, is to be) the 16-byte
        steady-state header."""
        same_sig = sig == self._last_sig
        last_cpu = self._last_cpu
        versions = [t._version for t in cpu]   # pylint: disable=protected-access
        if same_sig and len(cpu) == len(last_cpu) and all(a is b for a, b in zip(cpu, last_cpu)) and \
                versions == self._last_cpu_versions:    # same objects AND not written in place since they were sent
            if not defer_fast:
                self._sock.sendall(_ENV_HEAD.pack(0, -1))   # steady state: nothing but the header
            return True
        meta = b'' if same_sig else pickle.dumps(sig)
        self._last_sig = sig
        self._last_cpu = list(cpu)   # keeps the objects alive, so `is` cannot match a recycled id
        self._last_cpu_versions = versions
        parts = [t.contiguous().view(-1).view(torch.uint8).numpy().tobytes() for t in cpu if t.numel() > 0]
        blob_len = sum(len(part) for part in parts)
        self._sock.sendall(b''.join([_ENV_HEAD.pack(len(meta), blob_len), meta, *parts]))
        return False

    def _run(self):
        while not self._evt_stop_thread.is_set():
            t_wait = time.perf_counter()
            with self._queue_out.condition:
                while self._queue_out.empty():
                    if self._evt_stop_thread.is_set():
                        return
                    self._queue_out.condition.wait()
                payload = self._queue_out.get(block=False)
                self._queue_out.condition.notify_all()
            t_busy = time.perf_counter()
            self.stats['wait_s'] += t_busy - t_wait
            data = payload.data
            is_tuple = isinstance(data, tuple)
            objs = data if is_tuple else (data,)
            tensors = [o for o in objs if isinstance(o, torch.Tensor)]
            cpu = [t for t in tensors if not t.is_cuda]
            cuda = [t for t in tensors if t.is_cuda]
            fast = self._send_envelope(_signature(objs, is_tuple), cpu, defer_fast=bool(cuda))
            self._call_pre_hooks()
            if cuda:
                # envelope header + NCCL sends + event record in one GIL-free call (CUDA tensors exist only in a process
                # with CUDA, where open_hop has joined the hop's communicator)
                hop = self._hop
                for tensor in cuda:
                    tensor.record_stream(self._stream)
                if self._timing_hooks:
                    # device-side hop time: events on the hop stream right before / after the sends
                    self._report_timed()
                    if payload.ready is not None:
                        self._stream.wait_event(payload.ready)
                    start = torch.cuda.Event(enable_timing=True)
                    start.record(self._stream)
                    done = torch.cuda.Event(enable_timing=True)
                    done.record(self._stream)   # creates the handle; re-recorded by the hop after the sends
                    hop.send(cuda, None, self._stream, done, write_envelope=fast)
                    self._timed.append((start, done, sum(t.numel() * t.element_size() for t in cuda) * 8e-6))
                else:
                    done = _fresh_event(self._stream)
                    hop.send(cuda, payload.ready, self._stream, done, write_envelope=fast)
                if payload.on_consumed is not None:
                    payload.on_consumed(done)
                self._inflight.append(done)
                # bound the number of sends the host may run ahead of the device
                while len(self._inflight) > 1 + queue_depth():
                    self._inflight.popleft().synchronize()
            elif payload.on_consumed is not None:
                payload.on_consumed(None)
            self._call_post_hooks(tuple(tensors))
            self.stats['busy_s'] += time.perf_counter() - t_busy
            self.stats['n'] += 1


class TensorRecvThread(AbstractTensorExchangeThread):
    """Thread for receiving payloads from `src_rank` (`p2p/__init__.py:207-258`)."""

    def __init__(self, queue_in: ConditionQueue, src_rank: int):
        super().__init__()
        self._queue_in = queue_in
        self._src_rank = src_rank
        self._sig = None
        self._last_cpu: List[torch.Tensor] = []
        self._conn = None
        self._hop = None
        self._rings = {}
        self._slots = ring_slots()
        self._count = 0

    def stop(self) -> None:
        """Direct the thread to stop."""
        self._evt_stop_thread.set()

    def _slot(self, pos: int, dtype, shape):
        """Next device receive buffer for payload position `pos`, plus its 'consumer finished' guard."""
        key = (pos, dtype, shape)
        ring = self._rings.get(key)
        if ring is None:
            ring = [[torch.empty(shape, dtype=dtype, device=torch.device('cuda', self._device)), None]
                    for _ in range(self._slots)]
            self._rings[key] = ring
        return ring[self._count % self._slots]

    def run(self):
        """Receive payloads and enqueue them."""
        self._enter_device()
        if self._conn is None:
            self.open_hop()
        conn, hop = self._conn, self._hop
        try:
            self._loop(conn, hop)
        finally:
            if hop is not None:
                if self._stream is not None:
                    self._stream.synchronize()
                hop.close()
            conn.close()

    def open_hop(self) -> None:
        """Accept the sender's connection and, on a GPU, join the hop's NCCL communicator."""
        self._conn = DistP2pContext.accept_from(self._src_rank)
        lib = _native_lib()
        self._hop = _NativeHop(lib, self._conn, False) if lib is not None else None

    def _loop(self, conn, hop):
        while True:
            # blocks until the sender's next payload or its closing envelope (sent by its shutdown); no polling
            # thread per message as in the reference (`p2p/__init__.py:224-232`)
            t_wait = time.perf_counter()
            if hop is not None:
                head = hop.wait_envelope()
                t_busy = time.perf_counter()
                self.stats['wait_s'] += t_busy - t_wait
                if head is None:
                    return      # the sender went away
                meta_len, cpu_len = head
            else:
                head = _recv_exact(conn, _ENV_HEAD.size)
                t_busy = time.perf_counter()
                self.stats['wait_s'] += t_busy - t_wait
                if not head:
                    return      # the sender went away
                meta_len, cpu_len = _ENV_HEAD.unpack(head)
            if meta_len < 0:
                return          # the sender closed the hop
            reuse_cpu = cpu_len < 0
            cpu_len = max(cpu_len, 0)
            body = _recv_exact(conn, meta_len + cpu_len) if meta_len + cpu_len > 0 else b''
            if meta_len > 0:
                self._sig = pickle.loads(body[:meta_len])
            sig = self._sig
            self._call_pre_hooks()
            objs: List[Any] = []
            cuda_slots = []
            off = meta_len
            cpu_iter = iter(self._last_cpu) if reuse_cpu else None
            new_cpu = []
            for pos, (plane, dtype, shape) in enumerate(sig[1:]):
                if plane == 'obj':
                    objs.append(pickle.loads(dtype))
                elif plane == 'cpu':
                    if reuse_cpu:
                        tensor = next(cpu_iter)   # read-only by contract: the same object is handed out again
                    else:
                        tensor = torch.empty(shape, dtype=dtype)
                        nbytes = tensor.numel() * tensor.element_size()
                        if nbytes > 0:
                            tensor.view(-1).view(torch.uint8).copy_(torch.frombuffer(bytearray(body[off:off + nbytes]), dtype=torch.uint8))
                            off += nbytes
                        new_cpu.append(tensor)
                    objs.append(tensor)
                else:
                    slot = self._slot(pos, dtype, shape)
                    cuda_slots.append(slot)
                    objs.append(slot[0])
            if not reuse_cpu:
                self._last_cpu = new_cpu
            ready = None
            on_consumed = None
            if cuda_slots:   # device buffers exist only with CUDA, where open_hop has joined the hop's communicator
                ready = _fresh_event(self._stream)
                hop.recv(cuda_slots, self._stream, ready)

                def on_consumed(evt, slots=tuple(cuda_slots)):
                    for slot in slots:
                        slot[1] = evt
            self._count += 1
            self._call_post_hooks(tuple(t for t in objs if isinstance(t, torch.Tensor)))
            data = tuple(objs) if sig[0] else objs[0]
            self.stats['busy_s'] += time.perf_counter() - t_busy
            self.stats['n'] += 1
            with self._queue_in.condition:
                while self._queue_in.full():
                    if self._evt_stop_thread.is_set():
                        return
                    self._queue_in.condition.wait(0.05)
                self._queue_in.put(_Payload(data, ready, on_consumed))
                self._queue_in.condition.notify_all()


class TensorWorkThread(threading.Thread):
    """Thread for processing payloads with `callback` (`p2p/__init__.py:261-295`)."""

    def __init__(self, queue_in: ConditionQueue, queue_out: Optional[ConditionQueue], callback: Callable):
        super().__init__(daemon=True)
        self._queue_in = queue_in
        self._queue_out = queue_out
        self._callback = callback
        self._evt_stop_thread = threading.Event()
        self._device = torch.cuda.current_device() if torch.cuda.is_available() else None
        self.stats = {'wait_s': 0.0, 'busy_s': 0.0, 'n': 0}
        self.exception: Optional[BaseException] = None

    def stop(self) -> None:
        """Direct the thread to stop."""
        with self._queue_in.condition:
            self._evt_stop_thread.set()
            self._queue_in.condition.notify_all()

    def run(self):
        """Dequeue, process, enqueue."""
        stream = None
        if self._device is not None:
            torch.cuda.set_device(self._device)
            stream = torch.cuda.Stream(device=self._device)
        while True:
            t_wait = time.perf_counter()
            with self._queue_in.condition:
                while self._queue_in.empty():
                    if self._evt_stop_thread.is_set():
                        return
                    self._queue_in.condition.wait()
                payload = self._queue_in.get(block=False)
                self._queue_in.condition.notify_all()
            t_busy = time.perf_counter()
            self.stats['wait_s'] += t_busy - t_wait
            try:
                if stream is not None:
                    with torch.cuda.stream(stream):
                        if payload.ready is not None:
                            stream.wait_event(payload.ready)
                        result = self._callback(payload.data)
                        done = torch.cuda.Event()
                        done.record(stream)
                    if payload.on_consumed is not None:
                        payload.on_consumed(done)
                else:
                    result = self._callback(payload.data)
                    done = None
                    if payload.on_consumed is not None:
                        payload.on_consumed(None)
                # A shard that writes its outputs into a ring of persistent buffers (CUDA-graph mode) must not reuse
                # a buffer before the hop has sent it: the sender's "sent" event goes back to the shard.
                guard = getattr(self._callback, 'output_guard', None)
                sent_cb = guard() if callable(guard) else None
            except BaseException as exc:   # pylint: disable=broad-except
                # the reference loses worker exceptions and hangs (SURVEY.md 8b); keep it for the owner to re-raise
                self.exception = exc
                raise
            self.stats['busy_s'] += time.perf_counter() - t_busy
            self.stats['n'] += 1
            if result is not None and self._queue_out is not None:
                with self._queue_out.condition:
                    while self._queue_out.full():
                        if self._evt_stop_thread.is_set():
                            return
                        self._queue_out.condition.wait(0.05)
                    self._queue_out.put(_Payload(result, done, sent_cb))
                    self._queue_out.condition.notify_all()


class CommandThread(threading.Thread):
    """Thread for receiving commands from any rank (`p2p/__init__.py:298-331`)."""

    def __init__(self, callback: DistCmdHandler):
        super().__init__(daemon=True)
        self._callback = callback
        self._evt_stop_thread = threading.Event()

    def stop(self) -> None:
        """Direct the thread to stop."""
        self._evt_stop_thread.set()

    def run(self):
        """Listen for commands."""
        while True:
            head = torch.zeros(3, dtype=torch.int)
            if not _poll(dist.irecv(head, tag=TAG_CMD), self._evt_stop_thread):
                return
            src = int(head[2])   # the sender names itself: any-source requests do not report their source
            cmd, count = int(head[0]), int(head[1])
            if cmd == _CMD_EXIT:
                return
            tensors = ()
            for _ in range(count):
                size = torch.zeros(1, dtype=torch.int64)
                dist.recv(size, src=src, tag=TAG_CMD_META)
                meta = torch.empty(int(size[0]), dtype=torch.uint8)
                dist.recv(meta, src=src, tag=TAG_CMD_META)
                dtype, shape = pickle.loads(meta.numpy().tobytes())
                tensor = torch.empty(shape, dtype=dtype)
                if tensor.numel() > 0:
                    dist.recv(tensor.view(-1), src=src, tag=TAG_CMD_DATA)
                tensors += (tensor,)
            self._callback(cmd, tensors)


class DistP2pPipelineStage:
    """The singleton distributed P2P pipeline stage context manager (`p2p/__init__.py:334-450`).

    `rank_src` / `rank_dst`: ranks to receive payloads from / send them to (None = not applicable);
    `work_cb(payload) -> payload | None`: the stage's shard (None relays); `results_cb(payload)`: consumer of
    the last stage's output on the data rank. Thread and queue topology follow the reference's `_create_stage`.
    """

    def __init__(self, rank_src: Optional[int], rank_dst: Optional[int], work_cb: Optional[Callable],
                 results_cb: Optional[Callable[[Any], None]]):
        self._initialized = False
        self._queues = {}
        self._threads = {}
        self._args = (rank_src, rank_dst, work_cb, results_cb)
        self._native = None            # _native.NativeStage once init() has chosen the native pipeline
        self._native_world = False     # every rank agreed on it (then shutdown ends with a drain barrier everywhere)
        self._create_stage(rank_src, rank_dst, work_cb, results_cb)

    # ------------------------------------------------------------------ native pipeline selection
    def _host_feeder(self) -> bool:
        """A data rank outside the stage pipeline (no worker, both ranks set) without a CUDA device: the native pipeline
        serves it through rings in shared memory (`_native.NativeHostFeeder`); the Python-thread path cannot."""
        rank_src, rank_dst, work_cb, results_cb = self._args
        return work_cb is None and results_cb is not None and rank_src is not None and rank_dst is not None and \
            not torch.cuda.is_available()

    def _native_capable(self) -> bool:
        """Whether THIS rank's role can run on the native pipeline (csrc/pipe.cu): a native shard as the worker, hooks
        that the link kernels account for, the reference's ring topology with the data rank on the first stage - or the
        data rank outside the stage pipeline (no worker, both ranks set), which feeds the first stage through a relay,
        or, without a CUDA device, through a ring in shared memory. A rank without a CUDA device is capable only in
        that role, or idle."""
        rank_src, rank_dst, work_cb, results_cb = self._args
        if os.environ.get('PIPEEDGE_NATIVE', '1') == '0':
            return False
        if rank_src is None and rank_dst is None and work_cb is None and results_cb is None:
            return True    # idle rank: neutral
        if not torch.cuda.is_available() and not self._host_feeder():
            return False
        try:
            from ._native import shard_is_native   # pylint: disable=import-outside-toplevel
        except ImportError:
            return False
        feeder = work_cb is None and results_cb is not None and rank_src is not None and rank_dst is not None
        if not feeder and (work_cb is None or not shard_is_native(work_cb)):
            return False
        if any(thr._pre_hooks or thr._post_hooks   # pylint: disable=protected-access
               for thr in self._threads.values() if isinstance(thr, AbstractTensorExchangeThread)):
            return False   # user hooks run on the Python exchange threads (send-timing hooks do not: device timestamps)
        if (rank_src is None) != (rank_dst is None):
            return False
        if results_cb is not None and not feeder and not work_cb.shard_config.is_first:
            return False
        return True

    def _choose_native(self) -> bool:
        capable = self._native_capable()
        if dist.is_initialized() and dist.get_world_size() > 1:
            # Every rank votes, with or without a CUDA device: [capable, -(host feeder), -(has a CUDA device)], MIN.
            # A data rank without a GPU outside the stage pipeline needs the native pipeline; so does the rest of the
            # world when any rank has a GPU (a world without one runs the Python threads over Gloo, as before).
            host_feeder = self._host_feeder()
            vote = torch.tensor([1 if capable else 0, -1 if host_feeder else 0, -1 if torch.cuda.is_available() else 0],
                                dtype=torch.int)
            dist.all_reduce(vote, op=dist.ReduceOp.MIN)    # control plane (Gloo); every rank builds a stage object
            native = bool(vote[0] == 1)
            if not native and int(vote[1]) < 0 and int(vote[2]) < 0:
                raise RuntimeError("the data rank has no CUDA device: only the native pipeline can serve it, and not "
                                   "every rank can run it (PIPEEDGE_NATIVE=0, exchange hooks, or a shard it does not "
                                   "support); give the data rank a GPU or run every rank natively")
            return native
        return capable and self._args[0] is None and self._args[1] is None

    def _create_stage(self, rank_src, rank_dst, work_cb, results_cb):
        depth = queue_depth()
        self._queues['in'] = ConditionQueue(maxsize=depth)
        self._queues['out'] = ConditionQueue(maxsize=depth)
        self._queues['res'] = ConditionQueue(maxsize=depth)
        if work_cb is None:
            self._queues['out'] = self._queues['in']   # relay without a worker
        else:
            self._threads['work'] = TensorWorkThread(self._queues['in'], self._queues['out'], work_cb)
            if hasattr(work_cb, 'num_slots'):
                # outputs in flight between the worker and the wire: queued + being sent + being produced
                work_cb.num_slots = max(int(work_cb.num_slots), 2 * depth + 3)
        if results_cb is not None:
            queue_res = self._queues['out'] if rank_dst is None else self._queues['res']
            self._threads['res'] = TensorWorkThread(queue_res, None, results_cb)
        if rank_dst is not None:
            self._threads['send'] = TensorSendThread(self._queues['out'], rank_dst)
        if rank_src is not None:
            queue_in = self._queues['in'] if results_cb is None else self._queues['res']
            self._threads['recv'] = TensorRecvThread(queue_in, rank_src)

    def init(self) -> None:
        """Start the threads - or, when every rank runs a native shard with hooks the link kernels account for, the
        native pipeline (one CUDA graph per micro-batch, stage loop in C; `_native.py`)."""
        assert not self._initialized
        self._initialized = True
        if self._choose_native():
            self._native_world = True
            rank_src, rank_dst, work_cb, results_cb = self._args
            if work_cb is not None:
                from ._native import NativeStage   # pylint: disable=import-outside-toplevel
                self._native = NativeStage(rank_src, rank_dst, work_cb, results_cb)
            elif results_cb is not None and self._host_feeder():   # ... outside the stage pipeline, without a GPU
                from ._native import NativeHostFeeder   # pylint: disable=import-outside-toplevel
                self._native = NativeHostFeeder(rank_src, rank_dst, results_cb)
            elif results_cb is not None:   # the data rank outside the stage pipeline
                from ._native import NativeFeeder   # pylint: disable=import-outside-toplevel
                self._native = NativeFeeder(rank_src, rank_dst, results_cb)
            if self._native is not None:
                send = self._threads.get('send')
                for hook, args in (send._timing_hooks if send is not None else ()):   # pylint: disable=protected-access
                    self._native.add_send_timing_hook(hook, args)   # registered before init(): stamps from the start
                self._native.init(DistP2pContext.connect_to, DistP2pContext.accept_from)
            return
        # Open this rank's hops in ascending order of the hop's SENDER rank before any thread runs. Opening blocks
        # until the peer joins (socket accept, NCCL communicator init); a global order rules out circular waits.
        hops = []
        if 'send' in self._threads:
            hops.append((dist.get_rank(), self._threads['send']))
        if 'recv' in self._threads:
            hops.append((self._threads['recv']._src_rank, self._threads['recv']))   # pylint: disable=protected-access
        for _, thr in sorted(hops, key=lambda h: h[0]):
            thr.open_hop()
        for thr in self._threads.values():
            thr.start()

    def shutdown(self) -> None:
        """Stop and join the threads."""
        assert self._initialized
        self._initialized = False
        if self._native_world:
            if self._native is not None:
                self._native.shutdown()
            elif dist.is_initialized() and dist.get_world_size() > 1:
                from ._native import drain_barrier   # pylint: disable=import-outside-toplevel
                drain_barrier()    # idle rank: the stages' drain barrier counts every rank
            return
        # workers drain first, then the sender closes its hop (which lets the peer's receiver finish), then our
        # receiver waits for the upstream sender's closing message
        for name in ('work', 'res', 'send', 'recv'):
            thr = self._threads.get(name)
            if thr is not None:
                thr.stop()
                thr.join(timeout=_STOP_GRACE_SEC + 5)

    def register_recv_pre_hook(self, hook: Callable[..., None], args: tuple) -> None:
        """Register a pre hook for tensor receive with signature: `hook(*args)`."""
        self._no_hooks_on_native()
        thr = self._threads.get('recv')
        if thr is not None:
            thr.register_pre_hook(hook, args)

    def register_recv_post_hook(self, hook: Callable[..., None], args: tuple) -> None:
        """Register a post hook for tensor receive with signature: `hook(tensors, *args)`."""
        self._no_hooks_on_native()
        thr = self._threads.get('recv')
        if thr is not None:
            thr.register_post_hook(hook, args)

    def register_send_pre_hook(self, hook: Callable[..., None], args: tuple) -> None:
        """Register a pre hook for tensor send with signature: `hook(*args)`."""
        self._no_hooks_on_native()
        thr = self._threads.get('send')
        if thr is not None:
            thr.register_pre_hook(hook, args)

    def register_send_post_hook(self, hook: Callable[..., None], args: tuple) -> None:
        """Register a post hook for tensor send with signature: `hook(tensors, *args)`."""
        self._no_hooks_on_native()
        thr = self._threads.get('send')
        if thr is not None:
            thr.register_post_hook(hook, args)

    def register_send_timing_hook(self, hook: Callable[..., None], args: tuple) -> None:
        """Register `hook(mbits, seconds, *args)`, called with each payload's DEVICE-side transfer time (CUDA events
        around the hop's NCCL sends). The send post hook above fires when a send is enqueued, not when it has
        finished, so bandwidth-driven policies (`runtime.py:121-216` in the reference) read this instead. No
        reference equivalent: there the blocking send itself is timed on the host.

        Legal before or after `init()` on the native pipeline too: there `seconds` is the send's duration from the
        graph's device timestamps (send start -> payload published; it includes waiting for a free slot, like the
        NCCL send includes waiting for the receiver) and `mbits` is what the thread path reports for the same payload."""
        if self._native is not None:
            self._native.add_send_timing_hook(hook, args)
            return
        if self._native_world:
            return   # idle rank: it sends nothing
        thr = self._threads.get('send')
        if thr is not None:
            thr.register_timing_hook(hook, args)

    def _no_hooks_on_native(self) -> None:
        if self._native_world:
            raise RuntimeError("the native pipeline is running: register exchange hooks BEFORE init() (they select the "
                               "Python exchange threads) or set PIPEEDGE_NATIVE=0")

    @property
    def native(self):
        """The `_native.NativeStage` driving this rank (a `_native.NativeFeeder` on a data rank outside the stage
        pipeline, a `_native.NativeHostFeeder` on one without a CUDA device), or None (Python threads / idle rank)."""
        return self._native

    def prepare(self, ubatch: int, dim1: int = 0) -> None:
        """Optional: capture the stage's CUDA graph for micro-batches of `ubatch` items (`dim1`: BERT sequence length)
        before the first payload arrives. No-op on the Python-thread path. Call before any traffic."""
        if self._native is not None:
            self._native.prepare(ubatch, dim1)

    def __enter__(self):
        self.init()
        return self

    def __exit__(self, *args):
        self.shutdown()

    def stats(self) -> dict:
        """Per-thread host time: blocked waiting (`wait_s`) vs working (`busy_s`) and items handled."""
        if self._native_world:
            return {}
        return {name: dict(thr.stats) for name, thr in self._threads.items() if hasattr(thr, 'stats')}

    def check_workers(self) -> None:
        """Re-raise an exception that killed a worker thread (the reference would hang instead)."""
        if self._native is not None:
            self._native.check()
            return
        for thr in self._threads.values():
            exc = getattr(thr, 'exception', None)
            if exc is not None:
                raise RuntimeError("a pipeline worker thread failed") from exc

    def enqueue_tensor(self, tensor: torch.Tensor) -> None:
        """Insert data into the pipeline; blocks while the inbound queue is full (`p2p/__init__.py:442-450`)."""
        assert self._initialized
        if self._native is not None:
            self._native.enqueue(tensor)
            return
        queue_in = self._queues['in']
        with queue_in.condition:
            while queue_in.full():
                self.check_workers()
                queue_in.condition.wait(0.5)
            queue_in.put(_Payload(tensor))
            queue_in.condition.notify_all()
