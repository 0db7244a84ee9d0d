"""The harness of the multi-rank pipeline tests: one spawned process per rank, the shards and QuantPipe hooks those
ranks run (and the same shards back to back in the test process), the CPU oracle's bound, `runtime.py` launched on
several ranks, and a one-process pipe fed from the host that sends into a loop-back link."""
import ctypes
import faulthandler
import os
import socket
import subprocess
import sys
import numpy as np
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the model, batch, micro-batch and partition of every `runtime.py` run; a test adds its own -q, -r and -D
RUNTIME_MODEL = ('-m', 'facebook/deit-tiny-distilled-patch16-224', '-b', '64', '-u', '8', '-pt', '1,24,25,48')


def free_port() -> int:
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def ragged(i, n_ubatch, ubatch):
    """Items in micro-batch i: the last micro-batch is one short."""
    return ubatch - 1 if (i == n_ubatch - 1 and ubatch > 1) else ubatch


def make_shard(name, cuts, s, qbit=0, weights=None, hooks=(), monitor=False):
    """Stage `s` of the model cut after `cuts`, with the hooks `runtime.py` gives it, registered in its order: `hooks`
    and the monitor run before the encode in the forward, and the native stage inspects all of them."""
    import runtime as rt
    from pipeedge_b200.models import ModuleShardConfig
    from pipeedge_b200.models.transformers import bert, deit, vit
    from pipeedge_b200.synth import MODEL_SPECS, hf_config, synth_weights
    spec = MODEL_SPECS[name]
    classes = {'vit': vit.ViTShardForImageClassification, 'deit': deit.DeiTShardForImageClassification,
               'bert': bert.BertShardForSequenceClassification}
    lo = 1 if s == 0 else cuts[s - 1] + 1
    cfg = ModuleShardConfig(layer_start=lo, layer_end=cuts[s], is_first=lo == 1, is_last=cuts[s] == spec.layers)
    shard = classes[spec.family](hf_config(spec), cfg, weights if weights is not None else synth_weights(spec, seed=0))
    shard.register_buffer('quant_bit', torch.tensor(qbit), persistent=False)
    for hook in hooks:
        shard.register_forward_hook(hook)
    if monitor:
        shard.register_forward_hook(rt.forward_hook_monitor)
    if s != len(cuts) - 1:
        shard.register_forward_hook(rt.forward_hook_quant_encode)
    if s != 0:
        shard.register_forward_pre_hook(rt.forward_pre_hook_quant_decode)
    if monitor:
        shard.register_forward_pre_hook(rt.forward_pre_hook_monitor)
    return shard


def run_local(shards, inputs):
    """The shards back to back in this process (no communication): the logits of every input."""
    outs = []
    for x in inputs:
        for shard in shards:
            x = shard(x)
        outs.append(x.cpu().numpy())
    return outs


def assert_within_oracle(name, logits, inputs):
    """Each micro-batch's logits within 4e-3 * max|ref| of the whole model run by the CPU oracle."""
    from oracle import shards as osh
    from pipeedge_b200.synth import MODEL_SPECS, synth_weights
    spec = MODEL_SPECS[name]
    w = synth_weights(spec, seed=0)
    for i, (got, x) in enumerate(zip(logits, inputs)):
        want = osh.shard_forward(spec, w, 1, spec.layers, x).numpy()
        assert np.abs(got - want).max() <= 4e-3 * np.abs(want).max(), f"micro-batch {i}"


def _rank_main(rank, worker, world, port, args, env, hang_dump, hard_exit, out_q):
    if hang_dump:
        faulthandler.enable()   # a native crash prints every thread's Python stack into the test log
        faulthandler.dump_traceback_later(hang_dump, exit=True)   # a hung rank shows where, and ends
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), **env)
    if torch.cuda.is_available():   # the Gloo suite hides the GPUs
        os.environ.setdefault('PIPEEDGE_LINK_TIMEOUT_S', '60')   # ranks sharing one GPU are time-sliced
        torch.cuda.set_device(rank % torch.cuda.device_count())
    out_q.put((rank, worker(rank, world, *args)))
    faulthandler.cancel_dump_traceback_later()
    out_q.close()
    out_q.join_thread()
    sys.stdout.flush()
    sys.stderr.flush()
    if hard_exit:
        os._exit(0)   # pylint: disable=protected-access


def spawn(worker, world, args=(), env=None, get_timeout=600, join_timeout=180, hang_dump=None, hard_exit=False):
    """Run `worker(rank, world, *args)` in one spawned process per rank, with `env` set in each, and return
    {rank: what it returned}. `worker` is a module-level function of its test module (spawn pickles it by name).
    `hard_exit`: the ranks leave with os._exit(0), without the interpreter's exit-time teardown."""
    ctx = mp.get_context('spawn')
    out_q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_rank_main, args=(r, worker, world, port, args, env or {}, hang_dump, hard_exit, out_q))
             for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    try:
        for _ in range(world):
            rank, result = out_q.get(timeout=get_timeout)
            got[rank] = result
    finally:
        for p in procs:
            p.join(join_timeout)
            if p.is_alive():
                p.kill()
                p.join(10)
    for r, p in enumerate(procs):
        assert p.exitcode == 0, f"rank {r} exited with {p.exitcode}"
    return got


def run_runtime(tmp_path, world, args, env):
    """`runtime.py` on `world` ranks of this host with RUNTIME_MODEL and `args`, each rank's stdout and stderr merged:
    {rank: output}. Every rank must exit with 0."""
    port = free_port()
    procs = {}
    for rank in reversed(range(world)):
        argv = [sys.executable, os.path.join(ROOT, 'runtime.py'), str(rank), str(world), '--port', str(port),
                *RUNTIME_MODEL, *args]
        procs[rank] = subprocess.Popen(argv, cwd=str(tmp_path), env=dict(env, LOCAL_RANK=str(rank)),
                                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    outs = {}
    for rank, p in procs.items():
        try:
            outs[rank], _ = p.communicate(timeout=600)
        except subprocess.TimeoutExpired:
            p.kill()
            outs[rank], _ = p.communicate()
    for rank, p in procs.items():
        assert p.returncode == 0, outs[rank][-3000:]
    return outs


class LoopbackPipe:
    """A pipe whose input ring is fed from the host and whose sends go into a loop-back link in this process (raw
    receive, no stage kernels); with `results` it also drains its results from that link."""

    def __init__(self, in_bytes, out_bytes, slots=4, quant_hint=0, results=True):
        from pipeedge_b200._lib import LIB, check
        self.link_in, self.loop, self.pipe = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
        check(LIB.pe_link_open_host(in_bytes, slots, ctypes.byref(self.link_in)))
        check(LIB.pe_link_open_local(out_bytes, slots, quant_hint, ctypes.byref(self.loop)))
        check(LIB.pe_pipe_create(self.link_in, self.loop, self.loop if results else None, ctypes.byref(self.pipe)))
        self.buf = torch.zeros(in_bytes // 4, dtype=torch.float32, device='cuda')   # every capture's receive buffer

    def __enter__(self):
        return self

    def __exit__(self, *_):
        from pipeedge_b200._lib import LIB
        LIB.pe_pipe_destroy(self.pipe)
        LIB.pe_link_close(self.loop)
        LIB.pe_link_close(self.link_in)

    def capture(self, items, n, bit, raw_bytes):
        """Capture the graph of `items` raw inputs sending `n` values per item at `bit` bits: its kernel count."""
        from pipeedge_b200._lib import LIB, check
        kernels = ctypes.c_int()
        check(LIB.pe_pipe_set_out_dim(self.pipe, n))
        check(LIB.pe_pipe_capture_begin(self.pipe, items, 0, 0, self.buf.data_ptr(), None, 0, 0, raw_bytes))
        check(LIB.pe_pipe_capture_end(self.pipe, self.buf.data_ptr(), None, n, None, None, 0, items, bit,
                                      1 if bit else 0, 0, ctypes.byref(kernels)))
        return kernels.value

    def submit_and_drain(self, src, items, n):
        """Submit the pinned fp32 `src` and return a copy of its result."""
        from pipeedge_b200._lib import LIB, check
        check(LIB.pe_pipe_submit(self.pipe, src.data_ptr(), src.numel() * 4, 1, items, 0))
        ptr, got_items, got_n = ctypes.c_void_p(), ctypes.c_int(), ctypes.c_size_t()
        check(LIB.pe_pipe_next_result(self.pipe, ctypes.byref(ptr), ctypes.byref(got_items), ctypes.byref(got_n)))
        return np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_float)), shape=(items * n,)).copy()
