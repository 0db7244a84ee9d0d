"""CPU: replicas of the stage pipeline fed by one data rank outside them (`runtime.py --replicas R`) - the schedule and
its refusals, the command broadcast, each rank's neighbours, the data rank's round-robin fan-out and in-order fan-in
(with stand-in feeders that finish out of order), the host data rank end to end against stand-in stages that attach to
its shared-memory rings, and the refusal of every rank when one cannot run the native pipeline."""
import ctypes
import os
import subprocess
import sys
import threading
import time
import pytest
import torch

import model_cfg
import monitoring
import runtime as rt
from pipeedge_b200.comm.p2p import DistP2pPipelineStage
from pipeedge_b200.comm.p2p._native import InOrderResults, NativeReplicaFeeder

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _multirank as mr  # noqa: E402

MODEL = 'facebook/deit-tiny-distilled-patch16-224'   # 48 sub-layers
PT = [(1, 24), (25, 48)]
ENV = {'CUDA_VISIBLE_DEVICES': ''}


# ---------------------------------------------------------------------------------------------------- the schedule
def test_default_schedule_is_every_other_rank_ascending_and_leftovers_stay_idle():
    layers, quant, ranks = rt.replica_schedule(8, 3, PT, [8, 0], None, 0, MODEL)
    assert layers == PT and quant == [8, 0]
    assert ranks == [[1, 2], [3, 4], [5, 6]]   # rank 7 stays idle
    layers, quant, ranks = rt.replica_schedule(5, 2, PT, None, None, 2, MODEL)
    assert quant == [0, 0] and ranks == [[0, 1], [3, 4]]


def test_explicit_rank_order_is_replica_major():
    _, _, ranks = rt.replica_schedule(7, 3, PT, None, [6, 5, 4, 3, 2, 1], 0, MODEL)
    assert ranks == [[6, 5], [4, 3], [2, 1]]


def test_without_a_partition_each_replica_is_one_stage_of_every_layer():
    layers, quant, ranks = rt.replica_schedule(4, 3, None, None, None, 0, MODEL)
    assert layers == [(1, 48)] and quant == [0] and ranks == [[1], [2], [3]]


@pytest.mark.parametrize('kwargs,match', [
    (dict(world=5, rank_order=[0, 1, 2, 3]), 'inside a replica'),
    (dict(world=5, rank_order=[1, 2, 3, 4], data_rank=3), 'inside a replica'),
    (dict(world=4), 'the world has 4'),
    (dict(world=4, rank_order=[1, 2, 3, 0]), 'the world has 4'),
    (dict(world=6, rank_order=[1, 2, 2, 3]), 'a rank twice'),
    (dict(world=6, rank_order=[1, 2, 3]), 'take 4'),
    (dict(world=6, rank_order=[1, 2, 3, 9]), 'outside the world'),
    (dict(world=5, data_rank=5), 'not a rank'),
    (dict(world=5, automated=True), 'automated scheduling'),
    (dict(world=5, quant=[8]), '1 bit-widths'),
    (dict(world=5, partition=None, quant=[8]), 'partition with quantization'),
    (dict(world=5, replicas=0), 'at least 1'),
])
def test_schedules_that_cannot_run_are_refused(kwargs, match):
    args = dict(world=5, replicas=2, partition=PT, quant=None, rank_order=None, data_rank=0, automated=False)
    args.update(kwargs)
    with pytest.raises(ValueError, match=match):
        rt.replica_schedule(args['world'], args['replicas'], args['partition'], args['quant'], args['rank_order'],
                            args['data_rank'], MODEL, automated=args['automated'])


def test_runtime_refuses_a_bad_replica_command_line_before_joining_the_world(tmp_path):
    """Every rank checks its own command line first: no process group is created, nothing waits for rank 0."""
    for extra, match in ((['-r', '0,1,2,3'], 'inside a replica'), (['-H', 'a,b,c,d,e'], 'automated scheduling')):
        proc = subprocess.run([sys.executable, os.path.join(mr.ROOT, 'runtime.py'), '0', '5', '--replicas', '2',
                               '-m', MODEL, '-pt', '1,24,25,48', '-d', 'cpu', *extra], cwd=str(tmp_path),
                              capture_output=True, text=True, timeout=300, env=dict(os.environ, **ENV))
        assert proc.returncode != 0
        assert 'ValueError' in proc.stderr and match in proc.stderr, proc.stderr[-2000:]
    proc = subprocess.run([sys.executable, os.path.join(mr.ROOT, 'runtime.py'), '0', '4', '--replicas', '2', '-m', MODEL,
                           '-pt', '1,24,25,48', '-d', 'cpu'], cwd=str(tmp_path), capture_output=True, text=True,
                          timeout=300, env=dict(os.environ, **ENV))
    assert proc.returncode != 0 and 'the world has 4' in proc.stderr, proc.stderr[-2000:]


class _Broadcast(Exception):
    pass


def _broadcast_of(monkeypatch, tmp_path, replicas, rank_order):
    """The tensors rank 0 of a world of 5 broadcasts with CMD_SCHED (the run stops right after)."""
    sent = []

    class FakeContext:
        def __init__(self, *_args):
            pass

        def __enter__(self):
            return self

        def __exit__(self, *_args):
            return False

        def cmd_broadcast(self, cmd, tensors=None):
            sent.append((cmd, tensors))
            raise _Broadcast

    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(rt, 'DistP2pContext', FakeContext)
    try:
        with pytest.raises(_Broadcast):
            rt.run_pipeline_p2p(5, 0, MODEL, None, 16, 8, PT, [8, 0], rank_order, 0, replicas=replicas)
    finally:
        monitoring.finish()
    assert len(sent) == 1 and sent[0][0] == rt.CMD_SCHED
    return sent[0][1]


def test_one_replica_broadcasts_exactly_the_schedule_of_today(monkeypatch, tmp_path):
    got = _broadcast_of(monkeypatch, tmp_path, 1, [1, 2])
    layers, quant, ranks = rt.get_pipeline_sched(5, PT, [8, 0], [1, 2], MODEL)
    want = (torch.tensor(layers), torch.tensor(quant), torch.tensor(ranks), torch.tensor(0))
    assert len(got) == 4
    for a, b in zip(got, want):
        assert a.dtype == b.dtype and torch.equal(a, b)
    assert got[2].shape == (2,)


def test_replicas_broadcast_the_stage_ranks_as_a_replica_by_stage_tensor(monkeypatch, tmp_path):
    got = _broadcast_of(monkeypatch, tmp_path, 2, [4, 3, 2, 1])
    assert len(got) == 4
    assert torch.equal(got[0], torch.tensor(PT)) and torch.equal(got[1], torch.tensor([8, 0]))
    assert torch.equal(got[2], torch.tensor([[4, 3], [2, 1]])) and int(got[3]) == 0
    # what a receiver's command handler makes of it (`handle_cmd`): one rank list per replica
    assert [t.tolist() for t in got][2] == [[4, 3], [2, 1]]


# ---------------------------------------------------------------------------------------------------- neighbours
def test_neighbours_of_every_rank_of_a_data_rank_and_three_replicas_of_two_stages():
    replicas = [[1, 2], [3, 4], [5, 6]]
    want = {1: (0, 0, 0, 2), 2: (0, 1, 1, 0), 3: (1, 0, 0, 4), 4: (1, 1, 3, 0), 5: (2, 0, 0, 6), 6: (2, 1, 5, 0)}
    for rank in range(8):
        got = model_cfg.replica_neighbours(replicas, 0, rank)
        assert got == want.get(rank, (None, None, None, None)), rank
    results = lambda _t: None   # noqa: E731
    data = model_cfg.dist_p2p_pipeline_stage_factory(replicas, 0, 0, None, None, results)
    assert data._args == ([2, 4, 6], [1, 3, 5], None, results)   # pylint: disable=protected-access
    assert data._replicas == [(2, 1), (4, 3), (6, 5)]            # pylint: disable=protected-access
    shard = object()
    for rank, (_, stage, src, dst) in want.items():
        ctx = model_cfg.dist_p2p_pipeline_stage_factory(replicas, 0, rank, stage, shard, None)
        assert ctx._args == (src, dst, shard, None), rank      # pylint: disable=protected-access
    idle = model_cfg.dist_p2p_pipeline_stage_factory(replicas, 0, 7, None, None, None)
    assert idle._args == (None, None, None, None)               # pylint: disable=protected-access
    with pytest.raises(ValueError):
        model_cfg.dist_p2p_pipeline_stage_factory(replicas, 0, 3, 1, shard, None)   # rank 3 is stage 0


def test_replica_lists_are_only_for_a_data_rank_outside_the_pipeline():
    with pytest.raises(ValueError, match='replica'):
        DistP2pPipelineStage([2, 4], [1, 3], object(), None)
    with pytest.raises(ValueError, match='replica'):
        DistP2pPipelineStage([2, 4], [1], None, lambda _t: None)
    stage = DistP2pPipelineStage([2, 4], [1, 3], None, lambda _t: None)
    with pytest.raises(RuntimeError, match='do not feed pipeline replicas'):
        stage.register_send_pre_hook(lambda: None, ())


# ---------------------------------------------------------------------------------------------------- fan-out / fan-in
@pytest.mark.parametrize('replicas,n', [(3, 7), (2, 8), (1, 5), (4, 3)])
def test_results_arrive_in_enqueue_order_whatever_order_replicas_finish_in(replicas, n):
    """Each replica returns its own micro-batches in order (a ring is FIFO), but the replicas interleave at random."""
    gen = torch.Generator().manual_seed(replicas * 100 + n)
    for _ in range(20):
        got = []
        order = InOrderResults(replicas, got.append)
        queues = [list(range(k, n, replicas)) for k in range(replicas)]
        while any(queues):
            live = [k for k in range(replicas) if queues[k]]
            k = live[int(torch.randint(len(live), (1,), generator=gen))]
            order.sink(k)(queues[k].pop(0))
        assert got == list(range(n)) and order.delivered == n and order.held == []


class _FakeFeeder:
    """Stands in for one replica's feeder: it answers each micro-batch on its own thread after `delay(replica)`."""
    delays = ()

    def __init__(self, rank_src, rank_dst, results_cb):
        self.replica = rank_dst // 2
        self.pairs = (rank_src, rank_dst)
        self._results_cb = results_cb
        self._q = []
        self._cond = threading.Condition()
        self._closed = False
        self._thread = threading.Thread(target=self._run, daemon=True)
        self.exception = None
        self.input_geometry = (64, torch.float32, 2)
        self.enqueued = []
        self.hooks = []
        self.released = False

    def hops(self):
        return [(0, self.pairs[1], 'send'), (self.pairs[0], 0, 'recv')]

    def open_hop(self, kind, connect_to, accept_from):
        (connect_to if kind == 'send' else accept_from)(self.pairs[1] if kind == 'send' else self.pairs[0])

    def start(self):
        self._thread.start()

    def add_send_timing_hook(self, hook, args):
        self.hooks.append((hook, args))

    def enqueue(self, tensor):
        with self._cond:
            self.enqueued.append(int(tensor[0]))
            self._q.append(tensor)
            self._cond.notify_all()

    def _run(self):
        while True:
            with self._cond:
                self._cond.wait_for(lambda: self._q or self._closed)
                if not self._q:
                    return
                tensor = self._q.pop(0)
            time.sleep(self.delays[self.replica])
            self._results_cb(tensor * 10)

    def check(self):
        if self.exception is not None:
            raise RuntimeError("fake feeder failed") from self.exception

    def drain(self, timeout=120.0):
        with self._cond:
            self._closed = True
            self._cond.notify_all()
        self._thread.join(timeout)

    def release(self):
        self.released = True


@pytest.mark.parametrize('replicas,n', [(3, 10), (2, 7)])
def test_replica_feeder_fans_out_round_robin_and_delivers_in_order_through_shutdown(replicas, n):
    """Replica 0 is the slowest, the last one the fastest; shutdown comes right after the last enqueue, with most
    results still in flight: every result arrives once, in enqueue order, before shutdown returns."""
    _FakeFeeder.delays = tuple(0.02 * (replicas - k) for k in range(replicas))
    got = []
    opened = []
    pairs = [(2 * k + 2, 2 * k + 1) for k in range(replicas)]   # (last stage, first stage) of replica k
    feeder = NativeReplicaFeeder(pairs, lambda t: got.append(int(t[0])), host=False, factory=_FakeFeeder)
    hook = lambda mbits, sec: None   # noqa: E731
    feeder.add_send_timing_hook(hook, ())
    feeder.init(lambda dst: opened.append(('to', dst)), lambda src: opened.append(('from', src)))
    # one global order over every hop of the data rank: (sender, receiver) ascending
    assert opened == [('to', 2 * k + 1) for k in range(replicas)] + [('from', 2 * k + 2) for k in range(replicas)]
    assert feeder.input_geometry == (64, torch.float32, 2)
    for i in range(n):
        feeder.enqueue(torch.tensor([i, 0]))
    feeder.shutdown()
    assert got == [10 * i for i in range(n)]
    assert feeder.delivered == n
    for k, fake in enumerate(feeder.feeders):
        assert fake.enqueued == list(range(k, n, replicas))
        assert fake.hooks == [(hook, ())] and fake.released


def test_replica_feeder_refuses_replicas_that_take_different_inputs():
    class Odd(_FakeFeeder):
        def __init__(self, rank_src, rank_dst, results_cb):
            super().__init__(rank_src, rank_dst, results_cb)
            if rank_dst == 3:
                self.input_geometry = (128, torch.float32, 2)

    _FakeFeeder.delays = (0, 0)
    feeder = NativeReplicaFeeder([(2, 1), (4, 3)], lambda t: None, host=False, factory=Odd)
    with pytest.raises(ValueError, match='different inputs'):
        feeder.init(lambda dst: None, lambda src: None)
    feeder.shutdown()


def test_a_full_replica_blocks_the_round_robin():
    """Replica 0 takes no micro-batch until released: the enqueue of micro-batch 2 (replica 0's turn again) waits
    although replica 1 has room, and micro-batch 3 is not fed before it."""
    gate = threading.Event()

    class Gated(_FakeFeeder):
        def enqueue(self, tensor):
            if self.replica == 0 and int(tensor[0]) > 0:
                gate.wait(10)
            super().enqueue(tensor)

    _FakeFeeder.delays = (0, 0)
    got = []
    feeder = NativeReplicaFeeder([(2, 1), (4, 3)], lambda t: got.append(int(t[0])), host=False, factory=Gated)
    feeder.init(lambda dst: None, lambda src: None)
    thr = threading.Thread(target=lambda: [feeder.enqueue(torch.tensor([i])) for i in range(4)])
    thr.start()
    time.sleep(0.3)
    assert feeder.feeders[0].enqueued == [0] and feeder.feeders[1].enqueued == [1]
    gate.set()
    thr.join(10)
    feeder.shutdown()
    assert got == [0, 10, 20, 30]


# ---------------------------------------------------------------------------------------------------- host data rank
N_ELEMS = 4
RING_SLOTS = 3


def _host_input(i, n):
    return torch.arange(mr.ragged(i, n, 3) * N_ELEMS, dtype=torch.float32).view(-1, N_ELEMS) + 100 * i


def _stand_in_stage(rank):
    """A one-stage replica without a GPU: it announces [items, 4] fp32 inputs, attaches to the data rank's rings like a
    first / last stage's links do, and answers each input x with 2x + 1 - slowly on rank 1, so that the replicas finish
    out of order."""
    from pipeedge_b200._lib import LIB, check
    from pipeedge_b200.comm.p2p import DistP2pContext
    from pipeedge_b200.comm.p2p._native import drain_barrier, max_ubatch, send_input_geometry
    import torch.distributed as dist
    # the vote: a capable stage with a GPU
    dist.all_reduce(torch.tensor([1, 0, -1], dtype=torch.int), op=dist.ReduceOp.MIN)
    ring_in, ring_res = ctypes.c_void_p(), ctypes.c_void_p()
    sock_in = DistP2pContext.accept_from(0)       # hop 0 -> rank (sender 0) first, as a stage opens them
    send_input_geometry(sock_in, max_ubatch() * N_ELEMS * 4, torch.float32, 2)
    check(LIB.pe_hostring_attach(sock_in.fileno(), 0, 0, 0, ctypes.byref(ring_in)))
    sock_res = DistP2pContext.connect_to(0)
    check(LIB.pe_hostring_attach(sock_res.fileno(), 1, max_ubatch() * N_ELEMS * 4, RING_SLOTS, ctypes.byref(ring_res)))
    ticket = (ctypes.c_longlong * 2)()
    data = ctypes.c_void_p()
    answered = 0
    while True:
        rc = LIB.pe_hostring_next(ring_in, ticket)
        if rc == 1:
            break
        check(rc)
        items = int(ticket[0])
        nbytes = items * N_ELEMS * 4
        check(LIB.pe_hostring_wait(ring_in, items, nbytes, ctypes.byref(data)))
        x = torch.frombuffer((ctypes.c_float * (items * N_ELEMS)).from_address(data.value), dtype=torch.float32).clone()
        check(LIB.pe_hostring_release(ring_in))
        if rank == 1:
            time.sleep(0.05)
        out = (2 * x + 1).contiguous()
        check(LIB.pe_hostring_publish(ring_res, out.data_ptr(), nbytes, items, N_ELEMS))
        answered += 1
    check(LIB.pe_hostring_close_input(ring_res))
    drain_barrier()
    LIB.pe_hostring_close(ring_in)
    LIB.pe_hostring_close(ring_res)
    sock_in.close()
    sock_res.close()
    return answered


def _host_replicas_worker(rank, world, n):
    from pipeedge_b200.comm.p2p import DistP2pContext
    out = {}
    with DistP2pContext(('gloo',), {'world_size': world, 'rank': rank}, lambda c, t: None):
        if rank > 0:
            out['answered'] = _stand_in_stage(rank)
        else:
            results, done = [], threading.Event()

            def results_cb(t):
                results.append(t.clone())
                if len(results) == n:
                    done.set()

            with model_cfg.dist_p2p_pipeline_stage_factory([[1], [2]], 0, 0, None, None, results_cb) as stage:
                out['kind'] = type(stage.native).__name__
                out['feeders'] = [type(f).__name__ for f in stage.native.feeders]
                for i in range(n):
                    stage.enqueue_tensor(_host_input(i, n))
                out['arrived'] = done.wait(120)
                stage.check_workers()
            out['results'] = [t.tolist() for t in results]   # plain data across the process boundary
            out['shm'] = [f for f in os.listdir('/dev/shm') if f.startswith(f"pipeedge_b200_{os.environ['MASTER_PORT']}_")]
            out['cuda_initialized'] = torch.cuda.is_initialized()
    return out


def test_host_data_rank_feeds_two_replicas_and_delivers_in_order():
    """A data rank without a GPU and two stand-in replicas in a Gloo world of 3: 7 micro-batches (not a multiple of 2,
    the last one short) go out round-robin through shared-memory rings; replica 0 answers slowly, yet every result
    arrives once, in enqueue order, and no segment is left behind."""
    n = 7
    got = mr.spawn(_host_replicas_worker, 3, (n,), env=ENV, get_timeout=240, join_timeout=60, hang_dump=200)
    data = got[0]
    assert data['kind'] == 'NativeReplicaFeeder' and data['feeders'] == ['NativeHostFeeder'] * 2
    assert data['arrived']
    assert got[1]['answered'] == 4 and got[2]['answered'] == 3
    assert len(data['results']) == n
    for i, res in enumerate(data['results']):
        assert res == (2 * _host_input(i, n) + 1).tolist(), i
    assert data['shm'] == [] and data['cuda_initialized'] is False


# ---------------------------------------------------------------------------------------------------- refusal
def _refusal_worker(rank, world):
    from pipeedge_b200.comm.p2p import DistP2pContext
    replicas = [[1], [2]]
    with DistP2pContext(('gloo',), {'world_size': world, 'rank': rank}, lambda c, t: None):
        stage = None if rank == 0 else 0
        shard = None if rank == 0 else object()
        try:
            with model_cfg.dist_p2p_pipeline_stage_factory(replicas, 0, rank, stage, shard, lambda _t: None):
                return 'ran'
        except RuntimeError as exc:
            return str(exc)


def test_every_rank_refuses_replicas_when_one_cannot_run_the_native_pipeline():
    """PIPEEDGE_NATIVE=0 with a data rank that feeds two replicas: the Python threads run one pipeline only, so every
    rank stops with the same error, which names each rank's reason; every process exits cleanly."""
    got = mr.spawn(_refusal_worker, 3, env=dict(ENV, PIPEEDGE_NATIVE='0'), get_timeout=120, join_timeout=60)
    assert got[0] == got[1] == got[2], got
    assert 'feeds pipeline replicas' in got[0]
    for rank in range(3):
        assert f"rank {rank}: PIPEEDGE_NATIVE=0" in got[0], got[0]
