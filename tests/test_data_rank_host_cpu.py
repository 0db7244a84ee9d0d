"""CPU: a rank without a CUDA device (`runtime.py -d cpu`, or no visible GPU) - what the CLI lets it do, and how the
native pipeline's vote selects the host feeder for a data rank outside the stage pipeline, or refuses a world whose
stages cannot serve it."""
import os
import pytest
import torch
import torch.distributed as dist

import devices
import runtime as rt
from pipeedge_b200.comm.p2p import DistP2pPipelineStage


def test_init_env_records_a_host_only_rank(monkeypatch):
    """`-d cpu` hides every GPU from the process and makes the CPU its device; so does having no visible GPU. Neither
    raises."""
    monkeypatch.setattr(devices, 'DEVICE', None)
    for var in ('CUDA_VISIBLE_DEVICES', 'MASTER_ADDR', 'MASTER_PORT'):
        monkeypatch.setenv(var, 'unset')
    rt.init_env('cpu', '127.0.0.1', 29999, '')
    assert devices.DEVICE == torch.device('cpu')
    assert os.environ['CUDA_VISIBLE_DEVICES'] == ''
    monkeypatch.setenv('CUDA_VISIBLE_DEVICES', 'unset')
    monkeypatch.setattr(devices, 'DEVICE', None)
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: False)
    rt.init_env(None, '127.0.0.1', 29999, '')
    assert devices.DEVICE == torch.device('cpu')
    assert os.environ['CUDA_VISIBLE_DEVICES'] == 'unset'


def test_a_host_only_rank_may_not_own_a_stage(monkeypatch):
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: False)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        rt.check_host_only_role(0)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        rt.check_host_only_role(2)
    rt.check_host_only_role(None)   # a data rank outside the stage pipeline, or an idle rank


def _vote(monkeypatch, args, others, native='1'):
    """_choose_native() on a rank without a CUDA device in a world of 3, whose other ranks vote `others` (each
    [capable, -(host feeder), -(has a GPU)]): (this rank's vote, the outcome or the exception)."""
    stage = DistP2pPipelineStage(*args)
    sent = []

    def all_reduce(tensor, op):
        assert op == dist.ReduceOp.MIN
        sent.append(tensor.tolist())
        for other in others:
            tensor.copy_(torch.minimum(tensor, torch.tensor(other, dtype=tensor.dtype)))

    monkeypatch.setattr(torch.cuda, 'is_available', lambda: False)
    monkeypatch.setenv('PIPEEDGE_NATIVE', native)
    monkeypatch.setattr(dist, 'is_initialized', lambda: True)
    monkeypatch.setattr(dist, 'get_world_size', lambda: 3)
    monkeypatch.setattr(dist, 'all_reduce', all_reduce)
    try:
        outcome = stage._choose_native()   # pylint: disable=protected-access
    except RuntimeError as exc:
        outcome = exc
    monkeypatch.undo()
    return sent, outcome, stage


STAGES_NATIVE = [[1, 0, -1], [1, 0, -1]]     # two stage ranks with a GPU, both native-capable
STAGES_THREADS = [[0, 0, -1], [1, 0, -1]]    # ... one of them not (PIPEEDGE_NATIVE=0 or exchange hooks)


def test_the_host_only_data_rank_takes_part_in_the_vote(monkeypatch):
    """A data rank without a GPU outside the stage pipeline votes (it used to return before the all_reduce, leaving the
    other ranks waiting in it): capable, as a host feeder. The world then runs natively and this rank is a
    NativeHostFeeder."""
    results = lambda _t: None   # noqa: E731
    sent, outcome, stage = _vote(monkeypatch, (2, 1, None, results), STAGES_NATIVE)
    assert sent == [[1, -1, 0]]
    assert outcome is True
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: False)
    assert stage._host_feeder()   # pylint: disable=protected-access  (init() builds a NativeHostFeeder)


def test_a_host_only_idle_rank_is_neutral_and_a_host_only_stage_is_not_capable(monkeypatch):
    sent, outcome, _ = _vote(monkeypatch, (None, None, None, None), STAGES_NATIVE)
    assert sent == [[1, 0, 0]] and outcome is True
    sent, outcome, _ = _vote(monkeypatch, (2, 1, object(), None), STAGES_NATIVE)
    assert sent == [[0, 0, 0]] and outcome is False


@pytest.mark.parametrize('native,others', [('0', [[0, 0, -1], [0, 0, -1]]), ('1', STAGES_THREADS)])
def test_the_thread_path_refuses_a_host_only_data_rank_on_every_rank(monkeypatch, native, others):
    """PIPEEDGE_NATIVE=0, or a stage that cannot run natively: the Python threads carry CUDA payloads over NCCL and
    cannot serve a data rank without a GPU - the vote raises one clear error on that rank, and on the stages (which see
    the same reduced vote) instead of hanging."""
    results = lambda _t: None   # noqa: E731
    sent, outcome, _ = _vote(monkeypatch, (2, 1, None, results), others, native=native)
    assert sent == [[0 if native == '0' else 1, -1, 0]]
    assert isinstance(outcome, RuntimeError) and 'no CUDA device' in str(outcome)
    # a stage rank with a GPU receives the same reduced vote
    stage = DistP2pPipelineStage(0, 2, None, None)
    monkeypatch.setattr(stage, '_native_capable', lambda: native == '1')
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: True)
    monkeypatch.setattr(dist, 'is_initialized', lambda: True)
    monkeypatch.setattr(dist, 'get_world_size', lambda: 3)
    monkeypatch.setattr(dist, 'all_reduce', lambda t, op: t.copy_(torch.tensor([0, -1, -1], dtype=t.dtype)))
    with pytest.raises(RuntimeError, match='no CUDA device'):
        stage._choose_native()   # pylint: disable=protected-access


def test_a_world_without_any_gpu_keeps_the_thread_path(monkeypatch):
    """Every rank without a GPU (the Gloo path): a data rank outside the pipeline is not refused, the threads run."""
    results = lambda _t: None   # noqa: E731
    sent, outcome, _ = _vote(monkeypatch, (2, 1, None, results), [[0, 0, 0], [0, 0, 0]])
    assert sent == [[1, -1, 0]] and outcome is False
