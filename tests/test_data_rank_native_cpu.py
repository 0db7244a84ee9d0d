"""CPU: the native pipeline's vote for a data rank outside the stage pipeline (the feeder role), and the input
geometry the first stage announces to it over their hop's socket."""
import socket
import pytest
import torch

from pipeedge_b200.comm.p2p import DistP2pPipelineStage
from pipeedge_b200.comm.p2p import _native


def _capable(monkeypatch, args, native='1', hooked=False):
    stage = DistP2pPipelineStage(*args)   # (built first: its threads ask a CUDA runtime for the device when it claims one)
    if hooked:
        stage.register_send_pre_hook(lambda: None, ())
    with monkeypatch.context() as m:
        m.setattr(torch.cuda, 'is_available', lambda: True)
        m.setenv('PIPEEDGE_NATIVE', native)
        return stage._native_capable()   # pylint: disable=protected-access


def test_the_feeder_role_votes_native(monkeypatch):
    """No worker, a results callback and both ranks set (what `model_cfg.dist_p2p_pipeline_stage_factory` builds for a
    data rank outside the pipeline): native, unless PIPEEDGE_NATIVE=0. A relay without a results callback, or a feeder
    missing one of its ranks, is not; idle ranks stay neutral."""
    results = lambda _t: None   # noqa: E731
    assert _capable(monkeypatch, (2, 1, None, results))
    assert _capable(monkeypatch, (1, 1, None, results))          # a single stage: both hops go to the data rank
    assert not _capable(monkeypatch, (2, 1, None, results), native='0')
    assert not _capable(monkeypatch, (2, 1, None, None))         # a relay that collects nothing
    assert not _capable(monkeypatch, (None, 1, None, results))
    assert not _capable(monkeypatch, (2, None, None, results))
    assert _capable(monkeypatch, (None, None, None, None))        # idle rank
    assert not _capable(monkeypatch, (None, None, None, None), native='0')


def test_a_feeder_with_exchange_hooks_takes_the_thread_path(monkeypatch):
    """User pre / post hooks run on the Python exchange threads: as for every other role, they rule the feeder out."""
    assert not _capable(monkeypatch, (2, 1, None, lambda _t: None), hooked=True)


@pytest.mark.parametrize('nbytes,dtype,ndim', [
    (64 * 3 * 224 * 224 * 4, torch.float32, 4),    # images
    (64 * 512 * 8, torch.int64, 2),                # BERT token ids
])
def test_input_geometry_round_trips(nbytes, dtype, ndim):
    a, b = socket.socketpair()
    try:
        _native.send_input_geometry(a, nbytes, dtype, ndim)
        assert _native.recv_input_geometry(b) == (nbytes, dtype, ndim)
    finally:
        a.close()
        b.close()


def test_input_geometry_of_a_first_stage_shard(monkeypatch):
    """What the first stage announces: PIPEEDGE_MAX_UBATCH items of its longest sequence, in its input dtype."""
    monkeypatch.setenv('PIPEEDGE_MAX_UBATCH', '8')

    class Shard:
        def native_max_tokens(self):
            return 32

        def native_input_spec(self, ubatch, dim1):
            return [((ubatch, dim1), torch.int64)]

    assert _native.max_input_geometry(Shard()) == (8 * 32 * 8, torch.int64, 2)


def test_malformed_or_missing_geometry_is_refused():
    a, b = socket.socketpair()
    try:
        a.sendall(b'\0' * _native._GEOMETRY.size)   # pylint: disable=protected-access
        with pytest.raises(ConnectionError, match='malformed'):
            _native.recv_input_geometry(b)
        a.close()
        with pytest.raises(ConnectionError, match='closed'):
            _native.recv_input_geometry(b)
    finally:
        a.close()
        b.close()
    with pytest.raises(ValueError, match='cannot be announced'):
        _native.send_input_geometry(None, 8, torch.complex64, 1)
