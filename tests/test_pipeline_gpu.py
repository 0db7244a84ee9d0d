"""GPU: real multi-rank pipelines through the reference-shaped API (DistP2pContext + DistP2pPipelineStage + shard +
QuantPipe hooks), one process per rank, checked bit for bit against the same shards and hooks run locally and against
the CPU oracle. The native pipeline (peer-memory links, `comm/p2p/_native.py`) also runs with every rank on ONE GPU
(cudaIpc between processes of the same device), so these tests do not need a multi-GPU box; the NCCL / Python-thread
path (`PIPEEDGE_NATIVE=0`) needs one GPU per rank and is skipped otherwise."""
import os
import sys
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _multirank as mr  # noqa: E402


def _inputs(name, n_ubatch, ubatch):
    from pipeedge_b200.synth import MODEL_SPECS, synth_input
    return [synth_input(MODEL_SPECS[name], mr.ragged(i, n_ubatch, ubatch), seed=10 + i, seq_len=32)
            for i in range(n_ubatch)]


def _worker(rank, world, name, cuts, qbits, n_ubatch, ubatch, native):
    import threading
    from pipeedge_b200.comm.p2p import DistP2pContext, DistP2pPipelineStage
    shard = mr.make_shard(name, cuts, rank, qbits[rank])
    shard.use_cuda_graph = True
    stop = threading.Event()
    results = []
    done = threading.Event()

    def results_cb(t):
        results.append(t.cpu())
        if len(results) == n_ubatch:
            done.set()

    with DistP2pContext(('gloo',), {'world_size': world, 'rank': rank}, lambda c, t: stop.set() if c == 0 else None) as ctx:
        src = world - 1 if rank == 0 else rank - 1
        dst = 0 if rank == world - 1 else rank + 1
        with DistP2pPipelineStage(src, dst, shard, results_cb if rank == 0 else None) as stage:
            assert (stage.native is not None) == native, "unexpected pipeline implementation"
            if rank == 0:
                # the last micro-batch is ragged (one item short): a second graph is captured mid-stream
                for x in _inputs(name, n_ubatch, ubatch):
                    stage.enqueue_tensor(x)
                assert done.wait(300), "results did not arrive"
                stage.check_workers()
                ctx.cmd_broadcast(0)
            else:
                assert stop.wait(420)
                stage.check_workers()
    return [r.numpy() for r in results] if rank == 0 else None


def _run_pipeline(name, cuts, qbits, n_ubatch, ubatch, native):
    # NCCL path: the ranks leave without the exit-time teardown of the CUDA / NCCL libraries (it can crash after a clean
    # shutdown). The native pipeline owns no communicator and exits normally.
    got = mr.spawn(_worker, len(cuts), (name, cuts, qbits, n_ubatch, ubatch, native),
                   env={'PIPEEDGE_NATIVE': '1' if native else '0'},
                   get_timeout=300,   # a fresh box pages torch in for a minute per process
                   hang_dump=240, hard_exit=not native)
    return got[0]


def _check_against_local_and_oracle(name, cuts, qbits, n_ubatch, ubatch, got):
    """Against the same shards + QuantPipe hooks run back to back in THIS process on cuda:0 (no communication)."""
    assert len(got) == n_ubatch
    inputs = _inputs(name, n_ubatch, ubatch)
    local = mr.run_local([mr.make_shard(name, cuts, s, qbits[s]) for s in range(len(cuts))], inputs)
    for i, (logits, want) in enumerate(zip(got, local)):
        np.testing.assert_array_equal(logits, want, err_msg=f"micro-batch {i}")
    if not any(qbits):
        mr.assert_within_oracle(name, got, inputs)


@pytest.mark.parametrize('name,cuts,qbits', [
    ('test/vit-tiny', (6, 12), (0, 0)),            # mid-block cut after an output projection: deferred residual add
    ('test/vit-tiny', (5, 12), (8, 0)),            # tuple payload (ctx, skip), both quantised by the fused send kernel
    ('test/bert-tiny', (7, 12), (4, 0)),           # tuple payload (inter, data) of a post-LN model, 4-bit
    ('test/deit-tiny', (4, 6, 8), (8, 6, 0)),      # three ranks (the model has 8 sub-layers): fused 8-bit, staged 6-bit hops
    ('test/vit-tiny', (2, 4, 6, 8, 10, 12), (0, 8, 0, 4, 0, 0)),   # six ranks, every rank a half block
])
def test_native_pipeline_is_bit_identical_to_local_shards(name, cuts, qbits):
    """Peer-memory links + one graph per stage: results arrive in FIFO order and are BIT-IDENTICAL to running the same
    shards and QuantPipe hooks locally (18 micro-batches through 4-slot rings: every slot is reused; the last one is
    ragged). Ranks share GPUs when the box has fewer GPUs than ranks."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    n_ubatch, ubatch = 18, 3
    got = _run_pipeline(name, cuts, qbits, n_ubatch, ubatch, native=True)
    _check_against_local_and_oracle(name, cuts, qbits, n_ubatch, ubatch, got)


def test_native_single_rank_stage_matches_direct_forward():
    """World of one: host-fed input ring -> one graph -> loop-back results link, against calling the shard directly."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import sys
    import threading
    sys.path.insert(0, ROOT)
    from pipeedge_b200.comm.p2p import DistP2pPipelineStage
    from pipeedge_b200.models import ModuleShardConfig
    from pipeedge_b200.models.transformers import bert
    from pipeedge_b200.synth import MODEL_SPECS, hf_config, synth_input, synth_weights
    spec = MODEL_SPECS['test/bert-tiny']
    cfg = ModuleShardConfig(layer_start=1, layer_end=spec.layers, is_first=True, is_last=True)
    weights = synth_weights(spec, seed=0)
    shard = bert.BertShardForSequenceClassification(hf_config(spec), cfg, weights)
    ref = bert.BertShardForSequenceClassification(hf_config(spec), cfg, weights)
    inputs = [synth_input(spec, 4 if i != 5 else 2, seed=30 + i, seq_len=32 if i < 8 else 48) for i in range(12)]
    got, done = [], threading.Event()

    def results_cb(t):
        got.append(t.clone())
        if len(got) == len(inputs):
            done.set()

    with DistP2pPipelineStage(None, None, shard, results_cb) as stage:
        assert stage.native is not None
        for x in inputs:
            stage.enqueue_tensor(x.pin_memory() if x.shape[0] == 4 else x.cuda())   # host and device sources
        assert done.wait(120)
        stage.check_workers()
    for x, y in zip(inputs, got):
        assert torch.equal(y, ref(x).cpu())


@pytest.mark.parametrize('name,cuts,qbits', [('test/vit-tiny', (6, 12), (0, 0)), ('test/vit-tiny', (5, 12), (8, 0)),
                                             ('test/bert-tiny', (7, 12), (4, 0))])
def test_two_stage_pipeline_over_nccl(name, cuts, qbits):
    """The generic path (Python exchange threads, NCCL hop; `PIPEEDGE_NATIVE=0`): FIFO and bit-identical to the local
    shards + hooks; the unquantised case is also checked against the CPU oracle."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("the NCCL hop needs one GPU per rank")
    n_ubatch, ubatch = 7, 3
    got = _run_pipeline(name, cuts, qbits, n_ubatch, ubatch, native=False)
    _check_against_local_and_oracle(name, cuts, qbits, n_ubatch, ubatch, got)


@pytest.mark.parametrize('policy', ['HEURISTIC', 'HEURISTIC2', 'CONTROLLER'])
def test_runtime_cli_adaptive_quant(policy, tmp_path):
    """`runtime.py` on 2 ranks with an adaptive QuantPipe policy and a send-rate constraint no hop can meet: the policy
    reads the hop's device-side transfer times and must move the stage's bit-width off 'no quantization', and the run
    must still deliver every result (`runtime.py:121-216,465-477` of the reference)."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    env = dict(os.environ, ADAPTIVE_QUANT=policy, SEND_CONSTRAINT='1e9', WINDOW_SIZE='2', PYTHONUNBUFFERED='1',
               MONITORING='1' if policy == 'CONTROLLER' else '0')   # one run also with the opt-in device-timed heartbeats
    rank0 = mr.run_runtime(tmp_path, 2, ['-q', '0,0'], env)[0]
    assert 'throughput is' in rank0, rank0[-3000:]
    import re
    bits = [int(b) for b in re.findall(r'Adaptive quantization \(\w+\): bitwidth1?=(\d+)', rank0)]
    assert bits, rank0[-3000:]
    assert any(0 < b < 32 for b in bits), bits
    if policy == 'CONTROLLER':
        for key in ('shard', 'quant_encode', 'output', 'send'):
            assert f'{key}: Global Time' in rank0, rank0[-3000:]
