"""GPU: the stage executor's sub-layer timestamps and the profiler built on them.

Stamps must not change what a stage computes or, once off again, which kernels it launches; the profiler's output must
have the reference's schema and shapes (`tests/golden/profiler.json.gz`), times that add up to the plain forward, and the
memory of a layer's weights as this build stores them."""
import gzip
import json
import os
import subprocess
import sys
import pytest
import torch
import yaml

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def golden(golden_dir):
    with gzip.open(os.path.join(golden_dir, 'profiler.json.gz'), 'rt', encoding='utf8') as f:
        return json.load(f)


def _stage(name, layer_start, layer_end, ubatch, tokens):
    from pipeedge_b200.models.transformers._stage import EncoderStage
    from pipeedge_b200.synth import MODEL_SPECS, hf_config, synth_weights
    spec = MODEL_SPECS[name]
    weights = synth_weights(spec, seed=0)
    if spec.family == 'bert':
        weights = {k[len('bert.'):]: v for k, v in weights.items() if k.startswith('bert.')}
    return EncoderStage(spec.family, hf_config(spec), layer_start, layer_end, weights, tokens, max_ubatch=ubatch)


def _inputs(stage, ubatch):
    gen = torch.Generator().manual_seed(5)
    width = stage.inter if stage.first_sub == 3 else stage.hidden
    x = torch.randn(ubatch, stage.tokens, width, generator=gen).cuda()
    if stage.in_is_tuple:
        return x, torch.randn(ubatch, stage.tokens, stage.hidden, generator=gen).cuda()
    return x


def _outs(stage, ubatch):
    s0, s1 = stage.out_shapes(ubatch)
    return (torch.full(s0, float('nan'), device='cuda'),
            None if s1 is None else torch.full(s1, float('nan'), device='cuda'))


def _as_tuple(res):
    return tuple(t.clone() for t in (res if isinstance(res, tuple) else (res,)))


def _same(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


CUTS = [
    ('test/vit-tiny', 5, 8, None),      # block boundaries
    ('test/vit-tiny', 2, 7, None),      # mid-block: (ctx, skip) in, (inter, skip) out
    ('test/vit-tiny', 4, 9, None),      # mid-block: (inter, skip) in, (ctx, skip) out
    ('test/bert-tiny', 3, 10, 40),      # post-LN
    ('test/vit-huge-tiny', 2, 7, None),  # head_dim 80: the fall-back attention kernel
]


@pytest.mark.parametrize('name,layer_start,layer_end,tokens', CUTS)
def test_stamps_leave_outputs_and_kernels_unchanged(name, layer_start, layer_end, tokens):
    from pipeedge_b200.synth import MODEL_SPECS
    ubatch = 3
    tokens = tokens or MODEL_SPECS[name].tokens
    plain = _stage(name, layer_start, layer_end, ubatch, tokens)
    stamped = _stage(name, layer_start, layer_end, ubatch, tokens)
    data = _inputs(plain, ubatch)
    n_sub = layer_end - layer_start + 1
    cols = n_sub + 1
    rows = 8
    stamps = torch.zeros((rows, cols), dtype=torch.int64, device='cuda')
    row_ctr = torch.zeros(1, dtype=torch.int64, device='cuda')

    out = _outs(plain, ubatch)
    want_eager = _as_tuple(plain.forward(data, out=out))
    count_eager = plain.kernel_count()
    want_graph = []
    for _ in range(3):   # warm-up eager, capture, replay
        want_graph.append(_as_tuple(plain.forward(data, out=out, use_graph=True)))
    count_graph = plain.kernel_count()
    assert all(_same(w, want_eager) for w in want_graph)

    out_s = _outs(stamped, ubatch)
    stamped.forward(data, out=out_s, use_graph=True)   # a graph captured WITHOUT stamps for these pointers
    stamped.forward(data, out=out_s, use_graph=True)
    stamped.set_stamps(stamps, row_ctr, col0=1)
    stamped.stamp(stamps, row_ctr, 0)
    assert _same(_as_tuple(stamped.forward(data, out=out_s)), want_eager)
    assert stamped.kernel_count() == count_eager + n_sub
    for _ in range(3):   # the unstamped graph is not replayed: a stamped one is captured and replayed
        stamped.stamp(stamps, row_ctr, 0)
        assert _same(_as_tuple(stamped.forward(data, out=out_s, use_graph=True)), want_eager)
    torch.cuda.synchronize()
    assert int(row_ctr.item()) == 4
    got = stamps.cpu()
    assert (got[:4] > 0).all() and (got[4:] == 0).all()
    assert (got[:4, 1:] >= got[:4, :-1]).all(), got

    stamped.set_stamps(None)
    for _ in range(2):   # the graph captured before stamps were on is replayed again
        assert _same(_as_tuple(stamped.forward(data, out=out_s, use_graph=True)), want_eager)
    assert stamped.kernel_count() == count_graph
    assert _same(_as_tuple(stamped.forward(data, out=out_s)), want_eager)
    assert stamped.kernel_count() == count_eager
    torch.cuda.synchronize()
    assert int(row_ctr.item()) == 4, "a graph captured with stamps ran after they were turned off"
    plain.close()
    stamped.close()


def test_replays_fill_one_row_each():
    """K back-to-back replays of one stamped graph fill exactly K rows; replays past the table's rows are counted."""
    from pipeedge_b200.synth import MODEL_SPECS
    stage = _stage('test/vit-tiny', 1, 12, 2, MODEL_SPECS['test/vit-tiny'].tokens)
    data = _inputs(stage, 2)
    out = _outs(stage, 2)
    k = 9
    stamps = torch.zeros((k, 13), dtype=torch.int64, device='cuda')
    row_ctr = torch.zeros(1, dtype=torch.int64, device='cuda')
    stage.forward(data, out=out, use_graph=True)   # warm-up without stamps
    stage.set_stamps(stamps, row_ctr, col0=1)
    stage.forward(data, out=out, use_graph=True)   # eager first use of the stamped key
    stage.forward(data, out=out, use_graph=True)   # capture + launch
    torch.cuda.synchronize()
    row_ctr.zero_()
    stamps.zero_()
    for _ in range(k + 3):
        stage.forward(data, out=out, use_graph=True)
    torch.cuda.synchronize()
    assert int(row_ctr.item()) == k + 3
    got = stamps.cpu()[:, 1:]
    assert (got > 0).all() and (got[:, 1:] >= got[:, :-1]).all()
    stage.close()


def _param_bytes(hidden, inter, sub):
    """Parameter bytes of one ViT sub-layer: 2 per matrix element (fp16), 4 per vector element (fp32)."""
    return {0: 2 * 3 * hidden * hidden + 4 * (3 * hidden + 2 * hidden),
            1: 2 * hidden * hidden + 4 * hidden,
            2: 2 * inter * hidden + 4 * (inter + 2 * hidden),
            3: 2 * hidden * inter + 4 * hidden}[sub]


def _converters_accept(tmp_path, path):
    for script, args in (('profiler_results_to_models.py', ['-i', path, '-o', str(tmp_path / 'models.yml')]),
                         ('profiler_results_to_device_types.py', ['H100', '-i', path, '-o',
                                                                  str(tmp_path / 'dt.yml'), '-dtm', '81559',
                                                                  '-dtb', '3600000'])):
        proc = subprocess.run([sys.executable, os.path.join(ROOT, script)] + args, cwd=tmp_path, capture_output=True,
                              text=True, check=False, timeout=300, env=dict(os.environ, PYTHONPATH=ROOT))
        assert proc.returncode == 0, proc.stdout + proc.stderr


@pytest.mark.parametrize('name,batch', [('test/vit-tiny', 2), ('test/deit-tiny', 2), ('test/bert-tiny', 2),
                                        ('test/vit-huge-tiny', 2), ('google/vit-base-patch16-224', 2)])
def test_profile(golden, tmp_path, name, batch):
    import profiler
    from pipeedge_b200.synth import MODEL_SPECS
    spec = MODEL_SPECS[name]
    prof = profiler.profile_layers(name, batch, iterations=50)
    data = prof['profile_data']
    assert [pd['layer'] for pd in data] == list(range(1, spec.layers + 1))
    for pd, want in zip(data, golden['shapes'][name]):
        assert set(pd) == {'layer', 'shape_in', 'shape_out', 'memory', 'time'}
        assert (pd['shape_in'], pd['shape_out']) == (want['shape_in'], want['shape_out'])
        assert pd['time'] > 0 and pd['memory'] > 0
    assert sum(pd['time'] for pd in data) == pytest.approx(prof['plain_s'], rel=1e-9)
    assert prof['stamped_s'] > 0
    if name == 'google/vit-base-patch16-224':
        for layer in range(21, 25):   # block 6 of 12
            want = _param_bytes(spec.hidden, spec.inter, (layer - 1) % 4) / 1e6
            assert data[layer - 1]['memory'] == pytest.approx(want, abs=1e-9), layer
    results = profiler.merge_results(profiler.new_results(name, batch, spec.layers), data)
    path = str(tmp_path / 'r.yml')
    profiler.save_results(results, path)
    with open(path, encoding='utf-8') as f:
        loaded = yaml.safe_load(f)
    assert set(loaded) == {'model_name', 'dtype', 'batch_size', 'layers', 'profile_data'}
    assert loaded['dtype'] == 'torch.float32' and loaded['batch_size'] == batch
    _converters_accept(tmp_path, path)


def test_cli_extends_a_results_file(tmp_path):
    import profiler
    common = ['-m', 'google/vit-base-patch16-224', '-b', '2', '-i', '20']
    split, whole = str(tmp_path / 'split.yml'), str(tmp_path / 'whole.yml')
    assert profiler.main(common + ['-o', split, '-L', '24']) == 0
    assert profiler.main(common + ['-o', split, '-l', '25', '-s', '197,768']) == 0
    assert profiler.main(common + ['-o', whole]) == 0
    with open(split, encoding='utf-8') as f:
        got = yaml.safe_load(f)
    with open(whole, encoding='utf-8') as f:
        want = yaml.safe_load(f)
    assert [(pd['layer'], pd['shape_in'], pd['shape_out'], pd['memory']) for pd in got['profile_data']] == \
        [(pd['layer'], pd['shape_in'], pd['shape_out'], pd['memory']) for pd in want['profile_data']]
    assert {k: v for k, v in got.items() if k != 'profile_data'} == {k: v for k, v in want.items() if k != 'profile_data'}
    before = open(split, 'rb').read()
    assert profiler.main(common + ['-o', split, '-l', '25', '-L', '30', '-s', '197,768']) == 1
    assert open(split, 'rb').read() == before
