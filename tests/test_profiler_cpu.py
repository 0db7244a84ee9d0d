"""CPU: the profiler's host side and the two converters that turn its results into the scheduler's YAML files.

The converters are checked byte for byte against what the reference's converters wrote from the same inputs, and the
shapes the profiler derives on the host against the reference's shard classes (`tests/golden/profiler.json.gz`,
`python -m oracle.profiler_goldens`)."""
import gzip
import json
import os
import subprocess
import sys
import numpy as np
import pytest
import yaml

import profiler
import runtime as rt
from pipeedge_b200.synth import MODEL_SPECS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden():
    with gzip.open(os.path.join(ROOT, 'tests', 'golden', 'profiler.json.gz'), 'rt', encoding='utf8') as f:
        return json.load(f)


@pytest.fixture(scope='module')
def golden():
    return _golden()


def _run(script, args, cwd, env=None):
    full_env = dict(os.environ, PYTHONPATH=ROOT, **(env or {}))
    return subprocess.run([sys.executable, os.path.join(ROOT, script)] + list(args), cwd=cwd, env=full_env,
                          capture_output=True, text=True, check=False, timeout=300)


@pytest.mark.parametrize('idx', range(len(_golden()['converters'])))
def test_converters_match_the_reference(golden, tmp_path, idx):
    """Every fixture case: new files, extended files, `-f`, refusals (existing entries, mem_MB / bw_Mbps mismatches,
    a missing -dtm / -dtb) and layer-count mismatches give the reference's exit code and file texts."""
    case = golden['converters'][idx]
    for name, text in case['files_before'].items():
        (tmp_path / name).write_text(text, encoding='utf-8')
    proc = _run(f"profiler_results_to_{case['tool']}.py", case['args'], tmp_path)
    assert proc.returncode == case['exit'], proc.stdout + proc.stderr
    for name, text in case['files_after'].items():
        path = tmp_path / name
        if text is None:
            assert not path.exists(), name
        else:
            assert path.read_bytes() == text.encode('utf-8'), name
    assert sorted(os.listdir(tmp_path)) == sorted(n for n, t in case['files_after'].items() if t is not None)


def test_fixture_covers_every_refusal(golden):
    """The golden cases exercise what the converters must refuse, so the byte-for-byte test above pins it."""
    stdout = '\n'.join(c['stdout'] for c in golden['converters'] if c['exit'] != 0)
    for msg in ('Model already exists', 'Model profile already exists', 'Mismatch for existing device type: bw_Mbps',
                'Mismatch for existing device type: mem_MB', 'must specify memory', 'must specify bandwidth',
                'Declared layer count does not match'):
        assert msg in stdout, msg
    assert any('Overwriting' in c['stdout'] and c['exit'] == 0 for c in golden['converters'])


@pytest.mark.parametrize('name', sorted(MODEL_SPECS))
def test_host_shapes_equal_the_reference(golden, name):
    spec = MODEL_SPECS[name]
    want = golden['shapes'][name]
    got = profiler.layer_shapes(spec, profiler.seq_len_from_shapes(spec, None, 1))
    assert golden['bert_tokens'] == profiler.BERT_TOKENS
    assert len(got) == len(want) == spec.layers
    for row, (shape_in, shape_out) in zip(want, got):
        assert (row['shape_in'], row['shape_out']) == (shape_in, shape_out), row['layer']


def test_recorded_dtype_is_what_runtime_passes_to_the_scheduler(monkeypatch):
    """`runtime.load_yaml_sched` runs `sched-pipeline -d <dtype>`; the scheduler looks profiles up by that dtype."""
    seen = {}

    def fake_run(args, **_):
        seen['args'] = args

        class Proc:   # pylint: disable=too-few-public-methods
            stdout = b"- '0': [1, 48]\n"
        return Proc()

    monkeypatch.setattr(subprocess, 'run', fake_run)
    rt.load_yaml_sched('textattack/bert-base-uncased-CoLA', 8, None, 'm.yml', 'd.yml', 'dev.yml')
    args = seen['args']
    assert args[args.index('-d') + 1] == profiler.DTYPE == 'torch.float32'
    for name in ('textattack/bert-base-uncased-CoLA', 'google/vit-base-patch16-224'):
        assert profiler.new_results(name, 8, 48)['dtype'] == 'torch.float32'


def _rows(intervals, start=1_000_000):
    """Stamp rows whose consecutive differences are `intervals` ([rows, cols - 1] ns)."""
    intervals = np.asarray(intervals, dtype=np.int64)
    return np.concatenate([np.full((intervals.shape[0], 1), start), start + np.cumsum(intervals, axis=1)], axis=1)


def test_layer_times_sum_to_the_plain_forward():
    rng = np.random.default_rng(3)
    intervals = rng.integers(2_000, 40_000, size=(50, 6))
    raw, times = profiler.layer_times(_rows(intervals), 6, False, 123e-6)
    assert np.allclose(raw, intervals.mean(axis=0))
    assert (times > 0).all()
    assert times.sum() == pytest.approx(123e-6, rel=1e-12)
    assert np.allclose(times / times.sum(), raw / raw.sum())


def test_layer_times_charge_the_head_to_the_last_layer():
    """A shard holding the model's last layer has one more column (after the head); its interval goes to the last
    layer, and the first interval (from before the embeddings) to the first."""
    intervals = np.array([[10, 20, 30, 5]] * 4)   # layers 46, 47, 48, then the head
    raw, times = profiler.layer_times(_rows(intervals), 3, True, 65e-9)
    assert raw.tolist() == [10, 20, 35]
    assert times == pytest.approx([10e-9, 20e-9, 35e-9])


@pytest.mark.parametrize('layer_start,layer_end,layers', [(1, 24, 48), (25, 48, 48), (7, 7, 12), (12, 12, 12)])
def test_layer_times_map_partial_ranges(layer_start, layer_end, layers):
    """Column k + 1 - column k is layer layer_start + k; rows that differ per layer keep their order."""
    n = layer_end - layer_start + 1
    last = layer_end == layers
    per_layer = np.array([1000 * layer for layer in range(layer_start, layer_end + 1)] + ([7] if last else []))
    raw, times = profiler.layer_times(_rows(np.tile(per_layer, (3, 1))), n, last, 1.0)
    want = per_layer[:n].astype(float)
    if last:
        want[-1] += 7
    assert raw.tolist() == want.tolist()
    assert times.sum() == pytest.approx(1.0)


def test_layer_times_refuse_bad_rows():
    with pytest.raises(ValueError):
        profiler.layer_times(np.zeros((2, 4)), 4, False, 1.0)
    with pytest.raises(profiler.ProfilerError):
        profiler.layer_times(_rows([[5, -1]]), 2, False, 1.0)


def test_results_checks():
    res = profiler.new_results('google/vit-base-patch16-224', 8, 48)
    res = profiler.merge_results(res, [{'layer': 3}, {'layer': 1}])
    assert [pd['layer'] for pd in res['profile_data']] == [1, 3]
    profiler.check_results(res, 'google/vit-base-patch16-224', 8, 48, 4, 48)
    for args in (('google/vit-large-patch16-224', 8, 48, 4, 4), ('google/vit-base-patch16-224', 2, 48, 4, 4),
                 ('google/vit-base-patch16-224', 8, 96, 4, 4), ('google/vit-base-patch16-224', 8, 48, 2, 3)):
        with pytest.raises(profiler.ProfilerError):
            profiler.check_results(res, *args)
    with pytest.raises(profiler.ProfilerError, match='dtype'):
        profiler.check_results(dict(res, dtype='torch.int64'), 'google/vit-base-patch16-224', 8, 48, 4, 4)


def test_shape_input_is_checked_against_the_model():
    vit, bert = MODEL_SPECS['google/vit-base-patch16-224'], MODEL_SPECS['bert-base-uncased']
    assert profiler.seq_len_from_shapes(vit, [[197, 768], [197, 768]], 2) == 128
    assert profiler.seq_len_from_shapes(bert, [[64]], 1) == 64
    assert profiler.seq_len_from_shapes(bert, [[64, 3072], [64, 768]], 4) == 64
    assert profiler.seq_len_from_shapes(bert, None, 5) == 128
    for spec, shapes, start in ((vit, [[197, 768]], 2), (vit, [[3, 224, 224]], 2), (bert, [[64, 768]], 4),
                                (bert, [[600]], 1)):
        with pytest.raises(profiler.ProfilerError):
            profiler.seq_len_from_shapes(spec, shapes, start)


@pytest.mark.parametrize('env,args', [({}, ['-d', 'cpu']), ({'CUDA_VISIBLE_DEVICES': ''}, [])])
def test_cli_without_a_gpu_fails_and_writes_nothing(tmp_path, env, args):
    proc = _run('profiler.py', ['-m', 'google/vit-base-patch16-224', '-b', '1', '-o', 'out.yml'] + args, tmp_path,
                env=env)
    assert proc.returncode != 0
    errors = [line for line in proc.stderr.splitlines() if 'error' in line.lower()]
    assert len(errors) == 1 and 'no CPU fallback' in errors[0], proc.stderr
    assert 'Traceback' not in proc.stderr
    assert os.listdir(tmp_path) == []


def test_cli_refuses_an_incompatible_results_file(tmp_path):
    existing = profiler.merge_results(profiler.new_results('google/vit-base-patch16-224', 8, 48),
                                      [{'layer': 5, 'shape_in': [[197, 768]], 'shape_out': [[197, 768]],
                                        'memory': 1.0, 'time': 1e-5}])
    profiler.save_results(existing, str(tmp_path / 'r.yml'))
    before = (tmp_path / 'r.yml').read_bytes()
    for extra in (['-l', '5', '-L', '5'], ['-b', '4']):
        proc = _run('profiler.py', ['-m', 'google/vit-base-patch16-224', '-o', 'r.yml', '-b', '8'] + extra, tmp_path)
        assert proc.returncode != 0 and 'error' in proc.stderr
        assert (tmp_path / 'r.yml').read_bytes() == before
    assert yaml.safe_load(before)['profile_data'][0]['layer'] == 5
