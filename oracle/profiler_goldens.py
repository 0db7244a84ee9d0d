"""Generate `tests/golden/profiler.json.gz` by executing the REFERENCE itself - TEST INFRASTRUCTURE.

`PIPEEDGE_REFERENCE=<checkout> python -m oracle.profiler_goldens` (see `oracle/make_goldens.py`). Stores:
* `shapes`: per-layer `shape_in` / `shape_out` of the reference's shard classes, one layer at a time on CPU as its
  `profile_layers_individually` chains them (batch 1, BERT at 128 tokens), for every registry and test model;
* `converters`: the files, exit codes and messages of the reference's `profiler_results_to_models.py` /
  `profiler_results_to_device_types.py` on fixed profiler results (new and extended files, `-f`, refusals).
"""
import gzip
import json
import os
import subprocess
import sys
import tempfile
import torch
import yaml
from oracle.make_goldens import OUT, REF_ROOT, REF_SRC, _ref
from pipeedge_b200.synth import MODEL_SPECS, hf_config, synth_input, synth_weights


def _shapes(tensors):
    """The reference profiler's `get_shapes`: one shape per tensor of the payload, without the batch dimension."""
    return [list(t.shape[1:]) for t in (tensors if isinstance(tensors, tuple) else (tensors,))]


def layer_shapes(name):
    sys.path.insert(0, REF_SRC)
    from pipeedge.models.transformers import bert   # pylint: disable=import-outside-toplevel,import-error
    shard_config_cls, classes, _, _ = _ref()
    spec = MODEL_SPECS[name]
    cls = classes[spec.family] if spec.family != 'bert' or spec.classify else bert.BertModelShard
    weights = synth_weights(spec, seed=0)
    data = synth_input(spec, 1, seed=1, seq_len=128)
    rows = []
    with torch.no_grad():
        for layer in range(1, spec.layers + 1):
            cfg = shard_config_cls(layer_start=layer, layer_end=layer, is_first=layer == 1, is_last=layer == spec.layers)
            shard = cls(hf_config(spec), cfg, weights)
            shard.eval()
            out = shard(data)
            rows.append({'layer': layer, 'shape_in': _shapes(data), 'shape_out': _shapes(out)})
            data = out
    return rows


def _results(model, layers, batch_size, n_data=None, scale=1.0):
    """A fixed `profiler_results.yml` text (made-up numbers)."""
    data = [{'layer': l, 'shape_in': [[197, 768]] if l > 1 else [[3, 224, 224]],
             'shape_out': [[197, 768], [197, 768]] if l % 4 == 1 else [[197, 768]],
             'memory': round(0.25 * l + 1.5, 6), 'time': scale * (1e-5 + 1.25e-6 * (l % 5))}
            for l in range(1, (layers if n_data is None else n_data) + 1)]
    return yaml.safe_dump({'model_name': model, 'dtype': 'torch.float32', 'batch_size': batch_size, 'layers': layers,
                           'profile_data': data}, default_flow_style=None)


CASES = [   # (tool, args, index of the case whose resulting files this one starts from, results files to add)
    ('models', ['-i', 'a.yml', '-o', 'models.yml'], None, ('a',)),
    ('models', ['-i', 'b.yml', '-o', 'models.yml'], 0, ('b',)),
    ('models', ['-i', 'a.yml', '-o', 'models.yml'], 1, ()),
    ('models', ['-i', 'c.yml', '-o', 'models.yml', '-f'], 1, ('c',)),
    ('models', ['-i', 'short.yml', '-o', 'models.yml'], None, ('short',)),
    ('models', ['-i', 'unknown.yml', '-o', 'models.yml'], None, ('unknown',)),
    ('device_types', ['H100', '-i', 'a.yml', '-o', 'dt.yml', '-dtm', '81559', '-dtb', '3600000'], None, ('a',)),
    ('device_types', ['H100', '-i', 'b.yml', '-o', 'dt.yml'], 6, ('b',)),
    ('device_types', ['H100', '-i', 'd.yml', '-o', 'dt.yml'], 7, ('d',)),
    ('device_types', ['H100', '-i', 'a.yml', '-o', 'dt.yml'], 7, ()),
    ('device_types', ['H100', '-i', 'c.yml', '-o', 'dt.yml', '-f'], 7, ('c',)),
    ('device_types', ['H100', '-i', 'd.yml', '-o', 'dt.yml', '-dtb', '1000'], 7, ('d',)),
    ('device_types', ['H100', '-i', 'd.yml', '-o', 'dt.yml', '-dtm', '1000'], 7, ('d',)),
    ('device_types', ['H100', '-i', 'd.yml', '-o', 'dt.yml', '-dtm', '81559', '-dtb', '3600000'], 7, ('d',)),
    ('device_types', ['A100', '-i', 'a.yml', '-o', 'dt.yml', '-dtm', '40000'], 7, ()),
    ('device_types', ['A100', '-i', 'a.yml', '-o', 'dt.yml', '-dtb', '2000'], None, ('a',)),
    ('device_types', ['A100', '-i', 'a.yml', '-o', 'dt.yml', '-dtm', '40000', '-dtb', '2000'], 7, ()),
    ('device_types', ['H100', '-i', 'short.yml', '-o', 'dt.yml'], 7, ('short',)),
]


def converter_cases():
    results = {'a': _results('google/vit-base-patch16-224', 48, 8),
               'b': _results('textattack/bert-base-uncased-CoLA', 48, 32, scale=3.0),
               'c': _results('google/vit-base-patch16-224', 48, 8, scale=2.0),
               'd': _results('google/vit-base-patch16-224', 48, 16, scale=1.5),
               'short': _results('google/vit-base-patch16-224', 48, 8, n_data=47),
               'unknown': _results('test/vit-tiny', 12, 2)}
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([REF_SRC, REF_ROOT]))
    cases = []
    for tool, args, start, adds in CASES:
        files = {k: v for k, v in (cases[start]['files_after'] if start is not None else {}).items() if v is not None}
        files.update({f"{name}.yml": results[name] for name in adds})
        with tempfile.TemporaryDirectory() as tmp:
            for name, text in files.items():
                with open(os.path.join(tmp, name), 'w', encoding='utf-8') as f:
                    f.write(text)
            proc = subprocess.run([sys.executable, os.path.join(REF_ROOT, f"profiler_results_to_{tool}.py")] + args,
                                  cwd=tmp, env=env, capture_output=True, text=True, check=False)
            after = {}
            for name in sorted(set(os.listdir(tmp)) | set(files)):
                path = os.path.join(tmp, name)
                after[name] = open(path, encoding='utf-8').read() if os.path.exists(path) else None
        cases.append({'tool': tool, 'args': args, 'files_before': files, 'exit': proc.returncode,
                      'stdout': proc.stdout, 'files_after': after})
    return cases


def main():
    if not os.path.isdir(os.path.join(REF_SRC, 'pipeedge')):
        raise SystemExit("set PIPEEDGE_REFERENCE to a checkout of the reference (it must contain src/pipeedge)")
    shapes = {name: layer_shapes(name) for name in sorted(MODEL_SPECS)}
    out = {'batch_size': 1, 'bert_tokens': 128, 'shapes': shapes, 'converters': converter_cases()}
    with gzip.GzipFile(os.path.join(OUT, 'profiler.json.gz'), 'wb', mtime=0) as f:
        f.write(json.dumps(out).encode('utf-8'))


if __name__ == '__main__':
    main()
