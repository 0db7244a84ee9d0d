"""Generate `tests/golden/*.npz` by executing the REFERENCE itself - TEST INFRASTRUCTURE.

Run where a checkout of the reference (usc-isi/PipeEdge) exists:
`PIPEEDGE_REFERENCE=<checkout> python -m oracle.make_goldens`. Imports `<checkout>/src/pipeedge` read-only, runs
the reference's shard classes and quantisation functions on seeded synthetic inputs, and stores the outputs. The
tests only read the fixtures, never the reference.

Fixture contents
----------------
* `shards_<model>.npz` for the tiny test models: the complete value after EVERY sub-layer boundary
  (tuples stored as `_0`/`_1`), the embeddings and the final logits, ubatch 2.
* `shards_<registry model>.npz` for ViT-B, DeiT-B and BERT-base-CoLA at full size: logits plus a
  strided sample of the hidden state after sub-layers 2, 24 and 48 (full tensors would be ~MBs).
* `quant.npz`: `tensor_encode_outerdim` outputs and `tensor_decode_outerdim` round trips for
  several bit widths, plus the two runtime hooks' clamp thresholds (restated in this script
  without the `monitoring` calls - `runtime.py` itself cannot be imported here, SURVEY.md 8c).
* `quant_bits.npz` (`python -m oracle.make_goldens quant_bits`): the same for the bit-widths `quant.npz` leaves out
  (1, 7, 9, 11, 12, 13, 14, 15) on normal, outlier, rounding-tie and every-code inputs, through the reference's
  `basic_op` and `clamp_op` only (no constant items: the reference asserts on them).
* `adaptive.json` (`python -m oracle.make_goldens adaptive`): outputs of the reference's adaptive-QuantPipe policy
  code (`<checkout>/utils/{quant,controller}.py`): `constrain_max_bitwidth` over a grid, Kalman-filter and
  bit-width-controller traces for fixed measurement sequences.
"""
import os
import sys
import numpy as np
import torch

REF_ROOT = os.environ.get('PIPEEDGE_REFERENCE', '')   # a checkout of the reference
REF_SRC = os.path.join(REF_ROOT, 'src')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'tests', 'golden')
SAMPLE_STRIDE = 97   # prime, so the sample walks across rows and columns

sys.path.insert(0, ROOT)
from pipeedge_b200.synth import MODEL_SPECS, hf_config, synth_input, synth_weights  # noqa: E402


def _ref():
    sys.path.insert(0, REF_SRC)
    # pylint: disable=import-outside-toplevel,import-error
    from pipeedge.models import ModuleShardConfig
    from pipeedge.models.transformers import bert, deit, vit
    from pipeedge.quantization import basic_op, clamp_op
    return ModuleShardConfig, {'vit': vit.ViTShardForImageClassification,
                               'deit': deit.DeiTShardForImageClassification,
                               'bert': bert.BertShardForSequenceClassification}, basic_op, clamp_op


def ref_shard(spec, weights, layer_start, layer_end):
    """Instantiate the reference shard class exactly as `model_cfg.module_shard_factory` does."""
    shard_config_cls, classes, _, _ = _ref()
    cfg = shard_config_cls(layer_start=layer_start, layer_end=layer_end,
                           is_first=layer_start == 1, is_last=layer_end == spec.layers)
    shard = classes[spec.family](hf_config(spec), cfg, weights)
    shard.eval()   # deviation: the reference leaves BERT dropout live (SURVEY.md section 0)
    return shard


def _store(out, key, val):
    if isinstance(val, tuple):
        for i, t in enumerate(val):
            out[f"{key}_{i}"] = t.numpy()
    else:
        out[key] = val.numpy()


def golden_tiny(name, ubatch=2, seq_len=24):
    spec = MODEL_SPECS[name]
    weights = synth_weights(spec, seed=0)
    x = synth_input(spec, ubatch, seed=1, seq_len=seq_len)
    out = {'input': x.numpy()}
    data = x
    with torch.no_grad():
        for layer in range(1, spec.layers + 1):
            # one reference shard per sub-layer: its output IS the boundary payload
            data = ref_shard(spec, weights, layer, layer)(data)
            _store(out, f"after_{layer}", data)
        out['logits_whole'] = ref_shard(spec, weights, 1, spec.layers)(x).numpy()
    np.savez_compressed(os.path.join(OUT, f"shards_{name.replace('/', '_')}.npz"), **out)
    print(name, 'done')


def golden_full(name, ubatch, cuts, seq_len=128):
    spec = MODEL_SPECS[name]
    weights = synth_weights(spec, seed=0)
    x = synth_input(spec, ubatch, seed=1, seq_len=seq_len)
    out = {'ubatch': np.int64(ubatch), 'seq_len': np.int64(seq_len), 'cuts': np.array(cuts),
           'stride': np.int64(SAMPLE_STRIDE)}
    data = x
    start = 1
    with torch.no_grad():
        for cut in cuts:
            data = ref_shard(spec, weights, start, cut)(data)
            start = cut + 1
            if cut == spec.layers:
                out['logits'] = data.numpy()
            else:
                out[f"after_{cut}_sample"] = data.numpy().reshape(-1)[::SAMPLE_STRIDE].copy()
                out[f"after_{cut}_norm"] = np.float64(data.double().norm().item())
    np.savez_compressed(os.path.join(OUT, f"shards_{name.replace('/', '_')}.npz"), **out)
    print(name, 'done')


def golden_quant():
    _, _, basic_op, clamp_op = _ref()
    out = {}
    gen = torch.Generator().manual_seed(7)
    shapes = {'a': (3, 17, 128), 'b': (2, 5, 77), 'c': (1, 33, 64)}
    for tag, shape in shapes.items():
        x = torch.randn(*shape, generator=gen) * 1.7 + 0.3
        out[f"x_{tag}"] = x.numpy()
        for bit in (2, 3, 4, 5, 6, 8, 10, 16):
            # encode hook restated (runtime.py:83-86)
            clamp = clamp_op.clamp_banner2019_laplace if x.min() < 0.2 else clamp_op.clamp_banner2019_gelu
            xc = clamp(x, bit)
            out[f"alpha_{tag}_{bit}"] = np.float32(xc.abs().max().item())   # == alpha when clamping bites
            enc = basic_op.tensor_encode_outerdim(xc, bit)
            for nm, t in zip(('comm', 'shape', 'scale', 'shift', 'bit'), enc):
                out[f"{nm}_{tag}_{bit}"] = t.numpy()
            out[f"dec_{tag}_{bit}"] = basic_op.tensor_decode_outerdim(enc).numpy()
    # GeLU-clamp branch: all values >= 0.2
    x = torch.rand(2, 9, 64, generator=gen) * 3 + 0.25
    out['x_g'] = x.numpy()
    for bit in (4, 8):
        xc = clamp_op.clamp_banner2019_gelu(x, bit)
        out[f"alpha_g_{bit}"] = np.float32(xc.abs().max().item())
        enc = basic_op.tensor_encode_outerdim(xc, bit)
        for nm, t in zip(('comm', 'shape', 'scale', 'shift', 'bit'), enc):
            out[f"{nm}_g_{bit}"] = t.numpy()
        out[f"dec_g_{bit}"] = basic_op.tensor_decode_outerdim(enc).numpy()
    # bit 0 passthrough
    enc = basic_op.tensor_encode_outerdim(x, 0)
    for nm, t in zip(('comm', 'shape', 'scale', 'shift', 'bit'), enc):
        out[f"{nm}_g_0"] = t.numpy()
    np.savez_compressed(os.path.join(OUT, "quant.npz"), **out)
    print('quant done')


QUANT_BITS = (1, 7, 9, 11, 12, 13, 14, 15)


def golden_quant_bits():
    """Stored per bit b and input kind k: x_k_b, alpha_k_b (the clamp's threshold), comm / shape / scale / shift /
    bit_k_b and dec_k_b, as `golden_quant`."""
    _, _, basic_op, clamp_op = _ref()
    out = {}
    gen = torch.Generator().manual_seed(17)
    for bit in QUANT_BITS:
        lv = (1 << bit) - 1
        xs = {'normal': torch.randn(3, 7, 41, generator=gen) * 1.3 + 0.1,
              'outliers': torch.randn(4, 300, generator=gen) * 1.3 + 0.1}
        xs['outliers'][0, :3] = torch.tensor([40.0, -35.0, 12.0])
        # ties: values v with lv * fp32(v / S) == k + 1/2 in fp32 (S = lv), the rest of the item spanning [0, S]; the
        # second item (+-100 S) keeps the Laplace threshold above S
        s = np.float32(lv)
        ties = [np.float32(0.0), s] + [np.float32(k + 0.5) for k in range(min(lv, 300))
                                      if float(np.float32(lv) * np.float32(np.float32(k + 0.5) / s)) == k + 0.5]
        ramp = np.arange(lv + 1, dtype=np.float32)
        for kind, vals in (('ties', ties), ('ramp', ramp)):
            vals = np.asarray(vals, dtype=np.float32)
            perm = torch.randperm(len(vals), generator=gen).numpy()
            guard = np.resize(np.array([-100 * s, 100 * s], np.float32), len(vals))
            xs[kind] = torch.from_numpy(np.stack([vals[perm], guard]))
        for kind, x in xs.items():
            key = f"{kind}_{bit}"
            out[f"x_{key}"] = x.numpy()
            clamp = clamp_op.clamp_banner2019_laplace if x.min() < 0.2 else clamp_op.clamp_banner2019_gelu
            xc = clamp(x, bit)
            out[f"alpha_{key}"] = np.float32(xc.abs().max().item())
            enc = basic_op.tensor_encode_outerdim(xc, bit)
            for nm, t in zip(('comm', 'shape', 'scale', 'shift', 'bit'), enc):
                out[f"{nm}_{key}"] = t.numpy()
            out[f"dec_{key}"] = basic_op.tensor_decode_outerdim(enc).numpy()
    np.savez_compressed(os.path.join(OUT, "quant_bits.npz"), **out)
    print('quant_bits done')


def _ref_utils():
    """The reference's top-level `utils` package, imported under another name (this repo has its own `utils`)."""
    import importlib.util   # pylint: disable=import-outside-toplevel
    sys.path.insert(0, REF_SRC)   # `utils/quant.py` imports pipeedge.quantization.basic_op
    pkg_dir = os.path.join(REF_ROOT, 'utils')
    spec = importlib.util.spec_from_file_location('ref_utils', os.path.join(pkg_dir, '__init__.py'),
                                                  submodule_search_locations=[pkg_dir])
    pkg = importlib.util.module_from_spec(spec)
    sys.modules['ref_utils'] = pkg
    spec.loader.exec_module(pkg)
    import ref_utils.controller as ref_controller   # pylint: disable=import-outside-toplevel,import-error
    import ref_utils.quant as ref_quant             # pylint: disable=import-outside-toplevel,import-error
    return ref_quant, ref_controller


def golden_adaptive():
    """Adaptive QuantPipe policy code of the reference on fixed inputs -> tests/golden/adaptive.json."""
    import json   # pylint: disable=import-outside-toplevel
    ref_quant, ref_controller = _ref_utils()
    out = {}
    grid = []
    for t_max in (0.0, 0.001, 0.004, 0.01, 0.05, 1.0, float('inf')):
        for d_size in (0.0, 4.84, 38.7, 154.9):            # Mbits of a payload
            for d_speed in (0.0, 10.0, 1000.0, 25000.0):   # Mbit/s
                for bw_max in (32, 16):
                    try:
                        got = int(ref_quant.constrain_max_bitwidth(torch.tensor(t_max), torch.tensor(d_size),
                                                                   torch.tensor(d_speed), torch.tensor(bw_max)))
                    except IndexError:   # 0/0 or inf*0: NaN compares false everywhere, the reference indexes []
                        got = -1
                    grid.append([t_max, d_size, d_speed, bw_max, got])
    out['constrain_max_bitwidth'] = grid
    rng = np.random.default_rng(5)
    kalman = []
    for x0, p0 in ((0.0, 1.0), (3.0, 0.5)):
        filt = ref_controller.KalmanFilter(x_hat_0=x0, p_0=p0)
        zs = (10.0 + rng.normal(0, 0.5, 20)).tolist()
        hs = (1.0 + rng.uniform(0, 2, 20)).tolist()
        kalman.append({'x0': x0, 'p0': p0, 'z': zs, 'h': hs, 'x_hat': [float(filt(z, h)) for z, h in zip(zs, hs)]})
    out['kalman'] = kalman
    xup = []
    for ref_value, u0, umax, pole in ((100.0, 1.0, 16.0, 0.0), (40.0, 2.0, 8.0, 0.5), (7.5, 1.0, float('inf'), 0.9)):
        ctl = ref_controller.AdaptiveIntegralXupController(ref_value, u0, u_max=umax, pole=pole)
        ys = (ref_value * rng.uniform(0.3, 1.6, 25)).tolist()
        xup.append({'reference': ref_value, 'u_0': u0, 'u_max': umax, 'pole': pole, 'y': ys,
                    'u': [float(ctl(y)) for y in ys]})
    out['xup'] = xup
    basic_op = _ref()[2]
    bitwidths = [i for i in range(32, 1, -1)
                 if int(basic_op.compression_factor(i)) > int(basic_op.compression_factor(i + 1))]
    out['bitwidths'] = bitwidths
    traces = []
    for constraint, start, window in ((100.0, 32, 10), (2500.0, 8, 10), (30.0, 2, 7), (0.0, 32, 10)):
        ctl = ref_quant.AdaptiveBitwidthPerformanceController(0, bitwidths, start)
        ctl.reference = constraint
        perf = (max(constraint, 10.0) * rng.uniform(0.2, 2.0, 30)).tolist()
        traces.append({'constraint': constraint, 'start': start, 'window': window, 'perf': perf,
                       'out': [list(map(int, ctl(p, window))) for p in perf]})
    out['bitwidth_controller'] = traces
    with open(os.path.join(OUT, 'adaptive.json'), 'w', encoding='utf8') as f:
        json.dump(out, f)
    print('adaptive done')


def golden_sched():
    """The reference's `parse_yaml_sched` (`runtime.py:260-288`; the script itself cannot be imported here, so the
    function is extracted from its source) on scheduler-format YAML -> tests/golden/sched.json."""
    import ast    # pylint: disable=import-outside-toplevel
    import json   # pylint: disable=import-outside-toplevel
    import logging   # pylint: disable=import-outside-toplevel
    import yaml   # pylint: disable=import-outside-toplevel
    with open(os.path.join(REF_ROOT, 'runtime.py'), encoding='utf8') as f:
        tree = ast.parse(f.read())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == 'parse_yaml_sched')
    from typing import List, Optional, Tuple   # pylint: disable=import-outside-toplevel
    scope = {'List': List, 'Optional': Optional, 'Tuple': Tuple, 'logger': logging.getLogger('ref')}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), 'ref_runtime', 'exec'), scope)   # pylint: disable=exec-used
    ref = scope['parse_yaml_sched']
    cases = [
        ("- mb-a: [1, 24]\n- mb-b: [25, 48]\n", ['mb-a', 'mb-b']),
        ("- mb-b: [1, 10]\n- mb-a: [11, 48]\n", ['mb-a', 'mb-b']),
        ("- '1': [1, 6]\n- '0': [7, 30]\n- '2': [31, 48]\n", None),
        ("- 3: [1, 96]\n", None),
        ("- gpu0: [1, 6]\n- gpu1: [7, 12]\n- gpu2: [13, 18]\n- gpu3: [19, 24]\n- gpu4: [25, 30]\n- gpu5: [31, 36]\n"
         "- gpu6: [37, 42]\n- gpu7: [43, 48]\n", [f'gpu{i}' for i in range(8)]),
        ("- nosuch: [1, 48]\n", ['mb-a']),
        ("- notarank: [1, 48]\n", None),
        ("[]\n", None),
    ]
    out = []
    for text, hosts in cases:
        sched = yaml.safe_load(text)
        try:
            layers, ranks = ref(sched, hosts)
            out.append({'yaml': text, 'hosts': hosts, 'layers': [list(l) for l in layers], 'ranks': ranks})
        except (ValueError, RuntimeError) as exc:
            out.append({'yaml': text, 'hosts': hosts, 'error': type(exc).__name__})
    with open(os.path.join(OUT, 'sched.json'), 'w', encoding='utf8') as f:
        json.dump(out, f, indent=1)
    print('sched done')


def main():
    if not os.path.isdir(os.path.join(REF_SRC, 'pipeedge')):
        raise SystemExit("set PIPEEDGE_REFERENCE to a checkout of the reference (it must contain src/pipeedge)")
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(8)
    if sys.argv[1:] == ['adaptive']:
        golden_adaptive()
        return
    if sys.argv[1:2] == ['tiny']:
        for name in sys.argv[2:]:
            golden_tiny(name)
        return
    if sys.argv[1:] == ['sched']:
        golden_sched()
        return
    if sys.argv[1:] == ['quant_bits']:
        golden_quant_bits()
        return
    if sys.argv[1:] == ['vit-large']:
        golden_full('google/vit-large-patch16-224', 2, (24, 48, 72, 96))
        return
    golden_adaptive()
    golden_sched()
    golden_quant()
    golden_quant_bits()
    for name in ('test/vit-tiny', 'test/deit-tiny', 'test/bert-tiny', 'test/vit-huge-tiny'):
        golden_tiny(name)
    golden_full('google/vit-base-patch16-224', 2, (2, 24, 48))
    golden_full('facebook/deit-base-distilled-patch16-224', 2, (6, 24, 48))
    golden_full('textattack/bert-base-uncased-CoLA', 2, (6, 24, 48), seq_len=128)
    golden_full('google/vit-large-patch16-224', 2, (24, 48, 72, 96))    # BASELINE config 3's model and 4-way cuts


if __name__ == '__main__':
    main()
