"""Sub-layer profiler: the scheduler's `profiler_results.yml` for this build's kernels on an H100.

Same command line and schema as the reference's `profiler.py`; like it, it extends an existing results file after
checking model, dtype, batch size and layer count, and refuses layers the file already holds. Times come from device
timestamps inside a CUDA graph of the whole `[-l, -L]` shard (`-i` replays, default 200, because a sub-layer takes
5-40 us), scaled so that the layers sum to the unstamped forward. Memory is the growth of
`torch.cuda.memory_allocated()` while one layer's shard is built (its weights, without the stage's workspace), and
`dtype` is `torch.float32` for every model. DESIGN.md section 7 gives the method and its deviations from the reference.
There is no CPU fallback: `-d cpu`, or a process without a CUDA sm_90 device, stops with one error and writes nothing.
"""
import argparse
import gc
import logging
import os
import subprocess
import sys
from typing import Callable, List, Optional, Sequence, Tuple
import numpy as np
import torch
import yaml
from pipeedge_b200.synth import MODEL_SPECS, ModelSpec, hf_config, synth_input, synth_weights

logger = logging.getLogger(__name__)

DTYPE = 'torch.float32'        # every hop's dtype; runtime.load_yaml_sched passes the same to sched-pipeline
DEFAULT_ITERATIONS = 200       # graph replays per timing (sub-layers are microseconds long)
WARMUP_REPLAYS = 20
BERT_TOKENS = 128


class ProfilerError(RuntimeError):
    """A profile that cannot be taken (no GPU, bad arguments, an incompatible results file)."""


# ------------------------------------------------------------------------------------------------ shapes
def layer_shapes(spec: ModelSpec, seq_len: int = BERT_TOKENS) -> List[Tuple[list, list]]:
    """(shape_in, shape_out) of every sub-layer 1..layers, per item as the reference's profiler records them: one shape
    per tensor of the payload, a `(data, skip)` tuple at a mid-block cut (SURVEY.md 8a-A2)."""
    tokens = seq_len if spec.family == 'bert' else spec.tokens
    hid, inter = [tokens, spec.hidden], [tokens, spec.inter]
    first = [[seq_len]] if spec.family == 'bert' else [[spec.channels, spec.image_size, spec.image_size]]
    last = [[spec.num_labels]] if spec.classify else [[spec.hidden]]   # classifier logits / BERT pooler
    out = []
    shape_in = first
    for layer in range(1, spec.layers + 1):
        if layer == spec.layers:
            shape_out = last
        else:
            shape_out = {0: [hid, hid], 1: [hid], 2: [inter, hid], 3: [hid]}[(layer - 1) % 4]
        out.append((shape_in, shape_out))
        shape_in = shape_out
    return out


def seq_len_from_shapes(spec: ModelSpec, shapes: Optional[Sequence[Sequence[int]]], layer_start: int) -> int:
    """BERT's sequence length stated by `-s` (the first dimension of the first shape), else the default (128, or the
    model's longest); checks that the shapes are the model's input shapes at `layer_start`."""
    seq_len = min(BERT_TOKENS, spec.max_pos)
    if shapes and spec.family == 'bert':
        seq_len = int(shapes[0][0])
        if not 1 <= seq_len <= spec.max_pos:
            raise ProfilerError(f"sequence length {seq_len} is outside [1, {spec.max_pos}] for {spec.name}")
    if shapes:
        want = layer_shapes(spec, seq_len)[layer_start - 1][0]
        if [list(s) for s in shapes] != want:
            raise ProfilerError(f"-s {shapes} is not the input of layer {layer_start} of {spec.name}: {want}")
    return seq_len


# ------------------------------------------------------------------------------------------------ time arithmetic
def layer_times(stamps: np.ndarray, n_layers: int, includes_last: bool, plain_s: float) -> Tuple[np.ndarray, np.ndarray]:
    """Per-layer (raw ns, seconds) from stamp rows of a stamped shard of `n_layers` sub-layers.

    Row columns: 0 before the shard (before the embeddings of layer 1), 1..n after each sub-layer, and, when the
    shard holds the model's last layer, n + 1 after the head, which is charged to the last layer. Seconds are the raw
    means scaled so that they sum to `plain_s`, the unstamped forward's time."""
    stamps = np.asarray(stamps, dtype=np.int64)
    cols = n_layers + 1 + (1 if includes_last else 0)
    if stamps.ndim != 2 or stamps.shape[1] != cols or stamps.shape[0] < 1:
        raise ValueError(f"stamps must be [rows, {cols}], got {stamps.shape}")
    intervals = np.diff(stamps, axis=1).astype(np.float64)
    if (intervals < 0).any():
        raise ProfilerError("device timestamps decrease within a forward")
    raw = intervals[:, :n_layers].mean(axis=0)
    if includes_last:
        raw[-1] += intervals[:, n_layers].mean()
    total = raw.sum()
    if total <= 0:
        raise ProfilerError("stamped forward took no time")
    return raw, raw * (plain_s / total)


# ------------------------------------------------------------------------------------------------ device
def require_gpu(device: Optional[str]) -> torch.device:
    """The CUDA sm_90 device to profile on; ProfilerError for `cpu` or when the process sees none."""
    if device is not None and torch.device(device).type != 'cuda':
        raise ProfilerError(f"device {device!r}: the profiler times this build's sm_90a kernels and needs a CUDA "
                            "device (there is no CPU fallback)")
    if not torch.cuda.is_available():
        raise ProfilerError("no CUDA device: the profiler needs an H100 (sm_90a); there is no CPU fallback")
    dev = torch.device(device if device is not None else 'cuda')
    if dev.index is None:
        dev = torch.device('cuda', torch.cuda.current_device())
    if torch.cuda.get_device_capability(dev) != (9, 0):
        raise ProfilerError(f"{torch.cuda.get_device_name(dev)} is not an sm_90 device")
    return dev


def device_description(dev: torch.device) -> str:
    """Card name and power limit (read-only `nvidia-smi` query), e.g. 'NVIDIA H100 80GB HBM3, power limit 700.00 W'."""
    name = torch.cuda.get_device_name(dev)
    limit = 'unknown'
    try:
        uuid = str(torch.cuda.get_device_properties(dev).uuid)
        proc = subprocess.run(['nvidia-smi', '--query-gpu=uuid,power.limit', '--format=csv,noheader,nounits'],
                              capture_output=True, text=True, timeout=30, check=True)
        for line in proc.stdout.splitlines():
            fields = [f.strip() for f in line.split(',')]
            if len(fields) == 2 and fields[0].lower().endswith(uuid.lower()):
                limit = f"{fields[1]} W"
    except (OSError, subprocess.SubprocessError, AttributeError):
        pass
    return f"{name}, power limit {limit}"


# ------------------------------------------------------------------------------------------------ shards
def _shard_class(spec: ModelSpec):
    # pylint: disable=import-outside-toplevel
    from pipeedge_b200.models.transformers import bert, deit, vit
    if spec.family == 'bert':
        return bert.BertShardForSequenceClassification if spec.classify else bert.BertModelShard
    return {'vit': vit.ViTShardForImageClassification, 'deit': deit.DeiTShardForImageClassification}[spec.family]


def make_shard(spec: ModelSpec, weights, layer_start: int, layer_end: int):
    """The shard of `[layer_start, layer_end]` on the current device, as `model_cfg.module_shard_factory` builds it."""
    from pipeedge_b200.models import ModuleShardConfig   # pylint: disable=import-outside-toplevel
    cfg = ModuleShardConfig(layer_start=layer_start, layer_end=layer_end, is_first=layer_start == 1,
                            is_last=layer_end == spec.layers)
    return _shard_class(spec)(hf_config(spec), cfg, weights)


def load_weights(spec: ModelSpec, model_file: Optional[str]):
    """`runtime.py`'s rule: the npz file if it exists, else seeded synthetic weights in the same layout."""
    if model_file and os.path.exists(model_file):
        with np.load(model_file) as npz:
            return dict(npz)
    logger.warning("weights file %s not found: using seeded synthetic weights", model_file)
    return synth_weights(spec, seed=0)


def shard_inputs(spec: ModelSpec, batch_size: int, layer_start: int, seq_len: int, dev: torch.device):
    """Seeded inputs of layer `layer_start`: images / token ids for layer 1, fp32 boundary payloads otherwise."""
    if layer_start == 1:
        return synth_input(spec, batch_size, seed=1, seq_len=seq_len).to(dev)
    gen = torch.Generator().manual_seed(1)
    shapes = layer_shapes(spec, seq_len)[layer_start - 1][0]
    data = tuple(torch.randn(batch_size, *s, generator=gen).to(dev) for s in shapes)
    return data[0] if len(data) == 1 else data


def layer_memory_mb(spec: ModelSpec, weights, layer: int) -> float:
    """MB (10^6 bytes) of device memory the shard of `layer` alone allocates through torch: its weights and edge
    tables. The stage workspace is cudaMalloc'd by the library and not counted."""
    gc.collect()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    shard = make_shard(spec, weights, layer, layer)
    torch.cuda.synchronize()
    grown = torch.cuda.memory_allocated() - before
    shard.stage.close()
    del shard
    gc.collect()
    return grown / 1e6


def time_graphs(forwards: Sequence[Callable[[], object]], iterations: int, warmup: bool,
                before_timing: Sequence[Optional[Callable[[], None]]]) -> List[float]:
    """Capture each forward into a CUDA graph, then per graph: (warm-up replays,) `before_timing`, `iterations`
    back-to-back replays between two CUDA events. Returns seconds per forward."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graphs = []
    with torch.cuda.stream(side):
        for fwd in forwards:
            fwd()   # eager first run: one-time kernel attributes, BERT's workspace for this sequence length
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=side, capture_error_mode='thread_local'):
                fwd()
            graphs.append(graph)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    out = []
    for graph, prepare in zip(graphs, before_timing):
        if warmup:
            for _ in range(WARMUP_REPLAYS):
                graph.replay()
        if prepare is not None:
            prepare()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(iterations):
            graph.replay()
        end.record()
        end.synchronize()
        out.append(start.elapsed_time(end) / 1e3 / iterations)
    return out


def time_shard(shard, inputs, n_layers: int, includes_last: bool, iterations: int, warmup: bool) -> dict:
    """Plain and stamped graph times of one forward of `shard` and the stamp rows of the stamped replays:
    {'plain_s', 'stamped_s', 'stamps' [iterations, cols] ns}."""
    from pipeedge_b200.models.transformers._stage import EncoderStage   # pylint: disable=import-outside-toplevel
    dev = shard.stage.device
    cols = n_layers + 1 + (1 if includes_last else 0)
    stamps = torch.zeros((iterations, cols), dtype=torch.int64, device=dev)
    row_ctr = torch.zeros(1, dtype=torch.int64, device=dev)

    def plain():
        return shard(inputs)

    def stamped():
        shard.stage.set_stamps(stamps, row_ctr, col0=1)
        try:
            EncoderStage.stamp(stamps, row_ctr, 0)
            out = shard(inputs)
            if includes_last:
                EncoderStage.stamp(stamps, row_ctr, cols - 1, bump_row=True)
            return out
        finally:
            shard.stage.set_stamps(None)

    def reset():
        stamps.zero_()
        row_ctr.zero_()

    plain_s, stamped_s = time_graphs([plain, stamped], iterations, warmup, [None, reset])
    rows = int(row_ctr.item())
    if rows != iterations:
        raise ProfilerError(f"{iterations} stamped replays filled {rows} rows")
    return {'plain_s': plain_s, 'stamped_s': stamped_s, 'stamps': stamps.cpu().numpy()}


def profile_layers(model_name: str, batch_size: int, layer_start: int = 1, layer_end: Optional[int] = None,
                   weights=None, shapes_in: Optional[Sequence[Sequence[int]]] = None, warmup: bool = True,
                   iterations: int = DEFAULT_ITERATIONS, device: Optional[str] = None) -> dict:
    """Profile sub-layers `[layer_start, layer_end]` of `model_name` (a `pipeedge_b200.synth.MODEL_SPECS` name) on the
    GPU. Returns {'profile_data': [{layer, shape_in, shape_out, memory, time}], 'plain_s', 'stamped_s', 'device'}.
    `weights`: a loaded npz mapping (default: seeded synthetic weights); `shapes_in`: the `-s` shapes."""
    if model_name not in MODEL_SPECS:
        raise ProfilerError(f"unknown model {model_name}")
    spec = MODEL_SPECS[model_name]
    layer_end = spec.layers if layer_end is None else layer_end
    if not 1 <= layer_start <= layer_end <= spec.layers:
        raise ProfilerError(f"layers [{layer_start}, {layer_end}] are not within [1, {spec.layers}]")
    if batch_size < 1 or iterations < 1:
        raise ProfilerError("batch size and iterations must be positive")
    seq_len = seq_len_from_shapes(spec, shapes_in, layer_start)
    dev = require_gpu(device)
    torch.cuda.set_device(dev)
    described = device_description(dev)
    logger.info("Profiling %s layers [%d, %d] at batch %d on %s", model_name, layer_start, layer_end, batch_size,
                described)
    if weights is None:
        weights = synth_weights(spec, seed=0)
    memory = [layer_memory_mb(spec, weights, layer) for layer in range(layer_start, layer_end + 1)]
    shard = make_shard(spec, weights, layer_start, layer_end)
    n_layers = layer_end - layer_start + 1
    inputs = shard_inputs(spec, batch_size, layer_start, seq_len, dev)
    with torch.no_grad():
        timed = time_shard(shard, inputs, n_layers, layer_end == spec.layers, iterations, warmup)
    shard.stage.close()
    _, times = layer_times(timed['stamps'], n_layers, layer_end == spec.layers, timed['plain_s'])
    shapes = layer_shapes(spec, seq_len)
    # fresh lists per entry: YAML would write shared ones as anchors and aliases
    data = [{'layer': layer, 'shape_in': [list(s) for s in shapes[layer - 1][0]],
             'shape_out': [list(s) for s in shapes[layer - 1][1]],
             'memory': memory[i], 'time': float(times[i])}
            for i, layer in enumerate(range(layer_start, layer_end + 1))]
    logger.info("Plain forward %.3f us, stamped %.3f us: stamps cost x%.4f", timed['plain_s'] * 1e6,
                timed['stamped_s'] * 1e6, timed['stamped_s'] / timed['plain_s'])
    return {'profile_data': data, 'plain_s': timed['plain_s'], 'stamped_s': timed['stamped_s'], 'device': described}


# ------------------------------------------------------------------------------------------------ results file
def new_results(model_name: str, batch_size: int, layers: int) -> dict:
    """An empty results file's content."""
    return {'model_name': model_name, 'dtype': DTYPE, 'batch_size': batch_size, 'layers': layers, 'profile_data': []}


def check_results(results: dict, model_name: str, batch_size: int, layers: int, layer_start: int,
                  layer_end: int) -> None:
    """ProfilerError unless an existing results file can be extended by these layers."""
    checks = (('model name', results.get('model_name'), model_name), ('dtype', results.get('dtype'), DTYPE),
              ('batch size', results.get('batch_size'), batch_size), ('layer count', results.get('layers'), layers))
    for what, have, want in checks:
        if have != want:
            raise ProfilerError(f"{what} mismatch with existing results: {have} != {want}")
    done = sorted({pd['layer'] for pd in results.get('profile_data') or []} & set(range(layer_start, layer_end + 1)))
    if done:
        raise ProfilerError(f"layers {done} are already in the existing results")


def merge_results(results: dict, data: List[dict]) -> dict:
    """`results` with `data` added, sorted by layer."""
    results['profile_data'] = sorted(list(results.get('profile_data') or []) + data, key=lambda pd: pd['layer'])
    return results


def save_results(results: dict, path: str) -> None:
    with open(path, 'w', encoding='utf-8') as yfile:
        yaml.safe_dump(results, yfile, default_flow_style=None)


def main(argv: Optional[List[str]] = None) -> int:
    """Main function."""
    import model_cfg   # pylint: disable=import-outside-toplevel
    parser = argparse.ArgumentParser(description="Module Shard Profiler (in-context sub-layer times on an H100)",
                                     formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("-o", "--results-yml", default="profiler_results.yml", type=str, help="output YAML file")
    parser.add_argument("-d", "--device", type=str, default=None,
                        help="CUDA device, e.g. 'cuda' or 'cuda:1' (there is no CPU fallback); default: the current one")
    parser.add_argument("-m", "--model-name", type=str, default="google/vit-base-patch16-224",
                        choices=model_cfg.get_model_names(), help="the neural network model for loading")
    parser.add_argument("-M", "--model-file", type=str,
                        help="the model file, if not in working directory (seeded synthetic weights if it is missing)")
    parser.add_argument("-l", "--layer-start", default=1, type=int, help="start layer")
    parser.add_argument("-L", "--layer-end", type=int, help="end layer; default: last layer in the model")
    parser.add_argument("-s", "--shape-input", type=str, action='append',
                        help="comma-delimited input shape without the batch dimension, once per tensor, e.g. "
                             "'197,768'; for BERT '128' at layer 1 sets the sequence length (default 128); "
                             "checked against the model")
    parser.add_argument("-b", "--batch-size", default=8, type=int, help="batch size")
    parser.add_argument("-w", "--warmup", action="store_true", default=True,
                        help=f"replay each graph {WARMUP_REPLAYS} times before timing it")
    parser.add_argument("--no-warmup", action="store_false", dest="warmup", help="don't replay before timing")
    parser.add_argument("-i", "--iterations", default=DEFAULT_ITERATIONS, type=int,
                        help="graph replays to average each layer's time over")
    args = parser.parse_args(argv)
    logging.basicConfig(level=logging.INFO, format="%(message)s")
    try:
        shapes = None
        if args.shape_input:
            try:
                shapes = [[int(d) for d in shp.split(',')] for shp in args.shape_input]
            except ValueError as exc:
                raise ProfilerError(f"-s {args.shape_input}: {exc}") from exc
        layers = model_cfg.get_model_layers(args.model_name)
        layer_end = layers if args.layer_end is None else args.layer_end
        if os.path.exists(args.results_yml):
            logger.info("Using existing results file")
            with open(args.results_yml, 'r', encoding='utf-8') as yfile:
                results = yaml.safe_load(yfile)
            check_results(results, args.model_name, args.batch_size, layers, args.layer_start, layer_end)
        else:
            results = new_results(args.model_name, args.batch_size, layers)
        spec = MODEL_SPECS[args.model_name]
        seq_len_from_shapes(spec, shapes, args.layer_start)   # bad -s fails before any device work
        require_gpu(args.device)
        model_file = args.model_file or model_cfg.get_model_default_weights_file(args.model_name)
        prof = profile_layers(args.model_name, args.batch_size, args.layer_start, layer_end,
                              weights=load_weights(spec, model_file), shapes_in=shapes, warmup=args.warmup,
                              iterations=args.iterations, device=args.device)
    except ProfilerError as exc:
        print(f"profiler.py: error: {exc}", file=sys.stderr)
        return 1
    save_results(merge_results(results, prof['profile_data']), args.results_yml)
    logger.info("Wrote %s (%s)", args.results_yml, prof['device'])
    return 0


if __name__ == "__main__":
    sys.exit(main())
