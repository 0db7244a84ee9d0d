"""Does the profile predict what a stage costs? Profiles ViT-B at micro-batch 8 and BERT-base-CoLA at micro-batch 32
(128 tokens) with `profiler.profile_layers`, then times every stage of the even 2-, 4- and 8-way partitions and of one
mid-block cut as its own shard graph, the way the profiler times its plain graph, and prints the predicted time (the
sum of the stage's layer times) against the measured one, with the card and its power limit.

    python scripts/profile_vs_stages.py [--iterations 200] [--json out.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import profiler  # noqa: E402
from pipeedge_b200.synth import MODEL_SPECS, synth_weights  # noqa: E402

WORKLOADS = [('google/vit-base-patch16-224', 8), ('textattack/bert-base-uncased-CoLA', 32)]


def partitions(layers):
    """The even 2-, 4- and 8-way partitions and one mid-block cut."""
    out = {}
    for ways in (2, 4, 8):
        step = layers // ways
        out[f"{ways}-way"] = [(1 + i * step, (i + 1) * step) for i in range(ways)]
    out['mid-block'] = [(1, 22), (23, layers)]
    return out


def stage_time(spec, weights, batch, layer_start, layer_end, iterations):
    """Device seconds per forward of the shard [layer_start, layer_end] replayed as one CUDA graph."""
    shard = profiler.make_shard(spec, weights, layer_start, layer_end)
    seq_len = profiler.seq_len_from_shapes(spec, None, layer_start)
    inputs = profiler.shard_inputs(spec, batch, layer_start, seq_len, shard.stage.device)
    with torch.no_grad():
        (seconds,) = profiler.time_graphs([lambda: shard(inputs)], iterations, True, [None])
    shard.stage.close()
    return seconds


def main():
    parser = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    parser.add_argument('--iterations', type=int, default=profiler.DEFAULT_ITERATIONS)
    parser.add_argument('--json', type=str, default=None, help='also write the rows here')
    args = parser.parse_args()
    dev = profiler.require_gpu(None)
    device = profiler.device_description(dev)
    print(f"device: {device}")
    rows, overheads = [], {}
    for name, batch in WORKLOADS:
        spec = MODEL_SPECS[name]
        weights = synth_weights(spec, seed=0)
        prof = profiler.profile_layers(name, batch, weights=weights, iterations=args.iterations)
        times = {pd['layer']: pd['time'] for pd in prof['profile_data']}
        overheads[name] = prof['stamped_s'] / prof['plain_s']
        print(f"\n{name} micro-batch {batch}: whole model {prof['plain_s'] * 1e6:.1f} us plain, "
              f"{prof['stamped_s'] * 1e6:.1f} us stamped (stamps x{overheads[name]:.4f})")
        print(f"{'partition':>10} {'stage':>9} {'predicted us':>13} {'measured us':>12} {'rel err':>8}")
        for part, stages in partitions(spec.layers).items():
            for lo, hi in stages:
                predicted = sum(times[l] for l in range(lo, hi + 1))
                measured = stage_time(spec, weights, batch, lo, hi, args.iterations)
                err = (predicted - measured) / measured
                rows.append({'model': name, 'batch': batch, 'partition': part, 'stage': [lo, hi],
                             'predicted_s': predicted, 'measured_s': measured, 'rel_err': err})
                print(f"{part:>10} {f'[{lo},{hi}]':>9} {predicted * 1e6:13.1f} {measured * 1e6:12.1f} {err:+8.1%}")
    if args.json:
        with open(args.json, 'w', encoding='utf-8') as f:
            json.dump({'device': device, 'stamp_overhead': overheads, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
