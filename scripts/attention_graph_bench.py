"""In-graph cost of pe_attention (the wgmma attention kernel) at the supported models' flagship shapes (DESIGN.md 4a).

For each shape: microseconds per launch in a CUDA graph of R back-to-back launches (PDL on, as in a stage's graph), the
median and range of several timed windows. Prints a line naming the card, its power limit and maximum SM clock, then one
JSON line per shape. Uses only pe_attention, so the same script times any version of the kernel.

    python scripts/attention_graph_bench.py [--launches 48] [--replays 50] [--repeats 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pipeedge_b200._lib import LIB, check  # noqa: E402

# (name, micro-batch, tokens, heads): ViT-B ub 8, ViT-L ub 16, BERT-base ub 32 at S 128, DeiT-B distilled ub 32
SHAPES = [('vit-base', 8, 197, 12), ('vit-large', 16, 197, 16), ('bert-base', 32, 128, 12), ('deit-base', 32, 198, 12)]


def card():
    props = torch.cuda.get_device_properties(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30, check=False).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'unknown'
    return {'card': props.name, 'sms': props.multi_processor_count, 'power_limit, max_sm_clock': q}


def in_graph_us(fn, launches, replays, repeats):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(launches):
            fn()
    graph.replay()
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(replays):
            graph.replay()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e) * 1e3 / (replays * launches))
    times.sort()
    return times[len(times) // 2], times[0], times[-1]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--launches', type=int, default=48, help='attention launches per graph')
    ap.add_argument('--replays', type=int, default=50, help='graph replays per timed window')
    ap.add_argument('--repeats', type=int, default=5, help='timed windows (median reported)')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    print(json.dumps(card()), flush=True)
    for name, batch, tokens, heads in SHAPES:
        gen = torch.Generator(device='cuda').manual_seed(tokens)
        qkv = torch.randn(batch * tokens, 3 * heads * 64, device='cuda', generator=gen).half()
        ctx = torch.empty(batch * tokens, heads * 64, device='cuda', dtype=torch.float16)

        def attention():
            check(LIB.pe_attention(qkv.data_ptr(), ctx.data_ptr(), batch, tokens, heads, 64,
                                   torch.cuda.current_stream().cuda_stream))

        med, lo, hi = in_graph_us(attention, args.launches, args.replays, args.repeats)
        print(json.dumps({'shape': name, 'batch': batch, 'tokens': tokens, 'heads': heads, 'ctas': batch * heads *
                          ((tokens + 63) // 64), 'us_per_launch': round(med, 2), 'range': [round(lo, 2), round(hi, 2)]}),
              flush=True)


if __name__ == '__main__':
    main()
