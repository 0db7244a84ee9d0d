"""In-graph cost per launch of the long-K GEMMs under forced cluster plans, with the L2 -> SM operand traffic each plan
implies. The timing follows bench.py's dominant_kernel_us: back-to-back launches in one CUDA graph, each on a distinct
weight copy (copies total > 200 MB, four times the H100's L2), CUDA events around graph replays.

Modelled traffic: every tile streams its slice of an A row block (128/CN rows) and of a W panel (BN/CM rows) over the
whole K, so bytes = tiles * (128/CN + BN/CM) * K * 2. Multicast delivers each slice to the CN (A) or CM (W) CTAs that share
it without a second L2 read.

    python scripts/gemm_cluster_sweep.py            # every shape below
    python scripts/gemm_cluster_sweep.py vitb_fc2   # one shape
"""
import ctypes
import os
import subprocess
import sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pipeedge_b200 import _lib, ops  # noqa: E402

F32, F16, GELU = _lib.PE_EPI_F32, _lib.PE_EPI_F16, _lib.PE_EPI_GELU_F16
# name: (m, n, k, epilogue, forced plans "CM,CN,BN" or None for the planner's own choice)
SHAPES = {
    'vitb_fc2': (8 * 197, 768, 3072, F32, [None, '1,1,96', '1,8,96', '2,4,96', '4,2,96', '2,2,96', '1,2,96',
                                               '2,1,96']),
    'vitl_fc2': (16 * 197, 1024, 4096, F32, [None, '1,1,224', '2,1,224']),
    'bert_fc2': (32 * 128, 768, 3072, F32, [None, '1,1,192', '1,2,192', '1,4,192', '2,2,192', '2,4,192', '4,2,192']),
    'vitb_qkv': (8 * 197, 2304, 768, F16, [None]),
    'vitb_out': (8 * 197, 768, 768, F32, [None]),
    'vitb_fc1': (8 * 197, 3072, 768, GELU, [None]),
}


def plan_of(m, n, k, epi):
    out = (ctypes.c_int * 6)()
    _lib.check(_lib.LIB.pe_debug_gemm_plan(m, n, k, epi, out))
    return dict(zip(('cm', 'cn', 'bn', 'stages', 'tiles', 'ctas'), out))


def cta_tiles(m, n, p):
    """Tiles the launch runs, counting the idle tiles that pad a partial cluster (they issue their loads too)."""
    mb, nb = -(-m // 128), -(-n // p['bn'])
    return -(-mb // p['cm']) * p['cm'] * -(-nb // p['cn']) * p['cn']


def time_launch_us(m, n, k, epi, dev):
    copies = max(8, int(200e6 // (n * k * 2)) + 1)
    gen = torch.Generator(device=dev).manual_seed(7)
    a = torch.randn(m, k, device=dev, generator=gen).half()
    ws = [(torch.randn(n, k, device=dev, generator=gen) * 0.02).half() for _ in range(copies)]
    bias = torch.zeros(n, device=dev)
    out = torch.empty(m, n, device=dev, dtype=torch.float16 if epi in (F16, GELU) else torch.float32)
    side = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(side):
        for i in range(3):
            ops.linear(a, ws[i], bias, epi, out=out, static_w=True)
        side.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            for w in ws:
                ops.linear(a, w, bias, epi, out=out, static_w=True)
        for _ in range(3):
            graph.replay()
        reps = 20
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record(side)
        for _ in range(reps):
            graph.replay()
        end.record(side)
        side.synchronize()
    return start.elapsed_time(end) * 1e3 / (reps * copies)


def smi(fields):
    res = subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], capture_output=True,
                         text=True, check=False)
    return res.stdout.strip().splitlines()[0] if res.returncode == 0 and res.stdout.strip() else 'unavailable'


def main():
    assert torch.cuda.is_available(), "the sweep times kernels on a CUDA device"
    dev = torch.device('cuda', 0)
    print(f"device: {torch.cuda.get_device_name(dev)} | {smi('power.limit,clocks.max.sm')}", flush=True)
    only = [a for a in sys.argv[1:] if not a.startswith('-')] or list(SHAPES)
    for name in only:
        m, n, k, epi, plans = SHAPES[name]
        for force in plans:
            if force is None:
                os.environ.pop('PE_GEMM_FORCE', None)
            else:
                os.environ['PE_GEMM_FORCE'] = force
            p = plan_of(m, n, k, epi)
            us = time_launch_us(m, n, k, epi, dev)
            l2 = cta_tiles(m, n, p) * (128 // p['cn'] + p['bn'] // p['cm']) * k * 2
            flop = 2.0 * m * n * k
            print(f"{name:9s} {m}x{n}x{k} plan {force or 'auto':9s} cm {p['cm']} cn {p['cn']} bn {p['bn']:3d} "
                  f"stages {p['stages']} tiles {p['tiles']:3d} ctas {p['ctas']:3d}: {us:7.2f} us/launch  "
                  f"L2->SM {l2 / 1e6:6.1f} MB  {l2 / (us * 1e-6) / 1e12:5.2f} TB/s  {flop / (us * 1e-6) / 1e12:6.1f} TFLOP/s",
                  flush=True)
    os.environ.pop('PE_GEMM_FORCE', None)
    print(f"clocks after the sweep: {smi('clocks.sm,clocks.max.sm,power.draw,power.limit,temperature.gpu')}", flush=True)


if __name__ == '__main__':
    main()
