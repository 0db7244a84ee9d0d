"""Where a GEMM launch's time goes, per CTA, from the kernel's own clock64 stamps (pe_debug_gemm_trace).

For each ViT-B/16 GEMM at micro-batch 8 (M = 1576) the launches run back to back in one CUDA graph on distinct weight
copies, as in gemm_cluster_sweep.py; the stamps of the graph's last launch are read back. Stamps (trace slots): 0 start,
1 after pdl_wait, 2 first full stage, 3 main loop done, 5 epilogue done, 6 exit; 7, 8 and 10 are 2, 3 and 5 of a
CTA's second tile (multi-round plans). Phases, in SM cycles and in microseconds at the card's maximum SM clock:

    setup        start -> after pdl_wait (the predecessor's drain under programmatic dependent launch)
    first load   after pdl_wait -> first full stage
    main loop    first full stage -> last MMA retired
    epilogue     last MMA retired -> epilogue done (with TMA stores: stores issued, not completed)
    next wait    epilogue done -> the second tile's first full stage
    tail         last epilogue done -> exit (stores drained, CTA barrier)

    python scripts/gemm_phases.py                 # the four ViT-B GEMMs
    PE_GEMM_REG_STORE=1 python scripts/gemm_phases.py   # the same with the register-store epilogue
"""
import ctypes
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pipeedge_b200 import _lib, ops  # noqa: E402

F32, F16, GELU, RESID = _lib.PE_EPI_F32, _lib.PE_EPI_F16, _lib.PE_EPI_GELU_F16, _lib.PE_EPI_RESID_F32
SLOTS = 32
SHAPES = {   # name: (m, n, k, epilogue)
    'vitb_qkv': (8 * 197, 2304, 768, F16),
    'vitb_out': (8 * 197, 768, 768, RESID),
    'vitb_fc1': (8 * 197, 3072, 768, GELU),
    'vitb_fc2': (8 * 197, 768, 3072, RESID),
}


def smi(fields):
    res = subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader,nounits'], capture_output=True,
                         text=True, check=False)
    return res.stdout.strip().splitlines()[0] if res.returncode == 0 and res.stdout.strip() else 'unavailable'


def plan_of(m, n, k, epi):
    out = (ctypes.c_int * 6)()
    _lib.check(_lib.LIB.pe_debug_gemm_plan(m, n, k, epi, out))
    return dict(zip(('cm', 'cn', 'bn', 'stages', 'tiles', 'ctas'), out))


def trace_launches(m, n, k, epi, ctas, dev):
    """Per-CTA stamps [ctas, SLOTS] of the last of many back-to-back launches in one graph."""
    copies = max(8, int(200e6 // (n * k * 2)) + 1)
    gen = torch.Generator(device=dev).manual_seed(7)
    a = torch.randn(m, k, device=dev, generator=gen).half()
    ws = [(torch.randn(n, k, device=dev, generator=gen) * 0.02).half() for _ in range(copies)]
    bias = torch.randn(n, device=dev, generator=gen)
    resid = torch.randn(m, n, device=dev, generator=gen) if epi == RESID else None
    out = torch.empty(m, n, device=dev, dtype=torch.float16 if epi in (F16, GELU) else torch.float32)
    trace = torch.zeros(ctas * SLOTS, dtype=torch.int64, device=dev)
    side = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(side):
        for i in range(3):
            ops.linear(a, ws[i], bias, epi, resid=resid, out=out, static_w=True)
        side.synchronize()
        _lib.check(_lib.LIB.pe_debug_gemm_trace(ctypes.c_void_p(trace.data_ptr())))
        try:
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=side):
                for w in ws:
                    ops.linear(a, w, bias, epi, resid=resid, out=out, static_w=True)
        finally:
            _lib.check(_lib.LIB.pe_debug_gemm_trace(None))
        for _ in range(5):
            graph.replay()
        trace.zero_()
        graph.replay()
        side.synchronize()
    return trace.view(ctas, SLOTS).cpu()


def phases(t):
    """{phase: tensor of cycles over the CTAs that have it}."""
    t = t.double()
    two = t[:, 8] > 0
    last_epi = torch.where(two, t[:, 10], t[:, 5])
    ph = {
        'setup': t[:, 1] - t[:, 0],
        'first load': t[:, 2] - t[:, 1],
        'main loop': t[:, 3] - t[:, 2],
        'epilogue': t[:, 5] - t[:, 3],
    }
    if bool(two.any()):
        ph['next wait'] = (t[:, 7] - t[:, 5])[two]
        ph['main loop 2'] = (t[:, 8] - t[:, 7])[two]
        ph['epilogue 2'] = (t[:, 10] - t[:, 8])[two]
    ph['tail'] = t[:, 6] - last_epi
    ph['total'] = t[:, 6] - t[:, 0]
    return ph


def main():
    assert torch.cuda.is_available(), "the stamps come from a CUDA device"
    dev = torch.device('cuda', 0)
    path = 'registers' if os.environ.get('PE_GEMM_REG_STORE') == '1' else 'default'
    print(f"device: {torch.cuda.get_device_name(dev)} | power.limit W, clocks.max.sm MHz: "
          f"{smi('power.limit,clocks.max.sm')} | store path: {path}", flush=True)
    clk = smi('clocks.max.sm')
    mhz = float(clk) if clk.replace('.', '', 1).isdigit() else 0.0   # cycles -> us at the maximum SM clock
    only = [a for a in sys.argv[1:] if not a.startswith('-')] or list(SHAPES)
    for name in only:
        m, n, k, epi = SHAPES[name]
        p = plan_of(m, n, k, epi)
        t = trace_launches(m, n, k, epi, p['ctas'], dev)
        print(f"{name} {m}x{n}x{k} plan cm {p['cm']} cn {p['cn']} bn {p['bn']} stages {p['stages']} "
              f"tiles {p['tiles']} ctas {p['ctas']}", flush=True)
        print(f"  {'phase':12s} {'CTAs':>4s} {'median cyc':>10s} {'max cyc':>8s} {'median us':>9s} {'max us':>7s}")
        for ph, v in phases(t).items():
            med, mx = float(v.median()), float(v.max())
            us = (lambda c: c / mhz) if mhz > 0 else (lambda c: float('nan'))
            print(f"  {ph:12s} {v.numel():4d} {med:10.0f} {mx:8.0f} {us(med):9.2f} {us(mx):7.2f}", flush=True)


if __name__ == '__main__':
    main()
