"""Adaptive bit-widths on the native pipeline: what a stage pays for holding one graph variant per send bit-width.

A 2-rank pipeline (both ranks on cuda:0, peer-memory links between the processes) whose data rank declares the
adaptive policies' bit-widths (0, 2, 3, 4, 5, 6, 8, 10, 16). It prints, with the card's name and power limit:
  * capture_ms: host time of `prepare()` on the data rank - every variant of one shape captured (eager run + capture of
    both buffer parities per bit-width);
  * per micro-batch device time of the data rank (CUDA events around its graph launches over a phase) at a fixed
    bit-width, and alternating bit-widths every micro-batch; the phases are interleaved and repeated.

    python scripts/adaptive_native.py [--model google/vit-base-patch16-224] [--cut 24] [--ubatch 8] [--n 100]
"""
import argparse
import json
import os
import queue
import socket
import subprocess
import sys
import threading
import time
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BITS = (0, 2, 3, 4, 5, 6, 8, 10, 16)
PHASES = [('fixed 8', (8,)), ('alternating 8/4', (8, 4)), ('fixed 4', (4,)), ('alternating 8/6', (8, 6)),
          ('fixed 6', (6,))]


def _card() -> dict:
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], check=True,
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [f.strip() for f in out.split(',')]
    except (OSError, subprocess.SubprocessError, IndexError, ValueError):
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return {'gpu': name, 'power_limit': power}


def _worker(rank, port, args, out_q):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), PIPEEDGE_NATIVE='1')
    torch.cuda.set_device(0)
    import runtime as rt
    from pipeedge_b200.comm.p2p import DistP2pContext, DistP2pPipelineStage
    from pipeedge_b200.models import ModuleShardConfig
    from pipeedge_b200.synth import MODEL_SPECS, hf_config, synth_input, synth_weights
    import model_cfg
    spec = MODEL_SPECS[args.model]
    lo, hi = (1, args.cut) if rank == 0 else (args.cut + 1, spec.layers)
    cfg = ModuleShardConfig(layer_start=lo, layer_end=hi, is_first=lo == 1, is_last=hi == spec.layers)
    shard = model_cfg.get_model_dict(args.model)['shard_module'](hf_config(spec), cfg, synth_weights(spec, seed=0))
    shard.register_buffer('quant_bit', torch.tensor(8 if rank == 0 else 0), persistent=False)
    if rank == 0:
        declare = lambda *_: None   # noqa: E731
        declare._pe_native = True
        declare._pe_send_bits = BITS
        shard.register_forward_hook(declare)
        shard.register_forward_hook(rt.forward_hook_quant_encode)
    else:
        shard.register_forward_pre_hook(rt.forward_pre_hook_quant_decode)
    stop = threading.Event()
    count = [0]
    cond = threading.Condition()

    def results_cb(_t):
        with cond:
            count[0] += 1
            cond.notify_all()

    x = synth_input(spec, args.ubatch, seed=1).pin_memory()
    report = {}
    with DistP2pContext(('gloo',), {'world_size': 2, 'rank': rank}, lambda c, t: stop.set() if c == 0 else None) as ctx:
        with DistP2pPipelineStage(1 if rank == 0 else 0, 1 if rank == 0 else 0, shard,
                                  results_cb if rank == 0 else None) as stage:
            native = stage.native
            assert native is not None and (rank == 1 or native.adaptive), "not an adaptive native stage"
            if rank == 0:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                stage.prepare(args.ubatch)        # every variant of the shape; returns after the last capture
                report['capture_ms'] = (time.perf_counter() - t0) * 1e3
                report['variants'] = native.variants

                def phase(bits, n):
                    with cond:
                        start = count[0]
                    native.timing_reset()
                    for i in range(n):
                        shard.quant_bit = torch.tensor(bits[i % len(bits)])
                        stage.enqueue_tensor(x)
                    with cond:
                        assert cond.wait_for(lambda: count[0] >= start + n, 300), "results did not arrive"
                    native.sync()
                    return native.timing()['compute_ms'] / n

                phase(BITS, 2 * len(BITS))                      # warm-up: every variant launched
                times = {name: [] for name, _ in PHASES}
                for _ in range(args.repeats):
                    for name, bits in PHASES:
                        times[name].append(phase(bits, args.n))
                report['ms_per_ubatch'] = times
                report['captures'] = native.captures
                ctx.cmd_broadcast(0)
            else:
                assert stop.wait(1800)
    out_q.put((rank, report))


def main() -> None:
    parser = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    parser.add_argument('--model', default='google/vit-base-patch16-224')
    parser.add_argument('--cut', type=int, default=24, help="last sub-layer of the first stage")
    parser.add_argument('--ubatch', type=int, default=8)
    parser.add_argument('--n', type=int, default=100, help="micro-batches per timed phase")
    parser.add_argument('--repeats', type=int, default=3)
    args = parser.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("adaptive_native.py measures on a GPU; none is visible")
    ctx = mp.get_context('spawn')
    out_q = ctx.Queue()
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    procs = [ctx.Process(target=_worker, args=(r, port, args, out_q)) for r in range(2)]
    for p in procs:
        p.start()
    reports = {}
    try:
        while len(reports) < 2:
            try:
                rank, report = out_q.get(timeout=5)
                reports[rank] = report
            except queue.Empty:
                failed = [r for r, p in enumerate(procs) if p.exitcode not in (None, 0)]
                if failed:
                    raise SystemExit(f"rank {failed[0]} exited with {procs[failed[0]].exitcode}")
    finally:
        for p in procs:
            p.join(120 if len(reports) == 2 else 5)
            if p.is_alive():   # its peer failed: it would wait for a stop command that never comes
                p.kill()
                p.join(10)
    rep = reports[0]
    result = dict(_card(), model=args.model, cut=args.cut, ubatch=args.ubatch, n=args.n, bits=list(BITS),
                  capture_ms=round(rep['capture_ms'], 1), variants=rep['variants'], captures=rep['captures'],
                  ms_per_ubatch={k: [round(v, 4) for v in vs] for k, vs in rep['ms_per_ubatch'].items()})
    print(json.dumps(result))


if __name__ == '__main__':
    main()
