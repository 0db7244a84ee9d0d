"""Cost of the native pipeline's per-micro-batch timestamps: ms per micro-batch of ViT-B (micro-batch 8) on 1 and 2 ranks
with and without stamps, and the update step of %globaltimer seen in the records.

    python scripts/monitoring_overhead.py [--steps 200] [--warmup 20] [--reps 3] [--ranks 1 2]

Each rank is a process; ranks share GPUs when there are fewer GPUs than ranks. Per configuration the data rank feeds
`--warmup` micro-batches, then times `--steps` more: the pipe's device time from the first graph launch to the last
result copied out (`pe_pipe_timing`), divided by the steps. Stamps off and on alternate `--reps` times in one process
group. Prints one JSON line per rank count.
"""
import argparse
import json
import os
import socket
import subprocess
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODEL = 'google/vit-base-patch16-224'


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _worker(rank, world, port, args, out_q):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), PIPEEDGE_NATIVE='1')
    os.environ.setdefault('PIPEEDGE_LINK_TIMEOUT_S', '60')
    import torch
    from pipeedge_b200.comm.p2p import DistP2pContext, DistP2pPipelineStage
    from pipeedge_b200.models import ModuleShardConfig
    from pipeedge_b200.models.transformers.vit import ViTShardForImageClassification
    from pipeedge_b200.synth import MODEL_SPECS, hf_config, synth_input, synth_weights
    torch.cuda.set_device(rank % torch.cuda.device_count())
    spec = MODEL_SPECS[MODEL]
    weights = synth_weights(spec, seed=0)
    cut = spec.layers // 2 if world == 2 else spec.layers
    lo, hi = (1, cut) if rank == 0 else (cut + 1, spec.layers)
    x = synth_input(spec, args.ubatch, seed=1).pin_memory()
    phase_done = [threading.Event() for _ in range(2 * args.reps)]
    rows = []

    def run(ctx, phase, stamps):
        records = []
        cfg = ModuleShardConfig(layer_start=lo, layer_end=hi, is_first=lo == 1, is_last=hi == spec.layers)
        shard = ViTShardForImageClassification(hf_config(spec), cfg, weights)
        if stamps:   # a no-op hook that asks for every timestamp record: stamps on, nothing else
            marker = lambda *_: None   # noqa: E731
            marker._pe_native = True
            marker._pe_records = lambda _shard: records.append
            shard.register_forward_hook(marker)
        count, done = [0], threading.Event()
        want = [args.warmup]

        def results_cb(_t):
            count[0] += 1
            if count[0] == want[0]:
                done.set()

        src = None if world == 1 else 1 - rank
        with DistP2pPipelineStage(src, src, shard, results_cb if rank == 0 else None) as stage:
            assert stage.native is not None, "the native pipeline was not selected"
            if rank != 0:
                assert phase_done[phase].wait(600)
                return None
            for _ in range(args.warmup):
                stage.enqueue_tensor(x)
            assert done.wait(600)
            done.clear()
            want[0] += args.steps
            stage.native.timing_reset()
            for _ in range(args.steps):
                stage.enqueue_tensor(x)
            assert done.wait(600)
            stage.check_workers()
            timing = stage.native.timing()
            if world > 1:
                ctx.cmd_broadcast(phase)
            native = stage.native
        return {'stamps': stamps, 'ms_per_ubatch': timing['results_ms'] / args.steps, 'records': len(records),
                'dropped': native.records_dropped,
                'kernels': {f'{ub}x{dim}': k for (ub, dim), k in native.graph_kernels.items()},
                'stamp_ns': [v for r in records for v in (r.t_start, r.t_got, r.t_stage, r.t_send_start, r.t_send_end)]}

    with DistP2pContext(('gloo',), {'world_size': world, 'rank': rank},
                        lambda c, t: phase_done[c].set() if 0 <= c < len(phase_done) else None) as ctx:
        for rep in range(args.reps):
            for k, stamps in enumerate((False, True)):
                row = run(ctx, 2 * rep + k, stamps)
                if row is not None:
                    rows.append(row)
    if rank == 0:
        out_q.put(rows)
        out_q.close()
        out_q.join_thread()


def _granularity(stamps):
    """The smallest nonzero difference between two timestamps of the records, and the largest power of two dividing all."""
    values = sorted(set(stamps))
    steps = [b - a for a, b in zip(values, values[1:])]
    div = 1
    while div < (1 << 20) and all(v % (div * 2) == 0 for v in values):
        div *= 2
    return (min(steps) if steps else None), div


def main() -> None:
    parser = argparse.ArgumentParser(description=__doc__.split('\n', 1)[0])
    parser.add_argument('--steps', type=int, default=200)
    parser.add_argument('--warmup', type=int, default=20)
    parser.add_argument('--reps', type=int, default=3)
    parser.add_argument('--ubatch', type=int, default=8)
    parser.add_argument('--ranks', type=int, nargs='+', default=[1, 2])
    args = parser.parse_args()
    import torch
    import torch.multiprocessing as mp
    if not torch.cuda.is_available():
        raise SystemExit("monitoring_overhead.py needs a CUDA device")
    gpu = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        power = 'unknown'
    for world in args.ranks:
        ctx = mp.get_context('spawn')
        out_q = ctx.Queue()
        port = _free_port()
        procs = [ctx.Process(target=_worker, args=(r, world, port, args, out_q)) for r in range(world)]
        for p in procs:
            p.start()
        rows = out_q.get(timeout=1800)
        for p in procs:
            p.join(300)
        assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
        off = [r['ms_per_ubatch'] for r in rows if not r['stamps']]
        on = [r['ms_per_ubatch'] for r in rows if r['stamps']]
        stamps = [v for r in rows for v in r['stamp_ns']]
        step, div = _granularity(stamps)
        print(json.dumps({
            'model': MODEL, 'ubatch': args.ubatch, 'ranks': world, 'steps': args.steps, 'gpu': gpu, 'power_limit': power,
            'ms_per_ubatch_off': off, 'ms_per_ubatch_on': on,
            'median_off': sorted(off)[len(off) // 2], 'median_on': sorted(on)[len(on) // 2],
            'records_per_run': [r['records'] for r in rows if r['stamps']],
            'dropped': sum(r['dropped'] for r in rows),
            'kernels_off': rows[0]['kernels'], 'kernels_on': rows[1]['kernels'],
            'globaltimer_min_step_ns': step, 'globaltimer_values_divisible_by': div}), flush=True)


if __name__ == '__main__':
    main()
