"""R replicas of an S-stage pipeline fed by one data rank outside them (`runtime.py --replicas R`), against one
pipeline (R = 1) of the same stages, in the same session.

ViT-Base, unquantised, cut into S stages of equal sub-layer counts. Rank 0 is the data rank, with a GPU (`NativeFeeder`
per replica: each input crosses its GPU's relay) or without one (`CUDA_VISIBLE_DEVICES=''`, `NativeHostFeeder` per
replica: each first stage pulls its inputs over its own copy engine); replica k's stage s runs on rank 1 + k*S + s, on
GPU (rank mod the GPU count) - every rank on one GPU when only one is visible. Every configuration runs as its own set of
processes; configurations alternate, and each is repeated. Per run it prints one JSON line:
  * img_per_s: results-side throughput on the data rank (first enqueue of the timed phase to its last result);
  * ms_per_ubatch: the same phase's wall time per micro-batch;
  * replicas, stages, data_rank (gpu / host), gpus (visible GPUs);
  * checksum: sum over the first 16 results of the timed phase of (position + 1) * sum |logits|: it depends on the
    order results arrive in, so R > 1 must print the checksum of R = 1.
A last line per configuration gives the median and range of img/s over the repeats; the first line names the GPU, its
power limit and its SM clocks.

    python scripts/replicas.py [--replicas 1,2] [--stages 1] [--kinds gpu,host] [--ubatch 8] [--n 200] [--repeats 3]
"""
import argparse
import json
import os
import queue
import socket
import statistics
import subprocess
import sys
import threading
import time
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODEL = 'google/vit-base-patch16-224'
N_INPUTS = 16     # distinct micro-batches, cycled; the checksum covers this many results
CMD_STOP = 0


def _card() -> dict:
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                              '--format=csv,noheader'], check=True, capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power, sm, sm_max = [f.strip() for f in out.split(',')]
    except (OSError, subprocess.SubprocessError, IndexError, ValueError):
        name, power, sm, sm_max = torch.cuda.get_device_name(0), 'unknown', 'unknown', 'unknown'
    return {'gpu': name, 'power_limit': power, 'sm_clock_idle': sm, 'sm_clock_max': sm_max}


def _cuts(stages: int, layers: int):
    return [layers * (s + 1) // stages for s in range(stages)]


def _worker(rank, port, cfg, args, out_q):
    sys.path.insert(0, ROOT)
    host = cfg['kind'] == 'host' and rank == 0
    if host:
        os.environ['CUDA_VISIBLE_DEVICES'] = ''   # the data rank without a GPU, as `runtime.py -d cpu` makes it
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), PIPEEDGE_NATIVE='1')
    if not host:
        torch.cuda.set_device(rank % torch.cuda.device_count())
    import model_cfg
    import runtime as rt
    from pipeedge_b200.comm.p2p import DistP2pContext
    from pipeedge_b200.models import ModuleShardConfig
    from pipeedge_b200.synth import MODEL_SPECS, hf_config, synth_input, synth_weights
    spec = MODEL_SPECS[MODEL]
    replicas, stages = cfg['replicas'], cfg['stages']
    ranks = [list(range(1 + k * stages, 1 + (k + 1) * stages)) for k in range(replicas)]
    world = 1 + replicas * stages
    _, s, _, _ = model_cfg.replica_neighbours(ranks, 0, rank)
    shard = None
    if s is not None:
        cuts = _cuts(stages, spec.layers)
        lo, hi = (1 if s == 0 else cuts[s - 1] + 1), cuts[s]
        scfg = ModuleShardConfig(layer_start=lo, layer_end=hi, is_first=lo == 1, is_last=hi == spec.layers)
        shard = model_cfg.get_model_dict(MODEL)['shard_module'](hf_config(spec), scfg, synth_weights(spec, seed=0))
        shard.use_cuda_graph = True
        shard.register_buffer('quant_bit', torch.tensor(0), persistent=False)
        if s != stages - 1:
            shard.register_forward_hook(rt.forward_hook_quant_encode)
        if s != 0:
            shard.register_forward_pre_hook(rt.forward_pre_hook_quant_decode)
    stop = threading.Event()
    count, kept, cond = [0], [], threading.Condition()

    def results_cb(t):
        with cond:
            if len(kept) < N_INPUTS and count[0] >= args.warmup:
                kept.append(float(t.double().abs().sum()))
            count[0] += 1
            cond.notify_all()

    inputs = [synth_input(spec, args.ubatch, seed=100 + i) for i in range(N_INPUTS)]
    if not host:
        inputs = [x.pin_memory() for x in inputs]
    report = {}
    with DistP2pContext(('gloo',), {'world_size': world, 'rank': rank}, lambda c, _t: stop.set() if c == CMD_STOP
                        else None) as ctx:
        with model_cfg.dist_p2p_pipeline_stage_factory(ranks, 0, rank, s, shard, results_cb) as stage:
            if rank == 0:
                def phase(first, n):
                    t0 = time.perf_counter()
                    for i in range(first, first + n):
                        stage.enqueue_tensor(inputs[i % N_INPUTS])
                    with cond:
                        assert cond.wait_for(lambda: count[0] >= first + n, 600), "results did not arrive"
                    return time.perf_counter() - t0

                phase(0, args.warmup)
                seconds = phase(args.warmup, args.n)
                report = {'img_per_s': args.n * args.ubatch / seconds, 'ms_per_ubatch': seconds / args.n * 1e3,
                          'checksum': sum((i + 1) * v for i, v in enumerate(kept))}
                ctx.cmd_broadcast(CMD_STOP)
            else:
                assert stop.wait(1800)
    out_q.put((rank, report))
    out_q.close()
    out_q.join_thread()


def _run(cfg, args) -> dict:
    world = 1 + cfg['replicas'] * cfg['stages']
    ctx = mp.get_context('spawn')
    out_q = ctx.Queue()
    with socket.socket() as sock:
        sock.bind(('127.0.0.1', 0))
        port = sock.getsockname()[1]
    procs = [ctx.Process(target=_worker, args=(r, port, cfg, args, out_q)) for r in range(world)]
    for p in procs:
        p.start()
    reports = {}
    try:
        while len(reports) < world:
            try:
                rank, report = out_q.get(timeout=5)
                reports[rank] = report
            except queue.Empty:
                failed = [r for r, p in enumerate(procs) if p.exitcode not in (None, 0)]
                if failed:
                    raise SystemExit(f"{cfg}: rank {failed[0]} exited with {procs[failed[0]].exitcode}")
    finally:
        for p in procs:
            p.join(120 if len(reports) == world else 5)
            if p.is_alive():   # a peer failed: it would wait for a stop command that never comes
                p.kill()
                p.join(10)
    rep = reports[0]
    return {'replicas': cfg['replicas'], 'stages': cfg['stages'], 'data_rank': cfg['kind'],
            'gpus': torch.cuda.device_count(), 'img_per_s': round(rep['img_per_s'], 1),
            'ms_per_ubatch': round(rep['ms_per_ubatch'], 4), 'checksum': rep['checksum']}


def main() -> None:
    parser = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    parser.add_argument('--replicas', default='1,2', help="comma-separated R values; R = 1 is always included")
    parser.add_argument('--stages', type=int, default=1, help="stages per replica")
    parser.add_argument('--kinds', default='gpu,host', help="data rank kinds: gpu, host")
    parser.add_argument('--ubatch', type=int, default=8)
    parser.add_argument('--n', type=int, default=200, help="micro-batches in the timed phase")
    parser.add_argument('--warmup', type=int, default=50)
    parser.add_argument('--repeats', type=int, default=3)
    args = parser.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("replicas.py measures on a GPU; none is visible")
    if args.n < N_INPUTS:
        raise SystemExit(f"--n must be at least {N_INPUTS}: the checksum covers that many results")
    counts = sorted({1} | {int(r) for r in args.replicas.split(',')})
    configs = [dict(replicas=r, stages=args.stages, kind=kind) for kind in args.kinds.split(',') for r in counts]
    print(json.dumps(dict(_card(), model=MODEL, ubatch=args.ubatch, n=args.n, warmup=args.warmup,
                          gpus=torch.cuda.device_count())), flush=True)
    runs = {}
    for rep in range(args.repeats):
        for cfg in configs:
            res = _run(cfg, args)
            runs.setdefault((cfg['kind'], cfg['replicas']), []).append(res)
            print(json.dumps(dict(res, repeat=rep)), flush=True)
    for (kind, replicas), res in runs.items():
        rates = [r['img_per_s'] for r in res]
        print(json.dumps({'summary': True, 'replicas': replicas, 'stages': args.stages, 'data_rank': kind,
                          'img_per_s_median': round(statistics.median(rates), 1), 'img_per_s_min': min(rates),
                          'img_per_s_max': max(rates),
                          'ms_per_ubatch_median': round(statistics.median(r['ms_per_ubatch'] for r in res), 4),
                          'checksums': sorted({r['checksum'] for r in res})}), flush=True)


if __name__ == '__main__':
    main()
