"""The data rank inside vs outside the stage pipeline (`runtime.py -D 0` with and without `-r 1,2`).

ViT-Base cut into two stages `[1,24],[25,48]`, unquantised. Inside: ranks 0 (the data rank, stage 0) and 1. Outside:
rank 0 feeds stage 0 on rank 1 through the relay kernel and collects results from stage 1 on rank 2. Outside with a
host data rank: the same ranks, rank 0 without a GPU (CUDA_VISIBLE_DEVICES=''), feeding and collecting through rings in
shared memory (`NativeHostFeeder`). Every
configuration runs as its own set of processes; the configurations are interleaved and repeated. Per run it prints:
  * stage0_ms: device time per micro-batch on stage 0 over the timed phase (its first graph launch to the end of its
    last, `NativeStage.timing()`); null on the Python-thread path, which has no such timer;
  * items_per_s: results-side throughput on the data rank (first enqueue of the timed phase to its last result).
With one GPU all ranks share it. With one GPU per rank it also runs the outside topology with every rank on its own
GPU, on the native pipeline and on the Python-thread path (`PIPEEDGE_NATIVE=0`).

    python scripts/data_rank_outside.py [--model google/vit-base-patch16-224] [--ubatch 8] [--n 200] [--repeats 2]
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
CMD_STOP, CMD_RESET = 0, 1


def _card() -> dict:
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], check=True,
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [f.strip() for f in out.split(',')]
    except (OSError, subprocess.SubprocessError, IndexError, ValueError):
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return {'gpu': name, 'power_limit': power}


def _worker(rank, port, cfg, args, out_q):
    sys.path.insert(0, ROOT)
    host = cfg.get('host', False) and rank == 0
    if host:
        os.environ['CUDA_VISIBLE_DEVICES'] = ''   # the data rank without a GPU, as `runtime.py -d cpu` makes it
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), PIPEEDGE_NATIVE='1' if cfg['native'] else '0')
    if not host:
        torch.cuda.set_device(rank if cfg['own_gpu'] else 0)
    import model_cfg
    import runtime as rt
    from pipeedge_b200.comm.p2p import DistP2pContext
    from pipeedge_b200.models import ModuleShardConfig
    from pipeedge_b200.synth import MODEL_SPECS, hf_config, synth_input, synth_weights
    spec = MODEL_SPECS[args.model]
    stage_ranks = [1, 2] if cfg['outside'] else [0, 1]
    world = len(stage_ranks) + (1 if cfg['outside'] else 0)
    s = stage_ranks.index(rank) if rank in stage_ranks else None
    shard = None
    if s is not None:
        lo, hi = (1, args.cut) if s == 0 else (args.cut + 1, spec.layers)
        scfg = ModuleShardConfig(layer_start=lo, layer_end=hi, is_first=lo == 1, is_last=hi == spec.layers)
        shard = model_cfg.get_model_dict(args.model)['shard_module'](hf_config(spec), scfg, synth_weights(spec, seed=0))
        shard.use_cuda_graph = True
        shard.register_buffer('quant_bit', torch.tensor(0), persistent=False)
        if s == 0:
            shard.register_forward_hook(rt.forward_hook_quant_encode)
        else:
            shard.register_forward_pre_hook(rt.forward_pre_hook_quant_decode)
    stop, holder = threading.Event(), []
    count, cond = [0], threading.Condition()

    def on_cmd(cmd, _tensors):
        if cmd == CMD_STOP:
            stop.set()
        elif cmd == CMD_RESET and holder and holder[0].native is not None:
            holder[0].native.timing_reset()   # stage 0's next graph launch starts the timed phase

    def results_cb(_t):
        with cond:
            count[0] += 1
            cond.notify_all()

    x = synth_input(spec, args.ubatch, seed=1)
    x = x if host else x.pin_memory()
    report = {}
    with DistP2pContext(('gloo',), {'world_size': world, 'rank': rank}, on_cmd) as ctx:
        with model_cfg.dist_p2p_pipeline_stage_factory(stage_ranks, 0, rank, s, shard, results_cb) as stage:
            holder.append(stage)
            if rank == 0:
                def phase(n):
                    with cond:
                        start = count[0]
                    t0 = time.perf_counter()
                    for _ in range(n):
                        stage.enqueue_tensor(x)
                    with cond:
                        assert cond.wait_for(lambda: count[0] >= start + n, 600), "results did not arrive"
                    return time.perf_counter() - t0

                phase(args.warmup)
                ctx.cmd_broadcast(CMD_RESET)
                if stage.native is not None and s == 0:
                    stage.native.timing_reset()
                time.sleep(0.5)   # the reset command reaches stage 0 before the timed phase starts
                report['items_per_s'] = args.n * args.ubatch / phase(args.n)
                report['native'] = stage.native is not None
                if stage.native is not None and s == 0:
                    stage.native.sync()
                    report['stage0_ms'] = stage.native.timing()['compute_ms'] / args.n
                ctx.cmd_broadcast(CMD_STOP)
            else:
                assert stop.wait(1800)
                if s == 0 and stage.native is not None:
                    stage.native.sync()
                    report['stage0_ms'] = stage.native.timing()['compute_ms'] / args.n
    out_q.put((rank, report))
    out_q.close()
    out_q.join_thread()
    if not cfg['native']:
        # per-hop NCCL communicators: leave without the exit-time library teardown, as runtime.py does on that path
        sys.stdout.flush()
        os._exit(0)


def _run(cfg, args) -> dict:
    world = 3 if cfg['outside'] else 2
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
                    raise SystemExit(f"{cfg['name']}: rank {failed[0]} exited with {procs[failed[0]].exitcode}")
    finally:
        for p in procs:
            p.join(120 if len(reports) == world else 5)
            if p.is_alive():   # a peer failed: it would wait for a stop command that never comes
                p.kill()
                p.join(10)
    stage0 = next((rep['stage0_ms'] for rep in reports.values() if 'stage0_ms' in rep), None)
    return {'config': cfg['name'], 'native': reports[0]['native'], 'items_per_s': round(reports[0]['items_per_s'], 1),
            'stage0_ms': None if stage0 is None else round(stage0, 4)}


def main() -> None:
    parser = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    parser.add_argument('--model', default='google/vit-base-patch16-224')
    parser.add_argument('--cut', type=int, default=24, help="last sub-layer of stage 0")
    parser.add_argument('--ubatch', type=int, default=8)
    parser.add_argument('--n', type=int, default=200, help="micro-batches in the timed phase")
    parser.add_argument('--warmup', type=int, default=50)
    parser.add_argument('--repeats', type=int, default=2)
    args = parser.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("data_rank_outside.py measures on a GPU; none is visible")
    configs = [dict(name='inside, one GPU', outside=False, own_gpu=False, native=True),
               dict(name='outside, one GPU', outside=True, own_gpu=False, native=True),
               dict(name='outside, host data rank, one GPU', outside=True, own_gpu=False, native=True, host=True)]
    if torch.cuda.device_count() >= 3:
        configs += [dict(name='outside, GPU per rank', outside=True, own_gpu=True, native=True),
                    dict(name='outside, GPU per rank, PIPEEDGE_NATIVE=0', outside=True, own_gpu=True, native=False)]
    head = dict(_card(), model=args.model, cut=args.cut, ubatch=args.ubatch, n=args.n, warmup=args.warmup)
    print(json.dumps(head), flush=True)
    for rep in range(args.repeats):
        for cfg in configs:
            print(json.dumps(dict(_run(cfg, args), repeat=rep)), flush=True)


if __name__ == '__main__':
    main()
