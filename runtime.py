"""Distributed pipeline driver application - drop-in for the reference `runtime.py` p2p path.

Same CLI (`runtime.py:610-687`): `runtime.py RANK WORLDSIZE [-d] [-s] [--addr] [--port] [-c p2p] [-m] [-M] [-b]
[-u] [-pt] [-q] [-r] [-D]`, same schedule semantics (`-pt` 1-based inclusive sub-layer pairs, `-q` bits per
stage output, `-r` stage-to-rank order, `-D` data rank), same command protocol (CMD_STOP / CMD_SCHED) and the
same hook structure around the shard (`run_pipeline_p2p`, `runtime.py:418-511`). One rank per GPU:
activations stay in HBM, the hop is NCCL on a side stream, and the QuantPipe hooks call the fused device
kernels (bit-identical codes). The adaptive QuantPipe policies (`ADAPTIVE_QUANT=HEURISTIC|HEURISTIC2|CONTROLLER`
with `SEND_CONSTRAINT` items/s and `WINDOW_SIZE`, `runtime.py:121-216`) are carried over; they read the hop's
DEVICE-side transfer time (CUDA events around the NCCL sends, or the native pipeline's graph timestamps) through
`monitoring.py`'s window statistics.
Scheduler-generated partitions are ingested in the scheduler's own YAML format (`parse_yaml_sched`, `-H`, `--sched-file`, or
the reference's `sched-pipeline` binary when it is on PATH with `-sm/-sdt/-sd`). What is NOT carried over (out of scope,
SURVEY.md section 2): the RPC backend (`-c rpc`), the `sched-pipeline` planner itself, energy monitoring, and the dataset loaders that need the network; inputs are the reference's synthetic fallback (`runtime.py:386-400`)
generated locally, weights come from `-M` (an npz in the reference layout) or are synthesised.
"""
import argparse
import logging
import os
import queue
import sys
import threading
import time
from typing import List, Optional, Tuple, Union
import torch
from torch.utils.data import DataLoader, Dataset
from pipeedge_b200 import models
from pipeedge_b200.comm.p2p import DistP2pContext
from pipeedge_b200.quantization.basic_op import compression_factor, tensor_decode_outerdim, tensor_encode_outerdim
from pipeedge_b200.synth import MODEL_SPECS, synth_input, synth_weights
import devices
import model_cfg
import monitoring
from utils import quant as quantutil

logger = logging.getLogger(__name__)

CMD_STOP = 0
CMD_SCHED = 1

# A window period defines monitoring and configurability work intervals (`runtime.py:39-44`)
WINDOW_SIZE = 10
ENV_WINDOW_SIZE: str = "WINDOW_SIZE"


def get_window_size() -> int:
    """Get the window size."""
    return int(os.getenv(ENV_WINDOW_SIZE, str(WINDOW_SIZE)))


ENV_SEND_CONSTRAINT: str = "SEND_CONSTRAINT"

ENV_ADAPTIVE_QUANT: str = "ADAPTIVE_QUANT"
ADAPTIVE_QUANT_HEURISTIC = "HEURISTIC"
ADAPTIVE_QUANT_HEURISTIC2 = "HEURISTIC2"
ADAPTIVE_QUANT_CONTROLLER = "CONTROLLER"

MONITORING_KEY_MODEL = 'shard'
MONITORING_KEY_OUTPUT = 'output'
MONITORING_KEY_QUANT_DECODE = 'quant_decode'
MONITORING_KEY_QUANT_ENCODE = 'quant_encode'
MONITORING_KEY_RECV = 'recv'
MONITORING_KEY_SEND = 'send'

# Per-kernel-group heartbeats ('shard', 'quant_encode', 'quant_decode', 'output') cost four CUDA event records per
# micro-batch and stage on the Python-thread path, and timestamp kernels in every graph on the native pipeline, so
# unlike the reference they are opt-in: MONITORING=1. The 'send' key is always fed when an adaptive quantization policy
# is active.
ENV_MONITORING: str = "MONITORING"
_device_iters = None   # monitoring.DeviceIterations when MONITORING=1


def monitoring_enabled() -> bool:
    """Whether the opt-in heartbeats are on."""
    return _device_iters is not None


def enable_monitoring() -> None:
    """Turn the opt-in heartbeats on (MONITORING=1): their keys in the `monitoring` context `monitoring.init` made."""
    global _device_iters   # pylint: disable=global-statement
    monitoring.add_key(MONITORING_KEY_MODEL, work_type='tensors', acc_type='layers')
    monitoring.add_key(MONITORING_KEY_OUTPUT, work_type='classifications', acc_type='correct')
    monitoring.add_key(MONITORING_KEY_QUANT_DECODE, work_type='tensors', acc_type='bits')
    monitoring.add_key(MONITORING_KEY_QUANT_ENCODE, work_type='tensors', acc_type='bits')
    _device_iters = monitoring.DeviceIterations()


def disable_monitoring() -> None:
    """Report the heartbeats still in flight and turn them off."""
    global _device_iters   # pylint: disable=global-statement
    if _device_iters is not None:
        _device_iters.harvest(drain=True)
        _device_iters = None


def forward_pre_hook_monitor(_module, _inputs) -> None:
    """Register iteration start (`runtime.py:60-62`): a CUDA event on the shard's stream."""
    if _device_iters is not None:
        _device_iters.start(MONITORING_KEY_MODEL)


def forward_hook_monitor(module, _inputs, outputs) -> None:
    """Register iteration completion (`runtime.py:64-71`): work = micro-batch size, accuracy = layers processed; the
    duration is the device time between the two events."""
    if _device_iters is not None:
        n_items = models.get_microbatch_size(outputs, verify=True)
        n_layers = module.shard_config.layer_end - module.shard_config.layer_start + 1
        _device_iters.finish(MONITORING_KEY_MODEL, work=n_items, accuracy=n_layers)


def forward_hook_quant_encode(module, _input_arg, output: Union[torch.Tensor, Tuple[torch.Tensor, ...]]):
    """Encode tensors in the forward hook, after the shard (`runtime.py:73-91`).

    Clamp choice, threshold, per-item quantisation and bit-packing run fused on the device; the 5-tensor-per-
    payload-tensor wire format is the reference's. `quant_bit` is read per call, so adaptive policies may
    change it between micro-batches."""
    if isinstance(output, torch.Tensor):
        output = (output,)
    assert isinstance(output, tuple)
    quant_bit = int(module.quant_bit.item())
    if _device_iters is not None:
        _device_iters.start(MONITORING_KEY_QUANT_ENCODE)
    comm_tuple = []
    for tensor in output:
        assert isinstance(tensor, torch.Tensor)
        comm_tuple += tensor_encode_outerdim(tensor, quant_bit, clamp=quant_bit > 0)
    if _device_iters is not None:
        # work = micro-batch size, but quantization only does work if quant_bit > 0 (`runtime.py:88-90`)
        n_items = models.get_microbatch_size(output[0], verify=True) if quant_bit > 0 else 0
        _device_iters.finish(MONITORING_KEY_QUANT_ENCODE, work=n_items, accuracy=quant_bit)
    return tuple(comm_tuple)


def forward_pre_hook_quant_decode(_module, input_arg: Tuple[Tuple[torch.Tensor, ...]]):
    """Decode tensors in the pre-forward hook, before the shard (`runtime.py:93-119`)."""
    assert isinstance(input_arg, tuple) and len(input_arg) == 1
    input_tensors = input_arg[0]
    assert isinstance(input_tensors, tuple)
    assert len(input_tensors) % 5 == 0 and len(input_tensors) >= 5
    if _device_iters is not None:
        _device_iters.start(MONITORING_KEY_QUANT_DECODE)
    forward_tensor = [tensor_decode_outerdim(input_tensors[i * 5:i * 5 + 5]) for i in range(len(input_tensors) // 5)]
    if _device_iters is not None:
        quant_bit = int(input_tensors[4][0].item())     # same bit-width for all items (`runtime.py:103`)
        n_items = models.get_microbatch_size(forward_tensor[0], verify=True) if quant_bit > 0 else 0
        _device_iters.finish(MONITORING_KEY_QUANT_DECODE, work=n_items, accuracy=quant_bit)
    if len(forward_tensor) == 1:
        return tuple(forward_tensor)        # a single tensor payload
    return (tuple(forward_tensor),)         # a (data, skip) tuple payload


def native_heartbeats(rec, n_layers: int, encode: bool, decode: bool) -> List[Tuple[str, float, int, int]]:
    """The heartbeats `(key, seconds, work, accuracy)` the Python-thread path's hooks give for one micro-batch, from the
    native pipeline's timestamp record of it (`_native.StampRecord`; device nanoseconds). `encode` / `decode`: the
    stage has the quantisation hook of that side registered.

    * shard: receive done -> the stage's last kernel done; work = items, accuracy = layers.
    * quant_decode: on the native pipeline dequantisation is inside the receive kernel, so the key reports that
      kernel's duration, measured from the graph's start - it includes the kernel's wait for the upstream payload.
    * quant_encode: a staged send (generic bit-widths) reports its stand-alone encode kernels (send start -> encoded);
      a fused send (2 / 4 / 8 / 16 bits) quantises inside the send kernel, so the key reports that whole kernel.
    * An unquantised payload (bit 0) is not encoded or decoded: 0 s, like the thread path's pass-through hooks.
    Both quantisation keys: work = items if bit > 0 else 0, accuracy = bit (`runtime.py:88-90,124-126`)."""
    from pipeedge_b200._lib import PE_STAMP_STAGED   # pylint: disable=import-outside-toplevel
    beats = [(MONITORING_KEY_MODEL, (rec.t_stage - rec.t_got) * 1e-9, rec.items, n_layers)]
    if decode:
        bit = rec.bit_in
        beats.append((MONITORING_KEY_QUANT_DECODE, (rec.t_got - rec.t_start) * 1e-9 if bit > 0 else 0.0,
                      rec.items if bit > 0 else 0, bit))
    if encode:
        bit = rec.bit_out
        if bit == 0:
            seconds = 0.0
        elif rec.flags & PE_STAMP_STAGED:
            seconds = (rec.t_encoded - rec.t_send_start) * 1e-9
        else:
            seconds = (rec.t_send_end - rec.t_send_start) * 1e-9
        beats.append((MONITORING_KEY_QUANT_ENCODE, seconds, rec.items if bit > 0 else 0, bit))
    return beats


def _native_monitor_records(shard):
    """With MONITORING=1, the native pipeline's per-micro-batch record consumer of `shard`: the heartbeats of
    `native_heartbeats` for the hooks the shard carries. None (no timestamps) otherwise."""
    if _device_iters is None:
        return None
    n_layers = shard.shard_config.layer_end - shard.shard_config.layer_start + 1
    encode = forward_hook_quant_encode in shard._forward_hooks.values()            # pylint: disable=protected-access
    decode = forward_pre_hook_quant_decode in shard._forward_pre_hooks.values()    # pylint: disable=protected-access

    def consume(rec) -> None:
        for key, seconds, work, accuracy in native_heartbeats(rec, n_layers, encode, decode):
            monitoring.iteration(key, work=work, accuracy=accuracy, seconds=seconds)
    return consume


# What the native pipeline (pipeedge_b200/comm/p2p/_native.py) does with each hook: the quantisation pair is performed by
# the links' send / receive kernels (same codes, same decoded values); the monitor pair is fed from the graphs' device
# timestamps when MONITORING=1 (`_pe_records`: the stage turns timestamps on and hands it every record).
forward_hook_quant_encode._pe_native = True                 # pylint: disable=protected-access
forward_pre_hook_quant_decode._pe_native = True             # pylint: disable=protected-access
forward_pre_hook_monitor._pe_native = True                  # pylint: disable=protected-access
forward_hook_monitor._pe_native = True                      # pylint: disable=protected-access
forward_hook_monitor._pe_records = _native_monitor_records  # pylint: disable=protected-access


def _payload_tensors(outputs) -> Tuple[torch.Tensor, ...]:
    return (outputs,) if isinstance(outputs, torch.Tensor) else tuple(outputs)


def _send_window(*getters: str):
    """Consistent read of the send key's tag, window size and the requested `get_window_*` values."""
    with monitoring.get_locked_context(MONITORING_KEY_SEND) as mctx:
        tag = mctx.get_tag(key=MONITORING_KEY_SEND)
        window_size = mctx.get_window_size(key=MONITORING_KEY_SEND)
        values = tuple(getattr(mctx, 'get_window_' + g)(key=MONITORING_KEY_SEND) for g in getters)
    return (tag, window_size) + values


# (largest compression ratio, bit-width) steps of the heuristic; beyond the last step it sends with the floor
_HEURISTIC_STEPS = ((1, 0), (2, 16), (4, 8), (5, 6), (8, 4))
_HEURISTIC_FLOOR = 2


def forward_hook_set_quant_bandwidth_heuristic(module, _inputs, outputs) -> None:
    """Pick the quantization bit-width whose compression fits the window's send budget (`runtime.py:121-154`).

    Every `window_size` sends: budget = time the rate constraint allows for one window x measured hop bandwidth
    (Mbit/s); needed compression = what the window actually sent, scaled back to 32-bit, over that budget; mapped to
    32/16/8/6/4/2 bits by fixed thresholds."""
    tag, window_size, bandwidth, sent_mbits = _send_window('perf', 'work')
    if tag == 0 or tag % window_size != 0:
        return
    target_rate = module.rate_constraint.item()
    if target_rate > 0:
        ubatch_size = models.get_microbatch_size(outputs, verify=True)
        budget_mbits = ubatch_size * window_size / target_rate * bandwidth
    else:
        budget_mbits = float('inf')
    quant_bit = module.quant_bit.item()
    unquantized_mbits = sent_mbits * (32 / quant_bit) if quant_bit > 0 else sent_mbits
    compress_ratio = int(unquantized_mbits / budget_mbits) + 1
    for limit, bits in _HEURISTIC_STEPS:
        if compress_ratio <= limit:
            module.quant_bit = torch.tensor(bits)
            break
    else:
        module.quant_bit = torch.tensor(_HEURISTIC_FLOOR)
    logger.info("Adaptive quantization (heuristic): bitwidth=%d", int(module.quant_bit))


_HEURISTIC2_MIN_BIT = 2


def forward_hook_set_quant_bandwidth_heuristic_2(module, _inputs, outputs) -> None:
    """Largest bit-width that moves one micro-batch within its share of the rate constraint (`runtime.py:156-177`)."""
    tag, window_size, bandwidth = _send_window('perf')
    if tag == 0 or tag % window_size != 0:
        return
    tensors = _payload_tensors(outputs)
    ubatch_size = models.get_microbatch_size(outputs, verify=True)
    ubatch_time = ubatch_size / module.rate_constraint            # rate 0 -> inf: anything fits
    ubatch_mbits = sum(t.numel() * t.element_size() for t in tensors) * 8 / 1000000
    src_bit = torch.tensor(tensors[0].element_size() * 8)
    quant_bit = quantutil.constrain_max_bitwidth(ubatch_time, ubatch_mbits, bandwidth, src_bit)
    # at least 2 bits; the source width itself means "do not quantize" (0)
    module.quant_bit = max(torch.tensor(_HEURISTIC2_MIN_BIT), quant_bit) % src_bit
    logger.info("Adaptive quantization (heuristic2): bitwidth=%d", int(module.quant_bit))


# Largest bitwidths in range [2, 32] with unique discrete compressions (`runtime.py:179-181`)
BITWIDTHS = [i for i in range(32, 1, -1)
             if int(compression_factor(i)) > int(compression_factor(i + 1))]
# controllers are host objects and cannot live in a Module's buffers: cached per module
_MODULE_QUANT_CONTROLLERS = {}
_MODULE_QUANT_CONTROLLERS_LOCK = threading.Lock()


def forward_hook_set_quant_controller(module, _inputs, outputs) -> None:
    """Feedback controller: split each window between two adjacent bit-widths so that the measured send rate
    (items/s) tracks `rate_constraint` (`runtime.py:182-215`). The plan lives in the module's `bitwidth1`,
    `bitwidth2`, `bitwidth1_iters` buffers; `quant_bit` is set for the micro-batch about to be sent."""
    bw1 = int(module.bitwidth1.item()) if hasattr(module, 'bitwidth1') else 0
    bw2 = int(module.bitwidth2.item()) if hasattr(module, 'bitwidth2') else 0
    bw1_iters = int(module.bitwidth1_iters.item()) if hasattr(module, 'bitwidth1_iters') else 0
    tag, window_size, heartrate = _send_window('heartrate')
    if tag > 0 and tag % window_size == 0:
        with _MODULE_QUANT_CONTROLLERS_LOCK:
            bw_ctlr = _MODULE_QUANT_CONTROLLERS.get(module)
            if bw_ctlr is None:
                bw_start = module.quant_bit.item() or max(BITWIDTHS)        # not quantizing = the widest setting
                bw_ctlr = quantutil.AdaptiveBitwidthPerformanceController(0, BITWIDTHS, bw_start)
                _MODULE_QUANT_CONTROLLERS[module] = bw_ctlr
        bw_ctlr.reference = module.rate_constraint.item()
        send_rate = heartrate * models.get_microbatch_size(outputs, verify=True)
        bw1, bw2, bw1_iters = bw_ctlr(send_rate, window_size)
        module.register_buffer('bitwidth1', torch.tensor(bw1), persistent=False)
        module.register_buffer('bitwidth2', torch.tensor(bw2), persistent=False)
        logger.info("Adaptive quantization (controller): bitwidth1=%d (iters=%d), bitwidth2=%d", bw1, bw1_iters, bw2)
    bitwidth = bw1 if bw1_iters > 0 else bw2
    module.quant_bit = torch.tensor(bitwidth % max(BITWIDTHS))               # the widest setting = no quantization
    module.register_buffer('bitwidth1_iters', torch.tensor(max(0, bw1_iters - 1)), persistent=False)


def _native_policy_records(hook):
    """The native pipeline's record consumer factory for a policy hook (`_pe_records`): the consumer calls the same hook
    once per record of the stage, with a stand-in `outputs` of that micro-batch's geometry (meta fp32 tensors of
    [items, elements per item] per payload tensor, recovered from the record and the shapes the stage captured). The
    decision applies to the stage's next graph launch instead of the micro-batch the hook ran for."""
    def factory(shard):
        from pipeedge_b200.comm.p2p import _native   # pylint: disable=import-outside-toplevel

        def consume(rec) -> None:
            elems = _native.record_payload_elems(rec, shard.native_payload_shapes())
            outputs = tuple(torch.empty((rec.items, n), dtype=torch.float32, device='meta') for n in elems)
            hook(shard, None, outputs[0] if len(outputs) == 1 else outputs)
        return consume
    return factory


# The bit-widths each policy sets `quant_bit` to (the native pipeline captures one graph per member, `_pe_send_bits`).
# HEURISTIC: its steps and floor. HEURISTIC2: `max(_HEURISTIC2_MIN_BIT, b) % src_bit` of every b that
# `constrain_max_bitwidth` can return for an fp32 payload (src_bit 32, the native pipeline's payloads): src_bit itself,
# 0, and the largest bit-width of each packing ratio below src_bit. CONTROLLER: BITWIDTHS with the widest as 0.
_FP32_BITS = 32
QUANT_BITS_HEURISTIC = frozenset(b for _, b in _HEURISTIC_STEPS) | {_HEURISTIC_FLOOR}
QUANT_BITS_HEURISTIC2 = frozenset(max(_HEURISTIC2_MIN_BIT, b) % _FP32_BITS for b in range(_FP32_BITS, -1, -1)
                                  if b in (0, _FP32_BITS) or int(compression_factor(b)) > int(compression_factor(b + 1)))
QUANT_BITS_CONTROLLER = frozenset(b % max(BITWIDTHS) for b in BITWIDTHS)

for _hook, _bits in ((forward_hook_set_quant_bandwidth_heuristic, QUANT_BITS_HEURISTIC),
                     (forward_hook_set_quant_bandwidth_heuristic_2, QUANT_BITS_HEURISTIC2),
                     (forward_hook_set_quant_controller, QUANT_BITS_CONTROLLER)):
    _hook._pe_native = True                          # pylint: disable=protected-access
    _hook._pe_records = _native_policy_records(_hook)   # pylint: disable=protected-access
    _hook._pe_send_bits = _bits                      # pylint: disable=protected-access
del _hook, _bits


def hop_timing_hook_monitor(mbits: float, seconds: float, key: str) -> None:
    """One completed hop transfer -> one heartbeat of `key` with the device-measured duration (replaces the
    reference's host-timed `p2p_pre_hook_monitor` / `p2p_post_hook_monitor` pair, `runtime.py:218-230`)."""
    monitoring.iteration(key, work=mbits, seconds=seconds)


class ThreadSafeCounter:
    """Thread-safe counter (reference `utils/threads.py:57-91`)."""

    def __init__(self, value: int = 0):
        self._value = value
        self._cond = threading.Condition()

    @property
    def value(self) -> int:
        """Current counter value."""
        with self._cond:
            return self._value

    def add(self, quantity: int = 1) -> None:
        """Add to counter atomically."""
        with self._cond:
            self._value += quantity
            self._cond.notify_all()

    def wait_gte(self, threshold: int, timeout: Optional[float] = None) -> bool:
        """Wait until counter >= threshold."""
        with self._cond:
            return self._cond.wait_for(lambda: self._value >= threshold, timeout)


class RolloverTensorDataset(Dataset):
    """Like `TensorDataset`, but rolls over when the requested length exceeds the actual length
    (reference `utils/data.py:7-21`)."""

    def __init__(self, length: int, *tensors: torch.Tensor):
        assert all(tensors[0].size(0) == t.size(0) for t in tensors), "Size mismatch between tensors"
        self.length = length
        self.tensors = tensors

    def __getitem__(self, index):
        return tuple(t[index % len(t)] for t in self.tensors)

    def __len__(self):
        return self.length


results_counter = ThreadSafeCounter()
label_queue = queue.Queue()


def handle_results(tensors: torch.Tensor) -> None:
    """Process result tensors (`runtime.py:236-257`): argmax against the queued labels, count items."""
    n_items = models.get_microbatch_size(tensors, verify=True)
    if not label_queue.empty():
        ubatch_labels = label_queue.get()
        assert len(tensors) == len(ubatch_labels)
        pred = tensors.argmax(dim=1).cpu()
        acc = pred.eq(ubatch_labels).sum().item()
        logger.debug("micro-batch accuracy: %d/%d", acc, n_items)
    else:
        acc = 0
    if _device_iters is not None:
        # time BETWEEN results, not pipeline latency: a heartbeat series without an explicit start (`runtime.py:239-255`)
        monitoring.iteration(MONITORING_KEY_OUTPUT, work=n_items, accuracy=acc, safe=False)
    results_counter.add(n_items)


def parse_yaml_sched(sched: List[dict], hosts: Optional[List[str]]) -> Tuple[List[Tuple[int, int]], List[int]]:
    """Parse the scheduler's YAML (`sched-pipeline` prints a list of single-entry maps `host: [layer_start, layer_end]`)
    into `stage_layers` and `stage_ranks` (`runtime.py:260-288`): a host is looked up in `hosts` (its index is the rank)
    or, without a hosts list, is the rank itself."""
    assert isinstance(sched, list)
    if len(sched) == 0:
        raise RuntimeError("No viable schedule found")
    stage_layers, stage_ranks = [], []
    for stage in sched:
        assert len(stage) == 1          # one mapping per stage
        for host, layers in stage.items():
            assert len(layers) == 2
            stage_layers.append((int(layers[0]), int(layers[1])))
            if hosts:
                try:
                    stage_ranks.append(hosts.index(host))
                except ValueError:
                    logger.error("Scheduling: host not found in hosts list: %s", host)
                    raise
            else:
                try:
                    stage_ranks.append(int(host))
                except ValueError:
                    logger.error("Scheduling: 'hosts' not specified, failed to parse as rank: %s", host)
                    raise
    return stage_layers, stage_ranks


def load_yaml_sched(model_name: str, microbatch_size: int, sched_file: Optional[str], s_models_file: Optional[str],
                    s_dev_types_file: Optional[str], s_dev_file: Optional[str]) -> List[dict]:
    """The scheduler's output: read from `sched_file` (what `sched-pipeline` printed), or produced now by the
    reference's `sched-pipeline` binary if it is on PATH (same arguments as `sched/scheduler.py:24-70`; the
    scheduler itself is CPU planning code outside this build's scope and is not rebuilt here)."""
    import subprocess   # pylint: disable=import-outside-toplevel
    import yaml         # pylint: disable=import-outside-toplevel
    if sched_file:
        with open(sched_file, encoding='utf-8') as fh:
            return yaml.safe_load(fh)
    args = ['sched-pipeline', '-i', '2', '-o', '2', '-b', str(microbatch_size), '-d', 'torch.float32', '-m', model_name]
    for flag, val in (('-M', s_models_file), ('-T', s_dev_types_file), ('-D', s_dev_file)):
        if val:
            args += [flag, val]
    try:
        proc = subprocess.run(args, capture_output=True, check=True)
    except FileNotFoundError as exc:
        raise RuntimeError("Automated scheduling needs the reference's `sched-pipeline` on PATH (not built here): "
                           "pass its output with --sched-file, or a partition with -pt") from exc
    return yaml.safe_load(proc.stdout)


def get_pipeline_sched(world_size: int, partition: Optional[List[Tuple[int, int]]], quant: Optional[List[int]],
                       rank_order: Optional[List[int]], model_name: str, hosts: Optional[List[str]] = None,
                       microbatch_size: int = 8, sched_file: Optional[str] = None, s_models_file: Optional[str] = None,
                       s_dev_types_file: Optional[str] = None, s_dev_file: Optional[str] = None) \
        -> Tuple[List[Tuple[int, int]], List[int], List[int]]:
    """Get the pipeline schedule: `stage_layers`, `stage_quant`, `stage_ranks` (`runtime.py:291-355`)."""
    if partition:
        stage_layers = partition
        stage_quant = quant if quant else [0] * len(stage_layers)
        stage_ranks = rank_order if rank_order else list(range(len(stage_layers)))
    elif quant:
        raise RuntimeError("Must specify partition with quantization")
    elif rank_order:
        raise RuntimeError("Must specify partition with rank stage ordering")
    elif world_size <= 1:
        stage_layers = [(1, model_cfg.get_model_layers(model_name))]
        stage_quant = [0]
        stage_ranks = [0]
    else:
        # the scheduler's YAML (`runtime.py:334-351`): hosts must cover the world, no quantization for automated schedules
        if hosts and len(hosts) != world_size:
            raise RuntimeError("Specified hosts count != world size")
        sched = load_yaml_sched(model_name, microbatch_size, sched_file, s_models_file, s_dev_types_file, s_dev_file)
        stage_layers, stage_ranks = parse_yaml_sched(sched, hosts)
        stage_quant = [0] * len(stage_layers)
    logger.info("Scheduling: stage-to-layer mapping: %s", stage_layers)
    logger.info("Scheduling: stage output quantization: %s", stage_quant)
    logger.info("Scheduling: stage-to-rank mapping: %s", stage_ranks)
    return stage_layers, stage_quant, stage_ranks


def load_dataset(model_name: str, batch_size: int, ubatch_size: int) -> Dataset:
    """Synthetic inputs in place of the reference's downloaded image / `bert_input.npz` (`runtime.py:386-400`)."""
    spec = MODEL_SPECS[model_name]
    inputs = synth_input(spec, ubatch_size, seed=1)
    labels = torch.zeros(ubatch_size, dtype=torch.int64)
    return RolloverTensorDataset(batch_size, inputs, labels)


def resolve_weights(model_name: str, model_file: Optional[str]):
    """`-M` npz path if it exists, else seeded synthetic weights in the same layout (no network here)."""
    path = model_file or model_cfg.get_model_default_weights_file(model_name)
    if os.path.exists(path):
        return path
    logger.warning("weights file %s not found: using seeded synthetic weights", path)
    return synth_weights(MODEL_SPECS[model_name], seed=0)


sched_q = queue.Queue()
stop_event = threading.Event()


def handle_cmd(cmd: int, tensors: Tuple[torch.Tensor, ...]) -> None:
    """Process received commands (`runtime.py:406-415`)."""
    if cmd == CMD_STOP:
        logger.info("handle_cmd: stop")
        stop_event.set()
    elif cmd == CMD_SCHED:
        logger.info("handle_cmd: sched")
        sched_q.put(tuple(t.tolist() for t in tensors))
    else:
        logger.warning("handle_cmd: Unknown command: %s", cmd)


def run_pipeline_p2p(world_size: int, rank: int, model_name: str, model_file: Optional[str], batch_size: int,
                     ubatch_size: int, partition: Optional[List[Tuple[int, int]]], quant: Optional[List[int]],
                     rank_order: Optional[List[int]], data_rank: int, hosts: Optional[List[str]] = None,
                     sched_args: Optional[dict] = None) -> float:
    """Run the pipeline using P2P communication (`runtime.py:418-511`); returns throughput on the data rank."""
    throughput = 0.0
    monitoring.init(MONITORING_KEY_SEND, get_window_size(), work_type='Mbits')
    if os.getenv(ENV_MONITORING, '0') == '1':
        enable_monitoring()
    with DistP2pContext(('gloo',), {'world_size': world_size, 'rank': rank}, handle_cmd) as dist_ctx:
        if rank == 0:
            stage_layers, stage_quant, stage_ranks = get_pipeline_sched(world_size, partition, quant, rank_order,
                                                                        model_name, hosts=hosts,
                                                                        microbatch_size=ubatch_size, **(sched_args or {}))
            dist_ctx.cmd_broadcast(CMD_SCHED, (torch.tensor(stage_layers), torch.tensor(stage_quant),
                                               torch.tensor(stage_ranks), torch.tensor(data_rank)))
        else:
            stage_layers, stage_quant, stage_ranks, data_rank = sched_q.get()
        try:
            stage = stage_ranks.index(rank)
        except ValueError:
            stage = None
        check_host_only_role(stage)
        if stage is None:
            model = None
        else:
            weights = resolve_weights(model_name, model_file)
            shard_cls = model_cfg.get_model_dict(model_name)['shard_module']
            if isinstance(weights, str):
                model = model_cfg.module_shard_factory(model_name, weights, stage_layers[stage][0],
                                                       stage_layers[stage][1], stage)
            else:
                cfg = models.ModuleShardConfig(layer_start=stage_layers[stage][0], layer_end=stage_layers[stage][1],
                                               is_first=stage_layers[stage][0] == 1,
                                               is_last=stage_layers[stage][1] == model_cfg.get_model_layers(model_name))
                model = shard_cls(model_cfg.get_model_config(model_name), cfg, weights)
            model.use_cuda_graph = True
            model.register_buffer('quant_bit', torch.tensor(stage_quant[stage]), persistent=False)
            send_constraint = float(os.getenv(ENV_SEND_CONSTRAINT, str(0)))
            model.register_buffer('rate_constraint', torch.tensor(send_constraint), persistent=False)
            model.register_forward_hook(devices.forward_hook_to_cpu)
            model.register_forward_hook(forward_hook_monitor)
            if stage != len(stage_ranks) - 1:
                quant_impl = os.getenv(ENV_ADAPTIVE_QUANT)
                if quant_impl == ADAPTIVE_QUANT_CONTROLLER:
                    model.register_forward_hook(forward_hook_set_quant_controller)
                elif quant_impl == ADAPTIVE_QUANT_HEURISTIC:
                    model.register_forward_hook(forward_hook_set_quant_bandwidth_heuristic)
                elif quant_impl == ADAPTIVE_QUANT_HEURISTIC2:
                    model.register_forward_hook(forward_hook_set_quant_bandwidth_heuristic_2)
                model.register_forward_hook(forward_hook_quant_encode)
            if stage != 0:
                model.register_forward_pre_hook(forward_pre_hook_quant_decode)
            model.register_forward_pre_hook(forward_pre_hook_monitor)
            model.register_forward_pre_hook(devices.forward_pre_hook_to_device)
        with model_cfg.dist_p2p_pipeline_stage_factory(stage_ranks, data_rank, rank, stage, model,
                                                       handle_results) as stage_ctx:
            if model is not None:
                logger.info("Pipeline stage: %s", 'native' if stage_ctx.native is not None else 'Python threads')
            elif rank == data_rank:   # outside the stage pipeline: it feeds the first stage and collects results
                kind = 'Python threads' if stage_ctx.native is None else \
                    'native (host)' if not torch.cuda.is_available() else 'native'
                logger.info("Data rank: %s", kind)
            if os.getenv(ENV_ADAPTIVE_QUANT) or monitoring_enabled():
                stage_ctx.register_send_timing_hook(hop_timing_hook_monitor, (MONITORING_KEY_SEND,))
            if rank == data_rank:
                dataset = load_dataset(model_name, batch_size, ubatch_size)
                data_loader = DataLoader(dataset, batch_size=ubatch_size)
                tik_data = time.time()
                start_count = results_counter.value
                for ubatch, ubatch_labels in data_loader:
                    label_queue.put(ubatch_labels)
                    stage_ctx.enqueue_tensor(ubatch)
                while not results_counter.wait_gte(start_count + len(dataset), timeout=1.0):
                    stage_ctx.check_workers()
                latency = time.time() - tik_data
                throughput = batch_size / latency
                logger.info("Latency is %f, throughput is %f", latency, throughput)
                dist_ctx.cmd_broadcast(CMD_STOP)
                stop_event.set()
            else:
                stop_event.wait()
    disable_monitoring()
    monitoring.finish()
    return throughput


def check_host_only_role(stage: Optional[int]) -> None:
    """A rank without a CUDA device (`-d cpu`, or no visible GPU) may load data outside the stage pipeline or stay idle,
    as in the reference; a stage needs the GPU."""
    if stage is not None and not torch.cuda.is_available():
        raise RuntimeError(f"runtime.py: no CUDA device for stage {stage} - this build has no CPU fallback")


def init_env(device: Optional[str], net_addr: str, net_port: int, net_ifname: str) -> None:
    """Initialize the PyTorch environment (`runtime.py:581-602`). The compute device is CUDA, except on a rank with
    `-d cpu` or without a visible GPU: that rank is host-only (`devices.DEVICE` is the CPU) and never creates a CUDA
    context; with `-d cpu` every GPU is hidden from the process, so that no library can create one either."""
    if device is not None and torch.device(device).type == 'cpu':
        os.environ['CUDA_VISIBLE_DEVICES'] = ''
        devices.DEVICE = torch.device('cpu')
    elif not torch.cuda.is_available():
        devices.DEVICE = torch.device('cpu')
    else:
        if device is None or device == 'cuda':
            device = f"cuda:{int(os.environ.get('LOCAL_RANK', '0')) % torch.cuda.device_count()}"
        devices.DEVICE = torch.device(device)
        if devices.DEVICE.type != 'cuda':
            raise RuntimeError(f"runtime.py: device {device} is neither a CUDA device nor the CPU")
        torch.cuda.set_device(devices.DEVICE)
    os.environ['MASTER_ADDR'] = net_addr
    os.environ['MASTER_PORT'] = str(net_port)
    if net_ifname:
        os.environ["GLOO_SOCKET_IFNAME"] = net_ifname


def main() -> None:
    """Main function (`runtime.py:605-730`)."""
    parser = argparse.ArgumentParser(description="Pipeline Parallelism Runtime",
                                     formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("rank", type=int, help="the rank for the current node")
    parser.add_argument("worldsize", type=int, help="the world size (the number of nodes)")
    parser.add_argument("-d", "--device", type=str, default=None,
                        help="compute device, e.g.: 'cuda', 'cuda:1' (default: cuda:LOCAL_RANK or cuda:rank); 'cpu' only for a "
                             "data rank outside the stage pipeline or an idle rank")
    parser.add_argument("-s", "--socket-ifname", type=str, default="lo", help="socket interface name")
    parser.add_argument("--addr", type=str, default="127.0.0.1", help="ip address for the master node")
    parser.add_argument("--port", type=int, default=29500, help="communication port for the master node")
    parser.add_argument("-c", "--comm", type=str, default="p2p", choices=["p2p"],
                        help="the communication implementation (rpc is outside this build's scope)")
    parser.add_argument("-m", "--model-name", type=str, default="google/vit-base-patch16-224",
                        choices=model_cfg.get_model_names(), help="the neural network model for loading")
    parser.add_argument("-M", "--model-file", type=str, help="the model file, if not in working directory")
    parser.add_argument("-b", "--batch-size", default=64, type=int, help="batch size")
    parser.add_argument("-u", "--ubatch-size", default=8, type=int, help="microbatch size")
    usched = parser.add_argument_group('User-defined scheduling')
    usched.add_argument("-pt", "--partition", type=str,
                        help="comma-delimited list of start/end layer pairs, e.g.: '1,24,25,48'; "
                             "single-node default: all layers in the model")
    usched.add_argument("-q", "--quant", type=str,
                        help="comma-delimited list of quantization bits to use after each stage")
    usched.add_argument("-r", "--rank-order", type=str, default=None,
                        help="comma-delimited list of ranks in desired stage order; default: natural rank order")
    parser.add_argument("-H", "--hosts", type=str,
                        help="comma-delimited list of hosts in rank order; required for automated scheduling")
    asched = parser.add_argument_group('Automated scheduling')
    asched.add_argument("--sched-file", type=str,
                        help="YAML printed by the reference's sched-pipeline (list of `host: [start, end]` maps)")
    asched.add_argument("-sm", "--sched-models-file", default=None, type=str, help="models YAML file for sched-pipeline")
    asched.add_argument("-sdt", "--sched-dev-types-file", default=None, type=str, help="device types YAML file")
    asched.add_argument("-sd", "--sched-dev-file", default=None, type=str, help="devices YAML file")
    usched.add_argument("-D", "--data-rank", type=int, default=0,
                        help="rank where inputs are loaded and outputs are processed - must be "
                             "the same as stage=0 or not in the stage pipeline")
    args = parser.parse_args()

    if args.partition is None:
        partition = None
    else:
        parts = [int(i) for i in args.partition.split(',')]
        assert len(parts) % 2 == 0
        partition = [(parts[i], parts[i + 1]) for i in range(0, len(parts), 2)]
    quant = None if args.quant is None else [int(i) for i in args.quant.split(',')]
    rank_order = None if args.rank_order is None else [int(i) for i in args.rank_order.split(',')]

    tik = time.time()
    device = args.device
    if device is None and 'LOCAL_RANK' not in os.environ:
        device = f"cuda:{args.rank % max(1, torch.cuda.device_count())}"
    init_env(device, args.addr, args.port, args.socket_ifname if args.socket_ifname != 'lo0' else '')
    logger.info("Device: %s", devices.DEVICE)
    hosts = args.hosts.split(',') if args.hosts else None
    run_pipeline_p2p(args.worldsize, args.rank, args.model_name, args.model_file, args.batch_size,
                     args.ubatch_size, partition, quant, rank_order, args.data_rank, hosts=hosts,
                     sched_args={'sched_file': args.sched_file, 's_models_file': args.sched_models_file,
                                 's_dev_types_file': args.sched_dev_types_file, 's_dev_file': args.sched_dev_file})
    logger.info("Total program execution time = %f", time.time() - tik)


if __name__ == "__main__":
    logging.basicConfig(filename='runtime.log', level=logging.DEBUG)
    console_hndlr = logging.StreamHandler(sys.stdout)
    console_hndlr.setFormatter(logging.Formatter(fmt='%(message)s'))
    console_hndlr.setLevel(logging.INFO)
    logging.getLogger().addHandler(console_hndlr)
    main()
    from pipeedge_b200.comm import p2p as _p2p
    if torch.cuda.is_available() and _p2p.nccl_hops_opened():
        # Python-thread path only: everything is shut down, but the exit-time teardown of the CUDA / NCCL libraries can
        # crash after a clean multi-rank run with per-hop communicators. The native pipeline owns no communicator and
        # leaves through the normal interpreter exit (destroy graphs / events -> links -> process group, in that order).
        logging.shutdown()
        sys.stdout.flush()
        sys.stderr.flush()
        os._exit(0)
