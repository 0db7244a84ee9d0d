"""Entries of the scheduler's YAML files, checked for the types `sched-pipeline` expects."""
from typing import List, Optional, Sequence, Union

Number = Union[int, float]


def _check_list(values, types, what: str) -> None:
    if not isinstance(values, list) or not all(isinstance(v, types) for v in values):
        raise TypeError(f"{what} must be a list of {types}, got {values!r}")


def _check(value, types, what: str) -> None:
    if not isinstance(value, types):
        raise TypeError(f"{what} must be {types}, got {value!r}")


def yaml_model(num_layers: int, parameters_in: int, parameters_out: List[int], mem_MB: Sequence[Number]) -> dict:
    """A models-file entry: the layer count, the first layer's input elements per item, and per layer its output
    elements per item and its memory (MB)."""
    _check(num_layers, int, 'num_layers')
    _check(parameters_in, int, 'parameters_in')
    _check_list(parameters_out, int, 'parameters_out')
    _check_list(mem_MB, (int, float), 'mem_MB')
    return {'layers': num_layers, 'parameters_in': parameters_in, 'parameters_out': parameters_out, 'mem_MB': mem_MB}


def yaml_model_profile(dtype: str, batch_size: int, time_s: Sequence[Number]) -> dict:
    """One timing profile of a model on a device type; `sched-pipeline` finds it by (dtype, batch_size)."""
    _check(dtype, str, 'dtype')
    _check(batch_size, int, 'batch_size')
    _check_list(time_s, (int, float), 'time_s')
    return {'dtype': dtype, 'batch_size': batch_size, 'time_s': time_s}


def yaml_device_type(mem_MB: Number, bw_Mbps: Number, model_profiles: Optional[dict]) -> dict:
    """A device-types-file entry: memory, bandwidth and model name -> list of `yaml_model_profile`."""
    _check(mem_MB, (int, float), 'mem_MB')
    _check(bw_Mbps, (int, float), 'bw_Mbps')
    model_profiles = {} if model_profiles is None else model_profiles
    _check(model_profiles, dict, 'model_profiles')
    return {'mem_MB': mem_MB, 'bw_Mbps': bw_Mbps, 'model_profiles': model_profiles}
