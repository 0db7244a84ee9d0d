"""Load and save the scheduler's YAML files (each one a map at the top level)."""
import os
import yaml


def _load_map(file: str) -> dict:
    """The map in `file`, or an empty one when the file does not exist yet (the converters extend files)."""
    if not os.path.exists(file):
        return {}
    with open(file, 'r', encoding='utf-8') as yfile:
        return yaml.safe_load(yfile)


def yaml_models_load(file: str) -> dict:
    """A models file: model name -> `yaml_types.yaml_model`."""
    return _load_map(file)


def yaml_device_types_load(file: str) -> dict:
    """A device types file: device type name -> `yaml_types.yaml_device_type`."""
    return _load_map(file)


def yaml_save(yml: dict, file: str) -> None:
    """Write `yml` in the layout `sched-pipeline` reads (block maps, flow-style leaf lists)."""
    with open(file, 'w', encoding='utf-8') as yfile:
        yaml.safe_dump(yml, yfile, default_flow_style=None)
