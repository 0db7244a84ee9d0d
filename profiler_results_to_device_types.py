"""Turn a profiler results file into a model profile of a device type in the scheduler's device types YAML file
(extended if it exists).

`python profiler_results_to_device_types.py DEV_TYPE -i profiler_results.yml -o device_types.yml -dtm MB -dtb Mbps
[-f]`: a new device type needs its memory (`-dtm`) and bandwidth (`-dtb`); for an existing one they may be left out
but must not differ, because the profiles it already holds depend on them. A model profile is keyed on
(dtype, batch_size) and is replaced only with `-f`. Exits with status 1 when nothing was written.
"""
import argparse
import sys
import yaml
from pipeedge_b200.sched import yaml_files, yaml_types
from profiler_results_to_models import check_layers


def _dev_type_compatible(dev_type: dict, mem, bwdth) -> bool:
    if mem is not None and dev_type['mem_MB'] != mem:
        print(f"Mismatch for existing device type: mem_MB: {dev_type['mem_MB']} != {mem}")
        return False
    if bwdth is not None and dev_type['bw_Mbps'] != bwdth:
        print(f"Mismatch for existing device type: bw_Mbps: {dev_type['bw_Mbps']} != {bwdth}")
        return False
    return True


def save_device_types_yml(file: str, dev_type_name: str, mem, bwdth, model_name: str, dtype: str, batch_size: int,
                          time_s, overwrite_model: bool = False) -> bool:
    """Add the profile `time_s` of `model_name` at (dtype, batch_size) to device type `dev_type_name` in `file`;
    False (nothing written) on a conflicting device type, a missing -dtm/-dtb, or an existing profile without
    `overwrite_model`."""
    device_types = yaml_files.yaml_device_types_load(file)
    if dev_type_name in device_types:
        if not _dev_type_compatible(device_types[dev_type_name], mem, bwdth):
            return False
    elif mem is None:
        print("New device type: must specify memory argument")
        return False
    elif bwdth is None:
        print("New device type: must specify bandwidth argument")
        return False
    else:
        device_types[dev_type_name] = yaml_types.yaml_device_type(mem, bwdth, {})
    dev_type = device_types[dev_type_name]
    if dev_type['model_profiles'] is None:
        dev_type['model_profiles'] = {}
    profiles = dev_type['model_profiles'].setdefault(model_name, [])
    new = yaml_types.yaml_model_profile(dtype, batch_size, time_s)
    for idx, old in enumerate(profiles):
        if old['dtype'] == dtype and old['batch_size'] == batch_size:
            if not overwrite_model:
                print(f"Model profile already exists: {file}: {dev_type_name}: {model_name}: {old}")
                return False
            print(f"Overwriting existing model profile: {file}: {dev_type_name}: {model_name}: {old}")
            profiles[idx] = new
            break
    else:
        profiles.append(new)
    yaml_files.yaml_save(device_types, file)
    return True


def main() -> None:
    """Main function."""
    parser = argparse.ArgumentParser(description="Produce scheduler-compatible device types YAML file from profiling "
                                                 "results",
                                     formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("dev_type", type=str, help="device type name")
    parser.add_argument("-i", "--results-yml", type=str, default="profiler_results.yml",
                        help="profiler results input YAML file")
    parser.add_argument("-o", "--dev-types-yml", type=str, default="device_types.yml",
                        help="device types output YAML file")
    parser.add_argument("-dtm", "--dev-type-mem", type=int,
                        help="memory in MB (required if not already in DEV_TYPES_YML)")
    parser.add_argument("-dtb", "--dev-type-bw", type=int,
                        help="bandwidth in Mbps (required if not already in DEV_TYPES_YML)")
    parser.add_argument("-f", "--overwrite", action='store_true',
                        help="overwrite existing YAML device type model profile entries")
    args = parser.parse_args()

    with open(args.results_yml, 'r', encoding='utf-8') as yfile:
        results = yaml.safe_load(yfile)
    if not check_layers(results['model_name'], results['layers'], results['profile_data']):
        sys.exit(1)
    time_s = [r['time'] for r in results['profile_data']]
    if not save_device_types_yml(args.dev_types_yml, args.dev_type, args.dev_type_mem, args.dev_type_bw,
                                 results['model_name'], results['dtype'], results['batch_size'], time_s,
                                 overwrite_model=args.overwrite):
        sys.exit(1)


if __name__ == "__main__":
    main()
