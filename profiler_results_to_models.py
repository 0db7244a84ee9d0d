"""Turn a profiler results file into an entry of the scheduler's models YAML file (extended if it exists).

`python profiler_results_to_models.py -i profiler_results.yml -o models.yml [-f]`: the entry holds the layer count,
the first layer's input elements per item, each layer's output elements per item and its memory in MB. An existing
entry for the model is replaced only with `-f`. Exits with status 1 when nothing was written.
"""
import argparse
import sys
import numpy as np
import yaml
import model_cfg
from pipeedge_b200.sched import yaml_files, yaml_types


def _elements(shapes) -> int:
    """Elements per item of a layer's payload (a list of tensor shapes without the batch dimension)."""
    return int(sum(np.prod(shape) for shape in shapes))


def check_layers(model_name: str, layers: int, profile_data: list) -> bool:
    """Warn when `layers` differs from the registry's count; False when the profile does not hold every layer."""
    if model_name in model_cfg.get_model_names():
        expected = model_cfg.get_model_layers(model_name)
        if layers != expected:
            print(f"Warning: expected and actual layer counts differ: {expected} != {layers}")
    else:
        print(f"Warning: cannot verify layer count for unknown model: {model_name}: {layers}")
    if layers != len(profile_data):
        print(f"Declared layer count does not match profile data count: {layers} != {len(profile_data)}")
        return False
    return True


def save_models_yml(file: str, model_name: str, num_layers: int, parameters_in: int, parameters_out, mem,
                    overwrite_model: bool = False) -> bool:
    """Add (or with `overwrite_model` replace) `model_name` in the models file `file`; False if it is already there."""
    models = yaml_files.yaml_models_load(file)
    if model_name in models:
        if not overwrite_model:
            print(f"Model already exists: {file}: {model_name}: {models[model_name]}")
            return False
        print(f"Overwriting existing model: {file}: {model_name}: {models[model_name]}")
    models[model_name] = yaml_types.yaml_model(num_layers, parameters_in, parameters_out, mem)
    yaml_files.yaml_save(models, file)
    return True


def main() -> None:
    """Main function."""
    parser = argparse.ArgumentParser(description="Produce scheduler-compatible models YAML file from profiling results",
                                     formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("-i", "--results-yml", type=str, default="profiler_results.yml",
                        help="profiler results input YAML file")
    parser.add_argument("-o", "--models-yml", type=str, default="models.yml", help="models output YAML file")
    parser.add_argument("-f", "--overwrite", action='store_true', help="overwrite existing YAML model entries")
    args = parser.parse_args()

    with open(args.results_yml, 'r', encoding='utf-8') as yfile:
        results = yaml.safe_load(yfile)
    layers, model_name, profile_data = results['layers'], results['model_name'], results['profile_data']
    if not check_layers(model_name, layers, profile_data):
        sys.exit(1)
    if not profile_data:
        print("Empty profile data!")
        sys.exit(1)
    parameters_in = _elements(profile_data[0]['shape_in'])
    parameters_out = [_elements(r['shape_out']) for r in profile_data]
    mem = [r['memory'] for r in profile_data]
    if not save_models_yml(args.models_yml, model_name, layers, parameters_in, parameters_out, mem,
                           overwrite_model=args.overwrite):
        sys.exit(1)


if __name__ == "__main__":
    main()
