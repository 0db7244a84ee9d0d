"""The scheduler's YAML files: the models and device-types files that `profiler_results_to_models.py` and
`profiler_results_to_device_types.py` write and the reference's `sched-pipeline` reads (reference package
`pipeedge.sched`). The partitioner itself is not part of this build."""
