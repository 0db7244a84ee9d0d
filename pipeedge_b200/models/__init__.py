"""Model shard base types - same public names and semantics as the reference `pipeedge.models`
(`src/pipeedge/models/__init__.py:1-49`), so reference callers (`runtime.py`, `model_cfg.py`) work
unchanged against the native shards."""
from typing import Any, Tuple, Type, Union
from torch import nn, Tensor

ModuleShardData: Type = Union[Tensor, Tuple[Tensor, ...]]
"""A module shard input/output type."""


class ModuleShardConfig:
    """Shard (not model) configuration: `layer_start`/`layer_end` are 1-based inclusive sub-layer ids,
    `is_first`/`is_last` say whether the shard owns the embeddings / the head. Extra keyword arguments
    become attributes, as in the reference (`models/__init__.py:9-22`)."""
    # pylint: disable=too-few-public-methods

    def __init__(self, **kwargs: Any):
        defaults = {'layer_start': 0, 'layer_end': 0, 'is_first': False, 'is_last': False}
        defaults.update(kwargs)
        for key, value in defaults.items():
            setattr(self, key, value)


class ModuleShard(nn.Module):
    """Abstract parent class for module shards (`models/__init__.py:25-36`)."""
    # pylint: disable=abstract-method

    def __init__(self, config: Any, shard_config: ModuleShardConfig):
        super().__init__()
        self.config = config
        self.shard_config = shard_config

    def has_layer(self, layer: int) -> bool:
        """Whether `layer` lies in the shard's inclusive sub-layer range."""
        return self.shard_config.layer_start <= layer <= self.shard_config.layer_end


def get_microbatch_size(shard_data: ModuleShardData, verify: bool = False) -> int:
    """Micro-batch size = length of the outer dim of the (first) tensor (`models/__init__.py:39-49`)."""
    tensors = (shard_data,) if isinstance(shard_data, Tensor) else tuple(shard_data)
    if not tensors:
        return 0
    size = len(tensors[0])
    if verify:
        for tensor in tensors:
            assert isinstance(tensor, Tensor)
            assert len(tensor) == size
    return size
