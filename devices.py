"""Common device configuration - same module surface as the reference `devices.py`.

On the native GPU path activations never leave the GPU between the shard and the hop, so the two hooks the
reference installs around every shard forward (`devices.py:8-24`: H2D before, D2H after) are identities:
host inputs of the data rank are staged by the shard itself on a copy stream (see
`pipeedge_b200/models/transformers/_shard.py`), and there is no CPU fallback to move results to.
"""
from typing import Tuple, Union
import torch

# The torch.device to use for computation (set by `runtime.init_env`)
DEVICE = None


def forward_pre_hook_to_device(_module, inputs) -> Union[Tuple[torch.Tensor], Tuple[Tuple[torch.Tensor]]]:
    """Reference: move tensors to the compute device. Here: identity (the shard stages host inputs itself)."""
    return inputs


def forward_hook_to_cpu(_module, _inputs, outputs) -> Union[torch.Tensor, Tuple[torch.Tensor]]:
    """Reference: move tensors to the CPU. Here: identity (payloads stay in HBM for the NCCL hop)."""
    return outputs


# identities on every path, so the native pipeline may ignore them (see comm/p2p/_native.py: hook_is_native)
forward_pre_hook_to_device._pe_native = True   # pylint: disable=protected-access
forward_hook_to_cpu._pe_native = True          # pylint: disable=protected-access
