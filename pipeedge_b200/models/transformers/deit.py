"""DeiT shards on H100 - drop-in for `pipeedge.models.transformers.deit` (reference `deit.py`).

DeiT blocks are ViT blocks (`deit.py:27-69` copies `ViTLayerShard`); what differs is the timm `.npz` key
layout (`deit.py:119-156`), the extra distillation token (S = 198) and that only the `head` classifier is used
(`deit.py:215-218`). As in the reference, the distillation token is never loaded and stays zero
(`deit.py:119-124` vs HF `DeiTEmbeddings`).
"""
from collections.abc import Mapping
import numpy as np
from .vit import ViTModelShard, ViTShardForImageClassification


class DeiTModelShard(ViTModelShard):
    """Module shard based on `DeiTModel` (reference `deit.py:72-167`)."""
    FAMILY = 'deit'
    N_PREFIX = 2   # [CLS], [DIST]

    def _npz_first(self, weights: Mapping) -> dict:
        pos = np.asarray(weights["pos_embed"])[0]
        cls = np.asarray(weights["cls_token"]).reshape(1, -1)
        prefix = np.concatenate([cls + pos[:1], pos[1:2]], axis=0)   # zero distillation token + its position
        return {'conv': weights["patch_embed.proj.weight"], 'bias': weights["patch_embed.proj.bias"], 'pos': pos,
                'prefix': prefix}

    def _npz_last(self, weights: Mapping) -> dict:
        return {'ln_w': weights["norm.weight"], 'ln_b': weights["norm.bias"]}

    @staticmethod
    def save_weights(model_name: str, model_file: str, hub_repo: str = 'facebookresearch/deit:main',
                     hub_model_name=None) -> None:
        """The reference pulls the checkpoint from torch.hub (`deit.py:170-187`); this build has no network."""
        raise RuntimeError(f"cannot download weights for {model_name}: no network. Provide {model_file} in the "
                           "reference npz layout (pipeedge_b200.synth writes synthetic ones).")


class DeiTShardForImageClassification(ViTShardForImageClassification):
    """Module shard based on `DeiTForImageClassification` (reference `deit.py:190-233`)."""
    FAMILY = 'deit'
    _INNER = DeiTModelShard
    _HEAD_KEYS = ("head.weight", "head.bias", False)

    @property
    def deit(self):
        """The inner model shard under the reference's attribute name."""
        return self.vit

    @staticmethod
    def save_weights(model_name: str, model_file: str, hub_repo: str = 'facebookresearch/deit:main',
                     hub_model_name=None) -> None:
        """See `DeiTModelShard.save_weights`."""
        DeiTModelShard.save_weights(model_name, model_file, hub_repo=hub_repo, hub_model_name=hub_model_name)
