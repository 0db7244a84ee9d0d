"""Model configurations and default parameters - drop-in for the reference `model_cfg.py`.

Same registry names, layer counts and default weight-file names (`model_cfg.py:23-43`); the `shard_module`
entries point at the native shard classes, and `get_model_config` builds the HuggingFace config from the
architecture table in `pipeedge_b200.synth` instead of `AutoConfig.from_pretrained` (no network).
"""
import logging
from typing import Any, Callable, List, Optional, Tuple, Union
import torch
from pipeedge_b200.comm import p2p
from pipeedge_b200.models import ModuleShard, ModuleShardConfig
from pipeedge_b200.models.transformers import bert, deit, vit
from pipeedge_b200.synth import MODEL_SPECS, hf_config
import devices

_logger = logging.getLogger(__name__)

_MODEL_CONFIGS = {}


def _model_cfg_add(name, layers, weights_file, shard_module):
    _MODEL_CONFIGS[name] = {'name': name, 'layers': layers, 'weights_file': weights_file,
                            'shard_module': shard_module}


# Transformer blocks can be split 4 ways: ViT-Base has 12 blocks = 48 schedulable sub-layers
_model_cfg_add('google/vit-base-patch16-224', 48, 'ViT-B_16-224.npz', vit.ViTShardForImageClassification)
_model_cfg_add('google/vit-large-patch16-224', 96, 'ViT-L_16-224.npz', vit.ViTShardForImageClassification)
_model_cfg_add('google/vit-huge-patch14-224-in21k', 128, 'ViT-H_14.npz', vit.ViTShardForImageClassification)
_model_cfg_add('bert-base-uncased', 48, 'BERT-B.npz', bert.BertModelShard)
_model_cfg_add('bert-large-uncased', 96, 'BERT-L.npz', bert.BertModelShard)
_model_cfg_add('textattack/bert-base-uncased-CoLA', 48, 'BERT-B-CoLA.npz', bert.BertShardForSequenceClassification)
_model_cfg_add('facebook/deit-base-distilled-patch16-224', 48, 'DeiT_B_distilled.npz',
               deit.DeiTShardForImageClassification)
_model_cfg_add('facebook/deit-small-distilled-patch16-224', 48, 'DeiT_S_distilled.npz',
               deit.DeiTShardForImageClassification)
_model_cfg_add('facebook/deit-tiny-distilled-patch16-224', 48, 'DeiT_T_distilled.npz',
               deit.DeiTShardForImageClassification)


def get_model_names() -> List[str]:
    """Get a list of available model names."""
    return list(_MODEL_CONFIGS.keys())


def get_model_dict(model_name: str) -> dict:
    """Get a model's key/value properties - modify at your own risk."""
    return _MODEL_CONFIGS[model_name]


def get_model_layers(model_name: str) -> int:
    """Get a model's layer count."""
    return _MODEL_CONFIGS[model_name]['layers']


def get_model_config(model_name: str) -> Any:
    """Get a model's HuggingFace config (built locally; the reference calls `AutoConfig.from_pretrained`)."""
    return hf_config(MODEL_SPECS[model_name])


def get_model_default_weights_file(model_name: str) -> str:
    """Get a model's default weights file name."""
    return _MODEL_CONFIGS[model_name]['weights_file']


def save_model_weights_file(model_name: str, model_file: Optional[str] = None) -> None:
    """Save a model's weights file (`model_cfg.py:72-78`); needs the network in the reference."""
    if model_file is None:
        model_file = get_model_default_weights_file(model_name)
    _MODEL_CONFIGS[model_name]['shard_module'].save_weights(model_name, model_file)


def module_shard_factory(model_name: str, model_file: Optional[str], layer_start: int, layer_end: int,
                         stage: int) -> ModuleShard:
    """Get a shard instance on the current CUDA device (`model_cfg.py:80-95`)."""
    if model_file is None:
        model_file = get_model_default_weights_file(model_name)
    config = get_model_config(model_name)
    shard_config = ModuleShardConfig(layer_start=layer_start, layer_end=layer_end, is_first=layer_start == 1,
                                     is_last=layer_end == get_model_layers(model_name))
    module = _MODEL_CONFIGS[model_name]['shard_module']
    if devices.DEVICE is not None and torch.device(devices.DEVICE).type == 'cuda' and \
            torch.device(devices.DEVICE).index is not None:
        torch.cuda.set_device(torch.device(devices.DEVICE))
    shard = module(config, shard_config, model_file)
    _logger.info("======= %s Stage %d =======", module.__name__, stage)
    shard.to(device=devices.DEVICE)
    return shard


def replica_neighbours(replica_ranks: List[List[int]], data_rank: int, rank: int) \
        -> Tuple[Optional[int], Optional[int], Optional[int], Optional[int]]:
    """(replica, stage, rank_src, rank_dst) of `rank` among R replicas of one stage pipeline (`replica_ranks[k][s]`:
    replica k's stage s) fed by `data_rank` outside them: its neighbours are those of its own replica, and the data rank
    is the source of every replica's first stage and the destination of every last one. All None for the data rank and
    for an idle rank."""
    for replica, ranks in enumerate(replica_ranks):
        if rank in ranks:
            stage = ranks.index(rank)
            rank_src = data_rank if stage == 0 else ranks[stage - 1]
            rank_dst = data_rank if stage == len(ranks) - 1 else ranks[stage + 1]
            return replica, stage, rank_src, rank_dst
    return None, None, None, None


def dist_p2p_pipeline_stage_factory(stage_ranks: Union[List[int], List[List[int]]], data_rank: int, rank: int,
                                    stage: Optional[int], module: Optional[ModuleShard],
                                    handle_results_cb: Callable[[Any], None]) -> p2p.DistP2pPipelineStage:
    """Get a P2P pipeline stage instance with the reference's rank topology (`model_cfg.py:128-166`). `stage_ranks` may
    also be one list of ranks per replica of the stage pipeline (`runtime.py --replicas`, no reference equivalent): the
    data rank, outside every replica, then feeds all of them (`replica_neighbours`)."""
    if stage_ranks and isinstance(stage_ranks[0], (list, tuple)):
        if rank == data_rank:
            assert handle_results_cb is not None
            if stage is not None:
                raise ValueError("Data rank must be outside every replica of the stage pipeline")
            return p2p.DistP2pPipelineStage([ranks[-1] for ranks in stage_ranks], [ranks[0] for ranks in stage_ranks],
                                            None, handle_results_cb)
        _, own_stage, rank_src, rank_dst = replica_neighbours(stage_ranks, data_rank, rank)
        if stage != own_stage:
            raise ValueError(f"rank {rank} is stage {own_stage} of its replica, not stage {stage}")
        return p2p.DistP2pPipelineStage(rank_src, rank_dst, module if stage is not None else None, None)
    n_stages = len(stage_ranks)
    if rank == data_rank:
        assert handle_results_cb is not None
        results_cb = handle_results_cb
        if stage is None:          # data rank outside the pipeline: feeds stage 0, collects from the last stage
            rank_src, rank_dst, work_cb = stage_ranks[-1], stage_ranks[0], None
        else:                      # data rank inside the pipeline must be its first stage
            if stage != 0:
                raise ValueError(f"Data rank must be stage=0 or stage=None, but stage={stage}")
            rank_src = stage_ranks[-1] if n_stages > 1 else None
            rank_dst = stage_ranks[1] if n_stages > 1 else None
            work_cb = module
    elif stage is None:            # idle rank
        rank_src = rank_dst = work_cb = results_cb = None
    else:
        rank_src = data_rank if stage == 0 else stage_ranks[stage - 1]
        rank_dst = data_rank if stage == n_stages - 1 else stage_ranks[stage + 1]
        work_cb, results_cb = module, None
    return p2p.DistP2pPipelineStage(rank_src, rank_dst, work_cb, results_cb)
