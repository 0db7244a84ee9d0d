"""ViT shards on H100 - drop-in for `pipeedge.models.transformers.vit` (reference `vit.py`).

Same class names, constructor and `forward` contract; the arithmetic (HF `ViTEmbeddings`, `ViTSelfAttention`,
`ViTSelfOutput`, `ViTIntermediate`, `ViTOutput`, `nn.LayerNorm`, the classifier `nn.Linear`) runs as the
sm_90a kernels of `libpipeedge_b200.so`. Weights are read from the Google/JAX `.npz` layout the reference
loads (`vit.py:120-159,216-218`).
"""
from collections.abc import Mapping
import numpy as np
import torch
from ... import ops
from ..._lib import LIB, check
from .. import ModuleShardConfig
from . import TransformerShardData
from ._shard import GpuTransformerShard


class ViTModelShard(GpuTransformerShard):
    """Module shard based on `ViTModel` without pooling (reference `vit.py:73-170`)."""
    FAMILY = 'vit'
    N_PREFIX = 1   # [CLS]

    def _npz_first(self, weights: Mapping) -> dict:
        """Embedding tensors in canonical form: conv weight [H, C, P, P], bias, pos [S, H], prefix rows."""
        conv = np.transpose(np.asarray(weights["embedding/kernel"]), [3, 2, 0, 1])   # vit.py:125-128
        pos = np.asarray(weights["Transformer/posembed_input/pos_embedding"])[0]
        cls = np.asarray(weights["cls"]).reshape(1, -1)
        return {'conv': conv, 'bias': weights["embedding/bias"], 'pos': pos, 'prefix': cls + pos[:1]}

    def _npz_last(self, weights: Mapping) -> dict:
        return {'ln_w': weights["Transformer/encoder_norm/scale"], 'ln_b': weights["Transformer/encoder_norm/bias"]}

    def _build_shard(self, weights: Mapping) -> None:
        cfg = self.config
        n_patches = (cfg.image_size // cfg.patch_size) ** 2
        self.tokens = n_patches + self.N_PREFIX
        self.stage = self._make_stage(weights, self.tokens)
        dev = self.stage.device
        if self.shard_config.is_first:
            first = self._npz_first(weights)
            hidden = cfg.hidden_size
            kdim = cfg.num_channels * cfg.patch_size ** 2
            self._kpad = (kdim + 7) // 8 * 8
            conv = np.zeros((hidden, self._kpad), dtype=np.float32)
            conv[:, :kdim] = np.asarray(first['conv']).reshape(hidden, kdim)
            self._conv_w = self._f16(conv, dev)
            self._conv_b = self._f32(first['bias'], dev)
            self._pos = self._f32(first['pos'], dev)
            self._prefix = self._f32(first['prefix'], dev)
        if self.shard_config.is_last:
            last = self._npz_last(weights)
            self._ln_w, self._ln_b = self._f32(last['ln_w'], dev), self._f32(last['ln_b'], dev)

    def _embed(self, pixels: torch.Tensor) -> torch.Tensor:
        cfg = self.config
        batch = pixels.shape[0]
        if tuple(pixels.shape[1:]) != (cfg.num_channels, cfg.image_size, cfg.image_size):
            raise ValueError(f"expected pixel_values [B,{cfg.num_channels},{cfg.image_size},{cfg.image_size}], "
                             f"got {tuple(pixels.shape)}")
        n_patches = self.tokens - self.N_PREFIX
        out = (self._ring('embed', (batch, self.tokens, cfg.hidden_size)) if self.persistent else
               torch.empty((batch, self.tokens, cfg.hidden_size), dtype=torch.float32, device=pixels.device))
        work = self._ring('patches', (batch * n_patches, self._kpad), torch.float16) if self.persistent else \
            torch.empty((batch * n_patches, self._kpad), dtype=torch.float16, device=pixels.device)
        check(LIB.pe_patch_embed(pixels.data_ptr(), self._conv_w.data_ptr(), self._conv_b.data_ptr(),
                                 self._pos.data_ptr(), self._prefix.data_ptr(), out.data_ptr(), work.data_ptr(), batch,
                                 cfg.num_channels, cfg.image_size, cfg.patch_size, cfg.hidden_size, self.N_PREFIX,
                                 torch.cuda.current_stream().cuda_stream))
        return out

    def _features(self, data: TransformerShardData, cls_only: bool):
        data = self._to_device(data)
        if self.shard_config.is_first:
            data = self._embed(data)
        data = self._run_blocks(data)
        if self.shard_config.is_last:
            # LayerNorm is per token, so the classification shard normalises only the rows it reads
            rows = self._cls_rows(data) if cls_only else data
            f32, f16 = ops.layernorm(rows, self._ln_w, self._ln_b, self.config.layer_norm_eps,
                                     want_f32=not cls_only, want_f16=cls_only,
                                     out_f32=None if cls_only or not self._static else self._tmp('final_ln', rows.shape),
                                     out_f16=self._tmp('final_ln16', rows.shape, torch.float16)
                                     if cls_only and self._static else None)
            data = f16 if cls_only else f32
        return data

    def _first_input_spec(self, ubatch: int, dim1: int):
        cfg = self.config
        return ((ubatch, cfg.num_channels, cfg.image_size, cfg.image_size), torch.float32)

    def native_result_item_shape(self):
        return (self.tokens, self.config.hidden_size)

    @torch.no_grad()
    def forward(self, data: TransformerShardData) -> TransformerShardData:
        """Compute shard layers (`vit.py:161-170`)."""
        return self._features(data, cls_only=False)

    @staticmethod
    def save_weights(model_name: str, model_file: str, url=None, timeout_sec=None) -> None:
        """The reference downloads the Google checkpoint here (`vit.py:172-186`); this build has no network."""
        raise RuntimeError(f"cannot download weights for {model_name}: no network. Provide {model_file} in the "
                           "reference npz layout (pipeedge_b200.synth writes synthetic ones).")


class ViTShardForImageClassification(GpuTransformerShard):
    """Module shard based on `ViTForImageClassification` (reference `vit.py:189-232`)."""
    FAMILY = 'vit'
    _INNER = ViTModelShard
    _HEAD_KEYS = ("head/kernel", "head/bias", True)   # (weight key, bias key, weight stored [in, out])

    def _build_shard(self, weights: Mapping) -> None:
        self.vit = self._INNER(self.config, self.shard_config, weights)
        self.stage = self.vit.stage
        if self.shard_config.is_last:
            wkey, bkey, transposed = self._HEAD_KEYS
            head = np.asarray(weights[wkey])
            dev = self.stage.device
            self._head_w = self._f16(head.T if transposed else head, dev)
            self._head_b = self._f32(weights[bkey], dev)

    @torch.no_grad()
    def forward(self, data: TransformerShardData) -> TransformerShardData:
        """Compute shard layers; on the last stage `classifier(layernorm(x)[:, 0, :])` (`vit.py:220-226`)."""
        self.vit.use_cuda_graph, self.vit.num_slots = self.use_cuda_graph, self.num_slots
        data = self.vit._features(data, cls_only=True)   # pylint: disable=protected-access
        if self.shard_config.is_last:
            data = self._classify(data, self._head_w, self._head_b)
        return data

    def _inner(self):
        return self.vit

    def _first_input_spec(self, ubatch: int, dim1: int):
        return self.vit._first_input_spec(ubatch, dim1)   # pylint: disable=protected-access

    def native_result_item_shape(self):
        return (int(self.config.num_labels),)

    @staticmethod
    def save_weights(model_name: str, model_file: str, url=None, timeout_sec=None) -> None:
        """See `ViTModelShard.save_weights`."""
        ViTModelShard.save_weights(model_name, model_file, url=url, timeout_sec=timeout_sec)
