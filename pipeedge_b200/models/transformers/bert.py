"""BERT shards on H100 - drop-in for `pipeedge.models.transformers.bert` (reference `bert.py`).

Post-LN blocks (`bert.py:41-52`), no attention mask (`bert.py:45`), HF state_dict `.npz` layout
(`bert.py:104-140`; the classification shard strips a `bert.` prefix, `bert.py:191-196`). The reference leaves
dropout live on its layer shards (it never calls `.eval()`); this implementation is the deterministic
inference path (dropout = identity), which is what the oracle and the goldens pin.
"""
from collections.abc import Mapping
import numpy as np
import torch
from ... import _lib, ops
from ..._lib import LIB, check
from . import TransformerShardData
from ._shard import GpuTransformerShard


class BertModelShard(GpuTransformerShard):
    """Module shard based on `BertModel` (reference `bert.py:55-164`)."""
    FAMILY = 'bert'

    def _build_shard(self, weights: Mapping) -> None:
        cfg = self.config
        self.stage = self._make_stage(weights, tokens=128)   # re-sized on the first forward if S differs
        dev = self.stage.device
        if self.shard_config.is_first:
            self._pos_ids = torch.from_numpy(np.asarray(weights["embeddings.position_ids"]).reshape(-1)).to(
                device=dev, dtype=torch.int64)
            self._word = self._f32(weights["embeddings.word_embeddings.weight"], dev)
            self._pos = self._f32(weights["embeddings.position_embeddings.weight"], dev)
            self._type0 = self._f32(np.asarray(weights["embeddings.token_type_embeddings.weight"])[0], dev)
            self._emb_ln_w = self._f32(weights["embeddings.LayerNorm.weight"], dev)
            self._emb_ln_b = self._f32(weights["embeddings.LayerNorm.bias"], dev)
        if self.shard_config.is_last:
            self._pool_w = self._f16(weights["pooler.dense.weight"], dev)
            self._pool_b = self._f32(weights["pooler.dense.bias"], dev)
        del cfg

    def _embed(self, ids: torch.Tensor) -> torch.Tensor:
        batch, seq = ids.shape
        hidden = self.config.hidden_size
        out = (self._ring('embed', (batch, seq, hidden)) if self.persistent else
               torch.empty((batch, seq, hidden), dtype=torch.float32, device=ids.device))
        check(LIB.pe_bert_embed(ids.data_ptr(), self._pos_ids.data_ptr(), self._word.data_ptr(),
                                self._type0.data_ptr(), self._pos.data_ptr(), self._emb_ln_w.data_ptr(),
                                self._emb_ln_b.data_ptr(), float(self.config.layer_norm_eps), out.data_ptr(), batch, seq,
                                hidden, torch.cuda.current_stream().cuda_stream))
        return out

    @torch.no_grad()
    def forward(self, data: TransformerShardData) -> TransformerShardData:
        """Compute shard layers (`bert.py:142-151`); the last stage returns `tanh(dense(x[:, 0]))` (BertPooler)."""
        if self.shard_config.is_first:
            data = self._embed(self._to_device(data, dtype=torch.int64))
        else:
            data = self._to_device(data)
        data = self._run_blocks(data)
        if self.shard_config.is_last:
            first16 = self._cls_rows(data, torch.float16, 'first16')
            data = ops.linear(first16, self._pool_w, self._pool_b, _lib.PE_EPI_TANH_F32,
                              out=self._tmp('pooled', (first16.shape[0], self._pool_w.shape[0])) if self._static else None)
        return data

    def _first_input_spec(self, ubatch: int, dim1: int):
        return ((ubatch, dim1 or 128), torch.int64)

    def native_max_tokens(self) -> int:
        return int(self.config.max_position_embeddings)

    def native_result_item_shape(self):
        return (int(self.config.hidden_size),)

    @staticmethod
    def save_weights(model_name: str, model_file: str) -> None:
        """The reference pulls `BertModel.from_pretrained` here (`bert.py:153-161`); this build has no network."""
        raise RuntimeError(f"cannot download weights for {model_name}: no network. Provide {model_file} in the "
                           "reference npz layout (pipeedge_b200.synth writes synthetic ones).")


class BertShardForSequenceClassification(GpuTransformerShard):
    """Module shard based on `BertForSequenceClassification` (reference `bert.py:167-219`)."""
    FAMILY = 'bert'

    def _build_shard(self, weights: Mapping) -> None:
        inner = {k[len('bert.'):]: v for k, v in weights.items() if k.startswith('bert.')}   # bert.py:191-196
        self.bert = BertModelShard(self.config, self.shard_config, inner)
        self.stage = self.bert.stage
        if self.shard_config.is_last:
            dev = self.stage.device
            self._cls_w = self._f16(weights['classifier.weight'], dev)
            self._cls_b = self._f32(weights['classifier.bias'], dev)

    @torch.no_grad()
    def forward(self, data: TransformerShardData) -> TransformerShardData:
        """Compute shard layers; on the last stage `classifier(pooled)` (`bert.py:203-209`)."""
        self.bert.use_cuda_graph, self.bert.num_slots = self.use_cuda_graph, self.num_slots
        data = self.bert.forward(data) if self._static else self.bert(data)
        if self.shard_config.is_last:
            if self._static:
                pooled16 = self._tmp('pooled16', data.shape, torch.float16)
                pooled16.copy_(data)
            else:
                pooled16 = data.to(torch.float16)
            data = self._classify(pooled16, self._cls_w, self._cls_b)
        return data

    def _inner(self):
        return self.bert

    def _first_input_spec(self, ubatch: int, dim1: int):
        return self.bert._first_input_spec(ubatch, dim1)   # pylint: disable=protected-access

    def native_max_tokens(self) -> int:
        return self.bert.native_max_tokens()

    def native_result_item_shape(self):
        return (int(self.config.num_labels),)

    @staticmethod
    def save_weights(model_name: str, model_file: str) -> None:
        """See `BertModelShard.save_weights`."""
        BertModelShard.save_weights(model_name, model_file)
