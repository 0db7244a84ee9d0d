"""CPU oracle for the PipeEdge hot path - TEST INFRASTRUCTURE, NOT PRODUCT.

This package restates, on the CPU, the arithmetic that the reference (usc-isi/PipeEdge @ 1a68bbb)
performs on the path `BASELINE.json:north_star` names: the ViT / DeiT / BERT encoder-block shard
forward and the QuantPipe clamp / quantise / bit-pack (and its inverse).

Only `tests/`, `__graft_entry__.smoke()` and the `cpu_baseline` / `--impl reference` legs of
`bench.py` may import it, and only as the checker or the timed CPU baseline - never as the thing
shipped. Nothing under `pipeedge_b200/`, `runtime.py`, `model_cfg.py` or `devices.py` imports it;
`tests/test_host_cpu.py::test_product_never_imports_the_oracle` enforces that.

Where the arithmetic lives
--------------------------
The reference's shard classes contain no arithmetic of their own: they instantiate HuggingFace
`transformers` modules (`vit.py:12-14`, `deit.py:10-13`, `bert.py:10-12`; dependency declared
UNPINNED as `transformers>=4.6.0` in the reference `pyproject.toml:23`; this container has
5.5.0) and run them on ATen CPU kernels. `oracle/shards.py` restates those modules' published
algorithm (LayerNorm, Linear, unmasked softmax attention with scale d^-0.5, exact-erf GELU,
residuals) with plain `torch` fp32 CPU ops, citing the reference call site and the HF module for
each step. `oracle/quant.py` restates `pipeedge/quantization/{basic_op,clamp_op}.py` in NumPy.

Pinning
-------
The reference repo holds no golden vectors for the model path and only a round-trip property test
for quantisation (`test/quant/test_quant.py:7-30`). The oracle is therefore pinned against the
reference ITSELF: `oracle/make_goldens.py` imports a checkout of it (`PIPEEDGE_REFERENCE`, `src/pipeedge`) read-only, runs its shard classes and quantisation functions on
seeded inputs and writes `tests/golden/*.npz`; `tests/test_oracle_golden.py` (CPU) checks the oracle
against those fixtures and `tests/test_*_gpu.py` check the CUDA path against both.

One deliberate deviation: the reference never calls `.eval()` on BERT layer shards, so with
`hidden_dropout_prob=0.1` its BERT output is stochastic (SURVEY.md section 0). The goldens are
generated with the reference shards put in `.eval()`; the oracle has no dropout.
"""
