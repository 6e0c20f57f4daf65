"""FP8 KV cache counterpart of the oracle's decoder forward, for the GPU parity tests.

`KvFp8OracleModel` keeps its paged KV cache in fp32 and stores, per layer l, s·code with code = e4m3_rne(sat(y / s)) of
the bf16 K / V values y the oracle computes (s = k_scale[l] or v_scale[l], quant.quantize_kv_fp8): the values the
engine's attention reads from its e4m3 cache.  Everything else is the oracle's code unchanged; the decoder linears may be
`Fp8Weight`s as well (tests/fp8_ref.py), so the same model also stands for an FP8-weight target with an FP8 cache."""
from __future__ import annotations

import torch

import oracle.model as _om
from oracle import ops as _ops
from oracle.model import OracleModel
from ssd_b200.quant import quantize_kv_fp8
from tests.fp8_ref import _Fp8Ops


def dequantized(y: torch.Tensor, s: float) -> torch.Tensor:
    """s·code in fp32 (exact: one product of an e4m3 value and an fp32 scale, rounded once)."""
    return quantize_kv_fp8(y, s).float() * s


class _KvFp8Ops(_Fp8Ops):
    def __init__(self, model: "KvFp8OracleModel"):
        self.model = model

    def store_kvcache(self, k, v, k_cache, v_cache, slot_mapping):
        l = self.model.layer_of[k_cache.data_ptr()]
        _ops.store_kvcache(dequantized(k, self.model.k_scale[l]), dequantized(v, self.model.v_scale[l]), k_cache, v_cache,
                           slot_mapping)


class KvFp8OracleModel(OracleModel):
    def __init__(self, cfg, weights: dict, num_blocks: int, block_size: int = 256, compiled: bool = True,
                 k_scale: list[float] | None = None, v_scale: list[float] | None = None):
        super().__init__(cfg, weights, num_blocks, block_size, compiled)
        self.kv_cache = torch.zeros(self.kv_cache.shape, dtype=torch.float32)
        self.k_scale = list(k_scale) if k_scale is not None else [1.0] * cfg.layers
        self.v_scale = list(v_scale) if v_scale is not None else [1.0] * cfg.layers
        self.layer_of = {self.kv_cache[0, l].data_ptr(): l for l in range(cfg.layers)}

    def forward(self, *args, **kwargs):
        saved = _om.ops
        _om.ops = _KvFp8Ops(self)
        try:
            return super().forward(*args, **kwargs)
        finally:
            _om.ops = saved
