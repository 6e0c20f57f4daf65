"""FP8 (W8A16) counterpart of the oracle's decoder forward, for the GPU parity tests.

The target's four decoder linears are evaluated as bf16(s ⊙ (x · bf16(W8)ᵀ)) in fp32; everything else is the oracle's
code unchanged: `Fp8OracleModel.forward` runs `OracleModel.forward` with its `ops` module seen through a proxy whose
`linear` dispatches on `Fp8Weight`."""
from __future__ import annotations

import torch

import oracle.model as _om
from oracle import ops as _ops
from oracle.model import OracleModel
from ssd_b200.quant import FP8_LINEARS, quantize_fp8_rowwise


class Fp8Weight:
    def __init__(self, w8: torch.Tensor, scale: torch.Tensor):
        self.w8, self.scale = w8, scale


def linear_fp8(x: torch.Tensor, w8: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    y = x.to(torch.bfloat16).float() @ w8.float().t()  # e4m3 -> fp32 is exact, as is e4m3 -> bf16
    return (y * scale.float()[None, :]).to(torch.bfloat16)


class _Fp8Ops:
    def __getattr__(self, name):
        return getattr(_ops, name)

    @staticmethod
    def linear(x, w):
        if isinstance(w, Fp8Weight):
            return linear_fp8(x, w.w8, w.scale)
        return _ops.linear(x, w)


class Fp8OracleModel(OracleModel):
    def forward(self, *args, **kwargs):
        saved = _om.ops
        _om.ops = _Fp8Ops()
        try:
            return super().forward(*args, **kwargs)
        finally:
            _om.ops = saved


def quantize_weights(w: dict) -> tuple[dict, dict]:
    """(oracle weights with Fp8Weight linears, engine weights with float8 tensors + `<name>_scale`), both on the CPU."""
    wo = {k: v for k, v in w.items() if k != "layers"}
    we = dict(wo)
    wo["layers"], we["layers"] = [], []
    for lw in w["layers"]:
        lo, le = dict(lw), dict(lw)
        for name in FP8_LINEARS:
            w8, s = quantize_fp8_rowwise(lw[name])
            lo[name] = Fp8Weight(w8, s)
            le[name], le[name + "_scale"] = w8, s
        wo["layers"].append(lo)
        we["layers"].append(le)
    return wo, we
