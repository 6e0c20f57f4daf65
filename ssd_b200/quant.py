"""FP8 (e4m3fn) weight-only quantization of the decoder linears, of the target (Config.quantization) and of the draft
(Config.draft_quantization), each independently of the other.

One format, owned here and by ssdk_bind_weight_fp8 (include/ssdk.h): an FP8 matrix is a float8_e4m3fn tensor
W8 [N, K] in the bf16 matrix's row order plus fp32 per-row scales s [N]; row n stands for s[n] * W8[n, :].

    s[n] = amax(|W[n, :]|) / 448      (s = 1 for an all-zero row)
    W8   = e4m3_rne(clamp(W / s, -448, 448))

The quantization runs on whatever device the tensor is on, one tensor at a time, so a caller that replaces each bf16
matrix by its FP8 form as it goes never holds a second copy of the model."""
from __future__ import annotations

import math

import torch

E4M3_MAX = 448.0
FP8_LINEARS = ("qkv", "o", "gate_up", "down")  # the decoder linears of either model; embedding, lm_head and norms stay bf16


def quantize_fp8_rowwise(w: torch.Tensor, row_amax: torch.Tensor | None = None) -> tuple[torch.Tensor, torch.Tensor]:
    """bf16 (or fp32) [N, K] -> (float8_e4m3fn [N, K], fp32 [N]) with per-row amax scaling.  `row_amax` overrides the
    amax of the rows given (a column shard of a row-parallel matrix passes the amax of the full rows)."""
    wf = w.float()
    amax = wf.abs().amax(dim=1) if row_amax is None else row_amax.float()
    # divide by a tensor on the same device: torch's CUDA division by a Python scalar multiplies by its reciprocal,
    # which is not amax / 448 in every last bit, and the scales would then depend on where the weights were quantized
    s = amax / torch.full_like(amax, E4M3_MAX)
    s = torch.where(s > 0, s, torch.ones_like(s))
    w8 = (wf / s[:, None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return w8, s.contiguous()


def dequantize_fp8(w8: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """s[n] * W8[n, :] in fp32 (one fp32 rounding per element)."""
    return w8.float() * s.float()[:, None]


def quantize_layers_(w: dict, row_amax_max=None) -> dict:
    """Replace every decoder linear of a packed weight dict (loader / synth layout) by its FP8 form, in place, one
    tensor at a time: lw[name] becomes float8_e4m3fn and lw[name + "_scale"] holds the fp32 row scales.

    A tensor-parallel rank holds whole rows of qkv / gate_up but only a column shard of o / down.  `row_amax_max`
    (given on every rank of a tensor-parallel target) maps this rank's per-row amax of o / down to the maximum over all
    ranks, in place, so that every rank quantizes with the scales of the full rows: the shards are then exactly the
    shards of the quantized full matrix."""
    for lw in w["layers"]:
        for name in FP8_LINEARS:
            if lw[name].dtype != torch.float8_e4m3fn:
                amax = None
                if row_amax_max is not None and name in ("o", "down"):
                    amax = row_amax_max(lw[name].float().abs().amax(dim=1))
                w8, s = quantize_fp8_rowwise(lw[name], amax)
                lw[name] = w8  # drops the last reference to the bf16 matrix
                lw[name + "_scale"] = s
    return w


def checkpoint_quantization(hf) -> str | None:
    """'fp8' when config.json's quantization_config describes e4m3 weights with per-channel or per-tensor scales
    (compressed-tensors float8, fbgemm_fp8, or 'fp8' without weight blocks); None without a quantization_config.
    Block-wise scales and every other quantization method raise NotImplementedError."""
    qc = getattr(hf, "quantization_config", None)
    if not qc:
        return None
    method = qc.get("quant_method")
    if method == "fbgemm_fp8":
        return "fp8"
    if method == "fp8":
        if qc.get("weight_block_size"):
            raise NotImplementedError("block-wise FP8 scales (weight_block_size) are not supported: per-channel or "
                                      "per-tensor scales only")
        return "fp8"
    if method == "compressed-tensors":
        for group in (qc.get("config_groups") or {}).values():
            wq = group.get("weights") or {}
            if wq.get("type") == "float" and wq.get("num_bits") == 8:
                if wq.get("strategy") == "block":
                    raise NotImplementedError("block-wise FP8 scales (compressed-tensors strategy 'block') are not "
                                              "supported: per-channel or per-tensor scales only")
                return "fp8"
    raise NotImplementedError(f"quantization_config {qc!r}: only FP8 (e4m3) weight checkpoints are supported")


def parse_kv_cache_dtype(v: str) -> str:
    """Config.kv_cache_dtype -> "auto" (bf16 KV cache) or "fp8" (e4m3 target KV cache with per-layer scales)."""
    if v in ("auto", "bf16", "bfloat16"):
        return "auto"
    if v in ("fp8", "fp8_e4m3"):
        return "fp8"
    if v == "fp8_e5m2":
        raise NotImplementedError("kv_cache_dtype='fp8_e5m2' is not supported: the FP8 KV cache is e4m3 ('fp8')")
    raise ValueError(f"kv_cache_dtype={v!r}: supported values are 'auto' / 'bf16' / 'bfloat16' (bf16 KV cache) and "
                     "'fp8' / 'fp8_e4m3' (float8 e4m3 target KV cache)")


def quantize_kv_fp8(y: torch.Tensor, scale: float) -> torch.Tensor:
    """The FP8 KV store (ssdk_bind_kv_cache_fp8): e4m3_rne(clamp(y / scale, -448, 448)) of the bf16 values y, divided
    tensor by tensor (IEEE fp32 division on any device)."""
    yf = y.float()
    return (yf / torch.full_like(yf, scale)).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)


def resolve_kv_scales(found: dict[tuple[str, int], float], layers: int, where: str = "checkpoint"
                      ) -> tuple[list[float], list[float]]:
    """Per-layer (k_scale, v_scale) of an FP8 KV cache from the checkpoint's `model.layers.{i}.self_attn.k_scale` /
    `.v_scale` scalars (found[("k" | "v", i)]): all 1.0 when there are none.  Scales on some layers only, or a scale
    that is not finite or not > 0, raise ValueError."""
    if not found:
        return [1.0] * layers, [1.0] * layers
    missing = [f"{kind}_scale of layer {i}" for i in range(layers) for kind in ("k", "v") if (kind, i) not in found]
    if missing:
        raise ValueError(f"{where}: KV cache scales on some layers only (missing {', '.join(missing[:4])}"
                         f"{', ...' if len(missing) > 4 else ''})")
    for (kind, i), s in sorted(found.items()):
        if not (math.isfinite(s) and s > 0):
            raise ValueError(f"{where}: layer {i} {kind}_scale = {s!r}: KV cache scales must be finite and > 0")
    return [found[("k", i)] for i in range(layers)], [found[("v", i)] for i in range(layers)]


def parse_quantization(q: str | None) -> str | None:
    if q is None or q == "fp8":
        return q
    raise ValueError(f"quantization={q!r}: supported values are None (bf16 weights) and 'fp8' (e4m3 weight-only "
                     "quantization of the model's decoder linears)")
