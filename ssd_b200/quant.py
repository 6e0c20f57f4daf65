"""FP8 (e4m3fn) weight-only quantization of the decoder linears, of the target (Config.quantization) and of the draft
(Config.draft_quantization), each independently of the other.

One format, owned here and by ssdk_bind_weight_fp8 (include/ssdk.h): an FP8 matrix is a float8_e4m3fn tensor
W8 [N, K] in the bf16 matrix's row order plus fp32 per-row scales s [N]; row n stands for s[n] * W8[n, :].

    s[n] = amax(|W[n, :]|) / 448      (s = 1 for an all-zero row)
    W8   = e4m3_rne(clamp(W / s, -448, 448))

The quantization runs on whatever device the tensor is on, one tensor at a time, so a caller that replaces each bf16
matrix by its FP8 form as it goes never holds a second copy of the model."""
from __future__ import annotations

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


def parse_quantization(q: str | None) -> str | None:
    if q is None or q == "fp8":
        return q
    raise ValueError(f"quantization={q!r}: supported values are None (bf16 weights) and 'fp8' (e4m3 weight-only "
                     "quantization of the model's decoder linears)")
