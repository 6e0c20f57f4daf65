"""Shared helpers for the test-suite: golden loading and tiny-model construction."""
from __future__ import annotations

from pathlib import Path

import numpy as np
import torch

GOLDEN = Path(__file__).resolve().parent / "golden"


def bf16(a: np.ndarray) -> torch.Tensor:
    """int16 view stored in the npz -> bf16 tensor."""
    return torch.from_numpy(np.ascontiguousarray(a)).view(torch.bfloat16)


def load(name: str):
    return np.load(GOLDEN / name)


def trace_weights(z, prefix: str) -> dict:
    """Weights of the traced target ("t") or draft ("d").  The draft is the target's embedding, head, final norm and
    first layer, so only the target's weights are stored."""
    if prefix == "d":
        t = trace_weights(z, "t")
        return {**t, "layers": t["layers"][:1]}
    w = {k: bf16(z[f"{prefix}_{k}"]) for k in ("embed", "lm_head", "final_norm")}
    layers = []
    l = 0
    while f"{prefix}_l{l}_qkv" in z:
        lw = {}
        for k in ("input_norm", "qkv", "o", "post_norm", "gate_up", "down", "q_norm", "k_norm"):
            key = f"{prefix}_l{l}_{k}"
            if key in z:
                lw[k] = bf16(z[key])
        layers.append(lw)
        l += 1
    w["layers"] = layers
    return w


def trace_cfgs(family: str, z):
    from oracle.model import ModelCfg

    hd = 64 if family == "llama" else 128
    tc = ModelCfg(hidden=128, layers=2, heads=2, kv_heads=1, head_dim=hd, ffn=256, vocab=512, max_pos=512,
                  rms_eps=1e-5 if family == "llama" else 1e-6,
                  rope_theta=500000.0 if family == "llama" else 1000000.0, qk_norm=(family != "llama"))
    dc = ModelCfg(**{**tc.__dict__, "layers": 1})
    return tc, dc


def ulp_mismatch_fraction(a: torch.Tensor, b: torch.Tensor) -> float:
    return float((a.view(torch.int16) != b.view(torch.int16)).float().mean())
