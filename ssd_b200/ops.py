"""Tensor-level wrappers over the stand-alone ops of libssdk (same names/argument meaning as the
reference's layers so the parity tests read like tests of ssd.layers.*).

PyTorch is plumbing here: it owns the device memory and the stream; every op runs in the
hand-written sm_90a kernels behind the C-ABI.  All functions require CUDA tensors and raise if
the extension is missing — there is no eager fallback.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import lib as _L


def _ptr(t: torch.Tensor | None):
    return None if t is None else t.data_ptr()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _req(t: torch.Tensor, dtype, name: str):
    if not t.is_cuda:
        raise RuntimeError(f"{name}: CUDA tensor required (libssdk has no CPU path)")
    if t.dtype != dtype:
        raise TypeError(f"{name}: expected {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"{name}: must be contiguous")


def linear(x: torch.Tensor, weight: torch.Tensor, split_k: int = 0) -> torch.Tensor:
    """F.linear(x, weight) for M = x.shape[0] <= 64 tokens (layers/linear.py:98,196).

    x [M, K] bf16, weight [N, K] bf16 -> [M, N] bf16 (fp32 accumulate, one bf16 rounding)."""
    _req(x, torch.bfloat16, "x")
    _req(weight, torch.bfloat16, "weight")
    M, K = x.shape
    N = weight.shape[0]
    assert weight.shape[1] == K
    y = torch.empty(M, N, dtype=torch.bfloat16, device=x.device)
    nkb = K // 64
    if split_k == 1:
        parts = None
    else:
        if split_k == 0:  # same bound as auto_splits() in csrc/engine.cu
            tiles = (N + 127) // 128
            sms = torch.cuda.get_device_properties(x.device).multi_processor_count
            s_bound = max(1, min(max(1, nkb // 4), (2 * sms + tiles - 1) // tiles))
        else:
            s_bound = min(split_k, nkb)
        parts = torch.empty(s_bound * M * N, dtype=torch.float32, device=x.device)
    lib = _L.load()
    _L.check(lib.ssdk_gemm_small_m(_ptr(x), _ptr(weight), _ptr(y), _ptr(parts), M, N, K, N, split_k, _stream()),
             "ssdk_gemm_small_m")
    return y


def gate_up_silu(x: torch.Tensor, w_gate_up: torch.Tensor) -> torch.Tensor:
    """SiluAndMul(MergedColumnParallelLinear(x)) fused (models/llama3.py:130-133).
    w_gate_up [2*ffn, K] gate rows then up rows -> [M, ffn]."""
    _req(x, torch.bfloat16, "x")
    _req(w_gate_up, torch.bfloat16, "w_gate_up")
    M, K = x.shape
    ffn = w_gate_up.shape[0] // 2
    h = torch.empty(M, ffn, dtype=torch.bfloat16, device=x.device)
    lib = _L.load()
    _L.check(lib.ssdk_gemm_gate_up_silu(_ptr(x), _ptr(w_gate_up), _ptr(h), M, ffn, K, _stream()), "ssdk_gemm_gate_up_silu")
    return h


def rms_norm(x: torch.Tensor, weight: torch.Tensor, eps: float, residual: torch.Tensor | None = None):
    """RMSDNorm.forward (layers/layernorm.py:90-98).  Returns y if residual is None else (y, new_residual)."""
    _req(x, torch.bfloat16, "x")
    _req(weight, torch.bfloat16, "weight")
    M, d = x.shape
    y = torch.empty_like(x)
    res_out = torch.empty_like(x) if residual is not None else None
    if residual is not None:
        _req(residual, torch.bfloat16, "residual")
    lib = _L.load()
    _L.check(lib.ssdk_rmsnorm(_ptr(x), _ptr(residual), _ptr(weight), float(eps), _ptr(y), _ptr(res_out), M, d, _stream()),
             "ssdk_rmsnorm")
    return y if residual is None else (y, res_out)


def rope_store_kv(qkv: torch.Tensor, positions: torch.Tensor, slot_mapping: torch.Tensor, rope_table: torch.Tensor,
                  k_cache: torch.Tensor, v_cache: torch.Tensor, heads: int, kv_heads: int, head_dim: int,
                  q_norm_w: torch.Tensor | None = None, k_norm_w: torch.Tensor | None = None,
                  norm_eps: float = 1e-6) -> torch.Tensor:
    """[q/k RMSHeadNorm +] RotaryEmbedding.forward + store_kvcache (qwen3.py:97-105, rotary_embedding.py:40-60,
    attention.py:35-41).  Returns q [M, H*hd]; k (rotated) and v are written into the caches."""
    _req(qkv, torch.bfloat16, "qkv")
    _req(positions, torch.int64, "positions")
    _req(slot_mapping, torch.int32, "slot_mapping")
    _req(rope_table, torch.float32, "rope_table")
    M = qkv.shape[0]
    q = torch.empty(M, heads * head_dim, dtype=torch.bfloat16, device=qkv.device)
    lib = _L.load()
    _L.check(lib.ssdk_rope_store_kv(_ptr(qkv), _ptr(positions), _ptr(slot_mapping), _ptr(rope_table), _ptr(q_norm_w),
                                    _ptr(k_norm_w), float(norm_eps), _ptr(q), _ptr(k_cache), _ptr(v_cache), M, heads,
                                    kv_heads, head_dim, _stream()), "ssdk_rope_store_kv")
    return q


def silu_and_mul(x: torch.Tensor) -> torch.Tensor:
    """SiluAndMul.forward (layers/activation.py:11-14)."""
    _req(x, torch.bfloat16, "x")
    M, two_ffn = x.shape
    out = torch.empty(M, two_ffn // 2, dtype=torch.bfloat16, device=x.device)
    lib = _L.load()
    _L.check(lib.ssdk_silu_mul(_ptr(x), _ptr(out), M, two_ffn // 2, _stream()), "ssdk_silu_mul")
    return out


def paged_attention(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, block_tables: torch.Tensor,
                    context_lens: torch.Tensor, q_len: int, scale: float) -> torch.Tensor:
    """flash_attn_with_kvcache(q, k_cache, v_cache, cache_seqlens=context_lens, page_table=block_tables,
    causal=True[, cu_seqlens_q]) as called at layers/attention.py:107-111,128-131.

    q [B*q_len, H, hd]; caches [num_blocks, block_size, KV, hd]; returns [B*q_len, H*hd]."""
    _req(q, torch.bfloat16, "q")
    _req(k_cache, torch.bfloat16, "k_cache")
    _req(v_cache, torch.bfloat16, "v_cache")
    _req(block_tables, torch.int32, "block_tables")
    _req(context_lens, torch.int32, "context_lens")
    Mq, H, hd = q.shape
    B = Mq // q_len
    _, block_size, KV, _ = k_cache.shape
    max_blocks = block_tables.shape[1]
    lib = _L.load()
    nbytes = lib.ssdk_paged_attn_scratch_bytes(B, q_len, H, hd, max_blocks * block_size)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=q.device)
    out = torch.empty(Mq, H * hd, dtype=torch.bfloat16, device=q.device)
    _L.check(lib.ssdk_paged_attn(_ptr(q), _ptr(k_cache), _ptr(v_cache), _ptr(block_tables), _ptr(context_lens), _ptr(out),
                                 _ptr(scratch), B, q_len, H, KV, hd, block_size, max_blocks, float(scale), _stream()),
             "ssdk_paged_attn")
    return out


def paged_attention_plan(B: int, q_len: int, H: int, KV: int, max_ctx: int) -> dict:
    """The launch plan paged_attention takes for these sizes on the current device (max_ctx = block_size *
    max_blocks): query tokens per tile, 16-row MMA tiles, query tiles and KV splits."""
    out = (C.c_int32 * 4)()
    lib = _L.load()
    _L.check(lib.ssdk_paged_attn_plan(H, KV, B, q_len, max_ctx, out), "ssdk_paged_attn_plan")
    return {"TQ": out[0], "MT": out[1], "n_qtiles": out[2], "n_split": out[3]}


def sample(logits: torch.Tensor, temperatures: torch.Tensor, seed: int = 0, step_id: int = 0) -> torch.Tensor:
    """Sampler.forward (layers/sampler.py:14-36) — logits [B, V] bf16, temperatures [B] fp32 -> int64 [B]."""
    _req(logits, torch.bfloat16, "logits")
    _req(temperatures, torch.float32, "temperatures")
    B, V = logits.shape
    out = torch.empty(B, dtype=torch.int64, device=logits.device)
    lib = _L.load()
    _L.check(lib.ssdk_sample(_ptr(logits), V, _ptr(temperatures), B, V, seed, step_id, _ptr(out), _stream()), "ssdk_sample")
    return out


def verify(logits_p: torch.Tensor, logits_q: torch.Tensor, speculations: torch.Tensor, temperatures_target: torch.Tensor,
           temperatures_draft: torch.Tensor, cache_hits: torch.Tensor | None = None, jit_speculate: bool = False,
           seed: int = 0, step_id: int = 0):
    """ssd.utils.verify.verify (utils/verify.py:5-181), device-resident results:
    returns (n_accept int32 [B], recovery int64 [B]); the accepted suffix of row b is
    speculations[b, :1 + n_accept[b]]."""
    _req(logits_p, torch.bfloat16, "logits_p")
    _req(logits_q, torch.bfloat16, "logits_q")
    _req(speculations, torch.int64, "speculations")
    _req(temperatures_target, torch.float32, "temperatures_target")
    _req(temperatures_draft, torch.float32, "temperatures_draft")
    B, Kp1, V = logits_p.shape
    K = Kp1 - 1
    hits = None
    if cache_hits is not None:
        hits = cache_hits.to(torch.int32).contiguous()
    lib = _L.load()
    scratch = torch.empty(lib.ssdk_verify_scratch_bytes(B, K), dtype=torch.uint8, device=logits_p.device)
    n_acc = torch.empty(B, dtype=torch.int32, device=logits_p.device)
    rec = torch.empty(B, dtype=torch.int64, device=logits_p.device)
    _L.check(lib.ssdk_verify(_ptr(logits_p), _ptr(logits_q), _ptr(speculations), _ptr(temperatures_target),
                             _ptr(temperatures_draft), _ptr(hits), int(jit_speculate), B, K, V, seed, step_id, _ptr(n_acc),
                             _ptr(rec), _ptr(scratch), _stream()), "ssdk_verify")
    return n_acc, rec
