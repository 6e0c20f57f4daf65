"""Config — the keyword surface bench/bench.py:160-184 passes to LLM(...), same names and defaults as
ssd/config.py:7-49.  Options that belong to paths outside the sync-SD hot path (draft_async, use_eagle,
fan-out lists) are accepted and rejected loudly rather than silently ignored."""
from __future__ import annotations

import json
import os
from dataclasses import dataclass

from .paths import DEFAULT_DRAFT, DEFAULT_TARGET
from .quant import checkpoint_quantization, parse_kv_cache_dtype, parse_quantization


@dataclass
class Config:
    model: str = DEFAULT_TARGET
    max_num_batched_tokens: int = 16384
    max_num_seqs: int = 1
    max_model_len: int = 4096
    gpu_memory_utilization: float = 0.7
    num_gpus: int = 1
    enforce_eager: bool = False
    hf_config: object | None = None
    eos: int = -1
    kvcache_block_size: int = 256
    num_kvcache_blocks: int = -1
    device: str = "cuda"
    # speculation
    draft_hf_config: object | None = None
    speculate: bool = False
    draft: str = DEFAULT_DRAFT
    speculate_k: int = 1
    draft_async: bool = False
    async_fan_out: int = 3
    fan_out_list: list[int] | None = None
    fan_out_list_miss: list[int] | None = None
    sampler_x: float | None = None
    jit_speculate: bool = False
    use_eagle: bool = False
    eagle_layers: list[int] | None = None
    d_model_target: int | None = None
    tokenizer_path: str | None = None
    verbose: bool = False
    debug_mode: bool = False
    max_steps: int | None = None
    # ssd_b200 extensions (ignored by the reference's bench scripts)
    use_cuda_graph: bool = True
    use_pdl: bool = True
    seed: int = 0
    # prefill through ssdk_forward_varlen (PairRunner.prefill_varlen): prompts of any lengths and prefix-cache hits share
    # 256-token calls.  Opt-in until measured on the H100 (DESIGN.md §7).
    varlen_prefill: bool = False
    # "fp8": the target's four decoder linears (qkv, o, gate_up, down) run as e4m3 weights with fp32 per-row scales
    # (W8A16, DESIGN.md §3); bf16 checkpoints are quantized on load.  This changes the outputs.  An FP8 checkpoint is
    # loaded as FP8 whatever this says, and the field then reads "fp8".
    quantization: str | None = None
    # "fp8": the same for the draft's four decoder linears, independently of `quantization`.  At temperature 0 the engine
    # still emits the target's greedy chain and at temperature > 0 it still samples the target's distribution: an FP8
    # draft changes only the acceptance rate and the speed.  An FP8 draft checkpoint is loaded as FP8 whatever this says,
    # and the field then reads "fp8".
    draft_quantization: str | None = None
    # "fp8" (or "fp8_e4m3"): the TARGET's KV cache is stored as float8 e4m3 with one fp32 scale per layer for K and one
    # for V (the checkpoint's self_attn.k_scale / v_scale, else 1.0; DESIGN.md §3).  Half the bytes per token, twice the
    # pages in the same memory.  This changes the outputs.  The draft's cache stays bf16.  "auto" (or "bf16",
    # "bfloat16"): bf16, the default; the field then reads "auto".
    kv_cache_dtype: str = "auto"

    @property
    def max_blocks(self) -> int:
        return (self.max_model_len + self.kvcache_block_size - 1) // self.kvcache_block_size

    def __post_init__(self):
        if not os.path.isdir(self.model):
            raise AssertionError(f"model directory {self.model!r} does not exist (config.py:53)")
        if not 1 <= self.num_gpus <= 8:
            raise AssertionError("single node only: 1 <= num_gpus <= 8 (config.py:55)")
        if self.draft_async:
            raise NotImplementedError("draft_async (async SSD) is a SURVEY §8(f) 'next' row, not built yet")
        if self.use_eagle:
            raise NotImplementedError("EAGLE-3 drafts are out of scope of the sync-SD hot path")
        if self.enforce_eager:
            self.use_cuda_graph = False
        self.quantization = parse_quantization(self.quantization)
        self.draft_quantization = parse_quantization(self.draft_quantization)
        self.kv_cache_dtype = parse_kv_cache_dtype(self.kv_cache_dtype)
        self.hf_config = load_hf_config(self.model)
        if checkpoint_quantization(self.hf_config) == "fp8":
            self.quantization = "fp8"
        self.max_model_len = min(self.max_model_len, self.hf_config.max_position_embeddings)
        if self.speculate:
            if not os.path.isdir(self.draft):
                raise AssertionError(f"draft directory {self.draft!r} does not exist")
            self.draft_hf_config = load_hf_config(self.draft)
            if checkpoint_quantization(self.draft_hf_config) == "fp8":  # any other quantization raises
                self.draft_quantization = "fp8"
            self.max_model_len = min(self.max_model_len, self.draft_hf_config.max_position_embeddings)
        if self.max_num_batched_tokens < self.max_model_len:
            raise AssertionError("max_num_batched_tokens < max_model_len (config.py:94)")
        # limits of libssdk (DESIGN.md "Limits"), reported here rather than at the first step
        k1 = (self.speculate_k + 1) if self.speculate else 1
        if self.speculate and not 1 <= self.speculate_k <= 7:
            raise ValueError(f"speculate_k={self.speculate_k}: libssdk supports 1 <= k <= 7")
        if self.max_num_seqs > 32 or self.max_num_seqs * k1 > 256:
            raise ValueError(f"max_num_seqs={self.max_num_seqs} with {k1} tokens per sequence and step: libssdk runs at most 32 "
                             "sequences and 256 tokens per step")


class _HFConfig:
    """Minimal attribute bag over config.json (what ssd/config.py reads through transformers.AutoConfig)."""

    def __init__(self, d: dict):
        self.__dict__.update(d)
        self.model_type = d.get("model_type", "llama")
        if "head_dim" not in d or d["head_dim"] is None:
            self.head_dim = d["hidden_size"] // d["num_attention_heads"]
        self.tie_word_embeddings = d.get("tie_word_embeddings", False)
        if "rope_theta" not in d:
            rp = d.get("rope_parameters") or {}
            self.rope_theta = rp.get("rope_theta", 1000000.0 if "qwen" in self.model_type else 500000.0)


def load_hf_config(path: str) -> _HFConfig:
    with open(os.path.join(path, "config.json")) as f:
        return _HFConfig(json.load(f))
