"""Weights -> device, and construction of the PairRunner from a Config.

Real checkpoints: HF safetensors are read and packed exactly as ssd/utils/loader.py:186-218 + the weight_loader
callbacks do (q|k|v -> qkv_proj, gate|up -> gate_up_proj; column-parallel shards by output rows, row-parallel by
input columns, embedding / lm_head by vocab rows).  Synthetic directories: generated on the device (synth.py)."""
from __future__ import annotations

import glob
import json
import os

import torch

from . import lib as L
from .quant import FP8_LINEARS, quantize_layers_, resolve_kv_scales
from .runner import ModelSpec, PairRunner


def spec_from_config(hf) -> ModelSpec:
    return ModelSpec(hidden=hf.hidden_size, layers=hf.num_hidden_layers, heads=hf.num_attention_heads,
                     kv_heads=hf.num_key_value_heads, head_dim=hf.head_dim, ffn=hf.intermediate_size,
                     vocab=hf.vocab_size, rms_eps=hf.rms_norm_eps, rope_theta=float(hf.rope_theta),
                     qk_norm=("qwen3" in hf.model_type), tie_embed=bool(hf.tie_word_embeddings),
                     max_pos=hf.max_position_embeddings)


# decoder linears: checkpoint leaf -> (packed matrix, sub-matrix index); column-parallel ones pack q|k|v and gate|up
_LINEAR_LEAVES = {
    "self_attn.q_proj": ("qkv", 0), "self_attn.k_proj": ("qkv", 1), "self_attn.v_proj": ("qkv", 2),
    "self_attn.o_proj": ("o", 0), "mlp.gate_proj": ("gate_up", 0), "mlp.up_proj": ("gate_up", 1),
    "mlp.down_proj": ("down", 0),
}


def load_safetensors_weights(path: str, spec: ModelSpec, device, tp_size: int = 1, tp_rank: int = 0,
                             allow_fp8: bool = True, kv_scales: bool = False) -> dict:
    """Packed per-rank weights.  bf16 / fp16 / fp32 tensors are loaded as bf16.  A float8_e4m3fn decoder linear
    `<proj>.weight` stays e4m3 and pairs with `<proj>.weight_scale` (fp32 or bf16, shape [N, 1], [N], [1] or []); the
    packed matrix then gets fp32 per-row scales lw[name + "_scale"] (a per-tensor scale is broadcast to its rows, so
    q|k|v and gate|up with different per-tensor scales become one per-row vector).  `input_scale` / `input_scale_ub`
    are activation scales of W8A8 kernels and are ignored (listed in w["ignored"]).  Block-wise scales
    (`weight_scale_inv`) raise NotImplementedError, and so does any FP8 tensor when allow_fp8 is False.
    kv_scales: the scalar KV cache scales `model.layers.{i}.self_attn.k_scale` / `.v_scale` are read as fp32 into
    w["kv_scales"] (resolve_kv_scales); without it they are dropped, as every tensor the engine does not use."""
    from safetensors import safe_open

    H, KV, hd = spec.heads // tp_size, spec.kv_heads // tp_size, spec.head_dim
    ffn, Vs, d = spec.ffn // tp_size, spec.vocab // tp_size, spec.hidden
    bf, f8 = torch.bfloat16, torch.float8_e4m3fn
    w = {"layers": [dict() for _ in range(spec.layers)]}
    ignored: list[str] = []
    # per packed matrix: (rows of each sub-matrix in the checkpoint, rows of each on this rank, shape on this rank,
    # column-parallel?)
    full_rows = {"qkv": [spec.heads * hd, spec.kv_heads * hd, spec.kv_heads * hd], "gate_up": [spec.ffn, spec.ffn],
                 "o": [d], "down": [d]}
    rank_rows = {"qkv": [H * hd, KV * hd, KV * hd], "gate_up": [ffn, ffn], "o": [d], "down": [d]}
    shape = {"qkv": ((H + 2 * KV) * hd, d), "gate_up": (2 * ffn, d), "o": (d, H * hd), "down": (d, ffn)}
    scales_seen: dict[tuple[int, str, int], bool] = {}
    kv_found: dict[tuple[str, int], float] = {}

    def rows(t, n):  # column-parallel: shard output rows
        return t[tp_rank * n:(tp_rank + 1) * n]

    def cols(t, n):  # row-parallel: shard input columns
        return t[:, tp_rank * n:(tp_rank + 1) * n]

    def packed(lw, name, dtype):
        if name not in lw:
            lw[name] = torch.empty(*shape[name], dtype=dtype, device=device)
            if dtype == f8:
                lw[name + "_scale"] = torch.empty(shape[name][0], dtype=torch.float32, device=device)
        elif lw[name].dtype != dtype:
            raise ValueError(f"{path}: the parts of packed {name} mix FP8 and non-FP8 weights")
        return lw[name]

    def put_linear(lw, name, part, t):
        dst = packed(lw, name, f8 if t.dtype == f8 else bf)
        if name in ("o", "down"):
            dst.copy_(cols(t if t.dtype == f8 else t.to(bf), shape[name][1]).to(device))
            return
        r0 = sum(rank_rows[name][:part])
        n = rank_rows[name][part]
        dst[r0:r0 + n] = rows(t if t.dtype == f8 else t.to(bf), n).to(device)

    def put_scale(lw, layer, name, part, t):
        n_full = full_rows[name][part]
        t = t.float().reshape(-1)
        if t.numel() == 1:
            t = t.expand(n_full)
        elif t.numel() != n_full:
            raise ValueError(f"{path}: layer {layer} {name} weight_scale has {t.numel()} elements; expected 1 or "
                             f"{n_full} (per-tensor or per-channel)")
        sc = packed(lw, name, f8)
        r0, n = sum(rank_rows[name][:part]), rank_rows[name][part]
        # column-parallel: the scales follow their rows; row-parallel (o, down): every rank keeps all output-row
        # scales, since a row scale factors out of each rank's partial sum
        sc_rank = rows(t, n) if name in ("qkv", "gate_up") else t
        lw[name + "_scale"][r0:r0 + n] = sc_rank.to(device)
        scales_seen[(layer, name, part)] = True

    for file in sorted(glob.glob(os.path.join(path, "*.safetensors"))):
        with safe_open(file, "pt", "cpu") as f:
            for name in f.keys():
                if name.endswith(".weight_scale_inv"):
                    raise NotImplementedError(f"{path}: {name}: block-wise FP8 scales are not supported (per-channel or "
                                              "per-tensor scales only)")
                if name.endswith(".input_scale") or name.endswith(".input_scale_ub"):
                    ignored.append(name)  # activation scales: the FP8 path is weight-only
                    continue
                t = f.get_tensor(name)
                if kv_scales and name.startswith("model.layers.") and name.endswith((".self_attn.k_scale",
                                                                                     ".self_attn.v_scale")):
                    if t.numel() != 1:
                        raise ValueError(f"{path}: {name} has {t.numel()} elements; KV cache scales are per layer "
                                         "(one scalar)")
                    kv_found[(name[-7], int(name.split(".")[2]))] = float(t.to(torch.float32).reshape(-1)[0])
                    continue
                if t.dtype == f8 and not allow_fp8:
                    raise NotImplementedError(f"{path}: {name} is FP8 and allow_fp8=False asks for bf16 weights; FP8 "
                                              "decoder linears load for the draft as well, not for the target model "
                                              "only: pass allow_fp8=True")
                parts = name.split(".")
                if name.startswith("model.layers.") and ".".join(parts[3:-1]) in _LINEAR_LEAVES and \
                        parts[-1] in ("weight", "weight_scale"):
                    layer = int(parts[2])
                    lname, part = _LINEAR_LEAVES[".".join(parts[3:-1])]
                    if parts[-1] == "weight_scale":
                        put_scale(w["layers"][layer], layer, lname, part, t)
                    else:
                        put_linear(w["layers"][layer], lname, part, t)
                    continue
                if t.dtype == f8:
                    raise NotImplementedError(f"{path}: {name} is FP8; only the decoder linears may be FP8")
                t = t.to(bf)
                if name == "model.embed_tokens.weight":
                    w["embed"] = rows(t, Vs).to(device).contiguous()
                elif name == "lm_head.weight":
                    w["lm_head"] = rows(t, Vs).to(device).contiguous()
                elif name == "model.norm.weight":
                    w["final_norm"] = t.to(device)
                elif name.startswith("model.layers."):
                    lw, leaf = w["layers"][int(parts[2])], ".".join(parts[3:])
                    if leaf == "input_layernorm.weight":
                        lw["input_norm"] = t.to(device)
                    elif leaf == "post_attention_layernorm.weight":
                        lw["post_norm"] = t.to(device)
                    elif leaf == "self_attn.q_norm.weight":
                        lw["q_norm"] = t.to(device)
                    elif leaf == "self_attn.k_norm.weight":
                        lw["k_norm"] = t.to(device)
    for layer, lw in enumerate(w["layers"]):
        for lname, sub in full_rows.items():
            if lname in lw and lw[lname].dtype == f8:
                missing = [p for p in range(len(sub)) if (layer, lname, p) not in scales_seen]
                if missing:
                    raise ValueError(f"{path}: layer {layer} {lname}: FP8 weight without weight_scale")
    if "lm_head" not in w:  # tie_word_embeddings (models/llama3.py:321-322)
        w["lm_head"] = w["embed"]
    if ignored:
        w["ignored"] = ignored
    if kv_scales:
        w["kv_scales"] = resolve_kv_scales(kv_found, spec.layers, path)
    return w


def is_fp8(w: dict) -> bool:
    return any(lw[n].dtype == torch.float8_e4m3fn for lw in w["layers"] for n in FP8_LINEARS)


def shard_packed_weights(w: dict, spec: ModelSpec, tp_size: int, tp_rank: int) -> dict:
    """Slice full packed weights (tp=1 layout) into rank `tp_rank`'s shard with the reference's rules:
    qkv / gate_up column-parallel per sub-matrix (layers/linear.py:116-122,148-162), o / down row-parallel
    (:188-193), embedding / lm_head by vocab rows (embed_head.py:41-47), norms replicated."""
    H, KV, hd, ffn, V = spec.heads, spec.kv_heads, spec.head_dim, spec.ffn, spec.vocab
    h, kv, f, vs = H // tp_size, KV // tp_size, ffn // tp_size, V // tp_size
    r = tp_rank
    out = {"embed": w["embed"][r * vs:(r + 1) * vs].contiguous(), "lm_head": w["lm_head"][r * vs:(r + 1) * vs].contiguous(),
           "final_norm": w["final_norm"], "layers": []}
    for lw in w["layers"]:
        def col_par(name, t):  # q|k|v and gate|up rows (and their FP8 row scales) sliced per sub-matrix
            if name == "qkv":
                q, k, v = t.split([H * hd, KV * hd, KV * hd], dim=0)
                return torch.cat([q[r * h * hd:(r + 1) * h * hd], k[r * kv * hd:(r + 1) * kv * hd],
                                  v[r * kv * hd:(r + 1) * kv * hd]]).contiguous()
            gate, up = t.chunk(2, dim=0)
            return torch.cat([gate[r * f:(r + 1) * f], up[r * f:(r + 1) * f]]).contiguous()

        o = {"input_norm": lw["input_norm"], "post_norm": lw["post_norm"],
             "qkv": col_par("qkv", lw["qkv"]),
             "o": lw["o"][:, r * h * hd:(r + 1) * h * hd].contiguous(),
             "gate_up": col_par("gate_up", lw["gate_up"]),
             "down": lw["down"][:, r * f:(r + 1) * f].contiguous()}
        # FP8 row scales: column-parallel ones follow their rows; row-parallel (o, down) ones are replicated, since a
        # row scale factors out of each rank's partial sum
        for name in ("qkv", "gate_up"):
            if name + "_scale" in lw:
                o[name + "_scale"] = col_par(name, lw[name + "_scale"])
        for name in ("o", "down"):
            if name + "_scale" in lw:
                o[name + "_scale"] = lw[name + "_scale"]
        for k2 in ("q_norm", "k_norm"):
            if k2 in lw:
                o[k2] = lw[k2]
        out["layers"].append(o)
    return out


def tp_row_amax_max(amax: torch.Tensor) -> torch.Tensor:
    import torch.distributed as dist
    dist.all_reduce(amax, op=dist.ReduceOp.MAX)
    return amax


def load_weights(path: str, spec: ModelSpec, device, tp_size: int = 1, tp_rank: int = 0,
                 quantization: str | None = None, is_target: bool = True, kv_cache_dtype: str = "auto") -> dict:
    """Packed per-rank weights of a synthetic directory or a safetensors checkpoint.  quantization="fp8" replaces the
    decoder linears by e4m3 + per-row scales (quant.py) after loading, one tensor at a time; FP8 checkpoint tensors are
    kept as they are either way.  With tp_size > 1 every rank must call this together: the row scales of o / down come
    from the full rows (a MAX all-reduce over the ranks' column shards).  The draft (is_target=False) is a tp = 1
    replica on rank 0, so its rows are whole and need no reduction.
    kv_cache_dtype="fp8" (target only): w["kv_scales"] = (k_scale, v_scale), per-layer lists of floats from the
    checkpoint (1.0 without them; the same on every tensor-parallel rank)."""
    if not is_target and tp_size != 1:
        raise ValueError("the draft is loaded whole (tp_size = 1) on rank 0")
    if not is_target and kv_cache_dtype != "auto":
        raise ValueError("only the target's KV cache can be FP8; the draft's stays bf16")
    kv8 = kv_cache_dtype == "fp8"
    marker = os.path.join(path, "ssd_b200_synthetic.json")
    if os.path.exists(marker):
        from .synth import generate_weights
        with open(marker) as f:
            w = generate_weights(spec, json.load(f), device, tp_size, tp_rank)
        if kv8:
            w["kv_scales"] = resolve_kv_scales({}, spec.layers, path)
    elif glob.glob(os.path.join(path, "*.safetensors")):
        w = load_safetensors_weights(path, spec, device, tp_size, tp_rank, allow_fp8=True, kv_scales=kv8)
    else:
        raise FileNotFoundError(f"{path}: neither *.safetensors nor ssd_b200_synthetic.json")
    if quantization == "fp8":
        quantize_layers_(w, tp_row_amax_max if tp_size > 1 else None)
        # the freed bf16 matrices and fp32 temporaries go back to the device, so that kv_blocks_for sees them as free
        if torch.device(device).type == "cuda":
            torch.cuda.empty_cache()
    return w


def load_draft_weights(config, spec: ModelSpec, device) -> dict:
    """The draft's packed weights, a whole (tp = 1) replica.  config.draft_quantization="fp8" quantizes its decoder
    linears on load.  An FP8 draft checkpoint loads as FP8 either way (found by its quantization_config in Config, or
    here by its e4m3 tensors), and config.draft_quantization then reads "fp8".  A draft runs in one weight format, so a
    bf16 decoder linear next to FP8 ones is quantized too."""
    wd = load_weights(config.draft, spec, device, quantization=config.draft_quantization, is_target=False)
    if is_fp8(wd) and config.draft_quantization is None:
        config.draft_quantization = "fp8"
        quantize_layers_(wd)
        if torch.device(device).type == "cuda":
            torch.cuda.empty_cache()
    return wd


class _DraftCfg:
    num_kvcache_blocks = 0


def kv_block_bytes(config, spec: ModelSpec, tp_size: int, fp8: bool = False) -> int:
    """Bytes of one KV page (K and V of every layer): 2 bytes per element, 1 for an FP8 (e4m3) cache."""
    return 2 * spec.layers * config.kvcache_block_size * (spec.kv_heads // tp_size) * spec.head_dim * (1 if fp8 else 2)


def kv_blocks_for(config, spec: ModelSpec, tp_size: int, share: float, reserved: int = 0, fp8: bool = False) -> int:
    """allocate_kv_cache (engine/model_runner.py:446-476): blocks that fit in share * gpu_memory_utilization * free,
    capped at what max_num_seqs sequences of max_model_len (+ prefix-cache slack) can ever use.  `reserved` = bytes
    already promised to another cache out of the same free-memory snapshot (the reference sizes the draft cache from
    what REMAINS after the target's, draft_runner.py:27).  fp8: pages of an e4m3 cache (half the bytes)."""
    free, _ = torch.cuda.mem_get_info()
    free = max(0, free - reserved)
    block_bytes = kv_block_bytes(config, spec, tp_size, fp8)
    fit = int(free * config.gpu_memory_utilization * share) // block_bytes
    want = max(config.max_num_seqs, 1) * config.max_blocks * 2 + 2
    return max(1, min(fit, want))


def build_runner(config, tp_size: int = 1, tp_rank: int = 0, device=None, finalize: bool = True):
    device = torch.device(device or "cuda:0")
    torch.cuda.set_device(device)
    tspec = spec_from_config(config.hf_config)
    dspec = spec_from_config(config.draft_hf_config) if config.speculate else None
    kv8 = getattr(config, "kv_cache_dtype", "auto") == "fp8"
    wt = load_weights(config.model, tspec, device, tp_size, tp_rank, quantization=config.quantization,
                      kv_cache_dtype="fp8" if kv8 else "auto")
    if is_fp8(wt):  # an FP8 checkpoint found by its tensor dtypes
        config.quantization = "fp8"
    wd = load_draft_weights(config, dspec, device) if (dspec is not None and tp_rank == 0) else None
    if dspec is not None and tp_rank != 0:
        dspec = None  # the draft is a replica pinned to rank 0 (SURVEY §8e)
    nbt = kv_blocks_for(config, tspec, tp_size, 0.8 if dspec else 1.0, fp8=kv8)
    nbd = kv_blocks_for(config, dspec, 1, 0.75, reserved=nbt * kv_block_bytes(config, tspec, tp_size, kv8)) if dspec else None
    config.num_kvcache_blocks = nbt
    draft_cfg = _DraftCfg()
    draft_cfg.num_kvcache_blocks = nbd or nbt
    runner = PairRunner(tspec, dspec, spec_k=config.speculate_k if config.speculate else 0,  # workers keep K although they hold no draft
                        max_batch=max(1, config.max_num_seqs), block_size=config.kvcache_block_size,
                        max_model_len=config.max_model_len, num_blocks_target=nbt, num_blocks_draft=nbd, device=device,
                        use_graph=config.use_cuda_graph, use_pdl=config.use_pdl, jit_speculate=config.jit_speculate,
                        tp_size=tp_size, tp_rank=tp_rank, draft_fp8=wd is not None and is_fp8(wd),
                        target_kv_scales=wt["kv_scales"] if kv8 else None)
    runner.bind_weights(L.TARGET, wt)
    if wd is not None:
        runner.bind_weights(L.DRAFT, wd)
    if finalize:
        runner.finalize()
    return runner, draft_cfg
