#!/usr/bin/env python
"""Reference GPU arm: the UNMODIFIED reference engine (tanishqkumar/ssd, installed under oracle/_ref by
`__graft_entry__.build()` from the reference checkout, oracle/reference_build.py) driven through its own public
API — `ssd.LLM(...)`, `add_request`, `create_inference_step`, `step` — on this box's GPU: its `LlamaForCausalLM` /
`Qwen3ForCausalLM`, `F.linear` (cuBLAS), its `@torch.compile` regions (Inductor -> Triton), its Triton `store_kvcache`,
its CUDA-graph capture / replay (`capture_cudagraph`, `run_decode_cudagraph`, `run_verify_cudagraph`), its `Sampler`,
`verify()`, `Scheduler` and `BlockManager`.  None of ssd_b200's kernels or engine code is on this path.

What has to be supplied from outside, because the image is not the reference's pinned environment (SURVEY §7/§8c):
  1. `sgl_kernel.flash_attn` (FA3 wheel, absent, Hopper-only): two functions backed by flash_attn 2.8.3, which ships
     sm_90 SASS — the stub BASELINE.md §4.2 prescribes;
  2. checkpoints: none exist in the image, so `ssd.engine.model_runner.load_model` is replaced by a filler that writes
     ssd_b200.synth's seeded synthetic weights (the same tensors our engine runs on) into the reference's own
     nn.Parameters, and `AutoTokenizer.from_pretrained` returns the synthetic "<id>" tokenizer for synthetic dirs;
  3. transformers 5.5 vs the pinned 4.57: `rope_scaling` became an always-present dict, which Qwen3 forwards into an
     `lru_cache`d function (TypeError) — set to None on the loaded HF configs, explicit `rope_theta`.

Prints ONE JSON line: decode tokens/s = METRICS["decode_total_tokens"] / time over K timed `LLMEngine.step()` calls
after W warm-up steps (the reference's own metric, llm_engine.py:204-205), with the generated token ids so the caller can
compare them with ssd_b200's on the same weights and prompt.
"""
from __future__ import annotations

import argparse
import json
import os
import random
import sys
import tempfile
import time
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF_DIR = os.path.join(ROOT, "oracle", "_ref")


def install_flash_attn_stub():
    """`from sgl_kernel.flash_attn import flash_attn_varlen_func, flash_attn_with_kvcache` (ssd/layers/attention.py:6)
    with FA3's call signatures as used at attention.py:90-93,107-111,128-131, served by flash_attn 2.8.3."""
    import flash_attn as fa2

    def flash_attn_with_kvcache(q, k_cache, v_cache, cache_seqlens=None, page_table=None, softmax_scale=None,
                                causal=True, cu_seqlens_q=None, max_seqlen_q=None, **_):
        if cu_seqlens_q is not None:
            # verify: q [B*(K+1), H, hd] with the same K+1 rows per sequence (cu_seqlens_q = arange * (K+1)); FA2's
            # kv-cache kernel takes [B, q_len, H, hd] and aligns the causal mask to the END of cache_seqlens, like FA3
            n, H, hd = q.shape
            ql = int(max_seqlen_q)
            o = fa2.flash_attn_with_kvcache(q.view(n // ql, ql, H, hd), k_cache, v_cache, cache_seqlens=cache_seqlens,
                                            block_table=page_table, softmax_scale=softmax_scale, causal=causal)
            return o.view(n, H, hd)
        return fa2.flash_attn_with_kvcache(q, k_cache, v_cache, cache_seqlens=cache_seqlens, block_table=page_table,
                                           softmax_scale=softmax_scale, causal=causal)

    def flash_attn_varlen_func(q, k, v, max_seqlen_q=None, cu_seqlens_q=None, max_seqlen_k=None, cu_seqlens_k=None,
                               softmax_scale=None, causal=True, **_):
        return fa2.flash_attn_varlen_func(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k,
                                          softmax_scale=softmax_scale, causal=causal)

    m, sub = types.ModuleType("sgl_kernel"), types.ModuleType("sgl_kernel.flash_attn")
    sub.flash_attn_with_kvcache = flash_attn_with_kvcache
    sub.flash_attn_varlen_func = flash_attn_varlen_func
    m.flash_attn = sub
    sys.modules["sgl_kernel"] = m
    sys.modules["sgl_kernel.flash_attn"] = sub


def import_reference():
    if not os.path.isdir(os.path.join(REF_DIR, "ssd")):
        raise RuntimeError(f"{REF_DIR}/ssd missing: run `python -c 'import __graft_entry__ as g; g.build()'` with "
                           "a reference checkout (oracle/reference_build.py; SSD_REFERENCE_DIR overrides its location)")
    os.environ.setdefault("SSD_HF_CACHE", tempfile.gettempdir())
    os.environ.setdefault("SSD_DATASET_DIR", tempfile.gettempdir())
    os.environ.setdefault("SSD_CUDA_ARCH", "9.0")
    for mod in [k for k in sys.modules if k == "ssd" or k.startswith("ssd.")]:
        del sys.modules[mod]
    sys.path.insert(0, REF_DIR)
    sys.path.insert(1, ROOT)
    install_flash_attn_stub()
    try:
        import wandb  # noqa: F401
    except Exception:
        w = types.ModuleType("wandb")
        w.init = w.log = w.finish = lambda *a, **k: None
        sys.modules["wandb"] = w
    import ssd  # noqa: F401  (the reference package; oracle/_ref is first on sys.path)
    assert os.path.realpath(os.path.dirname(ssd.__file__)).startswith(os.path.realpath(REF_DIR)), ssd.__file__
    return ssd


def patch_environment():
    """Items 2 and 3 of the module docstring."""
    import torch
    import ssd.config as rcfg
    import ssd.engine.llm_engine as reng
    import ssd.engine.model_runner as rmr
    import ssd.engine.scheduler as rsch
    from ssd_b200 import synth
    from ssd_b200.runner import ModelSpec

    orig_autoconfig = rcfg.AutoConfig.from_pretrained

    def autoconfig(path, *a, **k):
        cfg = orig_autoconfig(path, *a, **k)
        with open(os.path.join(path, "config.json")) as f:
            raw = json.load(f)
        cfg.rope_scaling = None
        cfg.rope_theta = float(raw.get("rope_theta", 500000.0))
        if getattr(cfg, "head_dim", None) is None:
            cfg.head_dim = cfg.hidden_size // cfg.num_attention_heads
        if not isinstance(getattr(cfg, "torch_dtype", None), torch.dtype):
            cfg.torch_dtype = torch.bfloat16
        return cfg

    class _AC:
        from_pretrained = staticmethod(autoconfig)

    rcfg.AutoConfig = _AC

    class _Tok(synth.SyntheticTokenizer):
        def decode(self, ids, **_):
            return super().decode(ids)

    class _AT:
        @staticmethod
        def from_pretrained(path, *a, **k):
            return _Tok(path)

    reng.AutoTokenizer = _AT
    rmr.AutoTokenizer = _AT
    rsch.AutoTokenizer = _AT

    def fill_synthetic(model, path, target_path=None, target_hidden_size=None):
        with open(os.path.join(path, "ssd_b200_synthetic.json")) as f:
            meta = json.load(f)
        with open(os.path.join(path, "config.json")) as f:
            c = json.load(f)
        spec = ModelSpec(hidden=c["hidden_size"], layers=c["num_hidden_layers"], heads=c["num_attention_heads"],
                         kv_heads=c["num_key_value_heads"], head_dim=c["head_dim"], ffn=c["intermediate_size"],
                         vocab=c["vocab_size"], rms_eps=c["rms_norm_eps"], rope_theta=c["rope_theta"],
                         qk_norm=(c["model_type"] == "qwen3"))
        dev = next(model.parameters()).device
        names = {"input_norm": "input_layernorm.weight", "post_norm": "post_attention_layernorm.weight",
                 "qkv": "self_attn.qkv_proj.weight", "o": "self_attn.o_proj.weight", "gate_up": "mlp.gate_up_proj.weight",
                 "down": "mlp.down_proj.weight", "q_norm": "self_attn.q_norm.weight", "k_norm": "self_attn.k_norm.weight"}
        top = {"embed": "model.embed_tokens.weight", "lm_head": "lm_head.weight", "final_norm": "model.norm.weight"}
        n = 0
        with torch.no_grad():
            for item in synth.iter_weights(spec, meta, dev):
                if item[0] == "layer":
                    for k, t in item[2].items():
                        p = model.get_parameter(f"model.layers.{item[1]}.{names[k]}")
                        assert p.shape == t.shape, (k, p.shape, t.shape)
                        p.data.copy_(t)
                        n += 1
                else:
                    p = model.get_parameter(top[item[0]])
                    assert p.shape == item[1].shape, (item[0], p.shape, item[1].shape)
                    p.data.copy_(item[1])
                    n += 1
        print(f"[ref_gpu] filled {n} synthetic tensors into {type(model).__name__} from {path}", flush=True)

    rmr.load_model = fill_synthetic


def run(args) -> dict:
    import torch
    assert torch.cuda.is_available(), "the reference GPU arm needs a GPU"
    t_start = time.time()
    import_reference()
    patch_environment()
    from ssd import LLM, SamplingParams
    from ssd.engine import llm_engine as reng
    from ssd_b200 import synth
    sys.path.insert(0, ROOT)
    import bench as B  # workload table only

    tshape, dshape, desc = B.WORKLOADS[args.workload]
    K = args.spec_k
    root = tempfile.mkdtemp(prefix="ssd_ref_gpu_")
    need = args.prompt_len + (args.steps + args.warmup + 6) * (K + 1) + 64
    max_len = max(4096, -(-need // 256) * 256)
    tdir = synth.make_model_dir(root, tshape, "target", seed=0, alpha=args.alpha, layers=args.target_layers,
                                o_down_std=args.o_down_std, lm_scale=args.lm_scale)
    ddir = synth.make_model_dir(root, dshape, "draft", seed=0, alpha=args.alpha, o_down_std=args.o_down_std,
                                lm_scale=args.lm_scale)
    llm = LLM(tdir, speculate=True, draft=ddir, speculate_k=K, num_gpus=1, max_num_seqs=1, max_model_len=max_len,
              kvcache_block_size=256, jit_speculate=True, enforce_eager=bool(args.eager), verbose=False,
              max_num_batched_tokens=max(16384, max_len))
    init_s = time.time() - t_start
    random.seed(0)
    prompt = [random.randint(0, 10000) % synth.SHAPES[tshape][6] for _ in range(args.prompt_len)]
    budget = (args.steps + args.warmup + 4) * (K + 1) + 8
    temp = float(args.temp)
    llm.add_request(prompt, SamplingParams(temperature=temp, max_new_tokens=budget, ignore_eos=True))
    step = llm.create_inference_step(llm.config)
    M = reng.METRICS
    for k in M:
        M[k] = [] if isinstance(M[k], list) else 0
    seq = llm.scheduler.waiting[0]
    llm.step(step)  # prefill (target, then draft)
    for _ in range(args.warmup):
        llm.step(step)
    torch.cuda.synchronize()
    tok0 = M["decode_total_tokens"]
    n0 = len(M["accepted_suffix_lens_with_recovery"])
    t0 = time.perf_counter()
    for _ in range(args.steps):
        llm.step(step)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    toks = M["decode_total_tokens"] - tok0
    lens = M["accepted_suffix_lens_with_recovery"][n0:]
    out = {"impl": "reference-gpu", "metric": "decode tokens/sec (sync speculative decoding, accept-len reported)",
           "value": toks / dt, "unit": "tokens/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
           "ms_per_step": dt / args.steps * 1e3, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
           "dtype": "bf16", "data": "synthetic", "accept_len": sum(lens) / max(1, len(lens)),
           "config": {"workload": f"{desc}, sync SD k={K} b=1 temp={temp:g}, TP=1, prompt {args.prompt_len} random tokens, "
                                  f"synthetic bigram-agreement weights alpha={args.alpha} — UNMODIFIED reference engine "
                                  f"(oracle/_ref) on the GPU: F.linear/cuBLAS, torch.compile, its CUDA graphs, "
                                  f"flash_attn 2.8.3 behind the sgl_kernel.flash_attn stub",
                      "enforce_eager": bool(args.eager), "init_s": round(init_s, 1), "torch": torch.__version__},
           "e2e": {"value": toks / dt, "unit": "tokens/s", "h2d_bytes_per_step": None, "d2h_bytes_per_step": None},
           "tokens": [int(t) for t in seq.completion_token_ids[:args.emit_tokens]]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="70b")
    ap.add_argument("--steps", type=int, default=48)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--spec-k", type=int, default=6)
    ap.add_argument("--alpha", type=float, default=0.85)
    ap.add_argument("--prompt-len", type=int, default=128)
    ap.add_argument("--temp", type=float, default=0.0)
    ap.add_argument("--eager", type=int, default=0)
    ap.add_argument("--target-layers", type=int, default=None)
    ap.add_argument("--o-down-std", type=float, default=1e-5)
    ap.add_argument("--emit-tokens", type=int, default=256)
    ap.add_argument("--lm-scale", type=float, default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    try:
        out = run(args)
    except Exception as exc:  # noqa: BLE001 — the caller (bench.py) records the reason in its JSON line
        import traceback
        traceback.print_exc()
        out = {"impl": "reference-gpu", "unavailable": f"{type(exc).__name__}: {exc}"[:400]}
    line = json.dumps(out)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    print(line, flush=True)
    sys.stdout.flush()
    os._exit(0)  # the reference registers an atexit hook that hard-exits anyway (llm_engine.py:124-184)


if __name__ == "__main__":
    main()
