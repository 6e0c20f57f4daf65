"""bf16 vs FP8 (e4m3) target KV cache, on one card, with the card's name and power limit printed first.

  attn      the paged attention kernel (ops.paged_attention vs ops.paged_attention_fp8, + the split-KV merge when the
            plan splits) at the Llama-3.1-8B shape (H 32, KV 8, hd 128) and the Llama-3.1-70B TP=4 rank shape (H 16,
            KV 2): q_len 1, 7 and 256, contexts 1k ... 32k, batch 1 and 8 (q_len 256: batch 1); median of 20 CUDA-event
            timings, L2 flushed before each call.  Each call also allocates its output and scratch from torch's cache
            and clears 16 KB of scratch, the same for both dtypes.  KV MB is what one call streams (B * ctx * KV * hd * 2
            tensors * bytes per element), computed from the shapes.
  e2e       Llama-3.1-8B + Llama-3.2-1B synthetic pair (bench.py's workload: k = 6, b = 1, temp 0), bf16 KV vs
            kv_cache_dtype="fp8", both engines resident in one process and alternated, 3 runs each after a warm-up round,
            at a 128-token prompt and at long prompts: `value` (device-resident loop), `e2e` (LLMEngine.step) tok/s,
            step time, accept-len, and mismatches of both loops against the closed-form greedy chain.
  capacity  the target's KV pages, the tokens they hold and the longest single-sequence context (up to the 128k
            max_model_len), bf16 vs fp8, for the same pair at gpu_memory_utilization 0.5 (memory binds, not the page cap).
    python tools/bench_kv_fp8.py [--sections attn,e2e,capacity] [--prompts 128,4096,16384] [--out OUT.json]"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_fp8 import _close, _pair, _run_once, card, time_ms  # noqa: E402
from ssd_b200 import ops  # noqa: E402
from ssd_b200.quant import quantize_kv_fp8  # noqa: E402

ATTN_SHAPES = {"8B": (32, 8), "70B-tp4": (16, 2)}
CONTEXTS = (1024, 2048, 4096, 8192, 16384, 32768)


def bench_attn(a, out):
    dev = torch.device("cuda:0")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    hd, bs = 128, 256
    for shape, (H, KV) in ATTN_SHAPES.items():
        for q_len, B in ((1, 1), (1, 8), (7, 1), (7, 8), (256, 1)):
            for ctx in CONTEXTS:
                mb = (ctx + bs - 1) // bs
                g = torch.Generator(device=dev).manual_seed(ctx + q_len + B)
                kc = torch.randn(B * mb, bs, KV, hd, device=dev, generator=g).to(torch.bfloat16)
                vc = torch.randn(B * mb, bs, KV, hd, device=dev, generator=g).to(torch.bfloat16)
                k8, v8 = quantize_kv_fp8(kc, 0.05), quantize_kv_fp8(vc, 0.05)
                q = torch.randn(B * q_len, H, hd, device=dev, generator=g).to(torch.bfloat16)
                bt = torch.arange(B * mb, dtype=torch.int32, device=dev).view(B, mb)
                cl = torch.full((B,), ctx, dtype=torch.int32, device=dev)
                f16 = lambda: ops.paged_attention(q, kc, vc, bt, cl, q_len, hd ** -0.5)
                f8 = lambda: ops.paged_attention_fp8(q, k8, v8, bt, cl, q_len, hd ** -0.5, 0.05, 0.05)
                t16, t8 = time_ms(f16, flush), time_ms(f8, flush)
                kv_mb = B * ctx * KV * hd * 2 / 1e6
                rec = {"section": "attn", "shape": shape, "H": H, "KV": KV, "q_len": q_len, "batch": B, "ctx": ctx,
                       "plan": ops.paged_attention_plan(B, q_len, H, KV, mb * bs),
                       "bf16_us": round(t16 * 1e3, 1), "fp8_us": round(t8 * 1e3, 1),
                       "bf16_kv_MB": round(2 * kv_mb, 2), "fp8_kv_MB": round(kv_mb, 2),
                       "bf16_GBps": round(2 * kv_mb / t16, 1), "fp8_GBps": round(kv_mb / t8, 1),
                       "speedup": round(t16 / t8, 3)}
                print(json.dumps(rec), flush=True)
                out.append(rec)
                del kc, vc, k8, v8
    del flush
    torch.cuda.empty_cache()


def bench_e2e(a, out):
    from ssd_b200 import synth
    root = tempfile.mkdtemp(prefix="ssd_b200_kv8_")
    pi_t = synth.permutations(synth.SHAPES["llama-3.1-8b"][6], 0, 0.85, "cpu")[0].tolist()

    def mismatches(prompt, toks):
        bad, prev = 0, prompt[-1]
        for t in toks:
            bad += int(t != pi_t[prev])
            prev = t
        return bad

    prompts = [int(x) for x in a.prompts.split(",")]
    max_len = max(prompts) + (a.steps + 12) * 14 + 256
    llms = {kv: _pair(root, None, max_num_seqs=1, max_model_len=max_len, max_num_batched_tokens=max(16384, max_len),
                  kv_cache_dtype=kv) for kv in ("auto", "fp8")}
    for plen in prompts:
        res = {k: [] for k in llms}
        for rep in range(4):  # alternated; round 0 is a warm-up
            rng = random.Random(rep * 1000 + plen)
            prompt = [rng.randint(0, 10000) for _ in range(plen)]
            for k, llm in llms.items():
                v, e, acc, dlog, elog = _run_once(llm, prompt, a.steps, 8)
                if rep:
                    res[k].append({"value": v, "e2e": e, "accept_len": acc, "step_ms": 1e3 * acc / v,
                                   "tokens": len(dlog) + len(elog),
                                   "chain_mismatches": mismatches(prompt, dlog) + mismatches(prompt, elog)})
        for k, runs in res.items():
            rec = {"section": "e2e", "kv_cache_dtype": k, "prompt_len": plen,
                   "runs": [{kk: round(vv, 3) if isinstance(vv, float) else vv for kk, vv in r_.items()} for r_ in runs]}
            for m in ("value", "e2e", "step_ms"):
                xs = sorted(r_[m] for r_ in runs)
                rec[m] = {"median": round(xs[len(xs) // 2], 2), "min": round(xs[0], 2), "max": round(xs[-1], 2)}
            print(json.dumps(rec), flush=True)
            out.append(rec)
    for llm in llms.values():
        _close(llm)


def capacity_one(kv: str) -> dict:
    root = tempfile.mkdtemp(prefix="ssd_b200_kv8_cap_")
    # max_num_seqs 4 lifts the page cap (max_num_seqs * max_model_len) above what memory allows either way
    llm = _pair(root, None, max_num_seqs=4, max_model_len=131072, max_num_batched_tokens=131072,
                gpu_memory_utilization=0.5, kv_cache_dtype=kv)
    nb, bs = llm.config.num_kvcache_blocks, llm.config.kvcache_block_size
    rec = {"section": "capacity", "kv_cache_dtype": kv, "gpu_memory_utilization": 0.5, "target_pages": nb,
           "page_tokens": bs, "tokens_held": nb * bs, "longest_context": min(nb * bs, llm.config.max_model_len),
           "target_kv_GB": round(llm.runner.kv[0].numel() * llm.runner.kv[0].element_size() / 1e9, 2),
           "draft_pages": llm.draft_cfg.num_kvcache_blocks}
    _close(llm)
    return rec


def bench_capacity(a, out):
    # one process per dtype: both size their caches from the free memory of an otherwise empty device
    for kv in ("auto", "fp8"):
        res = subprocess.run([sys.executable, os.path.abspath(__file__), "--capacity-one", kv], capture_output=True,
                             text=True, timeout=900)
        line = [l for l in res.stdout.splitlines() if l.startswith('{"section": "capacity"')]
        if res.returncode != 0 or not line:
            raise RuntimeError(f"capacity run for {kv} failed:\n{res.stderr[-3000:]}")
        rec = json.loads(line[-1])
        print(json.dumps(rec), flush=True)
        out.append(rec)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sections", default="attn,e2e,capacity")
    ap.add_argument("--prompts", default="128,4096,16384")
    ap.add_argument("--steps", type=int, default=48)
    ap.add_argument("--out", default=None)
    ap.add_argument("--capacity-one", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kv_fp8 needs a CUDA device")
    if a.capacity_one:
        print(json.dumps(capacity_one(a.capacity_one)), flush=True)
        return
    info = card()
    print(json.dumps(info), flush=True)
    out = [info]
    for sec in a.sections.split(","):
        {"attn": bench_attn, "e2e": bench_e2e, "capacity": bench_capacity}[sec](a, out)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
