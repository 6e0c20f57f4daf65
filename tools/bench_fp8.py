"""bf16 vs FP8 (W8A16) target weights, on one card, with the card's name and power limit printed first.

  gemm     the weight-streaming GEMM instances at the shapes of tools/bench_gemm.py: median of 20 CUDA-event timings per
           case, L2 flushed before each launch; GB/s counts the bytes each variant actually streams (bf16: 2 B per
           weight; FP8: 1 B per weight + 4 B per row scale).
  e2e      Llama-3.1-8B + Llama-3.2-1B synthetic pair (bench.py's default workload: k = 6, b = 1, temp 0, 128-token
           prompt), bf16 target vs quantization="fp8", both engines resident in one process and alternated, 3 runs
           each: `value` (device-resident loop, as bench.py) and `e2e` (LLMEngine.step) tok/s, accept-len, and the
           tokens of both loops against the closed-form greedy chain of the synthetic target.
  prefill  the same pair prefilled (target + draft): 16 x 128-token prompts through prefill_many and the ragged set of
           tools/bench_prefill.py through prefill_many and prefill_varlen; median of three alternated warm runs.
  draft    the e2e workload in four configurations, target / draft = bf16 / bf16, bf16 / FP8, FP8 / bf16 and FP8 / FP8
           (quantization, draft_quantization), all resident in one process and alternated, 3 runs each after a warm-up
           round: `value` and `e2e` tok/s, accept-len, chain mismatches, the draft phase's device time per step (the
           streaming draft kernel, from torch.profiler over 16 resident steps) with the GB/s that implies over the draft's
           weight bytes per step (computed from its shapes, not measured), and the step time with a 3000-token prompt,
           where the draft runs kernel-per-op (as tools/check_draft_stream.py --prompt-len 3000).
    python tools/bench_fp8.py [--sections gemm,e2e,prefill,draft] [--m 1,7,16,64,256] [--out OUT.json]"""
import argparse
import atexit
import gc
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ssd_b200 import ops  # noqa: E402
from ssd_b200.quant import quantize_fp8_rowwise  # noqa: E402

SHAPES = {  # name: (N, K) — same as tools/bench_gemm.py
    "1B.qkv": (3072, 2048), "1B.o": (2048, 2048), "1B.gate_up": (16384, 2048), "1B.down": (2048, 8192),
    "8B.qkv": (6144, 4096), "8B.o": (4096, 4096), "8B.gate_up": (28672, 4096), "8B.down": (4096, 14336),
    "70B.qkv": (10240, 8192), "70B.o": (8192, 8192), "70B.gate_up": (57344, 8192), "70B.down": (8192, 28672),
}


def card() -> dict:
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # noqa: BLE001
        pl = f"unknown ({type(exc).__name__})"
    return {"gpu": name, "power_limit": pl}


def time_ms(fn, flush) -> float:
    for _ in range(3):
        fn()
    ts = []
    for _ in range(20):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def bench_gemm(a, out):
    dev = torch.device("cuda:0")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    for name, (N, K) in SHAPES.items():
        w = (torch.randn(N, K, device=dev) * 0.02).to(torch.bfloat16)
        w8, s = quantize_fp8_rowwise(w)
        silu = name.endswith("gate_up")
        for M in (int(m) for m in a.m.split(",")):
            x = torch.randn(M, K, device=dev).to(torch.bfloat16)
            if silu:
                f16, f8 = (lambda: ops.gate_up_silu(x, w)), (lambda: ops.gate_up_silu_fp8(x, w8, s))
            else:
                f16, f8 = (lambda: ops.linear(x, w)), (lambda: ops.linear_fp8(x, w8, s))
            t16, t8 = time_ms(f16, flush), time_ms(f8, flush)
            rec = {"shape": name, "M": M, "N": N, "K": K, "bf16_ms": round(t16, 4), "fp8_ms": round(t8, 4),
                   "bf16_GBps": round(N * K * 2 / t16 / 1e6, 1), "fp8_GBps": round((N * K + 4 * N) / t8 / 1e6, 1),
                   "speedup": round(t16 / t8, 3)}
            print(json.dumps(rec), flush=True)
            out.append(rec)
        del w, w8, s
    del flush
    torch.cuda.empty_cache()


def _close(llm) -> None:
    llm.exit()
    atexit.unregister(llm.exit)
    gc.collect()
    torch.cuda.empty_cache()


def _pair(root, quantization, draft_quantization=None, **kw):
    from ssd_b200 import synth
    from ssd_b200.llm import LLM
    t = synth.make_model_dir(root, "llama-3.1-8b", "target", seed=0)
    d = synth.make_model_dir(root, "llama-3.2-1b", "draft", seed=0)
    return LLM(t, speculate=True, draft=d, speculate_k=6, num_gpus=1, kvcache_block_size=256, jit_speculate=True,
               quantization=quantization, draft_quantization=draft_quantization, **kw)


def _run_once(llm, prompt, steps, warm):
    """One measurement as bench.py takes it: the device-resident loop (`value`), then LLMEngine.step (`e2e`)."""
    from ssd_b200 import lib as L
    from ssd_b200.engine import llm_engine
    from ssd_b200.sampling_params import SamplingParams
    r = llm.runner
    bt = list(range(r.max_blocks))
    rec = r.prefill(L.TARGET, prompt, bt)
    r.prefill(L.DRAFT, prompt, bt, want_sample=False)
    r.stage([len(prompt)], [rec], [bt], [bt], [0.0], [0.0])
    for _ in range(warm):
        r.step_resident(1)
    torch.cuda.synchronize()
    _, tot0, _ = r.fetch(1)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        r.step_resident(1)
    e1.record()
    torch.cuda.synchronize()
    _, tot1, _ = r.fetch(1)
    value = int(tot1[0] - tot0[0]) / (e0.elapsed_time(e1) / 1e3)
    dev_log = r.resident_log(0)
    llm.add_request(prompt, SamplingParams(temperature=0.0, max_new_tokens=(steps + warm + 4) * 7 + 8, ignore_eos=True))
    seq = llm.scheduler.waiting[-1]
    step = llm.create_inference_step(llm.config)
    for k in llm_engine.METRICS:
        llm_engine.METRICS[k] = [] if isinstance(llm_engine.METRICS[k], list) else 0
    for _ in range(warm + 1):
        llm.step(step)
    torch.cuda.synchronize()
    tok0 = llm_engine.METRICS["decode_total_tokens"]
    t0 = time.perf_counter()
    for _ in range(steps):
        llm.step(step)
    torch.cuda.synchronize()
    e2e = (llm_engine.METRICS["decode_total_tokens"] - tok0) / (time.perf_counter() - t0)
    lens = llm_engine.METRICS["accepted_suffix_lens_with_recovery"]
    while not seq.is_finished:  # retire the request so that the next run starts from an empty scheduler
        llm.step(step)
    return value, e2e, sum(lens) / max(1, len(lens)), dev_log, list(seq.completion_token_ids)


def bench_e2e(a, out):
    from ssd_b200 import synth
    root = tempfile.mkdtemp(prefix="ssd_b200_fp8_")
    pi_t = synth.permutations(synth.SHAPES["llama-3.1-8b"][6], 0, 0.85, "cpu")[0].tolist()

    def mismatches(prompt, toks):
        bad, prev = 0, prompt[-1]
        for t in toks:
            bad += int(t != pi_t[prev])
            prev = t
        return bad

    llms = {q or "bf16": _pair(root, q, max_num_seqs=1, max_model_len=4096) for q in (None, "fp8")}
    res = {k: [] for k in llms}
    for rep in range(4):  # alternated; round 0 is a warm-up
        # a fresh 128-token prompt per round (the same for both engines), so no round hits the prefix cache
        rng = random.Random(rep)
        prompt = [rng.randint(0, 10000) for _ in range(128)]
        for k, llm in llms.items():
            v, e, acc, dlog, elog = _run_once(llm, prompt, a.steps, 8)
            if rep:
                res[k].append({"value": v, "e2e": e, "accept_len": acc, "tokens": len(dlog) + len(elog),
                               "chain_mismatches": mismatches(prompt, dlog) + mismatches(prompt, elog)})
    for k, runs in res.items():
        rec = {"section": "e2e", "target": k, "runs": [{kk: round(vv, 2) if isinstance(vv, float) else vv
                                                         for kk, vv in r_.items()} for r_ in runs]}
        for m in ("value", "e2e"):
            xs = sorted(r_[m] for r_ in runs)
            rec[m] = {"median": round(xs[len(xs) // 2], 1), "min": round(xs[0], 1), "max": round(xs[-1], 1)}
        print(json.dumps(rec), flush=True)
        out.append(rec)
    for llm in llms.values():
        _close(llm)


def _resident(llm, prompt, warm):
    from ssd_b200 import lib as L
    r = llm.runner
    bt = list(range(r.max_blocks))
    rec = r.prefill(L.TARGET, prompt, bt)
    r.prefill(L.DRAFT, prompt, bt, want_sample=False)
    r.stage([len(prompt)], [rec], [bt], [bt], [0.0], [0.0])
    for _ in range(warm):
        r.step_resident(1)
    torch.cuda.synchronize()
    return r


def _draft_phase_ms(llm, prompt, steps=16):
    """Device time per step of the streaming draft kernel (the whole draft phase at this shape), by torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    r = _resident(llm, prompt, 4)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            r.step_resident(1)
        torch.cuda.synchronize()
    us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) for e in prof.key_averages()
             if "draft_stream_kernel" in e.key)
    return us / 1e3 / steps if us else None


def _step_ms(llm, prompt, steps=16):
    r = _resident(llm, prompt, 4)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        r.step_resident(1)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def _draft_bytes_per_step(llm) -> dict:
    """Weight bytes the K draft forwards of one step stream (arithmetic from the shapes): decoder linears at 2 B (bf16)
    or 1 B + 4 B per row scale (FP8), plus the bf16 lm_head."""
    h, k = llm.config.draft_hf_config, llm.config.speculate_k
    d, hd, ffn = h.hidden_size, h.head_dim, h.intermediate_size
    qkv = (h.num_attention_heads + 2 * h.num_key_value_heads) * hd
    weights = qkv * d + d * h.num_attention_heads * hd + 2 * ffn * d + d * ffn
    rows = qkv + d + 2 * ffn + d
    head = h.vocab_size * d * 2
    return {"bf16": k * (h.num_hidden_layers * weights * 2 + head),
            "fp8": k * (h.num_hidden_layers * (weights + 4 * rows) + head)}


def bench_draft(a, out):
    from ssd_b200 import synth
    root = tempfile.mkdtemp(prefix="ssd_b200_fp8_")
    pi_t = synth.permutations(synth.SHAPES["llama-3.1-8b"][6], 0, 0.85, "cpu")[0].tolist()

    def mismatches(prompt, toks):
        bad, prev = 0, prompt[-1]
        for t in toks:
            bad += int(t != pi_t[prev])
            prev = t
        return bad

    configs = {"bf16/bf16": (None, None), "bf16/fp8": (None, "fp8"), "fp8/bf16": ("fp8", None), "fp8/fp8": ("fp8", "fp8")}
    llms = {k: _pair(root, q, dq, max_num_seqs=1, max_model_len=4096) for k, (q, dq) in configs.items()}
    nbytes = _draft_bytes_per_step(next(iter(llms.values())))
    res = {k: [] for k in llms}
    for rep in range(4):  # alternated; round 0 is a warm-up
        rng = random.Random(100 + rep)
        prompt = [rng.randint(0, 10000) for _ in range(128)]
        long_prompt = [rng.randint(0, 10000) for _ in range(3000)]
        for k, llm in llms.items():
            v, e, acc, dlog, elog = _run_once(llm, prompt, a.steps, 8)
            dms = _draft_phase_ms(llm, prompt)
            lms = _step_ms(llm, long_prompt)
            if rep:
                res[k].append({"value": v, "e2e": e, "accept_len": acc, "tokens": len(dlog) + len(elog),
                               "chain_mismatches": mismatches(prompt, dlog) + mismatches(prompt, elog),
                               "draft_ms_per_step": dms, "step_ms_prompt3000": lms})
    for k, runs in res.items():
        fmt = "fp8" if configs[k][1] else "bf16"
        rec = {"section": "draft", "target/draft": k, "draft_GB_per_step": round(nbytes[fmt] / 1e9, 2),
               "runs": [{kk: round(vv, 3) if isinstance(vv, float) else vv for kk, vv in r_.items()} for r_ in runs]}
        for m in ("value", "e2e", "accept_len", "draft_ms_per_step", "step_ms_prompt3000"):
            xs = sorted(r_[m] for r_ in runs if r_[m] is not None)
            if xs:
                rec[m] = {"median": round(xs[len(xs) // 2], 3), "min": round(xs[0], 3), "max": round(xs[-1], 3)}
        rec["chain_mismatches"] = sum(r_["chain_mismatches"] for r_ in runs)
        if "draft_ms_per_step" in rec:
            rec["draft_GBps_implied"] = round(nbytes[fmt] / (rec["draft_ms_per_step"]["median"] * 1e6), 1)
        print(json.dumps(rec), flush=True)
        out.append(rec)
    for llm in llms.values():
        _close(llm)


def bench_prefill(a, out):
    from ssd_b200 import lib as L
    root = tempfile.mkdtemp(prefix="ssd_b200_fp8_")
    llms = {q or "bf16": _pair(root, q, max_num_seqs=16, max_model_len=1024) for q in (None, "fp8")}
    rng = random.Random(2)  # the prompt sets of tools/bench_prefill.py
    ragged = [[rng.randint(0, 10000) for _ in range(rng.randint(16, 600))] for _ in range(16)]
    # bench_prefill.py's shared-prefix set is drawn here (not run) so that the 16 x 128 set below is the same as its own
    _ = [rng.randint(0, 10000) for _ in range(512)]
    for _ in range(16):
        _ = [rng.randint(0, 10000) for _ in range(rng.randint(16, 128))]
    uniform = [[rng.randint(0, 10000) for _ in range(128)] for _ in range(16)]
    bs = next(iter(llms.values())).runner.block_size

    def tables(prompts):
        nxt, out_ = 0, []
        for p in prompts:
            n = -(-len(p) // bs)
            out_.append(list(range(nxt, nxt + n)))
            nxt += n
        return out_

    for name, prompts, fn in (("16 x 128 tokens", uniform, "prefill_many"), ("16 ragged (16-600 tokens)", ragged, "prefill_many"),
                              ("16 ragged (16-600 tokens)", ragged, "prefill_varlen")):
        bts = tables(prompts)
        times, first = {k: [] for k in llms}, {}
        for rep in range(4):
            for k, llm in llms.items():
                f = getattr(llm.runner, fn)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                first[k] = f(L.TARGET, prompts, bts, [0] * 16)
                f(L.DRAFT, prompts, bts, [0] * 16, want_sample=False)
                torch.cuda.synchronize()
                if rep:
                    times[k].append(time.perf_counter() - t0)
        rec = {"section": "prefill", "prompts": name, "path": fn, "tokens_per_model": sum(map(len, prompts))}
        for k, ts in times.items():
            ts.sort()
            rec[f"{k}_ms"] = round(ts[1] * 1e3, 1)
            rec[f"{k}_spread_ms"] = round((ts[-1] - ts[0]) * 1e3, 1)
        rec["fp8_over_bf16"] = round(rec["bf16_ms"] / rec["fp8_ms"], 3)
        print(json.dumps(rec), flush=True)
        out.append(rec)
    for llm in llms.values():
        _close(llm)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sections", default="gemm,e2e,prefill")
    ap.add_argument("--m", default="1,7,16,64,256")
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8 needs a CUDA device")
    out = [card()]
    print(json.dumps(out[0]), flush=True)
    for sec in a.sections.split(","):
        {"gemm": bench_gemm, "e2e": bench_e2e, "prefill": bench_prefill, "draft": bench_draft}[sec](a, out)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    sys.exit(main())
