"""Prefill (TTFT) timing of ssdk_forward_tokens in chunks of 64 (round 1) vs 256 tokens (UMMA N = 256 instances of the GEMM):
a 2048-token prompt through the 8B-width target (full depth) and an 8-layer 70B-width target; then the reference bench's
prompt set (16 prompts x 128 tokens) one prompt per call vs packed two to a call (PairRunner.prefill_many); then
prefill_many against prefill_varlen on ragged prompts, prompts sharing a 512-token prefix and the 16 x 128 set (calls, ms
as the median of three alternated warm runs, prompt tok/s, first tokens equal), with the card's name and power limit."""
import atexit
import gc
import os
import random
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ssd_b200 import lib as L, synth  # noqa: E402
from ssd_b200.llm import LLM  # noqa: E402


def close(llm) -> None:
    """Tear an engine down and give its memory back before the next one is built (LLM registers exit with atexit,
    which would otherwise keep its weights and KV cache alive for the whole run)."""
    llm.exit()
    atexit.unregister(llm.exit)
    gc.collect()
    torch.cuda.empty_cache()


for shape, layers in (("llama-3.1-8b", None), ("llama-3.1-70b", 8)):
    root = tempfile.mkdtemp()
    llm = LLM(synth.make_model_dir(root, shape, "target", layers=layers), speculate=True,
              draft=synth.make_model_dir(root, "llama-3.2-1b", "draft", layers=2), speculate_k=6, num_gpus=1, max_num_seqs=1,
              max_model_len=4096, jit_speculate=True)
    r = llm.runner
    random.seed(0)
    prompt = [random.randint(0, 10000) for _ in range(2048)]
    bt = list(range(r.max_blocks))
    out = {}
    for chunk in (64, 256):
        r.prefill(L.TARGET, prompt, bt, chunk=chunk)  # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        tok = r.prefill(L.TARGET, prompt, bt, chunk=chunk)
        torch.cuda.synchronize()
        out[chunk] = (time.perf_counter() - t0, tok)
    L_ = layers or synth.SHAPES[shape][1]
    print(f"{shape} ({L_} layers) 2048-token prefill: chunk 64 {out[64][0] * 1e3:.1f} ms, chunk 256 {out[256][0] * 1e3:.1f} ms "
          f"({out[64][0] / out[256][0]:.2f}x), {2048 / out[256][0]:.0f} tok/s, first token equal: {out[64][1] == out[256][1]}", flush=True)
    del r
    close(llm)
    del llm

# 16 x 128-token prompts (bench/bench.py --random: numseqs 16, input_len 128): one prompt per call vs prefill_many
root = tempfile.mkdtemp()
llm = LLM(synth.make_model_dir(root, "llama-3.1-8b", "target"), speculate=True,
          draft=synth.make_model_dir(root, "llama-3.2-1b", "draft", layers=2), speculate_k=6, num_gpus=1, max_num_seqs=16,
          max_model_len=1024, jit_speculate=True)
r = llm.runner
random.seed(1)
prompts = [[random.randint(0, 10000) for _ in range(128)] for _ in range(16)]
bts = [list(range(b * r.max_blocks, (b + 1) * r.max_blocks)) for b in range(16)]
res = {}
for mode in ("one by one", "packed"):
    for rep in range(2):  # first pass = warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if mode == "packed":
            toks = r.prefill_many(L.TARGET, prompts, bts, [0] * 16)
        else:
            toks = [r.prefill(L.TARGET, prompts[b], bts[b]) for b in range(16)]
        torch.cuda.synchronize()
        res[mode] = (time.perf_counter() - t0, toks)
a, b = res["one by one"], res["packed"]
print(f"llama-3.1-8b, 16 prompts x 128 tokens: one per call {a[0] * 1e3:.1f} ms, packed {b[0] * 1e3:.1f} ms ({a[0] / b[0]:.2f}x), "
      f"{16 * 128 / b[0]:.0f} prompt tok/s, first tokens equal: {a[1] == b[1]}", flush=True)
del r
close(llm)
del llm

# prefill_many (uniform chunk per call; prefix-cache hits one by one) against prefill_varlen (any lengths per call, hits
# join as soon as their pages are written), Llama-3.1-8B + Llama-3.2-1B widths at full depth, both models prefilled
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip().splitlines()[0]
print(f"card: {gpu}", flush=True)
root = tempfile.mkdtemp()
llm = LLM(synth.make_model_dir(root, "llama-3.1-8b", "target"), speculate=True,
          draft=synth.make_model_dir(root, "llama-3.2-1b", "draft"), speculate_k=6, num_gpus=1, max_num_seqs=16,
          max_model_len=1024, jit_speculate=True)
r = llm.runner
rng = random.Random(2)
ragged = [[rng.randint(0, 10000) for _ in range(rng.randint(16, 600))] for _ in range(16)]
prefix = [rng.randint(0, 10000) for _ in range(512)]
shared = [prefix + [rng.randint(0, 10000) for _ in range(rng.randint(16, 128))] for _ in range(16)]
uniform = [[rng.randint(0, 10000) for _ in range(128)] for _ in range(16)]
bs = r.block_size
nxt = 0


def pages(n):
    global nxt
    nxt += -(-n // bs)
    return list(range(nxt - -(-n // bs), nxt))


bts = [pages(len(p)) for p in ragged]
head = pages(512)
bts_shared = [head + pages(len(p) - 512) for p in shared]
starts_shared = [0] + [512] * 15
bts_uniform = [pages(128) for _ in uniform]
cache_blocks = min(r.kv[L.TARGET].shape[2], r.kv[L.DRAFT].shape[2])
print(f"KV cache: {cache_blocks} blocks of {bs} tokens, the prompt sets use {nxt}", flush=True)
assert nxt <= cache_blocks, "KV cache too small for the prompt sets"
for name, prompts, tables, starts in (("16 ragged prompts (16-600 tokens)", ragged, bts, [0] * 16),
                                      ("16 prompts, shared 512-token prefix + 16-128 own", shared, bts_shared, starts_shared),
                                      ("16 x 128 tokens", uniform, bts_uniform, [0] * 16)):
    fns = {"prefill_many": r.prefill_many, "prefill_varlen": r.prefill_varlen}
    res = {k: [] for k in fns}
    ncalls, first = {}, {}
    for rep in range(4):  # alternated; the first round is warm-up
        for k, fn in fns.items():
            calls = []
            fwd_t, fwd_v = r.forward_tokens, r.forward_varlen
            r.forward_tokens = lambda *a, _f=fwd_t, **kw: (calls.append(1), _f(*a, **kw))[1]
            r.forward_varlen = lambda *a, _f=fwd_v, **kw: (calls.append(1), _f(*a, **kw))[1]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            toks = fn(L.TARGET, prompts, tables, starts)
            fn(L.DRAFT, prompts, tables, starts, want_sample=False)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            r.forward_tokens, r.forward_varlen = fwd_t, fwd_v
            if rep > 0:
                res[k].append(dt)
            ncalls[k], first[k] = len(calls), toks
    n_tok = sum(len(p) - s for p, s in zip(prompts, starts))
    line = []
    for k in fns:
        ms = sorted(res[k])[len(res[k]) // 2] * 1e3
        line.append(f"{k}: {ncalls[k]} calls, {ms:.1f} ms, {n_tok / ms * 1e3:.0f} prompt tok/s")
    print(f"{name} ({n_tok} tokens per model, target + draft): " + "; ".join(line) +
          f"; first tokens equal: {first['prefill_many'] == first['prefill_varlen']}", flush=True)
close(llm)
