"""Validate the streaming draft kernel (csrc/draft_stream.cuh, one persistent launch per step for the K draft forwards
and their samplings) against the kernel-per-op path (SSDK_DRAFT_STREAM=0).

    python tools/check_draft_stream.py [--temp 0.7] [--prompt-len 3000] [--parallel]
                                                         # runs the modes in subprocesses and compares; --prompt-len > 1024
                                                         # exercises the long-context attention (16 KV splits); --parallel
                                                         # runs the modes at the same time (correctness only, timings mixed)

Workload: a 2-layer target at Llama-3.1-8B dimensions + the full 16-layer Llama-3.2-1B draft (real draft shapes, synthetic
bigram-agreement weights), k=6, b=1.  SD output equals AR output whatever the draft does, so the check is on the DRAFT
side: the speculated tokens and accept lengths of every step must be identical between the modes, the draft logits of the
last step must agree within bf16 GEMV-vs-tensor-core accumulation noise, and the step time of each mode is printed."""
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


TEMP = float(sys.argv[sys.argv.index("--temp") + 1]) if "--temp" in sys.argv else 0.0
PROMPT = int(sys.argv[sys.argv.index("--prompt-len") + 1]) if "--prompt-len" in sys.argv else 200


def worker(out_path):
    import random

    import numpy as np
    import torch

    from ssd_b200 import lib as L, synth
    from ssd_b200.llm import LLM

    root = tempfile.mkdtemp()
    llm = LLM(synth.make_model_dir(root, "llama-3.1-8b", "target", layers=2), speculate=True,
              draft=synth.make_model_dir(root, "llama-3.2-1b", "draft"), speculate_k=6, num_gpus=1, max_num_seqs=1,
              max_model_len=max(2048, (PROMPT + 24 * 7 + 263) // 256 * 256), jit_speculate=True)
    r = llm.runner
    random.seed(0)
    prompt = [random.randint(0, 10000) for _ in range(PROMPT)]
    bt = list(range(r.max_blocks))
    rec = r.prefill(L.TARGET, prompt, bt)
    r.prefill(L.DRAFT, prompt, bt, want_sample=False)
    ctx, toks_all, nacc_all = len(prompt), [], []
    for _ in range(24):
        toks, nacc, nrec = r.spec_step([ctx], [rec], [bt], [bt], [TEMP], [TEMP], seed=5)
        toks_all.append(toks[0].tolist())
        nacc_all.append(int(nacc[0]))
        ctx += int(nacc[0]) + 1
        rec = int(nrec[0])
    lq = r.logits_q(1).float().cpu().numpy()
    r.stage([ctx], [rec], [bt], [bt], [TEMP], [TEMP])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(4):
        r.step_resident(1)
    e0.record()
    for _ in range(16):
        r.step_resident(1)
    e1.record()
    torch.cuda.synchronize()
    np.savez(out_path, toks=np.array(toks_all), nacc=np.array(nacc_all), lq=lq, ms=e0.elapsed_time(e1) / 16)


def main():
    if len(sys.argv) > 2 and sys.argv[1] == "--worker":
        return worker(sys.argv[2])
    import numpy as np

    res = {}
    tmp = tempfile.mkdtemp()
    modes = (("regular", {"SSDK_DRAFT_STREAM": "0"}), ("stream", {"SSDK_DRAFT_STREAM": "1"}))
    extra = (["--temp", str(TEMP)] if TEMP else []) + ["--prompt-len", str(PROMPT)]
    procs = []
    for mode, env in modes:
        out = os.path.join(tmp, mode + ".npz")
        pr = subprocess.Popen([sys.executable, os.path.abspath(__file__), "--worker", out] + extra, env={**os.environ, **env})
        procs.append((mode, out, pr))
        if "--parallel" not in sys.argv:
            pr.wait(timeout=600)
    for mode, out, pr in procs:
        if pr.wait(timeout=600) != 0:
            sys.exit(f"{mode} run failed (rc={pr.returncode})")
        res[mode] = np.load(out)
    a = res["regular"]
    report = {"temp": TEMP, "prompt_len": PROMPT, "mean_accept_len": float(a["nacc"].mean() + 1), "ms_per_step": {}, "same_tokens": {},
              "draft_logits_max_abs_diff": {}, "draft_logits_max_abs": float(np.abs(a["lq"]).max())}
    bad = False
    for mode, _ in modes:
        b = res[mode]
        report["ms_per_step"][mode] = float(b["ms"])
        if mode == "regular":
            continue
        same = bool((a["toks"] == b["toks"]).all() and (a["nacc"] == b["nacc"]).all())
        err = float(np.abs(a["lq"] - b["lq"]).max())
        report["same_tokens"][mode] = same
        report["draft_logits_max_abs_diff"][mode] = err
        bad = bad or not same or err > 0.02 * report["draft_logits_max_abs"] + 0.05
    print(json.dumps(report))
    if bad:
        sys.exit("the streaming draft kernel disagrees with the kernel-per-op path")


if __name__ == "__main__":
    main()
