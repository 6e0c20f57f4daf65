"""The SOURCE of csrc/attention.cuh (paged_attn_kernel + attn_combine_kernel) compiled for the host with
tests/emu/cuda_emu.h — one OS thread per CUDA thread; cp.async, ldmatrix and mma.sync as per-warp exchanges with the
PTX ISA fragment layouts — and held to the fp64 reference within the rounding bound of tests/attn_ref.py.

This runs the kernel's own indexing on a machine without a GPU: page lookup once per chunk (page sizes that are
multiples of 64) and once per 16-byte segment (16, 80), GQA ratios that are and are not powers of two, ragged query
tiles, the causal limit, and the split-KV partials and their merge with one, three and 32 splits.  It says nothing about
the device memory model or speed; test_attention_gpu.py runs the same inputs on the device."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from tests import attn_ref as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "emu", "run_attention.cpp")
BIN = os.path.join(ROOT, "tests", "emu", "_build", "run_attention")

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
# SSD_B200_TSAN=1: build with -fsanitize=thread; a missing __syncthreads around the double-buffered K/V stages or the
# warp-merge buffer is then reported as a data race.
TSAN = os.environ.get("SSD_B200_TSAN") == "1"
if TSAN:
    BIN += "_tsan"

# (id, hd, H, KV, Q, block size, contexts, max_blocks, forced n_split, kind)
EMU_CASES = [
    ("g3_q7_bs80_split3", 64, 3, 1, 7, 80, [300, 7], None, 3, "needle"),          # per-token pages straddle chunks
    ("g1_q1_bs16_split32", 128, 4, 4, 1, 16, [1200], None, 32, "random"),         # 19 chunks: 19 of 32 splits active
    ("g16_q7_bs256_split1", 64, 16, 1, 7, 256, [700], None, 1, "needle"),         # 2 tokens x 16 heads per tile, 4 tiles
    ("g8_q33_bs16_split3", 128, 8, 1, 33, 16, [33], None, 3, "needle"),           # ctx == Q, ragged last tile (33 % 4)
    ("g4_q1_bs80_split32", 64, 8, 2, 1, 80, [1, 500, 1100], None, 32, "needle"),  # context 1, trailing empty splits
    ("g4_q33_bs256_split1", 64, 4, 1, 33, 256, [1100], None, 1, "random"),
    ("g3_q1_bs16_split32", 64, 6, 2, 1, 16, [1150], 80, 32, "needle"),            # 18 chunks: second batch of merge loads
]


def build():
    deps = [SRC, os.path.join(ROOT, "tests", "emu", "cuda_emu.h"), os.path.join(ROOT, "ssd_b200", "csrc", "attention.cuh"),
            os.path.join(ROOT, "ssd_b200", "csrc", "common.cuh")]
    if os.path.exists(BIN) and all(os.path.getmtime(BIN) >= os.path.getmtime(d) for d in deps):
        return
    os.makedirs(os.path.dirname(BIN), exist_ok=True)
    flags = ["-fsanitize=thread", "-g"] if TSAN else []
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-Wno-unknown-pragmas", "-Wno-attributes", *flags, "-o", BIN,
                    SRC], check=True)


def case_inputs(case):
    _, hd, H, KV, Q, bs, ctx, mb, ns, kind = case
    return A.make_inputs(hd, H, KV, Q, bs, ctx, kind=kind, seed=hash((hd, H, KV, Q, bs, len(ctx))) % 10007, max_blocks=mb,
                         n_split=ns)


def run_emu(tmp_path, case, inputs):
    """Run the emulated kernel on `inputs`; returns (plan (TQ, MT, n_qtiles, n_split), out [B*Q, H*hd] bf16)."""
    _, hd, H, KV, Q, bs, ctx, mb, ns, _ = case
    q, kc, vc, bt, cl = inputs
    u16 = lambda t: t.contiguous().view(torch.int16).numpy()
    blob = tmp_path / "in.bin"
    with open(blob, "wb") as f:
        np.array([len(ctx), Q, H, KV, hd, bs, bt.shape[1], kc.shape[0] * bs, ns], dtype=np.int32).tofile(f)
        np.array([hd ** -0.5], dtype=np.float32).tofile(f)
        for t in (q, kc, vc):
            u16(t).tofile(f)
        bt.numpy().astype(np.int32).tofile(f)
        cl.numpy().astype(np.int32).tofile(f)
    out = tmp_path / "out.bin"
    res = subprocess.run([BIN, str(blob), str(out)], capture_output=True, text=True, timeout=1800)
    assert res.returncode == 0, res.stderr[-2000:]
    assert "ThreadSanitizer" not in res.stderr, res.stderr[:3000]
    raw = np.fromfile(out, dtype=np.int32, count=4)
    o = np.fromfile(out, dtype=np.int16, offset=16)
    return tuple(int(x) for x in raw), torch.from_numpy(o.copy()).view(torch.bfloat16).reshape(len(ctx) * Q, H * hd)


@pytest.mark.parametrize("case", EMU_CASES, ids=[c[0] for c in EMU_CASES])
def test_attention_kernel_source_on_host_threads(tmp_path, case):
    build()
    _, hd, H, KV, Q, bs, ctx, mb, ns, kind = case
    inputs = case_inputs(case)
    plan, out = run_emu(tmp_path, case, inputs)
    assert plan[3] == ns
    ref, S = A.reference(*inputs, Q, hd ** -0.5)
    r = A.err_over_bound(out, ref, S)
    print(f"[attention emu] {case[0]} plan TQ={plan[0]} MT={plan[1]} n_qtiles={plan[2]} n_split={plan[3]}: "
          f"worst err/bound {r:.3f}")
    assert r <= 1.0, f"worst err/bound {r:.3f}"
