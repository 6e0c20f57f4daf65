"""The SOURCE of the varlen attention (paged_attn_varlen_kernel + attn_combine_kernel<true> in csrc/attention.cuh)
compiled for the host with tests/emu/cuda_emu.h and held to the fp64 reference within the rounding bound of
tests/attn_ref.py (tests/attn_ref_varlen.py for packed sequences).

Sequences of one launch have their own q_len: tiles come from the engine's tile table (attn_varlen_tiles), the causal
limit of each row is its own sequence's, and the split-KV merge finds the row's tile from the prefix sums.  The cases
cover q_len 1 next to longer ones, lengths that straddle a TQ boundary, one sequence of 256, pages of 16, 80 and 256,
G = 1, 3, 8 and 16, and n_split forced to 1, 3 and 32.  test_varlen_gpu.py runs the same inputs on the device."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from tests import attn_ref as A
from tests import attn_ref_varlen as AV

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "emu", "run_attention_varlen.cpp")
BIN = os.path.join(ROOT, "tests", "emu", "_build", "run_attention_varlen")

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
TSAN = os.environ.get("SSD_B200_TSAN") == "1"
if TSAN:
    BIN += "_tsan"

# (id, hd, H, KV, q_lens, block size, contexts, max_blocks, forced n_split, kind)
EMU_CASES = [
    ("g3_ragged_bs80_split3", 64, 3, 1, [7, 1, 12, 3], 80, [300, 1, 140, 90], None, 3, "needle"),  # TQ 10: 12 straddles
    ("g1_ragged_bs16_split32", 128, 4, 4, [1, 40, 33], 16, [700, 40, 1200], None, 32, "random"),   # TQ 32: 40, 33 straddle
    ("g16_ragged_bs256_split1", 64, 16, 1, [2, 5, 1], 256, [700, 5, 300], None, 1, "needle"),     # TQ 2
    ("g8_q256_bs16_split3", 128, 8, 1, [256], 16, [300], None, 3, "needle"),                        # one sequence of 256
    ("g8_ragged_bs80_split32", 64, 8, 1, [5, 1, 9, 4, 1], 80, [5, 500, 1100, 64, 65], None, 32, "needle"),
    ("g3_alias_bs16_split1", 64, 6, 2, [11, 3], 16, [400, 450], None, 1, "needle"),
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
    name, hd, H, KV, ql, bs, ctx, mb, ns, kind = case
    return AV.make_inputs_varlen(hd, H, KV, ql, bs, ctx, kind=kind, seed=sum(map(ord, name)), max_blocks=mb, n_split=ns,
                                alias=name.startswith("g3_alias"))


def run_emu(tmp_path, case, inputs):
    """Run the emulated kernel; returns (plan (TQ, MT, n_qtiles, n_split, n_tiles), out [sum q_lens, H*hd] bf16)."""
    _, hd, H, KV, ql, bs, ctx, _, ns, _ = case
    q, kc, vc, bt, cl = inputs
    u16 = lambda t: t.contiguous().view(torch.int16).numpy()
    blob = tmp_path / "in.bin"
    with open(blob, "wb") as f:
        np.array([len(ctx), H, KV, hd, bs, bt.shape[1], kc.shape[0] * bs, ns], dtype=np.int32).tofile(f)
        np.array(ql, dtype=np.int32).tofile(f)
        np.array([hd ** -0.5], dtype=np.float32).tofile(f)
        for t in (q, kc, vc):
            u16(t).tofile(f)
        bt.numpy().astype(np.int32).tofile(f)
        cl.numpy().astype(np.int32).tofile(f)
    out = tmp_path / "out.bin"
    res = subprocess.run([BIN, str(blob), str(out)], capture_output=True, text=True, timeout=1800)
    assert res.returncode == 0, res.stderr[-2000:]
    assert "ThreadSanitizer" not in res.stderr, res.stderr[:3000]
    raw = np.fromfile(out, dtype=np.int32, count=5)
    o = np.fromfile(out, dtype=np.int16, offset=20)
    return tuple(int(x) for x in raw), torch.from_numpy(o.copy()).view(torch.bfloat16).reshape(sum(ql), H * hd)


@pytest.mark.parametrize("case", EMU_CASES, ids=[c[0] for c in EMU_CASES])
def test_varlen_attention_kernel_source_on_host_threads(tmp_path, case):
    build()
    _, hd, H, KV, ql, bs, ctx, mb, ns, kind = case
    inputs = case_inputs(case)
    plan, out = run_emu(tmp_path, case, inputs)
    TQ = plan[0]
    assert plan[3] == ns
    assert plan[4] == sum((x + TQ - 1) // TQ for x in ql)
    ref, S = AV.reference_varlen(*inputs, ql, hd ** -0.5)
    r = A.err_over_bound(out, ref, S)
    print(f"[varlen attention emu] {case[0]} plan TQ={plan[0]} MT={plan[1]} n_split={plan[3]} tiles={plan[4]}: "
          f"worst err/bound {r:.3f}")
    assert r <= 1.0, f"worst err/bound {r:.3f}"
