"""The SOURCE of csrc/draft_stream.cuh on host threads (tests/emu/cuda_emu.h): forward 0 with a pending token as its
row 0 (the draft KV of the previous step's last draft token, written by the next step's first forward) must produce
exactly what two launches of one-row forwards produce — a headless forward of the pending token, then the step's
forwards of the recovery token: the same K/V bits at every position, the same logits bits of every forward and the same
sampled tokens.  Row 1's attention must see row 0's fresh K/V, which lives in another CTA's cache store; with
SSD_B200_TSAN=1 the emulated kernel is built with ThreadSanitizer and must report no race."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle.model import ModelCfg, OracleModel, random_weights

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "emu", "run_draft_fold.cpp")
BIN = os.path.join(ROOT, "tests", "emu", "_build", "run_draft_fold")

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
TSAN = os.environ.get("SSD_B200_TSAN") == "1"
if TSAN:
    BIN += "_tsan"


def _build():
    deps = [SRC, os.path.join(ROOT, "tests", "emu", "cuda_emu.h"), os.path.join(ROOT, "ssd_b200", "csrc", "draft_stream.cuh"),
            os.path.join(ROOT, "ssd_b200", "csrc", "common.cuh")]
    if os.path.exists(BIN) and all(os.path.getmtime(BIN) >= os.path.getmtime(d) for d in deps):
        return
    os.makedirs(os.path.dirname(BIN), exist_ok=True)
    flags = ["-fsanitize=thread", "-g"] if TSAN else []
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-Wno-unknown-pragmas", "-Wno-attributes", *flags, "-o", BIN, SRC],
                   check=True)


def _u16(t):
    return t.contiguous().view(torch.int16).numpy().astype(np.uint16)


@pytest.mark.parametrize("family,grid,dims,temp,n_fwd,ctx0,bs", [
    ("llama", 3, (256, 512), 0.0, 3, 22, 16),    # K <= 2048 everywhere; the pending token ends a 16-token page
    ("qwen", 2, (256, 512), 0.8, 2, 271, 64),    # q/k norm, head_dim 128, Philox sampling; 16 KV splits for both rows
    ("llama", 3, (256, 4096), 0.0, 2, 21, 16),   # down-proj K = 4096: 4 rows x 2 segments per job, both rows' partials
    ("llama", 2, (256, 512), 0.7, 2, 257, 16),   # row 0 sees 256 tokens (8 KV splits), row 1 257 (16 splits)
])
def test_two_row_forward0_equals_two_launches(tmp_path, family, grid, dims, temp, n_fwd, ctx0, bs):
    _build()
    torch.manual_seed(2)
    hd = 64 if family == "llama" else 128
    hidden, ffn = dims
    heads = hidden // hd if family == "llama" else max(2, hidden // hd)
    cfg = ModelCfg(hidden=hidden, layers=2, heads=heads, kv_heads=max(1, heads // 2), head_dim=hd, ffn=ffn, vocab=264,
                   max_pos=512, rms_eps=1e-5 if family == "llama" else 1e-6, rope_theta=500000.0,
                   qk_norm=(family != "llama"))
    w = random_weights(cfg, seed=11)
    nblk = max(6, (ctx0 + n_fwd) // bs + 2)
    model = OracleModel(cfg, w, num_blocks=nblk, block_size=bs)
    bt = [4, 1, 5, 0, 3, 2] + list(range(6, nblk))
    n = ctx0 - 1  # tokens with K/V in the cache; position ctx0 - 1 is pending
    prompt = torch.randint(0, cfg.vocab, (n,))
    slots = torch.tensor([bt[p // bs] * bs + p % bs for p in range(n)], dtype=torch.int32)
    model.forward(prompt, torch.arange(n), slots, torch.tensor([n], dtype=torch.int32), torch.tensor([bt], dtype=torch.int32), n)
    kv0 = model.kv_cache.clone()

    blob = tmp_path / "in.bin"
    with open(blob, "wb") as f:
        np.array([cfg.hidden, cfg.layers, cfg.heads, cfg.kv_heads, hd, cfg.ffn, cfg.vocab, int(cfg.qk_norm), bs, len(bt),
                  nblk * bs, ctx0, n_fwd, grid, cfg.max_pos, 3], dtype=np.int32).tofile(f)
        np.array([cfg.rms_eps, temp], dtype=np.float32).tofile(f)
        np.array([4321, 5 * 16], dtype=np.uint64).tofile(f)
        np.array([91, 77], dtype=np.int64).tofile(f)
        np.array(bt, dtype=np.int32).tofile(f)
        for t in (w["embed"], w["final_norm"], w["lm_head"]):
            _u16(t).tofile(f)
        model.rope.numpy().astype(np.float32).tofile(f)
        ones = torch.ones(hd, dtype=torch.bfloat16)
        for lw in w["layers"]:
            for k in ("qkv", "o", "gate_up", "down", "input_norm", "post_norm"):
                _u16(lw[k]).tofile(f)
            _u16(lw.get("q_norm", ones)).tofile(f)
            _u16(lw.get("k_norm", ones)).tofile(f)
        _u16(kv0[0]).tofile(f)
        _u16(kv0[1]).tofile(f)
    out = tmp_path / "out.bin"
    res = subprocess.run([BIN, str(blob), str(out)], capture_output=True, text=True, timeout=3000)
    assert res.returncode == 0, res.stderr[-2000:]
    assert "ThreadSanitizer" not in res.stderr, res.stderr[:3000]

    raw = np.fromfile(out, dtype=np.uint16)
    nl = n_fwd * cfg.vocab
    ncache = cfg.layers * nblk * bs * cfg.kv_heads * hd
    per = nl + 2 * ncache + 4 * (n_fwd + 1)
    assert raw.size == 2 * per
    folded, split = raw[:per], raw[per:]
    names = {"logits": (0, nl), "k cache": (nl, nl + ncache), "v cache": (nl + ncache, nl + 2 * ncache),
             "tokens": (nl + 2 * ncache, per)}
    for name, (a, b) in names.items():
        assert np.array_equal(folded[a:b], split[a:b]), f"{name} differs between the folded and the two-launch run"
    # row 0 stored its K/V: the pending slot of the last layer is no longer the (zero) value it had
    kc = torch.from_numpy(folded[nl:nl + ncache].astype(np.int16)).view(torch.bfloat16).reshape(kv0[0].shape)
    p = ctx0 - 1
    assert kv0[0][-1, bt[p // bs], p % bs].abs().max() == 0 and kc[-1, bt[p // bs], p % bs].abs().max() > 0
    toks = np.frombuffer(folded[nl + 2 * ncache:].tobytes(), dtype=np.int64).tolist()
    assert toks[0] == 77 and min(toks) >= 0
