"""The SOURCE of the FP8 instance of csrc/draft_stream.cuh (draft_stream_kernel<HD, GMAX, true>: e4m3 decoder linears
with fp32 row scales, bf16 lm_head) compiled for the host with tests/emu/cuda_emu.h and checked against the FP8 oracle
(tests/fp8_ref.py) used as the draft: logits of every forward, the K/V written, and the greedy or Philox tokens sampled on
the kernel's own logits.  The geometries cover every FP8 consume shape: K <= 2048 rows (16 per slot), gate|up pairs,
K > 2048 split units at 3072, 4096 and 5120, head_dim 64 and 128 with q/k norm, contexts across the 8 -> 16 KV-split switch,
and a two-row forward 0 with a pending token, which must also equal, bit for bit, a headless launch for the pending token
followed by the one-row forwards.  With SSD_B200_TSAN=1 the emulated kernel is built with ThreadSanitizer and must report
no race."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle.model import ModelCfg, random_weights
from tests.fp8_ref import Fp8OracleModel, quantize_weights

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "emu", "run_draft_stream_fp8.cpp")
BIN = os.path.join(ROOT, "tests", "emu", "_build", "run_draft_stream_fp8")

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


@pytest.mark.parametrize("family,grid,dims,temp,n_fwd,ctx0,bs,pending", [
    ("llama", 3, (256, 512), 0.0, 3, 21, 16, False),   # K <= 2048: 16 rows per slot; gate|up: 16 pairs in two slots
    ("qwen", 2, (256, 512), 0.8, 3, 270, 64, True),    # q/k norm, head_dim 128, Philox sampling, 16 KV splits, pending token
    ("llama", 3, (256, 4096), 0.0, 2, 21, 16, True),   # down K = 4096: 8 rows x 2 segments per slot, both rows' partials
    ("llama", 2, (256, 5120), 0.7, 2, 21, 16, False),  # down K = 5120: 4 rows x 4 segments per slot
    ("qwen", 3, (256, 3072), 0.0, 2, 40, 16, True),    # down K = 3072 (Qwen3-0.6B's): 8 rows x 2 segments of 1536
    ("llama", 2, (256, 512), 0.0, 4, 254, 16, False),  # context 255 .. 258 in one launch: 8 -> 16 KV splits at 257
])
def test_fp8_draft_stream_kernel_source_on_host_threads(tmp_path, family, grid, dims, temp, n_fwd, ctx0, bs, pending):
    from oracle import verify as V
    _build()
    torch.manual_seed(3)
    hd = 64 if family == "llama" else 128
    hidden, ffn = dims
    heads = hidden // hd if family == "llama" else max(2, hidden // hd)
    cfg = ModelCfg(hidden=hidden, layers=2, heads=heads, kv_heads=max(1, heads // 2), head_dim=hd, ffn=ffn, vocab=264,
                   max_pos=512, rms_eps=1e-5 if family == "llama" else 1e-6, rope_theta=500000.0,
                   qk_norm=(family != "llama"))
    w = random_weights(cfg, seed=13)
    wo, we = quantize_weights(w)
    nblk = max(6, (ctx0 + n_fwd) // bs + 2)
    model = Fp8OracleModel(cfg, wo, num_blocks=nblk, block_size=bs)
    bt = [4, 1, 5, 0, 3, 2] + list(range(6, nblk))
    btt = torch.tensor([bt], dtype=torch.int32)
    n = ctx0 - 1 if pending else ctx0  # tokens with K/V in the cache before the launch
    prompt = torch.randint(0, cfg.vocab, (n,))
    slots = torch.tensor([bt[p // bs] * bs + p % bs for p in range(n)], dtype=torch.int32)
    model.forward(prompt, torch.arange(n), slots, torch.tensor([n], dtype=torch.int32), btt, n)
    kv0 = model.kv_cache.clone()
    seed, call_base = 2468, 3 * 16
    pend_tok, first = (91 if pending else -1), 77

    blob = tmp_path / "in.bin"
    with open(blob, "wb") as f:
        np.array([cfg.hidden, cfg.layers, cfg.heads, cfg.kv_heads, hd, cfg.ffn, cfg.vocab, int(cfg.qk_norm), bs, len(bt),
                  nblk * bs, ctx0, n_fwd, grid, cfg.max_pos, 3], dtype=np.int32).tofile(f)
        np.array([cfg.rms_eps, temp], dtype=np.float32).tofile(f)
        np.array([seed, call_base], dtype=np.uint64).tofile(f)
        np.array([pend_tok, first], dtype=np.int64).tofile(f)
        np.array(bt, dtype=np.int32).tofile(f)
        for t in (w["embed"], w["final_norm"], w["lm_head"]):
            _u16(t).tofile(f)
        model.rope.numpy().astype(np.float32).tofile(f)
        ones = torch.ones(hd, dtype=torch.bfloat16)
        for lw in we["layers"]:
            for k in ("qkv", "o", "gate_up", "down"):
                lw[k].contiguous().view(torch.uint8).numpy().tofile(f)
                lw[k + "_scale"].float().numpy().tofile(f)
            for k in ("input_norm", "post_norm"):
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
    assert raw.size == (2 if pending else 1) * per
    if pending:  # the two-row forward 0 == a headless launch for the pending token + the one-row forwards, bit for bit
        for name, (a, b) in {"logits": (0, nl), "k cache": (nl, nl + ncache), "v cache": (nl + ncache, nl + 2 * ncache),
                             "tokens": (nl + 2 * ncache, per)}.items():
            assert np.array_equal(raw[a:b], raw[per + a:per + b]), f"{name}: two-row forward 0 != two launches"
    got = torch.from_numpy(raw[:nl].astype(np.int16)).view(torch.bfloat16).reshape(n_fwd, cfg.vocab)
    kc = torch.from_numpy(raw[nl:nl + ncache].astype(np.int16)).view(torch.bfloat16).float().numpy()
    vc = torch.from_numpy(raw[nl + ncache:nl + 2 * ncache].astype(np.int16)).view(torch.bfloat16).float().numpy()
    toks = np.frombuffer(raw[nl + 2 * ncache:per].tobytes(), dtype=np.int64).tolist()
    assert toks[0] == first and len(toks) == n_fwd + 1

    def fwd(tok, p):
        slot = torch.tensor([bt[p // bs] * bs + p % bs], dtype=torch.int32)
        return model.forward(torch.tensor([tok]), torch.tensor([p]), slot, torch.tensor([p + 1], dtype=torch.int32), btt, 1)

    if pending:
        fwd(pend_tok, ctx0 - 1)
    # the FP8 oracle, teacher-forced on the kernel's tokens
    for step in range(n_fwd):
        want = model.compute_logits(fwd(toks[step], ctx0 + step))[0].float().numpy()
        g = got[step].float().numpy()
        scale = np.abs(want).max()
        assert np.abs(g - want).max() <= 0.02 * scale + 0.02, (step, np.abs(g - want).max(), scale)
        mine = int(V.sample(got[step][None], torch.tensor([temp]), seed, call_base + step)[0])
        assert toks[step + 1] == mine, (step, toks[step + 1], mine)
    ref = model.kv_cache.float().numpy()
    assert np.abs(kc - ref[0].reshape(-1)).max() <= 0.02 * np.abs(ref[0]).max() + 1e-3
    assert np.abs(vc - ref[1].reshape(-1)).max() <= 0.02 * np.abs(ref[1]).max() + 1e-3
    if pending:  # row 0 stored the pending token's K/V
        p = ctx0 - 1
        assert kv0[0][-1, bt[p // bs], p % bs].abs().max() == 0
        assert np.abs(kc.reshape(kv0[0].shape)[-1, bt[p // bs], p % bs]).max() > 0
