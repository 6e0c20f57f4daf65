"""The FP8 KV cache kernels' SOURCE on host threads (tests/emu/cuda_emu.h):

* paged attention over e4m3 caches (paged_attn_kernel<HD, MT, true>, paged_attn_varlen_kernel<HD, MT, true> and the
  split-KV merge) on the case ladders of test_attention_emu_cpu.py and test_attention_varlen_emu_cpu.py (pages of 16,
  80 and 256 tokens; GQA 1-16; q_len 1, 7 and 33; 1, 3 and 32 splits; ragged varlen tiles), held to the fp64
  reference on the dequantized caches K = k_scale * code, V = v_scale * code within the unwidened bound of
  tests/attn_ref.py;
* the KV8 rope store (rope_store_kernel<HD, true>), whose bytes must equal e4m3_rne(sat(y / s)) of the bf16 values y
  the bf16 instance stores on the same inputs, bit for bit, with q unchanged and skipped slots (-1) untouched.

SSD_B200_TSAN=1 builds both drivers with ThreadSanitizer: a missing barrier around the raw stages or the widened K/V
buffer shows up as a data race."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from ssd_b200.quant import quantize_kv_fp8
from tests import attn_ref as A
from tests import attn_ref_varlen as AV
from tests import test_attention_emu_cpu as EU
from tests import test_attention_varlen_emu_cpu as EV

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
TSAN = os.environ.get("SSD_B200_TSAN") == "1"
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")

# (k_scale, v_scale): unit, powers of two, and values that are not
SCALES = [(1.0, 1.0), (0.0625, 0.125), (0.0371, 0.0213)]


def _build(name: str, deps: list[str]) -> str:
    src = os.path.join(EMU, name + ".cpp")
    out = os.path.join(EMU, "_build", name + ("_tsan" if TSAN else ""))
    deps = [src, os.path.join(EMU, "cuda_emu.h"), os.path.join(ROOT, "ssd_b200", "csrc", "common.cuh")] + \
        [os.path.join(ROOT, "ssd_b200", "csrc", d) for d in deps]
    if os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps):
        return out
    os.makedirs(os.path.dirname(out), exist_ok=True)
    flags = ["-fsanitize=thread", "-g"] if TSAN else []
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-Wno-unknown-pragmas", "-Wno-attributes", *flags, "-o", out,
                    src], check=True)
    return out


def build_attention() -> str:
    return _build("run_attention_fp8", ["attention.cuh"])


def build_rope() -> str:
    return _build("run_rope_store_fp8", ["elementwise.cuh", "gemm.cuh"])


def quantize_caches(kc, vc, ks, vs):
    """(k codes, v codes) as float8_e4m3fn and the dequantized caches K = ks * code, V = vs * code in fp64."""
    k8, v8 = quantize_kv_fp8(kc, ks), quantize_kv_fp8(vc, vs)
    return k8, v8, k8.double() * ks, v8.double() * vs


def run_attention_emu(tmp_path, binary, *, varlen, B, Q, q_lens, H, KV, hd, bs, ns, q, k8, v8, bt, cl, ks, vs):
    blob = tmp_path / "in.bin"
    with open(blob, "wb") as f:
        np.array([int(varlen), B, Q, H, KV, hd, bs, bt.shape[1], k8.shape[0] * bs, ns], dtype=np.int32).tofile(f)
        if varlen:
            np.array(q_lens, dtype=np.int32).tofile(f)
        np.array([hd ** -0.5, ks, vs], dtype=np.float32).tofile(f)
        q.contiguous().view(torch.int16).numpy().tofile(f)
        for t in (k8, v8):
            t.contiguous().view(torch.uint8).numpy().tofile(f)
        bt.numpy().astype(np.int32).tofile(f)
        cl.numpy().astype(np.int32).tofile(f)
    out = tmp_path / "out.bin"
    res = subprocess.run([binary, str(blob), str(out)], capture_output=True, text=True, timeout=1800)
    assert res.returncode == 0, res.stderr[-2000:]
    assert "ThreadSanitizer" not in res.stderr, res.stderr[:3000]
    plan = tuple(int(x) for x in np.fromfile(out, dtype=np.int32, count=4))
    o = np.fromfile(out, dtype=np.int16, offset=16)
    return plan, torch.from_numpy(o.copy()).view(torch.bfloat16).reshape(q.shape[0], H * hd)


@pytest.mark.parametrize("i", range(len(EU.EMU_CASES)), ids=[c[0] for c in EU.EMU_CASES])
def test_fp8_attention_source_on_host_threads(tmp_path, i):
    binary = build_attention()
    case = EU.EMU_CASES[i]
    name, hd, H, KV, Q, bs, ctx, mb, ns, kind = case
    ks, vs = SCALES[i % len(SCALES)]
    q, kc, vc, bt, cl = EU.case_inputs(case)
    k8, v8, kd, vd = quantize_caches(kc, vc, ks, vs)
    plan, out = run_attention_emu(tmp_path, binary, varlen=False, B=len(ctx), Q=Q, q_lens=None, H=H, KV=KV, hd=hd, bs=bs,
                                  ns=ns, q=q, k8=k8, v8=v8, bt=bt, cl=cl, ks=ks, vs=vs)
    assert plan[3] == ns
    ref, S = A.reference(q, kd, vd, bt, cl, Q, hd ** -0.5)
    r = A.err_over_bound(out, ref, S)
    print(f"[fp8 attention emu] {name} scales ({ks}, {vs}) plan {plan}: worst err/bound {r:.3f}")
    assert r <= 1.0, f"worst err/bound {r:.3f}"


@pytest.mark.parametrize("i", range(len(EV.EMU_CASES)), ids=[c[0] for c in EV.EMU_CASES])
def test_fp8_varlen_attention_source_on_host_threads(tmp_path, i):
    binary = build_attention()
    case = EV.EMU_CASES[i]
    name, hd, H, KV, ql, bs, ctx, mb, ns, kind = case
    ks, vs = SCALES[(i + 1) % len(SCALES)]
    q, kc, vc, bt, cl = EV.case_inputs(case)
    k8, v8, kd, vd = quantize_caches(kc, vc, ks, vs)
    plan, out = run_attention_emu(tmp_path, binary, varlen=True, B=len(ctx), Q=0, q_lens=ql, H=H, KV=KV, hd=hd, bs=bs,
                                  ns=ns, q=q, k8=k8, v8=v8, bt=bt, cl=cl, ks=ks, vs=vs)
    assert plan[3] == ns
    ref, S = AV.reference_varlen(q, kd, vd, bt, cl, ql, hd ** -0.5)
    r = A.err_over_bound(out, ref, S)
    print(f"[fp8 varlen attention emu] {name} scales ({ks}, {vs}) plan {plan}: worst err/bound {r:.3f}")
    assert r <= 1.0, f"worst err/bound {r:.3f}"


def rope_inputs(M, H, KV, hd, nslots, qk_norm, seed):
    g = torch.Generator().manual_seed(seed)
    max_pos = 4096
    pos = torch.randint(0, max_pos, (M,), generator=g, dtype=torch.int64)
    slots = torch.randperm(nslots, generator=g)[:M].to(torch.int32)
    slots[M // 2] = -1  # a skipped row (padding)
    inv = 1.0 / (10000.0 ** (torch.arange(0, hd, 2, dtype=torch.float32) / hd))
    fr = torch.arange(max_pos, dtype=torch.float32)[:, None] * inv[None]
    table = torch.cat([fr.cos(), fr.sin()], dim=1).contiguous()
    qn = (1.0 + 0.1 * torch.randn(hd, generator=g)).to(torch.bfloat16)
    kn = (1.0 + 0.1 * torch.randn(hd, generator=g)).to(torch.bfloat16)
    # wide dynamic range: values that saturate at 448 * s, normal codes and subnormal ones
    qkv = (torch.randn(M, (H + 2 * KV) * hd, generator=g) * torch.exp(3 * torch.randn(M, (H + 2 * KV) * hd,
                                                                                       generator=g))).to(torch.bfloat16)
    return pos, slots, table, qn, kn, qkv


def run_rope_emu(tmp_path, binary, M, H, KV, hd, nslots, qk_norm, ks, vs, inputs):
    pos, slots, table, qn, kn, qkv = inputs
    blob = tmp_path / "in.bin"
    with open(blob, "wb") as f:
        np.array([M, H, KV, hd, table.shape[0], nslots, int(qk_norm)], dtype=np.int32).tofile(f)
        np.array([1e-6, ks, vs], dtype=np.float32).tofile(f)
        pos.numpy().tofile(f)
        slots.numpy().tofile(f)
        table.numpy().tofile(f)
        for t in (qn, kn, qkv):
            t.contiguous().view(torch.int16).numpy().tofile(f)
    out = tmp_path / "out.bin"
    res = subprocess.run([binary, str(blob), str(out)], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    assert "ThreadSanitizer" not in res.stderr, res.stderr[:3000]
    raw = np.fromfile(out, dtype=np.uint8)
    nq, nc = M * H * hd, nslots * KV * hd
    sizes = [2 * nq, 2 * nc, 2 * nc, 2 * nq, nc, nc]
    parts, o = [], 0
    for s in sizes:
        parts.append(torch.from_numpy(raw[o:o + s].copy()))
        o += s
    bf = lambda t, n: t.view(torch.bfloat16).reshape(n, -1)
    return (bf(parts[0], M), bf(parts[1], nslots), bf(parts[2], nslots), bf(parts[3], M),
            parts[4].reshape(nslots, -1), parts[5].reshape(nslots, -1))


@pytest.mark.parametrize("hd,qk_norm", [(64, False), (64, True), (128, False), (128, True)])
def test_fp8_rope_store_equals_quantized_bf16_store(tmp_path, hd, qk_norm):
    binary = build_rope()
    M, H, KV, nslots = 9, 6, 2, 40
    for ks, vs in SCALES:
        inputs = rope_inputs(M, H, KV, hd, nslots, qk_norm, seed=hd + int(qk_norm))
        q, kc, vc, q8, kc8, vc8 = run_rope_emu(tmp_path, binary, M, H, KV, hd, nslots, qk_norm, ks, vs, inputs)
        slots = inputs[1]
        assert torch.equal(q.view(torch.int16), q8.view(torch.int16)), "q differs between the bf16 and KV8 instances"
        written = slots[slots >= 0].long()
        skipped = torch.ones(nslots, dtype=torch.bool)
        skipped[written] = False
        for name, c16, c8, s in (("k", kc, kc8, ks), ("v", vc, vc8, vs)):
            want = quantize_kv_fp8(c16[written], s).view(torch.uint8)
            got = c8[written]
            bad = (want != got).sum().item()
            assert bad == 0, f"{name} cache: {bad} bytes differ from e4m3(sat(bf16 store / {s}))"
            assert (c8[skipped] == 0x5A).all(), f"{name} cache: a skipped or unused slot was written"
        codes = kc8[written].view(torch.float8_e4m3fn).float().abs()
        print(f"[fp8 rope emu] hd {hd} qk_norm {qk_norm} scales ({ks}, {vs}): {written.numel()} rows bit-exact, "
              f"saturated k codes {(codes == 448).sum().item()}, subnormal k codes "
              f"{((codes > 0) & (codes < 2 ** -6)).sum().item()}")
