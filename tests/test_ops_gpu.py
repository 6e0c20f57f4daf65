"""GPU parity of the stand-alone ops, called through the C-ABI (ssd_b200.ops -> libssdk.so), against the
CPU oracle / a plain fp32 torch restatement on the same seeded inputs."""
import numpy as np
import pytest
import torch

from tests import attn_ref
from tests.helpers import bf16, load, ulp_mismatch_fraction

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from ssd_b200 import lib
    lib.load()  # fails loudly if libssdk.so is missing
    return torch.device("cuda:0")


def _ref_linear(x, w):
    return (x.double() @ w.double().t())


@pytest.mark.parametrize("M,N,K,split", [
    (1, 512, 128, 1), (7, 512, 128, 1), (7, 3072, 2048, 1), (1, 3072, 2048, 0), (7, 4096, 4096, 0),
    (16, 2048, 8192, 0), (7, 4096, 4096, 3), (33, 1024, 512, 1), (64, 1280, 1024, 0), (7, 16032, 2048, 1),
    (5, 200, 64, 1), (7, 2048, 8192, 8), (7, 1024, 4096, 16), (20, 1024, 2048, 4), (40, 512, 1024, 2),
    # prefill chunks / large batches: UMMA N = 128 and 256 (accumulator drained in passes of 64 token columns)
    (65, 1024, 512, 1), (128, 3072, 2048, 0), (200, 2048, 8192, 0), (256, 4096, 4096, 1), (129, 640, 1024, 2), (256, 512, 256, 1),
])
def test_linear_matches_fp64(dev, M, N, K, split):
    from ssd_b200 import ops
    g = torch.Generator().manual_seed(M * 1000 + N + K)
    x = torch.randn(M, K, generator=g).to(torch.bfloat16).to(dev)
    w = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16).to(dev)
    y = ops.linear(x, w, split_k=split)
    ref = _ref_linear(x, w)
    # fp32 accumulate + one bf16 rounding: error <= 2^-8 |ref| + accumulation noise
    err = (y.double() - ref).abs()
    tol = ref.abs() * 2 ** -8 + 1e-3 * (K ** 0.5) * 0.05
    assert bool((err <= tol).all()), f"max err {float(err.max())}"
    # and bit-level agreement with cuBLAS-style fp32 accumulation on nearly all elements
    y32 = (x.float() @ w.float().t()).to(torch.bfloat16)
    assert ulp_mismatch_fraction(y.cpu(), y32.cpu()) < 0.02


@pytest.mark.parametrize("M,ffn,K", [(1, 256, 128), (7, 8192, 2048), (7, 1024, 512), (40, 512, 256), (3, 200, 128),
                                     (100, 1024, 512), (256, 2048, 1024), (130, 14336, 4096)])
def test_gate_up_silu(dev, M, ffn, K):
    from oracle import ops as O
    from ssd_b200 import ops
    g = torch.Generator().manual_seed(ffn + K + M)
    x = torch.randn(M, K, generator=g).to(torch.bfloat16)
    w = (torch.randn(2 * ffn, K, generator=g) * 0.05).to(torch.bfloat16)
    h = ops.gate_up_silu(x.to(dev), w.to(dev)).cpu()
    gu = (x.float() @ w.float().t()).to(torch.bfloat16)
    ref = O.silu_and_mul(gu)
    # one bf16 ulp is 2^-8 .. 2^-7 relative: allow a one-ulp flip anywhere (rtol 3e-2), and only on a few per cent of the outputs
    torch.testing.assert_close(h.float(), ref.float(), rtol=3e-2, atol=2e-3)
    assert ulp_mismatch_fraction(h, ref) < 0.05


@pytest.mark.parametrize("M,d", [(1, 128), (7, 2048), (7, 8192), (64, 4096), (3, 5120), (256, 4096)])
def test_rms_norm(dev, M, d):
    from oracle import ops as O
    from ssd_b200 import ops
    g = torch.Generator().manual_seed(d + M)
    x = (torch.randn(M, d, generator=g) * 2).to(torch.bfloat16)
    r = (torch.randn(M, d, generator=g) * 2).to(torch.bfloat16)
    w = (1 + 0.2 * torch.randn(d, generator=g)).to(torch.bfloat16)
    y = ops.rms_norm(x.to(dev), w.to(dev), 1e-5).cpu()
    assert ulp_mismatch_fraction(y, O.rms_norm(x, w, 1e-5)) < 2e-3
    y2, r2 = ops.rms_norm(x.to(dev), w.to(dev), 1e-5, r.to(dev))
    ry, rr = O.rms_norm(x, w, 1e-5, r)
    assert torch.equal(r2.cpu(), rr)
    assert ulp_mismatch_fraction(y2.cpu(), ry) < 2e-3
    torch.testing.assert_close(y2.cpu().float(), ry.float(), rtol=1e-2, atol=1e-2)


def test_rms_norm_matches_reference_golden(dev):
    from ssd_b200 import ops
    z = load("layers_compiled.npz")
    x, res, w = bf16(z["norm_x"]).to(dev), bf16(z["norm_res"]).to(dev), bf16(z["norm_w"]).to(dev)
    y, r = ops.rms_norm(x, w, 1e-5, res)
    assert torch.equal(r.cpu(), bf16(z["norm_add_res"]))
    assert ulp_mismatch_fraction(y.cpu(), bf16(z["norm_add_y"])) < 2e-3
    sy = ops.silu_and_mul(bf16(z["silu_x"]).to(dev)).cpu()
    assert ulp_mismatch_fraction(sy, bf16(z["silu_y"])) < 5e-3


@pytest.mark.parametrize("H,KV,hd,qk_norm", [(4, 2, 64, False), (32, 8, 64, False), (8, 2, 128, True), (16, 8, 128, True)])
def test_rope_store_kv(dev, H, KV, hd, qk_norm):
    from oracle import ops as O
    from ssd_b200 import ops
    g = torch.Generator().manual_seed(H * hd)
    M, bs, nblk = 7, 16, 8
    qkv = torch.randn(M, (H + 2 * KV) * hd, generator=g).to(torch.bfloat16)
    pos = torch.tensor([0, 1, 5, 17, 100, 101, 127])
    slots = torch.tensor([3, 4, -1, 20, 21, 22, 127], dtype=torch.int32)
    table = O.rope_table(hd, 128, 500000.0)
    qn = (1 + 0.2 * torch.randn(hd, generator=g)).to(torch.bfloat16) if qk_norm else None
    kn = (1 + 0.2 * torch.randn(hd, generator=g)).to(torch.bfloat16) if qk_norm else None
    kc = torch.zeros(nblk, bs, KV, hd, dtype=torch.bfloat16)
    vc = torch.zeros_like(kc)
    q, k, v = qkv.split([H * hd, KV * hd, KV * hd], dim=-1)
    q, k, v = q.reshape(M, H, hd), k.reshape(M, KV, hd), v.reshape(M, KV, hd)
    if qk_norm:
        q = O.rms_norm(q.reshape(-1, hd), qn, 1e-6).reshape(M, H, hd)
        k = O.rms_norm(k.reshape(-1, hd), kn, 1e-6).reshape(M, KV, hd)
    qr, kr = O.apply_rope(q, pos, table), O.apply_rope(k, pos, table)
    O.store_kvcache(kr, v, kc, vc, slots)
    kcd, vcd = torch.zeros_like(kc).to(dev), torch.zeros_like(vc).to(dev)
    qd = ops.rope_store_kv(qkv.to(dev), pos.to(dev), slots.to(dev), table.to(dev), kcd, vcd, H, KV, hd,
                           qn.to(dev) if qk_norm else None, kn.to(dev) if qk_norm else None, 1e-6)
    assert ulp_mismatch_fraction(qd.cpu(), qr.reshape(M, -1)) < 5e-3
    assert ulp_mismatch_fraction(kcd.cpu(), kc) < 5e-3
    assert torch.equal(vcd.cpu(), vc)
    torch.testing.assert_close(qd.cpu().float(), qr.reshape(M, -1).float(), rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("H,KV,hd", [(4, 1, 64), (32, 8, 64), (32, 8, 128), (8, 1, 128), (16, 8, 128), (2, 2, 64)])
@pytest.mark.parametrize("q_len,ctx", [(1, [1]), (1, [63, 300]), (7, [7]), (7, [64, 65]), (5, [1000, 257]), (40, [40]),
                                       (64, [200]), (200, [200]), (256, [700]), (100, [100, 356])])
def test_paged_attention(dev, H, KV, hd, q_len, ctx):
    from ssd_b200 import ops
    g = torch.Generator().manual_seed(H + KV + hd + q_len + sum(ctx))
    B, bs = len(ctx), 256
    if B * q_len > 256:
        pytest.skip("more than 256 query tokens")
    mb = (max(ctx) + bs - 1) // bs + 1
    nblk = B * mb + 2
    kc = torch.randn(nblk, bs, KV, hd, generator=g).to(torch.bfloat16)
    vc = torch.randn(nblk, bs, KV, hd, generator=g).to(torch.bfloat16)
    perm = torch.randperm(nblk, generator=g)[:B * mb].view(B, mb).to(torch.int32)  # non-contiguous pages
    bt = perm.clone()
    for b in range(B):
        used = (ctx[b] + bs - 1) // bs
        bt[b, used:] = -1
    q = torch.randn(B * q_len, H, hd, generator=g).to(torch.bfloat16)
    cl = torch.tensor(ctx, dtype=torch.int32)
    out = ops.paged_attention(q.to(dev), kc.to(dev), vc.to(dev), bt.to(dev), cl.to(dev), q_len, hd ** -0.5).cpu()
    # fp64 reference, within twice the kernel's two bf16 roundings (tests/attn_ref.py; test_attention_gpu.py has the
    # needle inputs, page sizes, GQA ratios and split plans)
    ref, S = attn_ref.reference(q, kc, vc, bt, cl, q_len, hd ** -0.5)
    r = attn_ref.err_over_bound(out, ref, S)
    assert r <= 1.0, f"worst err/bound {r:.3f}"


def test_sample_greedy_and_ties(dev):
    from ssd_b200 import ops
    z = load("sampler_t0.npz")
    logits = bf16(z["logits"]).to(dev)
    toks = ops.sample(logits, torch.zeros(4, device=dev))
    assert toks.cpu().tolist() == z["tokens"].tolist()  # reference Sampler, incl. the lowest-index tie-break
    big = (torch.randn(3, 128256) * 3).to(torch.bfloat16)
    assert ops.sample(big.to(dev), torch.zeros(3, device=dev)).cpu().tolist() == big.float().argmax(-1).tolist()


def test_sample_temperature_matches_oracle_and_distribution(dev):
    from oracle import verify as V
    from ssd_b200 import ops
    g = torch.Generator().manual_seed(5)
    logits = (torch.randn(4, 4096, generator=g) * 2).to(torch.bfloat16)
    temps = torch.tensor([0.7, 1.0, 0.0, 1.3])
    agree = 0
    for step in range(8):
        got = ops.sample(logits.to(dev), temps.to(dev), seed=123, step_id=step).cpu()
        want = V.sample(logits, temps, seed=123, call_id=step)
        agree += int((got == want).sum())
    assert agree >= 30  # same Philox stream; only fp32 log rounding can flip a near-tie
    # distribution: 2000 draws of a 16-way categorical
    small = torch.tensor([[2.0, 1.0, 0.5, 0.0] * 4]).to(torch.bfloat16)
    cnt = torch.zeros(16)
    for step in range(2000):
        cnt[int(ops.sample(small.to(dev), torch.tensor([1.0], device=dev), seed=7, step_id=step))] += 1
    p = torch.softmax(small.float()[0], -1)
    assert float(((cnt / 2000 - p).abs()).max()) < 0.03


def test_verify_temp0_matches_reference_golden(dev):
    from ssd_b200 import ops
    z = load("verify_t0.npz")
    for c in range(int(z["n_cases"])):
        lp, lq, spec = bf16(z[f"c{c}_lp"]).to(dev), bf16(z[f"c{c}_lq"]).to(dev), torch.from_numpy(z[f"c{c}_spec"]).to(dev)
        B = lp.shape[0]
        zeros = torch.zeros(B, device=dev)
        n, rec = ops.verify(lp, lq, spec, zeros, zeros)
        assert n.cpu().tolist() == z[f"c{c}_nacc"].tolist()
        assert rec.cpu().tolist() == z[f"c{c}_rec"].tolist()


def test_verify_ratio_matches_oracle(dev):
    """temp>0 through the same Philox stream as the oracle: accept counts and recovery tokens agree
    (the oracle itself is pinned to the reference's acceptance probabilities / recovery distributions)."""
    from oracle import verify as V
    from ssd_b200 import ops
    z = load("verify_ratio.npz")
    tot = ok = 0
    for c in range(int(z["n_cases"])):
        lp, lq, spec = bf16(z[f"c{c}_lp"]), bf16(z[f"c{c}_lq"]), torch.from_numpy(z[f"c{c}_spec"])
        tt, tq, jit = z[f"c{c}_cfg"].tolist()
        B = lp.shape[0]
        hits = torch.from_numpy(z[f"c{c}_hits"]) if f"c{c}_hits" in z else None
        for step in range(6):
            suf, rec = V.verify(lp, lq, spec, torch.full((B,), tt), torch.full((B,), tq), hits, bool(jit), None, 99, step)
            n, r = ops.verify(lp.to(dev), lq.to(dev), spec.to(dev), torch.full((B,), tt, device=dev),
                              torch.full((B,), tq, device=dev), hits.to(dev) if hits is not None else None, bool(jit), 99, step)
            tot += 2 * B
            ok += sum(int(a == len(s) - 1) for a, s in zip(n.cpu().tolist(), suf))
            ok += sum(int(a == b) for a, b in zip(r.cpu().tolist(), rec))
    assert ok >= tot - 2, f"{ok}/{tot}"


def test_verify_full_vocab_sizes(dev):
    """BASELINE sizes: V = 128256 (Llama) and 151936 (Qwen), K = 6; size-independent properties."""
    from ssd_b200 import ops
    for V_, K in ((128256, 6), (151936, 6)):
        g = torch.Generator().manual_seed(V_)
        lp = (torch.randn(1, K + 1, V_, generator=g) * 3).to(torch.bfloat16)
        preds = lp.argmax(-1)
        for n_ok in (0, 3, K):
            spec = torch.zeros(1, K + 1, dtype=torch.int64)
            spec[0, 1:1 + n_ok] = preds[0, :n_ok]
            if n_ok < K:
                spec[0, 1 + n_ok] = (preds[0, n_ok] + 1) % V_
            lq = lp[:, :K].clone()
            n, rec = ops.verify(lp.to(dev), lq.to(dev), spec.to(dev), torch.zeros(1, device=dev), torch.zeros(1, device=dev))
            assert int(n) == n_ok and int(rec) == int(preds[0, n_ok])
        # identical p and q at temp>0: every draft token drawn from q is accepted (ratio == 1)
        spec = torch.zeros(1, K + 1, dtype=torch.int64)
        spec[0, 1:] = preds[0, :K]
        t = torch.full((1,), 0.8, device=dev)
        n, rec = ops.verify(lp.to(dev), lp[:, :K].contiguous().to(dev), spec.to(dev), t, t, None, True, 1, 2)
        assert int(n) == K and 0 <= int(rec) < V_
