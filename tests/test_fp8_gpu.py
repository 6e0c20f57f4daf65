"""GPU tests of the FP8 weight-only (W8A16) GEMM instances and of an FP8 target inside whole speculative steps."""
import pytest
import torch

from tests.fp8_ref import Fp8OracleModel, quantize_weights
from tests.helpers import load, trace_cfgs, trace_weights

pytestmark = pytest.mark.gpu
EPS = 0.08
F8 = torch.float8_e4m3fn


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from ssd_b200 import lib
    lib.load()
    return torch.device("cuda:0")


def _finite_codes() -> torch.Tensor:
    codes = torch.arange(256, dtype=torch.int32).to(torch.uint8)
    v = codes.view(F8).float()
    return codes[torch.isfinite(v)]  # 254 codes: everything but the two NaNs (+-0 included)


@pytest.mark.parametrize("M,N,K,split", [(1, 384, 512, 1), (16, 256, 1024, 3), (32, 640, 768, 1), (64, 512, 1024, 8),
                                         (100, 384, 512, 1), (256, 256, 1024, 3),
                                         # N % 128 != 0: the last tile's rows past N (TMA zero fill, no scale read)
                                         (7, 200, 512, 1), (64, 328, 1024, 3), (130, 72, 256, 1)])
@pytest.mark.parametrize("unit_scale", [True, False])
def test_every_e4m3_code_reaches_the_output_exactly(dev, M, N, K, split, unit_scale):
    """W8 holds every finite e4m3 code at many (row, k) positions; each X row is one-hot at a different k, so output
    [m, n] is exactly s[n] * value(W8[n, k_m]): one fp32 product, one bf16 rounding, no sum.  Any conversion,
    swizzle, permutation, tile or split-K indexing error changes an output bit."""
    from ssd_b200 import ops
    g = torch.Generator().manual_seed(M * 7 + N + K + split)
    codes = _finite_codes()
    w8 = codes[torch.randint(0, codes.numel(), (N, K), generator=g)].view(F8)
    ks = torch.randperm(K, generator=g)[:M]
    x = torch.zeros(M, K, dtype=torch.bfloat16)
    x[torch.arange(M), ks] = 1.0
    s = torch.ones(N) if unit_scale else torch.exp2(torch.randn(N, generator=g) * 4) * (1 + torch.rand(N, generator=g))
    y = ops.linear_fp8(x.to(dev), w8.to(dev), s.float().to(dev), split_k=split).cpu()
    want = (w8[:, ks].float().t() * s.float()[None, :]).to(torch.bfloat16)  # [M, N]
    # bit for bit, except that -0 comes out as +0: the accumulator adds the zero products of the other k
    same = (y.view(torch.int16) == want.view(torch.int16)) | ((y == 0) & (want == 0))
    assert bool(same.all()), f"{int((~same).sum())} outputs differ"


_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst_ratio():
    yield
    if _WORST:
        k = max(_WORST, key=_WORST.get)
        print(f"\n[fp8 linear] worst err/bound over {len(_WORST)} cases: {_WORST[k]:.3f} at (M, split) = {k[1:]}")


def _bound_ratio(y, x, w8, s):
    ref = x.double() @ (w8.double() * s.double()[:, None]).t()
    err = (y.double() - ref).abs()
    K = x.shape[1]
    # the bound of test_ops_gpu.py::test_linear_matches_fp64, not widened: one bf16 rounding + fp32 accumulation noise
    tol = ref.abs() * 2 ** -8 + 1e-3 * (K ** 0.5) * 0.05
    return float((err / tol).max())


@pytest.mark.parametrize("M", [1, 7, 16, 20, 40, 64, 65, 128, 200, 256])
@pytest.mark.parametrize("split", [1, 3, 8, 0])
def test_linear_fp8_matches_fp64(dev, M, split):
    from ssd_b200 import ops
    from ssd_b200.quant import quantize_fp8_rowwise
    N, K = 1280, 2048
    g = torch.Generator().manual_seed(M * 10 + split)
    x = torch.randn(M, K, generator=g).to(torch.bfloat16)
    w8, s = quantize_fp8_rowwise((torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16))
    y = ops.linear_fp8(x.to(dev), w8.to(dev), s.to(dev), split_k=split).cpu()
    r = _bound_ratio(y, x, w8, s)
    _WORST[("linear", M, split)] = r
    print(f"[fp8 linear M={M} split={split}] worst err/bound {r:.3f}")
    assert r <= 1.0


@pytest.mark.parametrize("M,split", [(1, 1), (7, 3), (16, 8), (33, 3), (64, 1), (100, 1), (256, 1)])
def test_gate_up_silu_fp8_matches_reference(dev, M, split):
    from oracle import ops as O
    from ssd_b200 import ops
    from ssd_b200.quant import quantize_fp8_rowwise
    from tests.fp8_ref import linear_fp8
    from tests.helpers import ulp_mismatch_fraction
    ffn, K = 1024, 1024
    g = torch.Generator().manual_seed(M + split)
    x = torch.randn(M, K, generator=g).to(torch.bfloat16)
    w8, s = quantize_fp8_rowwise((torch.randn(2 * ffn, K, generator=g) * 0.05).to(torch.bfloat16))
    h = ops.gate_up_silu_fp8(x.to(dev), w8.to(dev), s.to(dev), split_k=split).cpu()
    ref = O.silu_and_mul(linear_fp8(x, w8, s))
    # same tolerance as test_ops_gpu.py::test_gate_up_silu
    torch.testing.assert_close(h.float(), ref.float(), rtol=3e-2, atol=2e-3)
    assert ulp_mismatch_fraction(h, ref) < 0.05


def test_bind_rejects_bad_fp8_weights(dev):
    from ssd_b200 import lib as L
    from ssd_b200.runner import ModelSpec, PairRunner
    spec = ModelSpec(hidden=192, layers=1, heads=3, kv_heads=1, head_dim=64, ffn=256, vocab=512)
    r = PairRunner(spec, spec, spec_k=2, max_batch=1, block_size=64, max_model_len=256)
    w8 = torch.zeros(5 * 64, 192, dtype=F8, device=dev)
    s = torch.ones(5 * 64, device=dev)
    rc = r.lib.ssdk_bind_weight_fp8(r.h, L.TARGET, L.W_QKV, 0, w8.data_ptr(), s.data_ptr(), 320, 192)
    assert rc != 0 and "multiple of 128" in L.last_error()
    rc = r.lib.ssdk_bind_weight_fp8(r.h, L.DRAFT, L.W_QKV, 0, w8.data_ptr(), s.data_ptr(), 320, 192)
    assert rc != 0 and "target model only" in L.last_error()
    rc = r.lib.ssdk_bind_weight_fp8(r.h, L.TARGET, L.W_LM_HEAD, 0, w8.data_ptr(), s.data_ptr(), 512, 192)
    assert rc != 0 and "no FP8 form" in L.last_error()
    r.close()


def _to_dev(w, dev):
    out = {k: v.to(dev).contiguous() for k, v in w.items() if k != "layers"}
    out["layers"] = [{k: v.to(dev).contiguous() for k, v in lw.items()} for lw in w["layers"]]
    return out


def _spec(c):
    from ssd_b200.runner import ModelSpec
    return ModelSpec(hidden=c.hidden, layers=c.layers, heads=c.heads, kv_heads=c.kv_heads, head_dim=c.head_dim, ffn=c.ffn,
                     vocab=c.vocab, rms_eps=c.rms_eps, rope_theta=c.rope_theta, qk_norm=c.qk_norm, max_pos=c.max_pos)


@pytest.mark.parametrize("family", ["llama", "qwen"])
@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("temp", [0.0, 0.7])
def test_fp8_target_spec_steps_match_fp8_oracle(dev, family, use_graph, temp):
    """The trace models with an FP8 target (bf16 draft): 10 speculative steps, the engine's target and draft logits
    against the FP8 oracle (teacher-forced on the engine's tokens); at temperature 0 every decision with a top-2
    margin >= EPS must agree with the oracle's."""
    from oracle.model import OracleModel
    from oracle.spec import SpecSession, check_greedy_step, contiguous_block_tables
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    z = load(f"trace_{family}.npz")
    tc, dc = trace_cfgs(family, z)
    if tc.hidden % 128 or (tc.heads * tc.head_dim) % 128 or tc.ffn % 128:
        pytest.skip("trace shape has a K that is not a multiple of 128")
    K, bs, mb, B = int(z["K"]), int(z["block_size"]), int(z["max_blocks"]), 2
    wt, wd = trace_weights(z, "t"), trace_weights(z, "d")
    wo, we = quantize_weights(wt)
    r = PairRunner(_spec(tc), _spec(dc), spec_k=K, max_batch=B, block_size=bs, max_model_len=bs * mb, use_graph=use_graph,
                   use_pdl=False)
    r.bind_weights(L.TARGET, _to_dev(we, dev))
    r.bind_weights(L.DRAFT, _to_dev(wd, dev))
    r.finalize()
    s = SpecSession(Fp8OracleModel(tc, wo, B * mb, bs), OracleModel(dc, wd, B * mb, bs), K, mb)
    bt = contiguous_block_tables(B, mb)
    prompts = [z["prompt0"].tolist(), z["prompt1"].tolist()]
    rec_o = s.prefill(prompts, [0.0, 0.0], bt, bt.clone())
    bts = [bt[b].tolist() for b in range(B)]
    rec = []
    for b in range(B):
        rec.append(r.prefill(L.TARGET, prompts[b], bts[b]))
        r.prefill(L.DRAFT, prompts[b], bts[b], want_sample=False)
    assert sum(int(a != b_) for a, b_ in zip(rec, rec_o)) <= 1
    rec = list(rec_o)
    ctx = [len(p) for p in prompts]
    for step in range(10):
        toks, nacc, nrec = r.spec_step(ctx, rec, bts, bts, [temp] * B, [temp] * B, seed=5)
        spec = torch.from_numpy(toks)
        lp_o, lq_o = s.spec_step_forced(spec)
        torch.testing.assert_close(r.logits_p(B).cpu().float(), lp_o.float(), atol=0.08, rtol=0.03)
        torch.testing.assert_close(r.logits_q(B).cpu().float(), lq_o.float(), atol=0.08, rtol=0.03)
        if temp == 0.0:
            hard, _ = check_greedy_step(spec, nacc.tolist(), nrec.tolist(), lp_o, lq_o, EPS)
            assert not hard, f"step {step}: {hard}"
        ctx = [c + int(n) + 1 for c, n in zip(ctx, nacc)]
        rec = nrec.tolist()
        s.advance(nacc.tolist(), rec)
    r.close()


@pytest.mark.parametrize("B,prompt_len", [(1, 1012), (4, 60)])
def test_fp8_target_kernel_per_op_paths_match_fp8_oracle(dev, B, prompt_len):
    """A context past 1024 (the kernel-per-op draft at batch 1) and batch 4, with prefill_many, against the FP8 oracle."""
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession, check_greedy_step, contiguous_block_tables
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    K, bs, mb = 4, 64, 18
    tc = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024, max_pos=bs * mb)
    dc = ModelCfg(**{**tc.__dict__, "layers": 1})
    wt = random_weights(tc, 29)
    wd = {"embed": wt["embed"], "lm_head": wt["lm_head"], "final_norm": wt["final_norm"], "layers": [wt["layers"][0]]}
    wo, we = quantize_weights(wt)
    r = PairRunner(_spec(tc), _spec(dc), spec_k=K, max_batch=B, block_size=bs, max_model_len=bs * mb, use_graph=True)
    r.bind_weights(L.TARGET, _to_dev(we, dev))
    r.bind_weights(L.DRAFT, _to_dev(wd, dev))
    r.finalize()
    g = torch.Generator().manual_seed(5 + B)
    prompts = [torch.randint(0, tc.vocab, (prompt_len + 3 * b,), generator=g).tolist() for b in range(B)]
    bt = contiguous_block_tables(B, mb)
    bts = [bt[b].tolist() for b in range(B)]
    s = SpecSession(Fp8OracleModel(tc, wo, B * mb, bs), OracleModel(dc, wd, B * mb, bs), K, mb)
    rec_o = s.prefill(prompts, [0.0] * B, bt, bt.clone())
    rec = r.prefill_many(L.TARGET, prompts, bts, [0] * B)
    r.prefill_many(L.DRAFT, prompts, bts, [0] * B, want_sample=False)
    assert sum(int(a != b_) for a, b_ in zip(rec, rec_o)) <= 1, (rec, rec_o)
    rec, ctx = list(rec_o), [len(p) for p in prompts]
    for step in range(6):
        toks, nacc, nrec = r.spec_step(ctx, rec, bts, bts, [0.0] * B, [0.0] * B)
        spec = torch.from_numpy(toks)
        lp_o, lq_o = s.spec_step_forced(spec)
        torch.testing.assert_close(r.logits_p(B).cpu().float(), lp_o.float(), atol=0.08, rtol=0.03)
        torch.testing.assert_close(r.logits_q(B).cpu().float(), lq_o.float(), atol=0.08, rtol=0.03)
        hard, _ = check_greedy_step(spec, nacc.tolist(), nrec.tolist(), lp_o, lq_o, EPS)
        assert not hard, f"step {step}: {hard}"
        ctx = [c + int(n) + 1 for c, n in zip(ctx, nacc)]
        rec = nrec.tolist()
        s.advance(nacc.tolist(), rec)
    r.close()
