"""GPU tests of the FP8 (e4m3) target KV cache: the stand-alone attention and rope-store ops against the fp64 reference
and the bf16 store, whole speculative steps against the KV-FP8 oracle (tests/kv_fp8_ref.py), two layers at Llama-3.1-8B
widths, LLM.generate with kv_cache_dtype="fp8", checkpoint scales, and a 2-GPU target (skips on one GPU)."""
import socket

import pytest
import torch

from ssd_b200.quant import quantize_kv_fp8
from tests import attn_ref as A
from tests import attn_ref_varlen as AV
from tests.fp8_ref import quantize_weights
from tests.helpers import load, trace_cfgs, trace_weights
from tests.kv_fp8_ref import KvFp8OracleModel
from tests.test_attention_gpu import CASES, _max_blocks, plan_of

pytestmark = pytest.mark.gpu
EPS = 0.08
F8 = torch.float8_e4m3fn
# (k_scale, v_scale): unit, powers of two, and values that are not
SCALES = [(1.0, 1.0), (0.0625, 0.125), (0.0371, 0.0213)]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from ssd_b200 import lib
    lib.load()
    return torch.device("cuda:0")


def _to_dev(w, dev):
    out = {k: v.to(dev).contiguous() for k, v in w.items() if k != "layers"}
    out["layers"] = [{k: v.to(dev).contiguous() for k, v in lw.items()} for lw in w["layers"]]
    return out


def _spec(c):
    from ssd_b200.runner import ModelSpec
    return ModelSpec(hidden=c.hidden, layers=c.layers, heads=c.heads, kv_heads=c.kv_heads, head_dim=c.head_dim, ffn=c.ffn,
                     vocab=c.vocab, rms_eps=c.rms_eps, rope_theta=c.rope_theta, qk_norm=c.qk_norm, max_pos=c.max_pos)


# ------------------------------------------------------------------------------------------------ attention op
_WORST: dict[str, float] = {}


@pytest.mark.parametrize("kind", ["random", "needle"])
@pytest.mark.parametrize("i", range(len(CASES)), ids=[c[0] for c in CASES])
def test_paged_attention_fp8_matches_fp64(dev, i, kind):
    """Every case of test_attention_gpu.CASES over e4m3 caches: within the unwidened bound of the fp64 reference on
    K = k_scale * code, V = v_scale * code, with the plan of the bf16 op."""
    from ssd_b200 import ops
    case = CASES[i]
    name, hd, H, KV, Q, bs, ctx, _, alias = case
    ks, vs = SCALES[i % len(SCALES)]
    pl = plan_of(case)
    q, kc, vc, bt, cl = A.make_inputs(hd, H, KV, Q, bs, ctx, kind=kind, seed=sum(map(ord, name)),
                                      max_blocks=_max_blocks(case), alias=alias, n_split=pl["n_split"])
    k8, v8 = quantize_kv_fp8(kc, ks), quantize_kv_fp8(vc, vs)
    out = ops.paged_attention_fp8(q.to(dev), k8.to(dev), v8.to(dev), bt.to(dev), cl.to(dev), Q, hd ** -0.5, ks, vs).cpu()
    ref, S = A.reference(q, k8.double() * ks, v8.double() * vs, bt, cl, Q, hd ** -0.5)
    r = A.err_over_bound(out, ref, S)
    _WORST[kind] = max(_WORST.get(kind, 0.0), r)
    print(f"[fp8 attention gpu] {name} {kind} scales ({ks}, {vs}): plan {pl}, worst err/bound {r:.3f}")
    assert r <= 1.0, f"worst err/bound {r:.3f}"


@pytest.mark.parametrize("i", range(len(CASES)), ids=[c[0] for c in CASES])
def test_paged_attention_varlen_fp8_matches_fp64(dev, i):
    """The same cases through the varlen op, with the sequences' q_lens made ragged (q, q - 1, ...)."""
    from ssd_b200 import ops
    case = CASES[i]
    name, hd, H, KV, Q, bs, ctx, _, alias = case
    ks, vs = SCALES[(i + 1) % len(SCALES)]
    ql = [max(1, min(Q - (b % 3), ctx[b])) for b in range(len(ctx))]
    q, kc, vc, bt, cl = AV.make_inputs_varlen(hd, H, KV, ql, bs, ctx, kind="needle", seed=sum(map(ord, name)) + 1,
                                              max_blocks=_max_blocks(case), alias=alias)
    k8, v8 = quantize_kv_fp8(kc, ks), quantize_kv_fp8(vc, vs)
    out = ops.paged_attention_varlen_fp8(q.to(dev), k8.to(dev), v8.to(dev), bt.to(dev), cl.to(dev), ql, hd ** -0.5, ks,
                                         vs).cpu()
    ref, S = AV.reference_varlen(q, k8.double() * ks, v8.double() * vs, bt, cl, ql, hd ** -0.5)
    r = A.err_over_bound(out, ref, S)
    _WORST["varlen"] = max(_WORST.get("varlen", 0.0), r)
    print(f"[fp8 varlen attention gpu] {name} q_lens {ql[:4]} scales ({ks}, {vs}): worst err/bound {r:.3f}")
    assert r <= 1.0, f"worst err/bound {r:.3f}"


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("n_split_ctx", [200, 5000])
def test_every_e4m3_code_reaches_the_output_exactly(dev, hd, n_split_ctx):
    """The V cache holds every finite e4m3 code (in rows of hd); query row j singles out token t_j by a score margin that
    underflows every other weight to 0, so output row j is exactly bf16(v_scale * code) of token t_j, bit for bit
    (v_scale a power of two), through one split or many."""
    from ssd_b200 import ops
    codes = torch.arange(256, dtype=torch.int32).to(torch.uint8)
    finite = codes[torch.isfinite(codes.view(F8).float())]
    H = KV = 1
    bs, L = 64, n_split_ctx
    nrows = (finite.numel() + hd - 1) // hd
    mb = (L + bs - 1) // bs
    bt = torch.arange(mb, dtype=torch.int32)[None, :]
    v8 = torch.zeros(mb * bs, hd, dtype=torch.uint8)
    tokens = torch.linspace(0, L - 1, nrows).long()
    for j, t in enumerate(tokens.tolist()):
        chunk = finite[j * hd:(j + 1) * hd]
        v8[t, :chunk.numel()] = chunk
    # K: token t_j has 32 (code 0x60) in direction j, every other key is 0
    k8 = torch.zeros(mb * bs, hd, dtype=torch.uint8)
    for j, t in enumerate(tokens.tolist()):
        k8[t, j] = 0x60
    vs, ks = 0.25, 1.0
    Q = 1
    outs = []
    for j in range(nrows):
        q = torch.zeros(Q, H, hd)
        q[0, 0, j] = 64.0 * hd ** 0.5  # the chosen token scores ~2048 nats, every other one 0
        cl = torch.tensor([L], dtype=torch.int32)
        o = ops.paged_attention_fp8(q.to(torch.bfloat16).to(dev), k8.view(F8).view(mb, bs, 1, hd).to(dev),
                                    v8.view(F8).view(mb, bs, 1, hd).to(dev), bt.to(dev), cl.to(dev), Q, hd ** -0.5,
                                    ks, vs).cpu()
        outs.append(o[0])
    got = torch.stack(outs)  # [nrows, hd]
    want = (v8[tokens].view(F8).float() * vs).to(torch.bfloat16)
    same = (got.view(torch.int16) == want.view(torch.int16)) | ((got == 0) & (want == 0))
    assert bool(same.all()), f"{int((~same).sum())} outputs differ"


def test_fp8_op_at_unit_scales_equals_bf16_op_on_the_same_values(dev):
    """With k_scale = v_scale = 1 the fp8 op must equal the bf16 op run on the widened codes bit for bit: the same
    plan, splits and scratch layout (neither depends on the cache dtype) and the same arithmetic after widening."""
    from ssd_b200 import ops
    for case in CASES[:12]:
        name, hd, H, KV, Q, bs, ctx, _, alias = case
        q, kc, vc, bt, cl = A.make_inputs(hd, H, KV, Q, bs, ctx, kind="random", seed=7, max_blocks=_max_blocks(case),
                                          alias=alias)
        k8, v8 = quantize_kv_fp8(kc, 1.0), quantize_kv_fp8(vc, 1.0)
        a = ops.paged_attention(q.to(dev), k8.to(torch.bfloat16).to(dev), v8.to(torch.bfloat16).to(dev), bt.to(dev),
                                cl.to(dev), Q, hd ** -0.5)
        b = ops.paged_attention_fp8(q.to(dev), k8.to(dev), v8.to(dev), bt.to(dev), cl.to(dev), Q, hd ** -0.5, 1.0, 1.0)
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), name


# ------------------------------------------------------------------------------------------------ rope store
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("qk_norm", [False, True])
def test_rope_store_kv_fp8_equals_quantized_bf16_store(dev, hd, qk_norm):
    from ssd_b200 import ops
    M, H, KV, nslots = 37, 8, 2, 96
    g = torch.Generator().manual_seed(hd + int(qk_norm))
    qkv = (torch.randn(M, (H + 2 * KV) * hd, generator=g) *
           torch.exp(3 * torch.randn(M, (H + 2 * KV) * hd, generator=g))).to(torch.bfloat16).to(dev)
    pos = torch.randint(0, 2048, (M,), generator=g).to(dev)
    slots = torch.randperm(nslots, generator=g)[:M].to(torch.int32)
    slots[5] = -1
    slots = slots.to(dev)
    from ssd_b200.runner import rope_table
    table = rope_table(hd, 2048, 10000.0, dev)
    qn = (1 + 0.1 * torch.randn(hd, generator=g)).to(torch.bfloat16).to(dev) if qk_norm else None
    kn = (1 + 0.1 * torch.randn(hd, generator=g)).to(torch.bfloat16).to(dev) if qk_norm else None
    for ks, vs in SCALES:
        kc = torch.zeros(nslots, KV, hd, dtype=torch.bfloat16, device=dev)
        vc = torch.zeros_like(kc)
        q = ops.rope_store_kv(qkv, pos, slots, table, kc, vc, H, KV, hd, qn, kn)
        k8 = torch.full((nslots, KV, hd), 0x5A, dtype=torch.uint8, device=dev).view(F8)
        v8 = torch.full((nslots, KV, hd), 0x5A, dtype=torch.uint8, device=dev).view(F8)
        q8 = ops.rope_store_kv_fp8(qkv, pos, slots, table, k8, v8, H, KV, hd, ks, vs, qn, kn)
        assert torch.equal(q.view(torch.int16), q8.view(torch.int16))
        w = slots[slots >= 0].long()
        untouched = torch.ones(nslots, dtype=torch.bool, device=dev)
        untouched[w] = False
        for c16, c8, s in ((kc, k8, ks), (vc, v8, vs)):
            assert torch.equal(quantize_kv_fp8(c16[w], s).view(torch.uint8), c8[w].view(torch.uint8))
            assert bool((c8[untouched].view(torch.uint8) == 0x5A).all())


def test_bind_kv_cache_fp8_rejections(dev):
    import numpy as np
    from ssd_b200 import lib as L
    from ssd_b200.runner import ModelSpec, PairRunner
    spec = ModelSpec(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=512)
    r = PairRunner(spec, spec, spec_k=2, max_batch=1, block_size=64, max_model_len=256)
    kv = torch.zeros(2 * 2 * 4 * 64 * 2 * 64, dtype=torch.uint8, device=dev)
    one = np.ones(2, dtype=np.float32)
    p = lambda a: a.ctypes.data_as(L.c_f32p)
    assert r.lib.ssdk_bind_kv_cache_fp8(r.h, L.DRAFT, kv.data_ptr(), 4, p(one), p(one)) != 0
    assert "only the target" in L.last_error()
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        s = np.array([1.0, bad], dtype=np.float32)
        assert r.lib.ssdk_bind_kv_cache_fp8(r.h, L.TARGET, kv.data_ptr(), 4, p(one), p(s)) != 0
        assert "finite and > 0" in L.last_error()
    assert r.lib.ssdk_bind_kv_cache_fp8(r.h, L.TARGET, kv.data_ptr(), 4, p(one), p(one)) == 0
    r.close()


# ------------------------------------------------------------------------------------------------ whole steps
def _run_spec_steps(r, s, prompts, bts, temps, steps, seed=5, prefill="prefill", starts=None):
    from ssd_b200 import lib as L
    from oracle.spec import check_greedy_step
    B = len(prompts)
    bt = torch.tensor(bts, dtype=torch.int32)
    rec_o = s.prefill(prompts, [0.0] * B, bt, bt.clone())
    if prefill == "prefill":
        rec = [r.prefill(L.TARGET, prompts[b], bts[b]) for b in range(B)]
        for b in range(B):
            r.prefill(L.DRAFT, prompts[b], bts[b], want_sample=False)
    elif prefill == "many":
        rec = r.prefill_many(L.TARGET, prompts, bts, [0] * B)
        r.prefill_many(L.DRAFT, prompts, bts, [0] * B, want_sample=False)
    else:
        rec = r.prefill_varlen(L.TARGET, prompts, bts, starts)
        r.prefill_varlen(L.DRAFT, prompts, bts, starts, want_sample=False)
    assert sum(int(a != b_) for a, b_ in zip(rec, rec_o)) <= 1, (rec, rec_o)
    rec, ctx = list(rec_o), [len(p) for p in prompts]
    for step in range(steps):
        toks, nacc, nrec = r.spec_step(ctx, rec, bts, bts, temps, temps, seed=seed)
        spec = torch.from_numpy(toks)
        lp_o, lq_o = s.spec_step_forced(spec)
        lp = r.logits_p(B).cpu().float()
        torch.testing.assert_close(lp, lp_o.float(), atol=0.08, rtol=0.03)
        torch.testing.assert_close(r.logits_q(B).cpu().float(), lq_o.float(), atol=0.08, rtol=0.03)
        if temps[0] == 0.0:
            hard, _ = check_greedy_step(spec, nacc.tolist(), nrec.tolist(), lp_o, lq_o, EPS)
            assert not hard, f"step {step}: {hard}"
            # the engine's own decisions follow its own logits exactly: accepted drafts are its argmaxes
            for b in range(B):
                n = int(nacc[b])
                assert lp[b, :n].argmax(-1).tolist() == toks[b, 1:n + 1].tolist()
                assert int(lp[b, n].argmax()) == int(nrec[b])
        ctx = [c + int(n) + 1 for c, n in zip(ctx, nacc)]
        rec = nrec.tolist()
        s.advance(nacc.tolist(), rec)


@pytest.mark.parametrize("family", ["llama", "qwen"])
@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("temp", [0.0, 0.7])
def test_kv_fp8_spec_steps_match_kv_fp8_oracle(dev, family, use_graph, temp):
    """The trace models with an e4m3 target cache (per-layer scales that are not powers of two): 10 speculative steps,
    target and draft logits against the KV-FP8 oracle teacher-forced on the engine's tokens."""
    from oracle.model import OracleModel
    from oracle.spec import SpecSession, contiguous_block_tables
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    z = load(f"trace_{family}.npz")
    tc, dc = trace_cfgs(family, z)
    K, bs, mb, B = int(z["K"]), int(z["block_size"]), int(z["max_blocks"]), 2
    wt, wd = trace_weights(z, "t"), trace_weights(z, "d")
    ksc = [0.011 * (l + 1) for l in range(tc.layers)]
    vsc = [0.007 * (l + 2) for l in range(tc.layers)]
    r = PairRunner(_spec(tc), _spec(dc), spec_k=K, max_batch=B, block_size=bs, max_model_len=bs * mb, use_graph=use_graph,
                   use_pdl=False, target_kv_scales=(ksc, vsc))
    assert r.kv[L.TARGET].dtype == F8 and r.kv[L.DRAFT].dtype == torch.bfloat16
    r.bind_weights(L.TARGET, _to_dev(wt, dev))
    r.bind_weights(L.DRAFT, _to_dev(wd, dev))
    r.finalize()
    s = SpecSession(KvFp8OracleModel(tc, wt, B * mb, bs, k_scale=ksc, v_scale=vsc), OracleModel(dc, wd, B * mb, bs), K, mb)
    bts = contiguous_block_tables(B, mb).tolist()
    _run_spec_steps(r, s, [z["prompt0"].tolist(), z["prompt1"].tolist()], bts, [temp] * B, 10)
    r.close()


@pytest.mark.parametrize("B,prompt_len,fp8_weights", [(1, 1012, False), (4, 60, False), (2, 300, True)])
def test_kv_fp8_long_context_batch_and_fp8_weights_match_oracle(dev, B, prompt_len, fp8_weights):
    """A context past 1024 tokens, batch 4 through prefill_many, and an e4m3 cache together with quantization="fp8"."""
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession, contiguous_block_tables
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    K, bs, mb = 4, 64, 18
    tc = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024, max_pos=bs * mb)
    dc = ModelCfg(**{**tc.__dict__, "layers": 1})
    wt = random_weights(tc, 29)
    wd = {"embed": wt["embed"], "lm_head": wt["lm_head"], "final_norm": wt["final_norm"], "layers": [wt["layers"][0]]}
    ksc, vsc = [0.03, 0.05], [0.004, 0.0078125]
    if fp8_weights:
        wo, we = quantize_weights(wt)
    else:
        wo, we = wt, wt
    r = PairRunner(_spec(tc), _spec(dc), spec_k=K, max_batch=B, block_size=bs, max_model_len=bs * mb, use_graph=True,
                   target_kv_scales=(ksc, vsc))
    r.bind_weights(L.TARGET, _to_dev(we, dev))
    r.bind_weights(L.DRAFT, _to_dev(wd, dev))
    r.finalize()
    g = torch.Generator().manual_seed(5 + B)
    prompts = [torch.randint(0, tc.vocab, (prompt_len + 3 * b,), generator=g).tolist() for b in range(B)]
    bts = contiguous_block_tables(B, mb).tolist()
    s = SpecSession(KvFp8OracleModel(tc, wo, B * mb, bs, k_scale=ksc, v_scale=vsc), OracleModel(dc, wd, B * mb, bs), K, mb)
    _run_spec_steps(r, s, prompts, bts, [0.0] * B, 6, prefill="many")
    r.close()


def test_kv_fp8_prefill_varlen_with_prefix_hits_matches_oracle(dev):
    """prefill_varlen with prefix-cache hits: sequences 1 and 2 alias the first two pages of sequence 0, whose bytes
    (stored once, by their first writer) both read; then two speculative steps."""
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession
    from ssd_b200.runner import PairRunner
    from ssd_b200 import lib as L
    bs, mb, K = 64, 6, 4
    lens, starts = [200, 150, 200, 140], [0, 128, 128, 0]
    B = len(lens)
    c = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024, max_pos=bs * mb)
    dc = ModelCfg(**{**c.__dict__, "layers": 1})
    wt = random_weights(c, 41)
    wd = {"embed": wt["embed"], "lm_head": wt["lm_head"], "final_norm": wt["final_norm"], "layers": [wt["layers"][0]]}
    ksc, vsc = [0.02, 0.04], [0.01, 0.003]
    r = PairRunner(_spec(c), _spec(dc), spec_k=K, max_batch=B, block_size=bs, max_model_len=bs * mb, use_graph=True,
                   target_kv_scales=(ksc, vsc))
    r.bind_weights(L.TARGET, _to_dev(wt, dev))
    r.bind_weights(L.DRAFT, _to_dev(wd, dev))
    r.finalize()
    bts = [list(range(b * mb, (b + 1) * mb)) for b in range(B)]
    for i in (1, 2):
        bts[i][:2] = bts[0][:2]
    g = torch.Generator().manual_seed(17)
    prefix = torch.randint(0, c.vocab, (128,), generator=g).tolist()
    prompts = [prefix + torch.randint(0, c.vocab, (n - 128,), generator=g).tolist() for n in lens]
    s = SpecSession(KvFp8OracleModel(c, wt, B * mb, bs, k_scale=ksc, v_scale=vsc), OracleModel(dc, wd, B * mb, bs), K, mb)
    _run_spec_steps(r, s, prompts, bts, [0.0] * B, 2, prefill="varlen", starts=starts)
    r.close()


def test_kv_fp8_at_llama8b_widths_matches_oracle():
    """Two decoder layers at Llama-3.1-8B widths (H 32, KV 8, hd 128), full 128256 vocabulary, a 200-token prompt, e4m3
    target cache: first token and three speculative steps against the KV-FP8 oracle on the host, within the true-width
    test's logit bounds."""
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession, check_greedy_step
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    dev = torch.device("cuda:0")
    bs, mb, K = 256, 2, 4
    tc = ModelCfg(hidden=4096, layers=2, heads=32, kv_heads=8, head_dim=128, ffn=14336, vocab=128256, max_pos=bs * mb)
    dc = ModelCfg(hidden=2048, layers=1, heads=32, kv_heads=8, head_dim=64, ffn=8192, vocab=128256, max_pos=bs * mb)
    wt, wd = random_weights(tc, 3), random_weights(dc, 4)
    ksc, vsc = [0.0123, 0.0187], [0.0051, 0.0094]
    r = PairRunner(_spec(tc), _spec(dc), spec_k=K, max_batch=1, block_size=bs, max_model_len=bs * mb, use_graph=True,
                   target_kv_scales=(ksc, vsc))
    r.bind_weights(L.TARGET, _to_dev(wt, dev))
    r.bind_weights(L.DRAFT, _to_dev(wd, dev))
    r.finalize()
    g = torch.Generator().manual_seed(11)
    prompt = torch.randint(0, tc.vocab, (200,), generator=g).tolist()
    bt = torch.arange(mb, dtype=torch.int32)[None, :]
    s = SpecSession(KvFp8OracleModel(tc, wt, mb, bs, k_scale=ksc, v_scale=vsc), OracleModel(dc, wd, mb, bs), K, mb)
    rec_o = s.prefill([prompt], [0.0], bt, bt.clone())
    rec = r.prefill(L.TARGET, prompt, bt[0].tolist())
    r.prefill(L.DRAFT, prompt, bt[0].tolist(), want_sample=False)
    want = s.t.compute_logits(s._forward(s.t, torch.tensor(prompt), [0], len(prompt), bt)[-1:])[0].float()
    got = r.logits_last(1)[0].float().cpu()
    torch.testing.assert_close(got, want, atol=0.25, rtol=1 / 32)
    top2 = want.topk(2).values
    assert rec == rec_o[0] or float(top2[0] - top2[1]) < EPS, (rec, rec_o)
    rec, ctx = rec_o[0], len(prompt)
    for step in range(3):
        toks, nacc, nrec = r.spec_step([ctx], [rec], [bt[0].tolist()], [bt[0].tolist()], [0.0], [0.0])
        spec = torch.from_numpy(toks)
        lp_o, lq_o = s.spec_step_forced(spec)
        for eng, ref in ((r.logits_p(1), lp_o), (r.logits_q(1), lq_o)):
            torch.testing.assert_close(eng.cpu().float(), ref.float(), atol=0.25, rtol=1 / 32)
        hard, _ = check_greedy_step(spec, nacc.tolist(), nrec.tolist(), lp_o, lq_o, EPS)
        assert not hard, f"step {step}: {hard}"
        ctx += int(nacc[0]) + 1
        rec = int(nrec[0])
        s.advance(nacc.tolist(), [rec])
    r.close()


# ------------------------------------------------------------------------------------------------ public interface
def _generate(target, draft, prompts, **kw):
    from ssd_b200 import LLM, SamplingParams
    from ssd_b200 import lib as L
    llm = LLM(target, speculate=True, draft=draft, speculate_k=4, max_num_seqs=3, max_model_len=1024,
              kvcache_block_size=64, **kw)
    out, _ = llm.generate(prompts, SamplingParams(temperature=0.0, max_new_tokens=24, ignore_eos=True), use_tqdm=False)
    info = (llm.config.kv_cache_dtype, llm.runner.kv[L.TARGET].dtype, llm.runner.kv[L.DRAFT].dtype, llm.runner.kv_scales)
    llm.exit()
    return [o["token_ids"] for o in out], info


def test_llm_generate_synthetic_pair_with_kv_fp8(tmp_path):
    """LLM.generate on the synthetic pair with kv_cache_dtype="fp8" emits the bf16 run's tokens.  This is a weak check:
    the synthetic target's o / down projections are ~0, so attention barely moves its logits; the oracle tests above
    are the strong ones.  It pins the plumbing: the option, the e4m3 target cache, the bf16 draft cache, unit scales."""
    from ssd_b200 import synth
    t = synth.make_model_dir(str(tmp_path), "llama-tiny-target", "target", seed=0)
    d = synth.make_model_dir(str(tmp_path), "llama-tiny-draft", "draft", seed=0)
    g = torch.Generator().manual_seed(2)
    prompts = [torch.randint(2, 1000, (n,), generator=g).tolist() for n in (9, 130, 40)]
    ta, ia = _generate(t, d, prompts)
    tb, ib = _generate(t, d, prompts, kv_cache_dtype="fp8")
    assert ia[:3] == ("auto", torch.bfloat16, torch.bfloat16) and ia[3] is None
    assert ib[:3] == ("fp8", F8, torch.bfloat16)
    assert ib[3] == ([1.0] * len(ib[3][0]), [1.0] * len(ib[3][1]))
    assert ta == tb


def test_checkpoint_kv_scales_reach_the_device(tmp_path):
    """A checkpoint carrying fp32 self_attn.k_scale / v_scale scalars loaded with kv_cache_dtype="fp8": the runner binds
    exactly those fp32 values (not bf16-rounded ones); with "auto" the same checkpoint generates exactly as one without
    them."""
    from oracle.model import ModelCfg, random_weights
    from safetensors.torch import load_file, save_file
    from ssd_b200 import synth
    from tests.test_fp8_engine_gpu import _write_checkpoint
    c = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024, max_pos=2048)
    w = random_weights(c, 13)
    plain = _write_checkpoint(tmp_path / "llama-tiny-plain", c, w, fp8=False)
    scaled = _write_checkpoint(tmp_path / "llama-tiny-scaled", c, w, fp8=False)
    t = load_file(scaled + "/model.safetensors")
    ks = [0.0213, 0.0371]
    vs = [0.0119, 0.0078125]
    for l in range(c.layers):
        t[f"model.layers.{l}.self_attn.k_scale"] = torch.tensor(ks[l], dtype=torch.float32)
        t[f"model.layers.{l}.self_attn.v_scale"] = torch.tensor(vs[l], dtype=torch.float32)
    save_file(t, scaled + "/model.safetensors")
    draft = synth.make_model_dir(str(tmp_path), "llama-tiny-draft", "draft", seed=1, max_position_embeddings=2048)
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(2, 1000, (n,), generator=g).tolist() for n in (5, 70)]
    ta, _ = _generate(plain, draft, prompts, tokenizer_path=draft)
    tb, _ = _generate(scaled, draft, prompts, tokenizer_path=draft)
    assert ta == tb  # "auto" ignores the scale tensors
    _, info = _generate(scaled, draft, prompts, tokenizer_path=draft, kv_cache_dtype="fp8")
    assert info[0] == "fp8" and info[1] == F8
    assert info[3] == ([torch.tensor(x).item() for x in ks], [torch.tensor(x).item() for x in vs])


# ------------------------------------------------------------------------------------------------ tensor parallel
def _free_port():
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        return sk.getsockname()[1]


def _rank_main(rank, world, port, q):
    import torch.distributed as dist
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession, check_greedy_step, contiguous_block_tables
    from ssd_b200 import lib as L
    from ssd_b200.loader import shard_packed_weights
    from ssd_b200.parallel import bind_symmetric_memory, create_nccl_comm
    from ssd_b200.runner import PairRunner
    try:
        torch.cuda.set_device(rank)
        dev = torch.device("cuda", rank)
        dist.init_process_group("cpu:gloo,cuda:nccl", init_method=f"tcp://127.0.0.1:{port}", world_size=world, rank=rank,
                                device_id=dev)
        comm = create_nccl_comm(world, rank)
        K, B, bs, mb = 4, 2, 64, 3
        tc = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024, max_pos=256)
        dc = ModelCfg(**{**tc.__dict__, "layers": 1})
        wt = random_weights(tc, 41)
        wd = {"embed": wt["embed"], "lm_head": wt["lm_head"], "final_norm": wt["final_norm"], "layers": [wt["layers"][0]]}
        ksc, vsc = [0.02, 0.03], [0.005, 0.011]
        spec = _spec(tc)
        r = PairRunner(spec, _spec(dc) if rank == 0 else None, spec_k=K, max_batch=B, block_size=bs, max_model_len=bs * mb,
                       device=dev, use_graph=True, tp_size=world, tp_rank=rank, target_kv_scales=(ksc, vsc))
        r.bind_weights(L.TARGET, _to_dev(shard_packed_weights(wt, spec, world, rank), dev))
        if rank == 0:
            r.bind_weights(L.DRAFT, _to_dev(wd, dev))
        r.set_nccl_comm(comm)
        assert bind_symmetric_memory(r, world, rank), "symmetric memory could not be set up"
        r.finalize()
        bt = contiguous_block_tables(B, mb)
        bts = [bt[b].tolist() for b in range(B)]
        prompts = [[3, 14, 15, 92, 65, 35, 89, 79], [2, 71, 82, 81, 82]]
        rec = []
        for b in range(B):
            rec.append(r.prefill(L.TARGET, prompts[b], bts[b]))
            r.prefill(L.DRAFT, prompts[b], bts[b], want_sample=False)
        ctx = [len(p) for p in prompts]
        s = None
        if rank == 0:
            s = SpecSession(KvFp8OracleModel(tc, wt, B * mb, bs, k_scale=ksc, v_scale=vsc), OracleModel(dc, wd, B * mb, bs),
                            K, mb)
            s.prefill(prompts, [0.0, 0.0], bt, bt.clone())
        log = []
        for step in range(8):
            toks, nacc, nrec = r.spec_step(ctx, rec, bts, bts, [0.0] * B, [0.0] * B)
            log.append((toks.tolist(), nacc.tolist(), nrec.tolist()))
            if rank == 0:
                sp = torch.from_numpy(toks)
                lp, lq = s.spec_step_forced(sp)
                torch.testing.assert_close(r.logits_p(B).cpu().float(), lp.float(), atol=0.1, rtol=0.04)
                hard, _ = check_greedy_step(sp, nacc.tolist(), nrec.tolist(), lp, lq, EPS)
                assert not hard, f"step {step}: {hard}"
                s.advance(nacc.tolist(), nrec.tolist())
            ctx = [x + int(n) + 1 for x, n in zip(ctx, nacc)]
            rec = nrec.tolist()
        q.put((rank, "ok", None, log))
        r.close()
    except Exception:  # noqa: BLE001
        import traceback
        q.put((rank, "fail", traceback.format_exc(), None))


def test_tp2_kv_fp8_target_matches_oracle():
    """An e4m3 target cache split over 2 GPUs: each rank quantizes its own kv heads with the shared per-layer scales."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank_main, args=(rk, 2, port, q)) for rk in range(2)]
    for p in procs:
        p.start()
    res = {}
    try:
        for _ in range(2):
            rank, status, payload, log = q.get(timeout=300)
            res[rank] = (status, payload, log)
            assert status == "ok", f"rank {rank} failed:\n{payload}"
    finally:
        for p in procs:
            p.join(timeout=5)
            if p.is_alive():
                p.terminate()
    assert res[0][2] == res[1][2]
