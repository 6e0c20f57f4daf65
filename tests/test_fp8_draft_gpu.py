"""GPU tests of an FP8 draft: its four decoder linears as e4m3 weights with fp32 row scales, through the streaming draft
kernel (draft_stream_kernel<HD, GMAX, true>, batch 1 up to 1024 tokens of context) and through the kernel-per-op draft
(the FP8 GEMM instances: longer contexts, batch > 1, prefill, the one-token flush).  Whole speculative steps run against
the oracle with tests/fp8_ref.py's Fp8OracleModel as the draft, with a bf16 and with an FP8 target; LLM.generate covers
FP8 draft checkpoints, quantize-on-load, and the speculative-decoding guarantee that the draft's numerics change no
token at temperature 0."""
import pytest
import torch

from tests.fp8_ref import Fp8OracleModel, quantize_weights
from tests.test_fp8_engine_gpu import _write_checkpoint

pytestmark = pytest.mark.gpu
EPS = 0.08
F8 = torch.float8_e4m3fn
K = 4


def _to_dev(w, dev):
    out = {k: v.to(dev).contiguous() for k, v in w.items() if k != "layers"}
    out["layers"] = [{k: v.to(dev).contiguous() for k, v in lw.items()} for lw in w["layers"]]
    return out


def _spec(c):
    from ssd_b200.runner import ModelSpec
    return ModelSpec(hidden=c.hidden, layers=c.layers, heads=c.heads, kv_heads=c.kv_heads, head_dim=c.head_dim, ffn=c.ffn,
                     vocab=c.vocab, rms_eps=c.rms_eps, rope_theta=c.rope_theta, qk_norm=c.qk_norm, max_pos=c.max_pos)


# ------------------------------------------------------------------------------------------------ binding
def test_draft_fp8_bind_and_finalize_checks():
    from oracle.model import ModelCfg, random_weights
    from ssd_b200 import lib as L
    from ssd_b200.runner import ModelSpec, PairRunner
    dev = torch.device("cuda:0")
    spec = ModelSpec(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=512)
    c = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=512, max_pos=256)
    w = random_weights(c, 3)
    _, we = quantize_weights(w)

    def runner(draft_fp8):
        return PairRunner(spec, spec, spec_k=2, max_batch=1, block_size=64, max_model_len=256, draft_fp8=draft_fp8)

    # draft_fp8 = 0: the draft keeps refusing FP8 weights
    r = runner(False)
    w8, s = we["layers"][0]["qkv"].to(dev), we["layers"][0]["qkv_scale"].to(dev)
    assert r.lib.ssdk_bind_weight_fp8(r.h, L.DRAFT, L.W_QKV, 0, w8.data_ptr(), s.data_ptr(), *w8.shape) != 0
    assert "target model only" in L.last_error()
    r.close()
    # draft_fp8 = 1: accepted, with the target's checks
    r = runner(True)
    assert r.lib.ssdk_bind_weight_fp8(r.h, L.DRAFT, L.W_QKV, 0, w8.data_ptr(), s.data_ptr(), *w8.shape) == 0, L.last_error()
    bad = torch.zeros(5 * 64, 192, dtype=F8, device=dev)
    assert r.lib.ssdk_bind_weight_fp8(r.h, L.DRAFT, L.W_QKV, 0, bad.data_ptr(), s.data_ptr(), 320, 192) != 0
    assert "shape" in L.last_error() or "multiple of 128" in L.last_error()
    assert r.lib.ssdk_bind_weight_fp8(r.h, L.DRAFT, L.W_LM_HEAD, 0, w8.data_ptr(), s.data_ptr(), 512, 256) != 0
    assert "no FP8 form" in L.last_error()
    r.close()
    # finalize: a mixed draft and a draft without FP8 linears are refused when draft_fp8 = 1
    mixed = {**we, "layers": [dict(we["layers"][0]), dict(w["layers"][1])]}
    for wd, word in ((mixed, "partly bf16"), (w, "bf16")):
        r = runner(True)
        r.bind_weights(L.TARGET, _to_dev(w, dev))
        r.bind_weights(L.DRAFT, _to_dev(wd, dev))
        with pytest.raises(RuntimeError, match=word):
            r.finalize()
        r.close()
    r = runner(True)
    r.bind_weights(L.TARGET, _to_dev(w, dev))
    r.bind_weights(L.DRAFT, _to_dev(we, dev))
    r.finalize()
    r.close()


# ------------------------------------------------------------------------------------------------ spec steps vs oracle
def _pair(prompt_len, steps, target_fp8, B=1, bs=64, use_graph=True, draft_layers=2, seed=31):
    """A 2-layer target and an FP8 draft built from the same weights (draft_layers = 2: the draft equals the target up to
    FP8 rounding, so most steps accept every draft and the next step folds d_K into its first forward)."""
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession, contiguous_block_tables
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    mb = (prompt_len + (K + 1) * (steps + 1)) // bs + 2
    tc = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024, max_pos=bs * mb)
    wt = random_weights(tc, seed)
    dc = ModelCfg(**{**tc.__dict__, "layers": draft_layers})
    wd = {"embed": wt["embed"], "lm_head": wt["lm_head"], "final_norm": wt["final_norm"], "layers": wt["layers"][:draft_layers]}
    wdo, wde = quantize_weights(wd)
    dev = torch.device("cuda:0")
    r = PairRunner(_spec(tc), _spec(dc), spec_k=K, max_batch=B, block_size=bs, max_model_len=bs * mb, use_graph=use_graph,
                   draft_fp8=True)
    if target_fp8:
        wto, wte = quantize_weights(wt)
        r.bind_weights(L.TARGET, _to_dev(wte, dev))
        tgt = Fp8OracleModel(tc, wto, B * mb, bs)
    else:
        r.bind_weights(L.TARGET, _to_dev(wt, dev))
        tgt = OracleModel(tc, wt, B * mb, bs)
    r.bind_weights(L.DRAFT, _to_dev(wde, dev))
    r.finalize()
    s = SpecSession(tgt, Fp8OracleModel(dc, wdo, B * mb, bs), K, mb)
    return r, s, contiguous_block_tables(B, mb), tc, bs


def _draft_kv_matches(r, s, bts, ctx, bs):
    """After a flush, the engine's draft cache == the FP8 oracle's at every written position."""
    from ssd_b200 import lib as L
    r.flush_draft()
    got, want = r.kv[L.DRAFT].cpu().float(), s.d.kv_cache.float()
    for bt, n in zip(bts, ctx):
        blk = torch.tensor([bt[p // bs] for p in range(n)])
        slot = torch.tensor([p % bs for p in range(n)])
        torch.testing.assert_close(got[:, :, blk, slot], want[:, :, blk, slot], atol=0.08, rtol=0.03)


def _run(r, s, bt, tc, prompts, temp, steps, bs, check_every=6):
    from oracle.spec import check_greedy_step
    from ssd_b200 import lib as L
    B = len(prompts)
    bts = [bt[b].tolist() for b in range(B)]
    rec_o = s.prefill(prompts, [0.0] * B, bt, bt.clone())
    rec = r.prefill_many(L.TARGET, prompts, bts, [0] * B)
    r.prefill_many(L.DRAFT, prompts, bts, [0] * B, want_sample=False)
    assert sum(int(a != b_) for a, b_ in zip(rec, rec_o)) <= 1, (rec, rec_o)
    rec, ctx = list(rec_o), [len(p) for p in prompts]
    n_all = 0
    for step in range(steps):
        toks, nacc, nrec = r.spec_step(ctx, rec, bts, bts, [temp] * B, [temp] * B, seed=7)
        spec = torch.from_numpy(toks)
        lp_o, lq_o = s.spec_step_forced(spec)
        torch.testing.assert_close(r.logits_q(B).cpu().float(), lq_o.float(), atol=0.08, rtol=0.03)
        torch.testing.assert_close(r.logits_p(B).cpu().float(), lp_o.float(), atol=0.08, rtol=0.03)
        if temp == 0.0:
            hard, _ = check_greedy_step(spec, nacc.tolist(), nrec.tolist(), lp_o, lq_o, EPS)
            assert not hard, f"step {step} (ctx {ctx}): {hard}"
        n_all += int((nacc == K).sum())
        ctx = [c + int(n) + 1 for c, n in zip(ctx, nacc)]
        rec = nrec.tolist()
        s.advance(nacc.tolist(), rec)
        if step % check_every == check_every - 1 or step == steps - 1:
            _draft_kv_matches(r, s, bts, ctx, bs)
    return n_all, ctx


@pytest.mark.parametrize("target_fp8", [False, True])
@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("temp", [0.0, 0.7])
def test_fp8_draft_streaming_steps_match_oracle(target_fp8, use_graph, temp):
    """Batch 1 below 1024 tokens: the FP8 streaming draft kernel, with folded pending tokens after all-accept steps."""
    steps = 12
    r, s, bt, tc, bs = _pair(130, steps, target_fp8, use_graph=use_graph)
    g = torch.Generator().manual_seed(3)
    prompt = torch.randint(0, tc.vocab, (130,), generator=g).tolist()
    n_all, _ = _run(r, s, bt, tc, [prompt], temp, steps, bs)
    if temp == 0.0:
        assert n_all > 0, "no step accepted all drafts: the fold never ran"
    r.close()


@pytest.mark.parametrize("B,prompt_len,target_fp8", [(1, 1000, False), (1, 1000, True), (4, 60, False), (4, 60, True)])
def test_fp8_draft_kernel_per_op_paths_match_oracle(B, prompt_len, target_fp8):
    """A context past 1024 (the FP8 draft leaves the streaming kernel for the FP8 GEMMs mid-run) and batch 4."""
    steps = 10
    r, s, bt, tc, bs = _pair(prompt_len, steps, target_fp8, B=B, draft_layers=1)
    g = torch.Generator().manual_seed(prompt_len + B)
    prompts = [torch.randint(0, tc.vocab, (prompt_len + 3 * b,), generator=g).tolist() for b in range(B)]
    _, ctx = _run(r, s, bt, tc, prompts, 0.0, steps, bs, check_every=5)
    if prompt_len == 1000:
        assert ctx[0] > 1024, "the sequence never reached the kernel-per-op draft"
    r.close()


# ------------------------------------------------------------------------------------------------ true widths
@pytest.mark.parametrize("family", ["llama-3.2-1b", "qwen3-0.6b"])
def test_fp8_draft_at_true_widths_matches_fp8_oracle(family):
    """Two FP8 draft layers at Llama-3.2-1B widths (down K = 8192: 4 rows x 4 segments per slot) or Qwen3-0.6B widths
    (head_dim 128, q/k norm, down K = 3072), the full vocabulary, a 200-token prompt, batch 1: the streaming kernel against
    the FP8 oracle on the host.  The target is one bf16 layer at the same widths."""
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession, check_greedy_step
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    dev = torch.device("cuda:0")
    bs, mb = 256, 2
    if family == "llama-3.2-1b":
        dc = ModelCfg(hidden=2048, layers=2, heads=32, kv_heads=8, head_dim=64, ffn=8192, vocab=128256, max_pos=bs * mb)
    else:
        dc = ModelCfg(hidden=1024, layers=2, heads=16, kv_heads=8, head_dim=128, ffn=3072, vocab=151936, max_pos=bs * mb,
                      rms_eps=1e-6, rope_theta=1000000.0, qk_norm=True)
    tc = ModelCfg(**{**dc.__dict__, "layers": 1})
    wt, wd = random_weights(tc, 5), random_weights(dc, 6)
    wdo, wde = quantize_weights(wd)
    r = PairRunner(_spec(tc), _spec(dc), spec_k=K, max_batch=1, block_size=bs, max_model_len=bs * mb, use_graph=True,
                   draft_fp8=True)
    r.bind_weights(L.TARGET, _to_dev(wt, dev))
    r.bind_weights(L.DRAFT, _to_dev(wde, dev))
    r.finalize()
    del wde
    g = torch.Generator().manual_seed(12)
    prompt = torch.randint(0, dc.vocab, (200,), generator=g).tolist()
    bt = torch.arange(mb, dtype=torch.int32)[None, :]
    s = SpecSession(OracleModel(tc, wt, mb, bs), Fp8OracleModel(dc, wdo, mb, bs), K, mb)
    rec_o = s.prefill([prompt], [0.0], bt, bt.clone())
    r.prefill(L.TARGET, prompt, bt[0].tolist())
    r.prefill(L.DRAFT, prompt, bt[0].tolist(), want_sample=False)
    rec, ctx, worst = rec_o[0], len(prompt), 0.0  # the steps start from the oracle's first token
    for step in range(3):
        toks, nacc, nrec = r.spec_step([ctx], [rec], [bt[0].tolist()], [bt[0].tolist()], [0.0], [0.0])
        spec = torch.from_numpy(toks)
        lp_o, lq_o = s.spec_step_forced(spec)
        for eng, ref in ((r.logits_p(1), lp_o), (r.logits_q(1), lq_o)):
            torch.testing.assert_close(eng.cpu().float(), ref.float(), atol=0.25, rtol=1 / 32)
            worst = max(worst, float((eng.cpu().float() - ref.float()).abs().mean()))
        hard, _ = check_greedy_step(spec, nacc.tolist(), nrec.tolist(), lp_o, lq_o, EPS)
        assert not hard, f"step {step}: {hard}"
        ctx += int(nacc[0]) + 1
        rec = int(nrec[0])
        s.advance(nacc.tolist(), [rec])
    print(f"[fp8 draft {family} widths] worst mean |logit diff| {worst:.4f}")
    r.close()


# ------------------------------------------------------------------------------------------------ LLM.generate
def _generate(target, draft, prompts, **kw):
    from ssd_b200 import LLM, SamplingParams
    from ssd_b200 import lib as L
    llm = LLM(target, speculate=True, draft=draft, speculate_k=4, max_num_seqs=3, max_model_len=1024,
              kvcache_block_size=64, **kw)
    out, _ = llm.generate(prompts, SamplingParams(temperature=0.0, max_new_tokens=24, ignore_eos=True), use_tqdm=False)
    cfg = llm.config
    wd = [{n: (lw[n].view(torch.uint8).cpu(), lw[n + "_scale"].cpu()) if lw[n].dtype == F8 else (lw[n].cpu(), None)
           for n in ("qkv", "o", "gate_up", "down")} for lw in llm.runner.weights[L.DRAFT]["layers"]]
    llm.exit()
    return [o["token_ids"] for o in out], wd, cfg


def test_fp8_draft_checkpoint_generates_like_quantize_on_load(tmp_path):
    """An FP8 draft checkpoint and draft_quantization="fp8" on its bf16 source: the same tokens, bit-identical draft
    weights and scales on the device, and both configs read draft_quantization "fp8"."""
    from oracle.model import ModelCfg, random_weights
    from ssd_b200 import synth
    c = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024, max_pos=2048)
    w = random_weights(c, 17)
    target = synth.make_model_dir(str(tmp_path), "llama-tiny-target", "target", seed=1, max_position_embeddings=2048)
    bf_dir = _write_checkpoint(tmp_path / "llama-tiny-draft-bf16", c, w, fp8=False)
    f8_dir = _write_checkpoint(tmp_path / "llama-tiny-draft-fp8", c, w, fp8=True)
    g = torch.Generator().manual_seed(1)
    prompts = [torch.randint(2, 1000, (n,), generator=g).tolist() for n in (5, 70, 33)]
    ta, wa, ca = _generate(target, bf_dir, prompts, tokenizer_path=target, draft_quantization="fp8")
    tb, wb, cb = _generate(target, f8_dir, prompts, tokenizer_path=target)
    assert ca.draft_quantization == cb.draft_quantization == "fp8" and ca.quantization is None
    for l in range(c.layers):
        for n in ("qkv", "o", "gate_up", "down"):
            assert wa[l][n][1] is not None, (l, n)
            assert torch.equal(wa[l][n][0], wb[l][n][0]), (l, n, "weights")
            assert torch.equal(wa[l][n][1], wb[l][n][1]), (l, n, "scales")
    assert ta == tb


@pytest.mark.parametrize("quantization", [None, "fp8"])
def test_fp8_draft_emits_the_bf16_draft_tokens(tmp_path, quantization):
    """At temperature 0 the engine emits the target's greedy chain whatever the draft proposes: on the synthetic pair
    (whose margins make the chain exact) draft_quantization="fp8" gives exactly the tokens of the bf16-draft run, with a
    bf16 and with an FP8 target."""
    from ssd_b200 import synth
    t = synth.make_model_dir(str(tmp_path), "llama-tiny-target", "target", seed=0)
    d = synth.make_model_dir(str(tmp_path), "llama-tiny-draft", "draft", seed=0)
    g = torch.Generator().manual_seed(2)
    prompts = [torch.randint(2, 1000, (n,), generator=g).tolist() for n in (9, 130, 40)]
    ta, wa, ca = _generate(t, d, prompts, quantization=quantization)
    tb, wb, cb = _generate(t, d, prompts, quantization=quantization, draft_quantization="fp8")
    assert ca.draft_quantization is None and cb.draft_quantization == "fp8"
    assert wa[0]["qkv"][1] is None and wb[0]["qkv"][1] is not None
    assert ta == tb


def test_fp8_draft_prefill_varlen_with_prefix_hits_matches_oracle():
    """prefill_varlen on an FP8 draft: sequences 1 and 2 alias the first two 64-token pages of sequence 0 (prefix-cache
    hits joining the call that writes them); first tokens, then two speculative steps against the oracle."""
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession, check_greedy_step
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    dev = torch.device("cuda:0")
    bs, mb = 64, 6
    lens, starts = [200, 150, 200, 140], [0, 128, 128, 0]
    B = len(lens)
    c = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024, max_pos=bs * mb)
    dc = ModelCfg(**{**c.__dict__, "layers": 1})
    wt = random_weights(c, 43)
    wd = {"embed": wt["embed"], "lm_head": wt["lm_head"], "final_norm": wt["final_norm"], "layers": [wt["layers"][0]]}
    wdo, wde = quantize_weights(wd)
    r = PairRunner(_spec(c), _spec(dc), spec_k=K, max_batch=B, block_size=bs, max_model_len=bs * mb, use_graph=True,
                   draft_fp8=True)
    r.bind_weights(L.TARGET, _to_dev(wt, dev))
    r.bind_weights(L.DRAFT, _to_dev(wde, dev))
    r.finalize()
    bts = [list(range(b * mb, (b + 1) * mb)) for b in range(B)]
    for i in (1, 2):
        bts[i][:2] = bts[0][:2]
    g = torch.Generator().manual_seed(19)
    prefix = torch.randint(0, c.vocab, (128,), generator=g).tolist()
    prompts = [prefix + torch.randint(0, c.vocab, (n - 128,), generator=g).tolist() for n in lens]
    bt = torch.tensor(bts, dtype=torch.int32)
    s = SpecSession(OracleModel(c, wt, B * mb, bs), Fp8OracleModel(dc, wdo, B * mb, bs), K, mb)
    rec_o = s.prefill(prompts, [0.0] * B, bt, bt.clone())
    rec = r.prefill_varlen(L.TARGET, prompts, bts, starts)
    r.prefill_varlen(L.DRAFT, prompts, bts, starts, want_sample=False)
    assert sum(int(a != b_) for a, b_ in zip(rec, rec_o)) <= 1, (rec, rec_o)
    rec, ctx = list(rec_o), list(lens)
    for step in range(2):
        toks, nacc, nrec = r.spec_step(ctx, rec, bts, bts, [0.0] * B, [0.0] * B)
        spec = torch.from_numpy(toks)
        lp_o, lq_o = s.spec_step_forced(spec)
        torch.testing.assert_close(r.logits_p(B).cpu().float(), lp_o.float(), atol=0.08, rtol=0.03)
        torch.testing.assert_close(r.logits_q(B).cpu().float(), lq_o.float(), atol=0.08, rtol=0.03)
        hard, _ = check_greedy_step(spec, nacc.tolist(), nrec.tolist(), lp_o, lq_o, EPS)
        assert not hard, f"step {step}: {hard}"
        ctx = [x + int(n) + 1 for x, n in zip(ctx, nacc)]
        rec = nrec.tolist()
        s.advance(nacc.tolist(), rec)
    r.close()
