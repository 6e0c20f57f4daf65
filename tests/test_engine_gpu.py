"""GPU parity of the whole hot path through the C-ABI: prefill -> K+1 draft forwards -> verify forward ->
accept/reject, driven by ssdk_forward_tokens / ssdk_spec_step, checked step by step against the oracle
(teacher-forced on the engine's own tokens; decisions with a top-2 logit margin >= EPS must agree exactly)."""
import os

import numpy as np
import pytest
import torch

from tests.helpers import load, trace_cfgs, trace_weights

pytestmark = pytest.mark.gpu
EPS = 0.08


def _to_dev(w, dev):
    out = {k: v.to(dev).contiguous() for k, v in w.items() if k != "layers"}
    out["layers"] = [{k: v.to(dev).contiguous() for k, v in lw.items()} for lw in w["layers"]]
    return out


def _spec(c):
    from ssd_b200.runner import ModelSpec
    return ModelSpec(hidden=c.hidden, layers=c.layers, heads=c.heads, kv_heads=c.kv_heads, head_dim=c.head_dim, ffn=c.ffn,
                     vocab=c.vocab, rms_eps=c.rms_eps, rope_theta=c.rope_theta, qk_norm=c.qk_norm, max_pos=c.max_pos)


def _build(family, use_graph, K=None, max_batch=2):
    from oracle.model import OracleModel
    from oracle.spec import SpecSession, contiguous_block_tables
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    z = load(f"trace_{family}.npz")
    tc, dc = trace_cfgs(family, z)
    K = K or int(z["K"])
    bs, mb = int(z["block_size"]), int(z["max_blocks"])
    wt, wd = trace_weights(z, "t"), trace_weights(z, "d")
    dev = torch.device("cuda:0")
    r = PairRunner(_spec(tc), _spec(dc), spec_k=K, max_batch=max_batch, block_size=bs, max_model_len=bs * mb,
                   use_graph=use_graph, use_pdl=False)
    r.bind_weights(L.TARGET, _to_dev(wt, dev))
    r.bind_weights(L.DRAFT, _to_dev(wd, dev))
    r.finalize()
    B = max_batch
    t = OracleModel(tc, wt, B * mb, bs)
    d = OracleModel(dc, wd, B * mb, bs)
    s = SpecSession(t, d, K, mb)
    bt = contiguous_block_tables(B, mb)
    return z, r, s, bt, K


@pytest.mark.parametrize("family", ["llama", "qwen"])
@pytest.mark.parametrize("use_graph", [False, True])
def test_spec_steps_match_oracle(family, use_graph):
    from oracle.spec import check_greedy_step
    from ssd_b200 import lib as L
    z, r, s, bt, K = _build(family, use_graph)
    prompts = [z["prompt0"].tolist(), z["prompt1"].tolist()]
    B = 2
    rec_o = s.prefill(prompts, [0.0, 0.0], bt, bt.clone())
    rec = []
    for b in range(B):
        rec.append(r.prefill(L.TARGET, prompts[b], bt[b].tolist()))
        r.prefill(L.DRAFT, prompts[b], bt[b].tolist(), want_sample=False)
    # the first sampled tokens: engine == oracle == the reference's golden trace
    assert rec == rec_o, f"first tokens {rec} vs oracle {rec_o}"
    ctx = [len(p) for p in prompts]
    assert rec == z["rec0"].tolist(), f"first tokens {rec} vs reference {z['rec0'].tolist()}"
    soft_total = 0
    bts = [bt[b].tolist() for b in range(B)]
    for step in range(12):
        toks, nacc, nrec = r.spec_step(ctx, rec, bts, bts, [0.0] * B, [0.0] * B)
        spec = torch.from_numpy(toks)
        assert spec[:, 0].tolist() == rec
        lp_o, lq_o = s.spec_step_forced(spec)
        lp_e, lq_e = r.logits_p(B).cpu(), r.logits_q(B).cpu()
        torch.testing.assert_close(lq_e.float(), lq_o.float(), atol=0.08, rtol=0.03)
        torch.testing.assert_close(lp_e.float(), lp_o.float(), atol=0.08, rtol=0.03)
        # the engine's integer decisions are exact w.r.t. its OWN logits ...
        hard, soft = check_greedy_step(spec, nacc.tolist(), nrec.tolist(), lp_e, lq_e, 0.0)
        assert not hard and not soft, f"step {step}: engine decisions inconsistent with its logits: {hard + soft}"
        # ... and agree with the oracle's logits wherever the margin is not a near-tie
        hard, soft = check_greedy_step(spec, nacc.tolist(), nrec.tolist(), lp_o, lq_o, EPS)
        assert not hard, f"step {step}: {hard}"
        soft_total += len(soft)
        ctx = [c + int(n) + 1 for c, n in zip(ctx, nacc)]
        rec = nrec.tolist()
        s.advance(nacc.tolist(), rec)
    assert soft_total <= 6
    assert r.launch_count > 0
    r.close()


# golden steps (of 10, two sequences each) that must be reproduced EXACTLY — speculations, accept counts and recovery
# tokens of both sequences — before any near-tie may end the comparison
MIN_EXACT_GOLDEN_STEPS = {"llama": 2, "qwen": 4}


@pytest.mark.parametrize("family", ["llama", "qwen"])
def test_trace_matches_reference_tokens(family):
    """Follow the REFERENCE's golden trace (tests/golden/trace_<family>.npz, produced by running the reference's own
    model classes, Sampler and verify()): same prompts, the reference's recovery tokens and context lengths.  The engine
    must reproduce the reference's speculations / accept counts / recovery tokens step by step; the first step where it
    does not must be a near-tie (top-2 logit margin < EPS under the oracle), after which the KV state no longer follows
    the golden path and the comparison stops.  The number of exactly reproduced steps is reported and has a floor."""
    from oracle.spec import check_greedy_step
    from ssd_b200 import lib as L
    z, r, s, bt, K = _build(family, True)
    prompts = [z["prompt0"].tolist(), z["prompt1"].tolist()]
    B = 2
    s.prefill(prompts, [0.0, 0.0], bt, bt.clone())
    first = []
    for b in range(B):
        first.append(r.prefill(L.TARGET, prompts[b], bt[b].tolist()))
        r.prefill(L.DRAFT, prompts[b], bt[b].tolist(), want_sample=False)
    assert first == z["rec0"].tolist()
    ctx = [len(p) for p in prompts]
    bts = [bt[b].tolist() for b in range(B)]
    n_steps = z["spec"].shape[0]
    same = 0
    for step in range(n_steps):
        rec = z["spec"][step][:, 0].tolist()
        toks, nacc, nrec = r.spec_step(ctx, rec, bts, bts, [0.0] * B, [0.0] * B)
        nxt = z["spec"][step + 1][:, 0].tolist() if step + 1 < n_steps else z["final_recovery"].tolist()
        ok = (toks.tolist() == z["spec"][step].tolist() and nacc.tolist() == z["nacc"][step].tolist()
              and nrec.tolist() == nxt)
        if not ok:
            # the divergence must be explained by a near-tie: check the ENGINE's decisions against oracle logits
            # computed on the engine's own tokens from the (still golden) state
            lp, lq = s.spec_step_forced(torch.from_numpy(toks))
            hard, soft = check_greedy_step(torch.from_numpy(toks), nacc.tolist(), nrec.tolist(), lp, lq, EPS)
            assert not hard, f"step {step}: engine left the reference trace on a decision with a clear margin: {hard}"
            break
        same += 1
        s.spec_step_forced(torch.from_numpy(z["spec"][step]))  # keep the oracle's KV on the golden path
        s.advance(z["nacc"][step].tolist(), nxt)
        ctx = [c + int(n) + 1 for c, n in zip(ctx, z["nacc"][step])]
    print(f"[golden trace {family}] {same}/{n_steps} steps reproduced exactly (tokens, accept counts, recovery; 2 sequences)")
    assert same >= MIN_EXACT_GOLDEN_STEPS[family], f"only {same} golden steps reproduced exactly"
    r.close()


def test_temperature_step_runs_and_is_deterministic():
    from ssd_b200 import lib as L
    outs = []
    for _ in range(2):
        z, r, s, bt, K = _build("llama", True)
        prompts = [z["prompt0"].tolist(), z["prompt1"].tolist()]
        rec = []
        for b in range(2):
            rec.append(r.prefill(L.TARGET, prompts[b], bt[b].tolist(), temp=0.7, seed=3))
            r.prefill(L.DRAFT, prompts[b], bt[b].tolist(), want_sample=False)
        ctx = [len(p) for p in prompts]
        bts = [bt[b].tolist() for b in range(2)]
        log = []
        for step in range(6):
            toks, nacc, nrec = r.spec_step(ctx, rec, bts, bts, [0.7, 0.7], [0.7, 0.7], seed=3)
            assert ((0 <= nacc) & (nacc <= K)).all() and ((0 <= toks) & (toks < 512)).all()
            log.append((toks.tolist(), nacc.tolist(), nrec.tolist()))
            ctx = [c + int(n) + 1 for c, n in zip(ctx, nacc)]
            rec = nrec.tolist()
        outs.append(log)
        r.close()
    assert outs[0] == outs[1]


def test_resident_mode_matches_host_stepping():
    """Device-driven loop (no host I/O between steps) produces the same tokens as host-driven stepping."""
    from ssd_b200 import lib as L
    res = []
    for resident in (False, True):
        z, r, s, bt, K = _build("llama", True)
        prompts = [z["prompt0"].tolist(), z["prompt1"].tolist()]
        rec = []
        for b in range(2):
            rec.append(r.prefill(L.TARGET, prompts[b], bt[b].tolist()))
            r.prefill(L.DRAFT, prompts[b], bt[b].tolist(), want_sample=False)
        ctx = [len(p) for p in prompts]
        bts = [bt[b].tolist() for b in range(2)]
        n_steps = 8
        if resident:
            r.stage(ctx, rec, bts, bts, [0.0, 0.0], [0.0, 0.0])
            for _ in range(n_steps):
                r.step_resident(2)
            toks, total, nrec = r.fetch(2)
            res.append((total.tolist(), nrec.tolist()))
        else:
            total = [0, 0]
            for _ in range(n_steps):
                toks, nacc, nrec = r.spec_step(ctx, rec, bts, bts, [0.0, 0.0], [0.0, 0.0])
                ctx = [c + int(n) + 1 for c, n in zip(ctx, nacc)]
                total = [t + int(n) + 1 for t, n in zip(total, nacc)]
                rec = nrec.tolist()
            res.append((total, rec))
        r.close()
    assert res[0] == res[1]


def test_streaming_draft_kernel_matches_kernel_per_op_path():
    """csrc/draft_stream.cuh (default for batch 1) against SSDK_DRAFT_STREAM=0 at the real Llama-3.2-1B draft shape:
    identical speculations / accept lengths over 24 steps at temp 0 and at temp 0.7 (same Philox scores), draft logits
    within accumulation noise."""
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for extra in ([], ["--temp", "0.7"]):
        res = subprocess.run([sys.executable, os.path.join(root, "tools", "check_draft_stream.py")] + extra, capture_output=True,
                             text=True, timeout=1500)
        print(res.stdout[-600:])
        assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]


@pytest.mark.parametrize("chunk", [32, 64, 256])
def test_long_prompt_prefill_in_unsynchronised_chunks(chunk):
    """ADVICE r1 #1: ssdk_forward_tokens does not synchronise for non-final prefill chunks, so its pinned staging must not be
    reused before the queued H2D copy has run.  A 450-token prompt goes through 15 / 8 / 2 chunks (the first ones without a
    host sync); the sampled token and the last-position logits must match the oracle's single-pass prefill, and the KV it
    left behind must carry a correct decode step."""
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession, contiguous_block_tables
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    dev = torch.device("cuda:0")
    K, bs, mb = 4, 64, 8
    tc = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024, max_pos=512)
    dc = ModelCfg(**{**tc.__dict__, "layers": 1})
    wt = random_weights(tc, 23)
    wd = {"embed": wt["embed"], "lm_head": wt["lm_head"], "final_norm": wt["final_norm"], "layers": [wt["layers"][0]]}
    r = PairRunner(_spec(tc), _spec(dc), spec_k=K, max_batch=1, block_size=bs, max_model_len=bs * mb, use_graph=True)
    r.bind_weights(L.TARGET, _to_dev(wt, dev))
    r.bind_weights(L.DRAFT, _to_dev(wd, dev))
    r.finalize()
    g = torch.Generator().manual_seed(99)
    prompt = torch.randint(0, tc.vocab, (450,), generator=g).tolist()
    bt = contiguous_block_tables(1, mb)
    s = SpecSession(OracleModel(tc, wt, mb, bs), OracleModel(dc, wd, mb, bs), K, mb)
    rec_o = s.prefill([prompt], [0.0], bt, bt.clone())
    rec = r.prefill(L.TARGET, prompt, bt[0].tolist(), chunk=chunk)
    r.prefill(L.DRAFT, prompt, bt[0].tolist(), want_sample=False, chunk=chunk)
    # oracle logits of the last prompt position (teacher-forced single pass) vs the engine's
    ids = torch.tensor(prompt, dtype=torch.int64)
    o2 = OracleModel(tc, wt, mb, bs)
    h = SpecSession(o2, None, K, mb)._forward(o2, ids, [0], len(prompt), bt)
    want = o2.compute_logits(h[-1:])[0].float()
    got = r.logits_last(1)[0].float().cpu()
    torch.testing.assert_close(got, want, atol=0.08, rtol=0.03)
    margin = float(want.topk(2).values[0] - want.topk(2).values[1])
    assert rec == rec_o[0] or margin < EPS, (rec, rec_o, margin)
    # the KV written by the chunks carries a correct speculative step
    from oracle.spec import check_greedy_step
    toks, nacc, nrec = r.spec_step([len(prompt)], [rec_o[0]], [bt[0].tolist()], [bt[0].tolist()], [0.0], [0.0])
    lp, lq = s.spec_step_forced(torch.from_numpy(toks))
    hard, _ = check_greedy_step(torch.from_numpy(toks), nacc.tolist(), nrec.tolist(), lp, lq, EPS)
    assert not hard, hard
    r.close()


def test_large_batch_spec_steps_match_oracle():
    """20 sequences x (K+1 = 7) = 140 tokens per verify forward: the UMMA N = 256 instances of the GEMM inside the step graph,
    verify_kernel beyond 16 sequences, the kernel-per-op draft at M = 20.  Decisions checked against the oracle with the
    near-tie protocol; logits within tolerance."""
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession, check_greedy_step, contiguous_block_tables
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    dev = torch.device("cuda:0")
    B, K, bs, mb = 20, 6, 64, 2
    tc = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024, max_pos=256)
    dc = ModelCfg(**{**tc.__dict__, "layers": 1})
    wt = random_weights(tc, 31)
    wd = {"embed": wt["embed"], "lm_head": wt["lm_head"], "final_norm": wt["final_norm"], "layers": [wt["layers"][0]]}
    r = PairRunner(_spec(tc), _spec(dc), spec_k=K, max_batch=B, block_size=bs, max_model_len=bs * mb, use_graph=True)
    r.bind_weights(L.TARGET, _to_dev(wt, dev))
    r.bind_weights(L.DRAFT, _to_dev(wd, dev))
    r.finalize()
    g = torch.Generator().manual_seed(7)
    prompts = [torch.randint(0, tc.vocab, (int(n),), generator=g).tolist() for n in torch.randint(3, 40, (B,), generator=g)]
    bt = contiguous_block_tables(B, mb)
    bts = [bt[b].tolist() for b in range(B)]
    s = SpecSession(OracleModel(tc, wt, B * mb, bs), OracleModel(dc, wd, B * mb, bs), K, mb)
    rec_o = s.prefill(prompts, [0.0] * B, bt, bt.clone())
    rec = []
    for b in range(B):
        rec.append(r.prefill(L.TARGET, prompts[b], bts[b]))
        r.prefill(L.DRAFT, prompts[b], bts[b], want_sample=False)
    assert sum(int(a != b_) for a, b_ in zip(rec, rec_o)) <= 1  # a bf16 near-tie may flip one first token
    rec = list(rec_o)
    ctx = [len(p) for p in prompts]
    soft_total = 0
    for step in range(3):
        toks, nacc, nrec = r.spec_step(ctx, rec, bts, bts, [0.0] * B, [0.0] * B)
        spec = torch.from_numpy(toks)
        assert spec[:, 0].tolist() == rec
        lp_o, lq_o = s.spec_step_forced(spec)
        torch.testing.assert_close(r.logits_p(B).cpu().float(), lp_o.float(), atol=0.08, rtol=0.03)
        torch.testing.assert_close(r.logits_q(B).cpu().float(), lq_o.float(), atol=0.08, rtol=0.03)
        hard, soft = check_greedy_step(spec, nacc.tolist(), nrec.tolist(), lp_o, lq_o, EPS)
        assert not hard, f"step {step}: {hard}"
        soft_total += len(soft)
        ctx = [c + int(n) + 1 for c, n in zip(ctx, nacc)]
        rec = nrec.tolist()
        s.advance(nacc.tolist(), rec)
    assert soft_total <= 12
    r.close()


def test_packed_prefill_of_ragged_prompts_matches_oracle():
    """prefill_many: several prompts per call (uniform chunk per call, sizes planned on the host), ragged lengths incl. equal
    pairs and a 1-token prompt.  First tokens against the oracle (near-tie protocol), last-position logits of the sequences
    in the final call within tolerance, and the KV it wrote must carry two speculative steps for the whole batch."""
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession, check_greedy_step, contiguous_block_tables
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    dev = torch.device("cuda:0")
    lens = [100, 100, 37, 1, 180, 64, 100, 9]
    B, K, bs, mb = len(lens), 4, 64, 4
    tc = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024, max_pos=256)
    dc = ModelCfg(**{**tc.__dict__, "layers": 1})
    wt = random_weights(tc, 41)
    wd = {"embed": wt["embed"], "lm_head": wt["lm_head"], "final_norm": wt["final_norm"], "layers": [wt["layers"][0]]}
    r = PairRunner(_spec(tc), _spec(dc), spec_k=K, max_batch=B, block_size=bs, max_model_len=bs * mb, use_graph=True)
    r.bind_weights(L.TARGET, _to_dev(wt, dev))
    r.bind_weights(L.DRAFT, _to_dev(wd, dev))
    r.finalize()
    g = torch.Generator().manual_seed(17)
    prompts = [torch.randint(0, tc.vocab, (n,), generator=g).tolist() for n in lens]
    bt = contiguous_block_tables(B, mb)
    bts = [bt[b].tolist() for b in range(B)]
    s = SpecSession(OracleModel(tc, wt, B * mb, bs), OracleModel(dc, wd, B * mb, bs), K, mb)
    rec_o = s.prefill(prompts, [0.0] * B, bt, bt.clone())
    calls = []
    fwd = r.forward_tokens
    r.forward_tokens = lambda which, ids, *a, **k: (calls.append((which, len(ids), len(ids[0]))), fwd(which, ids, *a, **k))[1]
    rec = r.prefill_many(L.TARGET, prompts, bts, [0] * B)
    r.prefill_many(L.DRAFT, prompts, bts, [0] * B, want_sample=False)
    r.forward_tokens = fwd
    tgt_calls = [c for c in calls if c[0] == L.TARGET]
    assert sum(b * q for _, b, q in tgt_calls) == sum(lens) and max(b for _, b, _ in tgt_calls) > 1
    assert len(tgt_calls) < len(lens), tgt_calls  # fewer weight passes than one per prompt
    assert sum(int(a != b_) for a, b_ in zip(rec, rec_o)) <= 1, (rec, rec_o)
    rec = list(rec_o)
    ctx = list(lens)
    for step in range(2):
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


def test_spec_steps_across_the_draft_path_switch_match_oracle():
    """The step graph takes the streaming draft kernel while the context fits one load round of its attention phase
    (<= 1024 tokens incl. the K+1 new ones) and the kernel-per-op draft beyond (use_draft_stream, csrc/engine.cu).  A
    sequence that starts at 1012 tokens crosses the limit within ten steps: every step — whichever graph ran it, and the
    KV the other one left behind — must agree with the oracle (teacher-forced, near-tie protocol); the contexts in between
    also run the 16-split layout of the streaming kernel's attention (> 256 tokens)."""
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession, check_greedy_step, contiguous_block_tables
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    dev = torch.device("cuda:0")
    K, bs, mb = 4, 64, 18
    tc = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024, max_pos=bs * mb)
    dc = ModelCfg(**{**tc.__dict__, "layers": 1})
    wt = random_weights(tc, 29)
    wd = {"embed": wt["embed"], "lm_head": wt["lm_head"], "final_norm": wt["final_norm"], "layers": [wt["layers"][0]]}
    r = PairRunner(_spec(tc), _spec(dc), spec_k=K, max_batch=1, block_size=bs, max_model_len=bs * mb, use_graph=True)
    r.bind_weights(L.TARGET, _to_dev(wt, dev))
    r.bind_weights(L.DRAFT, _to_dev(wd, dev))
    r.finalize()
    g = torch.Generator().manual_seed(5)
    prompt = torch.randint(0, tc.vocab, (1012,), generator=g).tolist()
    bt = contiguous_block_tables(1, mb)
    s = SpecSession(OracleModel(tc, wt, mb, bs), OracleModel(dc, wd, mb, bs), K, mb)
    rec_o = s.prefill([prompt], [0.0], bt, bt.clone())
    r.prefill(L.TARGET, prompt, bt[0].tolist())
    r.prefill(L.DRAFT, prompt, bt[0].tolist(), want_sample=False)
    ctx, rec = len(prompt), rec_o[0]
    launches = []
    for step in range(10):
        n0 = r.launch_count
        toks, nacc, nrec = r.spec_step([ctx], [rec], [bt[0].tolist()], [bt[0].tolist()], [0.0], [0.0])
        launches.append(r.launch_count - n0)
        spec = torch.from_numpy(toks)
        lp_o, lq_o = s.spec_step_forced(spec)
        torch.testing.assert_close(r.logits_p(1).cpu().float(), lp_o.float(), atol=0.08, rtol=0.03)
        torch.testing.assert_close(r.logits_q(1).cpu().float(), lq_o.float(), atol=0.08, rtol=0.03)
        hard, _ = check_greedy_step(spec, nacc.tolist(), nrec.tolist(), lp_o, lq_o, EPS)
        assert not hard, f"step {step} (ctx {ctx}): {hard}"
        ctx += int(nacc[0]) + 1
        rec = int(nrec[0])
        s.advance(nacc.tolist(), [rec])
    assert ctx > 1024 - K - 1, "the sequence never reached the switch"
    if os.environ.get("SSDK_DRAFT_STREAM", "1") != "0":
        assert launches[0] < launches[-1], f"one launch for the draft phase below the limit, a kernel per op above: {launches}"
    r.close()
