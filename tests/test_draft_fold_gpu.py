"""The draft writes the KV of a step's last draft token d_K in the NEXT step's first draft forward (row 0 of a two-row
forward), or in a one-token flush when the sequence does not continue (PairRunner.flush_draft).  These tests run spec
steps through ssdk_spec_step on both draft paths (the streaming kernel at batch 1 up to 1024 tokens of context, the
kernel-per-op draft beyond and at batch > 1) and check them against the oracle, which runs the reference's K+1 draft
forwards per step: decisions (near-tie protocol), draft and target logits, and — after a flush — the engine's draft KV
cache on every written position.  A draft identical to the target accepts every draft at temperature 0, so the folded
path runs at every step; a one-layer draft mixes full and partial acceptance."""
import pytest
import torch

from tests.test_engine_gpu import EPS, _spec, _to_dev

pytestmark = pytest.mark.gpu
K = 4


def _pair(prompt_len, steps, same_draft, B=1, bs=64, seed=29):
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession, contiguous_block_tables
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    mb = (prompt_len + (K + 1) * (steps + 1)) // bs + 2
    tc = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024, max_pos=bs * mb)
    wt = random_weights(tc, seed)
    if same_draft:
        dc, wd = tc, wt
    else:
        dc = ModelCfg(**{**tc.__dict__, "layers": 1})
        wd = {"embed": wt["embed"], "lm_head": wt["lm_head"], "final_norm": wt["final_norm"], "layers": [wt["layers"][0]]}
    dev = torch.device("cuda:0")
    r = PairRunner(_spec(tc), _spec(dc), spec_k=K, max_batch=B, block_size=bs, max_model_len=bs * mb, use_graph=True)
    r.bind_weights(L.TARGET, _to_dev(wt, dev))
    r.bind_weights(L.DRAFT, _to_dev(wd, dev))
    r.finalize()
    s = SpecSession(OracleModel(tc, wt, B * mb, bs), OracleModel(dc, wd, B * mb, bs), K, mb)
    bt = contiguous_block_tables(B, mb)
    return r, s, bt, tc, bs


def _draft_kv_matches(r, s, bts, ctx, bs):
    """Engine draft cache == oracle draft cache (K+1 forwards per step) at every written position."""
    from ssd_b200 import lib as L
    r.flush_draft()
    got, want = r.kv[L.DRAFT].cpu().float(), s.d.kv_cache.float()
    for bt, n in zip(bts, ctx):
        idx = [(bt[p // bs], p % bs) for p in range(n)]
        blk = torch.tensor([i for i, _ in idx])
        slot = torch.tensor([j for _, j in idx])
        torch.testing.assert_close(got[:, :, blk, slot], want[:, :, blk, slot], atol=0.08, rtol=0.03)


def _run(r, s, bt, tc, bs, prompts, temp, steps, check_every=10):
    from oracle.spec import check_greedy_step
    from ssd_b200 import lib as L
    B = len(prompts)
    bts = [bt[b].tolist() for b in range(B)]
    s.prefill(prompts, [0.0] * B, bt, bt.clone())
    rec = [r.prefill(L.TARGET, prompts[b], bts[b], temp=temp, seed=3) for b in range(B)]
    for b in range(B):
        r.prefill(L.DRAFT, prompts[b], bts[b], want_sample=False)
    s.recovery = list(rec)
    ctx = [len(p) for p in prompts]
    n_all = n_part = 0
    for step in range(steps):
        toks, nacc, nrec = r.spec_step(ctx, rec, bts, bts, [temp] * B, [temp] * B, seed=3)
        spec = torch.from_numpy(toks)
        assert spec[:, 0].tolist() == rec
        lp_o, lq_o = s.spec_step_forced(spec)
        torch.testing.assert_close(r.logits_q(B).cpu().float(), lq_o.float(), atol=0.08, rtol=0.03)
        torch.testing.assert_close(r.logits_p(B).cpu().float(), lp_o.float(), atol=0.08, rtol=0.03)
        if temp == 0.0:
            hard, _ = check_greedy_step(spec, nacc.tolist(), nrec.tolist(), lp_o, lq_o, EPS)
            assert not hard, f"step {step} (ctx {ctx}): {hard}"
        n_all += int((nacc == K).sum())
        n_part += int((nacc < K).sum())
        ctx = [c + int(n) + 1 for c, n in zip(ctx, nacc)]
        rec = nrec.tolist()
        s.advance(nacc.tolist(), rec)
        if step % check_every == check_every - 1 or step == steps - 1:
            _draft_kv_matches(r, s, bts, ctx, bs)
    return n_all, n_part, ctx


@pytest.mark.parametrize("prompt_len", [130, 1000])
@pytest.mark.parametrize("temp", [0.0, 0.7])
def test_folded_steps_match_oracle(prompt_len, temp):
    """30+ steps with every draft accepted at temperature 0 (draft == target): each step folds the previous d_K into its
    first draft forward.  The 1000-token prompt crosses the 1024-token switch to the kernel-per-op draft."""
    steps = 32
    r, s, bt, tc, bs = _pair(prompt_len, steps, same_draft=True)
    g = torch.Generator().manual_seed(prompt_len)
    prompt = torch.randint(0, tc.vocab, (prompt_len,), generator=g).tolist()
    n_all, _, ctx = _run(r, s, bt, tc, bs, [prompt], temp, steps)
    assert n_all > 0, "no step accepted all drafts: the fold never ran"
    if temp == 0.0:
        assert n_all >= steps // 2
    if prompt_len == 1000:
        assert ctx[0] > 1024, "the sequence never reached the kernel-per-op draft"
    r.close()


def test_mixed_acceptance_matches_oracle():
    """A one-layer draft: full and partial acceptance alternate, so steps fold or not from one to the next."""
    steps = 30
    r, s, bt, tc, bs = _pair(130, steps, same_draft=False)
    g = torch.Generator().manual_seed(1)
    prompt = torch.randint(0, tc.vocab, (130,), generator=g).tolist()
    n_all, n_part, _ = _run(r, s, bt, tc, bs, [prompt], 0.0, steps)
    assert n_part > 0
    r.close()


@pytest.mark.parametrize("B", [2, 4])
def test_batch_kernel_per_op_fold_matches_oracle(B):
    """Batch > 1 runs the kernel-per-op draft: forward 0 is a two-row forward per sequence whose row 0 stores K/V only
    for sequences with a pending token."""
    steps = 12
    r, s, bt, tc, bs = _pair(100, steps, same_draft=(B == 2), B=B)
    g = torch.Generator().manual_seed(B)
    prompts = [torch.randint(0, tc.vocab, (n,), generator=g).tolist() for n in (100, 37, 64, 90)[:B]]
    n_all, _, _ = _run(r, s, bt, tc, bs, prompts, 0.0, steps, check_every=4)
    if B == 2:
        assert n_all > 0
    r.close()


def _prefix_case(flush_via_hit):
    """Sequence A ends right after an all-accept step whose d_K is the last token of a full page.  Sequence B starts with
    A's tokens on A's pages.  Its draft prefill either reuses those pages (a prefix-cache hit: the pending d_K must be
    flushed first) or computes the whole prompt on pages of its own.  Returns B's speculations and draft logits."""
    from ssd_b200 import lib as L
    bs = 16
    r, s, bt, tc, _ = _pair(64, 8, same_draft=True, B=2, bs=bs)
    g = torch.Generator().manual_seed(8)
    a_prompt = torch.randint(0, tc.vocab, (bs * 3 - K - 1,), generator=g).tolist()
    bt_a, bt_b = bt[0].tolist(), bt[1].tolist()
    rec = r.prefill(L.TARGET, a_prompt, bt_a)
    r.prefill(L.DRAFT, a_prompt, bt_a, want_sample=False)
    toks, nacc, nrec = r.spec_step([len(a_prompt)], [rec], [bt_a], [bt_a], [0.0], [0.0])
    assert int(nacc[0]) == K, "the draft equals the target: every draft must be accepted"
    a_tokens = a_prompt + toks[0].tolist()  # 3 full pages; d_K (the last one) is pending
    assert len(a_tokens) == 3 * bs
    b_prompt = a_tokens + torch.randint(0, tc.vocab, (20,), generator=g).tolist()
    if flush_via_hit:
        bt_bd = bt_a[:3] + bt_b[3:]
        rec_b = r.prefill(L.TARGET, b_prompt, bt_b)
        r.prefill(L.DRAFT, b_prompt, bt_bd, start=3 * bs, want_sample=False)
    else:
        bt_bd = bt_b
        rec_b = r.prefill(L.TARGET, b_prompt, bt_b)
        r.prefill(L.DRAFT, b_prompt, bt_bd, want_sample=False)
    out = []
    ctx = len(b_prompt)
    for _ in range(3):
        toks, nacc, nrec = r.spec_step([ctx], [rec_b], [bt_b], [bt_bd], [0.0], [0.0])
        out.append((toks.copy(), r.logits_q(1).cpu().float()))
        ctx += int(nacc[0]) + 1
        rec_b = int(nrec[0])
    r.close()
    return out


def test_pending_token_is_flushed_before_a_prefix_cache_hit():
    hit, scratch = _prefix_case(True), _prefix_case(False)
    for (ta, la), (tb, lb) in zip(hit, scratch):
        assert (ta == tb).all(), (ta, tb)
        torch.testing.assert_close(la, lb, atol=0.02, rtol=0.01)


def test_pending_token_is_flushed_when_another_chain_steps():
    """Sequence A leaves a pending d_K; a step of sequence B alone (A preempted) must write it first; A then resumes on
    its pages and must still match the oracle."""
    from oracle.spec import check_greedy_step
    from ssd_b200 import lib as L
    r, s, bt, tc, bs = _pair(60, 6, same_draft=True, B=2)
    g = torch.Generator().manual_seed(4)
    prompts = [torch.randint(0, tc.vocab, (n,), generator=g).tolist() for n in (60, 45)]
    bts = [bt[b].tolist() for b in range(2)]
    s.prefill(prompts, [0.0, 0.0], bt, bt.clone())
    rec = [r.prefill(L.TARGET, prompts[b], bts[b]) for b in range(2)]
    for b in range(2):
        r.prefill(L.DRAFT, prompts[b], bts[b], want_sample=False)
    s.recovery = list(rec)
    ctx = [len(p) for p in prompts]
    pending_seen = 0
    for rows in ([0, 1], [1], [0, 1], [0], [1], [0, 1]):
        toks, nacc, nrec = r.spec_step([ctx[b] for b in rows], [rec[b] for b in rows], [bts[b] for b in rows],
                                       [bts[b] for b in rows], [0.0] * len(rows), [0.0] * len(rows))
        pending_seen += len(r._pending)
        # the oracle steps the same rows
        s.ctx, s.recovery = [ctx[b] for b in rows], [rec[b] for b in rows]
        s.bt_t = s.bt_d = bt[rows]
        spec = torch.from_numpy(toks)
        lp_o, lq_o = s.spec_step_forced(spec)
        torch.testing.assert_close(r.logits_q(len(rows)).cpu().float(), lq_o.float(), atol=0.08, rtol=0.03)
        hard, _ = check_greedy_step(spec, nacc.tolist(), nrec.tolist(), lp_o, lq_o, EPS)
        assert not hard, hard
        for j, b in enumerate(rows):
            ctx[b] += int(nacc[j]) + 1
            rec[b] = int(nrec[j])
    assert pending_seen > 0
    _draft_kv_matches(r, s, bts, ctx, bs)
    r.close()
