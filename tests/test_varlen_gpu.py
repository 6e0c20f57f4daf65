"""Varlen prefill on the device: sequences of different lengths (and prefix-cache hits) in one call.

- ops.paged_attention_varlen (paged_attn_varlen_kernel + attn_combine_kernel<true>) against the fp64 bound of
  tests/attn_ref.py (tests/attn_ref_varlen.py) on random and needle inputs, bit-identical to ops.paged_attention when every q_len is equal, and on
  the host-thread emulation's inputs.
- PairRunner.prefill_varlen against the oracle: ceil(sum / 256) calls, first tokens (near-tie protocol), last-row logits
  of the final call, and two teacher-forced spec steps on the KV it wrote; with prefix-cache hits joining the calls of
  the sequence whose pages they read; bit-identical to prefill_many where both group the prompts the same way.
- Launch count, LLM.generate(varlen_prefill=True) against the default engine, and a 2-GPU case (skips on one GPU)."""
import math
import shutil

import numpy as np
import pytest
import torch

from tests import attn_ref as A
from tests import attn_ref_varlen as AV

pytestmark = pytest.mark.gpu

_RQ = [int(x) for x in np.random.default_rng(5).integers(1, 9, 32)]
_RC = [q + int(x) for q, x in zip(_RQ, np.random.default_rng(6).integers(0, 1500, 32))]

# (id, hd, H, KV, q_lens, block size, contexts, max_blocks (None: just enough pages), alias)
CASES = [
    ("split1_g1_bs16", 64, 4, 4, [1, 3, 2], 16, [1, 40, 64], 4, False),            # max_ctx 64: one split
    ("split5_g3_bs80", 64, 6, 2, [3, 12, 1, 7], 80, [3, 200, 81, 300], 4, False),   # 5 splits, TQ 10 straddled
    ("split32_g8_bs16_8k", 128, 8, 1, [1, 5, 3], 16, [8192, 100, 3000], 512, False),
    ("split32_g16_bs256_16k", 128, 16, 1, [2, 1], 256, [16384, 300], 64, False),
    ("b32_ragged_g4_bs32", 64, 4, 1, _RQ, 32, _RC, None, False),
    ("q256_g2_bs64", 64, 4, 2, [256], 64, [256], None, False),
    ("straddle_g2_bs80", 128, 16, 8, [17, 16, 33, 1], 80, [1300, 16, 700, 5], None, False),
    ("g12_bs64", 128, 12, 1, [5, 2, 3], 64, [500, 2, 4097], None, False),
    ("g4_h32kv8_bs32_8k", 128, 32, 8, [8, 1, 20], 32, [8192, 9, 600], None, False),
    ("alias_g4_bs16", 64, 8, 2, [7, 3], 16, [900, 1000], None, True),
]
WORST: dict[str, float] = {}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from ssd_b200 import lib
    lib.load()
    return torch.device("cuda:0")


def _mb(case):
    _, _, _, _, _, bs, ctx, mb, _ = case
    return mb if mb is not None else (max(ctx) + bs - 1) // bs + 1


def _plan(case):
    from ssd_b200 import ops
    _, hd, H, KV, ql, bs, ctx, _, _ = case
    return ops.paged_attention_varlen_plan(ql, H, KV, bs * _mb(case))


@pytest.mark.parametrize("kind", ["random", "needle"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_varlen_attention_matches_fp64(dev, case, kind):
    from ssd_b200 import ops
    name, hd, H, KV, ql, bs, ctx, _, alias = case
    pl = _plan(case)
    assert pl["n_tiles"] == sum(math.ceil(q / pl["TQ"]) for q in ql)
    q, kc, vc, bt, cl = AV.make_inputs_varlen(hd, H, KV, ql, bs, ctx, kind=kind, seed=sum(map(ord, name)),
                                             max_blocks=_mb(case), alias=alias, n_split=pl["n_split"])
    out = ops.paged_attention_varlen(q.to(dev), kc.to(dev), vc.to(dev), bt.to(dev), cl.to(dev), ql, hd ** -0.5).cpu()
    ref, S = AV.reference_varlen(q, kc, vc, bt, cl, ql, hd ** -0.5)
    r = A.err_over_bound(out, ref, S)
    WORST[kind] = max(WORST.get(kind, 0.0), r)
    print(f"[varlen attention gpu] {name} {kind}: plan {pl}, worst err/bound {r:.3f}")
    assert r <= 1.0, f"worst err/bound {r:.3f}"


def test_varlen_plans_reached(dev):
    """One split, a middle split count and the 32-way maximum all run."""
    ns = {c[0]: _plan(c)["n_split"] for c in CASES}
    print(f"[varlen attention plan] {ns}")
    assert 1 in ns.values() and A.MAX_SPLIT in ns.values() and any(1 < n < A.MAX_SPLIT for n in ns.values())


@pytest.mark.parametrize("shape", [(64, 4, 4, 3, 16, [1, 40, 64], 4), (64, 6, 2, 7, 80, [7, 200, 300], 4),
                                   (128, 8, 1, 5, 16, [8192, 100], 512), (128, 16, 8, 33, 64, [700, 33], None),
                                   (64, 4, 2, 256, 64, [256], None)])
def test_equal_q_lens_are_bit_identical_to_the_uniform_kernel(dev, shape):
    from ssd_b200 import ops
    hd, H, KV, Q, bs, ctx, mb = shape
    mb = mb or (max(ctx) + bs - 1) // bs + 1
    ql = [Q] * len(ctx)
    pu = ops.paged_attention_plan(len(ctx), Q, H, KV, bs * mb)
    pv = ops.paged_attention_varlen_plan(ql, H, KV, bs * mb)
    assert {k: pv[k] for k in pu} == pu and pv["n_tiles"] == len(ctx) * pu["n_qtiles"]
    q, kc, vc, bt, cl = [t.to(dev) for t in A.make_inputs(hd, H, KV, Q, bs, ctx, kind="random", seed=9, max_blocks=mb)]
    a = ops.paged_attention(q, kc, vc, bt, cl, Q, hd ** -0.5)
    b = ops.paged_attention_varlen(q, kc, vc, bt, cl, ql, hd ** -0.5)
    assert torch.equal(a, b), f"plan {pu}"


def test_host_emulation_inputs_on_device(dev, tmp_path):
    from ssd_b200 import ops
    from tests import test_attention_varlen_emu_cpu as E
    have_gxx = shutil.which("g++") is not None
    if have_gxx:
        E.build()
    for case in E.EMU_CASES:
        name, hd, H, KV, ql, bs, ctx, mb, ns, kind = case
        q, kc, vc, bt, cl = inputs = E.case_inputs(case)
        ref, S = AV.reference_varlen(q, kc, vc, bt, cl, ql, hd ** -0.5)
        out = ops.paged_attention_varlen(q.to(dev), kc.to(dev), vc.to(dev), bt.to(dev), cl.to(dev), ql, hd ** -0.5).cpu()
        r_dev = A.err_over_bound(out, ref, S)
        WORST["emulation inputs (device)"] = max(WORST.get("emulation inputs (device)", 0.0), r_dev)
        msg = f"[varlen attention gpu] emulation case {name}: device {r_dev:.3f}"
        if have_gxx:
            _, emu_out = E.run_emu(tmp_path, case, inputs)
            r_emu = A.err_over_bound(emu_out, ref, S)
            msg += f", host threads {r_emu:.3f}"
            assert r_emu <= 1.0, msg
        print(msg)
        assert r_dev <= 1.0, msg


def test_varlen_worst_err_over_bound_summary(dev):
    if not WORST:
        pytest.skip("run together with the tests above")
    for family, r in sorted(WORST.items()):
        print(f"[varlen attention gpu] worst err/bound, {family}: {r:.3f}")
    assert max(WORST.values()) <= 1.0


# ---------------------------------------------------------------------------------------------------------------- engine
def _pair(bs, mb, B, K=4, seed=41):
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    from tests.test_engine_gpu import _spec, _to_dev
    dev = torch.device("cuda:0")
    tc = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024, max_pos=bs * mb)
    dc = ModelCfg(**{**tc.__dict__, "layers": 1})
    wt = random_weights(tc, seed)
    wd = {"embed": wt["embed"], "lm_head": wt["lm_head"], "final_norm": wt["final_norm"], "layers": [wt["layers"][0]]}

    def runner():
        r = PairRunner(_spec(tc), _spec(dc), spec_k=K, max_batch=B, block_size=bs, max_model_len=bs * mb, use_graph=True)
        r.bind_weights(L.TARGET, _to_dev(wt, dev))
        r.bind_weights(L.DRAFT, _to_dev(wd, dev))
        r.finalize()
        return r

    return runner, lambda: SpecSession(OracleModel(tc, wt, B * mb, bs), OracleModel(dc, wd, B * mb, bs), K, mb), tc


def _check_against_oracle(lens, bs, mb, bts, starts, shared_prefix=0):
    from oracle.spec import check_greedy_step
    from ssd_b200 import lib as L
    from tests.test_engine_gpu import EPS
    B = len(lens)
    runner, session, tc = _pair(bs, mb, B)
    r, s = runner(), session()
    g = torch.Generator().manual_seed(17)
    prefix = torch.randint(0, tc.vocab, (shared_prefix,), generator=g).tolist()
    prompts = [prefix + torch.randint(0, tc.vocab, (n - shared_prefix,), generator=g).tolist() for n in lens]
    bt = torch.tensor(bts, dtype=torch.int32)
    rec_o = s.prefill(prompts, [0.0] * B, bt, bt.clone())
    calls = []
    fwd = r.forward_varlen
    r.forward_varlen = lambda which, ids, *a, **k: (calls.append((which, [len(x) for x in ids])), fwd(which, ids, *a, **k))[1]
    rec = r.prefill_varlen(L.TARGET, prompts, bts, starts)
    last = calls[-1][1]
    n_last = len(last)
    lg = r.logits_last(n_last).cpu().float()
    r.prefill_varlen(L.DRAFT, prompts, bts, starts, want_sample=False)
    r.forward_varlen = fwd
    tgt = [c for w, c in calls if w == L.TARGET]
    assert len(tgt) == math.ceil(sum(n - st for n, st in zip(lens, starts)) / 256), tgt
    assert sum(int(a != b_) for a, b_ in zip(rec, rec_o)) <= 1, (rec, rec_o)
    # last-row logits of the sequences of the final call (those are its last len(last) sequences in order)
    plan = r.plan_varlen_calls(lens, starts, bts, bs, 256, B)
    idx = [i for i, _, _ in plan[-1]]
    ref = []
    for i in idx:
        h = s._forward(s.t, torch.tensor(prompts[i], dtype=torch.int64), [0], lens[i], bt[i:i + 1])
        ref.append(s.t.compute_logits(h[-1:]).float())
    torch.testing.assert_close(lg, torch.cat(ref).cpu(), atol=0.08, rtol=0.03)
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


@pytest.mark.parametrize("bs", [64, 80])
def test_prefill_varlen_of_ragged_prompts_matches_oracle(bs):
    """A prompt longer than 256, a 1-token prompt, and one (211) that ends exactly on the end of the second call."""
    lens = [300, 1, 211, 40, 100, 60]
    mb = (max(lens) + 12 + bs - 1) // bs
    bts = [list(range(b * mb, (b + 1) * mb)) for b in range(len(lens))]
    _check_against_oracle(lens, bs, mb, bts, [0] * len(lens))


def test_prefill_varlen_with_prefix_hits_matches_oracle():
    """Sequences 1 and 2 alias the first two 64-token pages of sequence 0 and join the call that writes them."""
    bs, mb = 64, 6
    lens = [200, 150, 200, 140]
    bts = [list(range(b * mb, (b + 1) * mb)) for b in range(4)]
    for i in (1, 2):
        bts[i][:2] = bts[0][:2]
    _check_against_oracle(lens, bs, mb, bts, [0, 128, 128, 0], shared_prefix=128)


def test_prefill_varlen_is_bit_identical_to_prefill_many_on_uniform_prompts():
    from ssd_b200 import lib as L
    B, bs, mb = 16, 64, 3
    runner, _, tc = _pair(bs, mb, B)
    ra, rb = runner(), runner()
    g = torch.Generator().manual_seed(3)
    prompts = [torch.randint(0, tc.vocab, (128,), generator=g).tolist() for _ in range(B)]
    bts = [list(range(b * mb, (b + 1) * mb)) for b in range(B)]
    for temp in (0.0, 0.7):
        ta = ra.prefill_many(L.TARGET, prompts, bts, [0] * B, [temp] * B, seed=5)
        ra.prefill_many(L.DRAFT, prompts, bts, [0] * B, want_sample=False)
        tb = rb.prefill_varlen(L.TARGET, prompts, bts, [0] * B, [temp] * B, seed=5)
        rb.prefill_varlen(L.DRAFT, prompts, bts, [0] * B, want_sample=False)
        assert ta == tb, f"temp {temp}"
        for which in (L.TARGET, L.DRAFT):
            assert torch.equal(ra.kv[which], rb.kv[which]), f"temp {temp}, model {which}"
    ra.close()
    rb.close()


def test_varlen_call_launches_as_many_kernels_as_a_uniform_call():
    from ssd_b200 import lib as L
    runner, _, _ = _pair(64, 5, 4)
    r = runner()
    bts = [list(range(b * 5, (b + 1) * 5)) for b in range(2)]
    for which in (L.TARGET, L.DRAFT):
        for want in (True, False):
            n0 = r.launch_count
            r.forward_tokens(which, [[1] * 8, [2] * 8], [0, 0], bts, want_sample=want)
            n1 = r.launch_count
            r.forward_varlen(which, [[1] * 3, [2] * 13], [0, 0], bts, want_sample=want)
            n2 = r.launch_count
            assert n2 - n1 == n1 - n0 > 0, (which, want, n1 - n0, n2 - n1)
    r.close()


# ----------------------------------------------------------------------------------------------------------- LLM level
@pytest.fixture(scope="module")
def dirs(tmp_path_factory):
    from ssd_b200 import synth
    root = str(tmp_path_factory.mktemp("models"))
    t = synth.make_model_dir(root, "llama-tiny-target", "target", seed=1, alpha=0.7, max_position_embeddings=2048)
    d = synth.make_model_dir(root, "llama-tiny-draft", "draft", seed=1, alpha=0.7, max_position_embeddings=2048)
    return t, d


def _prompt_sets():
    g = torch.Generator().manual_seed(0)
    ragged = [torch.randint(2, 1000, (n,), generator=g).tolist() for n in (5, 300, 33, 1, 200, 70)]
    prefix = torch.randint(2, 1000, (128,), generator=g).tolist()
    shared = [prefix + torch.randint(2, 1000, (n,), generator=g).tolist() for n in (10, 40, 25, 60)]
    return ragged, shared


def _generate(t, d, prompts, **kw):
    from ssd_b200 import LLM, SamplingParams
    llm = LLM(t, speculate=True, draft=d, speculate_k=4, max_num_seqs=8, max_model_len=1024, kvcache_block_size=64,
              jit_speculate=True, **kw)
    out, _ = llm.generate(prompts, SamplingParams(temperature=0.0, max_new_tokens=24, ignore_eos=True), use_tqdm=False)
    llm.exit()
    return [o["token_ids"] for o in out]


def test_llm_generate_with_varlen_prefill_matches_the_default_engine(dirs):
    t, d = dirs
    for prompts in _prompt_sets():
        assert _generate(t, d, prompts, varlen_prefill=True) == _generate(t, d, prompts)


def test_tp2_varlen_prefill_matches_single_gpu(dirs):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    t, d = dirs
    prompts = _prompt_sets()[0]
    assert _generate(t, d, prompts, varlen_prefill=True, num_gpus=2) == _generate(t, d, prompts)
