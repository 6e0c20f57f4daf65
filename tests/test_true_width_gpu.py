"""Engine-level parity at the TRUE widths of the BASELINE models (VERDICT r1 'next round' 1a, ADVICE r1 #1).

Two decoder layers at the real dimensions of Llama-3.1-70B / 8B / Qwen3-32B (+ their drafts), full vocabulary,
NON-degenerate o_proj / down_proj, a 200-token prompt (4 prefill chunks, none of the first three synchronises) — the
oracle ran the same prompts on the same weights in the build container (oracle/gen_true_width_golden.py; the weights are
a pure integer function of (stream, row, column) and are regenerated here bit-for-bit on the device).  Checked, through
the C-ABI (ssdk_forward_tokens / ssdk_spec_step):
  * the first sampled token, every speculated token, accept count and recovery token: EXACT (all margins are in the
    thousands by construction, so there is no near-tie to excuse a mismatch);
  * logits_p / logits_q at 2048 sampled vocabulary columns of every row: |diff| <= 2.5 + 2^-5 |ref| everywhere AND a mean
    |diff| <= 0.6.  Calibration of these bounds (bf16 logits of magnitude 70-90, spacing 0.5): the oracle's OWN two
    arithmetic variants — Inductor single-rounding vs eager double-rounding norms / SiLU, oracle/ops.py `compiled` —
    differ from each other by mean 0.127 / max 1.0 (8B widths) and mean 0.348 / max 2.0 (70B widths): one-ulp noise.  A real
    defect is far outside: switching the attention branch or the MLP branch off moves the target's sampled logits by 9 on
    average (max 64), the 1B-width draft's by 2 on average;
  * the top-1 logit of every row within 2^-6 relative.
"""
import numpy as np
import pytest
import torch

from tests.helpers import bf16, load

pytestmark = pytest.mark.gpu


def _run(name: str):
    from oracle.gen_true_width_golden import CONFIGS, META, specs
    from ssd_b200 import lib as L, synth
    from ssd_b200.runner import PairRunner

    z = load(f"true_width_{name}.npz")
    tshape, dshape, B, plens, K, n_steps = CONFIGS[name]
    tms, _ = specs(tshape)
    dms, _ = specs(dshape)
    dev = torch.device("cuda:0")
    bs, mb = 256, 2
    r = PairRunner(tms, dms, spec_k=K, max_batch=B, block_size=bs, max_model_len=bs * mb, use_graph=True, use_pdl=True)
    r.bind_weights(L.TARGET, synth.generate_weights(tms, {**META, "role": "target"}, dev))
    r.bind_weights(L.DRAFT, synth.generate_weights(dms, {**META, "role": "draft"}, dev))
    r.finalize()
    cols = torch.from_numpy(z["cols"]).to(dev)
    bts = [list(range(b * mb, (b + 1) * mb)) for b in range(B)]
    prompts = [z[f"prompt{b}"].tolist() for b in range(B)]
    rec = []
    for b in range(B):
        rec.append(r.prefill(L.TARGET, prompts[b], bts[b]))
        r.prefill(L.DRAFT, prompts[b], bts[b], want_sample=False)
    assert rec == z["rec0"].tolist(), f"{name}: first tokens {rec} vs oracle {z['rec0'].tolist()}"
    ctx = [len(p) for p in prompts]
    worst = {"lp": 0.0, "lq": 0.0}
    for st in range(n_steps):
        toks, nacc, nrec = r.spec_step(ctx, rec, bts, bts, [0.0] * B, [0.0] * B)
        assert toks.tolist() == z[f"s{st}_spec"].tolist(), f"{name} step {st}: speculations differ"
        assert nacc.tolist() == z[f"s{st}_nacc"].tolist(), f"{name} step {st}: accept counts differ"
        assert nrec.tolist() == z[f"s{st}_rec"].tolist(), f"{name} step {st}: recovery tokens differ"
        for tag, eng in (("lp", r.logits_p(B)), ("lq", r.logits_q(B))):
            got = eng[..., cols].float().cpu()
            want = bf16(z[f"s{st}_{tag}"]).float()
            err = (got - want).abs()
            tol = 2.5 + want.abs() / 32
            ratio = err / tol
            i = int(ratio.argmax())
            assert float(ratio.max()) <= 1.0, (f"{name} step {st} {tag}: |diff| {float(err.flatten()[i]):.2f} at |ref| "
                                               f"{float(want.abs().flatten()[i]):.1f} (tolerance {float(tol.flatten()[i]):.2f}); "
                                               f"mean |diff| {float(err.mean()):.3f}")
            assert float(err.mean()) <= 0.6, f"{name} step {st} {tag}: mean |diff| {float(err.mean()):.3f}"
            worst[tag] = max(worst[tag], float(err.mean()))
            top = eng.float().max(-1).values.cpu()
            want_top = torch.from_numpy(z[f"s{st}_{tag}_top"])
            assert bool(((top - want_top).abs() <= want_top.abs() / 64 + 1.0).all()), f"{name} step {st} {tag}: top-1 logit"
        ctx = [c + int(n) + 1 for c, n in zip(ctx, nacc)]
        rec = nrec.tolist()
    r.close()
    return worst


@pytest.mark.parametrize("name", ["llama70b", "llama8b", "qwen32b"])
def test_true_width_steps_match_oracle(name):
    worst = _run(name)
    print(f"[true-width {name}] worst mean |logit diff| on sampled columns: p {worst['lp']:.3f}  q {worst['lq']:.3f}")
