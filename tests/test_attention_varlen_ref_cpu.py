"""Self-test of the varlen attention checker (tests/attn_ref_varlen.py): on needle inputs of packed
sequences with their own q_lens, each positional defect and each varlen defect (the causal limit taken from the call's
longest q_len, one sequence's rows read one packed row late) must fail the same bound the kernel tests use, and the
exact result rounded the way the kernel rounds must pass."""
import pytest
import torch

from tests import attn_ref as A
from tests import attn_ref_varlen as AV

# (hd, H, KV, q_lens, block size, contexts, n_split)
SHAPES = [
    (64, 8, 2, [7, 1, 12], 16, [300, 1, 140], 3),      # G 4, q_len 1, ctx == q_len
    (128, 6, 2, [5, 33, 2], 80, [1000, 33, 90], 5),    # G 3, pages of 80
    (128, 16, 1, [2, 1, 3], 256, [2000, 7, 600], 32),  # G 16, 32 splits
]
IDS = [f"hd{s[0]}_h{s[1]}_kv{s[2]}_q{'-'.join(map(str, s[3]))}_bs{s[4]}" for s in SHAPES]


def _rounded(x):
    return torch.from_numpy(A.to_bf16_values(x))


def _inputs(shape, kind):
    hd, H, KV, ql, bs, ctx, ns = shape
    return AV.make_inputs_varlen(hd, H, KV, ql, bs, ctx, kind=kind, seed=11, n_split=ns)


def test_equal_q_lens_give_the_uniform_inputs_and_reference():
    uni = A.make_inputs(64, 8, 2, 5, 16, [300, 40], kind="needle", seed=3, n_split=3)
    var = AV.make_inputs_varlen(64, 8, 2, [5, 5], 16, [300, 40], kind="needle", seed=3, n_split=3)
    assert all(torch.equal(a, b) for a, b in zip(uni, var))
    ru, _ = A.reference(*uni, 5, 0.125)
    rv, _ = AV.reference_varlen(*var, [5, 5], 0.125)
    assert (ru == rv).all()


@pytest.mark.parametrize("kind", ["needle", "random"])
@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_exact_varlen_result_rounded_like_the_kernel_passes(shape, kind):
    hd, ql = shape[0], shape[3]
    inp = _inputs(shape, kind)
    ref, S = AV.reference_varlen(*inp, ql, hd ** -0.5)
    rp, _ = AV.reference_varlen(*inp, ql, hd ** -0.5, round_p=True)
    r = A.err_over_bound(_rounded(rp), ref, S)
    print(f"[varlen attention checker] {kind}: P and output rounded {r:.3f}")
    assert r <= 0.5


@pytest.mark.parametrize("defect", A.DEFECTS_POSITIONAL + AV.DEFECTS_VARLEN)
@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_every_varlen_defect_fails_the_check_on_needles(shape, defect):
    hd, H, KV, ql, bs, ctx, ns = shape
    if defect == "swap_heads" and H // KV < 2:
        pytest.skip("no GQA group")
    inp = _inputs(shape, "needle")
    ref, S = AV.reference_varlen(*inp, ql, hd ** -0.5)
    bad, _ = AV.reference_varlen(*inp, ql, hd ** -0.5, defect=defect, n_split=ns)
    r = A.err_over_bound(_rounded(bad), ref, S)
    assert r > 1.0, f"{defect} passes the check (worst err/bound {r:.3f})"
