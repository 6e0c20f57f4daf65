"""Self-test of the attention checker (tests/attn_ref.py): the comparison the kernel tests use must fail for each kind of
defect a paged-attention kernel is prone to, and pass for the exact result rounded the way the kernel rounds.

Each defect is applied to the fp64 reference, the result is rounded to bf16 and compared with the unmutated reference
under the same bound as the kernel.  Positional and page defects must fail on needle inputs at every shape, and on
random inputs at contexts <= 1024 (beyond that a one-token error in a random average is about as small as the rounding
bound, which is why the needle inputs exist).  The scale defect must fail on random inputs.  So loosening the bound, or
weakening the inputs, turns this test red."""
import pytest
import torch

from tests import attn_ref as A

# (hd, H, KV, Q, block size, contexts, n_split)
SHAPES = [
    (64, 8, 2, 7, 16, [300, 7], 3),       # G 4, verify K = 6, pages of 16, ragged batch with ctx == Q
    (128, 6, 2, 5, 80, [1000], 5),        # G 3, pages of 80 straddle chunks
    (64, 4, 1, 8, 32, [8, 1024], 4),      # G 4, ctx == Q next to 1024
    (128, 12, 4, 33, 64, [33], 1),        # ragged prefill tile, one split
    (128, 16, 1, 2, 256, [2000], 32),     # G 16, 32 splits (needle inputs only for positional defects)
]
IDS = [f"hd{s[0]}_h{s[1]}_kv{s[2]}_q{s[3]}_bs{s[4]}_ctx{max(s[5])}" for s in SHAPES]


def _rounded(x):
    return torch.from_numpy(A.to_bf16_values(x))


def _inputs(shape, kind):
    hd, H, KV, Q, bs, ctx, ns = shape
    return A.make_inputs(hd, H, KV, Q, bs, ctx, kind=kind, seed=7, n_split=ns)


@pytest.mark.parametrize("kind", ["needle", "random"])
@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_exact_result_rounded_like_the_kernel_passes(shape, kind):
    hd, Q = shape[0], shape[3]
    inp = _inputs(shape, kind)
    ref, S = A.reference(*inp, Q, hd ** -0.5)
    r_out = A.err_over_bound(_rounded(ref), ref, S)
    rp, _ = A.reference(*inp, Q, hd ** -0.5, round_p=True)
    r_p = A.err_over_bound(_rounded(rp), ref, S)
    print(f"[attention checker] {kind}: output rounded {r_out:.3f}, P and output rounded {r_p:.3f}")
    # two bf16 roundings use at most half of the bound
    assert r_out <= 0.5 and r_p <= 0.5


@pytest.mark.parametrize("defect", A.DEFECTS)
@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_every_defect_fails_the_check(shape, defect):
    hd, H, KV, Q, bs, ctx, ns = shape
    if defect == "swap_heads" and H // KV < 2:
        pytest.skip("no GQA group")
    kinds = []
    if defect in A.DEFECTS_POSITIONAL:
        kinds.append("needle")
    if defect not in A.DEFECTS_POSITIONAL or max(ctx) <= 1024:
        kinds.append("random")
    for kind in kinds:
        inp = _inputs(shape, kind)
        ref, S = A.reference(*inp, Q, hd ** -0.5)
        bad, _ = A.reference(*inp, Q, hd ** -0.5, defect=defect, n_split=ns)
        r = A.err_over_bound(_rounded(bad), ref, S)
        assert r > 1.0, f"{defect} on {kind} inputs passes the check (worst err/bound {r:.3f})"
