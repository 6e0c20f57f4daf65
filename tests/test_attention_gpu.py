"""Paged attention on the device (ssd_b200.ops.paged_attention -> paged_attn_kernel + attn_combine_kernel) against the
fp64 reference of tests/attn_ref.py, within the bound the kernel's two bf16 roundings allow:
|out - ref| <= 2^-7·(|ref| + Σ p_i|v_i|) + 1e-6.

Every case runs twice: on random inputs, and on needle inputs whose outputs flip by O(1) when a position, a page, a head
or a KV split is read wrongly.  The cases cover head_dim 64 and 128; GQA ratios 1-8, 12 and 16, including the real
(32, 8), (64, 8) and (16, 8); verify lengths K+1 = 1..8 and prefill tiles of 16, 33, 64 and 256 tokens; pages of 16, 32,
64, 256 and 80 tokens (80 straddles the 64-token chunks, so the per-token page lookup runs); ctx == Q, a context of 1,
ragged batches of up to 32 sequences, contexts up to 8192 and one of 16384; -1 block-table tails and sequences that
share prefix pages.  max_blocks is chosen per case so that the planner takes each kind of plan on any H100
(test_plans_reached asserts which ones ran)."""
import shutil

import numpy as np
import pytest
import torch

from tests import attn_ref as A

pytestmark = pytest.mark.gpu

_RAGGED32 = [int(x) for x in np.random.default_rng(3).integers(8, 1500, 32)]
_RAGGED16 = [int(x) for x in np.random.default_rng(4).integers(16, 3000, 16)]

# (id, hd, H, KV, Q, block size, contexts, max_blocks (None: just enough pages), alias)
CASES = [
    ("ctx1_g1_bs16_split1", 64, 4, 4, 1, 16, [1], 4, False),                 # max_ctx 64: one split
    ("ctxq_g2_q2_bs32_split1", 128, 8, 4, 2, 32, [2], 2, False),
    ("ctxq_g12_q33_bs16_split1", 128, 12, 1, 33, 16, [33], 4, False),        # 2 tokens x 12 heads per tile, ragged tile
    ("g3_q3_bs80_split5", 64, 6, 2, 3, 80, [3, 200, 81], 4, False),          # max_ctx 320: five splits, -1 tails
    ("g4_h32kv8_q5_bs80_split5", 128, 32, 8, 5, 80, [300], 4, False),
    ("g5_q7_bs16_ragged", 64, 10, 2, 7, 16, [7, 1000, 64, 65], None, False),
    ("g6_q8_bs64", 128, 12, 2, 8, 64, [300, 8, 4097], None, False),
    ("g7_q7_bs80_split32", 64, 7, 1, 7, 80, [2100], 27, False),              # 33 chunks in 32 splits: 17 active, 2 each
    ("g8_q1_bs16_8k_split32", 128, 8, 1, 1, 16, [8192], 512, False),         # 128 chunks: 32 active splits of 4
    ("g16_q2_bs256_16k_split32", 128, 16, 1, 2, 256, [16384], 64, False),    # 256 chunks: splits of 8
    ("g4_q1_bs64_split32_trailing", 64, 4, 1, 1, 64, [300], 40, False),      # 5 chunks: 27 empty splits
    ("g8_h64kv8_q7_bs256", 128, 64, 8, 7, 256, [4000], None, False),
    ("g2_h16kv8_q8_bs256_8k", 128, 16, 8, 8, 256, [8192], None, False),
    ("g4_h32kv8_q8_bs32_8k", 128, 32, 8, 8, 32, [8192], None, False),
    ("g16_h32kv2_q1", 64, 32, 2, 1, 256, [5000, 17], None, False),
    ("g4_b32_q8_bs32_ragged", 64, 4, 1, 8, 32, _RAGGED32, None, False),
    ("g2_b16_q16_bs16_ragged", 128, 4, 2, 16, 16, _RAGGED16, None, False),
    ("g1_q64_bs256", 128, 2, 2, 64, 256, [1064, 64], None, False),
    ("g2_q256_bs64_ctxq", 64, 4, 2, 256, 64, [256], None, False),
    ("g1_q256_bs80", 128, 8, 8, 256, 80, [1300], None, False),
    ("g3_q33_bs80", 64, 3, 1, 33, 80, [33, 700], None, False),
    ("g1_q5_bs256", 128, 8, 8, 5, 256, [5, 300], None, False),
    ("alias_g4_q7_bs16", 64, 8, 2, 7, 16, [900, 1000], None, True),
    ("alias_g2_q8_bs64", 128, 16, 8, 8, 64, [2000, 2100], None, True),
]

WORST: dict[str, float] = {}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from ssd_b200 import lib
    lib.load()  # fails loudly if libssdk.so is missing
    return torch.device("cuda:0")


def _max_blocks(case):
    _, _, _, _, _, bs, ctx, mb, _ = case
    return mb if mb is not None else (max(ctx) + bs - 1) // bs + 1


def plan_of(case):
    """The device's plan for this case plus, per query tile, the chunks per split and the active splits (the formula
    the kernel and attn_combine_kernel use)."""
    from ssd_b200 import ops
    _, hd, H, KV, Q, bs, ctx, _, _ = case
    pl = ops.paged_attention_plan(len(ctx), Q, H, KV, bs * _max_blocks(case))
    tiles = []
    for L in ctx:
        for qt in range(pl["n_qtiles"]):
            tq = min(pl["TQ"], Q - qt * pl["TQ"])
            nch = (L - Q + qt * pl["TQ"] + tq + A.CHUNK - 1) // A.CHUNK
            cps = (nch + pl["n_split"] - 1) // pl["n_split"]
            tiles.append((cps, (nch + cps - 1) // cps))
    return {**pl, "max_cps": max(c for c, _ in tiles), "n_active": sorted({a for _, a in tiles})}


def _record(family, r):
    WORST[family] = max(WORST.get(family, 0.0), r)


@pytest.mark.parametrize("kind", ["random", "needle"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_paged_attention_matches_fp64(dev, case, kind):
    from ssd_b200 import ops
    name, hd, H, KV, Q, bs, ctx, _, alias = case
    assert len(ctx) * Q <= 256
    pl = plan_of(case)
    q, kc, vc, bt, cl = A.make_inputs(hd, H, KV, Q, bs, ctx, kind=kind, seed=sum(map(ord, name)),
                                      max_blocks=_max_blocks(case), alias=alias, n_split=pl["n_split"])
    out = ops.paged_attention(q.to(dev), kc.to(dev), vc.to(dev), bt.to(dev), cl.to(dev), Q, hd ** -0.5).cpu()
    ref, S = A.reference(q, kc, vc, bt, cl, Q, hd ** -0.5)
    r = A.err_over_bound(out, ref, S)
    _record(kind, r)
    print(f"[attention gpu] {name} {kind}: plan {pl}, worst err/bound {r:.3f}")
    assert r <= 1.0, f"worst err/bound {r:.3f}"


def test_plans_reached(dev):
    """Between them the cases take every kind of launch plan: one split, a middle split count, the 32-way maximum with
    more than 8 active splits (second batch of merge loads) and with empty trailing splits, splits that own several
    chunks, and one and two 16-row MMA tiles."""
    plans = {c[0]: plan_of(c) for c in CASES}
    for name, p in plans.items():
        print(f"[attention plan] {name}: TQ={p['TQ']} MT={p['MT']} n_qtiles={p['n_qtiles']} n_split={p['n_split']} "
              f"max chunks/split={p['max_cps']} active splits={p['n_active']}")
    ps = plans.values()
    assert any(p["n_split"] == 1 for p in ps)
    assert any(1 < p["n_split"] < A.MAX_SPLIT for p in ps)
    assert any(p["n_split"] == A.MAX_SPLIT and max(p["n_active"]) > 8 for p in ps)
    assert any(p["n_split"] == A.MAX_SPLIT and min(p["n_active"]) < A.MAX_SPLIT for p in ps)
    assert any(p["n_split"] == A.MAX_SPLIT and 8 < min(p["n_active"]) < A.MAX_SPLIT for p in ps)
    assert any(p["max_cps"] > 1 for p in ps)
    assert {1, 2} <= {p["MT"] for p in ps}


def test_host_emulation_inputs_on_device(dev, tmp_path):
    """The inputs of the host-thread emulation (test_attention_emu_cpu.py) on the device: both results within the bound.
    If the emulation's cp.async / ldmatrix / mma.sync stand-ins got a fragment layout wrong, the two would disagree."""
    from ssd_b200 import ops
    from tests import test_attention_emu_cpu as E
    have_gxx = shutil.which("g++") is not None
    if have_gxx:
        E.build()
    for case in E.EMU_CASES:
        name, hd, H, KV, Q, bs, ctx, mb, ns, kind = case
        q, kc, vc, bt, cl = inputs = E.case_inputs(case)
        ref, S = A.reference(q, kc, vc, bt, cl, Q, hd ** -0.5)
        out = ops.paged_attention(q.to(dev), kc.to(dev), vc.to(dev), bt.to(dev), cl.to(dev), Q, hd ** -0.5).cpu()
        r_dev = A.err_over_bound(out, ref, S)
        _record("emulation inputs (device)", r_dev)
        msg = f"[attention gpu] emulation case {name}: device {r_dev:.3f}"
        if have_gxx:
            _, emu_out = E.run_emu(tmp_path, case, inputs)
            r_emu = A.err_over_bound(emu_out, ref, S)
            _record("emulation inputs (host threads)", r_emu)
            msg += f", host threads {r_emu:.3f}"
            assert r_emu <= 1.0, msg
        print(msg)
        assert r_dev <= 1.0, msg


def test_worst_err_over_bound_summary(dev):
    if not WORST:
        pytest.skip("run together with the tests above")
    for family, r in sorted(WORST.items()):
        print(f"[attention gpu] worst err/bound, {family}: {r:.3f}")
    assert max(WORST.values()) <= 1.0
