"""Varlen counterpart of tests/attn_ref.py: sequences of one launch have their own q_len and their query rows are packed
in sequence order (q [sum q_lens, H, hd]).  Same fp64 semantics, the same bound (attn_ref.err_over_bound) and the same
needle construction, with each needle at its own sequence's last visible (L_b - q_b + j) or first masked position.

Shared by the varlen checker's self-test (test_attention_varlen_ref_cpu.py), the varlen kernel source on host threads
(test_attention_varlen_emu_cpu.py) and the device (test_varlen_gpu.py)."""
from __future__ import annotations

import numpy as np
import torch

from tests import attn_ref as A

# varlen launches: the causal limit taken from the call's longest q_len instead of the sequence's own, and the first
# sequence's query rows read one packed row late
DEFECTS_VARLEN = ("causal_from_qmax", "rows_shifted")


def reference_varlen(q, k_cache, v_cache, block_tables, context_lens, q_lens: list[int], scale: float, *,
                     defect: str | None = None, n_split: int = 1, round_p: bool = False):
    """attn_ref.reference for packed sequences of their own q_lens[b].  Returns (out, S) like attn_ref.reference.
    `defect` is one of attn_ref.DEFECTS (applied to every sequence) or DEFECTS_VARLEN."""
    cu = np.concatenate([[0], np.cumsum(q_lens)]).astype(int)
    qmax = max(q_lens)
    out, S = [], []
    for b, qb in enumerate(q_lens):
        rows = q[cu[b]:cu[b + 1]]
        if defect == "rows_shifted" and b == 0:
            rows = torch.roll(q, -1, 0)[cu[b]:cu[b + 1]]
        Q = qb
        if defect == "causal_from_qmax" and qb < qmax:
            # attn_ref.reference aligns query j of a q_len-Q call to L - Q + j: padding the rows to qmax (dummy rows
            # after them) puts row j at L - qmax + j
            rows = torch.cat([rows, torch.zeros(qmax - qb, *rows.shape[1:], dtype=rows.dtype)])
            Q = qmax
        o, s = A.reference(rows, k_cache, v_cache, block_tables[b:b + 1], context_lens[b:b + 1], Q, scale,
                           defect=defect if defect in A.DEFECTS else None, n_split=n_split, round_p=round_p)
        out.append(o[:qb])
        S.append(s[:qb])
    return np.concatenate(out), np.concatenate(S)


def make_inputs_varlen(hd: int, H: int, KV: int, q_lens: list[int], bs: int, ctx: list[int], *, kind: str, seed: int,
                       max_blocks: int | None = None, alias: bool = False, n_split: int = 1):
    """attn_ref.make_inputs for packed sequences of their own q_lens[b]: same draws in the same order, so equal q_lens
    give exactly attn_ref.make_inputs' tensors (test_attention_varlen_ref_cpu.py checks this)."""
    cu = np.concatenate([[0], np.cumsum(q_lens)]).astype(int)
    g = torch.Generator().manual_seed(seed)
    B, G = len(ctx), H // KV
    used = [(L + bs - 1) // bs for L in ctx]
    mb = max_blocks if max_blocks is not None else max(used) + 1
    assert mb >= max(used)
    nblk = sum(used) + 3
    perm = torch.randperm(nblk, generator=g).tolist()
    bt = torch.full((B, mb), -1, dtype=torch.int32)
    nxt = 0
    for b in range(B):
        for i in range(used[b]):
            bt[b, i] = perm[nxt]
            nxt += 1
    if alias and B > 1:
        shared = min(used[0], used[1]) - 1
        bt[1, :shared] = bt[0, :shared]
    q = torch.randn(int(cu[-1]), H, hd, generator=g)
    kc = torch.randn(nblk, bs, KV, hd, generator=g)
    if kind != "random":
        kc = 0.25 * kc
    vc = torch.randn(nblk, bs, KV, hd, generator=g)
    if kind == "needle":
        kflat = kc.view(-1, KV, hd)
        for kvh in range(KV):
            d = 0  # next free direction of this KV head (shared by all sequences: aliased pages stay unambiguous)
            for b in range(B):
                L = ctx[b]
                common = {0, L - 1}
                for step in (bs, A.CHUNK):
                    for x in range(step, L, step):
                        common |= {x - 1, x}
                for lo, _ in A.split_ranges(L, n_split)[1:]:
                    common |= {lo - 1, lo}
                common = sorted(c for c in common if 0 <= c < L)
                for j in range(q_lens[b]):
                    last = L - q_lens[b] + j
                    own = [last] + ([last + 1] if last + 1 < L else [])
                    for gg in range(G):
                        if d >= hd:
                            break
                        k = j * G + gg
                        n = own[k % len(own)] if k % 3 != 2 else common[(k // 3 * 7 + b) % len(common)]
                        q[cu[b] + j, kvh * G + gg] = 0.0
                        q[cu[b] + j, kvh * G + gg, d] = A.NEEDLE_Q
                        slot = int(bt[b, n // bs]) * bs + n % bs
                        kflat[slot, kvh, d] = A.NEEDLE_KEY
                        d += 1
    bf = lambda t: t.to(torch.bfloat16)
    return bf(q), bf(kc), bf(vc), bt, torch.tensor(ctx, dtype=torch.int32)
