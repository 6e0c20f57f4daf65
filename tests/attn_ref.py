"""fp64 reference of paged attention, the error bound the kernel's roundings allow, and the inputs that make indexing
errors visible.  Shared by the checker's self-test (test_attention_ref_cpu.py), the kernel source on host threads
(test_attention_emu_cpu.py) and the device (test_attention_gpu.py).

Semantics are those of oracle.ops.paged_attention: softmax(q kᵀ·scale + causal) v, the causal limit aligned to the end
of the context (query j of a sequence of context L sees positions <= L - Q + j), head h reads KV head h // G, pages are
looked up through the block table and entries past the context (-1) are never read.

Bound.  The kernel is exact up to two bf16 roundings: the softmax weights P (relative to the running maximum) are
rounded to bf16 before P·V, at most 2^-8 relative per weight, which moves an output by at most 2^-8·S with
S = Σ_i p_i·|v_i|; and the output is rounded to bf16, at most 2^-8·|out|.  Everything else is fp32.  The check is
|out - ref| <= 2^-7·(|ref| + S) + 1e-6: twice the worst case.

Needle inputs.  Background keys are 0.25·N(0, 1).  A needle row's query is c·e_d (e_d a basis direction of head_dim)
and the key at its chosen position n is given the component 4 in direction d, so the needle outscores every background
key by >= 30 nats: the row's output is v[n] if n is visible and a background average if it is masked.  Rows of one KV
head use distinct directions, so up to head_dim needles share a launch.  An off-by-one, a dropped position, a wrong
page or a lost KV split at a needle's position is then an O(1) error instead of a 1/L one.
"""
from __future__ import annotations

import math

import numpy as np
import torch

BOUND_REL = 2.0 ** -7
BOUND_ABS = 1e-6
CHUNK = 64           # KV positions per chunk of the kernel
MAX_SPLIT = 32       # most KV splits the planner picks (kAttnMaxSplit)
NEEDLE_KEY = 4.0
NEEDLE_Q = 256.0     # c: 4c·scale >= 90 nats at head_dim 128, background |c·k·scale| <= ~30

DEFECTS_POSITIONAL = ("causal_plus_1", "causal_minus_1", "drop_first", "drop_last", "wrong_page", "swap_heads",
                      "drop_split")
DEFECTS = DEFECTS_POSITIONAL + ("scale_no_log2e",)


def to_bf16_values(x: np.ndarray) -> np.ndarray:
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).double().numpy()


def split_ranges(L: int, n_split: int) -> list[tuple[int, int]]:
    """KV position ranges of the splits the kernel uses for the query tile that ends at position L (the last tile of a
    sequence of context L): each split owns ceil(chunks / n_split) consecutive 64-token chunks."""
    nch = (L + CHUNK - 1) // CHUNK
    cps = (nch + n_split - 1) // n_split
    return [(s * cps * CHUNK, min(L, (s + 1) * cps * CHUNK)) for s in range(n_split) if s * cps < nch]


def reference(q, k_cache, v_cache, block_tables, context_lens, q_len: int, scale: float, *, defect: str | None = None,
              n_split: int = 1, round_p: bool = False):
    """float64 paged attention.  Returns (out [B*Q, H, hd], S [B*Q, H, hd]) with S = Σ_i p_i·|v_i|.

    `defect` applies one of DEFECTS (the self-test's stand-ins for kernel bugs); `round_p` rounds the unnormalised
    weights to bf16 before P·V as the kernel does."""
    qn = q.double().numpy()
    kc, vc = k_cache.double().numpy(), v_cache.double().numpy()
    nblk, bs, KV, hd = kc.shape
    Mq, H, _ = qn.shape
    Q, B, G = q_len, Mq // q_len, H // KV
    kflat, vflat = kc.reshape(-1, KV, hd), vc.reshape(-1, KV, hd)
    bt, ctx = block_tables.numpy(), context_lens.numpy()
    sc = scale * (math.log(2.0) if defect == "scale_no_log2e" else 1.0)  # exp2(s·scale) instead of exp2(s·scale·log2 e)
    out, S = np.zeros((Mq, H, hd)), np.zeros((Mq, H, hd))
    for b in range(B):
        L = int(ctx[b])
        pos = np.arange(L)
        pages = bt[b, pos // bs].astype(np.int64)
        assert (pages >= 0).all(), "block table has -1 inside the context"
        slots = pages * bs + pos % bs
        if defect == "wrong_page":  # the second chunk (or the only one) read from the next physical page
            sel = pos // CHUNK == min(1, (L - 1) // CHUNK)
            slots[sel] = (slots[sel] + bs) % (nblk * bs)
        K, V = kflat[slots].transpose(1, 0, 2), vflat[slots].transpose(1, 0, 2)  # [KV, L, hd]
        qb = qn[b * Q:(b + 1) * Q].reshape(Q, KV, G, hd)
        if defect == "swap_heads":  # heads 0 and 1 of every GQA group exchanged
            qb = qb[:, :, [1, 0] + list(range(2, G))]
        rows = qb.transpose(1, 0, 2, 3).reshape(KV, Q * G, hd)  # row = j * G + g
        s = rows @ K.transpose(0, 2, 1) * sc  # [KV, Q*G, L]
        last = L - Q + np.arange(Q)  # last visible position of query j
        if defect == "causal_plus_1":
            last = last + 1
        elif defect == "causal_minus_1":
            last = last - 1
        vis = pos[None, :] <= last[:, None]  # [Q, L]
        if defect == "drop_first":
            vis &= pos[None, :] != 0
        elif defect == "drop_last":
            vis &= pos[None, :] != last[:, None]
        elif defect == "drop_split":  # the second split's partial lost (the first if there is only one)
            rg = split_ranges(L, n_split)
            lo, hi = rg[min(1, len(rg) - 1)]
            vis &= ~((pos[None, :] >= lo) & (pos[None, :] < hi))
        vis = np.repeat(vis, G, axis=0)[None]  # [1, Q*G, L]
        s = np.where(vis, s, -np.inf)
        m = s.max(-1, keepdims=True)
        m = np.where(np.isfinite(m), m, 0.0)
        e = np.exp(s - m)
        l = e.sum(-1, keepdims=True)
        inv = np.where(l > 0, 1.0 / np.where(l > 0, l, 1.0), 0.0)
        pe = to_bf16_values(e) if round_p else e
        o = (pe @ V) * inv
        sa = (e @ np.abs(V)) * inv
        out[b * Q:(b + 1) * Q] = o.reshape(KV, Q, G, hd).transpose(1, 0, 2, 3).reshape(Q, H, hd)
        S[b * Q:(b + 1) * Q] = sa.reshape(KV, Q, G, hd).transpose(1, 0, 2, 3).reshape(Q, H, hd)
    return out, S


def err_over_bound(out, ref: np.ndarray, S: np.ndarray) -> float:
    """max over elements of |out - ref| / bound; NaN or inf in `out` count as infinitely wrong."""
    o = out.double().numpy() if isinstance(out, torch.Tensor) else np.asarray(out, dtype=np.float64)
    o = o.reshape(ref.shape)
    err = np.nan_to_num(np.abs(o - ref), nan=np.inf)
    return float((err / (BOUND_REL * (np.abs(ref) + S) + BOUND_ABS)).max())


def make_inputs(hd: int, H: int, KV: int, Q: int, bs: int, ctx: list[int], *, kind: str, seed: int,
                max_blocks: int | None = None, alias: bool = False, n_split: int = 1):
    """bf16 inputs for one launch: q [B*Q, H, hd], caches [nblk, bs, KV, hd], block tables [B, max_blocks] (random
    non-contiguous pages, -1 past each context), context lengths [B].

    kind "random": q, k, v ~ N(0, 1).  kind "needle": see the module docstring; needles sit at position 0 and L-1, at
    each row's last visible and first masked position, at page, 64-token chunk and KV-split boundaries.  `alias`:
    sequence 1 shares the first pages of sequence 0, as the prefix cache does.  `n_split` only places needles on the
    split boundaries."""
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
    if kind == "random":
        q = torch.randn(B * Q, H, hd, generator=g)
        kc = torch.randn(nblk, bs, KV, hd, generator=g)
    else:
        q = torch.randn(B * Q, H, hd, generator=g)
        kc = 0.25 * torch.randn(nblk, bs, KV, hd, generator=g)
    vc = torch.randn(nblk, bs, KV, hd, generator=g)
    if kind == "needle":
        kflat = kc.view(-1, KV, hd)
        for kvh in range(KV):
            d = 0  # next free direction of this KV head (shared by all sequences: aliased pages stay unambiguous)
            for b in range(B):
                L = ctx[b]
                common = {0, L - 1}
                for step in (bs, CHUNK):
                    for x in range(step, L, step):
                        common |= {x - 1, x}
                for lo, _ in split_ranges(L, n_split)[1:]:
                    common |= {lo - 1, lo}
                common = sorted(c for c in common if 0 <= c < L)
                for j in range(Q):
                    last = L - Q + j
                    own = [last] + ([last + 1] if last + 1 < L else [])
                    for gg in range(G):
                        if d >= hd:
                            break
                        k = j * G + gg
                        n = own[k % len(own)] if k % 3 != 2 else common[(k // 3 * 7 + b) % len(common)]
                        q[b * Q + j, kvh * G + gg] = 0.0
                        q[b * Q + j, kvh * G + gg, d] = NEEDLE_Q
                        slot = int(bt[b, n // bs]) * bs + n % bs
                        kflat[slot, kvh, d] = NEEDLE_KEY
                        d += 1
    bf = lambda t: t.to(torch.bfloat16)
    return bf(q), bf(kc), bf(vc), bt, torch.tensor(ctx, dtype=torch.int32)
