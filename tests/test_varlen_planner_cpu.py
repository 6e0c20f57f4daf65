"""PairRunner.plan_varlen_calls and prefill_varlen's bookkeeping, with a fake forward_varlen: every prompt token runs
exactly once and in order, calls respect 256 tokens and max_batch sequences, prefix-cache hits only run once the pages
they read are written (the rule in plan_varlen_calls' docstring), batches without hits take ceil(sum / 256) calls, and
each sequence's first token comes from the call that holds its last prompt token."""
import math
import random

import pytest

from ssd_b200.runner import PairRunner

BS = 256


class FakeRunner:
    """prefill_varlen and plan_varlen_calls of PairRunner over a recording forward_varlen (no device)."""
    plan_varlen_calls = staticmethod(PairRunner.plan_varlen_calls)
    prefill_varlen = PairRunner.prefill_varlen

    def __init__(self, max_batch, block_size=BS):
        self.max_batch, self.block_size = max_batch, block_size
        self.calls = []

    def forward_varlen(self, which, ids, ctx_len, block_tables, temps=None, want_sample=True, seed=0):
        c = len(self.calls)
        self.calls.append((ids, ctx_len, want_sample))
        # token sampled for row b: identifies (call, position after the chunk)
        return [c * 100000 + ctx + len(x) for x, ctx in zip(ids, ctx_len)] if want_sample else None


def _batch(rng, n, lo, hi, bs=BS, hits=False):
    """n prompts with fresh pages; with hits, some sequences alias the first pages of an earlier one (chains too)."""
    lens = [rng.randint(lo, hi) for _ in range(n)]
    starts = [0] * n
    bts, nxt = [], 0
    for i in range(n):
        pages = list(range(nxt, nxt + math.ceil(lens[i] / bs)))
        nxt += len(pages)
        bts.append(pages)
    if hits:
        for i in range(1, n):
            if rng.random() < 0.5:
                src = rng.randrange(i)  # may itself be a hit: chains
                full = min(lens[src], lens[i] - 1) // bs
                if full >= 1:
                    k = rng.randint(1, full)
                    bts[i][:k] = bts[src][:k]
                    starts[i] = k * bs
    return lens, starts, bts


def _check(lens, starts, bts, calls, max_batch, bs=BS):
    n = len(lens)
    done = list(starts)
    for call in calls:
        assert 1 <= len(call) <= max_batch
        assert sum(q for _, _, q in call) <= 256
        assert [i for i, _, _ in call] == sorted({i for i, _, _ in call})
        for i, pos, q in call:
            assert pos == done[i] and q >= 1 and pos + q <= lens[i]  # in order, exactly once
            done[i] = pos + q
        for i, pos, q in call:  # the hit rule, with this call's tokens counted
            if starts[i] > 0:
                mine = set(bts[i][:math.ceil(starts[i] / bs)])
                for j in range(n):
                    if j != i and mine & set(bts[j]):
                        assert done[j] >= min(starts[i], lens[j]), (i, j, call)
    assert done == lens


@pytest.mark.parametrize("seed", range(40))
def test_random_batches_with_aliased_pages_and_chains_of_hits(seed):
    rng = random.Random(seed)
    bs = rng.choice([16, 64, 80, 256])
    max_batch = rng.choice([1, 3, 8, 32])
    lens, starts, bts = _batch(rng, rng.randint(1, 32), 1, 900, bs, hits=True)
    calls = PairRunner.plan_varlen_calls(lens, starts, bts, bs, 256, max_batch)
    _check(lens, starts, bts, calls, max_batch, bs)


@pytest.mark.parametrize("lens", [[100, 100, 37, 1, 180, 64, 100, 9], [128] * 16, [600, 1, 255, 256, 257]])
def test_without_hits_calls_are_ceil_of_tokens_over_256(lens):
    bts = [[i] * 4 for i in range(len(lens))]
    calls = PairRunner.plan_varlen_calls(lens, [0] * len(lens), bts, BS, 256, 32)
    _check(lens, [0] * len(lens), bts, calls, 32)
    assert len(calls) == math.ceil(sum(lens) / 256)


@pytest.mark.parametrize("seed", range(10))
def test_random_batches_without_hits(seed):
    rng = random.Random(100 + seed)
    lens, starts, bts = _batch(rng, 32, 1, 200)
    calls = PairRunner.plan_varlen_calls(lens, starts, bts, BS, 256, 32)
    _check(lens, starts, bts, calls, 32)
    assert len(calls) == math.ceil(sum(lens) / 256)


def test_uniform_prompts_group_like_prefill_many():
    """16 x 128 tokens: two prompts per call, in order — the grouping plan_prefill_call picks."""
    calls = PairRunner.plan_varlen_calls([128] * 16, [0] * 16, [[i] for i in range(16)], BS, 256, 16)
    assert [[(i, 0, 128) for i in (2 * c, 2 * c + 1)] for c in range(8)] == calls


def test_shared_prefix_batch_takes_seven_calls():
    """16 prompts of a 512-token shared prefix + 70 own tokens, 256-token pages: the first writes the two shared pages,
    the other 15 join as soon as those are written."""
    lens = [582] * 16
    bts = [[0, 1, 2 + i] for i in range(16)]
    starts = [0] + [512] * 15
    calls = PairRunner.plan_varlen_calls(lens, starts, bts, BS, 256, 16)
    _check(lens, starts, bts, calls, 16)
    assert len(calls) == math.ceil((582 + 15 * 70) / 256) == 7


def test_hits_may_join_the_call_that_writes_their_pages():
    # sequence 1 reads the first page of sequence 0, which is written in full by the first call
    calls = PairRunner.plan_varlen_calls([300, 300], [0, 256], [[0, 1], [0, 2]], BS, 256, 8)
    assert calls[0] == [(0, 0, 256)]
    assert (1, 256, 44) in calls[1]


@pytest.mark.parametrize("seed", range(10))
def test_prefill_varlen_samples_each_sequence_on_its_last_call(seed):
    rng = random.Random(200 + seed)
    max_batch = rng.choice([4, 32])
    lens, starts, bts = _batch(rng, rng.randint(1, 20), 1, 700, hits=True)
    fr = FakeRunner(max_batch)
    toks = [[rng.randrange(1000) for _ in range(n)] for n in lens]
    out = fr.prefill_varlen(0, toks, bts, starts, seed=1)
    calls = PairRunner.plan_varlen_calls(lens, starts, bts, BS, 256, max_batch)
    assert len(fr.calls) == len(calls)
    for c, (call, (ids, ctx, want)) in enumerate(zip(calls, fr.calls)):
        assert ids == [toks[i][pos:pos + q] for i, pos, q in call] and ctx == [pos for _, pos, _ in call]
        assert want == any(pos + q == lens[i] for i, pos, q in call)
        for i, pos, q in call:
            if pos + q == lens[i]:
                assert out[i] == c * 100000 + lens[i]
    assert fr.prefill_varlen(0, toks, bts, starts, want_sample=False) is None
