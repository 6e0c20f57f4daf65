"""Inference steps.  AutoRegressiveStep / SpecDecodeStep keep the reference's names and return values
(ssd/engine/step.py:15-163) but a decode is ONE extension call:

    reference  SpecDecodeStep.decode = K+1 x (host prep + graph replay + lm_head + sampler + .tolist())
                                       + target run + ~35-kernel verify() with 5 host syncs
    here       SpecDecodeStep.decode = PairRunner.spec_step -> ssdk_spec_step (one CUDA graph, one sync)
"""
from __future__ import annotations

from abc import ABC, abstractmethod
from time import perf_counter

from .. import lib as L
from .speculate_types import VerifyResult


class InferenceStep(ABC):
    def __init__(self, scheduler):
        self.scheduler = scheduler

    @abstractmethod
    def decode(self, seqs) -> int: ...

    @abstractmethod
    def prefill(self, seqs) -> int: ...


class AutoRegressiveStep(InferenceStep):
    """engine/step.py:29-53."""

    def __init__(self, scheduler, runner, tokenizer=None, seed: int = 0, varlen_prefill: bool = False):
        super().__init__(scheduler)
        self.runner, self.tokenizer, self.seed = runner, tokenizer, seed
        self.prefill_fn = runner.prefill_varlen if varlen_prefill else runner.prefill_many

    def prefill(self, seqs) -> int:
        toks = self.prefill_fn(L.TARGET, [s.token_ids for s in seqs], [s.block_table for s in seqs],
                               [min(s.num_cached_tokens, len(s) - 1) for s in seqs],
                               [s.temperature for s in seqs], seed=self.seed)
        self.scheduler.postprocess(seqs, toks, True)
        return sum(len(s) for s in seqs)

    def decode(self, seqs) -> int:
        toks = self.runner.forward_tokens(L.TARGET, [[s.last_token] for s in seqs], [len(s) - 1 for s in seqs],
                                          [s.block_table for s in seqs], [s.temperature for s in seqs], seed=self.seed)
        self.scheduler.postprocess(seqs, toks, False)
        return len(seqs)


class SpecDecodeStep(InferenceStep):
    """engine/step.py:56-163 for synchronous speculation."""

    def __init__(self, scheduler, runner, lookahead: int, metrics: dict, tokenizer=None, seed: int = 0,
                 varlen_prefill: bool = False):
        super().__init__(scheduler)
        self.runner, self.K, self.metrics, self.tokenizer, self.seed = runner, lookahead, metrics, tokenizer, seed
        self.prefill_fn = runner.prefill_varlen if varlen_prefill else runner.prefill_many

    def prefill(self, seqs) -> int:
        """Target prefill samples the first recovery token (verifier.py:32-52), then the draft caches the prompt
        (speculator_sync.py:14-23).  Prefix-cache hits skip the cached blocks (scheduler.py:71-72)."""
        ids = [s.token_ids for s in seqs]
        # always run at least the last token to get logits
        rec = self.prefill_fn(L.TARGET, ids, [s.block_table for s in seqs],
                              [min(s.num_cached_tokens, len(s) - 1) for s in seqs],
                              [s.temperature for s in seqs], seed=self.seed)
        self.prefill_fn(L.DRAFT, ids, [s.draft_block_table for s in seqs],
                        [min(s.num_draft_cached_tokens, len(s) - 1) for s in seqs], want_sample=False)
        for seq, r in zip(seqs, rec):
            seq.recovery_token_id = r
            seq.num_cached_tokens = seq.num_prompt_tokens
            seq.num_draft_cached_tokens = seq.num_prompt_tokens
        return sum(len(s) for s in seqs)

    def decode(self, seqs) -> int:
        t0 = perf_counter()
        toks, nacc, rec = self.runner.spec_step(
            [s.num_cached_tokens for s in seqs], [s.recovery_token_id for s in seqs],
            [s.block_table for s in seqs], [s.draft_block_table for s in seqs],
            [s.temperature for s in seqs], [s.effective_draft_temperature for s in seqs], seed=self.seed)
        self.metrics["target_verify_times"].append(perf_counter() - t0)
        suffixes = [toks[b, :int(nacc[b]) + 1].tolist() for b in range(len(seqs))]
        # counted BEFORE EOS / max-token truncation, like verifier.py:127 and step.py:163
        self.metrics["accepted_suffix_lens_with_recovery"].extend(len(s) for s in suffixes)
        result = VerifyResult(suffixes, [int(r) for r in rec])
        self.scheduler.postprocess_speculate(seqs, result.new_suffixes, result.recovery_tokens)
        return sum(len(s) for s in suffixes)
