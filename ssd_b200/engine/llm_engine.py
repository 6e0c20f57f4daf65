"""LLMEngine — the object bench/bench.py drives: LLM(model, **kwargs).generate(prompts, sampling_params)
-> (outputs, METRICS), with the METRICS keys and counting rules of ssd/engine/llm_engine.py:25-36,193-235,321-381.
Host orchestration stays Python; every model FLOP and the accept/reject logic run inside libssdk."""
from __future__ import annotations

import atexit
from dataclasses import fields
from time import perf_counter

from ..config import Config
from ..sampling_params import SamplingParams
from .scheduler import Scheduler
from .sequence import Sequence
from .step import AutoRegressiveStep, InferenceStep, SpecDecodeStep

METRICS = {
    "cache_hits": [],
    "accepted_suffix_lens_with_recovery": [],
    "accepted_suffix_lens_on_hit": [],
    "accepted_suffix_lens_on_miss": [],
    "prefill_total_time": 0,
    "decode_total_time": 0,
    "prefill_total_tokens": 0,
    "decode_total_tokens": 0,
    "target_step_times": [],
    "target_verify_times": [],
}


def infer_model_family(path: str) -> str:
    p = path.lower()
    return "llama" if "llama" in p else ("qwen" if "qwen" in p else "unknown")


class LLMEngine:
    def __init__(self, model, **kwargs):
        known = {f.name for f in fields(Config)}
        config = Config(model, **{k: v for k, v in kwargs.items() if k in known})  # unknown kwargs dropped (llm_engine.py:42-44)
        self.config = config
        Sequence.block_size = config.kvcache_block_size
        if config.kvcache_block_size < 2 * config.speculate_k + 2:
            raise AssertionError("block size < 2*k+2 is not supported (llm_engine.py:48-49)")
        if config.speculate:
            tf, df = infer_model_family(config.model), infer_model_family(config.draft)
            if tf != df:
                raise AssertionError("target and draft must be of the same model family (llm_engine.py:55-57)")
        self._workers = None
        if config.num_gpus > 1:
            from ..parallel import launch_tp_engine
            self.runner, self.draft_cfg, self._workers = launch_tp_engine(config, model, kwargs)
        else:
            from ..loader import build_runner
            self.runner, self.draft_cfg = build_runner(config)
        self.model_runner = self.runner
        self.tokenizer = _load_tokenizer(config)
        config.eos = getattr(self.tokenizer, "eos_token_id", -1)
        if config.eos is None:
            config.eos = -1
        self.scheduler = Scheduler(config, draft_cfg=self.draft_cfg if config.speculate else None)
        self._exiting = False
        atexit.register(self.exit)

    def exit(self, hard: bool = False):
        """Tear down TP workers and the runner (llm_engine.py:126-184).  The reference's atexit hook always ends with
        os._exit(0) to get rid of its helper processes; here that is only done when the caller asks for it (hard=True)."""
        if self._exiting:
            return
        self._exiting = True
        try:
            if self._workers is not None:
                self._workers.close()
        except Exception:
            pass
        try:
            self.runner.close()
        except Exception:
            pass
        if hard:
            import os
            os._exit(0)

    def add_request(self, prompt, sampling_params: SamplingParams):
        if isinstance(prompt, str):
            prompt = self.tokenizer.encode(prompt)
        self.scheduler.add(Sequence(prompt, sampling_params))

    def create_inference_step(self, config: Config) -> InferenceStep:
        if config.speculate:
            return SpecDecodeStep(self.scheduler, self.runner, config.speculate_k, METRICS, self.tokenizer, config.seed,
                                  varlen_prefill=config.varlen_prefill)
        return AutoRegressiveStep(self.scheduler, self.runner, self.tokenizer, config.seed,
                                  varlen_prefill=config.varlen_prefill)

    def step(self, step: InferenceStep):
        t = perf_counter()
        seqs, is_prefill = self.scheduler.schedule()
        retired, self.scheduler.retired = self.scheduler.retired, []
        if not seqs:  # every runnable sequence ran out of room below max_model_len and was finished by schedule()
            return [(s.seq_id, s.completion_token_ids) for s in retired]
        n = step.prefill(seqs) if is_prefill else step.decode(seqs)
        dt = perf_counter() - t
        if is_prefill:
            METRICS["prefill_total_time"] += dt
            METRICS["prefill_total_tokens"] += n
        else:
            METRICS["decode_total_time"] += dt
            METRICS["decode_total_tokens"] += n
        return [(s.seq_id, s.completion_token_ids) for s in seqs if s.is_finished] + \
               [(s.seq_id, s.completion_token_ids) for s in retired]

    def is_finished(self):
        return self.scheduler.is_finished()

    def log_metrics(self):
        if METRICS["prefill_total_time"]:
            print(f"Final Prefill Throughput: {int(METRICS['prefill_total_tokens'] / METRICS['prefill_total_time'])}tok/s", flush=True)
        if METRICS["decode_total_time"]:
            print(f"Final Decode Throughput: {int(METRICS['decode_total_tokens'] / METRICS['decode_total_time'])}tok/s", flush=True)
        lens = METRICS["accepted_suffix_lens_with_recovery"]
        if self.config.speculate and lens:
            mean = sum(lens) / len(lens)
            print(f"[metrics] Avg Tokens per step (incl recovery): {mean:.2f}", flush=True)
            print(f"[metrics] Avg Fraction of Speculated Tokens Accepted: {(mean - 1) / self.config.speculate_k:.2f}", flush=True)
            if METRICS["target_step_times"]:
                print(f"[metrics] Avg target time per full step (ms): "
                      f"{sum(METRICS['target_step_times']) * 1000 / len(METRICS['target_step_times']):.2f}", flush=True)

    def generate(self, prompts, sampling_params, use_tqdm: bool = True, stream_callback=None):
        for k in METRICS:
            METRICS[k] = [] if isinstance(METRICS[k], list) else 0
        if self._workers is not None:  # spawned TP ranks replay the same call (SPMD host engines)
            self._workers.generate(prompts, sampling_params, stream_callback is not None)
        if not isinstance(sampling_params, list):
            sampling_params = [sampling_params] * len(prompts)
        for p, sp in zip(prompts, sampling_params):
            self.add_request(p, sp)
        pbar = None
        if use_tqdm:
            from tqdm.auto import tqdm
            pbar = tqdm(total=len(prompts), desc="Generating", dynamic_ncols=True)
        outputs = {}
        step = self.create_inference_step(self.config)
        max_steps = self.config.max_steps if self.config.max_steps is not None else float("inf")
        i, seen = 0, {}
        while not self.is_finished() and i < max_steps:
            i += 1
            t = perf_counter()
            done = self.step(step)
            METRICS["target_step_times"].append(perf_counter() - t)
            if stream_callback:
                for seq in self.scheduler.running:
                    cur, prev = seq.num_completion_tokens, seen.get(seq.seq_id, 0)
                    if cur > prev:
                        stream_callback(seq.seq_id, seq.completion_token_ids[prev:cur])
                        seen[seq.seq_id] = cur
            for seq_id, toks in done:
                if stream_callback:
                    prev = seen.get(seq_id, 0)
                    if len(toks) > prev:
                        stream_callback(seq_id, toks[prev:])
                outputs[seq_id] = toks
                if pbar:
                    pbar.update(1)
        if pbar:
            pbar.close()
        outs = [{"text": self.tokenizer.decode(outputs[k]), "token_ids": outputs[k]} for k in sorted(outputs)]
        if not stream_callback:
            self.log_metrics()
        return outs, METRICS


def _load_tokenizer(config):
    """AutoTokenizer.from_pretrained(config.model) (llm_engine.py:116); synthetic model directories ship a
    WordLevel tokenizer.json, read directly with `tokenizers` to avoid transformers' network probes."""
    import os
    path = config.tokenizer_path or config.model
    marker = os.path.join(path, "ssd_b200_synthetic.json")
    if os.path.exists(marker):
        from ..synth import SyntheticTokenizer
        return SyntheticTokenizer(path)
    from transformers import AutoTokenizer
    return AutoTokenizer.from_pretrained(path, use_fast=True)
