"""The reference's OWN acceptance harness (bench/bench.py, unmodified, SURVEY §2 item 19) driving the ssd_b200 host
engine through the `ssd` compat shim — on CPU, with the device runner replaced by a deterministic test double.

The harness's calls into the engine were recorded by running it unmodified (oracle/gen_harness_golden.py ->
tests/golden/harness_<case>.json): the model path and kwargs of its `create_llm_kwargs` -> `LLM(...)`, and per
`generate()` the prompts, SamplingParams, the `llm.config.max_num_seqs` / `llm.scheduler.max_num_seqs` its sweep path
sets and the METRICS it resets.  The tests replay those calls, in order, through `import ssd.paths`,
`from ssd import LLM, SamplingParams` and `from ssd.engine.llm_engine import METRICS`, and check the drop-in boundary
end to end: the configuration the kwargs produce, `generate()`'s return value, the sweep reconfiguration, and the
scheduler / block-manager bookkeeping under random accept lengths."""
import importlib
import json
import os
import types

import numpy as np

from tests.helpers import GOLDEN

V = 128256


def _next(tok: int) -> int:
    """The fake target model: a fixed permutation-like map; greedy decoding follows it exactly."""
    return (tok * 31 + 7) % V


class FakeRunner:
    """Stands in for PairRunner: the target's greedy next token is _next(last); the draft agrees most of the time."""

    def __init__(self, K):
        self.K = K
        self.rng = np.random.default_rng(0)
        self.calls = {"prefill": 0, "spec_step": 0, "decode": 0}
        self.max_batch_seen = 0

    def prefill(self, which, tokens, block_table, start=0, temp=0.0, want_sample=True, chunk=64, seed=0):
        self.calls["prefill"] += 1
        assert len(block_table) * 256 >= len(tokens), "prefill without enough KV blocks"
        return _next(tokens[-1]) if want_sample else None

    def prefill_many(self, which, tokens, block_tables, starts, temps=None, want_sample=True, chunk=256, seed=0):
        out = [self.prefill(which, t, bt, start=s, want_sample=want_sample) for t, bt, s in zip(tokens, block_tables, starts)]
        return out if want_sample else None

    def forward_tokens(self, which, ids, ctx_len, block_tables, temps=None, want_sample=True, seed=0):
        self.calls["decode"] += 1
        return [_next(x[-1]) for x in ids]

    def spec_step(self, ctx_len, recovery, bt_target, bt_draft, temps_t, temps_q, seed=0):
        self.calls["spec_step"] += 1
        B, K = len(ctx_len), self.K
        self.max_batch_seen = max(self.max_batch_seen, B)
        toks = np.zeros((B, K + 1), dtype=np.int64)
        nacc = np.zeros(B, dtype=np.int32)
        rec = np.zeros(B, dtype=np.int64)
        for b in range(B):
            for t in (bt_target[b], bt_draft[b]):
                assert len(t) * 256 >= ctx_len[b] + K + 1, "look-ahead KV slots were not reserved"
            n = int(self.rng.integers(0, K + 1))
            cur = recovery[b]
            toks[b, 0] = cur
            for j in range(K):
                cur = _next(cur) if j < n else (_next(cur) + 1) % V  # first wrong token at position n
                toks[b, j + 1] = cur
            nacc[b] = n
            last = toks[b, n]
            rec[b] = _next(int(last))
        return toks, nacc, rec

    def close(self):
        pass


def _make_hf_cache(root):
    from ssd_b200 import synth
    for repo, shape, role in (("models--meta-llama--Llama-3.1-8B-Instruct", "llama-3.1-8b", "target"),
                              ("models--meta-llama--Llama-3.2-1B-Instruct", "llama-3.2-1b", "draft")):
        snap = os.path.join(root, repo, "snapshots")
        os.makedirs(snap, exist_ok=True)
        made = synth.make_model_dir(snap, shape, role)
        os.rename(made, os.path.join(snap, "synthetic"))


def _run_bench(tmp_path, monkeypatch, case):
    """Replay the reference harness's recorded calls (tests/golden/harness_<case>.json) on the engine."""
    with open(GOLDEN / f"harness_{case}.json") as f:
        rec = json.load(f)
    assert rec["exit_code"] == 0
    monkeypatch.setenv("SSD_HF_CACHE", str(tmp_path))
    monkeypatch.setenv("SSD_DATASET_DIR", str(tmp_path / "datasets"))
    _make_hf_cache(str(tmp_path))
    import ssd_b200.paths as P
    importlib.reload(P)
    import ssd_b200.compat as compat
    compat.install()
    fake = {}

    def fake_build_runner(config, tp_size=1, tp_rank=0, device=None, finalize=True):
        config.num_kvcache_blocks = 256
        fake["runner"] = FakeRunner(config.speculate_k)
        fake["config"] = config
        return fake["runner"], types.SimpleNamespace(num_kvcache_blocks=256)

    import ssd_b200.loader as loader
    monkeypatch.setattr(loader, "build_runner", fake_build_runner)

    import ssd.paths  # noqa: F401  (the harness's first import)
    from ssd import LLM, SamplingParams
    from ssd.engine.llm_engine import METRICS
    path = lambda v: v.replace("{HF_CACHE}", str(tmp_path)) if isinstance(v, str) else v
    llm = LLM(path(rec["llm"]["model"]), **{k: path(v) for k, v in rec["llm"]["kwargs"].items()})
    captured = {}
    for run in rec["runs"]:
        b = run["config_max_num_seqs"]
        assert b <= llm.config.max_num_seqs  # the harness's reconfigure_engine contract
        llm.config.max_num_seqs = b
        llm.scheduler.max_num_seqs = run["scheduler_max_num_seqs"]
        for k, v in METRICS.items():  # the harness's reset_metrics
            if isinstance(v, list):
                v.clear()
            else:
                METRICS[k] = 0
        assert {k: (list(v) if isinstance(v, list) else v) for k, v in METRICS.items()} == run["metrics_at_call"]
        prompts = run["prompts"]
        outs, metrics = llm.generate(prompts, [SamplingParams(**sp) for sp in run["sampling_params"]], use_tqdm=False)
        captured.setdefault("runs", []).append((prompts, outs, {k: (list(v) if isinstance(v, list) else v) for k, v in metrics.items()}))
    return captured, fake


def test_reference_bench_py_runs_unmodified_on_the_engine(tmp_path, monkeypatch):
    captured, fake = _run_bench(tmp_path, monkeypatch, "spec")
    cfg = fake["config"]
    assert cfg.speculate and cfg.speculate_k == 6 and cfg.jit_speculate and cfg.kvcache_block_size == 256
    assert cfg.max_num_seqs == 2 and cfg.max_model_len == 8192
    (prompts, outs, metrics), = captured["runs"]
    assert len(outs) == 5
    for p, o in zip(prompts, outs):
        want, cur = [], p[-1]
        for _ in range(60):
            cur = _next(cur)
            want.append(cur)
        assert o["token_ids"] == want, "speculative bookkeeping changed the greedy continuation"
    lens = metrics["accepted_suffix_lens_with_recovery"]
    assert lens and all(1 <= x <= 7 for x in lens)
    assert metrics["decode_total_tokens"] == sum(lens) and metrics["prefill_total_tokens"] == 5 * 40
    r = fake["runner"]
    assert r.max_batch_seen == 2 and r.calls["prefill"] == 2 * 5          # target + draft prefill per sequence
    assert r.calls["spec_step"] <= len(lens) <= 2 * r.calls["spec_step"]  # one suffix per running sequence per step


def test_reference_bench_py_sweep_and_autoregressive(tmp_path, monkeypatch):
    captured, fake = _run_bench(tmp_path, monkeypatch, "sweep_ar")
    assert not fake["config"].speculate
    assert len(captured["runs"]) == 2
    for prompts, outs, metrics in captured["runs"]:
        assert [len(o["token_ids"]) for o in outs] == [20, 20, 20]
        assert metrics["decode_total_tokens"] > 0 and not metrics["accepted_suffix_lens_with_recovery"]
