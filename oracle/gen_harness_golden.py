"""Record how the reference's own acceptance harness (bench/bench.py of a reference checkout named by SSD_REFERENCE_DIR,
run unmodified) drives the engine, as tests/golden/harness_<case>.json.

The harness runs on top of ssd_b200 through the `ssd` compat shim with the device runner replaced by the CPU test
double of tests/test_reference_harness_cpu.py.  Recorded at the engine boundary, in call order: the model path and
keyword arguments of `LLM(...)`, and for every `generate()` call the prompts, the SamplingParams fields, the
`config.max_num_seqs` / `scheduler.max_num_seqs` the harness set and the METRICS it left at the call.
tests/test_reference_harness_cpu.py replays these calls, so the test needs no reference checkout.

    SSD_REFERENCE_DIR=<checkout> python oracle/gen_harness_golden.py
"""
from __future__ import annotations

import copy
import importlib
import json
import os
import re
import runpy
import sys
import tempfile
import types
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))
OUT = REPO / "tests" / "golden"

CASES = {
    "spec": ["--size", "8", "--spec", "--k", "6", "--random", "--numseqs", "5", "--input_len", "40", "--output_len", "60",
             "--b", "2"],
    "sweep_ar": ["--size", "8", "--random", "--numseqs", "3", "--input_len", "16", "--output_len", "20", "--b", "2",
                 "--sweep", json.dumps([{"b": 2, "temp": 0.5}, {"b": 1}])],
}
SP_FIELDS = ("temperature", "draft_temperature", "ignore_eos", "max_new_tokens")


def record(ref: str, argv: list[str]) -> dict:
    from tests.test_reference_harness_cpu import FakeRunner, _make_hf_cache

    root = tempfile.mkdtemp(prefix="ssd_harness_")
    os.environ["SSD_HF_CACHE"] = root
    os.environ["SSD_DATASET_DIR"] = os.path.join(root, "datasets")
    _make_hf_cache(root)
    import ssd_b200.paths as P
    importlib.reload(P)
    import ssd_b200.compat as compat
    compat.install()
    wandb = types.ModuleType("wandb")
    wandb.init = wandb.log = wandb.finish = lambda *a, **k: None
    sys.modules["wandb"] = wandb

    # model directories relative to the HF cache the harness resolved them in (`{HF_CACHE}/models--...`)
    rel = lambda v: re.sub(r"^.*?/(?=models--)", "{HF_CACHE}/", v) if isinstance(v, str) else v
    rec = {"argv": argv, "llm": None, "runs": []}

    import ssd_b200.loader as loader
    import ssd_b200.engine.llm_engine as eng

    def fake_build_runner(config, tp_size=1, tp_rank=0, device=None, finalize=True):
        config.num_kvcache_blocks = 256
        return FakeRunner(config.speculate_k), types.SimpleNamespace(num_kvcache_blocks=256)

    orig_init, orig_generate, orig_build = eng.LLMEngine.__init__, eng.LLMEngine.generate, loader.build_runner

    def spy_init(self, model, **kwargs):
        rec["llm"] = {"model": rel(model), "kwargs": {k: rel(v) for k, v in kwargs.items()}}
        orig_init(self, model, **kwargs)

    def spy_generate(self, prompts, sampling_params, use_tqdm=True, stream_callback=None):
        rec["runs"].append({"prompts": [list(p) for p in prompts],
                            "sampling_params": [{f: getattr(sp, f) for f in SP_FIELDS} for sp in sampling_params],
                            "config_max_num_seqs": self.config.max_num_seqs,
                            "scheduler_max_num_seqs": self.scheduler.max_num_seqs,
                            "metrics_at_call": copy.deepcopy(dict(eng.METRICS))})
        return orig_generate(self, prompts, sampling_params, use_tqdm=False, stream_callback=stream_callback)

    eng.LLMEngine.__init__, eng.LLMEngine.generate, loader.build_runner = spy_init, spy_generate, fake_build_runner
    sys.argv = ["bench.py"] + argv
    sys.path.insert(0, os.path.join(ref, "bench"))
    try:
        runpy.run_path(os.path.join(ref, "bench", "bench.py"), run_name="__main__")
        code = 0
    except SystemExit as ex:
        code = ex.code
    finally:
        eng.LLMEngine.__init__, eng.LLMEngine.generate, loader.build_runner = orig_init, orig_generate, orig_build
        sys.path.remove(os.path.join(ref, "bench"))
    rec["exit_code"] = code
    return rec


def main():
    ref = os.environ["SSD_REFERENCE_DIR"]
    for name, argv in CASES.items():
        rec = record(ref, argv)
        assert rec["exit_code"] == 0, rec["exit_code"]
        (OUT / f"harness_{name}.json").write_text(json.dumps(rec, indent=1) + "\n")
        print(f"harness_{name}.json: {len(rec['runs'])} generate call(s)")


if __name__ == "__main__":
    main()
