"""ssd_b200 — H100-native sync speculative-decoding hot path behind the `ssd` API surface.

    from ssd_b200 import LLM, SamplingParams          # same call signatures as `from ssd import ...`
    import ssd_b200.compat; ssd_b200.compat.install()  # makes `import ssd` resolve to this package

Heavy imports (torch, the CUDA library) happen lazily so that `import ssd_b200` works on a CPU box."""
from .sampling_params import SamplingParams

__all__ = ["LLM", "SamplingParams", "Config", "LLMEngine", "METRICS"]


def __getattr__(name):
    if name == "LLM":
        from .llm import LLM
        return LLM
    if name in ("LLMEngine", "METRICS"):
        from .engine import llm_engine
        return getattr(llm_engine, name)
    if name == "Config":
        from .config import Config
        return Config
    raise AttributeError(name)
