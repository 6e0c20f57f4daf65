"""ctypes binding of libssdk.so — the only door between the Python host side and the CUDA hot path.

Every symbol declared in include/ssdk.h is bound here with explicit argtypes; the library is
built in-tree by ssd_b200.build.  There is NO fallback: if the shared object is missing or a
call fails, a RuntimeError is raised (a CPU/eager fallback would void every parity claim).
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_LIB_PATH = Path(__file__).resolve().parent / "_lib" / "libssdk.so"

c_i32p = C.POINTER(C.c_int32)
c_i64p = C.POINTER(C.c_int64)
c_f32p = C.POINTER(C.c_float)
VP = C.c_void_p


class ModelCfg(C.Structure):
    """struct ssdk_model_cfg (include/ssdk.h)."""

    _fields_ = [
        ("hidden", C.c_int32), ("layers", C.c_int32), ("heads", C.c_int32), ("kv_heads", C.c_int32),
        ("head_dim", C.c_int32), ("ffn", C.c_int32), ("vocab", C.c_int32), ("qk_norm", C.c_int32),
        ("rms_eps", C.c_float), ("max_pos", C.c_int32), ("tp_size", C.c_int32), ("tp_rank", C.c_int32),
    ]


class RuntimeCfg(C.Structure):
    """struct ssdk_runtime_cfg (include/ssdk.h)."""

    _fields_ = [
        ("spec_k", C.c_int32), ("max_batch", C.c_int32), ("block_size", C.c_int32),
        ("max_blocks_per_seq", C.c_int32), ("use_graph", C.c_int32), ("use_pdl", C.c_int32),
        ("jit_speculate", C.c_int32), ("reserved", C.c_int32),
    ]


# weight kinds (enum in include/ssdk.h)
W_EMBED, W_LM_HEAD, W_FINAL_NORM, W_INPUT_NORM, W_QKV, W_Q_NORM, W_K_NORM, W_O, W_POST_NORM, W_GATE_UP, W_DOWN, W_ROPE_TABLE = range(12)
TARGET, DRAFT = 0, 1

# name -> (restype, argtypes); must list every symbol of include/ssdk.h
SIGNATURES: dict[str, tuple] = {
    "ssdk_abi_version": (C.c_int, []),
    "ssdk_last_error": (C.c_char_p, []),
    "ssdk_create": (C.c_int, [C.POINTER(ModelCfg), C.POINTER(ModelCfg), C.POINTER(RuntimeCfg), C.POINTER(VP)]),
    "ssdk_destroy": (C.c_int, [VP]),
    "ssdk_bind_weight": (C.c_int, [VP, C.c_int, C.c_int, C.c_int, VP, C.c_int64, C.c_int64]),
    "ssdk_bind_kv_cache": (C.c_int, [VP, C.c_int, VP, C.c_int64]),
    "ssdk_workspace_bytes": (C.c_int64, [VP]),
    "ssdk_bind_workspace": (C.c_int, [VP, VP, C.c_int64]),
    "ssdk_set_nccl_comm": (C.c_int, [VP, VP]),
    "ssdk_symm_bytes": (C.c_int64, [VP]),
    "ssdk_bind_symm": (C.c_int, [VP, C.POINTER(VP), C.c_int]),
    "ssdk_finalize": (C.c_int, [VP, VP]),
    "ssdk_spec_step": (C.c_int, [VP, C.c_int, c_i32p, c_i64p, c_i32p, c_i32p, c_f32p, c_f32p, C.c_uint64, C.c_uint64,
                                 c_i64p, c_i32p, c_i64p, VP]),
    "ssdk_spec_step_stage": (C.c_int, [VP, C.c_int, c_i32p, c_i64p, c_i32p, c_i32p, c_f32p, c_f32p, C.c_uint64,
                                       C.c_uint64, VP]),
    "ssdk_spec_step_resident": (C.c_int, [VP, C.c_int, VP]),
    "ssdk_spec_step_fetch": (C.c_int, [VP, C.c_int, c_i64p, c_i32p, c_i64p, VP]),
    "ssdk_spec_step_log": (C.c_int, [VP, C.c_int, c_i64p, C.c_int, VP]),
    "ssdk_forward_tokens": (C.c_int, [VP, C.c_int, C.c_int, C.c_int, c_i64p, c_i32p, c_i32p, C.c_int, c_f32p,
                                      C.c_uint64, C.c_uint64, c_i64p, VP]),
    "ssdk_logits_p": (VP, [VP]),
    "ssdk_logits_q": (VP, [VP]),
    "ssdk_logits_last": (VP, [VP]),
    "ssdk_debug_trace": (C.c_int, [VP, C.c_int]),
    "ssdk_launch_count": (C.c_int64, [VP]),
    "ssdk_gemm_small_m": (C.c_int, [VP, VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, VP]),
    "ssdk_gemm_gate_up_silu": (C.c_int, [VP, VP, VP, C.c_int, C.c_int, C.c_int, VP]),
    "ssdk_rmsnorm": (C.c_int, [VP, VP, VP, C.c_float, VP, VP, C.c_int, C.c_int, VP]),
    "ssdk_rope_store_kv": (C.c_int, [VP, VP, VP, VP, VP, VP, C.c_float, VP, VP, VP, C.c_int, C.c_int, C.c_int,
                                     C.c_int, VP]),
    "ssdk_silu_mul": (C.c_int, [VP, VP, C.c_int, C.c_int, VP]),
    "ssdk_paged_attn_scratch_bytes": (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "ssdk_paged_attn": (C.c_int, [VP, VP, VP, VP, VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                  C.c_int, C.c_float, VP]),
    "ssdk_paged_attn_plan": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_i32p]),
    "ssdk_sample": (C.c_int, [VP, C.c_int64, VP, C.c_int, C.c_int, C.c_uint64, C.c_uint64, VP, VP]),
    "ssdk_verify_scratch_bytes": (C.c_int64, [C.c_int, C.c_int]),
    "ssdk_verify": (C.c_int, [VP, VP, VP, VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_uint64,
                              VP, VP, VP, VP]),
}

_lib = None


def lib_path() -> Path:
    return _LIB_PATH


def load(build_if_missing: bool = True) -> C.CDLL:
    """Load libssdk.so (building it with nvcc first if it is stale/missing and nvcc exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if build_if_missing:
        from . import build as _build

        try:
            if _build.is_stale():
                _build.build(verbose=False)
        except Exception as exc:  # no nvcc on this box: the prebuilt .so must be there
            if not _LIB_PATH.exists():
                raise RuntimeError(f"libssdk.so is missing and could not be built: {exc}") from exc
    if not _LIB_PATH.exists():
        raise RuntimeError(f"{_LIB_PATH} not found — run `python -m ssd_b200.build`; there is no CPU fallback")
    path = os.environ.get("SSDK_LIB") or str(_LIB_PATH)  # SSDK_LIB: an alternative build of the same library (trace variant)
    lib = C.CDLL(path, mode=os.RTLD_GLOBAL if hasattr(os, "RTLD_GLOBAL") else C.DEFAULT_MODE)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.ssdk_abi_version() != 1:
        raise RuntimeError("libssdk.so ABI version mismatch")
    _lib = lib
    return lib


def last_error() -> str:
    return load().ssdk_last_error().decode("utf-8", "replace")


def check(rc: int, what: str = "ssdk call") -> None:
    """Reference error convention is Python exceptions (SURVEY §8b): map rc<0 to RuntimeError."""
    if rc != 0:
        raise RuntimeError(f"{what} failed: {last_error()}")
