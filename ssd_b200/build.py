"""Build libssdk.so (the C-ABI hot path) in-tree with nvcc for sm_90a (H100).

    python -m ssd_b200.build            # build if stale
    python -m ssd_b200.build --force

The library links only against libcudart (static) and NCCL; it has no torch or Python
dependency.  The built .so lives next to the sources (ssd_b200/_lib/libssdk.so) so it
travels with the repo snapshot to the GPU box.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
OUT_DIR = ROOT / "_lib"
LIB = OUT_DIR / "libssdk.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xptxas=-v",
    "-Xcompiler", "-fPIC,-O2,-Wall,-Wno-unused-function",
    "--expt-relaxed-constexpr",
    "-shared",
]


def _nccl_paths() -> tuple[list[str], list[str]]:
    """Prefer the NCCL that torch bundles (2.28), fall back to the system one."""
    inc, lib = [], []
    try:
        import nvidia.nccl as _n  # type: ignore

        base = Path(_n.__path__[0])
        if (base / "include" / "nccl.h").exists():
            inc = ["-I", str(base / "include")]
            so = sorted((base / "lib").glob("libnccl.so*"))
            if so:
                lib = ["-L", str(base / "lib"), f"-l:{so[0].name}", f"-Xlinker=-rpath={base / 'lib'}"]
    except Exception:
        pass
    if not lib:
        lib = ["-lnccl"]
    return inc, lib


def sources() -> list[Path]:
    return [CSRC / "engine.cu"]


def headers() -> list[Path]:
    return sorted(CSRC.glob("*.cuh")) + [ROOT.parent / "include" / "ssdk.h"]


def is_stale() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    return any(p.stat().st_mtime > t for p in sources() + headers())


def build_trace_variant() -> Path:
    """libssdk_trace.so: same sources with -DSSDK_TRACE_FINE (phase marks inside the kernels for tools/trace_step.py).
    Loaded instead of libssdk.so when SSDK_LIB points at it; never used by the product path."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    inc, lib = _nccl_paths()
    out = OUT_DIR / "libssdk_trace.so"
    cmd = [nvcc, *NVCC_FLAGS, "-DSSDK_TRACE_FINE", *inc, "-o", str(out), *map(str, sources()), *lib, "-lcudart_static", "-ldl",
           "-lrt", "-lpthread"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed for the trace variant")
    return out


def build(force: bool = False, verbose: bool = True) -> Path:
    if not force and not is_stale():
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: libssdk.so cannot be built on this machine")
    OUT_DIR.mkdir(exist_ok=True)
    inc, lib = _nccl_paths()
    cmd = [nvcc, *NVCC_FLAGS, *inc, "-o", str(LIB), *map(str, sources()), *lib, "-lcudart_static", "-ldl", "-lrt", "-lpthread"]
    if verbose:
        print("[ssd_b200.build]", " ".join(cmd), flush=True)
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = OUT_DIR / "build.log"
    log.write_text(res.stdout + "\n" + res.stderr)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError(f"nvcc failed ({res.returncode}); see {log}")
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv)
    print(path)
    if "--trace-variant" in sys.argv:
        print(build_trace_variant())
