"""Install the unmodified reference package (tanishqkumar/ssd) into oracle/_ref for bench.py's reference GPU arm
(baseline/ref_gpu.py).

The source is the reference checkout: SSD_REFERENCE_DIR when set, else the first of DEFAULT_SOURCES that exists (a
checkout next to this repository, then the location the reference is mounted at in the project's build environment).
Without one nothing is installed and the reference arm reports itself unavailable.  --no-deps: the reference pins torch 2.8 / sgl-kernel / flashinfer, which the
project's environment does not provide; --no-index keeps the install offline (SSD_WHEELHOUSE may name a local wheel
directory for its build requirements)."""
from __future__ import annotations

import os
import shutil
import stat
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(ROOT, "oracle", "_ref")
DEFAULT_SOURCES = (os.path.join(os.path.dirname(ROOT), "reference"), "/root/reference")


def reference_source() -> str | None:
    env = os.environ.get("SSD_REFERENCE_DIR")
    for d in ([env] if env else list(DEFAULT_SOURCES)):
        if os.path.isfile(os.path.join(d, "ssd", "__init__.py")):
            return d
    return None


def install_reference() -> None:
    if os.path.isdir(os.path.join(DST, "ssd")):
        print("[build] oracle/_ref present")
        return
    src_dir = reference_source()
    if src_dir is None:
        print("[build] no reference checkout (SSD_REFERENCE_DIR): the reference GPU arm of bench.py will report 'unavailable'")
        return
    tmp = tempfile.mkdtemp(prefix="ssd_ref_src_")
    try:
        src = os.path.join(tmp, "ref")  # the build writes egg-info into the source tree
        shutil.copytree(src_dir, src)
        for d, _, files in os.walk(src):  # the checkout may be read-only, and copytree keeps its modes
            for path in [d] + [os.path.join(d, f) for f in files]:
                if not os.path.islink(path):
                    os.chmod(path, os.stat(path).st_mode | stat.S_IWUSR)
        cmd = [sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps", "--target", DST, src]
        if os.environ.get("SSD_WHEELHOUSE"):
            cmd[4:4] = ["--find-links", os.environ["SSD_WHEELHOUSE"]]
        res = subprocess.run(cmd, capture_output=True, text=True)
        print(f"[build] pip install reference ({src_dir}) -> oracle/_ref:", "ok" if res.returncode == 0 else res.stderr[-400:])
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
