"""Micro-benchmark of the weight-streaming GEMM at the shapes of the BASELINE models: achieved HBM GB/s
(weight bytes / CUDA-event time, L2 flushed between launches) next to torch (cuBLAS) on the same shapes.
    python tools/bench_gemm.py [OUT.json]"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ssd_b200 import ops

SHAPES = {  # name: (N, K)
    "1B.qkv": (3072, 2048), "1B.o": (2048, 2048), "1B.gate_up": (16384, 2048), "1B.down": (2048, 8192),
    "1B.lm_head": (128256, 2048),
    "8B.qkv": (6144, 4096), "8B.o": (4096, 4096), "8B.gate_up": (28672, 4096), "8B.down": (4096, 14336),
    "70B.qkv": (10240, 8192), "70B.o": (8192, 8192), "70B.gate_up": (57344, 8192), "70B.down": (8192, 28672),
}


def main():
    dev = torch.device("cuda:0")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    out = []
    for name, (N, K) in SHAPES.items():
        w = (torch.randn(N, K, device=dev) * 0.02).to(torch.bfloat16)
        for M in (1, 7):
            x = torch.randn(M, K, device=dev).to(torch.bfloat16)
            res = {}
            for impl in ("ssdk", "torch"):
                fn = (lambda: ops.linear(x, w)) if impl == "ssdk" else (lambda: torch.nn.functional.linear(x, w))
                if impl == "ssdk" and name.endswith("gate_up"):
                    fn = lambda: ops.gate_up_silu(x, w)
                for _ in range(3):
                    fn()
                ts = []
                for _ in range(10):
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    fn()
                    e1.record()
                    torch.cuda.synchronize()
                    ts.append(e0.elapsed_time(e1))
                ts.sort()
                ms = ts[len(ts) // 2]
                res[impl] = {"ms": ms, "GBps": N * K * 2 / ms / 1e6}
            rec = {"shape": name, "M": M, "N": N, "K": K, **{f"{k}_{kk}": vv for k, v in res.items() for kk, vv in v.items()}}
            print(json.dumps(rec), flush=True)
            out.append(rec)
        del w
    if len(sys.argv) > 1:  # optional file for the records printed above
        with open(sys.argv[1], "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    sys.exit(main())
