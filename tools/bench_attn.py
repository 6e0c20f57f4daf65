"""Stand-alone timing of ssdk_paged_attn (attention + split-KV combine) at the shapes of the speculative step, next to
flash_attn 2.8.3's `flash_attn_with_kvcache` (the library kernel the reference GPU arm runs behind its
sgl_kernel stub) on the SAME paged cache, for context 135 ... 8192.  Launches are captured in a CUDA graph (100 per replay)
so the number is the kernel time without host launch gaps; warm-L2 figure (as in the step, where the new tokens' K/V were
just written).  Also prints the achieved KV bytes/s of ours: ctx * KV * hd * 2 (K and V) * 2 B per launch."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ssd_b200 import ops  # noqa: E402

dev = torch.device("cuda")
torch.manual_seed(0)
SHAPES = [  # name, H, KV, hd, q_len
    ("70b verify tp1", 64, 8, 128, 7), ("70b verify tp8", 8, 1, 128, 7), ("8b verify", 32, 8, 128, 7),
    ("qwen32b verify tp4", 16, 2, 128, 7), ("1b decode", 32, 8, 64, 1), ("0.6b decode", 16, 8, 128, 1),
]
bs, nblk = 256, 32
CTXS = (135, 640, 2048, 4096, 8192)


def graph_time(fn):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        with torch.cuda.graph(g, stream=st):
            for _ in range(100):
                fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000 / 500  # us per call


def time_shape(H, KV, hd, Q):
    try:
        from flash_attn import flash_attn_with_kvcache
    except Exception:
        flash_attn_with_kvcache = None
    kc = torch.randn(nblk, bs, KV, hd, device=dev).bfloat16()
    vc = torch.randn(nblk, bs, KV, hd, device=dev).bfloat16()
    bt = torch.arange(nblk, dtype=torch.int32, device=dev)[None]
    q = torch.randn(Q, H, hd, device=dev).bfloat16()
    row = []
    for ctx in CTXS:
        cl = torch.tensor([ctx], dtype=torch.int32, device=dev)
        ours = graph_time(lambda: ops.paged_attention(q, kc, vc, bt, cl, Q, hd ** -0.5))
        fa = float("nan")
        if flash_attn_with_kvcache is not None:
            q4 = q.view(1, Q, H, hd)
            fa = graph_time(lambda: flash_attn_with_kvcache(q4, kc, vc, cache_seqlens=cl, block_table=bt, softmax_scale=hd ** -0.5,
                                                            causal=True))
            o1 = ops.paged_attention(q, kc, vc, bt, cl, Q, hd ** -0.5).float().view(Q, H, hd)
            o2 = flash_attn_with_kvcache(q4, kc, vc, cache_seqlens=cl, block_table=bt, softmax_scale=hd ** -0.5, causal=True)
            assert (o1 - o2.view(Q, H, hd).float()).abs().max() < 3e-2
        gbs = ctx * KV * hd * 2 * 2 / (ours * 1e-6) / 1e9
        row.append(f"ctx {ctx}: {ours:6.2f} us ({gbs:5.0f} GB/s) fa2 {fa:6.2f} us x{fa / ours:4.2f}")
    return "  ".join(row)


for name, H, KV, hd, Q in SHAPES:
    print(f"{name:20s} " + time_shape(H, KV, hd, Q), flush=True)
