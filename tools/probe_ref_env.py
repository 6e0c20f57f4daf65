"""GPU probe: do flash_attn 2.8.3 (paged kvcache) and torch.compile (Inductor -> Triton) work here?
Both are prerequisites of the reference GPU arm (bench.py --impl reference-gpu)."""
import time
import torch

t0 = time.time()
from flash_attn import flash_attn_with_kvcache, flash_attn_varlen_func  # noqa: E402
print("flash_attn import ok", time.time() - t0, flush=True)
dev = "cuda"
B, Q, H, KV, hd, bs, nb = 1, 7, 64, 8, 128, 256, 8
q = torch.randn(B, Q, H, hd, device=dev, dtype=torch.bfloat16)
kc = torch.randn(nb, bs, KV, hd, device=dev, dtype=torch.bfloat16)
vc = torch.randn(nb, bs, KV, hd, device=dev, dtype=torch.bfloat16)
bt = torch.arange(nb, device=dev, dtype=torch.int32)[None]
cl = torch.tensor([700], device=dev, dtype=torch.int32)
o = flash_attn_with_kvcache(q, kc, vc, cache_seqlens=cl, block_table=bt, softmax_scale=hd ** -0.5, causal=True)
torch.cuda.synchronize()
# reference: plain torch
k = kc.reshape(-1, KV, hd)[:700].float().repeat_interleave(H // KV, 1)
v = vc.reshape(-1, KV, hd)[:700].float().repeat_interleave(H // KV, 1)
s = torch.einsum("qhd,lhd->hql", q[0].float(), k) * hd ** -0.5
allowed = torch.arange(700, device=dev)[None, :] <= (torch.arange(Q, device=dev)[:, None] + (700 - Q))
s = s.masked_fill(~allowed[None], float("-inf"))
ref = torch.einsum("hql,lhd->qhd", torch.softmax(s, -1), v)
print("fa2 paged kvcache max err", (o[0].float() - ref).abs().max().item(), flush=True)

@torch.compile
def f(x, w):
    xf = x.float()
    return (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5)).to(x.dtype) * w

t0 = time.time()
x = torch.randn(7, 8192, device=dev, dtype=torch.bfloat16)
w = torch.ones(8192, device=dev, dtype=torch.bfloat16)
y = f(x, w)
torch.cuda.synchronize()
print("torch.compile ok", time.time() - t0, y.shape, flush=True)
g = torch.cuda.CUDAGraph()
with torch.cuda.graph(g):
    o2 = flash_attn_with_kvcache(q, kc, vc, cache_seqlens=cl, block_table=bt, softmax_scale=hd ** -0.5, causal=True)
g.replay()
torch.cuda.synchronize()
print("fa2 graph capture ok", (o2 - o).abs().max().item(), flush=True)
