"""Generate tests/golden/*.npz by importing and running the UNMODIFIED reference (a checkout
named by SSD_REFERENCE_DIR).

Runs only in the build container (the reference does not travel to the GPU box).  Usage:

    CXX=/usr/bin/g++ python oracle/gen_golden.py            # compiled (Inductor) numerics + everything else
    TORCHDYNAMO_DISABLE=1 python oracle/gen_golden.py eager  # eager numerics of the @torch.compile regions

Three stubs are needed to run the reference on CPU (SURVEY §8c): the absent `sgl_kernel.flash_attn`
wheel (two functions, replaced by a pure-torch paged attention with FlashAttention's documented
semantics) and the Triton `store_kvcache` (replaced by an index scatter).  Everything else —
ssd.utils.verify.verify, ssd.layers.sampler.Sampler, ssd.layers.{layernorm,rotary_embedding,activation},
ssd.models.{llama3,qwen3} with their weight_loader packing rules, ssd.utils.context — is the
reference's own code.
"""
from __future__ import annotations

import os
import sys
import types
from pathlib import Path

import numpy as np
import torch

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))
OUT = REPO / "tests" / "golden"
REF = os.environ["SSD_REFERENCE_DIR"]


# ----------------------------------------------------------------------------- stubs
def _paged_attn(q, k_cache, v_cache, cache_seqlens, page_table, softmax_scale, q_len):
    """q [B*q_len, H, hd]; causal aligned to the end of cache_seqlens; GQA; fp32 softmax."""
    Mq, H, hd = q.shape
    B = Mq // q_len
    bs, KV = k_cache.shape[1], k_cache.shape[2]
    out = torch.empty_like(q)
    for b in range(B):
        L = int(cache_seqlens[b])
        nb = (L + bs - 1) // bs
        pg = page_table[b, :nb].long()
        k = k_cache[pg].reshape(nb * bs, KV, hd)[:L].float().repeat_interleave(H // KV, 1)
        v = v_cache[pg].reshape(nb * bs, KV, hd)[:L].float().repeat_interleave(H // KV, 1)
        qq = q[b * q_len:(b + 1) * q_len].float()
        s = torch.einsum("qhd,lhd->hql", qq, k) * softmax_scale
        allowed = torch.arange(L)[None, :] <= (torch.arange(q_len)[:, None] + (L - q_len))
        s = s.masked_fill(~allowed[None], float("-inf"))
        out[b * q_len:(b + 1) * q_len] = torch.einsum("hql,lhd->qhd", torch.softmax(s, -1), v).to(q.dtype)
    return out


def flash_attn_with_kvcache(q, k_cache, v_cache, cache_seqlens=None, page_table=None, softmax_scale=None, causal=True,
                            cu_seqlens_q=None, max_seqlen_q=None, **_):
    if cu_seqlens_q is not None:  # verify: q [N, H, hd]
        return _paged_attn(q, k_cache, v_cache, cache_seqlens, page_table, softmax_scale, int(max_seqlen_q))
    B = q.shape[0]  # decode: q [B, 1, H, hd]
    o = _paged_attn(q.reshape(B, q.shape[2], q.shape[3]), k_cache, v_cache, cache_seqlens, page_table, softmax_scale, 1)
    return o.reshape(q.shape)


def flash_attn_varlen_func(q, k, v, max_seqlen_q=None, cu_seqlens_q=None, max_seqlen_k=None, cu_seqlens_k=None,
                           softmax_scale=None, causal=True, **_):
    H, KV = q.shape[1], k.shape[1]
    out = torch.empty_like(q)
    for b in range(cu_seqlens_q.numel() - 1):
        qs, qe = int(cu_seqlens_q[b]), int(cu_seqlens_q[b + 1])
        ks, ke = int(cu_seqlens_k[b]), int(cu_seqlens_k[b + 1])
        qq = q[qs:qe].float()
        kk = k[ks:ke].float().repeat_interleave(H // KV, 1)
        vv = v[ks:ke].float().repeat_interleave(H // KV, 1)
        Lq, Lk = qe - qs, ke - ks
        s = torch.einsum("qhd,lhd->hql", qq, kk) * softmax_scale
        allowed = torch.arange(Lk)[None, :] <= (torch.arange(Lq)[:, None] + (Lk - Lq))
        s = s.masked_fill(~allowed[None], float("-inf"))
        out[qs:qe] = torch.einsum("hql,lhd->qhd", torch.softmax(s, -1), vv).to(q.dtype)
    return out


def _store_kvcache(key, value, k_cache, v_cache, slot_mapping):
    KV, hd = key.shape[1], key.shape[2]
    keep = slot_mapping >= 0
    idx = slot_mapping[keep].long()
    k_cache.view(-1, KV, hd)[idx] = key[keep]
    v_cache.view(-1, KV, hd)[idx] = value[keep]


def import_reference():
    os.environ.setdefault("SSD_HF_CACHE", "/tmp/ssd_hf")
    os.environ.setdefault("SSD_DATASET_DIR", "/tmp/ssd_data")
    sys.path.insert(0, REF)
    m = types.ModuleType("sgl_kernel")
    fa = types.ModuleType("sgl_kernel.flash_attn")
    fa.flash_attn_varlen_func = flash_attn_varlen_func
    fa.flash_attn_with_kvcache = flash_attn_with_kvcache
    m.flash_attn = fa
    sys.modules["sgl_kernel"] = m
    sys.modules["sgl_kernel.flash_attn"] = fa
    import ssd  # noqa: F401
    import ssd.layers.attention as att

    att.store_kvcache = _store_kvcache
    return ssd


# ----------------------------------------------------------------------------- goldens
def gen_verify_t0(ssd):
    from ssd.utils.verify import verify

    g = torch.Generator().manual_seed(11)
    cases = {}
    for ci, (B, K, V) in enumerate([(1, 6, 1000), (3, 6, 512), (2, 4, 2048), (1, 7, 4096)]):
        lp = (torch.randn(B, K + 1, V, generator=g) * 3).to(torch.bfloat16)
        lq = (torch.randn(B, K, V, generator=g) * 3).to(torch.bfloat16)
        preds = lp.argmax(-1)
        spec = torch.randint(0, V, (B, K + 1), generator=g)
        for b in range(B):  # accept a random prefix of the target's greedy choices
            n = int(torch.randint(0, K + 1, (1,), generator=g))
            spec[b, 1:1 + n] = preds[b, :n]
        # force exact bf16 ties in one row: lowest index must win
        lp[0, 0, 7] = lp[0, 0].max()
        lp[0, 0, 3] = lp[0, 0].max()
        suf, rec = verify(lp, lq, spec, torch.zeros(B), torch.zeros(B))
        cases[f"c{ci}_lp"] = lp.view(torch.int16).numpy()
        cases[f"c{ci}_lq"] = lq.view(torch.int16).numpy()
        cases[f"c{ci}_spec"] = spec.numpy()
        cases[f"c{ci}_nacc"] = np.array([len(s) - 1 for s in suf], dtype=np.int32)
        cases[f"c{ci}_rec"] = np.array(rec, dtype=np.int64)
        cases[f"c{ci}_suffix_flat"] = np.array([t for s in suf for t in s], dtype=np.int64)
    cases["n_cases"] = np.array(4)
    np.savez_compressed(OUT / "verify_t0.npz", **cases)
    print("verify_t0 ok")


def gen_verify_ratio(ssd):
    """temp>0: pin the deterministic parts — acceptance probabilities, accept counts for injected uniforms,
    and the exact distributions handed to torch.multinomial (verify.py:155-159)."""
    import ssd.utils.verify as vmod

    g = torch.Generator().manual_seed(12)
    cases = {}
    real_rand_like, real_multinomial = torch.rand_like, torch.multinomial
    ci = 0
    for (B, K, V, tt, tq, jit) in [(2, 6, 512, 0.7, 0.7, True), (2, 5, 640, 1.0, 0.5, True), (2, 6, 512, 0.0, 0.8, True),
                                   (3, 4, 512, 0.9, 0.0, True), (2, 6, 512, 0.7, 0.7, False)]:
        lp = (torch.randn(B, K + 1, V, generator=g) * 2).to(torch.bfloat16)
        lq = (lp[:, :K].float() + torch.randn(B, K, V, generator=g)).to(torch.bfloat16)  # correlated draft
        spec = torch.randint(0, V, (B, K + 1), generator=g)
        pq = torch.softmax(lq.float() / max(tq, 1e-8), -1) if tq > 0 else None
        for b in range(B):
            for j in range(K):
                spec[b, j + 1] = int(torch.multinomial(pq[b, j], 1, generator=g)) if pq is not None else int(lq[b, j].argmax())
        uni = torch.rand(B, K, generator=g)
        captured = []
        torch.rand_like = lambda t, **kw: uni.to(t.dtype)
        def fake_multinomial(p, n, **kw):
            captured.append(p.clone())
            return p.argmax(dim=-1, keepdim=True)
        torch.multinomial = fake_multinomial
        try:
            temps_t, temps_q = torch.full((B,), tt), torch.full((B,), tq)
            hits = torch.tensor([1, 0, 1][:B]) if not jit else None
            suf, rec = vmod.verify(lp, lq, spec, temps_t, temps_q, cache_hits=hits, jit_speculate=jit)
        finally:
            torch.rand_like, torch.multinomial = real_rand_like, real_multinomial
        cases[f"c{ci}_lp"] = lp.view(torch.int16).numpy()
        cases[f"c{ci}_lq"] = lq.view(torch.int16).numpy()
        cases[f"c{ci}_spec"] = spec.numpy()
        cases[f"c{ci}_uni"] = uni.numpy()
        cases[f"c{ci}_cfg"] = np.array([tt, tq, float(jit)], dtype=np.float32)
        if hits is not None:
            cases[f"c{ci}_hits"] = hits.numpy().astype(np.int32)
        cases[f"c{ci}_nacc"] = np.array([len(s) - 1 for s in suf], dtype=np.int32)
        cases[f"c{ci}_rec_argmax"] = np.array(rec, dtype=np.int64)  # recovery when multinomial := argmax
        # captured: [adj_norm, fallbackDist] when any ratio row, else [fallbackDist]; may be empty when no temp_t>0
        for k, c in enumerate(captured):
            cases[f"c{ci}_dist{k}"] = c.numpy()
        cases[f"c{ci}_ndist"] = np.array(len(captured))
        ci += 1
    cases["n_cases"] = np.array(ci)
    np.savez_compressed(OUT / "verify_ratio.npz", **cases)
    print("verify_ratio ok")


def gen_verify_mixed(ssd):
    """Per-row temperatures (greedy and sampled rows in one batch), cache-hit gating without jit, K at both ends of the
    supported range: pins the row-selection logic of verify.py:57-62,127,146,167."""
    import ssd.utils.verify as vmod

    g = torch.Generator().manual_seed(15)
    cases = {}
    real_rand_like, real_multinomial = torch.rand_like, torch.multinomial
    cfgs = [
        (4, 6, 384, [0.0, 0.7, 1.0, 0.0], [0.0, 0.7, 0.5, 0.9], True, None),
        (4, 7, 256, [0.6, 0.6, 0.0, 1.2], [0.6, 0.0, 0.0, 1.2], False, [1, 0, 1, 1]),
        (3, 1, 512, [0.8, 0.0, 0.3], [0.8, 0.4, 0.3], True, None),
        (2, 3, 320, [0.0, 0.0], [0.0, 0.0], False, [0, 1]),
    ]
    for ci, (B, K, V, tts, tqs, jit, hits_l) in enumerate(cfgs):
        lp = (torch.randn(B, K + 1, V, generator=g) * 2).to(torch.bfloat16)
        lq = (lp[:, :K].float() + 0.7 * torch.randn(B, K, V, generator=g)).to(torch.bfloat16)
        spec = torch.randint(0, V, (B, K + 1), generator=g)
        for b in range(B):
            for j in range(K):
                if tqs[b] > 0:
                    spec[b, j + 1] = int(real_multinomial(torch.softmax(lq[b, j].float() / tqs[b], -1), 1, generator=g))
                else:
                    spec[b, j + 1] = int(lq[b, j].argmax())
        uni = torch.rand(B, K, generator=g)
        captured = []
        torch.rand_like = lambda t, **kw: uni.to(t.dtype)
        def fake_multinomial(p, n, **kw):
            captured.append(p.clone())
            return p.argmax(dim=-1, keepdim=True)
        torch.multinomial = fake_multinomial
        try:
            hits = torch.tensor(hits_l) if hits_l is not None else None
            suf, rec = vmod.verify(lp, lq, spec, torch.tensor(tts), torch.tensor(tqs), cache_hits=hits, jit_speculate=jit)
        finally:
            torch.rand_like, torch.multinomial = real_rand_like, real_multinomial
        cases[f"c{ci}_lp"] = lp.view(torch.int16).numpy()
        cases[f"c{ci}_lq"] = lq.view(torch.int16).numpy()
        cases[f"c{ci}_spec"] = spec.numpy()
        cases[f"c{ci}_uni"] = uni.numpy()
        cases[f"c{ci}_tt"] = np.array(tts, dtype=np.float32)
        cases[f"c{ci}_tq"] = np.array(tqs, dtype=np.float32)
        cases[f"c{ci}_jit"] = np.array(int(jit))
        if hits is not None:
            cases[f"c{ci}_hits"] = hits.numpy().astype(np.int32)
        cases[f"c{ci}_nacc"] = np.array([len(s) - 1 for s in suf], dtype=np.int32)
        cases[f"c{ci}_rec_argmax"] = np.array(rec, dtype=np.int64)
        cases[f"c{ci}_suffix_flat"] = np.array([t for s in suf for t in s], dtype=np.int64)
    cases["n_cases"] = np.array(len(cfgs))
    np.savez_compressed(OUT / "verify_mixed.npz", **cases)
    print("verify_mixed ok")


def gen_sampler(ssd):
    from ssd.layers.sampler import Sampler

    g = torch.Generator().manual_seed(13)
    logits = (torch.randn(4, 3000, generator=g) * 3).to(torch.bfloat16)
    logits[1, 17] = logits[1].max()
    logits[1, 5] = logits[1].max()
    toks = Sampler()(logits, torch.zeros(4))
    np.savez_compressed(OUT / "sampler_t0.npz", logits=logits.view(torch.int16).numpy(), tokens=toks.numpy())
    print("sampler ok")


def gen_layers(ssd, tag: str):
    from ssd.layers.activation import SiluAndMul
    from ssd.layers.layernorm import RMSDNorm, RMSHeadNorm
    from ssd.layers.rotary_embedding import RotaryEmbedding

    g = torch.Generator().manual_seed(14)
    out = {}
    d = 512
    x = (torch.randn(5, d, generator=g) * 2).to(torch.bfloat16)
    res = (torch.randn(5, d, generator=g) * 2).to(torch.bfloat16)
    w = (1 + 0.2 * torch.randn(d, generator=g)).to(torch.bfloat16)
    n = RMSDNorm(d, eps=1e-5).to(torch.bfloat16)
    n.weight.data.copy_(w)
    with torch.inference_mode():
        y0 = n(x.clone())
        y1, r1 = n(x.clone(), res.clone())
    out.update(norm_x=x, norm_res=res, norm_w=w, norm_y=y0, norm_add_y=y1, norm_add_res=r1)
    hd = 128
    xh = (torch.randn(12, hd, generator=g) * 2).to(torch.bfloat16)
    wh = (1 + 0.2 * torch.randn(hd, generator=g)).to(torch.bfloat16)
    hn = RMSHeadNorm(hd, eps=1e-6).to(torch.bfloat16)
    hn.weight.data.copy_(wh)
    with torch.inference_mode():
        out.update(hnorm_x=xh, hnorm_w=wh, hnorm_y=hn(xh.clone()))
    rope = RotaryEmbedding(64, 64, 512, 500000.0)
    q = torch.randn(6, 4 * 64, generator=g).to(torch.bfloat16)
    k = torch.randn(6, 2 * 64, generator=g).to(torch.bfloat16)
    pos = torch.tensor([0, 1, 2, 100, 101, 511])
    with torch.inference_mode():
        qo, ko = rope(pos, q.clone(), k.clone())
    out.update(rope_q=q, rope_k=k, rope_pos=pos, rope_qo=qo, rope_ko=ko, rope_table=rope.cos_sin_cache)
    gu = (torch.randn(5, 2 * 256, generator=g) * 2).to(torch.bfloat16)
    with torch.inference_mode():
        out.update(silu_x=gu, silu_y=SiluAndMul()(gu.clone()))
    npz = {}
    for kname, v in out.items():
        npz[kname] = v.view(torch.int16).numpy() if v.dtype == torch.bfloat16 else v.numpy()
    np.savez_compressed(OUT / f"layers_{tag}.npz", **npz)
    print(f"layers_{tag} ok")


def _hf_cfg(family, c):
    if family == "llama":
        from transformers import LlamaConfig as Cfg
    else:
        from transformers import Qwen3Config as Cfg
    cfg = Cfg(hidden_size=c.hidden, intermediate_size=c.ffn, num_hidden_layers=c.layers, num_attention_heads=c.heads,
              num_key_value_heads=c.kv_heads, head_dim=c.head_dim, vocab_size=c.vocab, rms_norm_eps=c.rms_eps,
              max_position_embeddings=c.max_pos, tie_word_embeddings=c.tie_embed, hidden_act="silu")
    cfg.rope_scaling = None  # SURVEY §8c(iv): transformers 5.5 makes this a dict; the reference needs None
    cfg.rope_theta = c.rope_theta
    cfg.torch_dtype = torch.bfloat16
    return cfg


def _build_ref_model(ssd, family, c, w, K, draft, num_blocks, block_size):
    from ssd.layers.rotary_embedding import get_rope
    get_rope.cache_clear()
    if family == "llama":
        from ssd.models.llama3 import LlamaForCausalLM as M
    else:
        from ssd.models.qwen3 import Qwen3ForCausalLM as M
    torch.set_default_dtype(torch.bfloat16)
    try:
        model = M(_hf_cfg(family, c), draft=draft, speculate=True, spec_k=K)
    finally:
        torch.set_default_dtype(torch.float32)
    H, KV, hd = c.heads, c.kv_heads, c.head_dim
    sd = dict(model.named_parameters())
    def load(name, tensor, *shard):
        p = sd[name]
        p.weight_loader(p, tensor, *shard) if hasattr(p, "weight_loader") else p.data.copy_(tensor)
    load("model.embed_tokens.weight", w["embed"])
    if not c.tie_embed:
        load("lm_head.weight", w["lm_head"])
    sd["model.norm.weight"].data.copy_(w["final_norm"])
    for l, lw in enumerate(w["layers"]):
        pre = f"model.layers.{l}."
        q, k, v = lw["qkv"].split([H * hd, KV * hd, KV * hd], dim=0)
        load(pre + "self_attn.qkv_proj.weight", q, "q")
        load(pre + "self_attn.qkv_proj.weight", k, "k")
        load(pre + "self_attn.qkv_proj.weight", v, "v")
        load(pre + "self_attn.o_proj.weight", lw["o"])
        gate, up = lw["gate_up"].chunk(2, dim=0)
        load(pre + "mlp.gate_up_proj.weight", gate, 0)
        load(pre + "mlp.gate_up_proj.weight", up, 1)
        load(pre + "mlp.down_proj.weight", lw["down"])
        sd[pre + "input_layernorm.weight"].data.copy_(lw["input_norm"])
        sd[pre + "post_attention_layernorm.weight"].data.copy_(lw["post_norm"])
        if c.qk_norm:
            sd[pre + "self_attn.q_norm.weight"].data.copy_(lw["q_norm"])
            sd[pre + "self_attn.k_norm.weight"].data.copy_(lw["k_norm"])
    # allocate_kv_cache (engine/model_runner.py:484-503)
    kv = torch.zeros(2, c.layers, num_blocks, block_size, KV, hd, dtype=torch.bfloat16)
    lid = 0
    for mod in model.modules():
        if hasattr(mod, "k_cache") and hasattr(mod, "v_cache"):
            mod.k_cache, mod.v_cache = kv[0, lid], kv[1, lid]
            lid += 1
    model.eval()
    return model, kv


def gen_trace(ssd, family):
    """Whole sync-SD token traces through the reference model classes + Sampler + verify(), temp 0."""
    from oracle.model import ModelCfg, random_weights
    from ssd.layers.sampler import Sampler
    from ssd.utils.context import reset_context, set_context
    from ssd.utils.verify import verify

    K, B, bs, mb = 4, 2, 64, 3
    hd = 64 if family == "llama" else 128
    tc = ModelCfg(hidden=128, layers=2, heads=2, kv_heads=1, head_dim=hd, ffn=256, vocab=512, max_pos=512,
                  rms_eps=1e-5 if family == "llama" else 1e-6, rope_theta=500000.0 if family == "llama" else 1000000.0,
                  qk_norm=(family != "llama"))
    dc = ModelCfg(**{**tc.__dict__, "layers": 1})
    wt = random_weights(tc, 21 if family == "llama" else 31)
    # correlated draft: the target's first layer + its embedding / head (gives accept lengths between 1 and K+1)
    wd = {"embed": wt["embed"], "lm_head": wt["lm_head"], "final_norm": wt["final_norm"], "layers": [wt["layers"][0]]}
    tgt, _ = _build_ref_model(ssd, family, tc, wt, K, False, B * mb, bs)
    drf, _ = _build_ref_model(ssd, family, dc, wd, K, True, B * mb, bs)
    sampler = Sampler()
    prompts = [[3, 14, 15, 92, 65, 35, 89, 79], [2, 71, 82, 81, 82]]
    bt = torch.arange(B * mb, dtype=torch.int32).view(B, mb)
    temps = torch.zeros(B)
    slot = lambda b, p: int(bt[b, p // bs]) * bs + p % bs

    @torch.inference_mode()
    def prefill(model):
        ids = torch.tensor([t for p in prompts for t in p])
        pos = torch.tensor([i for p in prompts for i in range(len(p))])
        cu = torch.tensor([0] + list(np.cumsum([len(p) for p in prompts])), dtype=torch.int32)
        sm = torch.tensor([slot(b, i) for b, p in enumerate(prompts) for i in range(len(p))], dtype=torch.int32)
        mx = max(len(p) for p in prompts)
        set_context(True, cu, cu, mx, mx, sm, None, None)  # model_runner.py:506-517
        h = model(ids, pos)
        logits = model.compute_logits(h, True)
        reset_context()
        return logits

    @torch.inference_mode()
    def decode(model, toks, ctx):  # model_runner.py:519-540 (non-verify)
        ids = torch.tensor(toks)
        pos = torch.tensor(ctx)
        sm = torch.tensor([slot(b, c) for b, c in enumerate(ctx)], dtype=torch.int32)
        cl = torch.tensor([c + 1 for c in ctx], dtype=torch.int32)
        set_context(False, None, None, 0, 0, sm, cl, bt)
        logits = model.compute_logits(model(ids, pos), True)
        reset_context()
        return logits

    @torch.inference_mode()
    def verify_fwd(model, spec, ctx):  # model_runner.py:526-533
        ids = spec.reshape(-1)
        pos = torch.tensor([c + j for c in ctx for j in range(K + 1)])
        sm = torch.tensor([slot(b, c + j) for b, c in enumerate(ctx) for j in range(K + 1)], dtype=torch.int32)
        cl = torch.tensor([c + K + 1 for c in ctx], dtype=torch.int32)
        cu = torch.arange(B + 1, dtype=torch.int32) * (K + 1)
        set_context(False, cu, None, K + 1, 0, sm, cl, bt)
        logits = model.compute_logits(model(ids, pos), False)
        reset_context()
        return logits.view(B, K + 1, -1)

    lg = prefill(tgt)
    prefill(drf)
    recovery = sampler(lg, temps).tolist()
    ctx = [len(p) for p in prompts]
    rec0 = list(recovery)
    steps_tokens, steps_nacc, first = [], [], {}
    for step in range(10):
        spec = torch.zeros(B, K + 1, dtype=torch.int64)
        spec[:, 0] = torch.tensor(recovery)
        lqs = []
        for k in range(K + 1):  # speculator_sync.py:47-65
            lq = decode(drf, spec[:, k].tolist(), [c + k for c in ctx])
            if k == K:
                break
            lqs.append(lq)
            spec[:, k + 1] = sampler(lq, temps)
        lq = torch.stack(lqs, 1)
        lp = verify_fwd(tgt, spec, ctx)
        suf, rec = verify(lp, lq, spec, temps, temps, None, None, None, True)
        if step == 0:
            first = dict(lp0=lp.view(torch.int16).numpy(), lq0=lq.view(torch.int16).numpy(), spec0=spec.numpy())
        steps_tokens.append(spec.numpy().copy())
        steps_nacc.append([len(s) - 1 for s in suf])
        ctx = [c + len(s) for c, s in zip(ctx, suf)]
        recovery = rec
    npz = dict(K=np.array(K), block_size=np.array(bs), max_blocks=np.array(mb), prompt0=np.array(prompts[0]),
               prompt1=np.array(prompts[1]), rec0=np.array(rec0), spec=np.stack(steps_tokens),
               nacc=np.array(steps_nacc, dtype=np.int32), final_recovery=np.array(recovery),
               prefill_logits=lg.view(torch.int16).numpy(), **first)
    # the draft's weights are a subset of the target's (tests/helpers.py:trace_weights rebuilds them)
    for kname in ("embed", "lm_head", "final_norm"):
        npz[f"t_{kname}"] = wt[kname].view(torch.int16).numpy()
    for l, lw in enumerate(wt["layers"]):
        for kname, v in lw.items():
            npz[f"t_l{l}_{kname}"] = v.view(torch.int16).numpy()
    np.savez_compressed(OUT / f"trace_{family}.npz", **npz)
    print(f"trace_{family} ok; accept lens per step: {steps_nacc}")


def main():
    OUT.mkdir(parents=True, exist_ok=True)
    tag = sys.argv[1] if len(sys.argv) > 1 else "compiled"
    torch.manual_seed(0)
    ssd = import_reference()
    if tag == "eager":
        assert os.environ.get("TORCHDYNAMO_DISABLE") == "1"
        gen_layers(ssd, "eager")
        return
    if tag == "mixed":  # incremental: only the per-row-temperature verify cases
        gen_verify_mixed(ssd)
        return
    gen_verify_t0(ssd)
    gen_verify_ratio(ssd)
    gen_verify_mixed(ssd)
    gen_sampler(ssd)
    gen_layers(ssd, "compiled")
    gen_trace(ssd, "llama")
    gen_trace(ssd, "qwen")


if __name__ == "__main__":
    main()
