"""GPU tests of an FP8 target through the public and the multi-call paths: LLM.generate from an FP8 checkpoint against
quantize-on-load of the bf16 checkpoint it came from, varlen prefill with prefix-cache hits, two decoder layers at
Llama-3.1-8B widths with the full vocabulary, and a 2-GPU tensor-parallel target (skips on one GPU)."""
import json
import socket

import pytest
import torch

from tests.fp8_ref import Fp8OracleModel, quantize_weights

pytestmark = pytest.mark.gpu
EPS = 0.08
F8 = torch.float8_e4m3fn


def _to_dev(w, dev):
    out = {k: v.to(dev).contiguous() for k, v in w.items() if k != "layers"}
    out["layers"] = [{k: v.to(dev).contiguous() for k, v in lw.items()} for lw in w["layers"]]
    return out


def _spec(c):
    from ssd_b200.runner import ModelSpec
    return ModelSpec(hidden=c.hidden, layers=c.layers, heads=c.heads, kv_heads=c.kv_heads, head_dim=c.head_dim, ffn=c.ffn,
                     vocab=c.vocab, rms_eps=c.rms_eps, rope_theta=c.rope_theta, qk_norm=c.qk_norm, max_pos=c.max_pos)


# ------------------------------------------------------------------------------------------------ checkpoint equivalence
def _write_checkpoint(path, c, w, fp8: bool):
    """HF Llama safetensors layout; FP8: e4m3 `<proj>.weight` + fp32 per-channel `weight_scale` [N, 1] + an unused
    `input_scale`, and a compressed-tensors float8 quantization_config (the layout of published FP8 Llama checkpoints)."""
    from safetensors.torch import save_file
    from ssd_b200.quant import quantize_fp8_rowwise
    path.mkdir()
    H, KV, hd = c.heads, c.kv_heads, c.head_dim
    t = {"model.embed_tokens.weight": w["embed"], "lm_head.weight": w["lm_head"], "model.norm.weight": w["final_norm"]}
    for l, lw in enumerate(w["layers"]):
        q, k, v = lw["qkv"].split([H * hd, KV * hd, KV * hd])
        gate, up = lw["gate_up"].chunk(2)
        mats = {"self_attn.q_proj": q, "self_attn.k_proj": k, "self_attn.v_proj": v, "self_attn.o_proj": lw["o"],
                "mlp.gate_proj": gate, "mlp.up_proj": up, "mlp.down_proj": lw["down"]}
        for leaf, m in mats.items():
            name = f"model.layers.{l}.{leaf}"
            if fp8:
                w8, s = quantize_fp8_rowwise(m)
                t[name + ".weight"], t[name + ".weight_scale"] = w8, s[:, None]
                t[name + ".input_scale"] = torch.ones(1)
            else:
                t[name + ".weight"] = m
        t[f"model.layers.{l}.input_layernorm.weight"] = lw["input_norm"]
        t[f"model.layers.{l}.post_attention_layernorm.weight"] = lw["post_norm"]
    save_file({k: v.contiguous() for k, v in t.items()}, str(path / "model.safetensors"))
    cfg = {"model_type": "llama", "hidden_size": c.hidden, "num_hidden_layers": c.layers, "num_attention_heads": H,
           "num_key_value_heads": KV, "head_dim": hd, "intermediate_size": c.ffn, "vocab_size": c.vocab,
           "rms_norm_eps": c.rms_eps, "rope_theta": c.rope_theta, "max_position_embeddings": 2048,
           "tie_word_embeddings": False, "bos_token_id": 0, "eos_token_id": 1}
    if fp8:
        cfg["quantization_config"] = {"quant_method": "compressed-tensors", "config_groups": {"group_0": {
            "targets": ["Linear"], "weights": {"num_bits": 8, "type": "float", "strategy": "channel", "symmetric": True}}},
            "ignore": ["lm_head"]}
    (path / "config.json").write_text(json.dumps(cfg))
    return str(path)


def test_fp8_checkpoint_generates_like_quantize_on_load(tmp_path):
    """LLM.generate from an FP8 checkpoint equals LLM.generate from the bf16 checkpoint it was quantized from with
    quantization="fp8": the same tokens, bit-identical device weights, and both engines report quantization "fp8"."""
    from oracle.model import ModelCfg, random_weights
    from ssd_b200 import LLM, SamplingParams, synth
    from ssd_b200 import lib as L
    c = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024, max_pos=2048)
    w = random_weights(c, 13)
    # the directory names carry the model family, as the engine reads it from the paths
    bf_dir = _write_checkpoint(tmp_path / "llama-tiny-bf16", c, w, fp8=False)
    f8_dir = _write_checkpoint(tmp_path / "llama-tiny-fp8", c, w, fp8=True)
    draft = synth.make_model_dir(str(tmp_path), "llama-tiny-draft", "draft", seed=1, max_position_embeddings=2048)
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(2, 1000, (n,), generator=g).tolist() for n in (5, 70, 33)]
    runs = {}
    for tag, path, q in (("quantize-on-load", bf_dir, "fp8"), ("fp8 checkpoint", f8_dir, None)):
        llm = LLM(path, speculate=True, draft=draft, speculate_k=4, max_num_seqs=3, max_model_len=1024,
                  kvcache_block_size=64, tokenizer_path=draft, quantization=q)
        assert llm.config.quantization == "fp8", tag
        out, _ = llm.generate(prompts, SamplingParams(temperature=0.0, max_new_tokens=24, ignore_eos=True), use_tqdm=False)
        wt = llm.runner.weights[L.TARGET]["layers"]
        runs[tag] = ([o["token_ids"] for o in out],
                     [{n: (lw[n].view(torch.uint8).cpu(), lw[n + "_scale"].cpu()) for n in ("qkv", "o", "gate_up", "down")}
                      for lw in wt])
        assert all(lw[n].dtype == F8 for lw in wt for n in ("qkv", "o", "gate_up", "down")), tag
        llm.exit()
    (ta, wa), (tb, wb) = runs["quantize-on-load"], runs["fp8 checkpoint"]
    for l in range(c.layers):
        for n in ("qkv", "o", "gate_up", "down"):
            assert torch.equal(wa[l][n][0], wb[l][n][0]), (l, n, "weights")
            assert torch.equal(wa[l][n][1], wb[l][n][1]), (l, n, "scales")
    assert ta == tb


# ------------------------------------------------------------------------------------------------ varlen prefill
def test_fp8_target_prefill_varlen_with_prefix_hits_matches_fp8_oracle():
    """prefill_varlen with an FP8 target: sequences 1 and 2 alias the first two 64-token pages of sequence 0 (prefix-cache
    hits joining the call that writes them); first tokens, then two speculative steps against the FP8 oracle."""
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession, check_greedy_step
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    dev = torch.device("cuda:0")
    bs, mb, K = 64, 6, 4
    lens, starts = [200, 150, 200, 140], [0, 128, 128, 0]
    B = len(lens)
    c = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024, max_pos=bs * mb)
    dc = ModelCfg(**{**c.__dict__, "layers": 1})
    wt = random_weights(c, 41)
    wd = {"embed": wt["embed"], "lm_head": wt["lm_head"], "final_norm": wt["final_norm"], "layers": [wt["layers"][0]]}
    wo, we = quantize_weights(wt)
    r = PairRunner(_spec(c), _spec(dc), spec_k=K, max_batch=B, block_size=bs, max_model_len=bs * mb, use_graph=True)
    r.bind_weights(L.TARGET, _to_dev(we, dev))
    r.bind_weights(L.DRAFT, _to_dev(wd, dev))
    r.finalize()
    bts = [list(range(b * mb, (b + 1) * mb)) for b in range(B)]
    for i in (1, 2):
        bts[i][:2] = bts[0][:2]
    g = torch.Generator().manual_seed(17)
    prefix = torch.randint(0, c.vocab, (128,), generator=g).tolist()
    prompts = [prefix + torch.randint(0, c.vocab, (n - 128,), generator=g).tolist() for n in lens]
    bt = torch.tensor(bts, dtype=torch.int32)
    s = SpecSession(Fp8OracleModel(c, wo, B * mb, bs), OracleModel(dc, wd, B * mb, bs), K, mb)
    rec_o = s.prefill(prompts, [0.0] * B, bt, bt.clone())
    rec = r.prefill_varlen(L.TARGET, prompts, bts, starts)
    r.prefill_varlen(L.DRAFT, prompts, bts, starts, want_sample=False)
    assert sum(int(a != b_) for a, b_ in zip(rec, rec_o)) <= 1, (rec, rec_o)
    rec, ctx = list(rec_o), list(lens)
    for step in range(2):
        toks, nacc, nrec = r.spec_step(ctx, rec, bts, bts, [0.0] * B, [0.0] * B)
        spec = torch.from_numpy(toks)
        lp_o, lq_o = s.spec_step_forced(spec)
        torch.testing.assert_close(r.logits_p(B).cpu().float(), lp_o.float(), atol=0.08, rtol=0.03)
        torch.testing.assert_close(r.logits_q(B).cpu().float(), lq_o.float(), atol=0.08, rtol=0.03)
        hard, _ = check_greedy_step(spec, nacc.tolist(), nrec.tolist(), lp_o, lq_o, EPS)
        assert not hard, f"step {step}: {hard}"
        ctx = [x + int(n) + 1 for x, n in zip(ctx, nacc)]
        rec = nrec.tolist()
        s.advance(nacc.tolist(), rec)
    r.close()


# ------------------------------------------------------------------------------------------------ true widths
def test_fp8_target_at_llama8b_widths_matches_fp8_oracle():
    """Two decoder layers at Llama-3.1-8B widths (K = 4096 / 14336: 32 / 112 FP8 k-blocks, the stage ring wraps many times,
    the engine's own split-K plan), full 128256 vocabulary, batch 1, a 200-token prompt; the draft is one layer at
    Llama-3.2-1B widths (bf16, streaming draft kernel).  First token, then three speculative steps: target and draft
    logits against the FP8 oracle on the host, decisions under the near-tie protocol."""
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession, check_greedy_step
    from ssd_b200 import lib as L
    from ssd_b200.runner import PairRunner
    dev = torch.device("cuda:0")
    bs, mb, K = 256, 2, 4
    tc = ModelCfg(hidden=4096, layers=2, heads=32, kv_heads=8, head_dim=128, ffn=14336, vocab=128256, max_pos=bs * mb)
    dc = ModelCfg(hidden=2048, layers=1, heads=32, kv_heads=8, head_dim=64, ffn=8192, vocab=128256, max_pos=bs * mb)
    wt, wd = random_weights(tc, 3), random_weights(dc, 4)
    wo, we = quantize_weights(wt)
    r = PairRunner(_spec(tc), _spec(dc), spec_k=K, max_batch=1, block_size=bs, max_model_len=bs * mb, use_graph=True)
    r.bind_weights(L.TARGET, _to_dev(we, dev))
    r.bind_weights(L.DRAFT, _to_dev(wd, dev))
    r.finalize()
    del we
    g = torch.Generator().manual_seed(11)
    prompt = torch.randint(0, tc.vocab, (200,), generator=g).tolist()
    bt = torch.arange(mb, dtype=torch.int32)[None, :]
    s = SpecSession(Fp8OracleModel(tc, wo, mb, bs), OracleModel(dc, wd, mb, bs), K, mb)
    rec_o = s.prefill([prompt], [0.0], bt, bt.clone())
    rec = r.prefill(L.TARGET, prompt, bt[0].tolist())
    r.prefill(L.DRAFT, prompt, bt[0].tolist(), want_sample=False)
    want = s.t.compute_logits(s._forward(s.t, torch.tensor(prompt), [0], len(prompt), bt)[-1:])[0].float()
    got = r.logits_last(1)[0].float().cpu()
    torch.testing.assert_close(got, want, atol=0.25, rtol=1 / 32)
    top2 = want.topk(2).values
    assert rec == rec_o[0] or float(top2[0] - top2[1]) < EPS, (rec, rec_o)
    rec, ctx, worst = rec_o[0], len(prompt), 0.0
    for step in range(3):
        toks, nacc, nrec = r.spec_step([ctx], [rec], [bt[0].tolist()], [bt[0].tolist()], [0.0], [0.0])
        spec = torch.from_numpy(toks)
        lp_o, lq_o = s.spec_step_forced(spec)
        for eng, ref in ((r.logits_p(1), lp_o), (r.logits_q(1), lq_o)):
            torch.testing.assert_close(eng.cpu().float(), ref.float(), atol=0.25, rtol=1 / 32)
            worst = max(worst, float((eng.cpu().float() - ref.float()).abs().mean()))
        hard, _ = check_greedy_step(spec, nacc.tolist(), nrec.tolist(), lp_o, lq_o, EPS)
        assert not hard, f"step {step}: {hard}"
        ctx += int(nacc[0]) + 1
        rec = int(nrec[0])
        s.advance(nacc.tolist(), [rec])
    print(f"[fp8 llama8b widths] worst mean |logit diff| {worst:.4f}")
    r.close()


# ------------------------------------------------------------------------------------------------ tensor parallel
DIMS = {"small": (256, 4, 2, 512, 1024),
        # o K = 512 / rank, down K = 2048 / rank (split-K ticket + publish), gate|up 64 tiles / rank (split-K SiLU)
        "wide": (1024, 16, 2, 8192, 2048)}


def _free_port():
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        return sk.getsockname()[1]


def _rank_main(rank, world, port, dims, fused_publish, q):
    import os
    os.environ["SSDK_FUSED_PUBLISH"] = fused_publish  # read once per process by libssdk
    import torch.distributed as dist
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession, check_greedy_step, contiguous_block_tables
    from ssd_b200 import lib as L
    from ssd_b200.loader import tp_row_amax_max, shard_packed_weights
    from ssd_b200.parallel import bind_symmetric_memory, create_nccl_comm
    from ssd_b200.quant import quantize_layers_
    from ssd_b200.runner import PairRunner
    try:
        torch.cuda.set_device(rank)
        dev = torch.device("cuda", rank)
        dist.init_process_group("cpu:gloo,cuda:nccl", init_method=f"tcp://127.0.0.1:{port}", world_size=world, rank=rank,
                                device_id=dev)
        comm = create_nccl_comm(world, rank)
        K, B, bs, mb = 4, 2, 64, 3
        hidden, heads, kvh, ffn, vocab = DIMS[dims]
        tc = ModelCfg(hidden=hidden, layers=2, heads=heads, kv_heads=kvh, head_dim=64, ffn=ffn, vocab=vocab, max_pos=256)
        dc = ModelCfg(**{**tc.__dict__, "layers": 1})
        wt = random_weights(tc, 41)
        wd = {"embed": wt["embed"], "lm_head": wt["lm_head"], "final_norm": wt["final_norm"], "layers": [wt["layers"][0]]}
        wo, we = quantize_weights(wt)
        spec = _spec(tc)
        mine = shard_packed_weights(we, spec, world, rank)
        # quantize-on-load of this rank's bf16 shard (the loader's path, MAX all-reduce of the o / down row amax) gives
        # exactly this rank's shard of the quantized full weights
        onload = quantize_layers_(_to_dev(shard_packed_weights(wt, spec, world, rank), dev), tp_row_amax_max)
        for l in range(tc.layers):
            for n in ("qkv", "o", "gate_up", "down"):
                assert torch.equal(onload["layers"][l][n].view(torch.uint8).cpu(), mine["layers"][l][n].view(torch.uint8))
                assert torch.equal(onload["layers"][l][n + "_scale"].cpu(), mine["layers"][l][n + "_scale"])
        r = PairRunner(spec, _spec(dc) if rank == 0 else None, spec_k=K, max_batch=B, block_size=bs, max_model_len=bs * mb,
                       device=dev, use_graph=True, tp_size=world, tp_rank=rank)
        r.bind_weights(L.TARGET, _to_dev(mine, dev))
        if rank == 0:
            r.bind_weights(L.DRAFT, _to_dev(wd, dev))
        r.set_nccl_comm(comm)
        assert bind_symmetric_memory(r, world, rank), "symmetric memory could not be set up"
        r.finalize()
        bt = contiguous_block_tables(B, mb)
        bts = [bt[b].tolist() for b in range(B)]
        prompts = [[3, 14, 15, 92, 65, 35, 89, 79], [2, 71, 82, 81, 82]]
        rec = []
        for b in range(B):
            rec.append(r.prefill(L.TARGET, prompts[b], bts[b]))
            r.prefill(L.DRAFT, prompts[b], bts[b], want_sample=False)
        ctx = [len(p) for p in prompts]
        s = None
        if rank == 0:
            s = SpecSession(Fp8OracleModel(tc, wo, B * mb, bs), OracleModel(dc, wd, B * mb, bs), K, mb)
            s.prefill(prompts, [0.0, 0.0], bt, bt.clone())
        log = []
        for step in range(8):
            toks, nacc, nrec = r.spec_step(ctx, rec, bts, bts, [0.0] * B, [0.0] * B)
            log.append((toks.tolist(), nacc.tolist(), nrec.tolist()))
            if rank == 0:
                sp = torch.from_numpy(toks)
                lp, lq = s.spec_step_forced(sp)
                torch.testing.assert_close(r.logits_p(B).cpu().float(), lp.float(), atol=0.1, rtol=0.04)
                hard, _ = check_greedy_step(sp, nacc.tolist(), nrec.tolist(), lp, lq, EPS)
                assert not hard, f"step {step}: {hard}"
                s.advance(nacc.tolist(), nrec.tolist())
            ctx = [x + int(n) + 1 for x, n in zip(ctx, nacc)]
            rec = nrec.tolist()
        q.put((rank, "ok", None, log))
        r.close()
    except Exception:  # noqa: BLE001
        import traceback
        q.put((rank, "fail", traceback.format_exc(), None))


@pytest.mark.parametrize("dims,fused", [("small", "0"), ("wide", "0"), ("wide", "1")])
def test_tp2_fp8_target_matches_fp8_oracle(dims, fused):
    """FP8 target split over 2 GPUs: column-parallel shards carry their row scales, row-parallel ones all of them; the
    wide shape reaches the in-kernel split-K SiLU epilogue, and fused = "1" the FP8 EPI_PUBLISH instances."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank_main, args=(rk, 2, port, dims, fused, q)) for rk in range(2)]
    for p in procs:
        p.start()
    res = {}
    try:
        for _ in range(2):
            rank, status, payload, log = q.get(timeout=300)
            res[rank] = (status, payload, log)
            assert status == "ok", f"rank {rank} failed:\n{payload}"
    finally:
        for p in procs:
            p.join(timeout=5)
            if p.is_alive():
                p.terminate()
    assert res[0][2] == res[1][2]
