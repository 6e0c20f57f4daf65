"""Tensor-parallel hot path on 2 GPUs (one process per GPU, NCCL): prefill + speculative steps through the C-ABI on
both ranks, rank 0's verdicts checked against the single-device CPU oracle (teacher-forced, near-tie protocol).
Covers the in-graph collectives: embedding all-reduce, row-parallel all-reduce, vocab-parallel lm_head all-gather,
draft-token broadcast, verdict broadcast.  Needs >= 2 GPUs; skips on one."""
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu
EPS = 0.08


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


DIMS = {
    # hidden, heads, kv_heads, ffn, vocab
    "small": (256, 4, 2, 512, 1024),
    # wide enough for the in-kernel split-K paths: o-proj K = 512 / rank (2 splits), down-proj K = 2048 / rank (8 splits,
    # ticket reduction + publish from the last CTA of a tile), gate|up 64 tiles / rank (split-K SiLU epilogue)
    "wide": (1024, 16, 2, 8192, 2048),
}


def _rank_main(rank, world, port, use_graph, use_symm, q, dims="small", fused_publish="0"):
    import os
    os.environ["SSDK_FUSED_PUBLISH"] = fused_publish  # read once per process by libssdk
    import torch.distributed as dist
    from oracle.model import ModelCfg, OracleModel, random_weights
    from oracle.spec import SpecSession, check_greedy_step, contiguous_block_tables
    from ssd_b200 import lib as L
    from ssd_b200.loader import shard_packed_weights
    from ssd_b200.parallel import create_nccl_comm
    from ssd_b200.runner import ModelSpec, PairRunner
    try:
        torch.cuda.set_device(rank)
        dist.init_process_group("cpu:gloo,cuda:nccl", init_method=f"tcp://127.0.0.1:{port}", world_size=world, rank=rank,
                                device_id=torch.device("cuda", rank))
        comm = create_nccl_comm(world, rank)
        K, B, bs, mb = 4, 2, 64, 3
        hidden, heads, kvh, ffn, vocab = DIMS[dims]
        tc = ModelCfg(hidden=hidden, layers=2, heads=heads, kv_heads=kvh, head_dim=64, ffn=ffn, vocab=vocab, max_pos=256)
        dc = ModelCfg(**{**tc.__dict__, "layers": 1})
        wt = random_weights(tc, 41)
        wd = {"embed": wt["embed"], "lm_head": wt["lm_head"], "final_norm": wt["final_norm"], "layers": [wt["layers"][0]]}
        spec = lambda c: ModelSpec(c.hidden, c.layers, c.heads, c.kv_heads, c.head_dim, c.ffn, c.vocab, c.rms_eps,
                                   c.rope_theta, c.qk_norm, False, c.max_pos)
        dev = torch.device("cuda", rank)
        to = lambda w: {**{k: v.to(dev).contiguous() for k, v in w.items() if k != "layers"},
                        "layers": [{k: v.to(dev).contiguous() for k, v in lw.items()} for lw in w["layers"]]}
        r = PairRunner(spec(tc), spec(dc) if rank == 0 else None, spec_k=K, max_batch=B, block_size=bs,
                       max_model_len=bs * mb, device=dev, use_graph=use_graph, tp_size=world, tp_rank=rank)
        r.bind_weights(L.TARGET, to(shard_packed_weights(wt, spec(tc), world, rank)))
        if rank == 0:
            r.bind_weights(L.DRAFT, to(wd))
        r.set_nccl_comm(comm)
        if use_symm:
            from ssd_b200.parallel import bind_symmetric_memory
            assert bind_symmetric_memory(r, world, rank), "symmetric memory could not be set up"
        r.finalize()
        bt = contiguous_block_tables(B, mb)
        bts = [bt[b].tolist() for b in range(B)]
        prompts = [[3, 14, 15, 92, 65, 35, 89, 79], [2, 71, 82, 81, 82]]
        rec = []
        for b in range(B):
            rec.append(r.prefill(L.TARGET, prompts[b], bts[b]))
            r.prefill(L.DRAFT, prompts[b], bts[b], want_sample=False)  # no-op on rank 1
        ctx = [len(p) for p in prompts]
        s = None
        if rank == 0:
            s = SpecSession(OracleModel(tc, wt, B * mb, bs), OracleModel(dc, wd, B * mb, bs), K, mb)
            rec_o = s.prefill(prompts, [0.0, 0.0], bt, bt.clone())
        log = []
        for step in range(8):
            toks, nacc, nrec = r.spec_step(ctx, rec, bts, bts, [0.0] * B, [0.0] * B)
            log.append((toks.tolist(), nacc.tolist(), nrec.tolist()))
            if rank == 0:
                sp = torch.from_numpy(toks)
                lp, lq = s.spec_step_forced(sp)
                lp_e = r.logits_p(B).cpu()
                torch.testing.assert_close(lp_e.float(), lp.float(), atol=0.1, rtol=0.04)
                hard, soft = check_greedy_step(sp, nacc.tolist(), nrec.tolist(), lp, lq, EPS)
                assert not hard, f"step {step}: {hard}"
                s.advance(nacc.tolist(), nrec.tolist())
            ctx = [c + int(n) + 1 for c, n in zip(ctx, nacc)]
            rec = nrec.tolist()
        q.put((rank, "ok", rec if rank != 0 else rec, log))
        r.close()
    except Exception as exc:  # noqa: BLE001
        import traceback
        q.put((rank, "fail", traceback.format_exc(), None))


@pytest.mark.parametrize("use_graph,use_symm,dims,fused", [
    (False, False, "small", "0"), (True, False, "small", "0"), (False, True, "small", "0"), (True, True, "small", "0"),
    (True, True, "wide", "0"), (False, True, "wide", "0"),
    (True, True, "small", "1"), (True, True, "wide", "1"), (False, True, "wide", "1"),  # GEMM-epilogue publish (EPI_PUBLISH)
])
def test_tp2_spec_steps(use_graph, use_symm, dims, fused):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank_main, args=(r, 2, port, use_graph, use_symm, q, dims, fused)) for r in range(2)]
    for p in procs:
        p.start()
    res = {}
    try:
        for _ in range(2):
            rank, status, payload, log = q.get(timeout=150)
            res[rank] = (status, payload, log)
            assert status == "ok", f"rank {rank} failed:\n{payload}"
    finally:
        for p in procs:
            p.join(timeout=5)
            if p.is_alive():
                p.terminate()
    for rank, (status, payload, _) in res.items():
        assert status == "ok", f"rank {rank} failed:\n{payload}"
    # the verdict broadcast makes every rank see identical tokens / accept counts / recovery tokens
    assert res[0][2] == res[1][2]
