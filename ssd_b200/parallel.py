"""Tensor parallelism of the target across up to 8 GPUs — one process per GPU.

The reference spawns one ModelRunner process per TP rank and drives them from rank 0 through pickle-over-shm RPC
(engine/llm_engine.py:61-76, engine/model_runner.py:404-428).  Here every rank runs the SAME deterministic host
engine (scheduler, block manager) in lock-step — SPMD — and the device keeps them in sync:

  * inside the step graph the K draft tokens (draft pinned to rank 0) are ncclBroadcast to the other ranks before the
    verify forward, row-parallel GEMM outputs are all-reduced, the vocab-parallel lm_head is all-gathered, and rank 0's
    verdict (tokens, accept counts, recovery) is broadcast back, so every rank's scheduler sees identical results;
  * no per-step host RPC exists at all.

Two launch modes:
  * torchrun / any launcher that sets RANK, WORLD_SIZE, LOCAL_RANK: every rank constructs LLM(num_gpus=WORLD_SIZE)
    and calls generate() with the same arguments (bench.py does this);
  * plain `LLM(model, num_gpus=N)` in one process (the reference's calling convention): N-1 worker processes are
    spawned; they build the same engine and replay every generate() call they receive over a multiprocessing queue.

The NCCL communicator handed to libssdk is created here with the same libnccl that the library links.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import torch
import torch.distributed as dist


# --------------------------------------------------------------------------------------------- NCCL comm
class _NcclUniqueId(C.Structure):
    _fields_ = [("internal", C.c_byte * 128)]


def _libnccl() -> C.CDLL:
    try:
        import nvidia.nccl as n
        so = sorted((Path(n.__path__[0]) / "lib").glob("libnccl.so*"))
        if so:
            return C.CDLL(str(so[0]), mode=C.RTLD_GLOBAL)
    except Exception:
        pass
    return C.CDLL("libnccl.so.2", mode=C.RTLD_GLOBAL)


def create_nccl_comm(world: int, rank: int, group=None) -> int:
    """ncclGetUniqueId on rank 0, broadcast through torch.distributed, ncclCommInitRank everywhere.
    Returns the raw ncclComm_t as an integer (kept alive for the life of the process)."""
    nccl = _libnccl()
    uid = _NcclUniqueId()
    if rank == 0:
        rc = nccl.ncclGetUniqueId(C.byref(uid))
        if rc != 0:
            raise RuntimeError(f"ncclGetUniqueId failed ({rc})")
    backend = dist.get_backend(group)
    dev = torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" else torch.device("cpu")
    buf = torch.tensor(list(bytes(uid)), dtype=torch.uint8, device=dev)
    dist.broadcast(buf, src=0, group=group)
    raw = bytes(buf.cpu().tolist())
    C.memmove(C.byref(uid), raw, 128)
    comm = C.c_void_p()
    nccl.ncclCommInitRank.argtypes = [C.POINTER(C.c_void_p), C.c_int, _NcclUniqueId, C.c_int]
    rc = nccl.ncclCommInitRank(C.byref(comm), world, uid, rank)
    if rc != 0:
        raise RuntimeError(f"ncclCommInitRank failed ({rc})")
    return comm.value


def bind_symmetric_memory(runner, world: int, rank: int, group=None) -> bool:
    """Allocate the NVLink symmetric buffer of the one-shot all-reduce (torch symmetric memory: cuMem + peer mapping),
    rendezvous with the other ranks and hand every rank's mapped pointer to libssdk (ssdk_bind_symm).  Returns False
    (the engine then keeps the in-graph NCCL all-reduce) ONLY when disabled with SSD_B200_NO_SYMM=1; if symmetric
    memory cannot be set up the launch fails loudly — a silent fall-back to NCCL would make every multi-GPU number
    unattributable (bench.py records which all-reduce ran in its "allreduce" key)."""
    if os.environ.get("SSD_B200_NO_SYMM") == "1":
        return False
    from . import lib as L
    nbytes = int(runner.lib.ssdk_symm_bytes(runner.h))
    if nbytes <= 0:
        return False
    try:
        import torch.distributed._symmetric_memory as symm_mem
        buf = symm_mem.empty(nbytes, dtype=torch.uint8, device=runner.device)
        buf.zero_()
        hdl = symm_mem.rendezvous(buf, group if group is not None else dist.group.WORLD)
        ptrs = [int(hdl.buffer_ptrs[r]) for r in range(world)]
        torch.cuda.synchronize()
        dist.barrier(group)  # every rank has zeroed its flags before anyone publishes
    except Exception as exc:  # noqa: BLE001
        raise RuntimeError(f"NVLink symmetric memory unavailable ({type(exc).__name__}: {exc}); set SSD_B200_NO_SYMM=1 to run "
                           "the tensor-parallel all-reduces through NCCL instead") from exc
    arr = (C.c_void_p * world)(*ptrs)
    L.check(runner.lib.ssdk_bind_symm(runner.h, arr, world), "ssdk_bind_symm")
    runner._keep.extend([buf, hdl])
    return True


# --------------------------------------------------------------------------------------------- engines
def _ensure_pg(world: int, rank: int, port: int | None = None) -> None:
    if dist.is_initialized():
        return
    if "MASTER_ADDR" in os.environ and port is None:
        dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    else:
        dist.init_process_group("cpu:gloo,cuda:nccl", init_method=f"tcp://127.0.0.1:{port}", world_size=world, rank=rank,
                                device_id=torch.device("cuda", torch.cuda.current_device()))


def build_tp_rank(config, world: int, rank: int, local_rank: int, port: int | None = None):
    """Build this rank's PairRunner (target shard [+ draft on rank 0]) and wire the NCCL communicator."""
    from .loader import build_runner
    torch.cuda.set_device(local_rank)
    _ensure_pg(world, rank, port)
    comm = create_nccl_comm(world, rank)
    runner, draft_cfg = build_runner(config, tp_size=world, tp_rank=rank, device=f"cuda:{local_rank}", finalize=False)
    runner.set_nccl_comm(comm)
    runner.symm = bind_symmetric_memory(runner, world, rank)
    runner.finalize()
    # all ranks must agree on the number of KV blocks so that the SPMD schedulers stay identical
    nb = torch.tensor([config.num_kvcache_blocks, draft_cfg.num_kvcache_blocks], dtype=torch.int64,
                      device="cuda" if dist.get_backend() == "nccl" else "cpu")
    dist.all_reduce(nb, op=dist.ReduceOp.MIN)
    config.num_kvcache_blocks, draft_cfg.num_kvcache_blocks = int(nb[0]), int(nb[1])
    return runner, draft_cfg


def _worker_main(model: str, kwargs: dict, world: int, rank: int, port: int, queue) -> None:
    os.environ["SSD_B200_SPAWNED_RANK"] = str(rank)
    os.environ["SSD_B200_SPAWNED_WORLD"] = str(world)
    os.environ["SSD_B200_SPAWNED_PORT"] = str(port)
    from .llm import LLM
    llm = LLM(model, **kwargs)
    while True:
        msg = queue.get()
        if msg[0] == "exit":
            break
        if msg[0] == "generate":
            llm.generate(msg[1], msg[2], use_tqdm=False, stream_callback=(lambda *a: None) if msg[3] else None)
    llm.exit()


class SpawnedWorkers:
    def __init__(self, model: str, kwargs: dict, world: int, port: int):
        import torch.multiprocessing as mp
        ctx = mp.get_context("spawn")
        self.queues, self.procs = [], []
        for r in range(1, world):
            q = ctx.Queue()
            p = ctx.Process(target=_worker_main, args=(model, kwargs, world, r, port, q), daemon=True)
            p.start()
            self.queues.append(q)
            self.procs.append(p)

    def generate(self, prompts, sampling_params, streaming: bool) -> None:
        for q in self.queues:
            q.put(("generate", prompts, sampling_params, streaming))

    def close(self) -> None:
        for q in self.queues:
            q.put(("exit",))
        for p in self.procs:
            p.join(timeout=10)
            if p.is_alive():
                p.terminate()


def launch_tp_engine(config, model: str, kwargs: dict):
    """Returns (runner, draft_cfg, workers|None) for this process."""
    world = config.num_gpus
    if "SSD_B200_SPAWNED_RANK" in os.environ:  # we ARE a spawned worker
        rank = int(os.environ["SSD_B200_SPAWNED_RANK"])
        port = int(os.environ["SSD_B200_SPAWNED_PORT"])
        runner, dcfg = build_tp_rank(config, world, rank, rank, port)
        return runner, dcfg, None
    if int(os.environ.get("WORLD_SIZE", "1")) == world:  # torchrun-style SPMD launch
        rank, local = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
        runner, dcfg = build_tp_rank(config, world, rank, local)
        return runner, dcfg, None
    # reference calling convention: spawn the other ranks ourselves
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    workers = SpawnedWorkers(model, kwargs, world, port)
    runner, dcfg = build_tp_rank(config, world, 0, 0, port)
    return runner, dcfg, workers
