"""PairRunner — host-side owner of the device state behind one ssdk handle.

Plays the role of the reference's ModelRunner (+ the in-process sync DraftRunner) for the hot path
(engine/model_runner.py:39-157,446-503; engine/draft_runner.py:27-38): it keeps the torch tensors
(weights in the reference's packed per-rank layout, the paged KV caches, the workspace) alive,
hands their raw pointers to libssdk and exposes the three calls the engine needs:

    prefill / decode   -> ssdk_forward_tokens   (ModelRunner.run with is_prefill / last_only)
    spec_step          -> ssdk_spec_step        (SpeculatorSync.speculate + Verifier.verify, one call)

PyTorch is plumbing only (allocation, streams); every FLOP of the path runs in libssdk.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import lib as L


@dataclass
class ModelSpec:
    """The HF-config fields the reference reads (models/llama3.py:157-183, models/qwen3.py:163-193)."""
    hidden: int
    layers: int
    heads: int
    kv_heads: int
    head_dim: int
    ffn: int
    vocab: int
    rms_eps: float = 1e-5
    rope_theta: float = 500000.0
    qk_norm: bool = False
    tie_embed: bool = False
    max_pos: int = 8192

    @classmethod
    def from_hf(cls, cfg) -> "ModelSpec":
        hd = getattr(cfg, "head_dim", None) or cfg.hidden_size // cfg.num_attention_heads
        theta = getattr(cfg, "rope_theta", None)
        if theta is None:
            rp = getattr(cfg, "rope_parameters", None) or {}
            theta = rp.get("rope_theta", 1000000.0 if "qwen" in cfg.model_type else 500000.0)
        return cls(hidden=cfg.hidden_size, layers=cfg.num_hidden_layers, heads=cfg.num_attention_heads,
                   kv_heads=cfg.num_key_value_heads, head_dim=hd, ffn=cfg.intermediate_size, vocab=cfg.vocab_size,
                   rms_eps=cfg.rms_norm_eps, rope_theta=float(theta), qk_norm=("qwen3" in cfg.model_type),
                   tie_embed=bool(getattr(cfg, "tie_word_embeddings", False)),
                   max_pos=cfg.max_position_embeddings)


def rope_table(head_dim: int, rows: int, base: float, device) -> torch.Tensor:
    """RotaryEmbedding.__init__ (layers/rotary_embedding.py:30-37); rope_scaling is dropped like the reference
    does (models/llama3.py:65-67).  Only `rows` <= max_model_len positions are materialised."""
    inv_freq = 1.0 / (base ** (torch.arange(0, head_dim, 2, dtype=torch.float, device=device) / head_dim))
    t = torch.arange(rows, dtype=torch.float, device=device)
    freqs = torch.einsum("i,j -> ij", t, inv_freq)
    return torch.cat((freqs.cos(), freqs.sin()), dim=-1).contiguous()


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


class PairRunner:
    def __init__(self, target: ModelSpec, draft: ModelSpec | None, *, spec_k: int, max_batch: int = 1,
                 block_size: int = 256, max_model_len: int = 4096, num_blocks_target: int | None = None,
                 num_blocks_draft: int | None = None, device: str | torch.device = "cuda:0", use_graph: bool = True,
                 use_pdl: bool = False, jit_speculate: bool = True, tp_size: int = 1, tp_rank: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("PairRunner needs a CUDA device: libssdk has no CPU path")
        self.lib = L.load()
        self.device = torch.device(device)
        torch.cuda.set_device(self.device)
        self.spec = {L.TARGET: target, L.DRAFT: draft}
        self.K, self.max_batch, self.block_size = spec_k, max_batch, block_size
        self.max_blocks = (max_model_len + block_size - 1) // block_size
        self.max_model_len = max_model_len
        self.tp_size, self.tp_rank = tp_size, tp_rank
        self._keep: list[torch.Tensor] = []  # tensors whose pointers libssdk holds
        self.weights: dict[int, dict] = {}

        def cfg(m: ModelSpec, tp: int, rank: int) -> L.ModelCfg:
            return L.ModelCfg(m.hidden, m.layers, m.heads, m.kv_heads, m.head_dim, m.ffn, m.vocab, int(m.qk_norm),
                              m.rms_eps, self.max_blocks * block_size, tp, rank)

        tcfg = cfg(target, tp_size, tp_rank)
        dcfg = cfg(draft, 1, 0) if draft is not None else None
        rt = L.RuntimeCfg(spec_k, max_batch, block_size, self.max_blocks, int(use_graph),
                          int(use_pdl), int(jit_speculate), 0)
        h = C.c_void_p()
        L.check(self.lib.ssdk_create(C.byref(tcfg), C.byref(dcfg) if dcfg is not None else None, C.byref(rt),
                                     C.byref(h)), "ssdk_create")
        self.h = h
        # KV caches: [2, L, num_blocks, block_size, KV/tp, hd] (engine/model_runner.py:484-491)
        self.kv = {}
        for which, m, nb, tp in ((L.TARGET, target, num_blocks_target, tp_size), (L.DRAFT, draft, num_blocks_draft, 1)):
            if m is None:
                continue
            nb = nb or max_batch * self.max_blocks
            kv = torch.zeros(2, m.layers, nb, block_size, m.kv_heads // tp, m.head_dim, dtype=torch.bfloat16,
                             device=self.device)
            self.kv[which] = kv
            L.check(self.lib.ssdk_bind_kv_cache(self.h, which, kv.data_ptr(), nb), "ssdk_bind_kv_cache")
            table = rope_table(m.head_dim, self.max_blocks * block_size, m.rope_theta, self.device)
            self._keep.append(table)
            L.check(self.lib.ssdk_bind_weight(self.h, which, L.W_ROPE_TABLE, 0, table.data_ptr(), table.shape[0],
                                              table.shape[1]), "bind rope table")
        nbytes = self.lib.ssdk_workspace_bytes(self.h)
        if nbytes <= 0:
            raise RuntimeError("ssdk_workspace_bytes failed: " + L.last_error())
        self.workspace = torch.zeros(nbytes + 1024, dtype=torch.uint8, device=self.device)
        off = (-self.workspace.data_ptr()) % 1024
        L.check(self.lib.ssdk_bind_workspace(self.h, self.workspace.data_ptr() + off, nbytes), "ssdk_bind_workspace")
        self.finalized = False
        self.step_id = 0

    # ------------------------------------------------------------------ weights
    def bind_weights(self, which: int, w: dict) -> None:
        """w: packed per-rank tensors on this device (bf16):
        embed, lm_head, final_norm, layers[l] = {input_norm, qkv, o, post_norm, gate_up, down[, q_norm, k_norm]}."""
        lib, h = self.lib, self.h

        def bind(kind, layer, t):
            if t.dtype != torch.bfloat16 or not t.is_cuda or not t.is_contiguous():
                raise ValueError("weights must be contiguous bf16 CUDA tensors")
            rows, cols = (t.shape[0], t.shape[1]) if t.dim() == 2 else (t.shape[0], 1)
            L.check(lib.ssdk_bind_weight(h, which, kind, layer, t.data_ptr(), rows, cols), f"bind kind={kind} layer={layer}")

        bind(L.W_EMBED, 0, w["embed"])
        bind(L.W_LM_HEAD, 0, w["lm_head"])
        bind(L.W_FINAL_NORM, 0, w["final_norm"])
        for l, lw in enumerate(w["layers"]):
            bind(L.W_INPUT_NORM, l, lw["input_norm"])
            bind(L.W_QKV, l, lw["qkv"])
            bind(L.W_O, l, lw["o"])
            bind(L.W_POST_NORM, l, lw["post_norm"])
            bind(L.W_GATE_UP, l, lw["gate_up"])
            bind(L.W_DOWN, l, lw["down"])
            if "q_norm" in lw:
                bind(L.W_Q_NORM, l, lw["q_norm"])
                bind(L.W_K_NORM, l, lw["k_norm"])
        self.weights[which] = w

    def set_nccl_comm(self, comm_ptr: int) -> None:
        L.check(self.lib.ssdk_set_nccl_comm(self.h, C.c_void_p(comm_ptr)), "ssdk_set_nccl_comm")

    def finalize(self) -> None:
        L.check(self.lib.ssdk_finalize(self.h, torch.cuda.current_stream().cuda_stream), "ssdk_finalize")
        self.finalized = True

    # ------------------------------------------------------------------ calls
    def _bt(self, block_tables) -> np.ndarray:
        """list[list[int]] -> int32 [B, max_blocks] padded with -1 (helpers/runner_helpers.py:110-121)."""
        B = len(block_tables)
        out = np.full((B, self.max_blocks), -1, dtype=np.int32)
        for b, t in enumerate(block_tables):
            out[b, :len(t)] = t
        return out

    def forward_tokens(self, which: int, ids: list[list[int]], ctx_len: list[int], block_tables, temps=None,
                       want_sample: bool = True, seed: int = 0) -> list[int] | None:
        """ModelRunner.run for q_len tokens per sequence appended at ctx_len (prefill chunk or AR decode)."""
        if self.spec[which] is None:
            return None  # the draft replica lives on TP rank 0 only (SURVEY §8e); other ranks have nothing to do
        B, Q = len(ids), len(ids[0])
        assert all(len(x) == Q for x in ids)
        ids_a = np.ascontiguousarray(np.array(ids, dtype=np.int64).reshape(-1))
        ctx_a, bt_a = _i32(ctx_len), self._bt(block_tables)
        temps_a = np.ascontiguousarray(temps if temps is not None else [0.0] * B, dtype=np.float32)
        out = np.zeros(B, dtype=np.int64)
        st = torch.cuda.current_stream().cuda_stream
        L.check(self.lib.ssdk_forward_tokens(self.h, which, B, Q, ids_a.ctypes.data_as(L.c_i64p),
                                             ctx_a.ctypes.data_as(L.c_i32p), bt_a.ctypes.data_as(L.c_i32p),
                                             int(want_sample), temps_a.ctypes.data_as(L.c_f32p), seed, self.step_id,
                                             out.ctypes.data_as(L.c_i64p), st), "ssdk_forward_tokens")
        self.step_id += 1
        return out.tolist() if want_sample else None

    def prefill(self, which: int, tokens: list[int], block_table: list[int], start: int = 0, temp: float = 0.0,
                want_sample: bool = True, chunk: int = 256, seed: int = 0):
        """Prefill one sequence from position `start` in chunks of <= 256 tokens through the multi-query path: the
        weights are streamed once per chunk (UMMA N = 128 / 256 instances of the wgmma GEMM), attention is the paged
        multi-query kernel with one q tile per 4-32 query rows (layers/attention.py:85-93 semantics: causal over the
        cache, which already holds the earlier chunks)."""
        tok = None
        pos = start
        n = len(tokens)
        while pos < n:
            q = min(chunk, n - pos)
            last = pos + q == n
            tok = self.forward_tokens(which, [tokens[pos:pos + q]], [pos], [block_table], [temp],
                                      want_sample=(want_sample and last), seed=seed)
            pos += q
        return tok[0] if tok else None

    @staticmethod
    def plan_prefill_call(remaining: list[int], max_tokens: int, max_batch: int) -> tuple[list[int], int]:
        """Pick the sequences and the (uniform) chunk length of the next prefill call: among the groups made of the nb
        sequences with the most tokens left, the one that covers the most tokens under nb * q <= max_tokens.  Equal-length
        prompts (the reference bench: 16 x 128 tokens) pack two to a 256-token call; ragged ones degrade to one at a time."""
        order = sorted((i for i, r in enumerate(remaining) if r > 0), key=lambda i: (-remaining[i], i))
        best, best_q = [], 0
        for nb in range(1, min(len(order), max_batch) + 1):
            q = min(max_tokens // nb, remaining[order[nb - 1]])
            if q < 1:
                break
            if nb * q > len(best) * best_q:
                best, best_q = order[:nb], q
        return sorted(best), best_q

    def prefill_many(self, which: int, tokens: list[list[int]], block_tables: list[list[int]], starts: list[int],
                     temps: list[float] | None = None, want_sample: bool = True, chunk: int = 256, seed: int = 0):
        """Prefill several sequences (runner_helpers.py:123-180 batches them by cu_seqlens): every call carries up to
        `chunk` tokens of up to max_batch sequences, the same number of tokens from each (plan_prefill_call), through the
        multi-query path; a sequence's first token is sampled by the call that holds its last prompt token.  Returns one
        token per sequence (None without want_sample)."""
        n = len(tokens)
        pos = list(starts)
        temps = list(temps) if temps is not None else [0.0] * n
        out: list[int | None] = [None] * n
        # A prefix-cache hit (start > 0) reads pages that an EARLIER sequence of the same batch may still be writing
        # (block_manager hashes a block when it is allocated, the reference stores the whole batch's K/V before any
        # attention runs): only sequences that compute their whole prompt share calls; the hits follow one by one, in order.
        packed = [i for i in range(n) if starts[i] == 0]
        while True:
            idx, q = self.plan_prefill_call([len(tokens[i]) - pos[i] if i in packed else 0 for i in range(n)],
                                            min(chunk, 256), self.max_batch)
            if not idx:
                break
            done = [pos[i] + q == len(tokens[i]) for i in idx]
            toks = self.forward_tokens(which, [tokens[i][pos[i]:pos[i] + q] for i in idx], [pos[i] for i in idx],
                                       [block_tables[i] for i in idx], [temps[i] for i in idx],
                                       want_sample=(want_sample and any(done)), seed=seed)
            for j, i in enumerate(idx):
                pos[i] += q
                if done[j] and toks is not None:
                    out[i] = toks[j]
        for i in range(n):
            if starts[i] != 0:
                out[i] = self.prefill(which, tokens[i], block_tables[i], start=starts[i], temp=temps[i],
                                      want_sample=want_sample, chunk=chunk, seed=seed)
        return out if want_sample else None

    def spec_step(self, ctx_len: list[int], recovery: list[int], bt_target, bt_draft, temps_t: list[float],
                  temps_q: list[float], seed: int = 0):
        """One sync speculative step.  Returns (speculations [B,K+1], n_accept [B], recovery [B]) as numpy."""
        B, K = len(ctx_len), self.K
        ctx_a, rec_a = _i32(ctx_len), np.ascontiguousarray(recovery, dtype=np.int64)
        btt, btd = self._bt(bt_target), self._bt(bt_draft)
        tt, tq = np.ascontiguousarray(temps_t, dtype=np.float32), np.ascontiguousarray(temps_q, dtype=np.float32)
        toks = np.zeros((B, K + 1), dtype=np.int64)
        nacc = np.zeros(B, dtype=np.int32)
        rec = np.zeros(B, dtype=np.int64)
        st = torch.cuda.current_stream().cuda_stream
        L.check(self.lib.ssdk_spec_step(self.h, B, ctx_a.ctypes.data_as(L.c_i32p), rec_a.ctypes.data_as(L.c_i64p),
                                        btt.ctypes.data_as(L.c_i32p), btd.ctypes.data_as(L.c_i32p),
                                        tt.ctypes.data_as(L.c_f32p), tq.ctypes.data_as(L.c_f32p), seed, self.step_id,
                                        toks.ctypes.data_as(L.c_i64p), nacc.ctypes.data_as(L.c_i32p),
                                        rec.ctypes.data_as(L.c_i64p), st), "ssdk_spec_step")
        self.step_id += 1
        return toks, nacc, rec

    # resident (device-driven) mode used by bench.py's kernel-only measurement
    def stage(self, ctx_len, recovery, bt_target, bt_draft, temps_t, temps_q, seed: int = 0):
        B = len(ctx_len)
        ctx_a, rec_a = _i32(ctx_len), np.ascontiguousarray(recovery, dtype=np.int64)
        btt, btd = self._bt(bt_target), self._bt(bt_draft)
        tt, tq = np.ascontiguousarray(temps_t, dtype=np.float32), np.ascontiguousarray(temps_q, dtype=np.float32)
        st = torch.cuda.current_stream().cuda_stream
        L.check(self.lib.ssdk_spec_step_stage(self.h, B, ctx_a.ctypes.data_as(L.c_i32p), rec_a.ctypes.data_as(L.c_i64p),
                                              btt.ctypes.data_as(L.c_i32p), btd.ctypes.data_as(L.c_i32p),
                                              tt.ctypes.data_as(L.c_f32p), tq.ctypes.data_as(L.c_f32p), seed,
                                              self.step_id, st), "ssdk_spec_step_stage")

    def step_resident(self, batch: int) -> None:
        L.check(self.lib.ssdk_spec_step_resident(self.h, batch, torch.cuda.current_stream().cuda_stream),
                "ssdk_spec_step_resident")

    def fetch(self, batch: int):
        K = self.K
        toks = np.zeros((batch, K + 1), dtype=np.int64)
        total = np.zeros(batch, dtype=np.int32)
        rec = np.zeros(batch, dtype=np.int64)
        L.check(self.lib.ssdk_spec_step_fetch(self.h, batch, toks.ctypes.data_as(L.c_i64p), total.ctypes.data_as(L.c_i32p),
                                              rec.ctypes.data_as(L.c_i64p), torch.cuda.current_stream().cuda_stream),
                "ssdk_spec_step_fetch")
        return toks, total, rec

    def resident_log(self, seq: int = 0, cap: int = 16384) -> list[int]:
        """Tokens sequence `seq` emitted in resident mode since stage() (recovery + accepted drafts of every step)."""
        out = np.zeros(cap, dtype=np.int64)
        n = self.lib.ssdk_spec_step_log(self.h, seq, out.ctypes.data_as(L.c_i64p), cap, torch.cuda.current_stream().cuda_stream)
        if n < 0:
            raise RuntimeError("ssdk_spec_step_log failed: " + L.last_error())
        return out[:n].tolist()

    # debug taps (parity tests compare these with the oracle's logits)
    def logits_p(self, batch: int) -> torch.Tensor:
        return _from_ptr(self.lib.ssdk_logits_p(self.h), (batch, self.K + 1, self.spec[L.TARGET].vocab), self.device)

    def logits_q(self, batch: int) -> torch.Tensor:
        return _from_ptr(self.lib.ssdk_logits_q(self.h), (batch, self.K, self.spec[L.TARGET].vocab), self.device)

    def logits_last(self, batch: int, which: int = L.TARGET) -> torch.Tensor:
        return _from_ptr(self.lib.ssdk_logits_last(self.h), (batch, self.spec[which].vocab), self.device)

    def step_io_bytes(self) -> tuple[int, int]:
        """(H2D, D2H) bytes ssdk_spec_step moves per call: the step block and the result block
        (layout_step() in csrc/engine.cu; every field 16-byte aligned)."""
        a = lambda n: (n + 15) // 16 * 16
        MB, mbk, K = self.max_batch, self.max_blocks, self.K
        h2d = a(MB * 4) + a(MB * 8) + 2 * a(MB * 4) + 16 + 2 * a(MB * mbk * 4)
        d2h = a(a(MB * (K + 1) * 8) + a(MB * 4) + MB * 8)
        return h2d, d2h

    @property
    def launch_count(self) -> int:
        return int(self.lib.ssdk_launch_count(self.h))

    def close(self) -> None:
        if getattr(self, "h", None):
            self.lib.ssdk_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _from_ptr(ptr: int, shape, device) -> torch.Tensor:
    """View `ptr` (inside the workspace tensor we own) as a bf16 tensor, returned as a copy."""
    n = int(np.prod(shape))

    class _Holder:
        pass

    holder = _Holder()
    holder.__cuda_array_interface__ = {"shape": (n,), "typestr": "<u2", "data": (int(ptr), False), "version": 3}
    t = torch.as_tensor(holder, device=device)
    return t.view(torch.bfloat16).view(*shape).clone()
