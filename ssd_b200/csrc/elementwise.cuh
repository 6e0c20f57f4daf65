// elementwise.cuh — the HBM/launch-bound glue between GEMMs: embedding + RMSNorm(+residual),
// per-head norm + RoPE + KV-cache scatter, SiLU*mul, and the per-forward index prep.
// Every kernel also folds in the fixed-order reduction of the producer GEMM's split-K
// partials (fp32 [S, M, N]) and the bf16 rounding the reference applies to every
// F.linear output (SURVEY §8a checklist 1).
#pragma once
#include "common.cuh"

namespace ssdk {

// A GEMM result as seen by its consumer: either a plain bf16 matrix [M, ld] or
// S split-K partials fp32 [S, M, N] to be summed (s = 0..S-1 in order) and rounded to bf16.
struct GemmOut {
  const __nv_bfloat16* dense;  // used when S == 0
  const float* partial;        // used when S >= 1
  int S;
  int M;   // rows in the partial buffer
  int N;   // row width of the partial buffer / dense ld
};

// Split-K partials are summed in the fixed order s = 0..S-1 (deterministic), but the loads are issued in
// batches of 8 so that the reduction costs ~S/8 L2 round trips instead of S.
SSDK_DEVINL float gemm_out_at(const GemmOut& g, int m, int n) {
  if (g.S == 0) return bf2f(g.dense[(size_t)m * g.N + n]);
  const float* base = g.partial + (size_t)m * g.N + n;
  const size_t stride = (size_t)g.M * g.N;
  float acc = 0.f;
  for (int s0 = 0; s0 < g.S; s0 += 8) {
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = (s0 + u < g.S) ? __ldcg(base + (size_t)(s0 + u) * stride) : 0.f;
#pragma unroll
    for (int u = 0; u < 8; ++u) acc += v[u];
  }
  return bf16_round(acc);
}
// 8 consecutive columns starting at n (n % 8 == 0).  NB = slabs requested per batch: 8 keeps 16 float4 loads
// (64 registers) in flight; callers that hold more live state per thread use 4.
template <int NB = 8>
SSDK_DEVINL void gemm_out_at8(const GemmOut& g, int m, int n, float* f) {
  if (g.S == 0) {
    uint4 v = *reinterpret_cast<const uint4*>(g.dense + (size_t)m * g.N + n);
    unpack_bf16x8(v, f);
    return;
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = 0.f;
  const float* base = g.partial + (size_t)m * g.N + n;
  const size_t stride = (size_t)g.M * g.N;
  for (int s0 = 0; s0 < g.S; s0 += NB) {
    float4 a[NB], b[NB];
#pragma unroll
    for (int u = 0; u < NB; ++u) {
      if (s0 + u < g.S) {
        const float4* p = reinterpret_cast<const float4*>(base + (size_t)(s0 + u) * stride);
        a[u] = __ldcg(p);
        b[u] = __ldcg(p + 1);
      } else {
        a[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        b[u] = a[u];
      }
    }
#pragma unroll
    for (int u = 0; u < NB; ++u) {
      f[0] += a[u].x; f[1] += a[u].y; f[2] += a[u].z; f[3] += a[u].w;
      f[4] += b[u].x; f[5] += b[u].y; f[6] += b[u].z; f[7] += b[u].w;
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = bf16_round(f[i]);
}

// two 2-column groups (cols a, a+1 and b, b+1; a, b even) with every load of a batch in flight together
SSDK_DEVINL void gemm_out_at2x2(const GemmOut& g, int m, int a, int b, float* fa, float* fb) {
  if (g.S == 0) {
    const float2 va = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(g.dense + (size_t)m * g.N + a));
    const float2 vb = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(g.dense + (size_t)m * g.N + b));
    fa[0] = va.x; fa[1] = va.y; fb[0] = vb.x; fb[1] = vb.y;
    return;
  }
  fa[0] = fa[1] = fb[0] = fb[1] = 0.f;
  const float* base = g.partial + (size_t)m * g.N;
  const size_t stride = (size_t)g.M * g.N;
  for (int s0 = 0; s0 < g.S; s0 += 8) {
    float2 va[8], vb[8];
    // unconditional loads from a clamped slab index (straight-line code: all 16 requests are in flight together), the
    // out-of-range copies are dropped by the selects below
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const float* row = base + (size_t)min(s0 + u, g.S - 1) * stride;
      va[u] = __ldcg(reinterpret_cast<const float2*>(row + a));
      vb[u] = __ldcg(reinterpret_cast<const float2*>(row + b));
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const bool in = s0 + u < g.S;
      fa[0] += in ? va[u].x : 0.f; fa[1] += in ? va[u].y : 0.f;
      fb[0] += in ? vb[u].x : 0.f; fb[1] += in ? vb[u].y : 0.f;
    }
  }
  fa[0] = bf16_round(fa[0]); fa[1] = bf16_round(fa[1]); fb[0] = bf16_round(fb[0]); fb[1] = bf16_round(fb[1]);
}

// ----------------------------------------------------------------------------------
// prep: positions / slot_mapping / context_lens for one forward of `batch` sequences
// with q_len tokens each, token j of sequence b at position ctx0[b] + pos_offset + j.
// Mirrors prepare_decode_tensors_from_seqs (helpers/runner_helpers.py:50-108) on device.
// pend (may be null): token 0 of sequence b gets slot -1 (no K/V store) unless pend[b] >= 0 — the two-row first draft
// forward of a spec step, whose row 0 writes the K/V of a pending token only.
// ----------------------------------------------------------------------------------
__global__ void prep_kernel(const int32_t* __restrict__ ctx0, const int32_t* __restrict__ block_tables,
                            int max_blocks, int block_size, int batch, int q_len, int pos_offset,
                            const int64_t* __restrict__ pend,
                            int64_t* __restrict__ positions, int32_t* __restrict__ slot_mapping,
                            int32_t* __restrict__ context_lens, unsigned* __restrict__ fwd_seq) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) trace_mark(TR_PREP);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < batch * q_len) {
    const int b = i / q_len, j = i - b * q_len;
    const int pos = ctx0[b] + pos_offset + j;
    positions[i] = pos;
    const int blk = block_tables[(size_t)b * max_blocks + pos / block_size];
    const bool masked = pend && j == 0 && pend[b] < 0;
    slot_mapping[i] = (blk < 0 || masked) ? -1 : blk * block_size + pos % block_size;
  }
  if (i < batch) context_lens[i] = ctx0[i] + pos_offset + q_len;
  if (fwd_seq && i == 0) *fwd_seq += 1u;  // epoch base of this forward's one-shot all-reduces (tensor parallel target)
}

// prep_kernel for a varlen forward: sequence b owns packed rows cu_q[b] .. cu_q[b+1]-1, appended at ctx0[b].
// One CTA of kMaxTokens threads, one per row.
__global__ void prep_varlen_kernel(const int32_t* __restrict__ ctx0, const int32_t* __restrict__ cu_q,
                                   const int32_t* __restrict__ block_tables, int max_blocks, int block_size, int batch,
                                   int64_t* __restrict__ positions, int32_t* __restrict__ slot_mapping,
                                   int32_t* __restrict__ context_lens, unsigned* __restrict__ fwd_seq) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) trace_mark(TR_PREP);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cu_q[batch]) {
    int b = 0;
    while (cu_q[b + 1] <= i) ++b;
    const int pos = ctx0[b] + i - cu_q[b];
    positions[i] = pos;
    const int blk = block_tables[(size_t)b * max_blocks + pos / block_size];
    slot_mapping[i] = (blk < 0) ? -1 : blk * block_size + pos % block_size;
  }
  if (i < batch) context_lens[i] = ctx0[i] + cu_q[i + 1] - cu_q[i];
  if (fwd_seq && i == 0) *fwd_seq += 1u;
}

// ----------------------------------------------------------------------------------
// (embedding gather |) (split-K reduce |) residual add + RMSNorm.   grid = M rows.
//   x row      = embed[ids[m*ids_stride] - vocab_start]  (ids != nullptr; rows outside the
//                local vocab shard contribute zeros — VocabParallelEmbedding, embed_head.py:49-58)
//              | GEMM output (dense or partials)
//   r          = x + residual_in            (fp32; residual_in may be null: r = x)
//   residual_out = bf16(r)
//   y          = bf16(r * rsqrt(mean(r^2) + eps) * w)        (layers/layernorm.py:64-88, compiled form)
// ----------------------------------------------------------------------------------
// One-shot, low-latency ("LL") all-reduce input (tensor parallel).  Every rank's bf16 contribution sits in THIS
// rank's symmetric buffer as 8-byte words {2 x bf16, flag}: ar_publish_kernel pushes them over NVLink with plain
// vector stores (an aligned 8-byte store is atomic, so data and flag become visible together — no fence, no separate
// signal), and the consumer simply re-reads a word until its flag equals the expected epoch.  The epoch is
// (target-forward sequence number) * 512 + (static index of the all-reduce inside the forward) + 1, so it needs no
// cross-kernel bookkeeping and a static CUDA graph can replay it.  Slots are double-buffered by a parity that runs on
// across forwards (symm_parity_of, common.cuh); a rank cannot run two all-reduces ahead of a peer because it needs that
// peer's words of the previous one first.
struct SymmIn {
  const uint8_t* base;      // this rank's symmetric buffer; nullptr = not used
  const unsigned* fwd_seq;  // local: sequence number of the current target forward
  int no_dep_wait;          // 1: the consumer may skip griddepcontrol.wait (see add_rmsnorm_kernel)
  int call_idx;             // static index of this all-reduce inside the forward
  int n_calls;              // all-reduces per forward (slot parity runs on across forwards, see symm_parity_of)
  int n_ranks;
  unsigned slot_bytes;
};
constexpr int kSymmMaxRanks = 8;
// NOTE (robustness item for the next round): fwd_seq is bumped by prep_kernel at the START of the forward.  A dataflow
// consumer reads it without a grid-dependency wait, i.e. formally it could run before prep_kernel has finished if the
// whole PDL chain (>= 9 launches) were co-resident and launched within prep's ~2 us — impossible at model shapes
// (the GEMM grids serialise the chain) and never observed, but not excluded by construction.  Moving the bump into a
// one-thread kernel after the forward's last consumer makes it stable long before the next forward starts.
SSDK_DEVINL size_t symm_slot_off(unsigned parity, int rank, unsigned slot_bytes) {
  return ((size_t)parity * kSymmMaxRanks + rank) * slot_bytes;
}

struct NormParams {
  GemmOut x;
  SymmIn symm;
  const int64_t* ids;
  int ids_stride;
  const __nv_bfloat16* embed;
  int vocab_start, vocab_rows;
  const __nv_bfloat16* residual_in;
  const __nv_bfloat16* w;
  float eps;
  __nv_bfloat16* y;
  __nv_bfloat16* residual_out;
  int d;
};

// One 8-element slice of the row: x = (all-reduced | embedded | GEMM) input + residual; writes the new residual.
template <int NB>
SSDK_DEVINL void norm_slice(const NormParams& p, int m, int i, const uint8_t* symm_slots, unsigned symm_e,
                            const __nv_bfloat16* erow, bool zero_row, float* x) {
  const int d = p.d;
  uint4 res = make_uint4(0, 0, 0, 0);
  // A dataflow (no grid-dependency wait) all-reduce consumer may run while kernels several steps back in the chain are
  // still executing — with small grids the whole PDL chain is co-resident — so it must not touch `residual` before it has
  // seen its own rank's flagged words (which imply that the local chain up to the publish kernel has completed).
  if (p.residual_in && !symm_slots) res = *reinterpret_cast<const uint4*>(p.residual_in + (size_t)m * d + i);
  if (symm_slots) {
    // sum the ranks' bf16 contributions in rank order (identical on every rank), fp32 accumulate, one bf16 rounding.
    // 8 elements = 4 words {2 x bf16, flag} = two 16-byte loads per rank; all ranks' loads are issued before any flag is
    // looked at, and the pass is repeated until all four flags of every rank show this epoch.
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] = 0.f;
    const size_t word0 = ((size_t)m * d + i) / 2;
    uint4 lo[kSymmMaxRanks], hi[kSymmMaxRanks];
    const long long t0 = clock64();
    bool ready = false;
    while (!ready) {
#pragma unroll
      for (int r = 0; r < kSymmMaxRanks; ++r) {
        if (r < p.symm.n_ranks) {
          const uint4* src = reinterpret_cast<const uint4*>(symm_slots + (size_t)r * p.symm.slot_bytes) + word0 / 2;
          lo[r] = ld_volatile_v4(src);
          hi[r] = ld_volatile_v4(src + 1);
        }
      }
      ready = true;
#pragma unroll
      for (int r = 0; r < kSymmMaxRanks; ++r)
        if (r < p.symm.n_ranks)
          ready = ready && lo[r].y == symm_e && lo[r].w == symm_e && hi[r].y == symm_e && hi[r].w == symm_e;
      if (!ready && clock64() - t0 > 8000000000LL) __trap();
    }
#pragma unroll
    for (int r = 0; r < kSymmMaxRanks; ++r) {
      if (r < p.symm.n_ranks) {
        const uint32_t w4[4] = {lo[r].x, lo[r].z, hi[r].x, hi[r].z};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 c = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w4[q]));
          x[2 * q] += c.x;
          x[2 * q + 1] += c.y;
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] = bf16_round(x[j]);
    asm volatile("" ::: "memory");  // keep the residual load below the polling loop
    if (p.residual_in) res = *reinterpret_cast<const uint4*>(p.residual_in + (size_t)m * d + i);
  } else if (p.ids) {
    if (zero_row) {
#pragma unroll
      for (int j = 0; j < 8; ++j) x[j] = 0.f;
    } else {
      unpack_bf16x8(*reinterpret_cast<const uint4*>(erow + i), x);
    }
  } else {
    gemm_out_at8<NB>(p.x, m, i, x);
  }
  if (p.residual_in) {
    float r[8];
    unpack_bf16x8(res, r);
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] += r[j];
  }
  if (p.residual_out) *reinterpret_cast<uint4*>(p.residual_out + (size_t)m * d + i) = pack_bf16x8(x);
}

// SLICES = 1 / 2: the row is register-resident, d <= SLICES * 8 * blockDim.x; every thread issues all the loads of a slice
// (weights, residual, <= 8 / 4 split-K slabs or all ranks' all-reduce words) before it uses any of them, so a slice costs
// one L2 round trip; the kernel is ~SLICES round trips + one block reduction.  SLICES = 0: any d, row staged in shared
// memory.  (With a single instantiation ptxas ran out of its 128 registers at 512 threads and serialised the slab loads:
// one round trip per slab, 3-4 us per call.)
template <int SLICES>
__global__ void __launch_bounds__(512) add_rmsnorm_kernel(NormParams p) {
  SSDK_DYN_SMEM(float, rbuf);  // d floats (SLICES == 0 only)
  SSDK_STATIC_SMEM(float, red, 32);
  pdl_launch_dependents();
  // All-reduce consumers after a row-parallel GEMM are pure dataflow: every input word (including THIS rank's own
  // contribution) carries the epoch flag, so the kernel does not have to wait for the publishing kernel to *complete*
  // (which would include the acknowledgement of its remote NVLink stores, ~4 us at TP=8) — it can start polling as soon
  // as it is resident.  Seeing this rank's own flagged words implies the local chain up to the publish has run, which is
  // what protects `hidden` / `residual` (read by earlier kernels of the chain) from being overwritten too early.
  if (!(p.symm.base && p.symm.no_dep_wait)) pdl_wait();
  if (threadIdx.x == 0) trace_mark(TR_NORM);
  const int m = blockIdx.x;
  const int d = p.d;
  // ---- one-shot all-reduce input: words carry their own flag, nothing to wait for up front ----
  const uint8_t* symm_slots = nullptr;
  unsigned symm_e = 0;
  if (p.symm.base) {
    const unsigned seq = __ldcg(p.symm.fwd_seq);
    symm_e = symm_epoch_of(seq, p.symm.call_idx);
    symm_slots = p.symm.base + symm_slot_off(symm_parity_of(seq, p.symm.call_idx, p.symm.n_calls), 0, p.symm.slot_bytes);
  }
  const __nv_bfloat16* erow = nullptr;
  bool zero_row = false;
  if (p.ids) {
    const long long id = p.ids[(size_t)m * p.ids_stride] - p.vocab_start;
    if (id < 0 || id >= p.vocab_rows) zero_row = true;
    else erow = p.embed + (size_t)id * d;
  }
  float ss = 0.f;
  if constexpr (SLICES > 0) {
    constexpr int NB = (SLICES == 1) ? 8 : 4;
    float xreg[SLICES][8];
    uint4 wpk[SLICES];
#pragma unroll
    for (int c = 0; c < SLICES; ++c) {
      const int i = (c * blockDim.x + threadIdx.x) * 8;
      if (i < d && p.y) wpk[c] = *reinterpret_cast<const uint4*>(p.w + i);
    }
#pragma unroll
    for (int c = 0; c < SLICES; ++c) {
      const int i = (c * blockDim.x + threadIdx.x) * 8;
      if (i < d) {
        norm_slice<NB>(p, m, i, symm_slots, symm_e, erow, zero_row, xreg[c]);
#pragma unroll
        for (int j = 0; j < 8; ++j) ss += xreg[c][j] * xreg[c][j];
      }
    }
    if (threadIdx.x == 0) trace_fine(TRF_NORM + 0);  // inputs arrived (thread 0's slices)
    ss = block_sum(ss, red);
    if (threadIdx.x == 0) trace_fine(TRF_NORM + 1);  // row statistic reduced
    const float rstd = rsqrtf(ss / (float)d + p.eps);
    if (p.y) {
#pragma unroll
      for (int c = 0; c < SLICES; ++c) {
        const int i = (c * blockDim.x + threadIdx.x) * 8;
        if (i < d) {
          float w[8], o[8];
          unpack_bf16x8(wpk[c], w);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = xreg[c][j] * rstd * w[j];
          *reinterpret_cast<uint4*>(p.y + (size_t)m * d + i) = pack_bf16x8(o);
        }
      }
    }
  } else {
    for (int i = threadIdx.x * 8; i < d; i += blockDim.x * 8) {
      float x[8];
      norm_slice<4>(p, m, i, symm_slots, symm_e, erow, zero_row, x);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        rbuf[i + j] = x[j];
        ss += x[j] * x[j];
      }
    }
    ss = block_sum(ss, red);
    const float rstd = rsqrtf(ss / (float)d + p.eps);
    if (p.y) {
      for (int i = threadIdx.x * 8; i < d; i += blockDim.x * 8) {
        float w[8], o[8];
        unpack_bf16x8(*reinterpret_cast<const uint4*>(p.w + i), w);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rbuf[i + j] * rstd * w[j];
        *reinterpret_cast<uint4*>(p.y + (size_t)m * d + i) = pack_bf16x8(o);
      }
    }
  }
  if (threadIdx.x == 0) trace_fine(TRF_NORM + 2);
}

// ----------------------------------------------------------------------------------
// ar_publish_kernel — first half of the one-shot all-reduce that replaces dist.all_reduce on the row-parallel
// boundaries (layers/linear.py:195-199, embed_head.py:56).  Each rank reduces its split-K partials (or gathers its
// masked embedding rows), rounds to bf16 exactly like the reference's per-rank F.linear output, and PUSHES the
// result as {2 x bf16, epoch} words over NVLink into slot[call parity][my_rank] of EVERY rank's symmetric buffer.
// The consumer (add_rmsnorm_kernel with SymmIn) spins on the words themselves, sums the ranks in rank order and
// continues with residual add + RMSNorm — no NCCL call, no fence, no extra pass over the data.
// ----------------------------------------------------------------------------------
struct ArPublishParams {
  GemmOut x;
  const int64_t* ids;  // embedding mode when non-null
  int ids_stride;
  const __nv_bfloat16* embed;
  int vocab_start, vocab_rows;
  int M, d, n_ranks, rank;
  uint8_t* peer[kSymmMaxRanks];
  unsigned slot_bytes;
  const unsigned* fwd_seq;
  int call_idx, n_calls;
};

__global__ void __launch_bounds__(256) ar_publish_kernel(ArPublishParams p) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) trace_mark(TR_MISC);
  const unsigned seq = __ldcg(p.fwd_seq);
  const unsigned e = symm_epoch_of(seq, p.call_idx);
  const size_t slot_off = symm_slot_off(symm_parity_of(seq, p.call_idx, p.n_calls), p.rank, p.slot_bytes);
  const int total = p.M * p.d;
  for (int idx = (blockIdx.x * blockDim.x + threadIdx.x) * 8; idx < total; idx += gridDim.x * blockDim.x * 8) {
    const int m = idx / p.d, i = idx - m * p.d;
    float x[8];
    if (p.ids) {
      const long long id = p.ids[(size_t)m * p.ids_stride] - p.vocab_start;
      if (id < 0 || id >= p.vocab_rows) {
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = 0.f;
      } else {
        unpack_bf16x8(*reinterpret_cast<const uint4*>(p.embed + (size_t)id * p.d + i), x);
      }
    } else {
      gemm_out_at8(p.x, m, i, x);
    }
    const uint4 v = pack_bf16x8(x);
    const uint4 lo = make_uint4(v.x, e, v.y, e), hi = make_uint4(v.z, e, v.w, e);
    // gridDim.y == 1: every thread pushes its words to all ranks; gridDim.y == n_ranks: CTA column y serves peer y only —
    // the (cheap, L2-resident) reduction is repeated per peer, the NVLink stores of the 8 peers are issued from 8x as many
    // SMs instead of back to back from one thread
    const int r_lo = gridDim.y > 1 ? (int)blockIdx.y : 0, r_hi = gridDim.y > 1 ? (int)blockIdx.y + 1 : p.n_ranks;
#pragma unroll
    for (int r = 0; r < kSymmMaxRanks; ++r) {
      if (r >= r_lo && r < r_hi) {
        uint4* dst = reinterpret_cast<uint4*>(p.peer[r] + slot_off) + idx / 4;
        dst[0] = lo;
        dst[1] = hi;
      }
    }
  }
}

// ----------------------------------------------------------------------------------
// (split-K reduce |) [per-head RMSNorm |] NeoX RoPE on q,k + KV-cache scatter.
// grid = (M, ceil((H+2KV)/4)), block = 128: one warp per head.
//   q,k: optional RMSHeadNorm (qwen3.py:97-103; layernorm.py:16-27 compiled form:
//        bf16(x * rsqrt(mean x^2 + eps) * w)), then
//        y1 = x1*cos - x2*sin, y2 = x2*cos + x1*sin in fp32 -> bf16 (rotary_embedding.py:6-17)
//   k,v rows go to cache slot slot_mapping[m] (skip -1)  (attention.py:10-41)
// ----------------------------------------------------------------------------------
struct RopeParams {
  GemmOut qkv;
  const int64_t* positions;
  const int32_t* slot_mapping;
  const float* rope_table;  // [max_pos, hd]: cos[0:hd/2] | sin[0:hd/2]
  const __nv_bfloat16* q_norm_w;
  const __nv_bfloat16* k_norm_w;
  float norm_eps;
  __nv_bfloat16* q_out;    // [M, H*hd]
  __nv_bfloat16* k_cache;  // [slots, KV*hd]  (KV8: e4m3 codes, one byte per element)
  __nv_bfloat16* v_cache;
  int heads, kv_heads, head_dim;
  float k_scale, v_scale;  // KV8 only: the layer's cache scales
};

// KV8: one k or v element pair, code = e4m3_rne(sat(y / s)) of the bf16 value y the bf16 instance stores (IEEE division)
SSDK_DEVINL void store_kv8_pair(uint8_t* dst, float a, float b, float s) {
  *reinterpret_cast<uint16_t*>(dst) = float2_to_e4m3x2(bf16_round(a) / s, bf16_round(b) / s);
}

// HD is a template parameter so that the per-lane element pairs are static registers (a run-time head_dim turned the
// x1/x2 arrays into local memory and made ptxas recycle the load registers, i.e. one L2 round trip per split-K slab).
// KV8: k and v go to the cache as e4m3 codes (store_kv8_pair); q is stored as in the bf16 instance.
template <int HD, bool KV8 = false>
__global__ void __launch_bounds__(128) rope_store_kernel(RopeParams p) {
  constexpr int HALF = HD / 2;
  constexpr int NP = (HALF + 63) / 64;  // (i, i+1) / (i + HALF, i + HALF + 1) pairs per lane, i = 2 * lane + 64 * t
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) trace_mark(TR_ROPE);
  const int m = blockIdx.x;
  const int head = blockIdx.y * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int H = p.heads, KV = p.kv_heads;
  if (head >= H + 2 * KV) return;
  const int kind = head < H ? 0 : (head < H + KV ? 1 : 2);  // q, k, v
  const int col0 = head * HD;
  // the slot, the position and the projection values are requested together; nothing below waits for one of them
  // before the others are in flight
  const int slot = p.slot_mapping[m];
  const long long pos = p.positions[m];

  float x1[NP][2], x2[NP][2];
  float ss = 0.f;
#pragma unroll
  for (int t = 0; t < NP; ++t) {
    const int i = 2 * lane + 64 * t;
    if (i < HALF) {
      gemm_out_at2x2(p.qkv, m, col0 + i, col0 + HALF + i, x1[t], x2[t]);
      ss += x1[t][0] * x1[t][0] + x1[t][1] * x1[t][1] + x2[t][0] * x2[t][0] + x2[t][1] * x2[t][1];
    } else {
      x1[t][0] = x1[t][1] = x2[t][0] = x2[t][1] = 0.f;
    }
  }
  if (kind != 0 && slot < 0) return;
  if (kind == 2 && KV8) {
    uint8_t* dst = reinterpret_cast<uint8_t*>(p.v_cache) + ((size_t)slot * KV + (head - H - KV)) * HD;
#pragma unroll
    for (int t = 0; t < NP; ++t) {
      const int i = 2 * lane + 64 * t;
      if (i < HALF) {
        store_kv8_pair(dst + i, x1[t][0], x1[t][1], p.v_scale);
        store_kv8_pair(dst + HALF + i, x2[t][0], x2[t][1], p.v_scale);
      }
    }
    return;
  }
  if (kind == 2) {
    __nv_bfloat16* dst = p.v_cache + ((size_t)slot * KV + (head - H - KV)) * HD;
#pragma unroll
    for (int t = 0; t < NP; ++t) {
      const int i = 2 * lane + 64 * t;
      if (i < HALF) {
        *reinterpret_cast<__nv_bfloat162*>(dst + i) = __floats2bfloat162_rn(x1[t][0], x1[t][1]);
        *reinterpret_cast<__nv_bfloat162*>(dst + HALF + i) = __floats2bfloat162_rn(x2[t][0], x2[t][1]);
      }
    }
    return;
  }
  if (threadIdx.x == 0) trace_fine(TRF_ROPE + 0);  // projection row reduced from the partials
  const __nv_bfloat16* nw = (kind == 0) ? p.q_norm_w : p.k_norm_w;
  if (nw) {
    ss = warp_sum(ss);
    const float rstd = rsqrtf(ss / (float)HD + p.norm_eps);
#pragma unroll
    for (int t = 0; t < NP; ++t) {
      const int i = 2 * lane + 64 * t;
      if (i < HALF) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          x1[t][e] = bf16_round(x1[t][e] * rstd * bf2f(nw[i + e]));
          x2[t][e] = bf16_round(x2[t][e] * rstd * bf2f(nw[HALF + i + e]));
        }
      }
    }
  }
  const float* cs = p.rope_table + (size_t)pos * HD;
  if (KV8 && kind == 1) {
    uint8_t* dst = reinterpret_cast<uint8_t*>(p.k_cache) + ((size_t)slot * KV + (head - H)) * HD;
#pragma unroll
    for (int t = 0; t < NP; ++t) {
      const int i = 2 * lane + 64 * t;
      if (i < HALF) {
        const float2 c = *reinterpret_cast<const float2*>(cs + i), sn = *reinterpret_cast<const float2*>(cs + HALF + i);
        store_kv8_pair(dst + i, x1[t][0] * c.x - x2[t][0] * sn.x, x1[t][1] * c.y - x2[t][1] * sn.y, p.k_scale);
        store_kv8_pair(dst + HALF + i, x2[t][0] * c.x + x1[t][0] * sn.x, x2[t][1] * c.y + x1[t][1] * sn.y, p.k_scale);
      }
    }
    if (threadIdx.x == 0) trace_fine(TRF_ROPE + 1);
    return;
  }
  __nv_bfloat16* dst = (kind == 0) ? p.q_out + (size_t)m * H * HD + (size_t)head * HD
                                   : p.k_cache + ((size_t)slot * KV + (head - H)) * HD;
#pragma unroll
  for (int t = 0; t < NP; ++t) {
    const int i = 2 * lane + 64 * t;
    if (i < HALF) {
      const float2 c = *reinterpret_cast<const float2*>(cs + i), sn = *reinterpret_cast<const float2*>(cs + HALF + i);
      *reinterpret_cast<__nv_bfloat162*>(dst + i) =
          __floats2bfloat162_rn(x1[t][0] * c.x - x2[t][0] * sn.x, x1[t][1] * c.y - x2[t][1] * sn.y);
      *reinterpret_cast<__nv_bfloat162*>(dst + HALF + i) =
          __floats2bfloat162_rn(x2[t][0] * c.x + x1[t][0] * sn.x, x2[t][1] * c.y + x1[t][1] * sn.y);
    }
  }
  if (threadIdx.x == 0) trace_fine(TRF_ROPE + 1);
}

// ----------------------------------------------------------------------------------
// SiLU(gate) * up for the split-K (non-fused-epilogue) gate|up GEMM and the stand-alone op.
// x: [M, 2*ffn] (dense or partials) -> out bf16 [M, ffn]
// ----------------------------------------------------------------------------------
__global__ void silu_mul_kernel(GemmOut x, __nv_bfloat16* __restrict__ out, int M, int ffn) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) trace_mark(TR_MISC);
  const int idx = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (idx >= M * ffn) return;
  const int m = idx / ffn, n = idx - m * ffn;
  float g[8], u[8], h[8];
  gemm_out_at8(x, m, n, g);
  gemm_out_at8(x, m, ffn + n, u);
#pragma unroll
  for (int j = 0; j < 8; ++j) h[j] = (g[j] / (1.0f + __expf(-g[j]))) * u[j];
  *reinterpret_cast<uint4*>(out + (size_t)m * ffn + n) = pack_bf16x8(h);
}

// gather `rows` rows (the last token of each sequence) of a [M, d] matrix: out[b] = x[b*q_len + q_len-1]
__global__ void gather_last_rows_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ out, int batch,
                                        int q_len, int d) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) trace_mark(TR_MISC);
  const int b = blockIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(x + ((size_t)b * q_len + q_len - 1) * d);
  uint4* dst = reinterpret_cast<uint4*>(out + (size_t)b * d);
  for (int i = threadIdx.x; i < d / 8; i += blockDim.x) dst[i] = src[i];
}

// varlen forward: the last row of sequence b is packed row cu_q[b+1] - 1
__global__ void gather_last_rows_varlen_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ out,
                                               const int32_t* __restrict__ cu_q, int d) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) trace_mark(TR_MISC);
  const int b = blockIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(x + (size_t)(cu_q[b + 1] - 1) * d);
  uint4* dst = reinterpret_cast<uint4*>(out + (size_t)b * d);
  for (int i = threadIdx.x; i < d / 8; i += blockDim.x) dst[i] = src[i];
}

}  // namespace ssdk
