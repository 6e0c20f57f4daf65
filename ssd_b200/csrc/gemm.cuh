// gemm.cuh — weight-streaming small-M GEMM on Hopper warpgroup MMA (wgmma, sm_90a).
//
//   Y[M, N] = X[M, K] · W[N, K]^T        M <= 64 tokens, bf16 in, fp32 accumulate, bf16 out
//
// Replaces every F.linear on the decode/verify path of the reference
// (layers/linear.py:98,196; layers/embed_head.py:95,111).  With M <= 7 the op is a pure
// HBM stream of W (arithmetic intensity ~M flop/B), so the design goal is bytes in
// flight, not tensor throughput:
//   * swap-AB: the 128 weight rows of a tile are the MMA "M" dimension (two warpgroups x
//     m64), the (padded) tokens are the MMA "N" dimension (16/32/64, 64-column chunks
//     beyond), so one wgmma consumes a 64x16 (x bf16) weight slab whatever M is; the
//     fp32 accumulator lives in the consumer warpgroups' registers.
//   * W and X tiles arrive by TMA (cp.async.bulk.tensor.2d) into 128B-swizzled shared
//     memory, kStages deep, mbarrier full/empty ring; W is tagged evict-first (read
//     once per forward), X evict-last (re-read by every CTA from L2).
//   * warp-specialised: warps 0-3 / 4-7 = consumer warpgroups (wgmma on weight rows
//     0-63 / 64-127), warp 8 = TMA producer (one lane).  The accumulator is staged through
//     the (then idle) pipeline shared memory so that warpgroup 0 runs the epilogue with
//     one weight row per thread.
//   * split-K over blockIdx.y fills the SMs when N/128 is small; partial sums go to
//     an fp32 [S, M, N] buffer which the *consumer* kernel (norm / rope / silu) reduces
//     in a fixed order, so results are deterministic.
//   * epilogues: bf16 store, fp32 split-K partial, or fused SiLU(gate)*up where a tile is
//     64 gate rows + 64 up rows of the packed gate|up matrix (layers/activation.py:11-14).
//   * PDL: weight tiles of the first kStages are requested BEFORE griddepcontrol.wait, so
//     the HBM stream of this GEMM starts under the tail of the previous kernel.
#pragma once
#include <cuda.h>
#include "common.cuh"

namespace ssdk {

constexpr int kBlockK = 64;    // bf16 per k-block = 128 B = one swizzle row
constexpr int kTileRows = 128; // weight rows per CTA = 2 x wgmma M (64)
constexpr int kGemmConsumers = 256;                // two consumer warpgroups
constexpr int kGemmThreads = kGemmConsumers + 32;  // + the TMA producer warp

enum GemmEpi { EPI_BF16 = 0, EPI_PARTIAL = 1, EPI_SILU = 2, EPI_PUBLISH = 3 };

// EPI_PUBLISH — row-parallel linear + the first half of the one-shot tensor-parallel all-reduce in ONE kernel
// (layers/linear.py:195-199: y = x W^T, then dist.all_reduce).  Every split-K CTA stores its fp32 partial tile and takes a
// ticket; the LAST CTA of a tile sums the S partials in the fixed order s = 0..S-1 (bit-identical to the unfused path),
// rounds to bf16 like the reference's per-rank F.linear output and pushes {2 x bf16, epoch} words straight from its
// registers into slot[parity][rank] of every rank's NVLink symmetric buffer.  The consumer (add_rmsnorm_kernel with
// SymmIn) polls the words themselves, so no separate publish kernel, no re-read of the partials by another grid and no
// kernel boundary sit between the GEMM and the all-reduce.
constexpr int kPubMaxRanks = 8;
struct PublishParams {
  uint8_t* peer[kPubMaxRanks];  // symmetric buffer of every rank (peer-mapped)
  const unsigned* fwd_seq;      // sequence number of the running target forward (epoch base)
  unsigned slot_bytes;
  int call_idx, n_calls;        // static index of this all-reduce inside the forward / all-reduces per forward
  int n_ranks, rank;
};

struct GemmParams {
  void* out;          // EPI_BF16/EPI_SILU: bf16 [M, ldo]; EPI_PARTIAL: fp32 [S, M, N]
  int M;              // valid tokens (<= UMMA_N)
  int N;              // output width (weight rows; for EPI_SILU the ffn width)
  int ldo;            // output row stride in elements
  int num_kb;         // total k-blocks (K / 64)
  int kb_per_split;   // k-blocks per blockIdx.y
  int tile_rows;      // output columns per tile: 128 (plain) or 64 (silu)
  int hi_row_offset;  // W row offset of the second 64-row half: 64 (plain) or ffn (silu)
  // in-kernel split-K reduction (EPI_PUBLISH, EPI_SILU with gridDim.y > 1): every split stores its fp32 partial tile and
  // takes a ticket; the last CTA of a tile sums the S partials in the fixed order s = 0..S-1 and runs the epilogue
  float* sk_partials;     // fp32 [S, M, sk_width]
  unsigned* sk_counters;  // [tiles] arrival tickets, zero on entry and on exit
  int sk_width;           // row width of the partial buffer (N, or 2 * ffn for gate|up)
  PublishParams pub;      // EPI_PUBLISH only
};

// Split-K ticket reduction run by the 4 epilogue warps (threads 0..127).  `col` = this thread's column in the partial
// buffer (< 0: no column).  Returns true in the CTA that arrived last, with r[m] replaced by the sum over all splits.
template <int UMMA_N>
SSDK_DEVINL bool splitk_ticket_reduce(uint32_t* r, const GemmParams& p, int col, int tile, int* smem_flag) {
  const int S = (int)gridDim.y;
  if (S <= 1) return true;
  if (col >= 0) {
    float* out = p.sk_partials + (size_t)blockIdx.y * p.M * p.sk_width;
#pragma unroll
    for (int m = 0; m < UMMA_N; ++m)
      if (m < p.M) out[(size_t)m * p.sk_width + col] = __uint_as_float(r[m]);
  }
  // the partial stores of the 128 epilogue threads are ordered before thread 64's acq_rel ticket by the named barrier
  // (one MEMBAR on one thread instead of a __threadfence on all of them); the same atomic is the acquire for the last CTA
  asm volatile("bar.sync 1, 128;" ::: "memory");
  if (threadIdx.x == 0) *smem_flag = (atom_add_acq_rel_gpu(&p.sk_counters[tile], 1u) == (unsigned)S - 1u) ? 1 : 0;
  asm volatile("bar.sync 1, 128;" ::: "memory");
  if (*smem_flag == 0) return false;
  if (threadIdx.x == 0) st_relaxed_gpu_u32(&p.sk_counters[tile], 0u);  // every CTA of this tile has taken its ticket
  if (col >= 0) {
    const size_t stride = (size_t)p.M * p.sk_width;
#pragma unroll
    for (int m = 0; m < UMMA_N; ++m) {
      if (m < p.M) {
        const float* src = p.sk_partials + (size_t)m * p.sk_width + col;
        float v[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) v[q] = (q < S && q != (int)blockIdx.y) ? __ldcg(src + (size_t)q * stride) : 0.f;
        float acc = 0.f;
#pragma unroll
        for (int q = 0; q < 8; ++q)
          if (q < S) acc += (q == (int)blockIdx.y) ? __uint_as_float(r[m]) : v[q];
        r[m] = __float_as_uint(acc);
      }
    }
  }
  return true;
}


template <int UMMA_N>
struct GemmCfg {
  static constexpr int kABytes = kTileRows * kBlockK * 2;  // 16384
  static constexpr int kBBytes = UMMA_N * kBlockK * 2;     // 2048 / 4096 / 8192 / 16384 / 32768
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = (UMMA_N == 16) ? 6 : (UMMA_N == 32 ? 5 : 4);
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024;  // + alignment slack
  // UMMA_N <= 64 (decode / verify: weight streaming, two CTAs per SM keep ~190 KB of loads in flight); 128 / 256 (prefill
  // chunks and large batches: 128-192 KB of stages, one CTA per SM, the weights are read once per 128 / 256 tokens)
  static constexpr int kCtasPerSm = UMMA_N <= 64 ? 2 : 1;
  static constexpr int kEpiCols = UMMA_N < 64 ? UMMA_N : 64;       // accumulator columns handled per epilogue pass
  static constexpr int kPasses = UMMA_N / kEpiCols;                // = wgmma N-chunks per k-step
  // epilogue shared memory, carved from the drained pipeline: accumulator stage [128][kEpiCols + 1] fp32, then the
  // SiLU exchange of the same size
  static constexpr int kEpiBytes = kTileRows * (kEpiCols + 1) * 4;
  static_assert(2 * kEpiBytes <= kStages * kStageBytes, "epilogue staging must fit in the pipeline stages");
};

template <int UMMA_N, int EPI>
__global__ void __launch_bounds__(kGemmThreads, GemmCfg<UMMA_N>::kCtasPerSm)
gemm_ws_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX, GemmParams p) {
  using Cfg = GemmCfg<UMMA_N>;
  constexpr int kStages = Cfg::kStages;
  constexpr int CW = Cfg::kEpiCols;

  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kStages];
  __shared__ __align__(8) uint64_t empty_bar[kStages];
  __shared__ int pub_last;

  // 128B swizzle needs 1024 B aligned tiles
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tile = blockIdx.x;
  const int kb0 = blockIdx.y * p.kb_per_split;
  const int nkb = min(p.kb_per_split, p.num_kb - kb0);
  const int row_lo = (EPI == EPI_SILU) ? tile * 64 : tile * kTileRows;
  const int row_hi = row_lo + p.hi_row_offset;

  if (threadIdx.x == kGemmConsumers) {
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmX);
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kGemmConsumers / 32);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  // let the next kernel in the stream start its own prologue / weight prefetch
  pdl_launch_dependents();

  if (threadIdx.x >= kGemmConsumers) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      const int pre = min(nkb, kStages);
      // weights do not depend on the previous kernel: request them before the grid dependency
      for (int i = 0; i < pre; ++i) {
        uint8_t* a_s = smem + i * Cfg::kStageBytes;
        mbar_arrive_expect_tx(&full_bar[i], Cfg::kStageBytes);
        const int k = (kb0 + i) * kBlockK;
        tma_load_2d(a_s, &tmW, &full_bar[i], k, row_lo, kEvictFirst);
        tma_load_2d(a_s + Cfg::kABytes / 2, &tmW, &full_bar[i], k, row_hi, kEvictFirst);
      }
      pdl_wait();  // X is produced by the previous kernel
      trace_mark(TR_GEMM);
      for (int i = 0; i < pre; ++i) {
        uint8_t* b_s = smem + i * Cfg::kStageBytes + Cfg::kABytes;
        tma_load_2d(b_s, &tmX, &full_bar[i], (kb0 + i) * kBlockK, 0, kEvictLast);
      }
      for (int i = pre; i < nkb; ++i) {
        const int s = i % kStages;
        const uint32_t ph = (uint32_t)(i / kStages) & 1u;
        mbar_wait(&empty_bar[s], ph ^ 1u);
        uint8_t* a_s = smem + s * Cfg::kStageBytes;
        mbar_arrive_expect_tx(&full_bar[s], Cfg::kStageBytes);
        const int k = (kb0 + i) * kBlockK;
        tma_load_2d(a_s, &tmW, &full_bar[s], k, row_lo, kEvictFirst);
        tma_load_2d(a_s + Cfg::kABytes / 2, &tmW, &full_bar[s], k, row_hi, kEvictFirst);
        tma_load_2d(a_s + Cfg::kABytes, &tmX, &full_bar[s], k, 0, kEvictLast);
      }
    }
  } else {
    // ===================== consumer warpgroups: MMA, then epilogue =====================
    const int wg = warp >> 2;  // weight rows 64 wg .. 64 wg + 63 of the tile
    float acc[Cfg::kPasses][CW / 2];
#pragma unroll
    for (int c = 0; c < Cfg::kPasses; ++c)
#pragma unroll
      for (int j = 0; j < CW / 2; ++j) acc[c][j] = 0.f;
    for (int i = 0; i < nkb; ++i) {
      const int s = i % kStages;
      const uint32_t ph = (uint32_t)(i / kStages) & 1u;
      mbar_wait(&full_bar[s], ph);
      uint8_t* a_s = smem + s * Cfg::kStageBytes;
      const uint64_t adesc = make_wgmma_desc_k128(a_s + wg * (Cfg::kABytes / 2));
      const uint64_t bdesc = make_wgmma_desc_k128(a_s + Cfg::kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k) {
        // advance 16 bf16 = 32 B along K inside the 128 B swizzle row: +2 in 16 B units; the next 64-token chunk of X
        // starts 64 rows x 128 B = 8 KB further on
#pragma unroll
        for (int c = 0; c < Cfg::kPasses; ++c)
          wgmma_bf16_ss<CW>(acc[c], adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k + c * (CW * 128 / 16)), 1u);
      }
      wgmma_commit();
      wgmma_wait_all();
      if (lane == 0) mbar_arrive(&empty_bar[s]);  // frees the smem stage: this warp's MMAs have retired
    }

    pdl_wait();
    if (threadIdx.x == 0) trace_fine(TRF_GEMM + 0);  // CTA 0's accumulator complete
    // every consumer warp is past its last MMA and every TMA load has landed: the stages are free for the epilogue
    asm volatile("bar.sync 2, %0;" ::"n"(kGemmConsumers) : "memory");
    float* stage = reinterpret_cast<float*>(smem);
    constexpr int LD = CW + 1;
    const int frag_row = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int frag_col = 2 * (lane & 3);
    const int row = threadIdx.x;  // epilogue (warpgroup 0): one weight row per thread
    bool stop = false;            // SiLU split-K: another CTA of this tile finishes it
    // the accumulator is drained in passes of CW token columns (one pass for UMMA_N <= 64); token index = m0 + m
#pragma unroll
    for (int c = 0; c < Cfg::kPasses; ++c) {
    const int m0 = c * CW;
    if (m0 >= p.M || stop) break;
#pragma unroll
    for (int j = 0; j < CW / 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        stage[(frag_row + 8 * h) * LD + 8 * j + frag_col] = acc[c][4 * j + 2 * h];
        stage[(frag_row + 8 * h) * LD + 8 * j + frag_col + 1] = acc[c][4 * j + 2 * h + 1];
      }
    asm volatile("bar.sync 2, %0;" ::"n"(kGemmConsumers) : "memory");
    if (threadIdx.x < kTileRows) {
    uint32_t r[CW];
#pragma unroll
    for (int m = 0; m < CW; ++m) r[m] = __float_as_uint(stage[row * LD + m]);

    if (EPI == EPI_BF16) {
      const int n = row_lo + row;
      if (n < p.N) {
        __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out);
#pragma unroll
        for (int m = 0; m < CW; ++m)
          if (m0 + m < p.M) out[(size_t)(m0 + m) * p.ldo + n] = f2bf(__uint_as_float(r[m]));
      }
    } else if (EPI == EPI_PARTIAL) {
      const int n = row_lo + row;
      if (n < p.N) {
        float* out = reinterpret_cast<float*>(p.out) + (size_t)blockIdx.y * p.M * p.N;
#pragma unroll
        for (int m = 0; m < CW; ++m)
          if (m0 + m < p.M) out[(size_t)(m0 + m) * p.N + n] = __uint_as_float(r[m]);
      }
    } else if (EPI == EPI_PUBLISH) {
      const PublishParams& pb = p.pub;
      const int n = row_lo + row;
      // in-kernel split-K (ticket) is only planned for single-pass shapes (UMMA_N <= 64: decode / verify)
      const bool last = splitk_ticket_reduce<CW>(r, p, n < p.N ? n : -1, tile, &pub_last);
      if (last) {
        const unsigned seq = __ldcg(pb.fwd_seq);
        const unsigned e = symm_epoch_of(seq, pb.call_idx);
        const size_t slot_off = ((size_t)symm_parity_of(seq, pb.call_idx, pb.n_calls) * kPubMaxRanks + pb.rank) * pb.slot_bytes;
#pragma unroll
        for (int m = 0; m < CW; ++m) {
          if (m0 + m < p.M) {
            const __nv_bfloat16 mine = f2bf(__uint_as_float(r[m]));
            const uint32_t bits = (uint32_t)__bfloat16_as_ushort(mine);
            const uint32_t nb = __shfl_down_sync(0xffffffffu, bits, 1);
            if ((lane & 1) == 0 && n < p.N) {
              const uint2 word = make_uint2(bits | (nb << 16), e);
              const size_t off = slot_off + (((size_t)(m0 + m) * p.N + n) >> 1) * 8;
#pragma unroll
              for (int rk = 0; rk < kPubMaxRanks; ++rk)
                if (rk < pb.n_ranks) st_global_v2_u32(pb.peer[rk] + off, word.x, word.y);  // ONE 8-byte store: data + flag
            }
          }
        }
      }
    } else {
      // SiLU(gate) * up: rows 0..63 = gate, 64..127 = up of the same 64 output columns.
      // With split-K (narrow tensor-parallel shards: too few 64-column tiles to fill the machine) the last CTA of a
      // tile first sums the partial gate / up rows of all splits; the nonlinearity is applied once, on the full sums.
      {
        const int j = row & 63;
        const int ncol = row_lo + j;
        const int col = ncol < p.N ? (row < 64 ? ncol : p.N + ncol) : -1;
        if (!splitk_ticket_reduce<CW>(r, p, col, tile, &pub_last)) goto epilogue_pass_done;
      }
      // the exchange (128 x (CW + 1) floats) sits behind the accumulator stage in the drained pipeline memory
      float* ex = reinterpret_cast<float*>(smem + Cfg::kEpiBytes);
#pragma unroll
      for (int m = 0; m < CW; ++m) ex[row * LD + m] = __uint_as_float(r[m]);
      asm volatile("bar.sync 1, 128;" ::: "memory");
      const int e = threadIdx.x;  // 0..127
      __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out);
      const int mc = min(CW, p.M - m0);
      for (int idx = e; idx < 64 * mc; idx += 128) {
        const int j = idx & 63, m = idx >> 6;
        const int n = row_lo + j;
        if (n < p.N) {
          // the reference rounds the gate|up linear output to bf16 before SiluAndMul
          const float g = bf16_round(ex[j * LD + m]);
          const float u = bf16_round(ex[(64 + j) * LD + m]);
          const float h = (g / (1.0f + __expf(-g))) * u;
          out[(size_t)(m0 + m) * p.ldo + n] = f2bf(h);
        }
      }
    }
    }  // epilogue warpgroup
  epilogue_pass_done:
    // the next pass rewrites the stage; a SiLU split-K CTA that did not arrive last leaves the tile to the one that did
    asm volatile("bar.sync 2, %0;" ::"n"(kGemmConsumers) : "memory");
    stop = (EPI == EPI_SILU) && gridDim.y > 1 && pub_last == 0;
    }  // accumulator passes
  }

  __syncthreads();
  if (threadIdx.x == 0) trace_fine(TRF_GEMM + 1);  // CTA 0's epilogue stored
}

// y[m, n] = bf16( sum_s P[s, m, n] )  — fixed-order split-K reduction (stand-alone op only;
// inside the engine the consumer kernels fold this in).
__global__ void splitk_reduce_kernel(const float* __restrict__ P, __nv_bfloat16* __restrict__ y, int S, int M, int N,
                                     int ldy) {
  pdl_launch_dependents();
  pdl_wait();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * N) return;
  const int m = idx / N, n = idx - m * N;
  float acc = 0.f;
  for (int s = 0; s < S; ++s) acc += P[(size_t)s * M * N + idx];
  y[(size_t)m * ldy + n] = f2bf(acc);
}

}  // namespace ssdk
