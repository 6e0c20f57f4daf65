// attention.cuh — paged attention for decode (q_len = 1), verify (q_len = K+1) and
// prefill chunks (q_len <= 256) over the paged KV cache (any page size; 256 tokens in the reference).
// Replaces sgl_kernel.flash_attn.flash_attn_with_kvcache at layers/attention.py:107-111,128-131:
//   softmax(q k^T * hd^-1/2 + causal) v, GQA (query head h -> kv head h / (H/KV)),
//   causal mask aligned to the END of the cache (query j of a sequence sees kv positions
//   <= context_len - q_len + j), K/V read back from the paged cache (attention.py:82-83).
//
// Work decomposition (the problem is tiny and latency-bound at b=1, so the aim is to
// spread a few hundred KB of KV over as many SMs as possible):
//   grid = (kv_heads, n_split, batch * n_qtiles), 128 threads.
//   A CTA owns one kv head, up to TQ query tokens x G=H/KV query heads (R = G*tq <= 64 rows,
//   padded to MT 16-row MMA tiles) and a contiguous range of 64-token KV chunks.
//   K/V chunks are staged in shared memory with 16-byte cp.async (coalesced 256 B rows of a
//   page), double buffered; QK^T and PV run on mma.sync m16n8k16 (bf16, fp32 accumulate)
//   with ldmatrix fragments; softmax is online in fp32 (exp2 domain).
//   Warps split (m-tile, token-slice); their partial (m, l, O) are merged through smem,
//   split-KV partials through a global fp32 scratch + attn_combine_kernel.
// The grid is static (CUDA-graph friendly): each CTA derives its chunk range from
// context_lens[] at run time.
#pragma once
#include "common.cuh"

namespace ssdk {

// warps per CTA: 8 for the 32/64-row q tiles (four or two token slices per m-tile), 4 for single-m-tile decode.
// One CTA per SM is resident, so the kernel is bound by the length of each warp's serial instruction chain (address
// generation, softmax, epilogue merge) rather than by bandwidth: more warps = shorter chains.
constexpr int attn_warps(int MT) { return MT == 1 ? 4 : 8; }
constexpr int kAttChunk = 64;
constexpr int kAttnMaxSplit = 32;  // split-KV partials per (token, head) row; attn_combine_kernel merges up to 32

// Launch plan (host code, shared by the engine and the host-thread test driver).
struct AttnPlan {
  int TQ;        // query tokens per CTA tile
  int MT;        // 16-row MMA tiles per CTA (G * TQ rows, padded)
  int n_qtiles;  // ceil(Q / TQ)
  int n_split;   // KV splits per (kv head, sequence, q tile)
};
// q tile of <= 32 rows (two 16-row MMA tiles, 8 warps = 4 token slices each): faster per verify layer than one 56-row
// tile or 16-row tiles.  KV is split until there are about two CTAs per SM, at most kAttnMaxSplit ways and at most one
// split per 64-token chunk of max_ctx.  Returns 1 for an unsupported GQA ratio, 2 for a tile that is too large.
inline int attn_make_plan(int H, int KV, int B, int Q, int max_ctx, int n_sms, AttnPlan* pl) {
  if (KV < 1) return 1;
  const int G = H / KV;
  if (G < 1|| G > 16 || (H % KV) != 0) return 1;
  int tq = 32 / G;
  if (tq < 1) tq = 1;
  if (tq > Q) tq = Q;
  int mt = (G * tq + 15) / 16;
  if (mt == 3) mt = 4;
  if (mt > 4) return 2;
  pl->TQ = tq;
  pl->MT = mt;
  pl->n_qtiles = (Q + tq - 1) / tq;
  const int ctas = KV * B * pl->n_qtiles;
  int ns = (2 * n_sms + ctas - 1) / ctas;
  const int max_chunks = max_ctx > kAttChunk ? (max_ctx + kAttChunk - 1) / kAttChunk : 1;
  if (ns > kAttnMaxSplit) ns = kAttnMaxSplit;
  if (ns > max_chunks) ns = max_chunks;
  pl->n_split = ns < 1 ? 1 : ns;
  return 0;
}
// AttnParams::g_shift
inline int attn_g_shift(int H, int KV) {
  for (int sft = 0; sft < 5; ++sft)
    if (H / KV == (1 << sft)) return sft;
  return -1;
}

struct AttnParams {
  const __nv_bfloat16* q;        // [B*Q, H, hd]
  const __nv_bfloat16* k_cache;  // [slots, KV, hd]
  const __nv_bfloat16* v_cache;
  const int32_t* block_tables;   // [B, max_blocks]
  const int32_t* context_lens;   // [B], includes the Q new tokens
  __nv_bfloat16* out;            // [B*Q, H*hd]
  float* part_o;                 // [B*Q*H, n_split, hd]
  float* part_lse;               // [B*Q*H, n_split]
  int B, Q, H, KV, block_size, max_blocks, n_split, TQ, n_qtiles;
  int g_shift;                   // log2(H / KV) when the GQA ratio is a power of two, else -1
  float scale_log2;              // softmax scale * log2(e)
};

#ifndef SSDK_HOST_EMU
// tests/emu/cuda_emu.h supplies host stand-ins for these five
SSDK_DEVINL void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(sz)
               : "memory");
}
SSDK_DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
SSDK_DEVINL void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
SSDK_DEVINL void ldmatrix_x4(uint32_t* r, const void* smem_row) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(smem_row)));
}
SSDK_DEVINL void ldmatrix_x4_trans(uint32_t* r, const void* smem_row) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(smem_row)));
}
SSDK_DEVINL void mma_bf16_16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
#endif
SSDK_DEVINL uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

template <int HD, int MT>
__global__ void __launch_bounds__(attn_warps(MT) * 32) paged_attn_kernel(AttnParams p) {
  constexpr int NW = attn_warps(MT);
  constexpr int kAttThreads = NW * 32;
  constexpr int LDS = HD + 8;               // padded smem row (bf16 elements)
  constexpr int TSL = NW / MT;              // token slices per chunk
  constexpr int TW = kAttChunk / TSL;       // tokens per warp per chunk (16 * MT)
  constexpr int NT = TW / 8;                // 8-token score tiles per warp
  constexpr int KS = HD / 16;               // k-steps over head_dim
  constexpr int ND = HD / 8;                // 8-wide output tiles over head_dim
  constexpr int SEG = HD / 8;               // 16-byte segments per K/V row

  SSDK_DYN_SMEM(uint8_t, att_smem);
  __nv_bfloat16* sK = reinterpret_cast<__nv_bfloat16*>(att_smem);            // [2][64][LDS]
  __nv_bfloat16* sV = sK + 2 * kAttChunk * LDS;                              // [2][64][LDS]

  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) trace_mark(TR_ATTN);

  const int kvh = blockIdx.x, split = blockIdx.y;
  const int b = blockIdx.z / p.n_qtiles, qt = blockIdx.z % p.n_qtiles;
  const int G = p.H / p.KV;
  const int tq = min(p.TQ, p.Q - qt * p.TQ);
  const int R = G * tq;
  const int ctx = p.context_lens[b];
  const int ctx0 = ctx - p.Q;                         // tokens before this forward
  const int kv_max = ctx0 + qt * p.TQ + tq;           // exclusive upper bound of visible kv for this q-tile
  const int nch_total = (kv_max + kAttChunk - 1) / kAttChunk;
  const int cps = (nch_total + p.n_split - 1) / p.n_split;
  const int ch_begin = split * cps;
  const int ch_end = min(nch_total, ch_begin + cps);
  // splits without chunks own no partial: attn_combine_kernel only reads the first ceil(nch_total / cps) splits
  if (p.n_split > 1 && ch_begin >= ch_end) return;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int mtile = warp % MT, tslice = warp / MT;
  const int32_t* bt = p.block_tables + (size_t)b * p.max_blocks;

  // ---- Q fragments (registers, whole kernel) ----
  uint32_t qa[KS][4];
  {
    const int r0 = mtile * 16 + g, r1 = r0 + 8;
    const __nv_bfloat16* q0 = nullptr;
    const __nv_bfloat16* q1 = nullptr;
    if (r0 < R) q0 = p.q + ((size_t)(b * p.Q + qt * p.TQ + r0 / G) * p.H + kvh * G + r0 % G) * HD;
    if (r1 < R) q1 = p.q + ((size_t)(b * p.Q + qt * p.TQ + r1 / G) * p.H + kvh * G + r1 % G) * HD;
#pragma unroll
    for (int kk = 0; kk < KS; ++kk) {
      const int c = kk * 16 + 2 * t;
      qa[kk][0] = q0 ? *reinterpret_cast<const uint32_t*>(q0 + c) : 0u;
      qa[kk][1] = q1 ? *reinterpret_cast<const uint32_t*>(q1 + c) : 0u;
      qa[kk][2] = q0 ? *reinterpret_cast<const uint32_t*>(q0 + c + 8) : 0u;
      qa[kk][3] = q1 ? *reinterpret_cast<const uint32_t*>(q1 + c + 8) : 0u;
    }
  }
  // causal limits (exclusive) of this thread's two rows
  int lim[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = mtile * 16 + g + 8 * h;
    lim[h] = (r < R) ? (ctx0 + qt * p.TQ + r / G + 1) : 0;
  }

  float o[ND][4];
#pragma unroll
  for (int i = 0; i < ND; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};

  // A 64-token chunk never straddles a page when block_size % 64 == 0 (the reference uses 256): one block-table
  // lookup per chunk instead of one dependent global load per 16-byte segment.
  const bool page_aligned = (p.block_size % kAttChunk) == 0;
  auto load_chunk = [&](int ch, int stage) {
    const int base = ch * kAttChunk;
    __nv_bfloat16* dk = sK + stage * kAttChunk * LDS;
    __nv_bfloat16* dv = sV + stage * kAttChunk * LDS;
    int chunk_blk = -1, chunk_off = 0;
    if (page_aligned) {
      chunk_blk = bt[base / p.block_size];
      chunk_off = base % p.block_size;
    }
#pragma unroll 4
    for (int idx = threadIdx.x; idx < kAttChunk * SEG; idx += kAttThreads) {
      const int tok = idx / SEG, seg = idx - tok * SEG;
      const int pos = base + tok;
      bool valid = pos < kv_max;
      size_t off = 0;
      if (valid) {
        int blk, in_blk;
        if (page_aligned) {
          blk = chunk_blk;
          in_blk = chunk_off + tok;
        } else {
          blk = bt[pos / p.block_size];
          in_blk = pos % p.block_size;
        }
        valid = blk >= 0;
        off = (((size_t)blk * p.block_size + in_blk) * p.KV + kvh) * HD + seg * 8;
      }
      cp_async16(dk + tok * LDS + seg * 8, p.k_cache + off, valid);
      cp_async16(dv + tok * LDS + seg * 8, p.v_cache + off, valid);
    }
  };

  if (ch_begin < ch_end) {
    load_chunk(ch_begin, 0);
    cp_async_commit();
    if (threadIdx.x == 0) trace_fine(TRF_ATTN + 0);  // q + first chunk requested
    for (int ch = ch_begin; ch < ch_end; ++ch) {
      const int stage = (ch - ch_begin) & 1;
      if (ch + 1 < ch_end) load_chunk(ch + 1, stage ^ 1);
      cp_async_commit();
      cp_async_wait<1>();
      __syncthreads();
      if (threadIdx.x == 0 && ch == ch_begin) trace_fine(TRF_ATTN + 1);  // first chunk landed

      const __nv_bfloat16* cK = sK + stage * kAttChunk * LDS;
      const __nv_bfloat16* cV = sV + stage * kAttChunk * LDS;
      const int tok0 = tslice * TW;

      // ---- S = Q K^T ----
      float s[NT][4];
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
        for (int kk = 0; kk < KS; kk += 2) {
          uint32_t kb[4];
          const int mi = lane >> 3, rr = lane & 7;
          const __nv_bfloat16* addr = cK + (tok0 + nt * 8 + rr) * LDS + kk * 16 + (mi & 1) * 8 + (mi >> 1) * 16;
          ldmatrix_x4(kb, addr);
          mma_bf16_16816(s[nt], qa[kk], kb[0], kb[1]);
          mma_bf16_16816(s[nt], qa[kk + 1], kb[2], kb[3]);
        }
      }
      // ---- scale, causal mask, online softmax ----
      const int pos_base = ch * kAttChunk + tok0 + 2 * t;
      float mnew[2] = {mrow[0], mrow[1]};
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int h = e >> 1;
          const int pos = pos_base + nt * 8 + (e & 1);
          const float v = (pos < lim[h]) ? s[nt][e] * p.scale_log2 : -INFINITY;
          s[nt][e] = v;
          mnew[h] = fmaxf(mnew[h], v);
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mnew[h] = fmaxf(mnew[h], __shfl_xor_sync(0xffffffffu, mnew[h], 1));
        mnew[h] = fmaxf(mnew[h], __shfl_xor_sync(0xffffffffu, mnew[h], 2));
      }
      float corr[2], msafe[2], psum[2] = {0.f, 0.f};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        msafe[h] = (mnew[h] == -INFINITY) ? 0.f : mnew[h];
        corr[h] = exp2f(mrow[h] - msafe[h]);  // mrow = -inf -> 0
        mrow[h] = mnew[h];
      }
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int h = e >> 1;
          const float pv = exp2f(s[nt][e] - msafe[h]);
          s[nt][e] = pv;
          psum[h] += pv;
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) lrow[h] = lrow[h] * corr[h] + psum[h];
#pragma unroll
      for (int i = 0; i < ND; ++i) {
        o[i][0] *= corr[0];
        o[i][1] *= corr[0];
        o[i][2] *= corr[1];
        o[i][3] *= corr[1];
      }
      // ---- O += P V ----
#pragma unroll
      for (int kk = 0; kk < TW / 16; ++kk) {
        uint32_t pa[4];
        pa[0] = pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);
        pa[1] = pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
        pa[2] = pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
        pa[3] = pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
        for (int nd = 0; nd < ND; nd += 2) {
          uint32_t vb[4];
          const int mi = lane >> 3, rr = lane & 7;
          const __nv_bfloat16* addr = cV + (tok0 + kk * 16 + (mi & 1) * 8 + rr) * LDS + nd * 8 + (mi >> 1) * 8;
          ldmatrix_x4_trans(vb, addr);
          mma_bf16_16816(o[nd], pa, vb[0], vb[1]);
          mma_bf16_16816(o[nd + 1], pa, vb[2], vb[3]);
        }
      }
      __syncthreads();  // everyone done with this stage before it is refilled
    }
  }
  cp_async_wait<0>();
  __syncthreads();
  if (threadIdx.x == 0) trace_fine(TRF_ATTN + 2);  // chunk loop done

  // ---- finish row sums across the quad, merge token slices through smem ----
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    lrow[h] += __shfl_xor_sync(0xffffffffu, lrow[h], 1);
    lrow[h] += __shfl_xor_sync(0xffffffffu, lrow[h], 2);
  }
  // Row stride HD + 8 floats (= 8 banks mod 32): the 8-byte fragment stores of a half-warp (rows g = 0..3, column
  // pairs t = 0..3) and the 16-byte row reads of the merge loop are both bank-conflict free.  With 8 warps the buffer
  // is exactly as large as the K/V stages it reuses: 8 * 16 * (HD + 8) * 4 B.
  constexpr int LDO = HD + 8;
  float* sO = reinterpret_cast<float*>(att_smem);  // [NW warps][16 rows][LDO]: O | m | l
  {
    float* w = sO + warp * 16 * LDO;
#pragma unroll
    for (int i = 0; i < ND; ++i) {
      *reinterpret_cast<float2*>(w + g * LDO + i * 8 + 2 * t) = make_float2(o[i][0], o[i][1]);
      *reinterpret_cast<float2*>(w + (g + 8) * LDO + i * 8 + 2 * t) = make_float2(o[i][2], o[i][3]);
    }
    if (t == 0) {
      *reinterpret_cast<float2*>(w + g * LDO + HD) = make_float2(mrow[0], lrow[0]);
      *reinterpret_cast<float2*>(w + (g + 8) * LDO + HD) = make_float2(mrow[1], lrow[1]);
    }
  }
  __syncthreads();
  // one (row, 4 columns) slice per loop iteration: rows 0..R-1, columns 0..HD-1
  for (int idx = threadIdx.x; idx < R * (HD / 4); idx += kAttThreads) {
    const int r = idx / (HD / 4), d = (idx - r * (HD / 4)) * 4;
    const int mt = r >> 4, rr = r & 15;
    float mmax = -INFINITY;
#pragma unroll
    for (int sl = 0; sl < TSL; ++sl) mmax = fmaxf(mmax, sO[((sl * MT + mt) * 16 + rr) * LDO + HD]);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    float l = 0.f;
    if (mmax != -INFINITY) {
#pragma unroll
      for (int sl = 0; sl < TSL; ++sl) {
        const float* w = sO + ((sl * MT + mt) * 16 + rr) * LDO;
        const float2 ml = *reinterpret_cast<const float2*>(w + HD);
        const float4 v = *reinterpret_cast<const float4*>(w + d);
        const float wgt = exp2f(ml.x - mmax);
        acc.x += v.x * wgt; acc.y += v.y * wgt; acc.z += v.z * wgt; acc.w += v.w * wgt;
        l += ml.y * wgt;
      }
    }
    const int rt = (p.g_shift >= 0) ? (r >> p.g_shift) : r / G;  // token inside the tile; r - rt * G = head of the group
    const int row_q = b * p.Q + qt * p.TQ + rt;
    const int head = kvh * G + (r - rt * G);
    const float inv = (l > 0.f) ? 1.f / l : 0.f;
    acc.x *= inv; acc.y *= inv; acc.z *= inv; acc.w *= inv;
    if (p.n_split == 1) {
      __nv_bfloat16* dst = p.out + ((size_t)row_q * p.H + head) * HD + d;
      *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(acc.x, acc.y);
      *reinterpret_cast<__nv_bfloat162*>(dst + 2) = __floats2bfloat162_rn(acc.z, acc.w);
    } else {
      const size_t pr = ((size_t)row_q * p.H + head) * p.n_split + split;
      *reinterpret_cast<float4*>(p.part_o + pr * HD + d) = acc;
      if (d == 0) p.part_lse[pr] = (l > 0.f) ? mmax + log2f(l) : -INFINITY;
    }
  }
  if (threadIdx.x == 0) trace_fine(TRF_ATTN + 3);  // partials / output stored
}

// merge split-KV partials: out = sum_s 2^(lse_s - max) o_s / sum_s 2^(lse_s - max).
// One CTA per (token, head) row, HD/4 threads, each owning one float4 of the output.  Only the splits that had
// chunks (n_active, recomputed from context_lens with the attention kernel's formula) are read, and every thread
// issues all of its loads before using them, so the merge costs ~2 L2 round trips whatever n_split is.
__global__ void attn_combine_kernel(AttnParams p, int hd) {
  SSDK_STATIC_SMEM(float, sw, 32);
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) trace_mark(TR_ATTN);
  const size_t row = blockIdx.x;  // (token, head)
  const int tok = (int)(row / p.H);
  const int b = tok / p.Q, j = tok - b * p.Q;
  const int qt = j / p.TQ;
  const int tq = min(p.TQ, p.Q - qt * p.TQ);
  const int kv_max = p.context_lens[b] - p.Q + qt * p.TQ + tq;
  const int nch_total = (kv_max + kAttChunk - 1) / kAttChunk;
  const int cps = (nch_total + p.n_split - 1) / p.n_split;
  const int n_active = (cps > 0) ? min(p.n_split, (nch_total + cps - 1) / cps) : 0;
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    const float lse = (lane < n_active) ? __ldcg(p.part_lse + row * p.n_split + lane) : -INFINITY;
    const float mx = warp_max(lse);
    const float wgt = (mx == -INFINITY) ? 0.f : exp2f(lse - mx);
    const float wsum = warp_sum(wgt);
    sw[lane] = (wsum > 0.f) ? wgt / wsum : 0.f;
  }
  const int d4 = threadIdx.x;
  float4 v[8];
  const bool mine = d4 < hd / 4;
  // first batch of partial loads is issued before the weights are ready
#pragma unroll
  for (int u = 0; u < 8; ++u)
    v[u] = (mine && u < n_active) ? __ldcg(reinterpret_cast<const float4*>(p.part_o + (row * p.n_split + u) * hd) + d4)
                                  : make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();
  if (threadIdx.x == 0) trace_fine(TRF_COMB + 0);  // weights ready, first batch requested
  if (!mine) return;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int s0 = 0; s0 < n_active; s0 += 8) {
    if (s0 > 0) {
#pragma unroll
      for (int u = 0; u < 8; ++u)
        v[u] = (s0 + u < n_active) ? __ldcg(reinterpret_cast<const float4*>(p.part_o + (row * p.n_split + s0 + u) * hd) + d4)
                                   : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const float ws = (s0 + u < n_active) ? sw[s0 + u] : 0.f;
      acc.x += ws * v[u].x; acc.y += ws * v[u].y; acc.z += ws * v[u].z; acc.w += ws * v[u].w;
    }
  }
  __nv_bfloat16* dst = p.out + row * hd + d4 * 4;
  *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(acc.x, acc.y);
  *reinterpret_cast<__nv_bfloat162*>(dst + 2) = __floats2bfloat162_rn(acc.z, acc.w);
  if (threadIdx.x == 0) trace_fine(TRF_COMB + 1);
}

}  // namespace ssdk
