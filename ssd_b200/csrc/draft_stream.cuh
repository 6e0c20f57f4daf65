// draft_stream.cuh — the whole speculate phase of a sync-SD step (SpeculatorSync.speculate, engine/speculator_sync.py:25-69:
// K single-token draft forwards + K samplings) as ONE persistent kernel, batch 1.
//
// The reference runs a K+1-th draft forward that only writes the KV of the last draft token d_K (speculator_sync.py:46-56).
// Here that KV is written by the NEXT step instead: when the previous step accepted all K drafts, d_K sits at position
// ctx0 - 1 without draft KV ("pending"), and forward 0 carries it as a second, earlier row (row 0) next to the recovery
// token (row 1).  Both rows share every weight slot, so row 0 costs FMAs but no weight bytes.  Row 0 is computed with
// exactly the arithmetic of a one-token forward (same x values, same per-warp dot products and summation order), stores
// its K/V, and produces no logits; its attention units run before row 1's, one device-wide barrier apart, so row 1's
// attention reads row 0's K/V from the cache.
//
// Why: the 1B draft streams 2.47 GB per forward, but the kernel-per-op path has nine kernel boundaries per layer, during
// each of which HBM idles.  The weights
// do not depend on the activations, so here every CTA (one per SM) streams ITS share of every matrix, in program order
// and without ever waiting for a phase, through a ring of 32 KB shared-memory slots:
//   * a PRODUCER warp requests slot after slot with bulk async copies (cp.async.bulk global -> shared, mbarrier
//     transaction counts, L2 evict-first) as soon as the consumers release them — across phase and layer boundaries, so
//     while the CTAs meet at a device-wide barrier or recompute a norm the ring (132 x 160 KB = 21 MB on chip) fills with
//     the NEXT phases' weights;
//   * 8 CONSUMER warps run the phases.  A projection at one token is a GEMV: each warp keeps its 64-float slice of x in
//     registers for the whole phase and owns whole rows (K <= 2048: no cross-warp traffic at all), reads 16 bytes per
//     lane per step from the slot (conflict-free), and releases the slot with one mbarrier arrive per warp.
// History: a persistent kernel with weights read straight from global memory was no faster than the kernel-per-op path;
// a first ring version (thread 0 issuing the copies between block-wide barriers, x read from shared memory) was bound by
// the consume loop, not HBM.
//
// Program order per forward (the five dependent stages of the reference's decoder layer, models/llama3.py:185-199):
//   A  [residual add + input RMSNorm, recomputed by every CTA] -> q|k|v rows
//   B  q/k head norm + RoPE + KV store + split-KV attention for (kv head, split) units; the last split of a kv head to
//      finish merges the partials into the attention output vector
//   C  o-proj rows
//   D  [residual add + post-attention RMSNorm, every CTA] -> gate|up row pairs + SiLU*mul
//   E  down-proj rows
// then final norm -> lm_head rows -> in-kernel sampling (greedy argmax over the bf16 logits, lowest index wins, or the
// Philox exponential race of layers/sampler.py:27-34 — the SAME scores sample_kernel computes, so the tokens are identical)
// -> the next forward starts inside the same launch.  With skip_last_head the last forward only writes KV (the reference's
// K+1-th forward, speculator_sync.py:52-56); the engine no longer launches that forward (see the top of this file).
// Rounding points are the reference's (SURVEY §8a checklist 1-4): every linear output, the residual, the norm output, q/k
// after RoPE and the attention output are rounded to bf16; accumulation is fp32.
//
// Jobs: rows are dealt to CTAs in jobs of consecutive rows; job s of a matrix belongs to CTA s mod #CTAs.
//   K <= 2048  : 8 rows = one slot, ONE contiguous bulk copy; warp w owns row w.
//   gate|up    : 8 (gate, up) row pairs = two slots (8 gate rows | the 8 matching up rows); warp w owns pair w.
//   K >  2048  : R = 4 (K <= 4096) or 2 (K <= 8192) rows = one slot; the 8 warps split (row, K-segment) units and combine
//                their partial sums in a fixed order through shared memory.
//
// FP8 (draft_stream_kernel<HD, GMAX, true>): the four decoder linears are e4m3 bytes with fp32 per-row scales (quant.py);
// the lm_head stays bf16 and keeps the geometry above.  A lane reads 8 e4m3 bytes per 256-column step (one 8-byte shared
// load, conflict-free) where the bf16 path reads 16 bytes, so it keeps the same 8 columns per lane, the same x slice in
// registers (at most 64 floats) and the same per-lane and shuffle summation order.  A row then takes half the slot bytes, so
// every job carries TWICE the rows of its bf16 form and each warp owns two rows (w and w + 8, or the second R-row group of a
// split job): 16 rows per slot for K <= 2048, 16 gate|up pairs per two slots, 8 (K <= 4096) or 4 (K <= 8192) rows per slot
// above.  Slots stay full, so the bytes in flight per SM are the bf16 ring's.  Each warp widens e4m3 -> f16 -> f32 on the
// CUDA cores (exact), and the row scale multiplies the finished fp32 dot product (split rows: the segment sum) right
// before the one bf16 rounding: y[n] = bf16(s[n] * sum_k W8[n, k] x[k]).  gate and up are scaled each by its own scale
// before SiLU.
#pragma once
#include "common.cuh"
#include "sampling.cuh"

namespace ssdk {

constexpr int kDsConsumers = 256;                 // threads 0..255: 8 consumer warps
constexpr int kDsWarps = kDsConsumers / 32;
constexpr int kDsThreads = kDsConsumers + 32;     // + the producer warp
constexpr int kDsMaxLayers = 32;
constexpr int kDsSplits = 16;         // most KV splits per kv head in phase B (long contexts)
constexpr int kDsShortSplits = 8;     // splits up to kDsLongCtx tokens
constexpr int kDsLongCtx = 256;       // = kDsShortSplits x 8 warps x 4 tokens: the most ONE load round of the short layout covers
constexpr int kDsSlotBytes = 32768;   // one ring slot
constexpr int kDsMaxSlots = 6;
constexpr int kDsMaxSteps = 8;        // 256-column steps per K segment (segment <= 2048 columns)
constexpr int kDsBtSmem = 32;         // page-table entries staged in shared memory at kernel start (the table is launch-constant)

struct DsLayer {
  const __nv_bfloat16 *qkv, *o, *gate_up, *down, *in_norm, *post_norm, *q_norm, *k_norm;
};

struct DsParams {
  int d, L, H, KV, ffn, vocab, qk_norm;
  float eps, scale_log2;
  const __nv_bfloat16 *embed, *final_norm, *lm_head;
  const float* rope;  // [max_pos, hd]: cos | sin
  __nv_bfloat16 *k_cache, *v_cache;
  long long cache_layer_stride;  // elements between layers
  int block_size, max_blocks;
  int64_t* tok_buf;              // [n_fwd (+1)]: tok_buf[0] = first input token; the kernel writes tok_buf[f + 1]
  int n_fwd;                     // forwards in this launch
  int skip_last_head;            // 1: the last forward runs without lm_head / sampling (it only writes KV)
  const int32_t* ctx0;           // tokens in the cache before the first forward
  const int32_t* block_table;    // [max_blocks]
  __nv_bfloat16 *vec_qkv, *vec_attn, *vec_o, *vec_act, *vec_down, *resid0, *resid1;
  float* attn_part;              // [H][kDsSplits][hd + 2]: o | m | l
  __nv_bfloat16* logits;         // row f at logits + f * logits_ld (may be null: no logits kept)
  long long logits_ld;
  const float* temp;             // draft temperature [1] (device)
  const uint64_t* dyn;           // optional device {seed, step}: call_id = step * 16 + f
  uint64_t seed, call_base;      // used when dyn == nullptr: call_id = call_base + f
  ArgMax* samp_partial;          // [#CTAs]
  unsigned* bar_state;           // one 64-bit arrival counter (8-byte aligned), only ever grows; zero before the first launch
  unsigned* attn_ticket;         // [KV] arrival tickets of the split-KV units, zero between phases
  int n_slots;                   // ring depth (3 .. kDsMaxSlots)
  DsLayer layers[kDsMaxLayers];
  const int64_t* pend_tok;       // [1] (may be null): >= 0: the token at position ctx0 - 1, whose KV forward 0 writes as row 0
  __nv_bfloat16* vec_row0;       // row 0's vectors (ds_row0_vecs layout); read only when a token is pending
  // FP8 instance only: fp32 per-row scales of layer l's qkv / o / gate_up / down (indexed by DS_QKV .. DS_DOWN); the
  // DsLayer pointers of these four matrices then point at e4m3 bytes
  const float* fp8_scale[kDsMaxLayers][4];
};

// vectors of row 0 of a two-row forward 0, carved from p.vec_row0 like the engine carves the row-1 vectors
struct DsVecs {
  __nv_bfloat16 *qkv, *attn, *o, *down, *resid0, *resid1, *act;
  SSDK_DEVINL __nv_bfloat16* resid(int i) const { return i ? resid1 : resid0; }  // no indexed array: stays in registers
};
SSDK_DEVINL DsVecs ds_row0_vecs(const DsParams& p, int hd) {
  DsVecs v{};
  __nv_bfloat16* b = p.vec_row0;
  if (!b) return v;
  v.qkv = b; b += ((p.H + 2 * p.KV) * hd + 7) / 8 * 8;
  v.attn = b; b += p.H * hd;
  v.o = b; b += p.d;
  v.down = b; b += p.d;
  v.resid0 = b; b += p.d;
  v.resid1 = b; b += p.d;
  v.act = b;
  return v;
}
// floats of the x region of shared memory: one row of every GEMV input, two rows of the norm outputs (d each)
__host__ SSDK_DEVINL int ds_xs_floats(int d, int ffn, int q_width) {
  const int a = 2 * d > ffn ? 2 * d : ffn;
  return a > q_width ? a : q_width;
}

// consumer-only block barrier (the producer warp runs on its own)
SSDK_DEVINL void ds_sync() {
#ifdef SSDK_HOST_EMU
  ::emu::named_barrier(1, kDsConsumers);
#else
  asm volatile("bar.sync 1, 256;" ::: "memory");
#endif
}

// ---------------------------------------------------------------------------------------------
// device-wide barrier of the consumers: ONE 64-bit arrival counter that only ever grows.  Barrier number n of a launch
// is complete when the counter reaches base + n * #CTAs, where base = the counter rounded down to a multiple of #CTAs at
// kernel start (every launch performs whole barriers, and the first barrier of a launch cannot complete before this CTA
// has arrived, so every CTA computes the same base).  Arrival = one release-add without a return value; waiting = relaxed
// polling loads + one acquire fence at the end.  (A first version — acq_rel fetch-adds for arrival, counter reset and
// generation bump, acquire loads for polling — compiled to MEMBAR.ALL.GPU + ATOMG + CCTL.IVALL three times in a row on the
// last arriver and an L1 invalidation per poll.)
// ---------------------------------------------------------------------------------------------
struct DsGridBar {
  unsigned long long* counter;
  unsigned long long target;
  __device__ void init() {
    if (threadIdx.x == 0) {
      const unsigned long long c = ld_relaxed_gpu_u64(counter);
      target = c - c % (unsigned long long)gridDim.x;
    }
  }
  __device__ void sync() {
    ds_sync();  // every consumer thread's writes of this phase are ordered before thread 0's release
    if (threadIdx.x == 0) {
      target += (unsigned long long)gridDim.x;
      red_add_release_gpu_u64(counter, 1ull);
      const long long t0 = clock64();
      while (ld_relaxed_gpu_u64(counter) < target) {
        if (clock64() - t0 > 4000000000LL) __trap();  // a CTA never arrived: fail loudly instead of hanging the GPU
      }
      fence_acq_rel_gpu();
    }
    ds_sync();
  }
};

SSDK_DEVINL uint4 ds_ldcg16(const void* p) { return __ldcg(reinterpret_cast<const uint4*>(p)); }
SSDK_DEVINL float2 ds_bf2(uint32_t w) { return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w)); }

// timeline marks of the second forward of a launch (CTA 0, thread 0; only when ssdk_debug_trace is on): ids 64 + point
SSDK_DEVINL void ds_mark(int f, int point) {
  if (f == 1 && threadIdx.x == 0) trace_mark(64 + point);
}

// ---------------------------------------------------------------------------------------------
// matrix geometry and the per-CTA job sequence
// ---------------------------------------------------------------------------------------------
enum { DS_QKV = 0, DS_O = 1, DS_GU = 2, DS_DOWN = 3, DS_HEAD = 4 };
enum { DS_PLAIN = 0, DS_PAIR = 1, DS_SPLIT = 2 };
struct DsGeom {
  int K;     // row length
  int rows;  // output rows (gate|up: pairs)
  int kind;  // DS_PLAIN / DS_PAIR / DS_SPLIT
  int rpj;   // rows (pairs) per job
  int segs;  // K segments per row (DS_SPLIT; 1 otherwise)
  int nj;    // jobs of the matrix
};
__host__ SSDK_DEVINL bool ds_geometry(int K, int rows, bool pair, DsGeom* g) {
  g->K = K; g->rows = rows; g->segs = 1;
  if (K < 256 || K > 8192 || (K % 256) != 0) return false;
  if (pair) {
    if (K > 2048) return false;  // a pair job is 8 gate rows + 8 up rows in two slots
    g->kind = DS_PAIR; g->rpj = 8;
  } else if (K <= 2048) {
    g->kind = DS_PLAIN; g->rpj = 8;
  } else {
    g->kind = DS_SPLIT; g->rpj = K <= 4096 ? 4 : 2; g->segs = kDsWarps / g->rpj;
    if ((K % (256 * g->segs)) != 0) return false;
  }
  g->nj = (rows + g->rpj - 1) / g->rpj;
  return true;
}
// an FP8 decoder linear: the bf16 job shape (segments, x layout) with twice the rows per job (see the top of the file)
__host__ SSDK_DEVINL bool ds_geometry8(int K, int rows, bool pair, DsGeom* g) {
  if (!ds_geometry(K, rows, pair, g)) return false;
  g->rpj *= 2;
  g->nj = (rows + g->rpj - 1) / g->rpj;
  return true;
}
SSDK_DEVINL bool ds_has_head(const DsParams& p, int f) { return !(p.skip_last_head && f == p.n_fwd - 1); }
SSDK_DEVINL const __nv_bfloat16* ds_weight(const DsParams& p, int l, int m) {
  const DsLayer& lw = p.layers[l < p.L ? l : 0];
  return m == DS_QKV ? lw.qkv : (m == DS_O ? lw.o : (m == DS_GU ? lw.gate_up : (m == DS_DOWN ? lw.down : p.lm_head)));
}

// position in the program: forward f, layer l (l == L: the lm_head), matrix m, job s (s = CTA, CTA + #CTAs, ...)
struct DsCursor {
  int f, l, m, s;
  bool valid;
};
SSDK_DEVINL void ds_cursor_settle(const DsParams& p, const DsGeom* geom, DsCursor& c) {  // skip matrices without a job left
  while (c.valid && c.s >= geom[c.m].nj) {
    c.s = (int)blockIdx.x;
    if (c.m == DS_HEAD) {
      c.f++; c.l = 0; c.m = DS_QKV;
    } else if (c.m == DS_DOWN) {
      c.l++; c.m = DS_QKV;
      if (c.l == p.L) {
        if (ds_has_head(p, c.f)) c.m = DS_HEAD;
        else { c.f++; c.l = 0; }
      }
    } else {
      c.m++;
    }
    if (c.f >= p.n_fwd) c.valid = false;
  }
}

// the producer: one lane walks the job sequence of this CTA and refills slots as the consumers release them.  (An L2
// window beyond the ring — `cp.async.bulk.prefetch.L2` of the next jobs, continuously or only while every requested copy
// had landed — made the step slower and was removed.)
SSDK_DEVINL void ds_cursor_next(const DsParams& p, const DsGeom* geom, DsCursor& c) {
  c.s += (int)gridDim.x;
  if (c.s >= geom[c.m].nj) ds_cursor_settle(p, geom, c);
}
// FP8: the decoder linears are e4m3 (one byte per weight), the lm_head bf16
template <bool FP8>
SSDK_DEVINL void ds_producer(const DsParams& p, const DsGeom* geom, uint8_t* ring, uint64_t* full, uint64_t* empty) {
  DsCursor c;
  c.f = 0; c.l = 0; c.m = DS_QKV; c.s = (int)blockIdx.x; c.valid = p.n_fwd > 0;
  ds_cursor_settle(p, geom, c);
  unsigned n = 0;  // slots requested so far
  const unsigned S = (unsigned)p.n_slots;
  while (c.valid) {
    const DsGeom g = geom[c.m];
    const __nv_bfloat16* w = ds_weight(p, c.l, c.m);
    const int rows = min(g.rpj, g.rows - c.s * g.rpj);
    unsigned bytes = (unsigned)rows * (unsigned)g.K * 2u;
    if constexpr (FP8) {
      if (c.m != DS_HEAD) bytes >>= 1;
    }
    const int parts = g.kind == DS_PAIR ? 2 : 1;
    for (int q = 0; q < parts; ++q) {
      const unsigned slot = n % S, round = n / S;
      mbar_wait(&empty[slot], (round & 1u) ^ 1u);  // a fresh barrier passes the first round at once
      mbar_arrive_expect_tx(&full[slot], bytes);
      const void* src = w + ((size_t)(q ? g.rows : 0) + (size_t)c.s * g.rpj) * g.K;
      if constexpr (FP8) {
        if (c.m != DS_HEAD)
          src = reinterpret_cast<const uint8_t*>(w) + ((size_t)(q ? g.rows : 0) + (size_t)c.s * g.rpj) * g.K;
      }
      bulk_load_g2s(ring + (size_t)slot * kDsSlotBytes, src, bytes, &full[slot]);
      ++n;
    }
    ds_cursor_next(p, geom, c);
  }
}

// ---------------------------------------------------------------------------------------------
// consumers
// ---------------------------------------------------------------------------------------------
struct DsRing {
  uint8_t* base;
  uint64_t *full, *empty;
  unsigned n_slots;
  unsigned taken;  // slots consumed so far (uniform over the consumers)
};
SSDK_DEVINL const uint8_t* ds_acquire(DsRing& r, unsigned k) {  // wait for the k-th slot after `taken`
  const unsigned n = r.taken + k, slot = n % r.n_slots;
  mbar_wait(&r.full[slot], (n / r.n_slots) & 1u);
  return r.base + (size_t)slot * kDsSlotBytes;
}
SSDK_DEVINL void ds_release(DsRing& r, unsigned k, int lane) {  // one arrive per consumer warp, after its last read
  __syncwarp();
  if (lane == 0) mbar_arrive(&r.empty[(r.taken + k) % r.n_slots]);
}

// x stays in REGISTERS for a whole phase: a warp always works on the same K segment (<= 2048 columns), i.e. lane owns the
// 8 columns [256 j + 8 lane, +8) of every 256-column step j < 8 — 64 floats
SSDK_DEVINL void ds_load_x(const float* xseg, int steps, int lane, float (&xr)[kDsMaxSteps][8]) {
#pragma unroll
  for (int j = 0; j < kDsMaxSteps; ++j) {
    if (j < steps) {
      const float4 a = *reinterpret_cast<const float4*>(xseg + j * 256 + lane * 8);
      const float4 b = *reinterpret_cast<const float4*>(xseg + j * 256 + lane * 8 + 4);
      xr[j][0] = a.x; xr[j][1] = a.y; xr[j][2] = a.z; xr[j][3] = a.w;
      xr[j][4] = b.x; xr[j][5] = b.y; xr[j][6] = b.z; xr[j][7] = b.w;
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) xr[j][e] = 0.f;
    }
  }
}
// dot of one row segment held in shared memory (16 bytes per lane per step, conflict-free) with x in registers
SSDK_DEVINL float ds_dot_seg(const uint8_t* wseg, int steps, int lane, const float (&xr)[kDsMaxSteps][8]) {
  const uint4* wp = reinterpret_cast<const uint4*>(wseg) + lane;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
  for (int j = 0; j < kDsMaxSteps; ++j) {
    if (j < steps) {
      const uint4 w = wp[j * 32];
      float2 f = ds_bf2(w.x);
      a0 = fmaf(f.x, xr[j][0], a0); a1 = fmaf(f.y, xr[j][1], a1);
      f = ds_bf2(w.y);
      a2 = fmaf(f.x, xr[j][2], a2); a3 = fmaf(f.y, xr[j][3], a3);
      f = ds_bf2(w.z);
      a0 = fmaf(f.x, xr[j][4], a0); a1 = fmaf(f.y, xr[j][5], a1);
      f = ds_bf2(w.w);
      a2 = fmaf(f.x, xr[j][6], a2); a3 = fmaf(f.y, xr[j][7], a3);
    }
  }
  return warp_sum((a0 + a1) + (a2 + a3));
}

// ds_dot_seg for an e4m3 row segment: 8 bytes (the same 8 columns) per lane per step, the same summation order; the
// caller applies the row scale
SSDK_DEVINL float ds_dot_seg8(const uint8_t* wseg, int steps, int lane, const float (&xr)[kDsMaxSteps][8]) {
  const uint2* wp = reinterpret_cast<const uint2*>(wseg) + lane;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
  for (int j = 0; j < kDsMaxSteps; ++j) {
    if (j < steps) {
      const uint2 w = wp[j * 32];
      float2 f = e4m3x2_to_float2(w.x);
      a0 = fmaf(f.x, xr[j][0], a0); a1 = fmaf(f.y, xr[j][1], a1);
      f = e4m3x2_to_float2(w.x >> 16);
      a2 = fmaf(f.x, xr[j][2], a2); a3 = fmaf(f.y, xr[j][3], a3);
      f = e4m3x2_to_float2(w.y);
      a0 = fmaf(f.x, xr[j][4], a0); a1 = fmaf(f.y, xr[j][5], a1);
      f = e4m3x2_to_float2(w.y >> 16);
      a2 = fmaf(f.x, xr[j][6], a2); a3 = fmaf(f.y, xr[j][7], a3);
    }
  }
  return warp_sum((a0 + a1) + (a2 + a3));
}

// sampling state of the lm_head phase (lane 0 of every consumer warp follows its own rows)
struct DsSample {
  bool greedy;
  float invT;
  uint64_t seed, call_id;
  ArgMax best;
};
SSDK_DEVINL float ds_score(const DsSample& s, float logit, int idx) {
  if (s.greedy) return logit;
  // scores = softmax(l/T) / (E + 1e-10) in the log domain, the very expression of sample_kernel (sampling.cuh)
  const uint4 rnd = philox_draw((uint32_t)(idx >> 2), 0u, s.call_id, TAG_SAMPLE, s.seed);
  const float e = u32_to_exp1(u4_word(rnd, idx & 3)) + 1e-10f;
  return logit * s.invT - __logf(e);
}

// row 0 of a two-row forward 0: its x (a norm output in shared memory, or an L2-resident vector) and its output
struct DsRow0 {
  const float* xs;
  const __nv_bfloat16* xg;
  __nv_bfloat16* y;
};
// row 0's dot product: ds_dot_seg's arithmetic, with x read step by step from shared memory (a second x slice held in
// registers for the whole phase does not fit next to row 1's: the kernel is at its register limit, 168 per thread)
SSDK_DEVINL float ds_dot_seg0(const uint8_t* wseg, int steps, int lane, const float* x0) {
  const uint4* wp = reinterpret_cast<const uint4*>(wseg) + lane;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 2
  for (int j = 0; j < steps; ++j) {
    const float4 u = *reinterpret_cast<const float4*>(x0 + j * 256 + lane * 8);
    const float4 v = *reinterpret_cast<const float4*>(x0 + j * 256 + lane * 8 + 4);
    const uint4 w = wp[j * 32];
    float2 f = ds_bf2(w.x);
    a0 = fmaf(f.x, u.x, a0); a1 = fmaf(f.y, u.y, a1);
    f = ds_bf2(w.y);
    a2 = fmaf(f.x, u.z, a2); a3 = fmaf(f.y, u.w, a3);
    f = ds_bf2(w.z);
    a0 = fmaf(f.x, v.x, a0); a1 = fmaf(f.y, v.y, a1);
    f = ds_bf2(w.w);
    a2 = fmaf(f.x, v.z, a2); a3 = fmaf(f.y, v.w, a3);
  }
  return warp_sum((a0 + a1) + (a2 + a3));
}
// the same for an e4m3 row segment (ds_dot_seg8's arithmetic)
SSDK_DEVINL float ds_dot_seg08(const uint8_t* wseg, int steps, int lane, const float* x0) {
  const uint2* wp = reinterpret_cast<const uint2*>(wseg) + lane;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 2
  for (int j = 0; j < steps; ++j) {
    const float4 u = *reinterpret_cast<const float4*>(x0 + j * 256 + lane * 8);
    const float4 v = *reinterpret_cast<const float4*>(x0 + j * 256 + lane * 8 + 4);
    const uint2 w = wp[j * 32];
    float2 f = e4m3x2_to_float2(w.x);
    a0 = fmaf(f.x, u.x, a0); a1 = fmaf(f.y, u.y, a1);
    f = e4m3x2_to_float2(w.x >> 16);
    a2 = fmaf(f.x, u.z, a2); a3 = fmaf(f.y, u.w, a3);
    f = e4m3x2_to_float2(w.y);
    a0 = fmaf(f.x, v.x, a0); a1 = fmaf(f.y, v.y, a1);
    f = e4m3x2_to_float2(w.y >> 16);
    a2 = fmaf(f.x, v.z, a2); a3 = fmaf(f.y, v.w, a3);
  }
  return warp_sum((a0 + a1) + (a2 + a3));
}
SSDK_DEVINL void ds_load_vec(const __nv_bfloat16* v, int n, float* xs);
// row 0's x in shared memory: r.xs as is, or r.xg (an L2-resident vector of n elements) staged into xs once every warp
// holds row 1's x slice in registers
SSDK_DEVINL const float* ds_row0_x(const DsRow0& r, float* xs, int n) {
  if (r.xs) return r.xs;
  ds_sync();
  ds_load_vec(r.xg, n, xs);
  return xs;
}

// rows of a K <= 2048 matrix: y[row] = bf16(W[row] . x)   (HEAD: logits + the warp's running best score)
// TWO: the same for row 0 from the same slot (its dot product is the one-row arithmetic on its own x)
template <bool HEAD, bool TWO = false>
SSDK_DEVINL void ds_consume_plain(DsRing& ring, const DsGeom& g, float* xs, __nv_bfloat16* y, DsSample* smp,
                                  const DsRow0& r0 = DsRow0{}) {
  static_assert(!(HEAD && TWO), "row 0 has no lm_head");
  if ((int)blockIdx.x >= g.nj) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int steps = g.K >> 8;
  float xr[kDsMaxSteps][8];
  ds_load_x(xs, steps, lane, xr);
  const float* x0 = nullptr;
  if constexpr (TWO) x0 = ds_row0_x(r0, xs, g.K);
  for (int s = (int)blockIdx.x; s < g.nj; s += (int)gridDim.x) {
    const uint8_t* st = ds_acquire(ring, 0);
    const float acc = ds_dot_seg(st + (size_t)warp * g.K * 2, steps, lane, xr);
    float acc0 = 0.f;
    if constexpr (TWO) acc0 = ds_dot_seg0(st + (size_t)warp * g.K * 2, steps, lane, x0);
    ds_release(ring, 0, lane);
    ring.taken += 1u;
    const int row = s * 8 + warp;
    if (lane == 0 && row < g.rows) {
      const __nv_bfloat16 o = f2bf(acc);
      if (!HEAD) {
        y[row] = o;
        if constexpr (TWO) r0.y[row] = f2bf(acc0);
      } else {
        if (y) y[row] = o;
        smp->best = argmax_better(smp->best, ArgMax{ds_score(*smp, bf2f(o), row), row});
      }
    }
  }
}
// gate|up pairs: act[i] = bf16(silu(bf16 g_i) * bf16 u_i)   (layers/activation.py:11-14 on the bf16-rounded linear output)
SSDK_DEVINL float ds_silu_mul(float gate, float up) {
  gate = bf16_round(gate);
  up = bf16_round(up);
  return (gate / (1.0f + __expf(-gate))) * up;
}
template <bool TWO>
SSDK_DEVINL void ds_consume_pair(DsRing& ring, const DsGeom& g, float* xs, __nv_bfloat16* act, const DsRow0& r0) {
  if ((int)blockIdx.x >= g.nj) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int steps = g.K >> 8;
  float xr[kDsMaxSteps][8];
  ds_load_x(xs, steps, lane, xr);
  const float* x0 = nullptr;
  if constexpr (TWO) x0 = ds_row0_x(r0, xs, g.K);
  for (int s = (int)blockIdx.x; s < g.nj; s += (int)gridDim.x) {
    float gate0 = 0.f, up0 = 0.f;
    const uint8_t* sg = ds_acquire(ring, 0);
    const float gate = ds_dot_seg(sg + (size_t)warp * g.K * 2, steps, lane, xr);
    if constexpr (TWO) gate0 = ds_dot_seg0(sg + (size_t)warp * g.K * 2, steps, lane, x0);
    ds_release(ring, 0, lane);
    const uint8_t* su = ds_acquire(ring, 1);
    const float up = ds_dot_seg(su + (size_t)warp * g.K * 2, steps, lane, xr);
    if constexpr (TWO) up0 = ds_dot_seg0(su + (size_t)warp * g.K * 2, steps, lane, x0);
    ds_release(ring, 1, lane);
    ring.taken += 2u;
    const int i = s * 8 + warp;
    if (lane == 0 && i < g.rows) {
      act[i] = f2bf(ds_silu_mul(gate, up));
      if constexpr (TWO) r0.y[i] = f2bf(ds_silu_mul(gate0, up0));
    }
  }
}
// rows of a K > 2048 matrix: the warps split (row, K segment) units; partial sums meet in shared memory, summed in
// segment order.  res: [2 rows][2 buffers][kDsWarps]
template <bool TWO>
SSDK_DEVINL void ds_consume_split(DsRing& ring, const DsGeom& g, float* xs, float* res, __nv_bfloat16* y,
                                  const DsRow0& r0) {
  if ((int)blockIdx.x >= g.nj) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row_in_job = warp / g.segs, seg = warp - row_in_job * g.segs;
  const int seg_len = g.K / g.segs, steps = seg_len >> 8;
  float xr[kDsMaxSteps][8];
  ds_load_x(xs + seg * seg_len, steps, lane, xr);
  const float* x0 = nullptr;
  if constexpr (TWO) x0 = ds_row0_x(r0, xs, g.K);
  const size_t w_off = ((size_t)row_in_job * g.K + (size_t)seg * seg_len) * 2;
  unsigned it = 0;
  for (int s = (int)blockIdx.x; s < g.nj; s += (int)gridDim.x, ++it) {
    const uint8_t* st = ds_acquire(ring, 0);
    const float acc = ds_dot_seg(st + w_off, steps, lane, xr);
    float acc0 = 0.f;
    if constexpr (TWO) acc0 = ds_dot_seg0(st + w_off, steps, lane, x0 + seg * seg_len);
    ds_release(ring, 0, lane);
    ring.taken += 1u;
    float* rb = res + (it & 1u) * kDsWarps;  // double buffered: the readers of job i may still be busy while job i+1 is summed
    float* rb0 = rb + 2 * kDsWarps;
    if (lane == 0) {
      rb[warp] = acc;
      if constexpr (TWO) rb0[warp] = acc0;
    }
    ds_sync();
    if ((int)threadIdx.x < g.rpj) {
      const int row = s * g.rpj + (int)threadIdx.x;
      if (row < g.rows) {
        float v = 0.f;
        for (int q = 0; q < g.segs; ++q) v += rb[(int)threadIdx.x * g.segs + q];
        y[row] = f2bf(v);
        if constexpr (TWO) {
          float v0 = 0.f;
          for (int q = 0; q < g.segs; ++q) v0 += rb0[(int)threadIdx.x * g.segs + q];
          r0.y[row] = f2bf(v0);
        }
      }
    }
  }
}

// ---- FP8 (e4m3) forms of the three consume shapes: two rows per warp (see the top of the file), each output
//      y = bf16(s * dot) with the row scale s requested before the slot is waited for ----
// K <= 2048: 16 rows per slot, warp w owns rows w and w + 8
template <bool TWO>
SSDK_DEVINL void ds_consume_plain8(DsRing& ring, const DsGeom& g, float* xs, __nv_bfloat16* y, const DsRow0& r0,
                                   const float* scale) {
  if ((int)blockIdx.x >= g.nj) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int steps = g.K >> 8;
  float xr[kDsMaxSteps][8];
  ds_load_x(xs, steps, lane, xr);
  const float* x0 = nullptr;
  if constexpr (TWO) x0 = ds_row0_x(r0, xs, g.K);
  for (int s = (int)blockIdx.x; s < g.nj; s += (int)gridDim.x) {
    const int ra = s * 16 + warp, rb = ra + 8;
    const float sa = ra < g.rows ? scale[ra] : 0.f, sb = rb < g.rows ? scale[rb] : 0.f;
    const uint8_t* wa = ds_acquire(ring, 0) + (size_t)warp * g.K;
    const uint8_t* wb = wa + (size_t)8 * g.K;
    const float acc_a = ds_dot_seg8(wa, steps, lane, xr);
    const float acc_b = ds_dot_seg8(wb, steps, lane, xr);
    float acc0_a = 0.f, acc0_b = 0.f;
    if constexpr (TWO) {
      acc0_a = ds_dot_seg08(wa, steps, lane, x0);
      acc0_b = ds_dot_seg08(wb, steps, lane, x0);
    }
    ds_release(ring, 0, lane);
    ring.taken += 1u;
    if (lane == 0) {
      if (ra < g.rows) {
        y[ra] = f2bf(acc_a * sa);
        if constexpr (TWO) r0.y[ra] = f2bf(acc0_a * sa);
      }
      if (rb < g.rows) {
        y[rb] = f2bf(acc_b * sb);
        if constexpr (TWO) r0.y[rb] = f2bf(acc0_b * sb);
      }
    }
  }
}
// gate|up: 16 pairs per job (16 gate rows | the 16 matching up rows), warp w owns pairs w and w + 8; gate and up are
// scaled each by its own row scale (scale[i] and scale[g.rows + i]) before SiLU
template <bool TWO>
SSDK_DEVINL void ds_consume_pair8(DsRing& ring, const DsGeom& g, float* xs, __nv_bfloat16* act, const DsRow0& r0,
                                  const float* scale) {
  if ((int)blockIdx.x >= g.nj) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int steps = g.K >> 8;
  float xr[kDsMaxSteps][8];
  ds_load_x(xs, steps, lane, xr);
  const float* x0 = nullptr;
  if constexpr (TWO) x0 = ds_row0_x(r0, xs, g.K);
  for (int s = (int)blockIdx.x; s < g.nj; s += (int)gridDim.x) {
    const int ia = s * 16 + warp, ib = ia + 8;
    const float sga = ia < g.rows ? scale[ia] : 0.f, sua = ia < g.rows ? scale[g.rows + ia] : 0.f;
    const float sgb = ib < g.rows ? scale[ib] : 0.f, sub = ib < g.rows ? scale[g.rows + ib] : 0.f;
    float ga0 = 0.f, gb0 = 0.f, ua0 = 0.f, ub0 = 0.f;
    const uint8_t* sg = ds_acquire(ring, 0) + (size_t)warp * g.K;
    const float ga = ds_dot_seg8(sg, steps, lane, xr);
    const float gb = ds_dot_seg8(sg + (size_t)8 * g.K, steps, lane, xr);
    if constexpr (TWO) {
      ga0 = ds_dot_seg08(sg, steps, lane, x0);
      gb0 = ds_dot_seg08(sg + (size_t)8 * g.K, steps, lane, x0);
    }
    ds_release(ring, 0, lane);
    const uint8_t* su = ds_acquire(ring, 1) + (size_t)warp * g.K;
    const float ua = ds_dot_seg8(su, steps, lane, xr);
    const float ub = ds_dot_seg8(su + (size_t)8 * g.K, steps, lane, xr);
    if constexpr (TWO) {
      ua0 = ds_dot_seg08(su, steps, lane, x0);
      ub0 = ds_dot_seg08(su + (size_t)8 * g.K, steps, lane, x0);
    }
    ds_release(ring, 1, lane);
    ring.taken += 2u;
    if (lane == 0) {
      if (ia < g.rows) {
        act[ia] = f2bf(ds_silu_mul(ga * sga, ua * sua));
        if constexpr (TWO) r0.y[ia] = f2bf(ds_silu_mul(ga0 * sga, ua0 * sua));
      }
      if (ib < g.rows) {
        act[ib] = f2bf(ds_silu_mul(gb * sgb, ub * sub));
        if constexpr (TWO) r0.y[ib] = f2bf(ds_silu_mul(gb0 * sgb, ub0 * sub));
      }
    }
  }
}
// K > 2048: 2R rows per slot (R = kDsWarps / segs, the bf16 rows per job); warp w owns (row w / segs, segment w % segs)
// of both R-row groups.  Partial sums meet in shared memory and are summed in segment order, then scaled.
// res: [2 rows][2 buffers][2 groups][kDsWarps]
template <bool TWO>
SSDK_DEVINL void ds_consume_split8(DsRing& ring, const DsGeom& g, float* xs, float* res, __nv_bfloat16* y,
                                   const DsRow0& r0, const float* scale) {
  if ((int)blockIdx.x >= g.nj) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int R = kDsWarps / g.segs;
  const int row_in_job = warp / g.segs, seg = warp - row_in_job * g.segs;
  const int seg_len = g.K / g.segs, steps = seg_len >> 8;
  float xr[kDsMaxSteps][8];
  ds_load_x(xs + seg * seg_len, steps, lane, xr);
  const float* x0 = nullptr;
  if constexpr (TWO) x0 = ds_row0_x(r0, xs, g.K) + seg * seg_len;
  const size_t off_a = (size_t)row_in_job * g.K + (size_t)seg * seg_len, off_b = off_a + (size_t)R * g.K;
  unsigned it = 0;
  for (int s = (int)blockIdx.x; s < g.nj; s += (int)gridDim.x, ++it) {
    const int row = s * g.rpj + (int)threadIdx.x;  // the output row of a reducing thread (threadIdx.x < g.rpj)
    const float sc = ((int)threadIdx.x < g.rpj && row < g.rows) ? scale[row] : 0.f;
    const uint8_t* st = ds_acquire(ring, 0);
    const float acc_a = ds_dot_seg8(st + off_a, steps, lane, xr);
    const float acc_b = ds_dot_seg8(st + off_b, steps, lane, xr);
    float acc0_a = 0.f, acc0_b = 0.f;
    if constexpr (TWO) {
      acc0_a = ds_dot_seg08(st + off_a, steps, lane, x0);
      acc0_b = ds_dot_seg08(st + off_b, steps, lane, x0);
    }
    ds_release(ring, 0, lane);
    ring.taken += 1u;
    float* rb = res + (it & 1u) * 2 * kDsWarps;  // double buffered, as in ds_consume_split
    float* rb0 = rb + 4 * kDsWarps;
    if (lane == 0) {
      rb[warp] = acc_a;
      rb[kDsWarps + warp] = acc_b;
      if constexpr (TWO) {
        rb0[warp] = acc0_a;
        rb0[kDsWarps + warp] = acc0_b;
      }
    }
    ds_sync();
    if ((int)threadIdx.x < g.rpj && row < g.rows) {
      const int grp = (int)threadIdx.x / R;
      const int base = grp * kDsWarps + ((int)threadIdx.x - grp * R) * g.segs;
      float v = 0.f;
      for (int q = 0; q < g.segs; ++q) v += rb[base + q];
      y[row] = f2bf(v * sc);
      if constexpr (TWO) {
        float v0 = 0.f;
        for (int q = 0; q < g.segs; ++q) v0 += rb0[base + q];
        r0.y[row] = f2bf(v0 * sc);
      }
    }
  }
}

// two: two rows (row 0 = r0).  FP8: e4m3 weights with the per-row scales `scale`
template <bool FP8 = false>
SSDK_DEVINL void ds_consume(DsRing& ring, const DsGeom& g, float* xs, float* res, __nv_bfloat16* y, bool two,
                            const DsRow0& r0, const float* scale = nullptr) {
  if constexpr (FP8) {
    if (g.kind == DS_PLAIN) {
      if (two) ds_consume_plain8<true>(ring, g, xs, y, r0, scale);
      else ds_consume_plain8<false>(ring, g, xs, y, r0, scale);
    } else {
      if (two) ds_consume_split8<true>(ring, g, xs, res, y, r0, scale);
      else ds_consume_split8<false>(ring, g, xs, res, y, r0, scale);
    }
  } else {
    if (g.kind == DS_PLAIN) {
      if (two) ds_consume_plain<false, true>(ring, g, xs, y, nullptr, r0);
      else ds_consume_plain<false>(ring, g, xs, y, nullptr);
    } else {
      if (two) ds_consume_split<true>(ring, g, xs, res, y, r0);
      else ds_consume_split<false>(ring, g, xs, res, y, r0);
    }
  }
}
template <bool FP8 = false>
SSDK_DEVINL void ds_consume_gu(DsRing& ring, const DsGeom& g, float* xs, __nv_bfloat16* act, bool two, const DsRow0& r0,
                               const float* scale = nullptr) {
  if constexpr (FP8) {
    if (two) ds_consume_pair8<true>(ring, g, xs, act, r0, scale);
    else ds_consume_pair8<false>(ring, g, xs, act, r0, scale);
  } else {
    if (two) ds_consume_pair<true>(ring, g, xs, act, r0);
    else ds_consume_pair<false>(ring, g, xs, act, r0);
  }
}

SSDK_DEVINL float ds_block_sum(float v, float* red) {  // all consumer threads get the result
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  v = warp_sum(v);
  ds_sync();
  if (lane == 0) red[wid] = v;
  ds_sync();
  float t = (lane < kDsWarps) ? red[lane] : 0.f;
  return warp_sum(t);
}

// xs[i] = bf16r( r_i * rsqrt(mean r^2 + eps) * w_i ),  r = a (+ b) in fp32;  resid_out = bf16(r) (written by CTA 0 only).
// a / b are L2-resident vectors produced by earlier phases.  d is a multiple of 8.
// The operands of a norm prologue that do NOT depend on the phase that just ended — the norm weight (first touch of a layer:
// an HBM miss) and the residual written one phase earlier — are requested BEFORE the device-wide barrier and ride it out in
// registers (first 8-element slice of the thread; d > 8 * kDsConsumers loads the rest inside the prologue).
struct DsPre {
  uint4 w, b;
};
SSDK_DEVINL DsPre ds_preload(const __nv_bfloat16* b, const __nv_bfloat16* w, int d) {
  DsPre r;
  const int i = threadIdx.x * 8;
  r.w = r.b = make_uint4(0u, 0u, 0u, 0u);
  if (i < d) {
    r.w = *reinterpret_cast<const uint4*>(w + i);
    if (b) r.b = ds_ldcg16(b + i);
  }
  return r;
}
SSDK_DEVINL void ds_norm_prologue(const __nv_bfloat16* a, const __nv_bfloat16* b, __nv_bfloat16* resid_out,
                                  const __nv_bfloat16* w, float eps, int d, float* xs, float* red, const DsPre* pre) {
  float ss = 0.f;
  const int i0 = threadIdx.x * 8;
  for (int i = i0; i < d; i += kDsConsumers * 8) {
    float x[8];
    unpack_bf16x8(ds_ldcg16(a + i), x);
    if (b) {
      float y[8];
      unpack_bf16x8((pre && i == i0) ? pre->b : ds_ldcg16(b + i), y);
#pragma unroll
      for (int j = 0; j < 8; ++j) x[j] += y[j];
    }
    if (resid_out && blockIdx.x == 0) *reinterpret_cast<uint4*>(resid_out + i) = pack_bf16x8(x);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      xs[i + j] = x[j];
      ss += x[j] * x[j];
    }
  }
  ss = ds_block_sum(ss, red);
  const float rstd = rsqrtf(ss / (float)d + eps);
  for (int i = i0; i < d; i += kDsConsumers * 8) {
    float wv[8];
    unpack_bf16x8((pre && i == i0) ? pre->w : *reinterpret_cast<const uint4*>(w + i), wv);
#pragma unroll
    for (int j = 0; j < 8; ++j) xs[i + j] = bf16_round(xs[i + j] * rstd * wv[j]);
  }
  ds_sync();
}
// xs = fp32(v[0 .. n)) for an L2-resident bf16 vector
SSDK_DEVINL void ds_load_vec(const __nv_bfloat16* v, int n, float* xs) {
  for (int i = threadIdx.x * 8; i < n; i += kDsConsumers * 8) {
    float x[8];
    unpack_bf16x8(ds_ldcg16(v + i), x);
#pragma unroll
    for (int j = 0; j < 8; ++j) xs[i + j] = x[j];
  }
  ds_sync();
}

// ---------------------------------------------------------------------------------------------
// phase B unit: kv head h, split s.  Rebuilds the rotated q rows of the head group and the new token's k / v from the
// q|k|v vector, stores k / v into the page slot (split 0 only), runs the online-softmax over its token range (the new
// token comes from shared memory, never from the cache) and writes (o, m, l) per query head.
// ---------------------------------------------------------------------------------------------
// KV splits per kv head: kDsShortSplits as soon as every split has a few tokens (64 units keep 64 SMs busy for one or two
// 4-token iterations per warp); a single split only for the first tokens of a sequence.  (One split per 256 tokens looked
// attractive — no partials, ticket or merge below 256 — but the token loop is a chain of dependent L2 round trips per
// iteration: measured 8B + 1B 10.29 vs 8.34 ms/step.)
// The phase is bound by the number of dependent load ROUNDS per split (a round = warps x tokens in flight; each further
// round measured 5 - 8 us per layer): up to 256 tokens 8 splits x 8 warps x 4 tokens cover the context in one round; beyond,
// 16 splits per kv head (128 units for 8 kv heads) and 8 tokens per warp iteration keep it at one round up to 1024 tokens
// (the engine takes the kernel-per-op draft for longer contexts, use_draft_stream in engine.cu).
SSDK_DEVINL int ds_num_splits(int ctx) {
  return ctx > kDsLongCtx ? kDsSplits : min(kDsShortSplits, max(1, (ctx + 7) >> 3));
}
// page of token t: from the shared-memory copy of the (launch-constant) page table when it fits, else from global memory
SSDK_DEVINL int ds_page_of(const DsParams& p, const int* bt_s, int t) {
  const int i = t / p.block_size;
  return p.max_blocks <= kDsBtSmem ? bt_s[i] : p.block_table[i];
}
// K and V slices of TB tokens (tb, tb + kDsWarps, ...) of kv head h into registers; the new token (t == pos) and tokens past
// the split's end are left zero (the new token's k / v come from shared memory when the scores are computed)
template <int HD, int TB>
SSDK_DEVINL void ds_load_kv(const DsParams& p, const int* bt_s, const __nv_bfloat16* kbase, const __nv_bfloat16* vbase, int h,
                            int tb, int t1, int pos, int lane, float (&kv)[TB][HD / 32], float (&vv)[TB][HD / 32]) {
  constexpr int EPL = HD / 32;
  static_assert(EPL == 2 || EPL == 4, "head_dim 64 or 128");
#pragma unroll
  for (int u = 0; u < TB; ++u) {
    const int t = tb + u * kDsWarps;
#pragma unroll
    for (int e = 0; e < EPL; ++e) kv[u][e] = vv[u][e] = 0.f;
    if (t < t1 && t != pos) {
      const int blk = ds_page_of(p, bt_s, t);
      const size_t off = (((size_t)blk * p.block_size + t % p.block_size) * p.KV + h) * HD + lane * EPL;
      if constexpr (EPL == 2) {
        const float2 a = ds_bf2(__ldcg(reinterpret_cast<const uint32_t*>(kbase + off)));
        const float2 b = ds_bf2(__ldcg(reinterpret_cast<const uint32_t*>(vbase + off)));
        kv[u][0] = a.x; kv[u][1] = a.y; vv[u][0] = b.x; vv[u][1] = b.y;
      } else {
        const uint2 a = __ldcg(reinterpret_cast<const uint2*>(kbase + off));
        const uint2 b = __ldcg(reinterpret_cast<const uint2*>(vbase + off));
        float2 f = ds_bf2(a.x); kv[u][0] = f.x; kv[u][1] = f.y;
        f = ds_bf2(a.y); kv[u][EPL - 2] = f.x; kv[u][EPL - 1] = f.y;
        f = ds_bf2(b.x); vv[u][0] = f.x; vv[u][1] = f.y;
        f = ds_bf2(b.y); vv[u][EPL - 2] = f.x; vv[u][EPL - 1] = f.y;
      }
    }
  }
}
// vqkv / vattn: the q|k|v input and the attention output of the row (row 1: p.vec_qkv / p.vec_attn)
template <int HD, int GMAX, int TB>  // TB = tokens per warp iteration
SSDK_DEVINL void ds_attention_unit(const DsParams& p, const __nv_bfloat16* vqkv, __nv_bfloat16* vattn, int layer, int h,
                                   int s, int ns, int ctx, float* sm, int* flag, const int* bt_s) {
  constexpr int HALF = HD / 2;
  constexpr int EPL = HD / 32;  // elements per lane in the dot layout (dims lane*EPL ..)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int G = p.H / p.KV;
  const int pos = ctx - 1;
  float* sq = sm;                      // [G][HD] rotated q (bf16-rounded values)
  float* sk = sq + GMAX * HD;          // [HD] new k
  float* sv = sk + HD;                 // [HD] new v
  float* sred = sv + HD;               // [kDsWarps][G][HD + 2] per-warp partials

  // ---- token range of this split; the cached K / V of the first warp iteration are requested NOW: they do not depend on
  //      phase A, so their L2 / HBM round trip overlaps the one of the q|k|v vector below ----
  const int per = (ctx + ns - 1) / ns;
  const int t0 = s * per, t1 = min(ctx, t0 + per);
  const __nv_bfloat16* kbase = p.k_cache + (size_t)layer * p.cache_layer_stride;
  const __nv_bfloat16* vbase = p.v_cache + (size_t)layer * p.cache_layer_stride;
  float kv[TB][EPL], vv[TB][EPL];
  ds_load_kv<HD, TB>(p, bt_s, kbase, vbase, h, t0 + warp, t1, pos, lane, kv, vv);

  // ---- q rows, k, v: one warp per row, rotate-half pairs (i, i + HALF) ----
  const float* cs = p.rope + (size_t)pos * HD;
  for (int row = warp; row < G + 2; row += kDsWarps) {
    const int kind = row < G ? 0 : (row == G ? 1 : 2);
    const int col0 = (kind == 0 ? (h * G + row) : (kind == 1 ? p.H + h : p.H + p.KV + h)) * HD;
    float x1[(HALF + 31) / 32], x2[(HALF + 31) / 32];
    float ss = 0.f;
    // plain L2 loads (the vector was written by other SMs in phase A)
#pragma unroll
    for (int t = 0; t < (HALF + 31) / 32; ++t) {
      const int i = lane + 32 * t;
      x1[t] = x2[t] = 0.f;
      if (i < HALF) {
        const unsigned short a = __ldcg(reinterpret_cast<const unsigned short*>(vqkv + col0 + i));
        const unsigned short b = __ldcg(reinterpret_cast<const unsigned short*>(vqkv + col0 + HALF + i));
        x1[t] = __bfloat162float(__ushort_as_bfloat16(a));
        x2[t] = __bfloat162float(__ushort_as_bfloat16(b));
        ss += x1[t] * x1[t] + x2[t] * x2[t];
      }
    }
    float* dst = kind == 0 ? sq + row * HD : (kind == 1 ? sk : sv);
    if (kind == 2) {
#pragma unroll
      for (int t = 0; t < (HALF + 31) / 32; ++t) {
        const int i = lane + 32 * t;
        if (i < HALF) {
          dst[i] = x1[t];
          dst[HALF + i] = x2[t];
        }
      }
      continue;
    }
    const __nv_bfloat16* nw = p.qk_norm ? (kind == 0 ? p.layers[layer].q_norm : p.layers[layer].k_norm) : nullptr;
    if (nw) {
      ss = warp_sum(ss);
      const float rstd = rsqrtf(ss / (float)HD + p.eps);
#pragma unroll
      for (int t = 0; t < (HALF + 31) / 32; ++t) {
        const int i = lane + 32 * t;
        if (i < HALF) {
          x1[t] = bf16_round(x1[t] * rstd * bf2f(nw[i]));
          x2[t] = bf16_round(x2[t] * rstd * bf2f(nw[HALF + i]));
        }
      }
    }
#pragma unroll
    for (int t = 0; t < (HALF + 31) / 32; ++t) {
      const int i = lane + 32 * t;
      if (i < HALF) {
        const float c = cs[i], sn = cs[HALF + i];
        dst[i] = bf16_round(x1[t] * c - x2[t] * sn);
        dst[HALF + i] = bf16_round(x2[t] * c + x1[t] * sn);
      }
    }
  }
  ds_sync();

  // ---- KV store of the new token (one unit per kv head) ----
  const int blk_new = ds_page_of(p, bt_s, pos);
  if (s == 0 && blk_new >= 0) {
    const size_t slot = (size_t)blk_new * p.block_size + pos % p.block_size;
    __nv_bfloat16* kc = p.k_cache + (size_t)layer * p.cache_layer_stride + (slot * p.KV + h) * HD;
    __nv_bfloat16* vc = p.v_cache + (size_t)layer * p.cache_layer_stride + (slot * p.KV + h) * HD;
    for (int i = threadIdx.x; i < HD; i += kDsConsumers) {
      kc[i] = f2bf(sk[i]);
      vc[i] = f2bf(sv[i]);
    }
  }

  // dot layout: lane owns dims [lane * EPL, lane * EPL + EPL)
  float qreg[GMAX][EPL];
#pragma unroll
  for (int g = 0; g < GMAX; ++g)
#pragma unroll
    for (int e = 0; e < EPL; ++e) qreg[g][e] = (g < G) ? sq[g * HD + lane * EPL + e] : 0.f;
  float m[GMAX], l[GMAX], acc[GMAX][EPL];
#pragma unroll
  for (int g = 0; g < GMAX; ++g) {
    m[g] = -INFINITY;
    l[g] = 0.f;
#pragma unroll
    for (int e = 0; e < EPL; ++e) acc[g][e] = 0.f;
  }
  // TB tokens per warp iteration: all 2 TB K / V loads are in flight before the first score is computed (one token
  // per iteration exposed a full L2 / HBM round trip per token)
  for (int tb = t0 + warp; tb < t1; tb += TB * kDsWarps) {
    if (tb != t0 + warp) ds_load_kv<HD, TB>(p, bt_s, kbase, vbase, h, tb, t1, pos, lane, kv, vv);
#pragma unroll
    for (int u = 0; u < TB; ++u) {
      const int t = tb + u * kDsWarps;
      if (t < t1) {
        if (t == pos) {
#pragma unroll
          for (int e = 0; e < EPL; ++e) {
            kv[u][e] = sk[lane * EPL + e];
            vv[u][e] = sv[lane * EPL + e];
          }
        }
#pragma unroll
        for (int g = 0; g < GMAX; ++g) {
          if (g < G) {
            float sc = 0.f;
#pragma unroll
            for (int e = 0; e < EPL; ++e) sc = fmaf(qreg[g][e], kv[u][e], sc);
            sc = warp_sum(sc) * p.scale_log2;
            const float mn = fmaxf(m[g], sc);
            const float corr = exp2f(m[g] - mn);  // m = -inf -> 0
            const float pr = exp2f(sc - mn);
            l[g] = l[g] * corr + pr;
#pragma unroll
            for (int e = 0; e < EPL; ++e) acc[g][e] = acc[g][e] * corr + pr * vv[u][e];
            m[g] = mn;
          }
        }
      }
    }
  }
  // ---- merge the warps through shared memory, one thread per (head, dim) ----
  constexpr int LDR = HD + 2;
#pragma unroll
  for (int g = 0; g < GMAX; ++g) {
    if (g < G) {
      float* w = sred + ((size_t)warp * G + g) * LDR;
#pragma unroll
      for (int e = 0; e < EPL; ++e) w[lane * EPL + e] = acc[g][e];
      if (lane == 0) {
        w[HD] = m[g];
        w[HD + 1] = l[g];
      }
    }
  }
  ds_sync();
  for (int idx = threadIdx.x; idx < G * HD; idx += kDsConsumers) {
    const int g = idx / HD, dim = idx - g * HD;
    float mx = -INFINITY;
    for (int w = 0; w < kDsWarps; ++w) mx = fmaxf(mx, sred[((size_t)w * G + g) * LDR + HD]);
    float o = 0.f, ll = 0.f;
    if (mx != -INFINITY) {
      for (int w = 0; w < kDsWarps; ++w) {
        const float* r = sred + ((size_t)w * G + g) * LDR;
        const float wt = exp2f(r[HD] - mx);
        o += r[dim] * wt;
        ll += r[HD + 1] * wt;
      }
    }
    if (ns == 1) {  // the only split: this is the attention output
      vattn[(size_t)(h * G + g) * HD + dim] = f2bf(ll > 0.f ? o / ll : 0.f);
    } else {
      float* out = p.attn_part + ((size_t)(h * G + g) * kDsSplits + s) * LDR;
      out[dim] = o;  // un-normalised: sum_t 2^(s_t - mx) v_t
      if (dim == 0) {
        out[HD] = mx;
        out[HD + 1] = ll;
      }
    }
  }
  if (ns == 1) {
    ds_sync();  // scratch is reused by the next unit of this CTA
    return;
  }
  // ---- the LAST split of this kv head to finish merges the head group's partials into the attention output vector, so
  //      that phase C only has to load 2 * H * HD bytes (every CTA merging every head cost ~7 us per layer) ----
  ds_sync();  // the partials of every thread are ordered before thread 0's acq_rel ticket
  if (threadIdx.x == 0) *flag = (atom_add_acq_rel_gpu(p.attn_ticket + h, 1u) == (unsigned)ns - 1u) ? 1 : 0;
  ds_sync();
  if (*flag) {
    if (threadIdx.x == 0) st_relaxed_gpu_u32(p.attn_ticket + h, 0u);  // next use: a later phase B, device-wide barriers away
    for (int idx = threadIdx.x; idx < G * HD; idx += kDsConsumers) {
      const int g = idx / HD, dim = idx - g * HD;
      const float* base = p.attn_part + (size_t)(h * G + g) * kDsSplits * LDR;
      float ms[kDsSplits], ls[kDsSplits], os[kDsSplits];
      float mx = -INFINITY;
#pragma unroll
      for (int q = 0; q < kDsSplits; ++q) {
        const bool on = q < ns;
        ms[q] = on ? __ldcg(base + q * LDR + HD) : -INFINITY;
        ls[q] = on ? __ldcg(base + q * LDR + HD + 1) : 0.f;
        os[q] = on ? __ldcg(base + q * LDR + dim) : 0.f;
        mx = fmaxf(mx, ms[q]);
      }
      float o = 0.f, l = 0.f;
#pragma unroll
      for (int q = 0; q < kDsSplits; ++q) {
        const float wt = (ms[q] == -INFINITY) ? 0.f : exp2f(ms[q] - mx);
        o += os[q] * wt;
        l += ls[q] * wt;
      }
      vattn[(size_t)(h * G + g) * HD + dim] = f2bf(l > 0.f ? o / l : 0.f);
    }
  }
  ds_sync();
}


// the row scales of layer l's matrix m (FP8 instance; nullptr in the bf16 one)
template <bool FP8>
SSDK_DEVINL const float* ds_scale(const DsParams& p, int l, int m) {
  if constexpr (FP8) return p.fp8_scale[l][m];
  else return nullptr;
}

// FP8: the decoder linears are e4m3 with per-row scales (p.fp8_scale); embedding, lm_head and norms stay bf16
template <int HD, int GMAX, bool FP8 = false>
__global__ void __launch_bounds__(kDsThreads, 1) draft_stream_kernel(const __grid_constant__ DsParams p) {
  SSDK_DYN_SMEM(uint8_t, ds_smem);
  SSDK_STATIC_SMEM(uint64_t, full_bar, kDsMaxSlots);
  SSDK_STATIC_SMEM(uint64_t, empty_bar, kDsMaxSlots);
  SSDK_STATIC_SMEM(DsGeom, geom, 5);
  SSDK_STATIC_SMEM(float, red, 32);
  SSDK_STATIC_SMEM(float, res, (FP8 ? 8 : 4) * kDsWarps);
  SSDK_STATIC_SMEM(ArgMax, ared, 32);
  SSDK_SHARED_VAR(int, tok_s);
  SSDK_SHARED_VAR(int, flag_s);
  SSDK_STATIC_SMEM(int, bt_s, kDsBtSmem);
  // dynamic shared memory: [ring: n_slots x 32 KB][xs: ds_xs_floats floats][attention scratch]
  float* xs = reinterpret_cast<float*>(ds_smem + (size_t)p.n_slots * kDsSlotBytes);
  float* scratch = xs + ds_xs_floats(p.d, p.ffn, p.H * HD);
  if (threadIdx.x < kDsBtSmem && (int)threadIdx.x < p.max_blocks) bt_s[threadIdx.x] = p.block_table[threadIdx.x];
  if (threadIdx.x == 0) {
    trace_mark(TR_MISC);
    if constexpr (FP8) {
      ds_geometry8(p.d, (p.H + 2 * p.KV) * HD, false, &geom[DS_QKV]);
      ds_geometry8(p.H * HD, p.d, false, &geom[DS_O]);
      ds_geometry8(p.d, p.ffn, true, &geom[DS_GU]);
      ds_geometry8(p.ffn, p.d, false, &geom[DS_DOWN]);
    } else {
      ds_geometry(p.d, (p.H + 2 * p.KV) * HD, false, &geom[DS_QKV]);
      ds_geometry(p.H * HD, p.d, false, &geom[DS_O]);
      ds_geometry(p.d, p.ffn, true, &geom[DS_GU]);
      ds_geometry(p.ffn, p.d, false, &geom[DS_DOWN]);
    }
    ds_geometry(p.d, p.vocab, false, &geom[DS_HEAD]);
    for (int s = 0; s < p.n_slots; ++s) {
      mbar_init(&full_bar[s], 1);           // the producer's arrive.expect_tx + the copy's transaction bytes
      mbar_init(&empty_bar[s], kDsWarps);   // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();  // the only block-wide barrier: mbarriers and the geometry table exist before anybody uses them

  if (threadIdx.x >= kDsConsumers) {
    // ===================== producer warp: the weight stream never waits for a phase =====================
    if (threadIdx.x == kDsConsumers) ds_producer<FP8>(p, geom, ds_smem, full_bar, empty_bar);
    return;
  }

  // ===================== consumer warps =====================
  DsRing ring;
  ring.base = ds_smem;
  ring.full = full_bar;
  ring.empty = empty_bar;
  ring.n_slots = (unsigned)p.n_slots;
  ring.taken = 0u;
  DsGridBar bar;
  bar.counter = reinterpret_cast<unsigned long long*>(p.bar_state);
  bar.target = 0;
  bar.init();

  const int ctx_base = p.ctx0[0];
  const float T = p.temp ? p.temp[0] : 0.f;
  const uint64_t seed = p.dyn ? p.dyn[0] : p.seed;
  const uint64_t call0 = p.dyn ? p.dyn[1] * 16ull : p.call_base;
  __nv_bfloat16* resid[2] = {p.resid0, p.resid1};
  long long tok = p.tok_buf[0];
  // a pending token: forward 0 also runs row 0 (that token at position ctx_base - 1; its x in xs[d, 2d) for the norms)
  const long long tok0 = p.pend_tok ? p.pend_tok[0] : -1;
  const DsVecs v0 = ds_row0_vecs(p, HD);

  for (int f = 0; f < p.n_fwd; ++f) {
    if (threadIdx.x == 0 && f > 0) trace_mark(TR_MISC);
    const int ctx = ctx_base + f + 1;  // tokens visible to this forward, the new one included
    const __nv_bfloat16* emb = p.embed + (size_t)tok * p.d;
    const bool two = f == 0 && tok0 >= 0;
    int cur = 0;  // resid[cur] holds the residual entering the layer (layer 0: the embedding row itself)
    DsPre pre;    // operands of the next norm prologue, requested before the barrier in front of it
    for (int l = 0; l < p.L; ++l) {
      const DsLayer& lw = p.layers[l];
      // ---- A: (add +) input norm -> q|k|v ----
      if (l == 0) {
        // first layer: hidden = norm(embed), residual = embed (models/llama3.py:192-193)
        if (two) ds_norm_prologue(p.embed + (size_t)tok0 * p.d, nullptr, v0.resid(cur ^ 1), lw.in_norm, p.eps, p.d, xs + p.d, red,
                                  nullptr);
        ds_norm_prologue(emb, nullptr, resid[cur ^ 1], lw.in_norm, p.eps, p.d, xs, red, nullptr);
      } else {
        if (two) ds_norm_prologue(v0.down, v0.resid(cur), v0.resid(cur ^ 1), lw.in_norm, p.eps, p.d, xs + p.d, red, nullptr);
        ds_norm_prologue(p.vec_down, resid[cur], resid[cur ^ 1], lw.in_norm, p.eps, p.d, xs, red, &pre);
      }
      cur ^= 1;
      ds_mark(f, 0);
      ds_consume<FP8>(ring, geom[DS_QKV], xs, res, p.vec_qkv, two, DsRow0{xs + p.d, nullptr, v0.qkv},
                      ds_scale<FP8>(p, l, DS_QKV));
      ds_mark(f, 1);
      bar.sync();
      ds_mark(f, 2);
#ifdef SSDK_TRACE_FINE
      bar.sync();  // probe: a second barrier right after the first has no arrival skew -> its duration is the pure latency
      ds_mark(f, 12);
#endif
      // ---- B: RoPE + KV store + attention units (+ merge by the last split of each kv head) ----
      if (two) {
        // row 0 first: its K/V store must be visible (device-wide barrier) before row 1's units read position ctx_base - 1
        const int ns0 = ds_num_splits(ctx - 1);
        for (int u = blockIdx.x; u < p.KV * ns0; u += gridDim.x) {
          if (ns0 == kDsSplits)
            ds_attention_unit<HD, GMAX, 8>(p, v0.qkv, v0.attn, l, u / ns0, u % ns0, ns0, ctx - 1, scratch, &flag_s, bt_s);
          else ds_attention_unit<HD, GMAX, 4>(p, v0.qkv, v0.attn, l, u / ns0, u % ns0, ns0, ctx - 1, scratch, &flag_s, bt_s);
        }
        bar.sync();
      }
      const int ns = ds_num_splits(ctx);
      for (int u = blockIdx.x; u < p.KV * ns; u += gridDim.x) {
        if (ns == kDsSplits)
          ds_attention_unit<HD, GMAX, 8>(p, p.vec_qkv, p.vec_attn, l, u / ns, u % ns, ns, ctx, scratch, &flag_s, bt_s);
        else ds_attention_unit<HD, GMAX, 4>(p, p.vec_qkv, p.vec_attn, l, u / ns, u % ns, ns, ctx, scratch, &flag_s, bt_s);
      }
      ds_mark(f, 3);
      bar.sync();
      ds_mark(f, 4);
      // ---- C: o-proj ----
      ds_load_vec(p.vec_attn, p.H * HD, xs);
      ds_consume<FP8>(ring, geom[DS_O], xs, res, p.vec_o, two, DsRow0{nullptr, v0.attn, v0.o}, ds_scale<FP8>(p, l, DS_O));
      ds_mark(f, 5);
      pre = ds_preload(resid[cur], lw.post_norm, p.d);
      bar.sync();
      ds_mark(f, 6);
      // ---- D: add + post-attention norm -> gate|up with SiLU*mul ----
      if (two) ds_norm_prologue(v0.o, v0.resid(cur), v0.resid(cur ^ 1), lw.post_norm, p.eps, p.d, xs + p.d, red, nullptr);
      ds_norm_prologue(p.vec_o, resid[cur], resid[cur ^ 1], lw.post_norm, p.eps, p.d, xs, red, &pre);
      cur ^= 1;
      ds_mark(f, 7);
      ds_consume_gu<FP8>(ring, geom[DS_GU], xs, p.vec_act, two, DsRow0{xs + p.d, nullptr, v0.act},
                         ds_scale<FP8>(p, l, DS_GU));
      ds_mark(f, 8);
      bar.sync();
      ds_mark(f, 9);
      // ---- E: down-proj ----
      ds_load_vec(p.vec_act, p.ffn, xs);
      ds_consume<FP8>(ring, geom[DS_DOWN], xs, res, p.vec_down, two, DsRow0{nullptr, v0.act, v0.down},
                      ds_scale<FP8>(p, l, DS_DOWN));
      ds_mark(f, 10);
      pre = ds_preload(resid[cur], l + 1 < p.L ? p.layers[l + 1].in_norm : p.final_norm, p.d);
      bar.sync();
      ds_mark(f, 11);
    }
    if (!ds_has_head(p, f)) break;
    // ---- final add + norm (models/llama3.py:198) -> lm_head; logits rounded to bf16 like every linear output ----
    ds_norm_prologue(p.vec_down, resid[cur], nullptr, p.final_norm, p.eps, p.d, xs, red, &pre);
    DsSample smp;
    smp.greedy = (T == 0.f);
    smp.invT = smp.greedy ? 1.f : 1.f / T;
    smp.seed = seed;
    smp.call_id = call0 + (uint64_t)f;
    smp.best = ArgMax{-INFINITY, 0x7fffffff};
    ds_consume_plain<true>(ring, geom[DS_HEAD], xs, p.logits ? p.logits + (size_t)f * p.logits_ld : nullptr, &smp);
    // ---- sampling: per-warp best -> per-CTA best -> device-wide reduction (every CTA learns the token) ----
    if ((threadIdx.x & 31) == 0) ared[threadIdx.x >> 5] = smp.best;
    ds_sync();
    if (threadIdx.x == 0) {
      ArgMax b = ared[0];
      for (int w = 1; w < kDsWarps; ++w) b = argmax_better(b, ared[w]);
      p.samp_partial[blockIdx.x] = b;
    }
    bar.sync();
    {
      ArgMax a{-INFINITY, 0x7fffffff};
      for (int i = threadIdx.x; i < (int)gridDim.x; i += kDsConsumers) {
        ArgMax q;
        q.v = __ldcg(&p.samp_partial[i].v);
        q.i = __ldcg(&p.samp_partial[i].i);
        a = argmax_better(a, q);
      }
      a = warp_argmax(a);
      ds_sync();  // ared was read above by thread 0 of THIS CTA only before the device-wide barrier: safe to reuse
      if ((threadIdx.x & 31) == 0) ared[threadIdx.x >> 5] = a;
      ds_sync();
      if (threadIdx.x == 0) {
        ArgMax b = ared[0];
        for (int w = 1; w < kDsWarps; ++w) b = argmax_better(b, ared[w]);
        tok_s = b.i;
      }
      ds_sync();
      tok = tok_s;
      if (blockIdx.x == 0 && threadIdx.x == 0) p.tok_buf[f + 1] = tok;
    }
  }
}

}  // namespace ssdk
