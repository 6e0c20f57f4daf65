// engine.cu — host side of libssdk: plan objects, TMA descriptors, kernel launch glue, the
// one-call speculative step (CUDA graph) and the extern "C" surface declared in include/ssdk.h.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cudaTypedefs.h>
#include <nccl.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/ssdk.h"
#include "attention.cuh"
#include "common.cuh"
#include "elementwise.cuh"
#include "gemm.cuh"
#include "sampling.cuh"
#include "draft_stream.cuh"

using namespace ssdk;
typedef __nv_bfloat16 bf16;

// ------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------
static thread_local std::string g_err;
static int fail(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return -1;
}
#define CK(expr)                                                                              \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) return fail("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
  } while (0)
#define CKN(expr)                                                                             \
  do {                                                                                        \
    ncclResult_t _e = (expr);                                                                 \
    if (_e != ncclSuccess) return fail("%s:%d %s -> nccl error %d", __FILE__, __LINE__, #expr, (int)_e); \
  } while (0)
#define CKI(expr)                 \
  do {                            \
    int _r = (expr);              \
    if (_r != 0) return _r;       \
  } while (0)

static int env_int(const char* name, int dflt) {
  const char* s = getenv(name);
  return (s && *s) ? atoi(s) : dflt;
}

// ------------------------------------------------------------------------------------------
// launch helper (optional programmatic dependent launch)
// ------------------------------------------------------------------------------------------
struct Launcher {
  cudaStream_t st = nullptr;
  bool pdl = false;       // PDL enabled at all
  bool prev_kernel = false;  // the previous op on the stream was one of our kernels
  int64_t count = 0;

  template <typename... KArgs, typename... Args>
  int go(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = (pdl && prev_kernel) ? 1 : 0;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
    if (e != cudaSuccess) return fail("kernel launch failed: %s", cudaGetErrorString(e));
    prev_kernel = true;
    ++count;
    return 0;
  }
  void barrier_op() { prev_kernel = false; }  // memcpy / NCCL / anything that is not our kernel
};

// ------------------------------------------------------------------------------------------
// TMA descriptors
// ------------------------------------------------------------------------------------------
static PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;
static int get_encode() {
  if (g_encode) return 0;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn)
    return fail("cuTensorMapEncodeTiled unavailable (%s)", cudaGetErrorString(e));
  g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  return 0;
}
// bf16 row-major [rows, cols] matrix, box = [box_rows, 64 cols], 128B swizzle
static int make_tmap(CUtensorMap* tm, const void* ptr, int64_t rows, int64_t cols, int box_rows) {
  CKI(get_encode());
  if (cols % 8 != 0) return fail("TMA: row length %lld not a multiple of 8 elements", (long long)cols);
  if (((uintptr_t)ptr & 15) != 0) return fail("TMA: base pointer not 16-byte aligned");
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)cols * 2};
  cuuint32_t box[2] = {(cuuint32_t)kBlockK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld box_rows=%d", (int)r,
                                     (long long)rows, (long long)cols, box_rows);
  return 0;
}
// e4m3 row-major [rows, cols] weight as bytes, box = [64 rows, 128 cols (= one 128 B swizzle row)], 128B swizzle
static int make_tmap_e4m3(CUtensorMap* tm, const void* ptr, int64_t rows, int64_t cols) {
  CKI(get_encode());
  if (cols % kBlockK8 != 0) return fail("FP8 weight: K=%lld not a multiple of %d", (long long)cols, kBlockK8);
  if (((uintptr_t)ptr & 15) != 0) return fail("TMA: base pointer not 16-byte aligned");
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)cols};
  cuuint32_t box[2] = {(cuuint32_t)kBlockK8, 64u};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled (e4m3) failed (%d) rows=%lld cols=%lld", (int)r,
                                     (long long)rows, (long long)cols);
  return 0;
}

// ------------------------------------------------------------------------------------------
// GEMM planning + launch
// ------------------------------------------------------------------------------------------
static int g_num_sms = 0;
static int num_sms() {
  if (!g_num_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  return g_num_sms;
}
// add_rmsnorm_kernel geometry: <= 2 register-resident 8-element slices per thread (512 threads), smem staging beyond
static int norm_threads(int d) { return std::max(32, std::min(512, ((d / 8 + 31) / 32) * 32)); }
static int launch_norm(Launcher& L, int M, int d, const NormParams& np) {
  const int threads = norm_threads(d);
  const int slices = (d + 8 * threads - 1) / (8 * threads);
  if (slices == 1) return L.go(add_rmsnorm_kernel<1>, dim3(M), dim3(threads), 0, np);
  if (slices == 2) return L.go(add_rmsnorm_kernel<2>, dim3(M), dim3(threads), 0, np);
  return L.go(add_rmsnorm_kernel<0>, dim3(M), dim3(threads), (size_t)d * 4, np);
}
static int launch_rope(Launcher& L, int M, const RopeParams& rp, bool kv8 = false) {
  const dim3 grid(M, (rp.heads + 2 * rp.kv_heads + 3) / 4), block(128);
  if (kv8) {  // e4m3 KV cache: the head_dims paged attention is built for
    switch (rp.head_dim) {
      case 64: return L.go(rope_store_kernel<64, true>, grid, block, 0, rp);
      case 128: return L.go(rope_store_kernel<128, true>, grid, block, 0, rp);
      default: return fail("unsupported head_dim %d for an FP8 KV cache (64 and 128 are built)", rp.head_dim);
    }
  }
  switch (rp.head_dim) {
    case 64: return L.go(rope_store_kernel<64>, grid, block, 0, rp);
    case 128: return L.go(rope_store_kernel<128>, grid, block, 0, rp);
    case 256: return L.go(rope_store_kernel<256>, grid, block, 0, rp);
    default: return fail("unsupported head_dim %d for RoPE (64, 128 and 256 are built)", rp.head_dim);
  }
}
static int umma_n_for(int M) { return M <= 16 ? 16 : (M <= 32 ? 32 : (M <= 64 ? 64 : (M <= 128 ? 128 : 256))); }

static int auto_splits(int tiles, int num_kb, int ctas_per_sm = 2) {
  // Fill the machine in ONE wave: 2 CTAs/SM are resident (shared-memory bound), so tiles * S <= 2 * #SM; a partial
  // second wave doubles the kernel time (measured: 320 CTAs on 296 slots ran at 65 % of the HBM peak).  S <= 8 keeps
  // the consumers' split-K reduction to one batch of loads; >= 4 k-blocks per CTA keeps the TMA pipeline busy.
  const int slots = ctas_per_sm * num_sms();
  int S = std::max(1, slots / tiles);
  S = std::min(S, std::max(1, num_kb / 4));
  S = std::min(S, 8);
  const int per = (num_kb + S - 1) / S;
  return (num_kb + per - 1) / per;
}

template <int UN, int EPI, bool FP8>
static int launch_gemm_inst(Launcher& L, const CUtensorMap& tmW, const CUtensorMap& tmX, const GemmParams& p, int tiles,
                            int splits, const float* fp8_scale) {
  using Cfg = GemmCfg<UN, FP8>;
  static bool attr_set = false;
  if (!attr_set) {
    CK(cudaFuncSetAttribute(gemm_ws_kernel<UN, EPI, FP8>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_set = true;
  }
  return L.go(gemm_ws_kernel<UN, EPI, FP8>, dim3(tiles, splits), dim3(kGemmThreads), (size_t)Cfg::kSmemBytes, tmW, tmX, p,
              fp8_scale);
}
// fp8_scale != nullptr: tmW is an e4m3 byte map (make_tmap_e4m3) and p.num_kb counts 128-k blocks
static int launch_gemm(Launcher& L, int umma_n, int epi, const CUtensorMap& tmW, const CUtensorMap& tmX,
                       const GemmParams& p, int tiles, int splits, const float* fp8_scale = nullptr) {
#define SSDK_GEMM_CASE(UN, EP)                                                                                       \
  if (umma_n == UN && epi == EP)                                                                                     \
    return fp8_scale ? launch_gemm_inst<UN, EP, true>(L, tmW, tmX, p, tiles, splits, fp8_scale)                      \
                     : launch_gemm_inst<UN, EP, false>(L, tmW, tmX, p, tiles, splits, nullptr);
  SSDK_GEMM_CASE(16, EPI_BF16) SSDK_GEMM_CASE(16, EPI_PARTIAL) SSDK_GEMM_CASE(16, EPI_SILU) SSDK_GEMM_CASE(16, EPI_PUBLISH)
  SSDK_GEMM_CASE(32, EPI_BF16) SSDK_GEMM_CASE(32, EPI_PARTIAL) SSDK_GEMM_CASE(32, EPI_SILU) SSDK_GEMM_CASE(32, EPI_PUBLISH)
  SSDK_GEMM_CASE(64, EPI_BF16) SSDK_GEMM_CASE(64, EPI_PARTIAL) SSDK_GEMM_CASE(64, EPI_SILU) SSDK_GEMM_CASE(64, EPI_PUBLISH)
  SSDK_GEMM_CASE(128, EPI_BF16) SSDK_GEMM_CASE(128, EPI_PARTIAL) SSDK_GEMM_CASE(128, EPI_SILU)
  SSDK_GEMM_CASE(256, EPI_BF16) SSDK_GEMM_CASE(256, EPI_PARTIAL) SSDK_GEMM_CASE(256, EPI_SILU)
#undef SSDK_GEMM_CASE
  return fail("no GEMM instance for umma_n=%d epi=%d", umma_n, epi);
}

struct WeightMat {
  const bf16* ptr = nullptr;  // bf16 [rows, cols]; with `scale` set: e4m3 bytes [rows, cols] (ssdk_bind_weight_fp8)
  const float* scale = nullptr;  // fp32 [rows] per-row scales of an FP8 matrix, nullptr for bf16
  int64_t rows = 0, cols = 0;
  CUtensorMap tm;
  bool has_tm = false;
};
static int weight_tmap(WeightMat& w) {
  if (w.has_tm) return 0;
  if (!w.ptr) return fail("weight not bound");
  if (w.scale) CKI(make_tmap_e4m3(&w.tm, w.ptr, w.rows, w.cols));
  else CKI(make_tmap(&w.tm, w.ptr, w.rows, w.cols, 64));
  w.has_tm = true;
  return 0;
}

// activations buffers usable as the X operand: [kMaxTokens rows, K] bf16.  Decode / verify steps use <= 64 tokens
// (UMMA N 16 / 32 / 64); prefill chunks and larger batches up to 256 (UMMA N 128 / 256: the weights are then streamed once
// per 256 tokens instead of once per 64 — a 2k-token 70B prompt reads 139 GB 8 times instead of 32).
constexpr int kMaxTokens = 256;
struct XMapCache {
  std::map<std::tuple<const void*, int, int>, CUtensorMap> maps;
  int get(const void* ptr, int K, int umma_n, const CUtensorMap** out) {
    auto key = std::make_tuple(ptr, K, umma_n);
    auto it = maps.find(key);
    if (it == maps.end()) {
      CUtensorMap tm;
      CKI(make_tmap(&tm, ptr, kMaxTokens, K, umma_n));
      it = maps.emplace(key, tm).first;
    }
    *out = &it->second;
    return 0;
  }
};

// ------------------------------------------------------------------------------------------
// model / engine state
// ------------------------------------------------------------------------------------------
struct LayerW {
  const bf16* input_norm = nullptr;
  const bf16* post_norm = nullptr;
  const bf16* q_norm = nullptr;
  const bf16* k_norm = nullptr;
  WeightMat qkv, o, gate_up, down;
};
struct Model {
  ssdk_model_cfg cfg;
  bool present = false;
  WeightMat embed, lm_head;
  const bf16* final_norm = nullptr;
  const float* rope = nullptr;
  int64_t rope_rows = 0;
  std::vector<LayerW> layers;
  bf16* k_cache = nullptr;
  bf16* v_cache = nullptr;
  int64_t num_blocks = 0;
  // ssdk_bind_kv_cache_fp8: the caches hold e4m3 codes (k_cache / v_cache then point at bytes), layer l's K = k_scale[l] *
  // code and V = v_scale[l] * code
  bool kv_fp8 = false;
  std::vector<float> k_scale, v_scale;
  // derived (per TP rank)
  int H, KV, hd, d, ffn, qkv_dim, vocab_local;
};

struct Workspace {
  // activations (X-operand capable: kMaxTokens rows each)
  bf16 *hidden, *residual, *q, *attn_out, *act, *last_hidden, *dense_tmp;
  float* partials;
  float *att_o, *att_lse;
  unsigned* att_counters;
  unsigned* ar_state;  // [0] sequence number of the running target forward (epoch base of its one-shot all-reduces)
  unsigned* pub_counters;  // [512] split-K arrival tickets of the in-kernel reductions (EPI_PUBLISH / split EPI_SILU), zero between launches
  int64_t* positions;
  int32_t *slot_mapping, *context_lens;
  // step state
  uint8_t* out_dev;     // [tok_buf | n_accept | recovery] — one D2H per step
  int64_t* tok_buf;     // [max_batch, K+1]
  int64_t* fold_ids;    // [max_batch, 2]: {token at ctx-1, recovery} — the kernel-per-op draft's two-row forward 0
  int64_t* ids_in;     // [kMaxTokens]  (forward_tokens input), followed by the varlen inputs (kFwIn*)
  int32_t* var_cu_q;    // [kMaxTokens + 1]  (forward_varlen prefix sums of q_len)
  AttnTile* var_tiles;  // [kMaxTokens]      (forward_varlen attention tile table)
  int64_t* out_tok;     // [max_batch]   (forward_tokens sampled output)
  bf16 *logits_q, *logits_p, *logits_last;
  bf16 *logits_shard, *logits_gather;  // tensor-parallel lm_head: local [rows, V/tp] and all-gathered [tp, rows, V/tp]
  // device copy of the step parameters (one contiguous block, see StepBlock)
  uint8_t* step_dev;
  int32_t* n_accept;
  int64_t* recovery;
  // device-resident generation log (resident/benchmark mode): accepted tokens per sequence
  int64_t* log_tokens;  // [max_batch, kLogCap]
  int32_t* log_len;     // [max_batch]
  // sampling scratch
  ArgMax* samp_partial;
  unsigned* samp_counters;
  RowPart* ver_rows;
  RecPart* ver_rec;
  unsigned* ver_counters;
  size_t partial_floats = 0;
  // streaming draft kernel (draft_stream.cuh): inter-phase vectors, split-KV partials, device-wide barrier state
  bf16* ds_vec;
  bf16* ds_vec0;  // the same vectors for row 0 of a two-row forward 0
  float* ds_attn;
  unsigned* ds_sync;
};

constexpr int kSampleChunks = 64;
// forward inputs, staged through one pinned ring slot and copied in one H2D: ids | cu_q | varlen tile table
constexpr size_t kFwInCuOff = (size_t)kMaxTokens * 8;
constexpr size_t kFwInTileOff = kFwInCuOff + ((size_t)(kMaxTokens + 1) * 4 + 15) / 16 * 16;
constexpr size_t kFwInBytes = kFwInTileOff + (size_t)kMaxTokens * sizeof(AttnTile);
constexpr int kLogCap = 16384;
constexpr int kVerifyCtas = 128;

struct ssdk_engine {
  ssdk_runtime_cfg rt;
  Model model[2];
  Workspace ws;
  void* ws_base = nullptr;
  int64_t ws_bytes = 0;
  XMapCache xmaps;
  ncclComm_t comm = nullptr;
  bool finalized = false;
  int64_t launches = 0;
  // pinned staging: [StepBlock in][results out]
  uint8_t* pin_in = nullptr;
  uint8_t* pin_out = nullptr;
  // ssdk_forward_tokens does not synchronize when no token is sampled (prefill chunks), so its inputs go through a ring of
  // pinned slots [StepBlock | token ids]; a slot is rewritten only after the H2D copies that read it have completed
  // (one event per slot).  pin_in stays private to ssdk_spec_step / _stage, which synchronize before they return.
  static constexpr int kFwSlots = 4;
  uint8_t* pin_fw = nullptr;
  size_t fw_slot_bytes = 0;
  cudaEvent_t fw_ev[kFwSlots] = {nullptr};
  bool fw_ev_pending[kFwSlots] = {false};
  unsigned fw_next = 0;
  size_t step_bytes = 0;
  size_t out_bytes = 0;
  // offsets inside the step block
  size_t off_ctx, off_rec, off_pend, off_tt, off_tq, off_seed, off_btt, off_btd;
  size_t off_out_nacc, off_out_rec;
  // graphs
  std::map<int, cudaGraphExec_t> spec_graphs;  // keyed by batch * 2 + (draft path: 1 = streaming kernel)
  std::map<int, int64_t> spec_graph_launches;
  std::map<int, cudaGraphExec_t> spec_graphs_resident;
  int resident_ctx_bound = 0;  // upper bound of the resident loop's context length (staged value + (K+1) per step)
  int max_ctx_hint = 0;
  cudaStream_t cap_stream = nullptr;
  // one-shot all-reduce over NVLink symmetric memory (optional; NCCL is used when not bound)
  int symm_n = 0;
  uint8_t* symm_peer[kSymmMaxRanks] = {nullptr};
  unsigned symm_slot_bytes = 0;  // graphs are captured here (the caller's stream may be the legacy default stream)
};

static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// the decoder linears of every layer are FP8 (the draft: all of them or none, checked by ssdk_finalize)
static bool model_linears_fp8(const Model& m) {
  for (const LayerW& lw : m.layers)
    if (!lw.qkv.scale || !lw.o.scale || !lw.gate_up.scale || !lw.down.scale) return false;
  return !m.layers.empty();
}
static bool model_any_linear_fp8(const Model& m) {
  for (const LayerW& lw : m.layers)
    if (lw.qkv.scale || lw.o.scale || lw.gate_up.scale || lw.down.scale) return true;
  return false;
}

static void derive(Model& m) {
  const auto& c = m.cfg;
  m.H = c.heads / c.tp_size;
  m.KV = c.kv_heads / c.tp_size;
  m.hd = c.head_dim;
  m.d = c.hidden;
  m.ffn = c.ffn / c.tp_size;
  m.qkv_dim = (m.H + 2 * m.KV) * m.hd;
  m.vocab_local = c.vocab / c.tp_size;
}

// elements of one row's inter-phase vectors of the streaming draft kernel (enqueue_draft_stream / ds_row0_vecs carve them)
static size_t ds_vec_elems(int qkv, int d, int ffn, int q_width) { return (size_t)qkv + 4 * d + ffn + q_width + 64; }

// workspace carve-up (pass base = nullptr to measure)
static int64_t carve(ssdk_engine* e, uint8_t* base) {
  size_t off = 0;
  auto take = [&](size_t bytes) -> uint8_t* {
    off = align_up(off, 1024);
    uint8_t* p = base ? base + off : nullptr;
    off += bytes;
    return p;
  };
  int dmax = 0, qmax = 0, fmax = 0, vmax = 0, Hmax = 0, hdmax = 0;
  size_t part = 0;
  for (int w = 0; w < 2; ++w) {
    Model& m = e->model[w];
    if (!m.present) continue;
    dmax = std::max(dmax, m.d);
    qmax = std::max(qmax, m.qkv_dim);
    fmax = std::max(fmax, m.ffn);
    vmax = std::max(vmax, m.cfg.vocab);
    Hmax = std::max(Hmax, m.H);
    hdmax = std::max(hdmax, m.hd);
    // partial buffer: max over GEMMs of S*M*N with S bounded by auto_splits (<= 2*SMs/tiles + 1)
    auto need = [&](int N, int K) {
      const int tiles = (N + kTileRows - 1) / kTileRows;
      const int S = std::max(auto_splits(tiles, K / kBlockK), auto_splits(tiles, std::max(1, K / kBlockK8)));  // bf16 / FP8
      return (size_t)S * kMaxTokens * N;
    };
    part = std::max(part, need(m.qkv_dim, m.d));
    part = std::max(part, need(m.d, m.H * m.hd));
    part = std::max(part, need(2 * m.ffn, m.d));
    part = std::max(part, need(m.d, m.ffn));
  }
  Workspace scratch_ws;
  Workspace& w = base ? e->ws : scratch_ws;  // measuring (base == nullptr) must not clobber bound pointers
  const int K = e->rt.spec_k, MB = e->rt.max_batch;
  w.hidden = (bf16*)take((size_t)kMaxTokens * dmax * 2);
  w.residual = (bf16*)take((size_t)kMaxTokens * dmax * 2);
  w.q = (bf16*)take((size_t)kMaxTokens * Hmax * hdmax * 2);
  w.attn_out = (bf16*)take((size_t)kMaxTokens * Hmax * hdmax * 2);
  w.act = (bf16*)take((size_t)kMaxTokens * fmax * 2);
  w.last_hidden = (bf16*)take((size_t)kMaxTokens * dmax * 2);
  w.dense_tmp = (bf16*)take((size_t)kMaxTokens * std::max(dmax, qmax) * 2);
  w.partials = (float*)take(part * 4);
  w.partial_floats = part;
  w.att_o = (float*)take((size_t)kMaxTokens * Hmax * kAttnMaxSplit * hdmax * 4);
  w.att_lse = (float*)take((size_t)kMaxTokens * Hmax * kAttnMaxSplit * 4);
  w.att_counters = (unsigned*)take((size_t)kMaxTokens * 64 * 4);
  w.ar_state = (unsigned*)take(64);
  w.pub_counters = (unsigned*)take(512 * 4);
  w.positions = (int64_t*)take(kMaxTokens * 8);
  w.slot_mapping = (int32_t*)take(kMaxTokens * 4);
  w.context_lens = (int32_t*)take(kMaxTokens * 4);
  w.out_dev = take(e->out_bytes);
  w.tok_buf = (int64_t*)w.out_dev;
  w.n_accept = (int32_t*)(w.out_dev ? w.out_dev + e->off_out_nacc : nullptr);
  w.recovery = (int64_t*)(w.out_dev ? w.out_dev + e->off_out_rec : nullptr);
  w.log_tokens = (int64_t*)take((size_t)MB * kLogCap * 8);
  w.log_len = (int32_t*)take((size_t)MB * 4);
  w.ids_in = (int64_t*)take(kFwInBytes);
  w.var_cu_q = (int32_t*)(w.ids_in ? (uint8_t*)w.ids_in + kFwInCuOff : nullptr);
  w.var_tiles = (AttnTile*)(w.ids_in ? (uint8_t*)w.ids_in + kFwInTileOff : nullptr);
  w.out_tok = (int64_t*)take(kMaxTokens * 8);
  w.logits_q = (bf16*)take((size_t)MB * std::max(K, 1) * vmax * 2);
  w.logits_p = (bf16*)take((size_t)MB * (K + 1) * vmax * 2);
  w.logits_last = (bf16*)take((size_t)kMaxTokens * vmax * 2);
  w.logits_shard = (bf16*)take((size_t)kMaxTokens * vmax * 2);
  w.logits_gather = (bf16*)take((size_t)kMaxTokens * vmax * 2);
  w.step_dev = take(e->step_bytes);
  w.samp_partial = (ArgMax*)take((size_t)kMaxTokens * kSampleChunks * sizeof(ArgMax));
  w.samp_counters = (unsigned*)take(kMaxTokens * 4);
  w.ver_rows = (RowPart*)take((size_t)kVerifyMaxRows * kVerifyCtas * sizeof(RowPart));
  w.ver_rec = (RecPart*)take((size_t)kVerifyMaxBatch * kVerifyCtas * sizeof(RecPart));
  w.ver_counters = (unsigned*)take(64);
  const size_t ds_elems = ds_vec_elems(qmax, dmax, fmax, Hmax * hdmax);
  w.ds_vec = (bf16*)take(ds_elems * 2);
  w.ds_vec0 = (bf16*)take(ds_elems * 2);
  w.fold_ids = (int64_t*)take((size_t)MB * 2 * 8);
  w.ds_attn = (float*)take((size_t)Hmax * kDsSplits * (hdmax + 2) * 4);
  w.ds_sync = (unsigned*)take(256);
  return (int64_t)align_up(off, 1024);
}

// ------------------------------------------------------------------------------------------
// one forward pass (enqueue only)
// ------------------------------------------------------------------------------------------
// a varlen forward (ssdk_forward_varlen): prefix sums and attention tiles on the device, the plan made on the host
struct VarlenFwd {
  AttnVarlen attn;
  AttnPlan plan;
  int n_tiles;
  int M;
};
struct Fwd {
  int which;
  int B, Q;
  const int64_t* ids;
  int ids_stride;
  const int32_t* ctx0;
  const int32_t* block_tables;
  int pos_offset;
  int logits_mode;  // 0 none, 1 all rows, 2 last row per sequence
  bf16* logits_out;
  int64_t logits_ld;
  const VarlenFwd* var = nullptr;  // set: B sequences of their own q_len packed into M rows (Q unused)
  const int64_t* pend = nullptr;   // set: row 0 of sequence b stores no K/V unless pend[b] >= 0 (prep_kernel)
};

static int attn_plan_raw(int H, int KV, int B, int Q, int max_ctx, int* TQ, int* MT, int* nqt, int* nsplit) {
  AttnPlan pl;
  const int rc = attn_make_plan(H, KV, B, Q, max_ctx, num_sms(), &pl);
  if (rc == 1) return fail("unsupported GQA ratio %d/%d", H, KV);
  if (rc != 0) return fail("attention tile too large");
  *TQ = pl.TQ;
  *MT = pl.MT;
  *nqt = pl.n_qtiles;
  *nsplit = pl.n_split;
  return 0;
}
static int attn_plan(const Model& m, int B, int Q, int* TQ, int* MT, int* nqt, int* nsplit, int max_ctx) {
  return attn_plan_raw(m.H, m.KV, B, Q, max_ctx, TQ, MT, nqt, nsplit);
}

template <int HD, int MT, bool KV8>
static int launch_attn_inst(Launcher& L, const AttnParams& p, const AttnVarlen* var, dim3 grid) {
  const size_t smem = (size_t)attn_smem_bytes(HD);
  static bool attr_set = false;
  if (!attr_set) {
    CK(cudaFuncSetAttribute(paged_attn_kernel<HD, MT, KV8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK(cudaFuncSetAttribute(paged_attn_varlen_kernel<HD, MT, KV8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set = true;
  }
  if (var) return L.go(paged_attn_varlen_kernel<HD, MT, KV8>, grid, dim3(attn_warps(MT) * 32), smem, p, *var);
  return L.go(paged_attn_kernel<HD, MT, KV8>, grid, dim3(attn_warps(MT) * 32), smem, p);
}
template <bool KV8>
static int launch_attn_kv(Launcher& L, const AttnParams& p, const AttnVarlen* var, int hd, int MT, dim3 grid) {
  if (hd == 128 && MT == 1) return launch_attn_inst<128, 1, KV8>(L, p, var, grid);
  if (hd == 128 && MT == 2) return launch_attn_inst<128, 2, KV8>(L, p, var, grid);
  if (hd == 128 && MT == 4) return launch_attn_inst<128, 4, KV8>(L, p, var, grid);
  if (hd == 64 && MT == 1) return launch_attn_inst<64, 1, KV8>(L, p, var, grid);
  if (hd == 64 && MT == 2) return launch_attn_inst<64, 2, KV8>(L, p, var, grid);
  if (hd == 64 && MT == 4) return launch_attn_inst<64, 4, KV8>(L, p, var, grid);
  return fail("unsupported head_dim %d (64 and 128 are built)", hd);
}
static int launch_attn(Launcher& L, const AttnParams& p, const AttnVarlen* var, int hd, int MT, dim3 grid, bool kv8) {
  return kv8 ? launch_attn_kv<true>(L, p, var, hd, MT, grid) : launch_attn_kv<false>(L, p, var, hd, MT, grid);
}

// The cache dtype of one attention call: kv8 = e4m3 caches (kc / vc point at bytes) with K = k_scale * code and
// V = v_scale * code.  The launch plan does not depend on it.
struct KvDtype {
  bool kv8 = false;
  float k_scale = 1.f, v_scale = 1.f;
};

static int enqueue_attention(Launcher& L, const bf16* q, const bf16* kc, const bf16* vc, const int32_t* bt,
                             const int32_t* ctx_lens, bf16* out, float* part_o, float* part_lse, unsigned* counters,
                             int B, int Q, int H,
                             int KV, int hd, int block_size, int max_blocks, float scale, int TQ, int MT, int nqt,
                             int nsplit, const VarlenFwd* var = nullptr, KvDtype kvd = KvDtype{}) {
  AttnParams a;
  a.q = q; a.k_cache = kc; a.v_cache = vc; a.block_tables = bt; a.context_lens = ctx_lens; a.out = out;
  a.part_o = part_o; a.part_lse = part_lse;
  (void)counters;
  a.B = B; a.Q = Q; a.H = H; a.KV = KV; a.block_size = block_size; a.max_blocks = max_blocks;
  a.n_split = nsplit; a.TQ = TQ; a.n_qtiles = nqt;
  a.g_shift = attn_g_shift(H, KV);
  a.scale_log2 = scale * 1.4426950408889634f;
  a.v_scale = 1.f;
  if (kvd.kv8) {
    a.scale_log2 *= kvd.k_scale;
    a.v_scale = kvd.v_scale;
  }
  if (var) {
    CKI(launch_attn(L, a, &var->attn, hd, MT, dim3(KV, nsplit, var->n_tiles), kvd.kv8));
    if (nsplit > 1) CKI(L.go(attn_combine_kernel<true>, dim3(var->M * H), dim3(32), 0, a, hd, var->attn));
    return 0;
  }
  CKI(launch_attn(L, a, nullptr, hd, MT, dim3(KV, nsplit, B * nqt), kvd.kv8));
  if (nsplit > 1) CKI(L.go(attn_combine_kernel<false>, dim3(B * Q * H), dim3(32), 0, a, hd, AttnVarlen{}));
  return 0;
}

static int enqueue_gemm(ssdk_engine* e, Launcher& L, const bf16* x, WeightMat& w, int M, int epi, void* out, int ldo,
                        int N_out, int* splits_out, const PublishParams* pub = nullptr) {
  CKI(weight_tmap(w));
  const int K = (int)w.cols;
  const int kbk = w.scale ? kBlockK8 : kBlockK;  // an FP8 stage holds 128 k (bytes) of weights, a bf16 one 64 k
  if (K % kbk) return fail("GEMM K=%d not a multiple of %d", K, kbk);
  const int un = umma_n_for(M);
  const CUtensorMap* tmX;
  CKI(e->xmaps.get(x, K, un, &tmX));
  GemmParams p;
  p.out = out; p.M = M; p.N = N_out; p.ldo = ldo; p.num_kb = K / kbk;
  int tiles, splits;
  p.sk_partials = nullptr; p.sk_counters = nullptr; p.sk_width = 0;
  if (epi == EPI_SILU) {
    tiles = (N_out + 63) / 64;
    // narrow (tensor-parallel) shards: too few 64-column tiles to fill the machine -> split K, reduced inside the kernel
    splits = (un <= 64 && tiles < num_sms() && out != nullptr && e->ws.partials) ? auto_splits(tiles, p.num_kb) : 1;
    if (splits > 1 && (tiles > 512 || (size_t)splits * M * 2 * N_out > e->ws.partial_floats)) splits = 1;
    p.tile_rows = 64;
    p.hi_row_offset = N_out;
    if (splits > 1) {
      p.sk_partials = e->ws.partials; p.sk_counters = e->ws.pub_counters; p.sk_width = 2 * N_out;
    }
  } else {
    tiles = (N_out + kTileRows - 1) / kTileRows;
    splits = (epi == EPI_PARTIAL || epi == EPI_PUBLISH) ? auto_splits(tiles, p.num_kb, un <= 64 ? 2 : 1) : 1;
    p.tile_rows = kTileRows;
    p.hi_row_offset = 64;
  }
  if (epi == EPI_PUBLISH) {
    if (!pub) return fail("EPI_PUBLISH without publish parameters");
    if (un > 64) return fail("EPI_PUBLISH is planned for <= 64 tokens");
    if (tiles > 512) return fail("EPI_PUBLISH: %d tiles > 512 ticket counters", tiles);
    if ((size_t)splits * M * N_out > e->ws.partial_floats) return fail("split-K partial buffer too small");
    p.pub = *pub;
    p.sk_partials = e->ws.partials; p.sk_counters = e->ws.pub_counters; p.sk_width = N_out;
  }
  p.kb_per_split = (p.num_kb + splits - 1) / splits;
  if (epi == EPI_PARTIAL && (size_t)splits * M * N_out > e->ws.partial_floats && out == e->ws.partials)
    return fail("split-K partial buffer too small");
  if (splits_out) *splits_out = splits;
  return launch_gemm(L, un, epi, w.tm, *tmX, p, tiles, splits, w.scale);
}

// y = allreduce_sum(bf16(sum_s partials)) for tensor-parallel row-parallel linears
// (layers/linear.py:195-199): reduce split-K locally, round to bf16 like F.linear, NCCL bf16 sum.
static SymmIn symm_in(ssdk_engine* e, int call_idx, bool no_dep_wait = false) {
  SymmIn s;
  s.no_dep_wait = no_dep_wait ? 1 : 0;
  s.base = e->symm_peer[e->model[SSDK_TARGET].cfg.tp_rank];
  s.fwd_seq = e->ws.ar_state;
  s.call_idx = call_idx;
  s.n_calls = 2 * e->model[SSDK_TARGET].cfg.layers + 1;
  s.n_ranks = e->symm_n;
  s.slot_bytes = e->symm_slot_bytes;
  return s;
}
// first half of the one-shot all-reduce: reduce split-K locally, push bf16 to every rank, release flags
static int enqueue_ar_publish(ssdk_engine* e, Launcher& L, const GemmOut* x, const NormParams* embed_src, int M, int d,
                              int call_idx) {
  Model& m = e->model[SSDK_TARGET];
  ArPublishParams ap;
  memset(&ap, 0, sizeof(ap));
  if (x) ap.x = *x;
  if (embed_src) {
    ap.ids = embed_src->ids; ap.ids_stride = embed_src->ids_stride; ap.embed = embed_src->embed;
    ap.vocab_start = embed_src->vocab_start; ap.vocab_rows = embed_src->vocab_rows;
  }
  ap.M = M; ap.d = d; ap.n_ranks = e->symm_n; ap.rank = m.cfg.tp_rank;
  for (int r = 0; r < e->symm_n; ++r) ap.peer[r] = e->symm_peer[r];
  ap.slot_bytes = e->symm_slot_bytes;
  ap.fwd_seq = e->ws.ar_state; ap.call_idx = call_idx; ap.n_calls = 2 * m.cfg.layers + 1;
  const int n8 = M * d / 8;
  // one CTA column per destination rank (see ar_publish_kernel): default at 8 ranks, where it measured 12.20 vs 12.57 ms/step
  // (Llama-3.1-70B TP=8); SSDK_PUBLISH_PER_PEER=0/1 overrides
  static int per_peer = -1;
  if (per_peer < 0) per_peer = env_int("SSDK_PUBLISH_PER_PEER", e->symm_n >= 8 ? 1 : 0) != 0 ? 1 : 0;
  const int gx = std::max(1, std::min((n8 + 255) / 256, num_sms()));
  return L.go(ar_publish_kernel, dim3(gx, per_peer ? e->symm_n : 1), dim3(256), 0, ap);
}

// row-parallel GEMM whose epilogue publishes the rank's bf16 result to every peer (EPI_PUBLISH)
static PublishParams publish_params(ssdk_engine* e, int call_idx) {
  Model& m = e->model[SSDK_TARGET];
  PublishParams pb;
  memset(&pb, 0, sizeof(pb));
  for (int r = 0; r < e->symm_n; ++r) pb.peer[r] = e->symm_peer[r];
  pb.fwd_seq = e->ws.ar_state;
  pb.slot_bytes = e->symm_slot_bytes;
  pb.call_idx = call_idx;
  pb.n_calls = 2 * m.cfg.layers + 1;
  pb.n_ranks = e->symm_n;
  pb.rank = m.cfg.tp_rank;
  return pb;
}
// SSDK_FUSED_PUBLISH=1: the row-parallel GEMM publishes from its own epilogue (EPI_PUBLISH).  Off by default: the ticket +
// reduce + 8-byte remote stores of the last split-K CTA of a tile lengthen the GEMM's tail, while the publish kernel
// spreads the same work over 28 CTAs x 256 threads with 16-byte stores (DESIGN.md §5).
static bool fused_publish_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* s = getenv("SSDK_FUSED_PUBLISH");
    v = (s && *s) ? (atoi(s) != 0 ? 1 : 0) : 0;
  }
  return v == 1;
}

static int enqueue_tp_allreduce(ssdk_engine* e, Launcher& L, int S, int M, int N, GemmOut* out) {
  Workspace& w = e->ws;
  const int n = M * N;
  CKI(L.go(splitk_reduce_kernel, dim3((n + 255) / 256), dim3(256), 0, (const float*)w.partials, w.dense_tmp, S, M, N, N));
  CKN(ncclAllReduce(w.dense_tmp, w.dense_tmp, (size_t)n, ncclBfloat16, ncclSum, e->comm, L.st));
  L.barrier_op();
  out->dense = w.dense_tmp; out->partial = nullptr; out->S = 0; out->M = M; out->N = N;
  return 0;
}

// [tp, rows, Vs] (all-gather layout) -> [rows, ld] with column r*Vs + v   (torch.cat(parts, -1), embed_head.py:98-99)
__global__ void unshard_logits_kernel(const bf16* __restrict__ gathered, bf16* __restrict__ out, int tp, int rows, int Vs,
                                      int64_t ld) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t n8 = (int64_t)tp * rows * (Vs / 8);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
    const int v8 = (int)(i % (Vs / 8));
    const int64_t t = i / (Vs / 8);
    const int m = (int)(t % rows), r = (int)(t / rows);
    const uint4 val = *reinterpret_cast<const uint4*>(gathered + ((size_t)r * rows + m) * Vs + (size_t)v8 * 8);
    *reinterpret_cast<uint4*>(out + (size_t)m * ld + (size_t)r * Vs + (size_t)v8 * 8) = val;
  }
}

static int enqueue_forward(ssdk_engine* e, Launcher& L, const Fwd& f) {
  Model& m = e->model[f.which];
  Workspace& w = e->ws;
  const int M = f.var ? f.var->M : f.B * f.Q;
  if (M < 1 || M > kMaxTokens) return fail("forward: %d tokens (max %d)", M, kMaxTokens);
  const int tp = m.cfg.tp_size;
  if (tp > 1 && !e->comm) return fail("tensor parallel forward without a NCCL communicator");
  const int bs = e->rt.block_size, mb = e->rt.max_blocks_per_seq;
  const int64_t cache_layer_stride = m.num_blocks * bs * m.KV * m.hd;

  unsigned* fwd_seq = (f.which == SSDK_TARGET && tp > 1 && e->symm_n == tp) ? w.ar_state : (unsigned*)nullptr;
  int TQ = 1, MT = 1, nqt = 1, nsplit = 1;
  if (f.var) {
    CKI(L.go(prep_varlen_kernel, dim3(1), dim3(kMaxTokens), 0, f.ctx0, f.var->attn.cu_q, f.block_tables, mb, bs, f.B,
             w.positions, w.slot_mapping, w.context_lens, fwd_seq));
    TQ = f.var->plan.TQ; MT = f.var->plan.MT; nqt = f.var->plan.n_qtiles; nsplit = f.var->plan.n_split;
  } else {
    CKI(L.go(prep_kernel, dim3(1), dim3(kMaxTokens), 0, f.ctx0, f.block_tables, mb, bs, f.B, f.Q, f.pos_offset, f.pend,
             w.positions, w.slot_mapping, w.context_lens, fwd_seq));
    CKI(attn_plan(m, f.B, f.Q, &TQ, &MT, &nqt, &nsplit, e->max_ctx_hint));
  }
  const float scale = 1.0f / sqrtf((float)m.hd);

  const bool use_symm = tp > 1 && e->symm_n == tp;
  bool prev_symm = false;
  int ar_idx = 0, prev_idx = 0;  // static index of each one-shot all-reduce inside this forward (epoch = seq*512+idx+1)
  GemmOut prev;  // output of the previous row-parallel GEMM feeding the next norm
  prev.dense = nullptr; prev.partial = nullptr; prev.S = 0; prev.M = M; prev.N = m.d;

  for (int l = 0; l < m.cfg.layers; ++l) {
    LayerW& lw = m.layers[l];
    // ---- input norm (layer 0: embedding gather, no residual) ----
    NormParams np;
    memset(&np, 0, sizeof(np));
    np.eps = m.cfg.rms_eps; np.d = m.d; np.w = lw.input_norm; np.y = w.hidden; np.residual_out = w.residual;
    if (l == 0) {
      if (tp == 1) {
        np.ids = f.ids; np.ids_stride = f.ids_stride; np.embed = m.embed.ptr;
        np.vocab_start = 0; np.vocab_rows = m.vocab_local;
      } else {
        // vocab-parallel embedding: masked local lookup + all-reduce (embed_head.py:49-58)
        NormParams ep;
        memset(&ep, 0, sizeof(ep));
        ep.ids = f.ids; ep.ids_stride = f.ids_stride; ep.embed = m.embed.ptr;
        ep.vocab_start = m.cfg.tp_rank * m.vocab_local; ep.vocab_rows = m.vocab_local;
        if (use_symm) {
          CKI(enqueue_ar_publish(e, L, nullptr, &ep, M, m.d, ar_idx));
          np.symm = symm_in(e, ar_idx++);
        } else {
          ep.eps = m.cfg.rms_eps; ep.d = m.d; ep.residual_out = w.dense_tmp;  // y = null: gather only
          CKI(launch_norm(L, M, m.d, ep));
          CKN(ncclAllReduce(w.dense_tmp, w.dense_tmp, (size_t)M * m.d, ncclBfloat16, ncclSum, e->comm, L.st));
          L.barrier_op();
          np.x.dense = w.dense_tmp; np.x.S = 0; np.x.M = M; np.x.N = m.d;
        }
      }
    } else {
      np.x = prev;
      if (prev_symm) np.symm = symm_in(e, prev_idx, true);
      np.residual_in = w.residual;
    }
    CKI(launch_norm(L, M, m.d, np));

    // ---- QKV projection -> RoPE (+qk norm) -> KV store ----
    int S = 1;
    CKI(enqueue_gemm(e, L, w.hidden, lw.qkv, M, EPI_PARTIAL, w.partials, 0, m.qkv_dim, &S));
    RopeParams rp;
    rp.qkv.dense = nullptr; rp.qkv.partial = w.partials; rp.qkv.S = S; rp.qkv.M = M; rp.qkv.N = m.qkv_dim;
    rp.positions = w.positions; rp.slot_mapping = w.slot_mapping; rp.rope_table = m.rope;
    rp.q_norm_w = m.cfg.qk_norm ? lw.q_norm : nullptr;
    rp.k_norm_w = m.cfg.qk_norm ? lw.k_norm : nullptr;
    rp.norm_eps = m.cfg.rms_eps;
    rp.q_out = w.q;
    KvDtype kvd;
    if (m.kv_fp8) {  // e4m3 caches: a layer is cache_layer_stride bytes
      rp.k_cache = reinterpret_cast<bf16*>(reinterpret_cast<uint8_t*>(m.k_cache) + (size_t)l * cache_layer_stride);
      rp.v_cache = reinterpret_cast<bf16*>(reinterpret_cast<uint8_t*>(m.v_cache) + (size_t)l * cache_layer_stride);
      kvd.kv8 = true; kvd.k_scale = m.k_scale[l]; kvd.v_scale = m.v_scale[l];
    } else {
      rp.k_cache = m.k_cache + (size_t)l * cache_layer_stride;
      rp.v_cache = m.v_cache + (size_t)l * cache_layer_stride;
    }
    rp.heads = m.H; rp.kv_heads = m.KV; rp.head_dim = m.hd;
    rp.k_scale = kvd.k_scale; rp.v_scale = kvd.v_scale;
    CKI(launch_rope(L, M, rp, kvd.kv8));

    // ---- attention over the paged cache ----
    CKI(enqueue_attention(L, w.q, rp.k_cache, rp.v_cache, f.block_tables, w.context_lens, w.attn_out, w.att_o,
                          w.att_lse, w.att_counters, f.B, f.Q, m.H, m.KV, m.hd, bs, mb, scale, TQ, MT, nqt, nsplit,
                          f.var, kvd));

    // ---- output projection (row-parallel) ----
    const bool fuse_pub = use_symm && fused_publish_enabled() && M <= 64;
    GemmOut oproj;
    bool oproj_symm = false;
    int oproj_idx = 0;
    if (fuse_pub) {
      const PublishParams pb = publish_params(e, ar_idx);
      CKI(enqueue_gemm(e, L, w.attn_out, lw.o, M, EPI_PUBLISH, w.partials, 0, m.d, &S, &pb));
      oproj_idx = ar_idx++;
      oproj_symm = true;
    } else {
      CKI(enqueue_gemm(e, L, w.attn_out, lw.o, M, EPI_PARTIAL, w.partials, 0, m.d, &S));
    }
    oproj.dense = nullptr; oproj.partial = w.partials; oproj.S = S; oproj.M = M; oproj.N = m.d;
    if (tp > 1 && !fuse_pub) {
      if (use_symm) {
        CKI(enqueue_ar_publish(e, L, &oproj, nullptr, M, m.d, ar_idx));
        oproj_idx = ar_idx++;
        oproj_symm = true;
      } else {
        CKI(enqueue_tp_allreduce(e, L, S, M, m.d, &oproj));
      }
    }

    // ---- post-attention norm ----
    NormParams pn;
    memset(&pn, 0, sizeof(pn));
    pn.x = oproj; pn.residual_in = w.residual; pn.w = lw.post_norm; pn.eps = m.cfg.rms_eps;
    if (oproj_symm) pn.symm = symm_in(e, oproj_idx, true);
    pn.y = w.hidden; pn.residual_out = w.residual; pn.d = m.d;
    CKI(launch_norm(L, M, m.d, pn));

    // ---- MLP: gate|up with fused SiLU*mul (split-K inside the kernel when the shard is too narrow to fill the machine) ----
    CKI(enqueue_gemm(e, L, w.hidden, lw.gate_up, M, EPI_SILU, w.act, m.ffn, m.ffn, nullptr));
    if (fuse_pub) {
      const PublishParams pb = publish_params(e, ar_idx);
      CKI(enqueue_gemm(e, L, w.act, lw.down, M, EPI_PUBLISH, w.partials, 0, m.d, &S, &pb));
      prev_idx = ar_idx++;
      prev_symm = true;
    } else {
      CKI(enqueue_gemm(e, L, w.act, lw.down, M, EPI_PARTIAL, w.partials, 0, m.d, &S));
    }
    prev.dense = nullptr; prev.partial = w.partials; prev.S = S; prev.M = M; prev.N = m.d;
    if (tp > 1 && !fuse_pub) {
      if (use_symm) {
        CKI(enqueue_ar_publish(e, L, &prev, nullptr, M, m.d, ar_idx));
        prev_idx = ar_idx++;
        prev_symm = true;
      } else {
        CKI(enqueue_tp_allreduce(e, L, S, M, m.d, &prev));
      }
    }
  }
  // ---- final norm ----
  NormParams fn;
  memset(&fn, 0, sizeof(fn));
  fn.x = prev; fn.residual_in = w.residual; fn.w = m.final_norm; fn.eps = m.cfg.rms_eps; fn.y = w.hidden;
  if (prev_symm) fn.symm = symm_in(e, prev_idx, true);
  fn.residual_out = nullptr; fn.d = m.d;
  CKI(launch_norm(L, M, m.d, fn));

  // ---- lm_head ----
  if (f.logits_mode != 0) {
    const bf16* x = w.hidden;
    int rows = M;
    if (f.logits_mode == 2 && f.var) {
      if (M > f.B) {
        CKI(L.go(gather_last_rows_varlen_kernel, dim3(f.B), dim3(256), 0, (const bf16*)w.hidden, w.last_hidden,
                 f.var->attn.cu_q, m.d));
        x = w.last_hidden;
      }
      rows = f.B;
    } else if (f.logits_mode == 2 && f.Q > 1) {
      CKI(L.go(gather_last_rows_kernel, dim3(f.B), dim3(256), 0, (const bf16*)w.hidden, w.last_hidden, f.B, f.Q, m.d));
      x = w.last_hidden;
      rows = f.B;
    } else if (f.logits_mode == 2) {
      rows = f.B;
    }
    if (tp == 1) {
      CKI(enqueue_gemm(e, L, x, m.lm_head, rows, EPI_BF16, f.logits_out, (int)f.logits_ld, m.vocab_local, nullptr));
    } else {
      // ParallelLMHead (embed_head.py:94-116): per-rank vocab shard, gathered and concatenated on rank 0
      const int Vs = m.vocab_local;
      if (Vs % 8) return fail("tensor-parallel lm_head: vocab shard %d not a multiple of 8", Vs);
      CKI(enqueue_gemm(e, L, x, m.lm_head, rows, EPI_BF16, w.logits_shard, Vs, Vs, nullptr));
      CKN(ncclAllGather(w.logits_shard, w.logits_gather, (size_t)rows * Vs, ncclBfloat16, e->comm, L.st));
      L.barrier_op();
      if (m.cfg.tp_rank == 0 && f.logits_out)
        CKI(L.go(unshard_logits_kernel, dim3(num_sms()), dim3(256), 0, (const bf16*)w.logits_gather, f.logits_out, tp, rows,
                 Vs, f.logits_ld));
    }
  }
  return 0;
}

// ------------------------------------------------------------------------------------------
// step block layout (host pinned <-> device), all offsets 16-byte aligned
// ------------------------------------------------------------------------------------------
static void layout_step(ssdk_engine* e) {
  const int MB = e->rt.max_batch, mbk = e->rt.max_blocks_per_seq;
  size_t off = 0;
  auto take = [&](size_t n) { size_t o = off; off = align_up(off + n, 16); return o; };
  e->off_ctx = take((size_t)MB * 4);
  e->off_rec = take((size_t)MB * 8);
  e->off_pend = take((size_t)MB * 8);
  e->off_tt = take((size_t)MB * 4);
  e->off_tq = take((size_t)MB * 4);
  e->off_seed = take(16);
  e->off_btt = take((size_t)MB * mbk * 4);
  e->off_btd = take((size_t)MB * mbk * 4);
  e->step_bytes = off;
  e->off_out_nacc = align_up((size_t)MB * (e->rt.spec_k + 1) * 8, 16);
  e->off_out_rec = e->off_out_nacc + align_up((size_t)MB * 4, 16);
  e->out_bytes = align_up(e->off_out_rec + (size_t)MB * 8, 16);
}



// copy the recovery tokens into column 0 of the speculation buffer (speculator_sync.py:38-45), and the ids of the
// kernel-per-op draft's two-row forward 0: {token at ctx-1 (the recovery token again when nothing is pending: computed,
// never stored), recovery}
__global__ void init_tokens_kernel(const int64_t* __restrict__ recovery, const int64_t* __restrict__ pend,
                                   int64_t* __restrict__ tok_buf, int64_t* __restrict__ fold_ids, int B, int Kp1) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = threadIdx.x;
  if (b < B) {
    tok_buf[(size_t)b * Kp1] = recovery[b];
    fold_ids[2 * b] = pend[b] >= 0 ? pend[b] : recovery[b];
    fold_ids[2 * b + 1] = recovery[b];
  }
}

// Device-resident bookkeeping between two spec steps (resident mode only): what
// Scheduler.postprocess_speculate does to num_cached_tokens / recovery_token_id
// (engine/scheduler.py:248-262), plus an on-device log of the accepted tokens.  A step that accepted all K drafts leaves
// the draft KV of d_K (position ctx-1 of the next step) to the next step's first draft forward: pend = d_K, else -1.
__global__ void advance_kernel(int32_t* __restrict__ ctx, int64_t* __restrict__ recovery_in, int64_t* __restrict__ pend,
                               uint64_t* __restrict__ seed_step, const int64_t* __restrict__ tok_buf,
                               const int32_t* __restrict__ n_accept, const int64_t* __restrict__ recovery_out,
                               int64_t* __restrict__ log_tokens, int32_t* __restrict__ log_len, int B, int Kp1, int log_cap) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = threadIdx.x;
  if (b < B) {
    const int n = n_accept[b] + 1;  // recovery + accepted drafts
    int len = log_len[b];
    for (int j = 0; j < n && len < log_cap; ++j) log_tokens[(size_t)b * log_cap + len++] = tok_buf[(size_t)b * Kp1 + j];
    log_len[b] = len;
    ctx[b] += n;
    recovery_in[b] = recovery_out[b];
    pend[b] = (n == Kp1) ? tok_buf[(size_t)b * Kp1 + Kp1 - 1] : -1;
  }
  if (threadIdx.x == 0) seed_step[1] += 1;
}

// ------------------------------------------------------------------------------------------
// spec step: K draft forwards -> (K+1)-token target forward -> verify      (enqueue only)
// The reference's K+1-th draft forward (KV of d_K only) is folded into the next step's first draft forward as its row 0
// when the step accepted all K drafts (pend[b] >= 0, the token at ctx-1); the host flushes it with a one-token draft
// forward when the sequence does not continue (PairRunner).
// ------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------
// streaming draft kernel: the K draft forwards + K samplings of a step in ONE cooperative launch (draft_stream.cuh)
// SSDK_DRAFT_STREAM=0 keeps the kernel-per-op path.
// ------------------------------------------------------------------------------------------
static bool draft_stream_enabled() {
  static int v = -1;
  if (v < 0) v = env_int("SSDK_DRAFT_STREAM", 1) != 0 ? 1 : 0;
  return v == 1;
}
constexpr int kMaxDynSmem = 227 * 1024 - 2048;  // opt-in limit per CTA minus the kernel's static shared memory (1.8 KB)
static size_t ds_fixed_smem(const Model& m) {
  const int G = m.H / m.KV, gmax = G <= 4 ? 4 : 8;
  const size_t xs = (size_t)ds_xs_floats(m.d, m.ffn, m.H * m.hd);
  const size_t scratch = (size_t)gmax * m.hd + 2 * m.hd + (size_t)kDsWarps * gmax * (m.hd + 2);
  return (xs + scratch) * 4 + 256;
}
static int ds_ring_slots(const Model& m) {
  const size_t fixed = ds_fixed_smem(m);
  if (fixed + 3 * (size_t)kDsSlotBytes > (size_t)kMaxDynSmem) return 0;
  return (int)std::min<size_t>(kDsMaxSlots, ((size_t)kMaxDynSmem - fixed) / kDsSlotBytes);
}
static bool draft_stream_supported(const Model& m, int B) {
  const int G = m.KV ? m.H / m.KV : 0;
  DsGeom g;
  return B == 1 && m.cfg.tp_size == 1 && m.cfg.layers <= kDsMaxLayers && (m.hd == 64 || m.hd == 128) && G >= 1 && G <= 8 &&
         m.H % m.KV == 0 && m.KV <= 32 && m.d % 8 == 0 && (m.H * m.hd) % 8 == 0 && m.ffn % 8 == 0 &&
         ds_geometry(m.d, m.qkv_dim, false, &g) && ds_geometry(m.H * m.hd, m.d, false, &g) &&
         ds_geometry(m.d, m.ffn, true, &g) && ds_geometry(m.ffn, m.d, false, &g) && ds_geometry(m.d, m.cfg.vocab, false, &g) &&
         ds_ring_slots(m) >= 3;
}
// Which draft path a step takes.  The streaming kernel wins while the attention phase of a KV split is ONE round of loads
// (16 splits x 8 warps x 8 tokens = 1024 tokens); every further round costs more than the kernel-per-op draft's tensor-core
// attention, so longer contexts take the
// kernel-per-op graph.  Both graphs compute the same step; ctx_bound = the longest context of the batch before the step.
static int draft_stream_max_ctx() {
  static int v = -1;
  if (v < 0) v = std::max(0, env_int("SSDK_DRAFT_STREAM_MAX_CTX", 1024));
  return v;
}
static bool use_draft_stream(ssdk_engine* e, int B, int ctx_bound) {
  const Model& drf = e->model[SSDK_DRAFT];
  return drf.present && draft_stream_enabled() && draft_stream_supported(drf, B) &&
         ctx_bound + e->rt.spec_k + 1 <= draft_stream_max_ctx();
}
template <int HD, int GMAX, bool FP8>
static int launch_draft_stream(Launcher& L, const DsParams& p, size_t smem) {
  static bool attr_set = false;
  if (!attr_set) {
    CK(cudaFuncSetAttribute(draft_stream_kernel<HD, GMAX, FP8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(num_sms());
  cfg.blockDim = dim3(kDsThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = L.st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;  // all CTAs must be co-resident: the phases meet at device-wide barriers
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;  // (a plain launch measured the same step time: 5.70 vs 5.66 ms — the attribute costs nothing between steps)
  cudaError_t err = cudaLaunchKernelEx(&cfg, draft_stream_kernel<HD, GMAX, FP8>, p);
  if (err != cudaSuccess) return fail("draft stream launch failed: %s", cudaGetErrorString(err));
  L.barrier_op();  // not a PDL primary: the next kernel starts after this grid has drained
  ++L.count;
  return 0;
}
// forwards 0 .. n_fwd-1 of the draft on tok_buf[0 ..]; samples tok_buf[f + 1] after every forward; forward 0 also writes
// the KV of pend[0] at ctx0 - 1 when pend[0] >= 0
static int enqueue_draft_stream(ssdk_engine* e, Launcher& L, int64_t* tok_buf, int n_fwd, const int64_t* pend,
                                const int32_t* ctx0, const int32_t* block_table, const float* temp, const uint64_t* dyn,
                                bf16* logits, int64_t logits_ld) {
  Model& m = e->model[SSDK_DRAFT];
  Workspace& w = e->ws;
  DsParams p;
  memset(&p, 0, sizeof(p));
  p.d = m.d; p.L = m.cfg.layers; p.H = m.H; p.KV = m.KV; p.ffn = m.ffn; p.vocab = m.cfg.vocab; p.qk_norm = m.cfg.qk_norm;
  p.eps = m.cfg.rms_eps;
  p.scale_log2 = (1.0f / sqrtf((float)m.hd)) * 1.4426950408889634f;
  p.embed = m.embed.ptr; p.final_norm = m.final_norm; p.lm_head = m.lm_head.ptr; p.rope = m.rope;
  p.k_cache = m.k_cache; p.v_cache = m.v_cache;
  p.cache_layer_stride = (long long)m.num_blocks * e->rt.block_size * m.KV * m.hd;
  p.block_size = e->rt.block_size; p.max_blocks = e->rt.max_blocks_per_seq;
  p.tok_buf = tok_buf; p.n_fwd = n_fwd; p.skip_last_head = 0;
  p.pend_tok = pend; p.vec_row0 = w.ds_vec0;
  p.ctx0 = ctx0; p.block_table = block_table;
  bf16* v = w.ds_vec;
  p.vec_qkv = v; v += align_up((size_t)m.qkv_dim, 8);
  p.vec_attn = v; v += (size_t)m.H * m.hd;
  p.vec_o = v; v += m.d;
  p.vec_down = v; v += m.d;
  p.resid0 = v; v += m.d;
  p.resid1 = v; v += m.d;
  p.vec_act = v;
  p.attn_part = w.ds_attn;
  p.logits = logits; p.logits_ld = logits_ld;
  p.temp = temp; p.dyn = dyn;
  p.samp_partial = w.samp_partial;
  p.bar_state = w.ds_sync;
  p.attn_ticket = w.ds_sync + 8;
  p.n_slots = ds_ring_slots(m);
  for (int l = 0; l < p.L; ++l) {
    const LayerW& lw = m.layers[l];
    p.layers[l] = DsLayer{lw.qkv.ptr, lw.o.ptr, lw.gate_up.ptr, lw.down.ptr, lw.input_norm, lw.post_norm, lw.q_norm, lw.k_norm};
    const WeightMat* mats[4] = {&lw.qkv, &lw.o, &lw.gate_up, &lw.down};  // DS_QKV .. DS_DOWN
    for (int i = 0; i < 4; ++i) p.fp8_scale[l][i] = mats[i]->scale;
  }
  const int G = m.H / m.KV, gmax = G <= 4 ? 4 : 8;
  const size_t smem = ds_fixed_smem(m) + (size_t)p.n_slots * kDsSlotBytes;
  if (model_linears_fp8(m)) {  // every decoder linear is FP8 (ssdk_finalize refuses a mixed draft)
    if (m.hd == 64 && gmax == 4) return launch_draft_stream<64, 4, true>(L, p, smem);
    if (m.hd == 64 && gmax == 8) return launch_draft_stream<64, 8, true>(L, p, smem);
    if (m.hd == 128 && gmax == 4) return launch_draft_stream<128, 4, true>(L, p, smem);
    return launch_draft_stream<128, 8, true>(L, p, smem);
  }
  if (m.hd == 64 && gmax == 4) return launch_draft_stream<64, 4, false>(L, p, smem);
  if (m.hd == 64 && gmax == 8) return launch_draft_stream<64, 8, false>(L, p, smem);
  if (m.hd == 128 && gmax == 4) return launch_draft_stream<128, 4, false>(L, p, smem);
  return launch_draft_stream<128, 8, false>(L, p, smem);
}

static int enqueue_spec_step(ssdk_engine* e, Launcher& L, int B, bool host_io, bool advance, bool stream_draft) {
  Workspace& w = e->ws;
  const int K = e->rt.spec_k;
  Model& tgt = e->model[SSDK_TARGET];
  Model& drf = e->model[SSDK_DRAFT];
  const int V = tgt.cfg.vocab;
  if (host_io) {
    CK(cudaMemcpyAsync(w.step_dev, e->pin_in, e->step_bytes, cudaMemcpyHostToDevice, L.st));
    L.barrier_op();
  }
  int32_t* ctx = (int32_t*)(w.step_dev + e->off_ctx);
  int64_t* rec_in = (int64_t*)(w.step_dev + e->off_rec);
  int64_t* pend = (int64_t*)(w.step_dev + e->off_pend);
  const float* tt = (const float*)(w.step_dev + e->off_tt);
  const float* tq = (const float*)(w.step_dev + e->off_tq);
  uint64_t* seed_step = (uint64_t*)(w.step_dev + e->off_seed);
  const int32_t* btt = (const int32_t*)(w.step_dev + e->off_btt);
  const int32_t* btd = (const int32_t*)(w.step_dev + e->off_btd);

  const int tp = tgt.cfg.tp_size, tp_rank = tgt.cfg.tp_rank;
  if (tp > 1 && !e->comm) return fail("tensor parallel spec step without a NCCL communicator");
  if (tp_rank == 0 && !drf.present) return fail("rank 0 needs the draft model");
  if (drf.present)
    CKI(L.go(init_tokens_kernel, dim3(1), dim3(64), 0, (const int64_t*)rec_in, (const int64_t*)pend, w.tok_buf, w.fold_ids,
             B, K + 1));
  if (stream_draft)
    CKI(enqueue_draft_stream(e, L, w.tok_buf, K, pend, ctx, btd, tq, seed_step, w.logits_q, (int64_t)V));
  for (int k = 0; k < K && drf.present && !stream_draft; ++k) {
    Fwd f;
    f.which = SSDK_DRAFT; f.B = B; f.Q = 1; f.ids = w.tok_buf + k; f.ids_stride = K + 1;
    f.ctx0 = ctx; f.block_tables = btd; f.pos_offset = k;
    f.logits_mode = 1;
    if (k == 0) {
      // two rows per sequence: the token at ctx-1 (K/V stored only when pending) and the recovery token; logits of row 1
      f.Q = 2; f.ids = w.fold_ids; f.ids_stride = 1; f.pos_offset = -1; f.logits_mode = 2; f.pend = pend;
    }
    f.logits_out = w.logits_q + (size_t)k * V;
    f.logits_ld = (int64_t)K * V;
    CKI(enqueue_forward(e, L, f));
    SampleParams sp;
    sp.logits = w.logits_q + (size_t)k * V; sp.ld = (int64_t)K * V; sp.temps = tq; sp.V = drf.cfg.vocab;
    sp.seed = 0; sp.call_id = 0; sp.out = w.tok_buf + k + 1; sp.out_stride = K + 1;
    sp.partial = w.samp_partial; sp.counters = w.samp_counters; sp.dyn = seed_step; sp.sub = k;
    CKI(L.go(sample_kernel, dim3(kSampleChunks, B), dim3(256), 0, sp));
  }
  if (tp > 1) {
    // the draft is pinned to rank 0: ship its K tokens (+ recovery) to the other ranks device-side
    CKN(ncclBroadcast(w.tok_buf, w.tok_buf, (size_t)B * (K + 1), ncclInt64, 0, e->comm, L.st));
    L.barrier_op();
  }
  {
    Fwd f;
    f.which = SSDK_TARGET; f.B = B; f.Q = K + 1; f.ids = w.tok_buf; f.ids_stride = 1;
    f.ctx0 = ctx; f.block_tables = btt; f.pos_offset = 0; f.logits_mode = 1;
    f.logits_out = w.logits_p; f.logits_ld = V;
    CKI(enqueue_forward(e, L, f));
  }
  if (tp_rank == 0) {
    VerifyParams vp;
    vp.lp = w.logits_p; vp.lq = w.logits_q; vp.spec = w.tok_buf; vp.temps_t = tt; vp.temps_q = tq;
    vp.cache_hits = nullptr; vp.jit = e->rt.jit_speculate; vp.B = B; vp.K = K; vp.V = V;
    vp.seed = 0; vp.call_id = 0; vp.n_accept = w.n_accept; vp.recovery = w.recovery;
    vp.row_part = w.ver_rows; vp.rec_part = w.ver_rec; vp.counters = w.ver_counters;
    vp.dyn = seed_step; vp.sub = 15;
    CKI(L.go(verify_kernel, dim3(kVerifyCtas), dim3(kVerifyThreads), 0, vp));
  }
  if (tp > 1) {
    // rank 0 holds the verdict: broadcast it so that every rank (SPMD host engines, resident loop) sees the same
    // tokens / accept counts / recovery tokens
    CKN(ncclBroadcast(w.out_dev, w.out_dev, e->out_bytes, ncclChar, 0, e->comm, L.st));
    L.barrier_op();
  }
  if (advance) {
    CKI(L.go(advance_kernel, dim3(1), dim3(64), 0, ctx, rec_in, pend, seed_step, (const int64_t*)w.tok_buf,
             (const int32_t*)w.n_accept, (const int64_t*)w.recovery, w.log_tokens, w.log_len, B, K + 1, kLogCap));
  }
  if (host_io) {
    CK(cudaMemcpyAsync(e->pin_out, w.out_dev, e->out_bytes, cudaMemcpyDeviceToHost, L.st));
    L.barrier_op();
  }
  return 0;
}

static int get_spec_graph(ssdk_engine* e, int B, bool host_io, bool stream_draft, cudaStream_t st, cudaGraphExec_t* out,
                          int64_t* nlaunch) {
  auto& cache = host_io ? e->spec_graphs : e->spec_graphs_resident;
  const int key = B * 2 + (stream_draft ? 1 : 0);
  auto it = cache.find(key);
  if (it != cache.end()) {
    *out = it->second;
    *nlaunch = e->spec_graph_launches[key];
    return 0;
  }
  (void)st;
  if (!e->cap_stream) CK(cudaStreamCreateWithFlags(&e->cap_stream, cudaStreamNonBlocking));
  Launcher L;
  L.st = e->cap_stream;
  L.pdl = e->rt.use_pdl != 0;
  cudaGraph_t graph = nullptr;
  CK(cudaStreamBeginCapture(e->cap_stream, cudaStreamCaptureModeThreadLocal));
  const int rc = enqueue_spec_step(e, L, B, host_io, !host_io, stream_draft);
  cudaError_t ce = cudaStreamEndCapture(e->cap_stream, &graph);
  if (rc != 0) {
    if (graph) cudaGraphDestroy(graph);
    return rc;
  }
  if (ce != cudaSuccess) return fail("graph capture failed: %s", cudaGetErrorString(ce));
  cudaGraphExec_t exec = nullptr;
  ce = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ce != cudaSuccess) return fail("graph instantiate failed: %s", cudaGetErrorString(ce));
  cache[key] = exec;
  e->spec_graph_launches[key] = L.count;
  *out = exec;
  *nlaunch = L.count;
  return 0;
}

// pre-set >48 KB dynamic smem opt-ins so nothing but launches happens during capture
static int init_kernel_attrs() {
#define SSDK_ATTR_G(UN, EP)                                                                                    \
  CK(cudaFuncSetAttribute(gemm_ws_kernel<UN, EP, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,          \
                          GemmCfg<UN>::kSmemBytes));                                                           \
  CK(cudaFuncSetAttribute(gemm_ws_kernel<UN, EP, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,           \
                          GemmCfg<UN, true>::kSmemBytes));
  SSDK_ATTR_G(16, EPI_BF16) SSDK_ATTR_G(16, EPI_PARTIAL) SSDK_ATTR_G(16, EPI_SILU) SSDK_ATTR_G(16, EPI_PUBLISH)
  SSDK_ATTR_G(32, EPI_BF16) SSDK_ATTR_G(32, EPI_PARTIAL) SSDK_ATTR_G(32, EPI_SILU) SSDK_ATTR_G(32, EPI_PUBLISH)
  SSDK_ATTR_G(64, EPI_BF16) SSDK_ATTR_G(64, EPI_PARTIAL) SSDK_ATTR_G(64, EPI_SILU) SSDK_ATTR_G(64, EPI_PUBLISH)
  SSDK_ATTR_G(128, EPI_BF16) SSDK_ATTR_G(128, EPI_PARTIAL) SSDK_ATTR_G(128, EPI_SILU)
  SSDK_ATTR_G(256, EPI_BF16) SSDK_ATTR_G(256, EPI_PARTIAL) SSDK_ATTR_G(256, EPI_SILU)
#undef SSDK_ATTR_G
#define SSDK_ATTR_A(HD, MT)                                                                                      \
  CK(cudaFuncSetAttribute(paged_attn_kernel<HD, MT, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, attn_smem_bytes(HD))); \
  CK(cudaFuncSetAttribute(paged_attn_kernel<HD, MT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, attn_smem_bytes(HD)));
  SSDK_ATTR_A(128, 1) SSDK_ATTR_A(128, 2) SSDK_ATTR_A(128, 4) SSDK_ATTR_A(64, 1) SSDK_ATTR_A(64, 2) SSDK_ATTR_A(64, 4)
#undef SSDK_ATTR_A
#define SSDK_ATTR_AV(HD, MT)                                                                                     \
  CK(cudaFuncSetAttribute(paged_attn_varlen_kernel<HD, MT, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, attn_smem_bytes(HD))); \
  CK(cudaFuncSetAttribute(paged_attn_varlen_kernel<HD, MT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, attn_smem_bytes(HD)));
  SSDK_ATTR_AV(128, 1) SSDK_ATTR_AV(128, 2) SSDK_ATTR_AV(128, 4) SSDK_ATTR_AV(64, 1) SSDK_ATTR_AV(64, 2) SSDK_ATTR_AV(64, 4)
#undef SSDK_ATTR_AV
  CK(cudaFuncSetAttribute(add_rmsnorm_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
  return 0;
}

// lazily allocated device scratch for the stand-alone sampler op
static void* g_op_scratch = nullptr;
static int op_scratch(void** out, cudaStream_t st) {
  if (!g_op_scratch) {
    CK(cudaMalloc(&g_op_scratch, 1 << 20));
    CK(cudaMemsetAsync(g_op_scratch, 0, 1 << 20, st));
  }
  *out = g_op_scratch;
  return 0;
}

// ==========================================================================================
// extern "C" surface
// ==========================================================================================
extern "C" {

int ssdk_abi_version(void) { return SSDK_ABI_VERSION; }
const char* ssdk_last_error(void) { return g_err.c_str(); }

int ssdk_create(const ssdk_model_cfg* target, const ssdk_model_cfg* draft, const ssdk_runtime_cfg* rt, ssdk_handle* out) {
  if (!target || !rt || !out) return fail("ssdk_create: null argument");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail("ssdk_create: no CUDA device");
  if (rt->spec_k < 0 || rt->spec_k > 7) return fail("spec_k=%d out of range [0,7]", rt->spec_k);
  if (rt->max_batch < 1 || rt->max_batch * (rt->spec_k + 1) > kMaxTokens || rt->max_batch > kVerifyMaxBatch)
    return fail("max_batch=%d: need max_batch*(K+1) <= %d and max_batch <= %d", rt->max_batch, kMaxTokens, kVerifyMaxBatch);
  if (rt->spec_k > 0 && !draft && target->tp_rank == 0) return fail("spec_k>0 needs a draft model on rank 0");
  if (rt->draft_fp8 != 0 && rt->draft_fp8 != 1) return fail("draft_fp8=%d: 0 (bf16 draft) or 1 (FP8 draft)", rt->draft_fp8);
  ssdk_engine* e = new ssdk_engine();
  e->rt = *rt;
  const ssdk_model_cfg* cfgs[2] = {target, draft};
  for (int w = 0; w < 2; ++w) {
    if (!cfgs[w]) continue;
    Model& m = e->model[w];
    m.cfg = *cfgs[w];
    m.present = true;
    const ssdk_model_cfg c = m.cfg;  // by value: the error paths below free the engine before formatting the message
    if (c.tp_size < 1 || c.heads % c.tp_size || c.kv_heads % c.tp_size || c.ffn % c.tp_size || c.vocab % c.tp_size) {
      delete e;
      return fail("model %d: tp_size %d does not divide heads/kv_heads/ffn/vocab", w, c.tp_size);
    }
    if (c.head_dim != 64 && c.head_dim != 128) {
      delete e;
      return fail("model %d: head_dim %d unsupported", w, c.head_dim);
    }
    if (c.hidden % 64 || (c.ffn / c.tp_size) % 64) {
      delete e;
      return fail("model %d: hidden/ffn must be multiples of 64", w);
    }
    derive(m);
    m.layers.resize(c.layers);
  }
  if (draft && draft->vocab != target->vocab) {
    delete e;
    return fail("draft and target vocab differ (model_runner.py:49)");
  }
  layout_step(e);
  e->max_ctx_hint = rt->max_blocks_per_seq * rt->block_size;
  if (cudaHostAlloc((void**)&e->pin_in, e->step_bytes, cudaHostAllocDefault) != cudaSuccess ||
      cudaHostAlloc((void**)&e->pin_out, e->out_bytes + 64 * 8, cudaHostAllocDefault) != cudaSuccess) {
    delete e;
    return fail("pinned staging allocation failed");
  }
  memset(e->pin_in, 0, e->step_bytes);
  e->fw_slot_bytes = align_up(e->step_bytes, 64) + kFwInBytes;
  if (cudaHostAlloc((void**)&e->pin_fw, e->fw_slot_bytes * ssdk_engine::kFwSlots, cudaHostAllocDefault) != cudaSuccess) {
    cudaFreeHost(e->pin_in);
    cudaFreeHost(e->pin_out);
    delete e;
    return fail("pinned staging allocation failed");
  }
  memset(e->pin_fw, 0, e->fw_slot_bytes * ssdk_engine::kFwSlots);
  for (int i = 0; i < ssdk_engine::kFwSlots; ++i) {
    if (cudaEventCreateWithFlags(&e->fw_ev[i], cudaEventDisableTiming) != cudaSuccess) {
      delete e;
      return fail("event creation failed");
    }
  }
  *out = e;
  return 0;
}

int ssdk_destroy(ssdk_handle h) {
  if (!h) return 0;
  for (auto& kv : h->spec_graphs) cudaGraphExecDestroy(kv.second);
  for (auto& kv : h->spec_graphs_resident) cudaGraphExecDestroy(kv.second);
  if (h->cap_stream) cudaStreamDestroy(h->cap_stream);
  if (h->pin_in) cudaFreeHost(h->pin_in);
  if (h->pin_out) cudaFreeHost(h->pin_out);
  if (h->pin_fw) cudaFreeHost(h->pin_fw);
  for (int i = 0; i < ssdk_engine::kFwSlots; ++i)
    if (h->fw_ev[i]) cudaEventDestroy(h->fw_ev[i]);
  delete h;
  return 0;
}

int ssdk_bind_weight(ssdk_handle h, int which, int kind, int layer, const void* dev_ptr, int64_t rows, int64_t cols) {
  if (!h || which < 0 || which > 1 || !h->model[which].present) return fail("bind_weight: bad handle/model");
  Model& m = h->model[which];
  if (!dev_ptr) return fail("bind_weight: null pointer");
  auto mat = [&](WeightMat& w, int64_t er, int64_t ec) -> int {
    if (rows != er || cols != ec)
      return fail("bind_weight kind %d layer %d: shape [%lld,%lld], expected [%lld,%lld]", kind, layer, (long long)rows,
                  (long long)cols, (long long)er, (long long)ec);
    w.ptr = (const bf16*)dev_ptr; w.scale = nullptr; w.rows = rows; w.cols = cols; w.has_tm = false;
    return 0;
  };
  auto vec = [&](const bf16** dst, int64_t n) -> int {
    if (rows * std::max<int64_t>(cols, 1) != n) return fail("bind_weight kind %d: %lld elements, expected %lld", kind,
                                                            (long long)(rows * std::max<int64_t>(cols, 1)), (long long)n);
    *dst = (const bf16*)dev_ptr;
    return 0;
  };
  const bool per_layer = kind >= SSDK_W_INPUT_NORM && kind <= SSDK_W_DOWN;
  if (per_layer && (layer < 0 || layer >= m.cfg.layers)) return fail("bind_weight: layer %d out of range", layer);
  switch (kind) {
    case SSDK_W_EMBED: return mat(m.embed, m.vocab_local, m.d);
    case SSDK_W_LM_HEAD: return mat(m.lm_head, m.vocab_local, m.d);
    case SSDK_W_FINAL_NORM: return vec(&m.final_norm, m.d);
    case SSDK_W_INPUT_NORM: return vec(&m.layers[layer].input_norm, m.d);
    case SSDK_W_QKV: return mat(m.layers[layer].qkv, m.qkv_dim, m.d);
    case SSDK_W_Q_NORM: return vec(&m.layers[layer].q_norm, m.hd);
    case SSDK_W_K_NORM: return vec(&m.layers[layer].k_norm, m.hd);
    case SSDK_W_O: return mat(m.layers[layer].o, m.d, (int64_t)m.H * m.hd);
    case SSDK_W_POST_NORM: return vec(&m.layers[layer].post_norm, m.d);
    case SSDK_W_GATE_UP: return mat(m.layers[layer].gate_up, 2 * (int64_t)m.ffn, m.d);
    case SSDK_W_DOWN: return mat(m.layers[layer].down, m.d, m.ffn);
    case SSDK_W_ROPE_TABLE:
      if (cols != m.hd) return fail("rope table width %lld != head_dim %d", (long long)cols, m.hd);
      m.rope = (const float*)dev_ptr;
      m.rope_rows = rows;
      return 0;
    default: return fail("bind_weight: unknown kind %d", kind);
  }
}

int ssdk_bind_weight_fp8(ssdk_handle h, int which, int kind, int layer, const void* w_e4m3, const float* row_scale,
                         int64_t rows, int64_t cols) {
  if (!h || which < 0 || which > 1 || !h->model[which].present) return fail("bind_weight_fp8: bad handle/model");
  if (which != SSDK_TARGET && !h->rt.draft_fp8)
    return fail("bind_weight_fp8: FP8 weights are supported for the target model only unless the runtime config sets "
                "draft_fp8 = 1");
  if (!w_e4m3 || !row_scale) return fail("bind_weight_fp8: null pointer");
  Model& m = h->model[which];
  if (layer < 0 || layer >= m.cfg.layers) return fail("bind_weight_fp8: layer %d out of range", layer);
  LayerW& lw = m.layers[layer];
  WeightMat* w = nullptr;
  int64_t er = 0, ec = 0;
  switch (kind) {
    case SSDK_W_QKV: w = &lw.qkv; er = m.qkv_dim; ec = m.d; break;
    case SSDK_W_O: w = &lw.o; er = m.d; ec = (int64_t)m.H * m.hd; break;
    case SSDK_W_GATE_UP: w = &lw.gate_up; er = 2 * (int64_t)m.ffn; ec = m.d; break;
    case SSDK_W_DOWN: w = &lw.down; er = m.d; ec = m.ffn; break;
    default: return fail("bind_weight_fp8: kind %d has no FP8 form (qkv, o, gate_up and down only)", kind);
  }
  if (rows != er || cols != ec)
    return fail("bind_weight_fp8 kind %d layer %d: shape [%lld,%lld], expected [%lld,%lld]", kind, layer, (long long)rows,
                (long long)cols, (long long)er, (long long)ec);
  if (cols % kBlockK8) return fail("bind_weight_fp8 kind %d: K=%lld is not a multiple of %d", kind, (long long)cols, kBlockK8);
  if (((uintptr_t)w_e4m3 & 15) != 0) return fail("bind_weight_fp8: weight pointer not 16-byte aligned");
  w->ptr = (const bf16*)w_e4m3; w->scale = row_scale; w->rows = rows; w->cols = cols; w->has_tm = false;
  return 0;
}

int ssdk_bind_kv_cache(ssdk_handle h, int which, void* kv_base, int64_t num_blocks) {
  if (!h || which < 0 || which > 1 || !h->model[which].present) return fail("bind_kv_cache: bad handle/model");
  Model& m = h->model[which];
  if (!kv_base || num_blocks < 1) return fail("bind_kv_cache: bad arguments");
  m.num_blocks = num_blocks;
  m.k_cache = (bf16*)kv_base;
  m.v_cache = m.k_cache + (size_t)m.cfg.layers * num_blocks * h->rt.block_size * m.KV * m.hd;
  m.kv_fp8 = false;
  return 0;
}

int ssdk_bind_kv_cache_fp8(ssdk_handle h, int which, void* kv_base, int64_t num_blocks, const float* k_scale,
                           const float* v_scale) {
  if (!h || which < 0 || which > 1 || !h->model[which].present) return fail("bind_kv_cache_fp8: bad handle/model");
  if (which != SSDK_TARGET) return fail("bind_kv_cache_fp8: only the target's KV cache can be FP8 (the draft's stays bf16)");
  if (h->finalized) return fail("bind_kv_cache_fp8: the engine is already finalized");
  Model& m = h->model[which];
  if (!kv_base || num_blocks < 1 || !k_scale || !v_scale) return fail("bind_kv_cache_fp8: bad arguments");
  if (m.hd != 64 && m.hd != 128) return fail("bind_kv_cache_fp8: head_dim %d (64 and 128 are built)", m.hd);
  if (((uintptr_t)kv_base & 15) != 0) return fail("bind_kv_cache_fp8: cache pointer not 16-byte aligned");
  for (int l = 0; l < m.cfg.layers; ++l)
    if (!(std::isfinite(k_scale[l]) && k_scale[l] > 0.f && std::isfinite(v_scale[l]) && v_scale[l] > 0.f))
      return fail("bind_kv_cache_fp8: layer %d scales k=%g v=%g (finite and > 0 required)", l, k_scale[l], v_scale[l]);
  m.num_blocks = num_blocks;
  m.k_cache = (bf16*)kv_base;
  m.v_cache = (bf16*)((uint8_t*)kv_base + (size_t)m.cfg.layers * num_blocks * h->rt.block_size * m.KV * m.hd);
  m.k_scale.assign(k_scale, k_scale + m.cfg.layers);
  m.v_scale.assign(v_scale, v_scale + m.cfg.layers);
  m.kv_fp8 = true;
  return 0;
}

int64_t ssdk_workspace_bytes(ssdk_handle h) {
  if (!h) return fail("null handle");
  return carve(h, nullptr);
}
int ssdk_bind_workspace(ssdk_handle h, void* dev_ptr, int64_t bytes) {
  if (!h || !dev_ptr) return fail("bind_workspace: null");
  const int64_t need = carve(h, nullptr);
  if (bytes < need) return fail("workspace too small: %lld < %lld", (long long)bytes, (long long)need);
  if (((uintptr_t)dev_ptr & 1023) != 0) return fail("workspace must be 1024-byte aligned");
  carve(h, (uint8_t*)dev_ptr);
  h->ws_base = dev_ptr;
  h->ws_bytes = bytes;
  h->xmaps.maps.clear();
  return 0;
}

int ssdk_set_nccl_comm(ssdk_handle h, void* nccl_comm) {
  if (!h) return fail("null handle");
  h->comm = (ncclComm_t)nccl_comm;
  return 0;
}
int64_t ssdk_symm_bytes(ssdk_handle h) {
  if (!h) return fail("null handle");
  const Model& m = h->model[SSDK_TARGET];
  if (m.cfg.tp_size <= 1) return 0;
  const int64_t slot = (int64_t)kMaxTokens * m.d * 4;  // {2 x bf16, flag} words
  return 2 * kSymmMaxRanks * slot;
}
int ssdk_bind_symm(ssdk_handle h, void* const* peer_ptrs, int n_peers) {
  if (!h || !peer_ptrs) return fail("bind_symm: null argument");
  const Model& m = h->model[SSDK_TARGET];
  if (n_peers != m.cfg.tp_size || n_peers > kSymmMaxRanks) return fail("bind_symm: %d peers, tp_size %d", n_peers, m.cfg.tp_size);
  for (int r = 0; r < n_peers; ++r) {
    if (!peer_ptrs[r]) return fail("bind_symm: null peer pointer %d", r);
    h->symm_peer[r] = (uint8_t*)peer_ptrs[r];
  }
  h->symm_n = n_peers;
  h->symm_slot_bytes = (unsigned)((size_t)kMaxTokens * m.d * 4);
  return 0;
}

int ssdk_finalize(ssdk_handle h, void* stream) {
  if (!h) return fail("null handle");
  if (!h->ws_base) return fail("finalize: workspace not bound");
  cudaStream_t st = (cudaStream_t)stream;
  for (int w = 0; w < 2; ++w) {
    Model& m = h->model[w];
    if (!m.present) continue;
    if (!m.embed.ptr || !m.lm_head.ptr || !m.final_norm || !m.rope) return fail("model %d: embed/lm_head/final_norm/rope not bound", w);
    if (!m.k_cache) return fail("model %d: KV cache not bound", w);
    if (m.rope_rows < h->max_ctx_hint) return fail("model %d: rope table has %lld rows < max context %d", w, (long long)m.rope_rows, h->max_ctx_hint);
    for (int l = 0; l < m.cfg.layers; ++l) {
      LayerW& lw = m.layers[l];
      if (!lw.input_norm || !lw.post_norm || !lw.qkv.ptr || !lw.o.ptr || !lw.gate_up.ptr || !lw.down.ptr)
        return fail("model %d layer %d: weights missing", w, l);
      if (m.cfg.qk_norm && (!lw.q_norm || !lw.k_norm)) return fail("model %d layer %d: q/k norm missing", w, l);
      CKI(weight_tmap(lw.qkv));
      CKI(weight_tmap(lw.o));
      CKI(weight_tmap(lw.gate_up));
      CKI(weight_tmap(lw.down));
    }
    CKI(weight_tmap(m.lm_head));
  }
  // one weight format per draft, so one streaming-kernel instance: draft_fp8 = 1 asks for every decoder linear in FP8
  const Model& drf = h->model[SSDK_DRAFT];
  if (drf.present && h->rt.draft_fp8 && !model_linears_fp8(drf))
    return fail("finalize: draft_fp8 = 1 but the draft's decoder linears are %s: bind qkv, o, gate_up and down of every "
                "draft layer with ssdk_bind_weight_fp8", model_any_linear_fp8(drf) ? "partly bf16" : "bf16");
  CKI(init_kernel_attrs());
  CK(cudaMemsetAsync(h->ws_base, 0, (size_t)carve(h, nullptr), st));
  CK(cudaStreamSynchronize(st));
  h->finalized = true;
  return 0;
}

static int fill_step(ssdk_handle h, int batch, const int32_t* ctx_len, const int64_t* recovery, const int64_t* pending,
                     const int32_t* btt, const int32_t* btd, const float* tt, const float* tq, uint64_t seed,
                     uint64_t step_id) {
  if (batch < 1 || batch > h->rt.max_batch) return fail("batch %d out of range", batch);
  const int mbk = h->rt.max_blocks_per_seq;
  memcpy(h->pin_in + h->off_ctx, ctx_len, (size_t)batch * 4);
  memcpy(h->pin_in + h->off_rec, recovery, (size_t)batch * 8);
  int64_t* pend = (int64_t*)(h->pin_in + h->off_pend);
  for (int b = 0; b < batch; ++b) {
    pend[b] = pending ? pending[b] : -1;
    if (pend[b] >= 0 && ctx_len[b] < 1) return fail("spec_step: sequence %d has a pending token but no context", b);
  }
  memcpy(h->pin_in + h->off_tt, tt, (size_t)batch * 4);
  memcpy(h->pin_in + h->off_tq, tq, (size_t)batch * 4);
  uint64_t ss[2] = {seed, step_id};
  memcpy(h->pin_in + h->off_seed, ss, 16);
  memcpy(h->pin_in + h->off_btt, btt, (size_t)batch * mbk * 4);
  memcpy(h->pin_in + h->off_btd, btd, (size_t)batch * mbk * 4);
  return 0;
}
static void read_step(ssdk_handle h, int batch, int64_t* out_tokens, int32_t* out_n_accept, int64_t* out_recovery) {
  const int K = h->rt.spec_k;
  if (out_tokens) memcpy(out_tokens, h->pin_out, (size_t)batch * (K + 1) * 8);
  if (out_n_accept) memcpy(out_n_accept, h->pin_out + h->off_out_nacc, (size_t)batch * 4);
  if (out_recovery) memcpy(out_recovery, h->pin_out + h->off_out_rec, (size_t)batch * 8);
}

int ssdk_spec_step(ssdk_handle h, int batch, const int32_t* ctx_len, const int64_t* recovery, const int64_t* pending,
                   const int32_t* block_tables_target, const int32_t* block_tables_draft, const float* temp_t,
                   const float* temp_q, uint64_t seed, uint64_t step_id, int64_t* out_tokens, int32_t* out_n_accept,
                   int64_t* out_recovery, void* stream) {
  if (!h || !h->finalized) return fail("spec_step: engine not finalized");
  if (h->rt.spec_k < 1) return fail("spec_step: engine built without speculation");
  cudaStream_t st = (cudaStream_t)stream;
  CKI(fill_step(h, batch, ctx_len, recovery, pending, block_tables_target, block_tables_draft, temp_t, temp_q, seed,
                step_id));
  const bool stream_draft = use_draft_stream(h, batch, *std::max_element(ctx_len, ctx_len + batch));
  if (h->rt.use_graph) {
    cudaGraphExec_t g;
    int64_t n;
    CKI(get_spec_graph(h, batch, true, stream_draft, st, &g, &n));
    CK(cudaGraphLaunch(g, st));
    h->launches += n;
  } else {
    Launcher L;
    L.st = st;
    L.pdl = h->rt.use_pdl != 0;
    CKI(enqueue_spec_step(h, L, batch, true, false, stream_draft));
    h->launches += L.count;
  }
  CK(cudaStreamSynchronize(st));
  read_step(h, batch, out_tokens, out_n_accept, out_recovery);
  return 0;
}

int ssdk_spec_step_stage(ssdk_handle h, int batch, const int32_t* ctx_len, const int64_t* recovery, const int64_t* pending,
                         const int32_t* block_tables_target, const int32_t* block_tables_draft, const float* temp_t,
                         const float* temp_q, uint64_t seed, uint64_t step_id, void* stream) {
  if (!h || !h->finalized) return fail("spec_step_stage: engine not finalized");
  cudaStream_t st = (cudaStream_t)stream;
  CKI(fill_step(h, batch, ctx_len, recovery, pending, block_tables_target, block_tables_draft, temp_t, temp_q, seed,
                step_id));
  h->resident_ctx_bound = *std::max_element(ctx_len, ctx_len + batch);
  CK(cudaMemcpyAsync(h->ws.step_dev, h->pin_in, h->step_bytes, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(h->ws.log_len, 0, (size_t)h->rt.max_batch * 4, st));
  CK(cudaStreamSynchronize(st));
  return 0;
}

int ssdk_spec_step_resident(ssdk_handle h, int batch, void* stream) {
  if (!h || !h->finalized) return fail("spec_step_resident: engine not finalized");
  if (h->rt.spec_k < 1) return fail("spec_step: engine built without speculation");
  cudaStream_t st = (cudaStream_t)stream;
  // the context lives on the device here; the host keeps an upper bound (every step appends at most K+1 tokens)
  const bool stream_draft = use_draft_stream(h, batch, h->resident_ctx_bound);
  h->resident_ctx_bound += h->rt.spec_k + 1;
  if (h->rt.use_graph) {
    cudaGraphExec_t g;
    int64_t n;
    CKI(get_spec_graph(h, batch, false, stream_draft, st, &g, &n));
    CK(cudaGraphLaunch(g, st));
    h->launches += n;
  } else {
    Launcher L;
    L.st = st;
    L.pdl = h->rt.use_pdl != 0;
    CKI(enqueue_spec_step(h, L, batch, false, true, stream_draft));
    h->launches += L.count;
  }
  return 0;
}

// resident mode read-back: out_tokens receives the LAST step's speculation row, out_n_accept
// the per-sequence TOTAL number of tokens produced since ssdk_spec_step_stage (log length),
// out_recovery the current recovery token.
int ssdk_spec_step_fetch(ssdk_handle h, int batch, int64_t* out_tokens, int32_t* out_n_accept, int64_t* out_recovery,
                         void* stream) {
  if (!h || !h->finalized) return fail("spec_step_fetch: engine not finalized");
  cudaStream_t st = (cudaStream_t)stream;
  CK(cudaMemcpyAsync(h->pin_out, h->ws.out_dev, h->out_bytes, cudaMemcpyDeviceToHost, st));
  int32_t* lens = (int32_t*)(h->pin_out + h->out_bytes);
  CK(cudaMemcpyAsync(lens, h->ws.log_len, (size_t)batch * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  read_step(h, batch, out_tokens, nullptr, out_recovery);
  if (out_n_accept) memcpy(out_n_accept, lens, (size_t)batch * 4);
  return 0;
}

int ssdk_spec_step_log(ssdk_handle h, int seq, int64_t* out_tokens, int cap, void* stream) {
  if (!h || !h->finalized) return fail("spec_step_log: engine not finalized");
  if (seq < 0 || seq >= h->rt.max_batch || !out_tokens || cap < 0) return fail("spec_step_log: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  int32_t len = 0;
  CK(cudaMemcpyAsync(&len, h->ws.log_len + seq, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const int n = std::min(std::min((int)len, cap), kLogCap);
  if (n > 0) {
    CK(cudaMemcpyAsync(out_tokens, h->ws.log_tokens + (size_t)seq * kLogCap, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  return n;
}

// ssdk_forward_tokens (q_lens == nullptr: q_len tokens per sequence) and ssdk_forward_varlen (q_lens[b] tokens of
// sequence b, packed).  Arguments are checked by the callers.
static int forward_call(ssdk_handle h, int which, int batch, int q_len, const int32_t* q_lens, const int64_t* ids,
                        const int32_t* ctx_len, const int32_t* block_tables, int want_sample, const float* temps,
                        uint64_t seed, uint64_t step_id, int64_t* out_tokens, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  Workspace& w = h->ws;
  Model& m = h->model[which];
  const int mbk = h->rt.max_blocks_per_seq;
  VarlenFwd var;
  int M = batch * q_len;
  if (q_lens) {
    int32_t n_tiles = 0;
    const int rc = attn_make_plan_varlen(m.H, m.KV, batch, q_lens, h->max_ctx_hint, num_sms(), &var.plan, &n_tiles);
    if (rc == 1) return fail("unsupported GQA ratio %d/%d", m.H, m.KV);
    if (rc != 0) return fail("attention tile too large");
    var.n_tiles = n_tiles;
    M = 0;
    for (int b = 0; b < batch; ++b) M += q_lens[b];
    var.M = M;
    var.attn.cu_q = w.var_cu_q;
    var.attn.tiles = w.var_tiles;
  }
  // stage inputs through one slot of the pinned ring (block tables go to the step-block field of `which`); wait for the
  // copies that last read this slot before overwriting it — a non-sampling call returns without synchronizing, and its
  // H2D copies are queued behind the previous chunk's kernels
  const int slot = (int)(h->fw_next++ % ssdk_engine::kFwSlots);
  if (h->fw_ev_pending[slot]) {
    CK(cudaEventSynchronize(h->fw_ev[slot]));
    h->fw_ev_pending[slot] = false;
  }
  uint8_t* pin = h->pin_fw + (size_t)slot * h->fw_slot_bytes;
  memcpy(pin + h->off_ctx, ctx_len, (size_t)batch * 4);
  float zero[kVerifyMaxBatch] = {0};
  memcpy(pin + h->off_tt, temps ? temps : zero, (size_t)batch * 4);
  uint64_t ss[2] = {seed, step_id};
  memcpy(pin + h->off_seed, ss, 16);
  memcpy(pin + (which == SSDK_TARGET ? h->off_btt : h->off_btd), block_tables, (size_t)batch * mbk * 4);
  CK(cudaMemcpyAsync(w.step_dev, pin, h->step_bytes, cudaMemcpyHostToDevice, st));
  uint8_t* pin_in = pin + align_up(h->step_bytes, 64);  // ids | cu_q | tile table, as w.ids_in
  memcpy(pin_in, ids, (size_t)M * 8);
  size_t in_bytes = (size_t)M * 8;
  if (q_lens) {
    attn_varlen_tiles(batch, q_lens, var.plan.TQ, (AttnTile*)(pin_in + kFwInTileOff), (int32_t*)(pin_in + kFwInCuOff));
    in_bytes = kFwInTileOff + (size_t)var.n_tiles * sizeof(AttnTile);
  }
  CK(cudaMemcpyAsync(w.ids_in, pin_in, in_bytes, cudaMemcpyHostToDevice, st));
  CK(cudaEventRecord(h->fw_ev[slot], st));
  h->fw_ev_pending[slot] = true;
  // sampled tokens come back through the tail of the result staging buffer (read after the synchronize below)
  int64_t* pin_ids = (int64_t*)(h->pin_out + h->out_bytes);

  Launcher L;
  L.st = st;
  L.pdl = h->rt.use_pdl != 0;
  Fwd f;
  f.which = which; f.B = batch; f.Q = q_len; f.ids = w.ids_in; f.ids_stride = 1;
  f.ctx0 = (const int32_t*)(w.step_dev + h->off_ctx);
  f.block_tables = (const int32_t*)(w.step_dev + (which == SSDK_TARGET ? h->off_btt : h->off_btd));
  f.pos_offset = 0;
  f.logits_mode = want_sample ? 2 : 0;
  f.logits_out = w.logits_last;
  f.logits_ld = m.cfg.vocab;
  f.var = q_lens ? &var : nullptr;
  CKI(enqueue_forward(h, L, f));
  const bool do_sample = want_sample && m.cfg.tp_rank == 0;
  if (do_sample) {
    SampleParams sp;
    sp.logits = w.logits_last; sp.ld = m.cfg.vocab; sp.temps = (const float*)(w.step_dev + h->off_tt);
    sp.V = m.cfg.vocab; sp.seed = seed; sp.call_id = step_id * 16ull + 14ull; sp.out = w.out_tok; sp.out_stride = 1;
    sp.partial = w.samp_partial; sp.counters = w.samp_counters; sp.dyn = nullptr; sp.sub = 0;
    CKI(L.go(sample_kernel, dim3(kSampleChunks, batch), dim3(256), 0, sp));
  }
  if (want_sample) {
    if (m.cfg.tp_size > 1) CKN(ncclBroadcast(w.out_tok, w.out_tok, (size_t)batch, ncclInt64, 0, h->comm, st));
    CK(cudaMemcpyAsync(pin_ids, w.out_tok, (size_t)batch * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (out_tokens) memcpy(out_tokens, pin_ids, (size_t)batch * 8);
  }
  h->launches += L.count;
  return 0;
}

int ssdk_forward_tokens(ssdk_handle h, int which, int batch, int q_len, const int64_t* ids, const int32_t* ctx_len,
                        const int32_t* block_tables, int want_sample, const float* temps, uint64_t seed,
                        uint64_t step_id, int64_t* out_tokens, void* stream) {
  if (!h || !h->finalized) return fail("forward_tokens: engine not finalized");
  if (which < 0 || which > 1 || !h->model[which].present) return fail("forward_tokens: model %d absent", which);
  if (batch < 1 || batch > h->rt.max_batch || q_len < 1 || batch * q_len > kMaxTokens)
    return fail("forward_tokens: batch=%d q_len=%d out of range", batch, q_len);
  return forward_call(h, which, batch, q_len, nullptr, ids, ctx_len, block_tables, want_sample, temps, seed, step_id,
                      out_tokens, stream);
}

int ssdk_forward_varlen(ssdk_handle h, int which, int n_seqs, const int32_t* q_lens, const int64_t* ids,
                        const int32_t* ctx_len, const int32_t* block_tables, int want_sample, const float* temps,
                        uint64_t seed, uint64_t step_id, int64_t* out_tokens, void* stream) {
  if (!h || !h->finalized) return fail("forward_varlen: engine not finalized");
  if (which < 0 || which > 1 || !h->model[which].present) return fail("forward_varlen: model %d absent", which);
  if (n_seqs < 1 || n_seqs > h->rt.max_batch)
    return fail("forward_varlen: n_seqs=%d out of range [1, %d]", n_seqs, h->rt.max_batch);
  if (!q_lens || !ids || !ctx_len || !block_tables) return fail("forward_varlen: null argument");
  int total = 0;
  for (int b = 0; b < n_seqs; ++b) {
    if (q_lens[b] < 1) return fail("forward_varlen: q_lens[%d]=%d < 1", b, q_lens[b]);
    total += q_lens[b];
    if (total > kMaxTokens) return fail("forward_varlen: more than %d tokens in one call", kMaxTokens);
  }
  return forward_call(h, which, n_seqs, 0, q_lens, ids, ctx_len, block_tables, want_sample, temps, seed, step_id,
                      out_tokens, stream);
}

// debug: route the kernels' timeline marks into `dev_buf` (uint64 [cap][2]); dev_buf = NULL disables tracing
int ssdk_debug_trace(void* dev_buf, int cap) {
  unsigned long long* p = (unsigned long long*)dev_buf;
  unsigned c = (unsigned)cap, zero = 0;
  CK(cudaMemcpyToSymbol(g_trace_buf, &p, sizeof(p)));
  CK(cudaMemcpyToSymbol(g_trace_cap, &c, sizeof(c)));
  CK(cudaMemcpyToSymbol(g_trace_n, &zero, sizeof(zero)));
  return 0;
}

const void* ssdk_logits_p(ssdk_handle h) { return h ? h->ws.logits_p : nullptr; }
const void* ssdk_logits_q(ssdk_handle h) { return h ? h->ws.logits_q : nullptr; }
const void* ssdk_logits_last(ssdk_handle h) { return h ? h->ws.logits_last : nullptr; }
int64_t ssdk_launch_count(ssdk_handle h) { return h ? h->launches : 0; }

// ------------------------------------------------------------------------------------------
// stand-alone ops
// ------------------------------------------------------------------------------------------
int ssdk_gemm_small_m(const void* x, const void* w, void* y, float* partials, int M, int N, int K, int ldy, int split_k,
                      void* stream) {
  if (M < 1 || M > kMaxTokens) return fail("gemm_small_m: M=%d out of [1,%d]", M, kMaxTokens);
  if (K % kBlockK) return fail("gemm_small_m: K must be a multiple of 64");
  Launcher L;
  L.st = (cudaStream_t)stream;
  CUtensorMap tmW, tmX;
  CKI(make_tmap(&tmW, w, N, K, 64));
  const int un = umma_n_for(M);
  CKI(make_tmap(&tmX, x, M, K, un));
  const int tiles = (N + kTileRows - 1) / kTileRows;
  const int num_kb = K / kBlockK;
  int S = split_k > 0 ? std::min(split_k, num_kb) : auto_splits(tiles, num_kb, un <= 64 ? 2 : 1);
  if (S > 1 && !partials) return fail("gemm_small_m: split_k=%d needs a partials buffer", S);
  GemmParams p;
  p.M = M; p.N = N; p.ldo = ldy; p.num_kb = num_kb; p.tile_rows = kTileRows; p.hi_row_offset = 64;
  p.kb_per_split = (num_kb + S - 1) / S;
  S = (num_kb + p.kb_per_split - 1) / p.kb_per_split;
  if (S == 1) {
    p.out = y;
    return launch_gemm(L, un, EPI_BF16, tmW, tmX, p, tiles, 1);
  }
  p.out = partials;
  CKI(launch_gemm(L, un, EPI_PARTIAL, tmW, tmX, p, tiles, S));
  const int n = M * N;
  return L.go(splitk_reduce_kernel, dim3((n + 255) / 256), dim3(256), 0, (const float*)partials, (bf16*)y, S, M, N, ldy);
}

int ssdk_gemm_gate_up_silu(const void* x, const void* w_gate_up, void* hout, int M, int ffn, int K, void* stream) {
  if (M < 1 || M > kMaxTokens) return fail("gemm_gate_up_silu: M=%d out of range", M);
  if (K % kBlockK || ffn % 8) return fail("gemm_gate_up_silu: K %% 64 or ffn %% 8 violated");
  Launcher L;
  L.st = (cudaStream_t)stream;
  CUtensorMap tmW, tmX;
  CKI(make_tmap(&tmW, w_gate_up, 2 * (int64_t)ffn, K, 64));
  const int un = umma_n_for(M);
  CKI(make_tmap(&tmX, x, M, K, un));
  GemmParams p;
  p.out = hout; p.M = M; p.N = ffn; p.ldo = ffn; p.num_kb = K / kBlockK; p.kb_per_split = p.num_kb;
  p.tile_rows = 64; p.hi_row_offset = ffn;
  return launch_gemm(L, un, EPI_SILU, tmW, tmX, p, (ffn + 63) / 64, 1);
}

int ssdk_gemm_small_m_fp8(const void* x, const void* w8, const float* scale, void* y, float* partials, int M, int N, int K,
                          int ldy, int split_k, void* stream) {
  if (M < 1 || M > kMaxTokens) return fail("gemm_small_m_fp8: M=%d out of [1,%d]", M, kMaxTokens);
  if (K % kBlockK8) return fail("gemm_small_m_fp8: K=%d is not a multiple of %d", K, kBlockK8);
  if (!scale) return fail("gemm_small_m_fp8: null scale");
  Launcher L;
  L.st = (cudaStream_t)stream;
  CUtensorMap tmW, tmX;
  CKI(make_tmap_e4m3(&tmW, w8, N, K));
  const int un = umma_n_for(M);
  CKI(make_tmap(&tmX, x, M, K, un));
  const int tiles = (N + kTileRows - 1) / kTileRows;
  const int num_kb = K / kBlockK8;
  int S = split_k > 0 ? std::min(split_k, num_kb) : auto_splits(tiles, num_kb, un <= 64 ? 2 : 1);
  if (S > 1 && !partials) return fail("gemm_small_m_fp8: split_k=%d needs a partials buffer", S);
  GemmParams p;
  p.M = M; p.N = N; p.ldo = ldy; p.num_kb = num_kb; p.tile_rows = kTileRows; p.hi_row_offset = 64;
  p.kb_per_split = (num_kb + S - 1) / S;
  S = (num_kb + p.kb_per_split - 1) / p.kb_per_split;
  if (S == 1) {
    p.out = y;
    return launch_gemm(L, un, EPI_BF16, tmW, tmX, p, tiles, 1, scale);
  }
  p.out = partials;
  CKI(launch_gemm(L, un, EPI_PARTIAL, tmW, tmX, p, tiles, S, scale));
  const int n = M * N;
  return L.go(splitk_reduce_kernel, dim3((n + 255) / 256), dim3(256), 0, (const float*)partials, (bf16*)y, S, M, N, ldy);
}

int ssdk_gemm_gate_up_silu_fp8(const void* x, const void* w8_gate_up, const float* scale, void* hout, float* partials,
                               unsigned* counters, int M, int ffn, int K, int split_k, void* stream) {
  if (M < 1 || M > kMaxTokens) return fail("gemm_gate_up_silu_fp8: M=%d out of range", M);
  if (K % kBlockK8 || ffn % 8) return fail("gemm_gate_up_silu_fp8: K %% 128 or ffn %% 8 violated");
  if (!scale) return fail("gemm_gate_up_silu_fp8: null scale");
  Launcher L;
  L.st = (cudaStream_t)stream;
  CUtensorMap tmW, tmX;
  CKI(make_tmap_e4m3(&tmW, w8_gate_up, 2 * (int64_t)ffn, K));
  const int un = umma_n_for(M);
  CKI(make_tmap(&tmX, x, M, K, un));
  const int tiles = (ffn + 63) / 64;
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.out = hout; p.M = M; p.N = ffn; p.ldo = ffn; p.num_kb = K / kBlockK8;
  p.tile_rows = 64; p.hi_row_offset = ffn;
  const int S = std::max(1, std::min(split_k, p.num_kb));
  p.kb_per_split = (p.num_kb + S - 1) / S;
  const int splits = (p.num_kb + p.kb_per_split - 1) / p.kb_per_split;
  if (splits > 1) {
    // in-kernel split-K (the engine's path for narrow tensor-parallel shards): fp32 [S, M, 2 ffn] partials and one
    // zeroed ticket counter per 64-column tile
    if (!partials || !counters) return fail("gemm_gate_up_silu_fp8: split_k=%d needs partials and counters", splits);
    if (un > 64 || tiles > 512) return fail("gemm_gate_up_silu_fp8: split-K is planned for <= 64 tokens, <= 512 tiles");
    p.sk_partials = partials; p.sk_counters = counters; p.sk_width = 2 * ffn;
  }
  return launch_gemm(L, un, EPI_SILU, tmW, tmX, p, tiles, splits, scale);
}

int ssdk_rmsnorm(const void* x, const void* residual_in, const void* w, float eps, void* y, void* residual_out, int M,
                 int d, void* stream) {
  if (d % 8 || d > 16384) return fail("rmsnorm: d=%d unsupported", d);
  Launcher L;
  L.st = (cudaStream_t)stream;
  CKI(init_kernel_attrs());
  NormParams np;
  memset(&np, 0, sizeof(np));
  np.x.dense = (const bf16*)x; np.x.S = 0; np.x.M = M; np.x.N = d;
  np.residual_in = (const bf16*)residual_in; np.w = (const bf16*)w; np.eps = eps;
  np.y = (bf16*)y; np.residual_out = (bf16*)residual_out; np.d = d;
  return launch_norm(L, M, d, np);
}

int ssdk_rope_store_kv(const void* qkv, const int64_t* positions, const int32_t* slot_mapping, const float* rope_table,
                       const void* q_norm_w, const void* k_norm_w, float norm_eps, void* q_out, void* k_cache,
                       void* v_cache, int M, int heads, int kv_heads, int head_dim, void* stream) {
  if (head_dim > 256 || head_dim % 2) return fail("rope: head_dim %d unsupported", head_dim);
  Launcher L;
  L.st = (cudaStream_t)stream;
  RopeParams rp;
  rp.qkv.dense = (const bf16*)qkv; rp.qkv.partial = nullptr; rp.qkv.S = 0; rp.qkv.M = M;
  rp.qkv.N = (heads + 2 * kv_heads) * head_dim;
  rp.positions = positions; rp.slot_mapping = slot_mapping; rp.rope_table = rope_table;
  rp.q_norm_w = (const bf16*)q_norm_w; rp.k_norm_w = (const bf16*)k_norm_w; rp.norm_eps = norm_eps;
  rp.q_out = (bf16*)q_out; rp.k_cache = (bf16*)k_cache; rp.v_cache = (bf16*)v_cache;
  rp.heads = heads; rp.kv_heads = kv_heads; rp.head_dim = head_dim;
  return launch_rope(L, M, rp);
}

static int check_kv_scales(const char* what, float k_scale, float v_scale) {
  if (!(std::isfinite(k_scale) && k_scale > 0.f && std::isfinite(v_scale) && v_scale > 0.f))
    return fail("%s: scales k=%g v=%g (finite and > 0 required)", what, k_scale, v_scale);
  return 0;
}

int ssdk_rope_store_kv_fp8(const void* qkv, const int64_t* positions, const int32_t* slot_mapping, const float* rope_table,
                           const void* q_norm_w, const void* k_norm_w, float norm_eps, void* q_out, void* k_cache,
                           void* v_cache, int M, int heads, int kv_heads, int head_dim, float k_scale, float v_scale,
                           void* stream) {
  CKI(check_kv_scales("rope_store_kv_fp8", k_scale, v_scale));
  Launcher L;
  L.st = (cudaStream_t)stream;
  RopeParams rp;
  rp.qkv.dense = (const bf16*)qkv; rp.qkv.partial = nullptr; rp.qkv.S = 0; rp.qkv.M = M;
  rp.qkv.N = (heads + 2 * kv_heads) * head_dim;
  rp.positions = positions; rp.slot_mapping = slot_mapping; rp.rope_table = rope_table;
  rp.q_norm_w = (const bf16*)q_norm_w; rp.k_norm_w = (const bf16*)k_norm_w; rp.norm_eps = norm_eps;
  rp.q_out = (bf16*)q_out; rp.k_cache = (bf16*)k_cache; rp.v_cache = (bf16*)v_cache;
  rp.heads = heads; rp.kv_heads = kv_heads; rp.head_dim = head_dim;
  rp.k_scale = k_scale; rp.v_scale = v_scale;
  return launch_rope(L, M, rp, true);
}

int ssdk_silu_mul(const void* gate_up, void* out, int M, int ffn, void* stream) {
  if (ffn % 8) return fail("silu_mul: ffn %% 8 != 0");
  Launcher L;
  L.st = (cudaStream_t)stream;
  GemmOut g;
  g.dense = (const bf16*)gate_up; g.partial = nullptr; g.S = 0; g.M = M; g.N = 2 * ffn;
  return L.go(silu_mul_kernel, dim3((M * ffn / 8 + 255) / 256), dim3(256), 0, g, (bf16*)out, M, ffn);
}

int ssdk_paged_attn_plan(int heads, int kv_heads, int batch, int q_len, int max_ctx, int* out4) {
  if (batch < 1 || q_len < 1 || kv_heads < 1 || out4 == nullptr) return fail("paged_attn_plan: bad arguments");
  return attn_plan_raw(heads, kv_heads, batch, q_len, max_ctx, &out4[0], &out4[1], &out4[2], &out4[3]);
}

int64_t ssdk_paged_attn_scratch_bytes(int batch, int q_len, int heads, int head_dim, int max_ctx) {
  (void)max_ctx;
  return (int64_t)batch * q_len * heads * kAttnMaxSplit * (head_dim + 1) * 4 + 1024 + 16384;
}

static int paged_attn_op(const void* q, const void* k_cache, const void* v_cache, const int32_t* block_tables,
                         const int32_t* context_lens, void* out, void* scratch, int batch, int q_len, int heads,
                         int kv_heads, int head_dim, int block_size, int max_blocks_per_seq, float scale, void* stream,
                         KvDtype kvd) {
  if (batch * q_len > kMaxTokens) return fail("paged_attn: too many query tokens");
  Launcher L;
  L.st = (cudaStream_t)stream;
  CKI(init_kernel_attrs());
  int TQ, MT, nqt, nsplit;
  CKI(attn_plan_raw(heads, kv_heads, batch, q_len, block_size * max_blocks_per_seq, &TQ, &MT, &nqt, &nsplit));
  // the first 16 KB of the scratch hold the arrival counters (zero on entry)
  CK(cudaMemsetAsync(scratch, 0, 16384, L.st));
  float* part_o = (float*)((uint8_t*)scratch + 16384);
  float* part_lse = part_o + (size_t)batch * q_len * heads * kAttnMaxSplit * head_dim;
  return enqueue_attention(L, (const bf16*)q, (const bf16*)k_cache, (const bf16*)v_cache, block_tables, context_lens,
                           (bf16*)out, part_o, part_lse, (unsigned*)scratch, batch, q_len, heads, kv_heads, head_dim, block_size,
                           max_blocks_per_seq, scale, TQ, MT, nqt, nsplit, nullptr, kvd);
}

int ssdk_paged_attn(const void* q, const void* k_cache, const void* v_cache, const int32_t* block_tables,
                    const int32_t* context_lens, void* out, void* scratch, int batch, int q_len, int heads, int kv_heads,
                    int head_dim, int block_size, int max_blocks_per_seq, float scale, void* stream) {
  return paged_attn_op(q, k_cache, v_cache, block_tables, context_lens, out, scratch, batch, q_len, heads, kv_heads,
                       head_dim, block_size, max_blocks_per_seq, scale, stream, KvDtype{});
}

int ssdk_paged_attn_fp8(const void* q, const void* k_cache, const void* v_cache, const int32_t* block_tables,
                        const int32_t* context_lens, void* out, void* scratch, int batch, int q_len, int heads,
                        int kv_heads, int head_dim, int block_size, int max_blocks_per_seq, float scale, float k_scale,
                        float v_scale, void* stream) {
  CKI(check_kv_scales("paged_attn_fp8", k_scale, v_scale));
  KvDtype kvd;
  kvd.kv8 = true; kvd.k_scale = k_scale; kvd.v_scale = v_scale;
  return paged_attn_op(q, k_cache, v_cache, block_tables, context_lens, out, scratch, batch, q_len, heads, kv_heads,
                       head_dim, block_size, max_blocks_per_seq, scale, stream, kvd);
}

int ssdk_paged_attn_varlen_plan(int heads, int kv_heads, int batch, const int32_t* q_lens, int max_ctx, int* out5) {
  if (batch < 1 || batch > kMaxTokens || !q_lens || kv_heads < 1 || out5 == nullptr)
    return fail("paged_attn_varlen_plan: bad arguments");
  int total = 0;
  for (int b = 0; b < batch; ++b) {
    if (q_lens[b] < 1) return fail("paged_attn_varlen_plan: q_lens[%d]=%d < 1", b, q_lens[b]);
    total += q_lens[b];
  }
  if (total > kMaxTokens) return fail("paged_attn_varlen_plan: %d query tokens (max %d)", total, kMaxTokens);
  AttnPlan pl;
  const int rc = attn_make_plan_varlen(heads, kv_heads, batch, q_lens, max_ctx, num_sms(), &pl, &out5[4]);
  if (rc == 1) return fail("unsupported GQA ratio %d/%d", heads, kv_heads);
  if (rc != 0) return fail("attention tile too large");
  out5[0] = pl.TQ; out5[1] = pl.MT; out5[2] = pl.n_qtiles; out5[3] = pl.n_split;
  return 0;
}

static int paged_attn_varlen_op(const void* q, const void* k_cache, const void* v_cache, const int32_t* block_tables,
                                const int32_t* context_lens, const int32_t* q_lens, void* out, void* scratch, int batch,
                                int heads, int kv_heads, int head_dim, int block_size, int max_blocks_per_seq,
                                float scale, void* stream, KvDtype kvd) {
  int plan[5];
  CKI(ssdk_paged_attn_varlen_plan(heads, kv_heads, batch, q_lens, block_size * max_blocks_per_seq, plan));
  Launcher L;
  L.st = (cudaStream_t)stream;
  CKI(init_kernel_attrs());
  // the first 16 KB of the scratch hold the prefix sums (at 0) and the tile table (at 8 KB)
  int32_t cu_q[kMaxTokens + 1];
  AttnTile tiles[kMaxTokens];
  VarlenFwd var;
  var.plan.TQ = plan[0]; var.plan.MT = plan[1]; var.plan.n_qtiles = plan[2]; var.plan.n_split = plan[3];
  var.n_tiles = attn_varlen_tiles(batch, q_lens, plan[0], tiles, cu_q);
  var.M = cu_q[batch];
  var.attn.cu_q = (const int32_t*)scratch;
  var.attn.tiles = (const AttnTile*)((uint8_t*)scratch + 8192);
  CK(cudaMemcpyAsync(scratch, cu_q, (size_t)(batch + 1) * 4, cudaMemcpyHostToDevice, L.st));
  CK(cudaMemcpyAsync((uint8_t*)scratch + 8192, tiles, (size_t)var.n_tiles * sizeof(AttnTile), cudaMemcpyHostToDevice, L.st));
  L.barrier_op();
  float* part_o = (float*)((uint8_t*)scratch + 16384);
  float* part_lse = part_o + (size_t)var.M * heads * kAttnMaxSplit * head_dim;
  return enqueue_attention(L, (const bf16*)q, (const bf16*)k_cache, (const bf16*)v_cache, block_tables, context_lens,
                           (bf16*)out, part_o, part_lse, nullptr, batch, 0, heads, kv_heads, head_dim, block_size,
                           max_blocks_per_seq, scale, var.plan.TQ, var.plan.MT, var.plan.n_qtiles, var.plan.n_split, &var,
                           kvd);
}

int ssdk_paged_attn_varlen(const void* q, const void* k_cache, const void* v_cache, const int32_t* block_tables,
                           const int32_t* context_lens, const int32_t* q_lens, void* out, void* scratch, int batch,
                           int heads, int kv_heads, int head_dim, int block_size, int max_blocks_per_seq, float scale,
                           void* stream) {
  return paged_attn_varlen_op(q, k_cache, v_cache, block_tables, context_lens, q_lens, out, scratch, batch, heads,
                              kv_heads, head_dim, block_size, max_blocks_per_seq, scale, stream, KvDtype{});
}

int ssdk_paged_attn_varlen_fp8(const void* q, const void* k_cache, const void* v_cache, const int32_t* block_tables,
                               const int32_t* context_lens, const int32_t* q_lens, void* out, void* scratch, int batch,
                               int heads, int kv_heads, int head_dim, int block_size, int max_blocks_per_seq,
                               float scale, float k_scale, float v_scale, void* stream) {
  CKI(check_kv_scales("paged_attn_varlen_fp8", k_scale, v_scale));
  KvDtype kvd;
  kvd.kv8 = true; kvd.k_scale = k_scale; kvd.v_scale = v_scale;
  return paged_attn_varlen_op(q, k_cache, v_cache, block_tables, context_lens, q_lens, out, scratch, batch, heads,
                              kv_heads, head_dim, block_size, max_blocks_per_seq, scale, stream, kvd);
}

int ssdk_sample(const void* logits, int64_t ld, const float* temps, int B, int V, uint64_t seed, uint64_t step_id,
                int64_t* out_tokens, void* stream) {
  if (B < 1 || B > kMaxTokens) return fail("sample: B out of range");
  Launcher L;
  L.st = (cudaStream_t)stream;
  void* scr = nullptr;
  CKI(op_scratch(&scr, L.st));
  SampleParams sp;
  sp.logits = (const bf16*)logits; sp.ld = ld; sp.temps = temps; sp.V = V; sp.seed = seed; sp.call_id = step_id;
  sp.out = out_tokens; sp.out_stride = 1;
  sp.counters = (unsigned*)scr;
  sp.partial = (ArgMax*)((uint8_t*)scr + 4096);
  sp.dyn = nullptr; sp.sub = 0;
  return L.go(sample_kernel, dim3(kSampleChunks, B), dim3(256), 0, sp);
}

int64_t ssdk_verify_scratch_bytes(int B, int K) {
  return (int64_t)B * (2 * K + 1) * kVerifyCtas * sizeof(RowPart) + (int64_t)B * kVerifyCtas * sizeof(RecPart) + 1024;
}

int ssdk_verify(const void* logits_p, const void* logits_q, const int64_t* speculations, const float* temps_t,
                const float* temps_q, const int32_t* cache_hits, int jit_speculate, int B, int K, int V, uint64_t seed,
                uint64_t step_id, int32_t* n_accept, int64_t* recovery, void* scratch, void* stream) {
  if (B < 1 || B > kVerifyMaxBatch || K < 1 || B * (2 * K + 1) > kVerifyMaxRows) return fail("verify: B=%d K=%d out of range", B, K);
  Launcher L;
  L.st = (cudaStream_t)stream;
  // counters live in the first 1 KB of the scratch and must be zero on entry
  CK(cudaMemsetAsync(scratch, 0, 1024, L.st));
  VerifyParams vp;
  vp.lp = (const bf16*)logits_p; vp.lq = (const bf16*)logits_q; vp.spec = speculations;
  vp.temps_t = temps_t; vp.temps_q = temps_q; vp.cache_hits = cache_hits; vp.jit = jit_speculate;
  vp.B = B; vp.K = K; vp.V = V; vp.seed = seed; vp.call_id = step_id;
  vp.n_accept = n_accept; vp.recovery = recovery;
  vp.counters = (unsigned*)scratch;
  vp.row_part = (RowPart*)((uint8_t*)scratch + 1024);
  vp.rec_part = (RecPart*)((uint8_t*)scratch + 1024 + (size_t)B * (2 * K + 1) * kVerifyCtas * sizeof(RowPart));
  vp.dyn = nullptr; vp.sub = 0;
  return L.go(verify_kernel, dim3(kVerifyCtas), dim3(kVerifyThreads), 0, vp);
}

}  // extern "C"
