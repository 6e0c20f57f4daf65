/*
 * ssdk.h — C-ABI of libssdk.so, the sm_90a (H100) speculative-decoding hot path.
 *
 * The reference (tanishqkumar/ssd) has no native code and no FFI: its hot path is
 * Python/torch calling cuBLAS, torch.compile(Triton), FlashAttention-3, FlashInfer
 * and NCCL.  Every entry point below therefore replaces a *Python* interface of the
 * reference; the file:line each one replaces is cited on the declaration
 * (paths relative to the reference root).  INTEGRATION.md shows the ctypes stub a
 * reference maintainer would add to bind them.
 *
 * Conventions
 *  - plain C types only: raw device/host pointers, sizes, `void* stream`
 *    (a cudaStream_t); no torch types.
 *  - every function returns 0 on success, <0 on error; ssdk_last_error() returns a
 *    thread-local, NUL-terminated description of the last failure.
 *  - the caller (PyTorch on the host side) owns all device memory: weights,
 *    KV cache, workspace, logits.  The library owns only its plan objects, CUDA
 *    graphs, TMA descriptors and a few KB of pinned staging for step I/O.
 *  - not thread-safe per handle; one handle per rank process; all work is enqueued
 *    on the caller's stream.
 *  - bf16 storage everywhere unless stated; fp32 accumulation and statistics.
 */
#ifndef SSDK_H_
#define SSDK_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SSDK_ABI_VERSION 1

typedef struct ssdk_engine* ssdk_handle;

/* which model of the pair an argument refers to */
enum { SSDK_TARGET = 0, SSDK_DRAFT = 1 };

/* weight kinds for ssdk_bind_weight (shapes are per tensor-parallel rank) */
enum {
  SSDK_W_EMBED      = 0,  /* [vocab/tp, hidden]            layers/embed_head.py:33-47 */
  SSDK_W_LM_HEAD    = 1,  /* [vocab/tp, hidden]            layers/embed_head.py:78-116 */
  SSDK_W_FINAL_NORM = 2,  /* [hidden]                      models/llama3.py:246,266 */
  SSDK_W_INPUT_NORM = 3,  /* [hidden]           per layer  models/llama3.py:182 */
  SSDK_W_QKV        = 4,  /* [(H+2KV)*hd/tp, hidden]       layers/linear.py:125-162 (q|k|v packed) */
  SSDK_W_Q_NORM     = 5,  /* [hd]  (Qwen3 only)            models/qwen3.py:87-88 */
  SSDK_W_K_NORM     = 6,  /* [hd]  (Qwen3 only) */
  SSDK_W_O          = 7,  /* [hidden, H*hd/tp]             layers/linear.py:165-199 */
  SSDK_W_POST_NORM  = 8,  /* [hidden]                      models/llama3.py:183 */
  SSDK_W_GATE_UP    = 9,  /* [2*ffn/tp, hidden] gate|up    layers/linear.py:101-122 */
  SSDK_W_DOWN       = 10, /* [hidden, ffn/tp]              layers/linear.py:165-199 */
  SSDK_W_ROPE_TABLE = 11, /* fp32 [max_pos, hd] cos|sin    layers/rotary_embedding.py:30-37 */
  SSDK_W_KIND_COUNT = 12
};

/* Mirrors the HF config fields the reference reads (models/llama3.py:157-183,
 * models/qwen3.py:163-193) after tensor-parallel division. */
typedef struct ssdk_model_cfg {
  int32_t hidden;        /* d */
  int32_t layers;        /* L */
  int32_t heads;         /* total query heads H */
  int32_t kv_heads;      /* total KV heads */
  int32_t head_dim;      /* hd */
  int32_t ffn;           /* total intermediate size */
  int32_t vocab;         /* total vocab V */
  int32_t qk_norm;       /* 1 = per-head RMSNorm on q,k before RoPE (Qwen3) */
  float   rms_eps;
  int32_t max_pos;       /* rows in the RoPE table that will be bound */
  int32_t tp_size;       /* 1 for the draft (replica on one GPU) */
  int32_t tp_rank;
} ssdk_model_cfg;

typedef struct ssdk_runtime_cfg {
  int32_t spec_k;             /* K (speculate_k); 0 = autoregressive only */
  int32_t max_batch;          /* max sequences per step (b); max_batch*(K+1) <= 256, max_batch <= 32 */
  int32_t block_size;         /* KV page size (kvcache_block_size, 256 in bench.py:40) */
  int32_t max_blocks_per_seq; /* ceil(max_model_len / block_size) */
  int32_t use_graph;          /* 1 = capture the spec step into one CUDA graph */
  int32_t use_pdl;            /* 1 = programmatic dependent launch between kernels */
  int32_t jit_speculate;      /* verify(): ratio acceptance on every temp>0 row (utils/verify.py:59-62) */
  int32_t draft_fp8;          /* 0 = bf16 draft; 1 = the draft's decoder linears are FP8 (ssdk_bind_weight_fp8),
                                 all of them: ssdk_finalize refuses a draft that is bf16 or only partly FP8 */
} ssdk_runtime_cfg;

/* ---- lifetime ------------------------------------------------------------- */
int  ssdk_abi_version(void);
const char* ssdk_last_error(void);

/* Replaces ModelRunner.__init__ / setup_and_warmup_model_and_cudagraphs
 * (engine/model_runner.py:39-157, 186-260) for both models of the pair.
 * `draft` may be NULL (autoregressive engine). */
int ssdk_create(const ssdk_model_cfg* target, const ssdk_model_cfg* draft,
                const ssdk_runtime_cfg* rt, ssdk_handle* out);
int ssdk_destroy(ssdk_handle h);

/* Replaces utils/loader.py:186-218 + the per-parameter weight_loader callbacks:
 * the host side shards/packs exactly as the reference does and hands over the
 * resulting device tensor.  `layer` is ignored for non-per-layer kinds. */
int ssdk_bind_weight(ssdk_handle h, int which, int kind, int layer,
                     const void* dev_ptr, int64_t rows, int64_t cols);

/* FP8 weight-only (W8A16) form of a decoder linear.  The reference has
 * no FP8 path.  kind: SSDK_W_QKV, SSDK_W_O, SSDK_W_GATE_UP or SSDK_W_DOWN;
 * which: SSDK_TARGET, or SSDK_DRAFT when the runtime config sets draft_fp8 = 1
 * (then every decoder linear of the draft must be FP8).  Layout, no packing step:
 *   w_e4m3    float8 e4m3fn [rows, cols] row-major, same shape and row order as
 *             the bf16 matrix of that kind (q|k|v and gate|up packed), 16-byte aligned;
 *   row_scale fp32 [rows]: row n of the matrix is row_scale[n] * W8[n, :].
 * cols (K) must be a multiple of 128.  Both buffers stay owned by the caller
 * and must outlive the handle.  The GEMM computes
 *   y[m, n] = bf16( s[n] * sum_k bf16(W8[n, k]) * x[m, k] )   (fp32 accumulate). */
int ssdk_bind_weight_fp8(ssdk_handle h, int which, int kind, int layer,
                         const void* w_e4m3, const float* row_scale,
                         int64_t rows, int64_t cols);

/* Replaces ModelRunner.allocate_kv_cache (engine/model_runner.py:446-503):
 * one tensor [2, L, num_blocks, block_size, kv_heads/tp, hd] (bf16);
 * k = base, v = base + L*num_blocks*block_size*kv_heads/tp*hd elements. */
int ssdk_bind_kv_cache(ssdk_handle h, int which, void* kv_base, int64_t num_blocks);

/* FP8 KV cache, called instead of ssdk_bind_kv_cache and before ssdk_finalize;
 * the reference has no FP8 KV path.  which: SSDK_TARGET only (the draft's cache
 * stays bf16).  Same [2, L, num_blocks, block_size, kv_heads/tp, hd] layout with
 * float8 e4m3fn elements (one byte each), 16-byte aligned; head_dim 64 or 128.
 * k_scale, v_scale: host fp32 arrays [L], finite and > 0, copied into the handle.
 * Layer l stores code = e4m3_rne(sat448(y / s)) of the bf16 value y the bf16
 * cache would hold, and attention reads K = k_scale[l] * code, V = v_scale[l] * code. */
int ssdk_bind_kv_cache_fp8(ssdk_handle h, int which, void* kv_base, int64_t num_blocks,
                           const float* k_scale, const float* v_scale);

/* Scratch owned by the caller (activations, split-K partials, attention partials,
 * logits_q/logits_p, token buffers). */
int64_t ssdk_workspace_bytes(ssdk_handle h);
int ssdk_bind_workspace(ssdk_handle h, void* dev_ptr, int64_t bytes);

/* Optional tensor-parallel plumbing (target only): a ncclComm_t created by the
 * host side over the TP ranks (replaces dist.new_group, engine/model_runner.py:100-107),
 * and the per-rank peer pointers of a symmetric buffer for the fused
 * GEMM + one-shot all-reduce (replaces dist.all_reduce, layers/linear.py:195-199). */
int ssdk_set_nccl_comm(ssdk_handle h, void* nccl_comm);
int64_t ssdk_symm_bytes(ssdk_handle h);
int ssdk_bind_symm(ssdk_handle h, void* const* peer_ptrs, int n_peers);

/* Finalise: builds TMA descriptors for every bound weight and (if use_graph)
 * captures the step graphs (replaces capture_cudagraph / capture_verify_cudagraph,
 * engine/helpers/cudagraph_helpers.py:440-633). */
int ssdk_finalize(ssdk_handle h, void* stream);

/* ---- the hot path ---------------------------------------------------------- */

/* One synchronous speculative-decoding step for `batch` sequences:
 *   K draft forwards (speculator_sync.py:25-69) -> one (K+1)-token target
 *   forward (verifier.py:54-106) -> accept/reject + recovery (utils/verify.py:5-181),
 * enqueued as ONE call with no host control flow per token.
 * The reference's K+1-th draft forward only writes the draft KV of the last draft token d_K.  It is not run here: when a
 * step accepts all K drafts (out_n_accept[b] == K), d_K's draft KV (position ctx_len + K) is NOT written.  Pass d_K as
 * pending[b] to the sequence's next step, whose first draft forward writes it; otherwise write it with a one-token
 * draft forward (ssdk_forward_tokens, want_sample = 0) before anything else uses the draft cache.
 *  in : ctx_len[b]      tokens already in both KV caches (= seq.num_cached_tokens,
 *                       engine/step.py:101) — the recovery token sits at this position
 *       recovery[b]     seq.recovery_token_id (speculator_sync.py:38-45)
 *       pending[b]      the token at ctx_len-1 when its draft KV is still to be written, else -1 (NULL: none)
 *       block_tables_*  [batch, max_blocks_per_seq] int32, -1 padded
 *                       (helpers/runner_helpers.py:110-121), covering ctx_len+K+1 slots
 *       temp_t/temp_q   per-sequence temperatures (verifier.py:83-90)
 *       seed, step_id   Philox key / counter for temp>0 (replaces torch's global RNG)
 *  out: out_tokens[b*(K+1) + j]  = [recovery, draft_1..draft_K]   (speculations)
 *       out_n_accept[b]          = number of accepted draft tokens (0..K)
 *       out_recovery[b]          = next recovery token
 * Host pointers; the call blocks until the results are on the host. */
int ssdk_spec_step(ssdk_handle h, int batch,
                   const int32_t* ctx_len, const int64_t* recovery, const int64_t* pending,
                   const int32_t* block_tables_target, const int32_t* block_tables_draft,
                   const float* temp_t, const float* temp_q,
                   uint64_t seed, uint64_t step_id,
                   int64_t* out_tokens, int32_t* out_n_accept, int64_t* out_recovery,
                   void* stream);

/* Device-resident variant for measurement: same work, inputs already staged on the
 * device by a previous ssdk_spec_step_stage(); nothing crosses PCIe.  The device carries
 * the pending token from step to step; the last step's d_K draft KV stays unwritten. */
int ssdk_spec_step_stage(ssdk_handle h, int batch,
                         const int32_t* ctx_len, const int64_t* recovery, const int64_t* pending,
                         const int32_t* block_tables_target, const int32_t* block_tables_draft,
                         const float* temp_t, const float* temp_q,
                         uint64_t seed, uint64_t step_id, void* stream);
int ssdk_spec_step_resident(ssdk_handle h, int batch, void* stream);
int ssdk_spec_step_fetch(ssdk_handle h, int batch, int64_t* out_tokens,
                         int32_t* out_n_accept, int64_t* out_recovery, void* stream);
/* Resident mode: copy the tokens sequence `seq` has emitted since ssdk_spec_step_stage (each step's recovery token +
 * accepted draft tokens, i.e. what Scheduler.postprocess_speculate appends, engine/scheduler.py:285-327) into
 * out_tokens[0 .. cap).  Returns the number of tokens copied (>= 0) or < 0 on error.  The device keeps at most
 * 16384 tokens per sequence. */
int ssdk_spec_step_log(ssdk_handle h, int seq, int64_t* out_tokens, int cap, void* stream);

/* Generic multi-token forward + sample of the last position of every sequence.
 * Replaces ModelRunner.run for prefill chunks (batch*q_len<=256 per call, causal over the
 * paged cache; engine/model_runner.py:634-680 with is_prefill) and for
 * single-token autoregressive decode (q_len=1; engine/step.py:36-47).
 *   ids[b*q_len + j] tokens, written to positions ctx_len[b]+j.
 *   want_sample: 1 = run lm_head on the last row of each sequence and sample with
 *   temps[b] (layers/sampler.py:14-36) into out_tokens[b].
 * Blocks until out_tokens is on the host when want_sample != 0. */
int ssdk_forward_tokens(ssdk_handle h, int which, int batch, int q_len,
                        const int64_t* ids, const int32_t* ctx_len,
                        const int32_t* block_tables, int want_sample,
                        const float* temps, uint64_t seed, uint64_t step_id,
                        int64_t* out_tokens, void* stream);

/* ssdk_forward_tokens for sequences of different lengths in one call (the reference's
 * cu_seqlens prefill, engine/helpers/runner_helpers.py:123-180): q_lens[b] tokens of
 * sequence b, packed in sequence order in ids (sum of q_lens long), written to positions
 * ctx_len[b] .. ctx_len[b]+q_lens[b]-1; ctx_len[b] tokens are already in the cache.
 * 1 <= n_seqs <= max_batch, every q_lens[b] >= 1, sum <= 256.  want_sample: lm_head on the
 * last row of every sequence, sampled into out_tokens[b]; ssdk_logits_last then holds
 * [n_seqs, V].  Blocks until out_tokens is on the host when want_sample != 0. */
int ssdk_forward_varlen(ssdk_handle h, int which, int n_seqs, const int32_t* q_lens,
                        const int64_t* ids, const int32_t* ctx_len,
                        const int32_t* block_tables, int want_sample,
                        const float* temps, uint64_t seed, uint64_t step_id,
                        int64_t* out_tokens, void* stream);

/* Debug/parity taps: device pointers to the logits of the last spec step
 * (bf16 [batch, K+1, V] and [batch, K, V]) and of the last ssdk_forward_tokens
 * or ssdk_forward_varlen (bf16 [batch, V]).  Valid until the next call. */
const void* ssdk_logits_p(ssdk_handle h);
const void* ssdk_logits_q(ssdk_handle h);
const void* ssdk_logits_last(ssdk_handle h);
/* Debug timeline: CTA 0 of every kernel appends (kernel id, %globaltimer ns) to dev_buf (uint64 [cap][2]) right
 * after its grid dependency resolves; replaces the reference's SSD_PROFILE perf_counter prints (engine/step.py:92-161).
 * dev_buf = NULL turns tracing off. */
int ssdk_debug_trace(void* dev_buf, int cap);
/* number of kernels this library launched (or replayed inside graphs) so far */
int64_t ssdk_launch_count(ssdk_handle h);

/* ---- stand-alone ops (parity tests call these through the same C-ABI) ------ */

/* y[M,N] = x[M,K] · w[N,K]^T  (bf16 in, fp32 accumulate in registers, bf16 out),
 * M <= 64: weight-streaming wgmma GEMM with TMA-fed 128B-swizzled smem tiles.
 * Replaces F.linear at layers/linear.py:98,196 and embed_head.py:95,111.
 * split_k = 0 lets the library choose; `partials` (fp32 [split_k, M, N]) is only
 * needed when split_k != 1.  When split_k > 1 the result is left in `partials`
 * AND reduced+rounded into y. */
int ssdk_gemm_small_m(const void* x, const void* w, void* y, float* partials,
                      int M, int N, int K, int ldy, int split_k, void* stream);

/* h[M,ffn] = silu(x·Wg^T) * (x·Wu^T) with gate|up packed [2*ffn, K]
 * (layers/linear.py:101-122 + layers/activation.py:11-14), fused epilogue. */
int ssdk_gemm_gate_up_silu(const void* x, const void* w_gate_up, void* h,
                           int M, int ffn, int K, void* stream);

/* FP8-weight (e4m3 + fp32 per-row scale, layout of ssdk_bind_weight_fp8)
 * versions of the two GEMMs above; the reference has no FP8 path.  M <= 256,
 * K a multiple of 128.  The scale multiplies the fp32 accumulator before any
 * rounding; split-K partials are stored scaled.  gate_up_silu_fp8: split_k <= 1
 * runs one split; split_k > 1 (M <= 64) reduces inside the kernel and needs
 * fp32 partials [split_k, M, 2*ffn] and ceil(ffn/64) zeroed uint32 counters
 * (left zeroed on return). */
int ssdk_gemm_small_m_fp8(const void* x, const void* w8, const float* scale,
                          void* y, float* partials, int M, int N, int K,
                          int ldy, int split_k, void* stream);
int ssdk_gemm_gate_up_silu_fp8(const void* x, const void* w8_gate_up,
                               const float* scale, void* h, float* partials,
                               unsigned* counters, int M, int ffn, int K,
                               int split_k, void* stream);

/* RMSDNorm (layers/layernorm.py:53-98), compiled single-rounding semantics:
 * r = x (+ residual); residual_out = bf16(r); y = bf16(r * rsqrt(mean r^2 + eps) * w).
 * residual_in may be NULL (first layer: y = norm(x), residual_out = x). */
int ssdk_rmsnorm(const void* x, const void* residual_in, const void* w, float eps,
                 void* y, void* residual_out, int M, int d, void* stream);

/* Optional per-head RMSNorm (RMSHeadNorm, layers/layernorm.py:5-50) + NeoX RoPE
 * (layers/rotary_embedding.py:6-60) on q,k, then KV-cache scatter
 * (store_kvcache, layers/attention.py:10-41).  qkv [M, (H+2KV)*hd] packed;
 * positions int64 [M]; slot_mapping int32 [M] (-1 = skip);
 * q_out [M, H*hd]; caches viewed as [num_slots, KV*hd]. */
int ssdk_rope_store_kv(const void* qkv, const int64_t* positions, const int32_t* slot_mapping,
                       const float* rope_table, const void* q_norm_w, const void* k_norm_w,
                       float norm_eps, void* q_out, void* k_cache, void* v_cache,
                       int M, int heads, int kv_heads, int head_dim, void* stream);
/* ssdk_rope_store_kv into e4m3 caches (layout of ssdk_bind_kv_cache_fp8, one byte
 * per element; head_dim 64 or 128): k and v are stored as
 * e4m3_rne(sat448(y / scale)) of the bf16 values y the bf16 op stores; q_out as
 * in the bf16 op.  The reference has no FP8 KV path. */
int ssdk_rope_store_kv_fp8(const void* qkv, const int64_t* positions, const int32_t* slot_mapping,
                           const float* rope_table, const void* q_norm_w, const void* k_norm_w,
                           float norm_eps, void* q_out, void* k_cache, void* v_cache,
                           int M, int heads, int kv_heads, int head_dim,
                           float k_scale, float v_scale, void* stream);

/* silu(x[:, :ffn]) * x[:, ffn:]  (layers/activation.py:11-14). */
int ssdk_silu_mul(const void* gate_up, void* out, int M, int ffn, void* stream);

/* Paged attention for decode (q_len=1) and verify/prefill-chunk (q_len>1):
 * replaces flash_attn_with_kvcache at layers/attention.py:107-111,128-131.
 * q [batch*q_len, H, hd]; caches [num_blocks, block_size, KV, hd];
 * context_lens[b] INCLUDES the q_len new tokens; causal, bottom-right aligned.
 * `scratch` fp32, at least ssdk_paged_attn_scratch_bytes(...) bytes. */
int64_t ssdk_paged_attn_scratch_bytes(int batch, int q_len, int heads, int head_dim, int max_ctx);
int ssdk_paged_attn(const void* q, const void* k_cache, const void* v_cache,
                    const int32_t* block_tables, const int32_t* context_lens,
                    void* out, void* scratch,
                    int batch, int q_len, int heads, int kv_heads, int head_dim,
                    int block_size, int max_blocks_per_seq, float scale, void* stream);
/* The launch plan ssdk_paged_attn picks for these sizes on the current device (max_ctx = block_size *
 * max_blocks_per_seq): out4 = {TQ query tokens per tile, MT 16-row MMA tiles per tile, n_qtiles, n_split KV splits}.
 * Launches nothing. */
int ssdk_paged_attn_plan(int heads, int kv_heads, int batch, int q_len, int max_ctx, int* out4);
/* ssdk_paged_attn for `batch` sequences of their own q_lens[b] (host array), packed in sequence
 * order: q [sum q_lens, H, hd] -> out [sum q_lens, H*hd]; context_lens[b] includes the q_lens[b]
 * new tokens.  Query tiles never cross a sequence.  `scratch`: at least
 * ssdk_paged_attn_scratch_bytes(1, sum q_lens, heads, head_dim, max_ctx) bytes. */
int ssdk_paged_attn_varlen(const void* q, const void* k_cache, const void* v_cache,
                           const int32_t* block_tables, const int32_t* context_lens,
                           const int32_t* q_lens, void* out, void* scratch,
                           int batch, int heads, int kv_heads, int head_dim,
                           int block_size, int max_blocks_per_seq, float scale, void* stream);
/* Its plan: out5 = {TQ, MT, n_qtiles of the longest sequence, n_split, tiles in the launch}.
 * With every q_lens[b] equal the first four are ssdk_paged_attn_plan's. */
int ssdk_paged_attn_varlen_plan(int heads, int kv_heads, int batch, const int32_t* q_lens, int max_ctx, int* out5);
/* ssdk_paged_attn and ssdk_paged_attn_varlen over e4m3 caches (layout of
 * ssdk_bind_kv_cache_fp8): attention over K = k_scale * code, V = v_scale * code,
 * q and out bf16, the same plans and scratch sizes as the bf16 ops.  The
 * reference has no FP8 KV path. */
int ssdk_paged_attn_fp8(const void* q, const void* k_cache, const void* v_cache,
                        const int32_t* block_tables, const int32_t* context_lens,
                        void* out, void* scratch,
                        int batch, int q_len, int heads, int kv_heads, int head_dim,
                        int block_size, int max_blocks_per_seq, float scale,
                        float k_scale, float v_scale, void* stream);
int ssdk_paged_attn_varlen_fp8(const void* q, const void* k_cache, const void* v_cache,
                               const int32_t* block_tables, const int32_t* context_lens,
                               const int32_t* q_lens, void* out, void* scratch,
                               int batch, int heads, int kv_heads, int head_dim,
                               int block_size, int max_blocks_per_seq, float scale,
                               float k_scale, float v_scale, void* stream);

/* Sampler.forward (layers/sampler.py:14-36): greedy where temp==0, else
 * argmax(softmax(l/T) / Exp(1)) with Philox(seed, step_id) exponentials.
 * logits bf16 [B, V] with row stride ld (elements); out int64 [B]. */
int ssdk_sample(const void* logits, int64_t ld, const float* temps, int B, int V,
                uint64_t seed, uint64_t step_id, int64_t* out_tokens, void* stream);

/* verify() (utils/verify.py:5-181), one fused kernel.
 * logits_p bf16 [B,K+1,V], logits_q bf16 [B,K,V], speculations int64 [B,K+1],
 * temps_* fp32 [B].  ratio_rows semantics follow jit_speculate / cache_hits
 * (cache_hits may be NULL).  Outputs on the device: n_accept int32 [B],
 * recovery int64 [B].  `scratch` >= ssdk_verify_scratch_bytes(B,K) bytes. */
int64_t ssdk_verify_scratch_bytes(int B, int K);
int ssdk_verify(const void* logits_p, const void* logits_q, const int64_t* speculations,
                const float* temps_t, const float* temps_q, const int32_t* cache_hits,
                int jit_speculate, int B, int K, int V, uint64_t seed, uint64_t step_id,
                int32_t* n_accept, int64_t* recovery, void* scratch, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SSDK_H_ */
