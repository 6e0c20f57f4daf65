// common.cuh — shared device helpers for the sm_90a kernels of libssdk.
// PTX wrappers (mbarrier, TMA, wgmma, PDL), bf16 helpers, reductions, Philox.
#pragma once
// SSDK_HOST_EMU: the kernels that use no TMA / wgmma / PTX-only feature can be compiled for the host by the test
// suite (tests/emu/cuda_emu.h supplies the CUDA vocabulary before this header is included); never defined in the product.
#ifndef SSDK_HOST_EMU
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#endif
#include <stdint.h>

#define SSDK_DEVINL __device__ __forceinline__

// shared-memory declarations inside a kernel body
#ifdef SSDK_HOST_EMU
#define SSDK_DYN_SMEM(T, name) T* name = reinterpret_cast<T*>(::emu::dyn_smem())
#define SSDK_STATIC_SMEM(T, name, n) T* name = ::emu::static_smem<T>(n, __LINE__)
#define SSDK_SHARED_VAR(T, name) T& name = *::emu::static_smem<T>(1, __LINE__)
#else
#define SSDK_DYN_SMEM(T, name) extern __shared__ __align__(16) T name[]
#define SSDK_STATIC_SMEM(T, name, n) __shared__ T name[n]
#define SSDK_SHARED_VAR(T, name) __shared__ T name
#endif

namespace ssdk {

// ----------------------------------------------------------------------------------
// bf16 helpers.  All "round to bf16" steps of the reference (every F.linear output,
// every norm/rope/silu output) are round-to-nearest-even, which __float2bfloat16_rn is.
// ----------------------------------------------------------------------------------
SSDK_DEVINL float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
SSDK_DEVINL float bf2f(__nv_bfloat16 x) { return __bfloat162float(x); }
SSDK_DEVINL __nv_bfloat16 f2bf(float x) { return __float2bfloat16_rn(x); }

SSDK_DEVINL void unpack_bf16x8(const uint4& v, float* f) {
  const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(p[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
SSDK_DEVINL uint4 pack_bf16x8(const float* f) {
  uint4 v;
  __nv_bfloat162* p = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) p[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return v;
}

// ----------------------------------------------------------------------------------
// warp / block reductions
// ----------------------------------------------------------------------------------
SSDK_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
SSDK_DEVINL float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// block-wide sum; `red` is >= 32 floats of shared memory; all threads get the result.
SSDK_DEVINL float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  float t = (lane < nw) ? red[lane] : 0.f;
  t = warp_sum(t);
  return t;
}

// (value, index) argmax with lowest-index tie-break == torch.argmax semantics
// (SURVEY §8a checklist 6).
struct ArgMax {
  float v;
  int i;
};
SSDK_DEVINL ArgMax argmax_better(ArgMax a, ArgMax b) {
  // NaN-free inputs assumed; larger value wins, ties -> lower index
  if (b.v > a.v || (b.v == a.v && b.i < a.i)) return b;
  return a;
}
SSDK_DEVINL ArgMax warp_argmax(ArgMax a) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ArgMax b;
    b.v = __shfl_xor_sync(0xffffffffu, a.v, o);
    b.i = __shfl_xor_sync(0xffffffffu, a.i, o);
    a = argmax_better(a, b);
  }
  return a;
}

// ----------------------------------------------------------------------------------
// Philox4x32-10 (counter-based RNG).  The reference draws from torch's global CUDA
// Philox stream (sampler.py:33, verify.py:115,158-159); a fused kernel cannot
// reproduce that stream, so the RNG is keyed explicitly: key = seed, counter =
// (element index, row, step_id, stream tag).  oracle/philox.py implements the same
// function bit-for-bit so temp>0 paths stay checkable token-for-token.
// ----------------------------------------------------------------------------------
SSDK_DEVINL uint4 philox4x32_10(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return ctr;
}
// uniform in (0,1]: (x + 1) * 2^-32 evaluated in fp32 the same way on host and device
SSDK_DEVINL float u32_to_unit_open0(uint32_t x) {
  // 24 high bits -> (k + 1) / 2^24, exactly representable; never 0, may be 1
  return (float)((x >> 8) + 1u) * (1.0f / 16777216.0f);
}
// Exp(1) sample from one 32-bit word
SSDK_DEVINL float u32_to_exp1(uint32_t x) { return -__logf(u32_to_unit_open0(x)); }

// epoch / slot parity of the one-shot all-reduce number call_idx of target forward number seq (n_calls all-reduces per
// forward).  The slot parity runs on ACROSS forwards: a forward has 2L+1 all-reduces — an odd number — so a per-forward
// parity would put the last all-reduce of forward n and the first one of forward n+1 into the same slot back to back, and
// a fast rank could overwrite words a slow peer is still polling (ADVICE r1).  With a continuous parity a slot is reused at
// distance 2 only, which the data dependence already protects (a rank needs every peer's words of all-reduce i+1 before
// it can publish i+2).
SSDK_DEVINL unsigned symm_epoch_of(unsigned seq, int call_idx) { return seq * 512u + (unsigned)call_idx + 1u; }
SSDK_DEVINL unsigned symm_parity_of(unsigned seq, int call_idx, int n_calls) {
  return (seq * (unsigned)n_calls + (unsigned)call_idx) & 1u;
}

#ifndef SSDK_HOST_EMU
// one 8-byte store (flag-in-word protocol: payload and flag must become visible together)
SSDK_DEVINL void st_global_v2_u32(void* p, uint32_t a, uint32_t b) {
  asm volatile("st.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(a), "r"(b) : "memory");
}
// ----------------------------------------------------------------------------------
// PTX: shared-address conversion, mbarrier, fences
// ----------------------------------------------------------------------------------
SSDK_DEVINL uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

SSDK_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
SSDK_DEVINL void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
SSDK_DEVINL void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
SSDK_DEVINL void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
SSDK_DEVINL void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
SSDK_DEVINL bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug turns into a trap (launch failure) instead of a hung GPU.
SSDK_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 8000000000LL) __trap();  // ~4 s at 2 GHz
  }
}

// ----------------------------------------------------------------------------------
// PTX: TMA (cp.async.bulk.tensor) 2D tile load, global -> shared, mbarrier completion
// ----------------------------------------------------------------------------------
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;

SSDK_DEVINL void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
SSDK_DEVINL void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "l"(policy)
      : "memory");
}

// non-tensor bulk copy global -> shared (contiguous bytes; 16-byte aligned addresses and size), mbarrier completion, weights
// tagged evict-first in L2; and its fire-and-forget sibling that only pulls the bytes into L2
SSDK_DEVINL void bulk_load_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
      ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(kEvictFirst)
      : "memory");
}

// ----------------------------------------------------------------------------------
// PTX: wgmma (Hopper warpgroup MMA), both operands from shared memory
// ----------------------------------------------------------------------------------
SSDK_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
SSDK_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
SSDK_DEVINL void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// Shared-memory matrix descriptor (sm_90 GMMA layout), K-major operand, 128-byte swizzle:
// 8-row x 128 B swizzle atoms stacked every 1024 B (SBO), LBO unused.
SSDK_DEVINL uint64_t make_wgmma_desc_k128(const void* smem_tile) {
  const uint32_t addr = smem_u32(smem_tile);
  uint64_t d = 0;
  d |= (uint64_t)((addr >> 4) & 0x3FFFu);  // start address, bits [0,14)
  d |= (uint64_t)1u << 16;                 // leading byte offset (ignored for SW128 K-major), bits [16,30)
  d |= (uint64_t)(1024u >> 4) << 32;       // stride byte offset = 1024 B, bits [32,46)
  d |= (uint64_t)1u << 62;                 // layout type SWIZZLE_128B, bits [62,64)
  return d;
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, A and B K-major bf16 in shared memory, D fp32 in registers of the
// warpgroup: thread t (warp w = t / 32 of the group, lane l) holds rows 16w + l/4 + {0, 8} and columns 8c + 2(l%4) + {0, 1}
// as d[4c + 2 * (row half) + column parity].  accumulate == 0 overwrites D.
template <int N>
SSDK_DEVINL void wgmma_bf16_ss(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate);
template <> SSDK_DEVINL void wgmma_bf16_ss<16>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}
template <> SSDK_DEVINL void wgmma_bf16_ss<32>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}
template <> SSDK_DEVINL void wgmma_bf16_ss<64>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, "
      "%19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}

// ----------------------------------------------------------------------------------
// PTX: programmatic dependent launch
// ----------------------------------------------------------------------------------
SSDK_DEVINL void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
SSDK_DEVINL void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ----------------------------------------------------------------------------------
// Timeline tracing (debug aid, off by default): CTA (0,0,0) of every kernel records
// (kernel id, %globaltimer) right after its grid dependency resolves.  Because each kernel's
// griddepcontrol.wait returns when its predecessor has fully completed, consecutive records are
// the real, PDL-overlapped, per-kernel increments of the critical path inside a graph replay —
// something ncu's serialised replay cannot show.  Enabled with ssdk_debug_trace().
// ----------------------------------------------------------------------------------
// The switch lives in constant memory: when tracing is off a kernel pays one uniform constant load, not a dependent
// global load on its first warp.
__constant__ unsigned long long* g_trace_buf = nullptr;  // [cap][2] = (id, time ns)
__constant__ unsigned g_trace_cap = 0;
__device__ unsigned g_trace_n = 0;
enum { TR_PREP = 1, TR_NORM, TR_GEMM, TR_ROPE, TR_ATTN, TR_SAMPLE, TR_VERIFY, TR_MISC };
SSDK_DEVINL void trace_mark(int id) {
  if (g_trace_buf == nullptr) return;
  if ((blockIdx.x | blockIdx.y | blockIdx.z) != 0) return;
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  const unsigned slot = atomicAdd(&g_trace_n, 1u);
  if (slot < g_trace_cap) {
    g_trace_buf[2 * slot] = (unsigned long long)id;
    g_trace_buf[2 * slot + 1] = t;
  }
}
// Phase marks inside a kernel (ids >= 16, tools/trace_step.py prints the mean gaps between them).  Each mark costs the
// marking thread an atomic round trip (~0.6 us), so they are compiled in only with -DSSDK_TRACE_FINE.
enum { TRF_ATTN = 16, TRF_NORM = 24, TRF_ROPE = 32, TRF_COMB = 40, TRF_GEMM = 48 };
SSDK_DEVINL void trace_fine(int id) {
#ifdef SSDK_TRACE_FINE
  trace_mark(id);
#else
  (void)id;
#endif
}

SSDK_DEVINL bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// streaming (read-once) 16-byte global load
SSDK_DEVINL uint4 ld_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
// the same with an L2 evict-first hint: a weight line that has been consumed is the first candidate for replacement, so
// lines prefetched for LATER phases (cp.async.bulk.prefetch.L2) survive in L2 until they are read
SSDK_DEVINL uint4 ld_nc_v4_evict_first(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p), "l"(kEvictFirst));
  return r;
}
// fetch-add with acquire-release semantics at device scope (tickets, device-wide barriers): orders this thread's earlier
// writes before the add and its later reads after it, without a separate fence
SSDK_DEVINL unsigned atom_add_acq_rel_gpu(unsigned* p, unsigned v) {
  unsigned old;
  asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}
// cheap device-wide barrier primitives: a release-add without a return value (the arriving thread does not wait for the
// L2 round trip), a relaxed polling load (no L1 invalidation per poll) and one acquire fence once the poll has succeeded
SSDK_DEVINL void red_add_release_gpu_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("red.release.gpu.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
SSDK_DEVINL unsigned long long ld_relaxed_gpu_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
SSDK_DEVINL void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
SSDK_DEVINL void st_relaxed_gpu_u32(unsigned* p, unsigned v) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// acquire load at device scope (flag / counter polling)
SSDK_DEVINL unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
SSDK_DEVINL void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
// 16-byte volatile load (flag-in-word polling: re-issued on every call, never cached in registers)
SSDK_DEVINL uint4 ld_volatile_v4(const void* p) {
  uint4 r;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

#else  // SSDK_HOST_EMU: host stand-ins for the few PTX helpers the emulated kernels use
enum { TR_PREP = 1, TR_NORM, TR_GEMM, TR_ROPE, TR_ATTN, TR_SAMPLE, TR_VERIFY, TR_MISC };
enum { TRF_ATTN = 16, TRF_NORM = 24, TRF_ROPE = 32, TRF_COMB = 40, TRF_GEMM = 48 };
SSDK_DEVINL void trace_mark(int) {}
SSDK_DEVINL void trace_fine(int) {}
SSDK_DEVINL void pdl_wait() {}
SSDK_DEVINL void pdl_launch_dependents() {}
SSDK_DEVINL uint4 ld_nc_v4(const void* p) { return *reinterpret_cast<const uint4*>(p); }
SSDK_DEVINL uint4 ld_nc_v4_evict_first(const void* p) { return *reinterpret_cast<const uint4*>(p); }
SSDK_DEVINL unsigned ld_acquire_u32(const unsigned* p) {
  std::this_thread::yield();
  return __atomic_load_n(p, __ATOMIC_ACQUIRE);
}
SSDK_DEVINL unsigned atom_add_acq_rel_gpu(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_ACQ_REL); }
SSDK_DEVINL void red_add_release_gpu_u64(unsigned long long* p, unsigned long long v) { __atomic_fetch_add(p, v, __ATOMIC_RELEASE); }
SSDK_DEVINL unsigned long long ld_relaxed_gpu_u64(const unsigned long long* p) {
  std::this_thread::yield();
#if defined(__SANITIZE_THREAD__)
  // ThreadSanitizer does not model atomic_thread_fence: the "relaxed poll + one acquire fence" of the device-wide barrier
  // would show up as races on everything the barrier orders.  Under TSan the poll itself acquires.
  return __atomic_load_n(p, __ATOMIC_ACQUIRE);
#else
  return __atomic_load_n(p, __ATOMIC_RELAXED);
#endif
}
SSDK_DEVINL void fence_acq_rel_gpu() { std::atomic_thread_fence(std::memory_order_acq_rel); }
SSDK_DEVINL void st_relaxed_gpu_u32(unsigned* p, unsigned v) { __atomic_store_n(p, v, __ATOMIC_RELAXED); }
SSDK_DEVINL void prefetch_l2(const void*) {}
// mbarrier + bulk copy stand-ins: one 64-bit word = {phase bit 63 | pending arrivals 32..47 | init count 48..62 | tx bytes 0..31},
// updated under one global lock (test infrastructure; the bulk copy is a synchronous memcpy by the issuing thread)
inline std::mutex& emu_mbar_mu() {
  static std::mutex m;
  return m;
}
inline void emu_mbar_settle(uint64_t& w) {
  const uint64_t pending = (w >> 32) & 0xFFFFu, init = (w >> 48) & 0x7FFFu;
  if (pending == 0 && (uint32_t)w == 0u) w = ((w ^ (1ull << 63)) & ~(0xFFFFull << 32)) | (init << 32);
}
SSDK_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
  std::lock_guard<std::mutex> g(emu_mbar_mu());
  *bar = ((uint64_t)count << 48) | ((uint64_t)count << 32);
}
SSDK_DEVINL void fence_mbar_init() {}
SSDK_DEVINL void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  std::lock_guard<std::mutex> g(emu_mbar_mu());
  uint64_t w = *bar;
  w = (w & ~0xFFFFFFFFull) | (uint32_t)((uint32_t)w + bytes);
  w -= (1ull << 32);
  emu_mbar_settle(w);
  *bar = w;
}
SSDK_DEVINL void mbar_arrive(uint64_t* bar) {
  std::lock_guard<std::mutex> g(emu_mbar_mu());
  uint64_t w = *bar;
  w -= (1ull << 32);
  emu_mbar_settle(w);
  *bar = w;
}
SSDK_DEVINL bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  std::lock_guard<std::mutex> g(emu_mbar_mu());
  return (uint32_t)(*bar >> 63) != parity;
}
SSDK_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
  for (;;) {
    {
      std::lock_guard<std::mutex> g(emu_mbar_mu());
      if ((uint32_t)(*bar >> 63) != parity) return;
    }
    std::this_thread::yield();
  }
}
SSDK_DEVINL void bulk_load_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  std::memcpy(smem_dst, gsrc, bytes);
  std::lock_guard<std::mutex> g(emu_mbar_mu());
  uint64_t w = *bar;
  w = (w & ~0xFFFFFFFFull) | (uint32_t)((uint32_t)w - bytes);
  emu_mbar_settle(w);
  *bar = w;
}
SSDK_DEVINL uint4 ld_volatile_v4(const void* p) {
  // two aligned 8-byte words {2 x bf16, epoch}: each is read atomically, like the device's 8-byte store granularity
  const uint64_t* q = reinterpret_cast<const uint64_t*>(p);
  const uint64_t a = __atomic_load_n(q, __ATOMIC_ACQUIRE), b = __atomic_load_n(q + 1, __ATOMIC_ACQUIRE);
  std::this_thread::yield();
  return make_uint4((uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32));
}
#endif

}  // namespace ssdk
