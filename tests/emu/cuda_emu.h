// cuda_emu.h — TEST INFRASTRUCTURE: the small CUDA vocabulary the non-TMA / non-wgmma kernels of ssd_b200/csrc use, mapped
// onto host threads so that a kernel's *source* (not a restatement of it) can be executed on a machine without a GPU:
// one OS thread per CUDA thread, __syncthreads = a per-CTA barrier, warp shuffles, ldmatrix and mma.sync = a per-warp
// exchange + barrier, cp.async = a copy at issue time, global atomics = host atomics.  Host memory is coherent and sequentially consistent enough for these tests, so this
// checks indexing, control flow, barrier placement (a shuffle or barrier that not all threads reach deadlocks here just
// as it is undefined on the device) and arithmetic — not the device memory model, cache behaviour or performance.
#pragma once
#include <atomic>
#include <barrier>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#define __device__
#define __global__
#define __host__
#define __forceinline__ inline
#define __grid_constant__
#define __launch_bounds__(...)
#define __align__(n) alignas(n)

struct uint2 { uint32_t x, y; };
struct alignas(16) uint4 { uint32_t x, y, z, w; };
struct float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
struct dim3 { unsigned x = 1, y = 1, z = 1; };
inline uint2 make_uint2(uint32_t x, uint32_t y) { return {x, y}; }
inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return {x, y, z, w}; }
inline float2 make_float2(float x, float y) { return {x, y}; }
inline float4 make_float4(float x, float y, float z, float w) { return {x, y, z, w}; }

// ---- bf16 (round-to-nearest-even, like cuda_bf16.h) ----
struct __nv_bfloat16 { uint16_t v; };
struct __nv_bfloat162 { __nv_bfloat16 x, y; };
inline __nv_bfloat16 __float2bfloat16_rn(float f) {
  uint32_t u;
  std::memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return {(uint16_t)((u >> 16) | 0x40)};  // NaN
  u += 0x7fffu + ((u >> 16) & 1u);
  return {(uint16_t)(u >> 16)};
}
inline __nv_bfloat16 __float2bfloat16(float f) { return __float2bfloat16_rn(f); }
inline float __bfloat162float(__nv_bfloat16 b) {
  uint32_t u = (uint32_t)b.v << 16;
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}
inline __nv_bfloat16 __ushort_as_bfloat16(unsigned short s) { return {s}; }
inline __nv_bfloat162 __floats2bfloat162_rn(float a, float b) { return {__float2bfloat16_rn(a), __float2bfloat16_rn(b)}; }
inline float2 __bfloat1622float2(__nv_bfloat162 v) { return {__bfloat162float(v.x), __bfloat162float(v.y)}; }

// ---- math ----
inline float rsqrtf(float x) { return 1.0f / std::sqrt(x); }
inline float __expf(float x) { return std::exp(x); }
inline float __logf(float x) { return std::log(x); }
inline uint32_t __umulhi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
using std::max;
using std::min;

namespace emu {
struct Warp {
  uint32_t slot[32];
  const void* ptr[32];    // ldmatrix row addresses
  uint32_t frag[32][6];   // mma.sync A and B fragments
  std::barrier<> bar{32};
};
struct Cta {
  explicit Cta(int threads, size_t dyn) : bar(threads), dyn_smem(dyn + 64), warps((threads + 31) / 32) {
    for (auto& w : warps) w = std::make_unique<Warp>();
  }
  std::barrier<> bar;
  std::vector<unsigned char> dyn_smem;
  std::vector<std::unique_ptr<Warp>> warps;
  std::mutex mu;
  std::map<int, std::vector<unsigned char>> statics;
  std::map<int, std::unique_ptr<std::barrier<>>> named;  // bar.sync id, count
};
struct ThreadCtx {
  Cta* cta = nullptr;
};
inline thread_local ThreadCtx tctx;
inline void* dyn_smem() {
  auto p = reinterpret_cast<uintptr_t>(tctx.cta->dyn_smem.data());
  return reinterpret_cast<void*>((p + 63) & ~uintptr_t(63));
}
template <typename T>
T* static_smem(size_t n, int key) {
  std::lock_guard<std::mutex> g(tctx.cta->mu);
  auto& v = tctx.cta->statics[key];
  if (v.empty()) v.resize(n * sizeof(T) + 64);
  return reinterpret_cast<T*>((reinterpret_cast<uintptr_t>(v.data()) + 63) & ~uintptr_t(63));
}
}  // namespace emu

inline thread_local dim3 threadIdx, blockIdx, blockDim, gridDim;

inline void __syncthreads() { emu::tctx.cta->bar.arrive_and_wait(); }
inline void __syncwarp(unsigned = 0xffffffffu) { emu::tctx.cta->warps[threadIdx.x >> 5]->bar.arrive_and_wait(); }
namespace emu {
// bar.sync id, count: a barrier among `count` threads of the CTA (the same `count` every time for a given id)
inline void named_barrier(int id, int count) {
  Cta* c = tctx.cta;
  std::barrier<>* b;
  {
    std::lock_guard<std::mutex> g(c->mu);
    auto& slot = c->named[id];
    if (!slot) slot = std::make_unique<std::barrier<>>(count);
    b = slot.get();
  }
  b->arrive_and_wait();
}
}  // namespace emu
inline void __threadfence() { std::atomic_thread_fence(std::memory_order_seq_cst); }
inline void __trap() {
  std::fprintf(stderr, "[cuda_emu] __trap()\n");
  std::abort();
}
inline long long clock64() {
  // ~2 "cycles" per ns keeps the kernels' cycle-count time-outs in the seconds range
  return 2 * std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
template <typename T>
inline T __shfl_xor_sync(unsigned, T v, int lane_mask) {
  static_assert(sizeof(T) == 4, "32-bit shuffles only");
  emu::Warp& w = *emu::tctx.cta->warps[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  std::memcpy(&w.slot[lane], &v, 4);
  w.bar.arrive_and_wait();
  T r;
  std::memcpy(&r, &w.slot[lane ^ lane_mask], 4);
  w.bar.arrive_and_wait();
  return r;
}

// ---- cp.async, ldmatrix, mma.sync (paged attention) ----
// cp.async.cg 16 bytes: copied, or zero-filled when the source size is 0, when issued; commit / wait have nothing left
// to order (a missing __syncthreads between the copy and its readers is still a race under TSan)
inline void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
  if (valid) std::memcpy(smem_dst, gsrc, 16);
  else std::memset(smem_dst, 0, 16);
}
inline void cp_async_commit() {}
template <int N>
inline void cp_async_wait() {}
namespace emu {
inline float bf16_bits_to_float(uint32_t h) {
  const uint32_t u = (h & 0xFFFFu) << 16;
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}
// ldmatrix.sync.aligned.m8n8.x4[.trans].shared.b16: lanes 8i..8i+7 give the addresses of rows 0..7 of 8x8 matrix i.
// Lane l receives in register i row l/4, columns 2(l%4) and 2(l%4)+1 of matrix i (of its transpose with .trans), the
// lower column in the low 16 bits.
inline void ldmatrix_x4(uint32_t* r, const void* smem_row, bool trans) {
  Warp& w = *tctx.cta->warps[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  w.ptr[lane] = smem_row;
  w.bar.arrive_and_wait();
  for (int i = 0; i < 4; ++i) {
    uint32_t e[2];
    for (int k = 0; k < 2; ++k) {
      const int row = trans ? 2 * (lane & 3) + k : lane >> 2;
      const int col = trans ? lane >> 2 : 2 * (lane & 3) + k;
      e[k] = static_cast<const uint16_t*>(w.ptr[8 * i + row])[col];
    }
    r[i] = e[0] | (e[1] << 16);
  }
  w.bar.arrive_and_wait();
}
}  // namespace emu
inline void ldmatrix_x4(uint32_t* r, const void* smem_row) { emu::ldmatrix_x4(r, smem_row, false); }
inline void ldmatrix_x4_trans(uint32_t* r, const void* smem_row) { emu::ldmatrix_x4(r, smem_row, true); }
// mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32, lane l = 4g + t:
//   A (16x16) a0: row g, a1: row g+8, a2: row g columns +8, a3: row g+8 columns +8 — each columns 2t, 2t+1;
//   B (16x8)  b0: rows 2t, 2t+1, b1: rows 2t+8, 2t+9 — each column g;
//   C/D (16x8) c0, c1: row g, c2, c3: row g+8 — columns 2t, 2t+1.
// Products of bf16 are exact in fp32; the 16 products are added to C in fp32, in k order.
inline void mma_bf16_16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  emu::Warp& w = *emu::tctx.cta->warps[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  for (int i = 0; i < 4; ++i) w.frag[lane][i] = a[i];
  w.frag[lane][4] = b0;
  w.frag[lane][5] = b1;
  w.bar.arrive_and_wait();
  float d[4];
  for (int e = 0; e < 4; ++e) {
    const int row = g + 8 * (e >> 1), col = 2 * t + (e & 1);
    float acc = c[e];
    for (int k = 0; k < 16; ++k) {
      const int sh = 16 * (k & 1);
      const uint32_t av = w.frag[4 * (row & 7) + ((k & 7) >> 1)][(row >> 3) + 2 * (k >> 3)] >> sh;
      const uint32_t bv = w.frag[4 * col + ((k & 7) >> 1)][4 + (k >> 3)] >> sh;
      acc += emu::bf16_bits_to_float(av) * emu::bf16_bits_to_float(bv);
    }
    d[e] = acc;
  }
  w.bar.arrive_and_wait();
  for (int e = 0; e < 4; ++e) c[e] = d[e];
}

inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
template <typename T>
inline T __ldcg(const T* p) { return *p; }

namespace emu {
// run kernel(params) on grid.x * grid.y * grid.z CTAs of `block` host threads each.  `wave` > 0 runs the CTAs in batches of that
// size (only valid for kernels whose CTAs never wait for one another: ticket / last-block patterns are fine, device-wide
// barriers are not); wave == 0 makes every CTA co-resident.
template <typename Kernel, typename Params>
void launch(Kernel kernel, const Params& params, dim3 grid, int block, size_t dyn_smem_bytes, int wave = 0) {
  if (block % 32) {
    std::fprintf(stderr, "[cuda_emu] block size must be a multiple of 32\n");
    std::abort();
  }
  const int total = (int)(grid.x * grid.y * grid.z);
  if (wave <= 0) wave = total;
  for (int first = 0; first < total; first += wave) {
    const int n = std::min(wave, total - first);
    std::vector<std::unique_ptr<Cta>> ctas;
    for (int b = 0; b < n; ++b) ctas.push_back(std::make_unique<Cta>(block, dyn_smem_bytes));
    std::vector<std::thread> ts;
    ts.reserve((size_t)n * block);
    for (int b = 0; b < n; ++b)
      for (int t = 0; t < block; ++t)
        ts.emplace_back([&, b, t] {
          tctx.cta = ctas[b].get();
          threadIdx.x = t;
          blockIdx.x = (unsigned)(first + b) % grid.x;
          blockIdx.y = (unsigned)(first + b) / grid.x % grid.y;
          blockIdx.z = (unsigned)(first + b) / (grid.x * grid.y);
          blockDim.x = block;
          gridDim = grid;
          kernel(params);
        });
    for (auto& t : ts) t.join();
  }
}
template <typename Kernel, typename Params>
void launch(Kernel kernel, const Params& params, int grid, int block, size_t dyn_smem_bytes) {
  dim3 g;
  g.x = (unsigned)grid;
  launch(kernel, params, g, block, dyn_smem_bytes, 0);
}
}  // namespace emu
