// Runs the SOURCE of rope_store_kernel (csrc/elementwise.cuh) on host threads twice on the same inputs: the bf16
// instance and the e4m3-cache instance (KV8).  TEST INFRASTRUCTURE.   run_rope_store_fp8 <in> <out>
// input: int32 M H KV hd max_pos nslots qk_norm ; float32 eps k_scale v_scale ; int64 positions[M] ; int32 slots[M] ;
//        float32 table[max_pos*hd] ; bf16 qn[hd] kn[hd] ; bf16 qkv[M*(H+2KV)*hd] (dense)
// output: bf16 q, k_cache, v_cache of the bf16 instance ; bf16 q of the KV8 instance ; uint8 k_cache, v_cache of the
//         KV8 instance.  The e4m3 caches start filled with 0x5A, so a slot the kernel must skip keeps that byte.
#include "cuda_emu.h"
#define SSDK_HOST_EMU 1
#include "../../ssd_b200/csrc/elementwise.cuh"

#include <fstream>

using bf16 = __nv_bfloat16;
template <typename T>
static std::vector<T> rd(std::ifstream& f, size_t n) {
  std::vector<T> v(n);
  f.read(reinterpret_cast<char*>(v.data()), (std::streamsize)(n * sizeof(T)));
  if (!f && n) std::exit(2);
  return v;
}
template <typename T>
static void wr(std::ofstream& o, const std::vector<T>& v) {
  o.write(reinterpret_cast<const char*>(v.data()), (std::streamsize)(v.size() * sizeof(T)));
}

template <bool KV8>
static void launch(const ssdk::RopeParams& p, int hd, dim3 grid) {
  if (hd == 64) emu::launch(ssdk::rope_store_kernel<64, KV8>, p, grid, 128, 0, 8);
  else emu::launch(ssdk::rope_store_kernel<128, KV8>, p, grid, 128, 0, 8);
}

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  std::ifstream f(argv[1], std::ios::binary);
  std::ofstream o(argv[2], std::ios::binary);
  auto h = rd<int32_t>(f, 7);
  const int M = h[0], H = h[1], KV = h[2], hd = h[3], max_pos = h[4], nslots = h[5], qk_norm = h[6];
  if (hd != 64 && hd != 128) return 3;
  auto sc = rd<float>(f, 3);
  auto pos = rd<int64_t>(f, M);
  auto slots = rd<int32_t>(f, M);
  auto table = rd<float>(f, (size_t)max_pos * hd);
  auto qn = rd<bf16>(f, hd), kn = rd<bf16>(f, hd);
  const int qkv_dim = (H + 2 * KV) * hd;
  auto qkv = rd<bf16>(f, (size_t)M * qkv_dim);
  std::vector<bf16> q((size_t)M * H * hd), kc((size_t)nslots * KV * hd), vc((size_t)nslots * KV * hd);
  std::vector<bf16> q8((size_t)M * H * hd);
  std::vector<uint8_t> kc8((size_t)nslots * KV * hd, 0x5A), vc8((size_t)nslots * KV * hd, 0x5A);
  ssdk::RopeParams p;
  std::memset(&p, 0, sizeof(p));
  p.qkv.dense = qkv.data(); p.qkv.S = 0; p.qkv.M = M; p.qkv.N = qkv_dim;
  p.positions = pos.data(); p.slot_mapping = slots.data(); p.rope_table = table.data();
  p.q_norm_w = qk_norm ? qn.data() : nullptr; p.k_norm_w = qk_norm ? kn.data() : nullptr; p.norm_eps = sc[0];
  p.heads = H; p.kv_heads = KV; p.head_dim = hd;
  dim3 grid;
  grid.x = (unsigned)M;
  grid.y = (unsigned)((H + 2 * KV + 3) / 4);
  p.q_out = q.data(); p.k_cache = kc.data(); p.v_cache = vc.data();
  launch<false>(p, hd, grid);
  p.q_out = q8.data();
  p.k_cache = reinterpret_cast<bf16*>(kc8.data()); p.v_cache = reinterpret_cast<bf16*>(vc8.data());
  p.k_scale = sc[1]; p.v_scale = sc[2];
  launch<true>(p, hd, grid);
  wr(o, q); wr(o, kc); wr(o, vc); wr(o, q8); wr(o, kc8); wr(o, vc8);
  return 0;
}
