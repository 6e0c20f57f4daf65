// Runs the SOURCE of csrc/attention.cuh (paged_attn_kernel + attn_combine_kernel) on host threads (cuda_emu.h).
// TEST INFRASTRUCTURE.
//   run_attention <input blob> <output blob>
// input: int32 B, Q, H, KV, hd, block_size, max_blocks, n_slots, n_split; float32 scale; bf16 q [B*Q, H, hd],
//        k_cache, v_cache [n_slots, KV, hd]; int32 block_tables [B, max_blocks], context_lens [B]
// output: int32 TQ, MT, n_qtiles, n_split; bf16 out [B*Q, H*hd]
// The tile plan is the engine's (attn_make_plan); n_split is forced from the input, so that one split, a few and the
// 32-way maximum all run whatever the host is.
#include "cuda_emu.h"
#define SSDK_HOST_EMU 1
#include "../../ssd_b200/csrc/attention.cuh"

#include <fstream>
#include <iostream>
#include <limits>
#include <utility>

using bf16 = __nv_bfloat16;

struct Reader {
  std::ifstream f;
  explicit Reader(const char* p) : f(p, std::ios::binary) {
    if (!f) {
      std::cerr << "cannot open " << p << "\n";
      std::exit(2);
    }
  }
  template <typename T>
  std::vector<T> vec(size_t n) {
    std::vector<T> v(n);
    f.read(reinterpret_cast<char*>(v.data()), (std::streamsize)(n * sizeof(T)));
    if (!f) {
      std::cerr << "short read\n";
      std::exit(2);
    }
    return v;
  }
  int i32() { return vec<int32_t>(1)[0]; }
  float f32() { return vec<float>(1)[0]; }
};

template <int HD, int MT>
void run(const ssdk::AttnParams& p, dim3 grid) {
  const size_t smem = (size_t)2 * 2 * ssdk::kAttChunk * (HD + 8) * 2;
  emu::launch(ssdk::paged_attn_kernel<HD, MT>, p, grid, ssdk::attn_warps(MT) * 32, smem, /*wave=*/4);
}

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  Reader r(argv[1]);
  const int B = r.i32(), Q = r.i32(), H = r.i32(), KV = r.i32(), hd = r.i32(), bs = r.i32(), mb = r.i32();
  const int nslots = r.i32(), n_split = r.i32();
  const float scale = r.f32();
  auto q = r.vec<bf16>((size_t)B * Q * H * hd);
  auto kc = r.vec<bf16>((size_t)nslots * KV * hd), vc = r.vec<bf16>((size_t)nslots * KV * hd);
  auto bt = r.vec<int32_t>((size_t)B * mb);
  auto ctx = r.vec<int32_t>(B);

  ssdk::AttnPlan pl;
  if (ssdk::attn_make_plan(H, KV, B, Q, bs * mb, /*n_sms=*/1 << 20, &pl) != 0) {
    std::cerr << "no plan\n";
    return 3;
  }
  if (n_split < 1 || n_split > ssdk::kAttnMaxSplit) return 3;
  pl.n_split = n_split;
  // unwritten outputs and partials are NaN, so a row the kernel forgets or a partial it never wrote shows up
  std::vector<bf16> out((size_t)B * Q * H * hd, __float2bfloat16_rn(std::numeric_limits<float>::quiet_NaN()));
  std::vector<float> part_o((size_t)B * Q * H * n_split * hd, std::numeric_limits<float>::quiet_NaN());
  std::vector<float> part_lse((size_t)B * Q * H * n_split, std::numeric_limits<float>::quiet_NaN());

  ssdk::AttnParams p;
  std::memset(&p, 0, sizeof(p));
  p.q = q.data(); p.k_cache = kc.data(); p.v_cache = vc.data(); p.block_tables = bt.data(); p.context_lens = ctx.data();
  p.out = out.data(); p.part_o = part_o.data(); p.part_lse = part_lse.data();
  p.B = B; p.Q = Q; p.H = H; p.KV = KV; p.block_size = bs; p.max_blocks = mb;
  p.n_split = pl.n_split; p.TQ = pl.TQ; p.n_qtiles = pl.n_qtiles;
  p.g_shift = ssdk::attn_g_shift(H, KV);
  p.scale_log2 = scale * 1.4426950408889634f;
  dim3 grid;
  grid.x = KV; grid.y = pl.n_split; grid.z = B * pl.n_qtiles;
  if (hd == 64 && pl.MT == 1) run<64, 1>(p, grid);
  else if (hd == 64 && pl.MT == 2) run<64, 2>(p, grid);
  else if (hd == 128 && pl.MT == 1) run<128, 1>(p, grid);
  else if (hd == 128 && pl.MT == 2) run<128, 2>(p, grid);
  else {
    std::cerr << "no instantiation for hd " << hd << " MT " << pl.MT << "\n";
    return 3;
  }
  if (pl.n_split > 1) {
    dim3 cg;
    cg.x = B * Q * H;
    auto combine = [](const std::pair<ssdk::AttnParams, int>& a) { ssdk::attn_combine_kernel(a.first, a.second); };
    emu::launch(combine, std::make_pair(p, hd), cg, 32, 0, /*wave=*/32);
  }
  std::ofstream o(argv[2], std::ios::binary);
  const int32_t plan[4] = {pl.TQ, pl.MT, pl.n_qtiles, pl.n_split};
  o.write(reinterpret_cast<const char*>(plan), sizeof(plan));
  o.write(reinterpret_cast<const char*>(out.data()), (std::streamsize)(out.size() * 2));
  return 0;
}
