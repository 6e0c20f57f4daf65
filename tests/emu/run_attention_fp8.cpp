// Runs the SOURCE of csrc/attention.cuh with e4m3 caches (paged_attn_kernel<HD, MT, true> or
// paged_attn_varlen_kernel<HD, MT, true>, + attn_combine_kernel) on host threads (cuda_emu.h).  TEST INFRASTRUCTURE.
//   run_attention_fp8 <input blob> <output blob>
// input: int32 varlen, B, Q, H, KV, hd, block_size, max_blocks, n_slots, n_split; int32 q_lens [B] (varlen only);
//        float32 scale, k_scale, v_scale; bf16 q [sum q_lens or B*Q, H, hd]; uint8 e4m3 k_cache, v_cache
//        [n_slots, KV, hd]; int32 block_tables [B, max_blocks], context_lens [B]
// output: int32 TQ, MT, n_qtiles, n_split; bf16 out [rows, H*hd]
// The plan is the engine's (attn_make_plan / attn_make_plan_varlen + attn_varlen_tiles) with n_split forced from the
// input; the scales are applied as the engine applies them (k_scale folded into scale_log2, v_scale in p.v_scale).
#include "cuda_emu.h"
#define SSDK_HOST_EMU 1
#include "../../ssd_b200/csrc/attention.cuh"

#include <fstream>
#include <iostream>
#include <limits>
#include <tuple>

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

using Args = std::pair<ssdk::AttnParams, ssdk::AttnVarlen>;

template <int HD, int MT>
void run(bool varlen, const Args& a, dim3 grid) {
  const size_t smem = (size_t)ssdk::attn_smem_bytes(HD);
  if (varlen) {
    auto k = [](const Args& x) { ssdk::paged_attn_varlen_kernel<HD, MT, true>(x.first, x.second); };
    emu::launch(k, a, grid, ssdk::attn_warps(MT) * 32, smem, /*wave=*/4);
  } else {
    auto k = [](const Args& x) { ssdk::paged_attn_kernel<HD, MT, true>(x.first); };
    emu::launch(k, a, grid, ssdk::attn_warps(MT) * 32, smem, /*wave=*/4);
  }
}

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  Reader r(argv[1]);
  const int varlen = r.i32(), B = r.i32(), Q = r.i32(), H = r.i32(), KV = r.i32(), hd = r.i32(), bs = r.i32();
  const int mb = r.i32(), nslots = r.i32(), n_split = r.i32();
  std::vector<int32_t> q_lens = varlen ? r.vec<int32_t>(B) : std::vector<int32_t>((size_t)B, Q);
  const float scale = r.f32(), k_scale = r.f32(), v_scale = r.f32();
  int M = 0;
  for (int b = 0; b < B; ++b) M += q_lens[b];
  auto q = r.vec<bf16>((size_t)M * H * hd);
  auto kc = r.vec<uint8_t>((size_t)nslots * KV * hd), vc = r.vec<uint8_t>((size_t)nslots * KV * hd);
  auto bt = r.vec<int32_t>((size_t)B * mb);
  auto ctx = r.vec<int32_t>(B);

  ssdk::AttnPlan pl;
  int n_tiles = 0;
  const int rc = varlen ? ssdk::attn_make_plan_varlen(H, KV, B, q_lens.data(), bs * mb, 1 << 20, &pl, &n_tiles)
                        : ssdk::attn_make_plan(H, KV, B, Q, bs * mb, 1 << 20, &pl);
  if (rc != 0) {
    std::cerr << "no plan\n";
    return 3;
  }
  if (n_split < 1 || n_split > ssdk::kAttnMaxSplit) return 3;
  pl.n_split = n_split;
  std::vector<ssdk::AttnTile> tiles((size_t)M);
  std::vector<int32_t> cu_q((size_t)B + 1);
  if (varlen && ssdk::attn_varlen_tiles(B, q_lens.data(), pl.TQ, tiles.data(), cu_q.data()) != n_tiles) return 3;
  // unwritten outputs and partials are NaN, so a row the kernel forgets or a partial it never wrote shows up
  std::vector<bf16> out((size_t)M * H * hd, __float2bfloat16_rn(std::numeric_limits<float>::quiet_NaN()));
  std::vector<float> part_o((size_t)M * H * n_split * hd, std::numeric_limits<float>::quiet_NaN());
  std::vector<float> part_lse((size_t)M * H * n_split, std::numeric_limits<float>::quiet_NaN());

  ssdk::AttnParams p;
  std::memset(&p, 0, sizeof(p));
  p.q = q.data();
  p.k_cache = reinterpret_cast<const bf16*>(kc.data());
  p.v_cache = reinterpret_cast<const bf16*>(vc.data());
  p.block_tables = bt.data(); p.context_lens = ctx.data();
  p.out = out.data(); p.part_o = part_o.data(); p.part_lse = part_lse.data();
  p.B = B; p.Q = varlen ? 0 : Q; p.H = H; p.KV = KV; p.block_size = bs; p.max_blocks = mb;
  p.n_split = pl.n_split; p.TQ = pl.TQ; p.n_qtiles = pl.n_qtiles;
  p.g_shift = ssdk::attn_g_shift(H, KV);
  p.scale_log2 = scale * 1.4426950408889634f;
  p.scale_log2 *= k_scale;
  p.v_scale = v_scale;
  ssdk::AttnVarlen v{};
  if (varlen) {
    v.tiles = tiles.data();
    v.cu_q = cu_q.data();
  }
  const Args args{p, v};
  dim3 grid;
  grid.x = KV; grid.y = pl.n_split; grid.z = varlen ? n_tiles : B * pl.n_qtiles;
  if (hd == 64 && pl.MT == 1) run<64, 1>(varlen, args, grid);
  else if (hd == 64 && pl.MT == 2) run<64, 2>(varlen, args, grid);
  else if (hd == 128 && pl.MT == 1) run<128, 1>(varlen, args, grid);
  else if (hd == 128 && pl.MT == 2) run<128, 2>(varlen, args, grid);
  else {
    std::cerr << "no instantiation for hd " << hd << " MT " << pl.MT << "\n";
    return 3;
  }
  if (pl.n_split > 1) {
    dim3 cg;
    cg.x = M * H;
    auto combine = [](const std::tuple<ssdk::AttnParams, int, ssdk::AttnVarlen, int>& a) {
      if (std::get<3>(a)) ssdk::attn_combine_kernel<true>(std::get<0>(a), std::get<1>(a), std::get<2>(a));
      else ssdk::attn_combine_kernel<false>(std::get<0>(a), std::get<1>(a), ssdk::AttnVarlen{});
    };
    emu::launch(combine, std::make_tuple(p, hd, v, varlen), cg, 32, 0, /*wave=*/32);
  }
  std::ofstream o(argv[2], std::ios::binary);
  const int32_t plan[4] = {pl.TQ, pl.MT, pl.n_qtiles, pl.n_split};
  o.write(reinterpret_cast<const char*>(plan), sizeof(plan));
  o.write(reinterpret_cast<const char*>(out.data()), (std::streamsize)(out.size() * 2));
  return 0;
}
