// Runs the SOURCE of the FP8 instance of csrc/draft_stream.cuh (draft_stream_kernel<HD, GMAX, true>) on host threads
// (cuda_emu.h).  TEST INFRASTRUCTURE.
//   run_draft_stream_fp8 <input blob> <output blob>
// blob layout: see tests/test_fp8_draft_emu_cpu.py (the writer).  The decoder linears are e4m3 bytes followed by their
// fp32 row scales.  Output: the run asked for (forward 0 two-row when a token is pending); with a pending token also the
// same work as two launches (a headless one-token launch for the pending token, then the forwards of the recovery token).
#include "cuda_emu.h"
#define SSDK_HOST_EMU 1
#include "../../ssd_b200/csrc/draft_stream.cuh"

#include <fstream>
#include <iostream>

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

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  Reader r(argv[1]);
  const int d = r.i32(), L = r.i32(), H = r.i32(), KV = r.i32(), hd = r.i32(), ffn = r.i32(), vocab = r.i32();
  const int qk_norm = r.i32(), block_size = r.i32(), max_blocks = r.i32(), nslots = r.i32(), ctx0 = r.i32();
  const int n_fwd = r.i32(), grid = r.i32(), max_pos = r.i32(), n_stages = r.i32();
  const float eps = r.f32();
  float temp = r.f32();
  auto rng = r.vec<uint64_t>(2);    // seed, call_base
  auto tokens = r.vec<int64_t>(2);  // pending token at position ctx0 - 1 (-1: none), first input token (position ctx0)
  auto block_table = r.vec<int32_t>(max_blocks);
  auto embed = r.vec<bf16>((size_t)vocab * d), final_norm = r.vec<bf16>(d), lm_head = r.vec<bf16>((size_t)vocab * d);
  auto rope = r.vec<float>((size_t)max_pos * hd);
  const int qkv_dim = (H + 2 * KV) * hd;
  struct LW {
    std::vector<uint8_t> qkv, o, gate_up, down;
    std::vector<float> s_qkv, s_o, s_gate_up, s_down;
    std::vector<bf16> in_norm, post_norm, q_norm, k_norm;
  };
  std::vector<LW> lw(L);
  for (auto& w : lw) {
    w.qkv = r.vec<uint8_t>((size_t)qkv_dim * d);
    w.s_qkv = r.vec<float>(qkv_dim);
    w.o = r.vec<uint8_t>((size_t)d * H * hd);
    w.s_o = r.vec<float>(d);
    w.gate_up = r.vec<uint8_t>((size_t)2 * ffn * d);
    w.s_gate_up = r.vec<float>(2 * ffn);
    w.down = r.vec<uint8_t>((size_t)d * ffn);
    w.s_down = r.vec<float>(d);
    w.in_norm = r.vec<bf16>(d);
    w.post_norm = r.vec<bf16>(d);
    w.q_norm = r.vec<bf16>(hd);
    w.k_norm = r.vec<bf16>(hd);
  }
  const size_t cache_layer = (size_t)nslots * KV * hd;
  const auto kc0 = r.vec<bf16>(cache_layer * L), vc0 = r.vec<bf16>(cache_layer * L);

  const size_t nvec = (size_t)qkv_dim + 4 * d + ffn + H * hd + 64;
  std::vector<bf16> vecs(nvec), vecs0(nvec);
  std::vector<float> attn((size_t)H * ssdk::kDsSplits * (hd + 2));
  std::vector<ssdk::ArgMax> partial(grid);
  alignas(8) unsigned sync[64] = {0};
  const int G = H / KV, gmax = G <= 4 ? 4 : 8;
  const size_t xs = (size_t)ssdk::ds_xs_floats(d, ffn, H * hd);
  const size_t scratch = (size_t)gmax * hd + 2 * hd + (size_t)ssdk::kDsWarps * gmax * (hd + 2);
  const size_t smem = (xs + scratch) * 4 + 256 + (size_t)n_stages * ssdk::kDsSlotBytes;
  const bool pending = tokens[0] >= 0;

  std::ofstream o(argv[2], std::ios::binary);
  for (int run = 0; run < (pending ? 2 : 1); ++run) {
    const bool folded = run == 0;  // run 0: the launch asked for; run 1: the same work as two launches
    std::vector<bf16> kc = kc0, vc = vc0, logits((size_t)n_fwd * vocab);
    std::vector<int64_t> tok_buf(n_fwd + 1, -1);
    const int launches = folded ? 1 : 2;
    for (int li = 0; li < launches; ++li) {
      const bool head_only = !folded && li == 0;
      int32_t ctx_dev = head_only ? ctx0 - 1 : ctx0;
      int64_t pend = folded ? tokens[0] : -1;
      std::vector<int64_t> tb1(2, -1);
      int64_t* tb = head_only ? tb1.data() : tok_buf.data();
      tb[0] = head_only ? tokens[0] : tokens[1];

      ssdk::DsParams p;
      std::memset(&p, 0, sizeof(p));
      p.d = d; p.L = L; p.H = H; p.KV = KV; p.ffn = ffn; p.vocab = vocab; p.qk_norm = qk_norm;
      p.eps = eps;
      p.scale_log2 = (1.0f / std::sqrt((float)hd)) * 1.4426950408889634f;
      p.embed = embed.data(); p.final_norm = final_norm.data(); p.lm_head = lm_head.data(); p.rope = rope.data();
      p.k_cache = kc.data(); p.v_cache = vc.data();
      p.cache_layer_stride = (long long)cache_layer;
      p.block_size = block_size; p.max_blocks = max_blocks;
      p.tok_buf = tb; p.n_fwd = head_only ? 1 : n_fwd; p.skip_last_head = head_only ? 1 : 0;
      p.ctx0 = &ctx_dev; p.block_table = block_table.data();
      p.pend_tok = folded ? &pend : nullptr;
      p.vec_row0 = vecs0.data();
      bf16* v = vecs.data();
      p.vec_qkv = v; v += (qkv_dim + 7) / 8 * 8;
      p.vec_attn = v; v += H * hd;
      p.vec_o = v; v += d;
      p.vec_down = v; v += d;
      p.resid0 = v; v += d;
      p.resid1 = v; v += d;
      p.vec_act = v;
      p.attn_part = attn.data();
      p.logits = head_only ? nullptr : logits.data(); p.logits_ld = vocab;
      p.temp = &temp; p.dyn = nullptr; p.seed = rng[0]; p.call_base = rng[1];
      p.samp_partial = partial.data();
      p.bar_state = sync;
      p.attn_ticket = sync + 8;
      p.n_slots = n_stages;
      for (int l = 0; l < L; ++l) {
        auto b = [](const std::vector<uint8_t>& x) { return reinterpret_cast<const bf16*>(x.data()); };
        p.layers[l] = ssdk::DsLayer{b(lw[l].qkv), b(lw[l].o), b(lw[l].gate_up), b(lw[l].down),
                                    lw[l].in_norm.data(), lw[l].post_norm.data(), lw[l].q_norm.data(), lw[l].k_norm.data()};
        p.fp8_scale[l][ssdk::DS_QKV] = lw[l].s_qkv.data();
        p.fp8_scale[l][ssdk::DS_O] = lw[l].s_o.data();
        p.fp8_scale[l][ssdk::DS_GU] = lw[l].s_gate_up.data();
        p.fp8_scale[l][ssdk::DS_DOWN] = lw[l].s_down.data();
      }
      if (hd == 64 && gmax == 4) emu::launch(ssdk::draft_stream_kernel<64, 4, true>, p, grid, ssdk::kDsThreads, smem);
      else if (hd == 64) emu::launch(ssdk::draft_stream_kernel<64, 8, true>, p, grid, ssdk::kDsThreads, smem);
      else if (gmax == 4) emu::launch(ssdk::draft_stream_kernel<128, 4, true>, p, grid, ssdk::kDsThreads, smem);
      else emu::launch(ssdk::draft_stream_kernel<128, 8, true>, p, grid, ssdk::kDsThreads, smem);
      for (int i = 2; i < 64; ++i)
        if (sync[i] != 0) {
          std::cerr << "attention ticket " << i << " not back to zero\n";
          return 3;
        }
      unsigned long long arrivals;
      std::memcpy(&arrivals, sync, 8);
      if (arrivals % (unsigned long long)grid != 0) {
        std::cerr << "barrier arrival counter is not a whole number of barriers\n";
        return 3;
      }
    }
    o.write(reinterpret_cast<const char*>(logits.data()), (std::streamsize)(logits.size() * 2));
    o.write(reinterpret_cast<const char*>(kc.data()), (std::streamsize)(kc.size() * 2));
    o.write(reinterpret_cast<const char*>(vc.data()), (std::streamsize)(vc.size() * 2));
    o.write(reinterpret_cast<const char*>(tok_buf.data()), (std::streamsize)(tok_buf.size() * 8));
  }
  return 0;
}
