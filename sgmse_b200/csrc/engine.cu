// Host side of the engine: architecture walk, weight packing, the network forward pass as a static
// launch sequence over a liveness-planned workspace, the predictor-corrector loop (captured as one CUDA
// graph), the cuFFT STFT/iSTFT front/back end, and the C-ABI of include/sgmse_b200.h.
//
// Reference call stack replaced: ScoreModel.enhance (model.py:426-465) -> get_pc_sampler
// (sampling/__init__.py:26-70) -> NCSNpp.forward (backbones/ncsnpp.py:256-419).
#include <cstring>

#include "engine.h"
#include "rk45.h"

#include <math.h>
#include <string.h>

#include <algorithm>
#include <tuple>

using namespace sgmse;
typedef sgmse_b200_engine Engine;

namespace sgmse {
static thread_local std::string g_last_error;
void set_last_error(const std::string& m) { g_last_error = m; }
const char* get_last_error() { return g_last_error.c_str(); }
}  // namespace sgmse

namespace {

constexpr float INV_SQRT2 = 0.70710678118654752440f;

int gn_groups(int c) { return std::min(c / 4, 32); }   // layerspp.py:219

// ------------------------------------------------------------------------------------------------
// architecture walk: mirrors NCSNpp.__init__ (ncsnpp.py:104-253) / NCSNpp_48k.__init__
// ------------------------------------------------------------------------------------------------
struct Walker {
  Engine& e;
  long long off = 0;
  int midx = 0;
  long long add(const std::string& name, long long numel) {
    e.manifest.push_back(ParamRef{name, numel, off});
    const long long o = off;
    off += numel;
    return o;
  }
  std::string mod(const char* leaf) const { return "all_modules." + std::to_string(midx) + "." + leaf; }

  void resblock(int cin, int cout, bool up, bool down) {
    Layer l{};
    l.kind = LK_RES; l.idx = midx; l.cin = cin; l.cout = cout; l.up = up; l.down = down;
    l.shortcut = (cin != cout) || up || down;                // layerspp.py:233
    const int temb_dim = 4 * e.cfg.nf;
    l.gn0_w = add(mod("GroupNorm_0.weight"), cin); l.gn0_b = add(mod("GroupNorm_0.bias"), cin);
    l.conv0_w = add(mod("Conv_0.weight"), (long long)cout * cin * 9); l.conv0_b = add(mod("Conv_0.bias"), cout);
    l.dense_w = add(mod("Dense_0.weight"), (long long)cout * temb_dim); l.dense_b = add(mod("Dense_0.bias"), cout);
    l.gn1_w = add(mod("GroupNorm_1.weight"), cout); l.gn1_b = add(mod("GroupNorm_1.bias"), cout);
    l.conv1_w = add(mod("Conv_1.weight"), (long long)cout * cout * 9); l.conv1_b = add(mod("Conv_1.bias"), cout);
    if (l.shortcut) { l.conv2_w = add(mod("Conv_2.weight"), (long long)cout * cin); l.conv2_b = add(mod("Conv_2.bias"), cout); }
    l.temb_off = e.total_temb_c;
    e.total_temb_c += cout;
    e.layers.push_back(l);
    ++midx;
  }
  void attn(int c) {
    Layer l{};
    l.kind = LK_ATTN; l.idx = midx; l.cin = l.cout = c;
    l.gn0_w = add(mod("GroupNorm_0.weight"), c); l.gn0_b = add(mod("GroupNorm_0.bias"), c);
    for (int k = 0; k < 4; ++k) {
      const std::string n = "NIN_" + std::to_string(k);
      l.nin_w[k] = add(mod((n + ".W").c_str()), (long long)c * c);
      l.nin_b[k] = add(mod((n + ".b").c_str()), c);
    }
    e.layers.push_back(l);
    ++midx;
  }
  void combine(int c) {
    Layer l{};
    l.kind = LK_COMBINE; l.idx = midx; l.cin = 4; l.cout = c;
    l.conv0_w = add(mod("Conv_0.weight"), (long long)c * 4); l.conv0_b = add(mod("Conv_0.bias"), c);
    e.layers.push_back(l);
    ++midx;
  }
  void outconv(int c) {
    Layer l{};
    l.kind = LK_OUTCONV; l.idx = midx; l.cin = c; l.cout = 4;
    l.gn0_w = add(mod("weight"), c); l.gn0_b = add(mod("bias"), c);
    ++midx;
    l.conv0_w = add(mod("weight"), (long long)4 * c * 9); l.conv0_b = add(mod("bias"), 4);
    ++midx;
    e.layers.push_back(l);
  }
};

void build_network(Engine& e) {
  const sgmse_b200_config& c = e.cfg;
  SG_CHECK(c.nf > 0 && c.nf % 8 == 0, "nf=%d must be a positive multiple of 8", c.nf);
  SG_CHECK(c.num_levels >= 1 && c.num_levels <= 8, "num_levels=%d out of range", c.num_levels);
  SG_CHECK(c.num_res_blocks >= 1, "num_res_blocks must be >= 1");
  SG_CHECK(c.backbone == SGMSE_B200_BACKBONE_NCSNPP || c.backbone == SGMSE_B200_BACKBONE_NCSNPP_48K ||
               c.backbone == SGMSE_B200_BACKBONE_NCSNPP_V2, "unknown backbone %d", c.backbone);
  SG_CHECK(c.backbone != SGMSE_B200_BACKBONE_NCSNPP_V2 || !c.scale_by_sigma, "'ncsnpp_v2' has no in-network scaling");
  SG_CHECK(c.sde_kind == SGMSE_B200_SDE_OUVE || c.sde_kind == SGMSE_B200_SDE_SBVE, "unknown SDE kind %d", c.sde_kind);
  SG_CHECK(c.loss_type >= 0 && c.loss_type <= 2 && c.network_scaling >= 0 && c.network_scaling <= 2 && c.c_in >= 0 &&
               c.c_in <= 1 && c.c_out >= 0 && c.c_out <= 3 && c.c_skip >= 0 && c.c_skip <= 1, "bad preconditioning settings");
  Walker w{e};
  const int nf = c.nf, L = c.num_levels, temb_dim = 4 * nf;
  e.outl_w = w.add("output_layer.weight", 8);          // assigned before all_modules (ncsnpp.py:104)
  e.outl_b = w.add("output_layer.bias", 2);
  e.gfp_w = w.add(w.mod("W"), nf); ++w.midx;
  e.lin1_w = w.add(w.mod("weight"), (long long)temb_dim * 2 * nf); e.lin1_b = w.add(w.mod("bias"), temb_dim); ++w.midx;
  e.lin2_w = w.add(w.mod("weight"), (long long)temb_dim * temb_dim); e.lin2_b = w.add(w.mod("bias"), temb_dim); ++w.midx;
  e.inconv_w = w.add(w.mod("weight"), (long long)nf * 4 * 9); e.inconv_b = w.add(w.mod("bias"), nf); ++w.midx;

  auto has_attn = [&](int res) {
    for (int i = 0; i < c.num_attn_resolutions; ++i) if (c.attn_resolutions[i] == res) return true;
    return false;
  };
  std::vector<int> hs_c{nf};
  int in_ch = nf;
  for (int lvl = 0; lvl < L; ++lvl) {
    const int res = c.image_size >> lvl;
    for (int b = 0; b < c.num_res_blocks; ++b) {
      const int out_ch = nf * c.ch_mult[lvl];
      w.resblock(in_ch, out_ch, false, false);
      in_ch = out_ch;
      if (has_attn(res)) w.attn(in_ch);
      hs_c.push_back(in_ch);
    }
    if (lvl != L - 1) {
      w.resblock(in_ch, in_ch, false, true);
      if (c.progressive_input_skip) w.combine(in_ch);
      hs_c.push_back(in_ch);
    }
  }
  in_ch = hs_c.back();
  w.resblock(in_ch, in_ch, false, false);
  w.attn(in_ch);
  w.resblock(in_ch, in_ch, false, false);
  for (int lvl = L - 1; lvl >= 0; --lvl) {
    const int res = c.image_size >> lvl;
    for (int b = 0; b < c.num_res_blocks + 1; ++b) {
      const int out_ch = nf * c.ch_mult[lvl];
      w.resblock(in_ch + hs_c.back(), out_ch, false, false);
      hs_c.pop_back();
      in_ch = out_ch;
    }
    if (has_attn(res)) w.attn(in_ch);
    if (c.progressive_output_skip) w.outconv(in_ch);
    if (lvl != 0) w.resblock(in_ch, in_ch, true, false);
  }
  SG_CHECK(hs_c.empty(), "internal: skip stack not empty");
  if (!c.progressive_output_skip) w.outconv(in_ch);
  e.weights_numel = w.off;
}

// ------------------------------------------------------------------------------------------------
// weight packing (host) + upload
// ------------------------------------------------------------------------------------------------
template <typename T> T from_float(float v);
template <> float from_float<float>(float v) { return v; }
template <> __half from_float<__half>(float v) { return __float2half_rn(v); }

// activation element type of the mode: fp32 in fp32 and tf32_tc, fp16 otherwise
DType act_dtype(const sgmse_b200_config& c) {
  return c.mode == SGMSE_B200_MODE_FP32 || c.mode == SGMSE_B200_MODE_TF32_TC ? DT_F32 : DT_F16;
}
// the modes whose convolutions run on the wgmma kernel where it tiles the shape
bool tc_mode(const sgmse_b200_config& c) { return c.mode == SGMSE_B200_MODE_FP16_TC || c.mode == SGMSE_B200_MODE_TF32_TC; }

void* upload(Engine& e, const void* host, size_t bytes) {
  void* d = nullptr;
  CUDA_OK(cudaMalloc(&d, bytes));
  CUDA_OK(cudaMemcpy(d, host, bytes, cudaMemcpyHostToDevice));
  e.dev_allocs.push_back(d);
  e.weights_bytes += bytes;
  return d;
}

// rows: list of (pointer to [Cout][Cin][kh*kw] fp32, Cin, taps)
struct PackSrc { const float* w; int cin; int taps; };
void pack_conv(Engine& e, const std::vector<PackSrc>& srcs, int cout, bool out_major_src, ConvW& cw,
               bool identity_tail = false) {
  // out_major_src: true for Conv2d weights [Cout][Cin][taps]; false for NIN weights [Cin][Cout]
  int ktot = 0;
  for (auto& s : srcs) ktot += s.taps * s.cin;
  cw.ktot = ktot; cw.cout = cout;
  std::vector<float> kd((size_t)ktot * cout);   // [k][cout]
  int kbase = 0;
  for (auto& s : srcs) {
    for (int tap = 0; tap < s.taps; ++tap)
      for (int ci = 0; ci < s.cin; ++ci) {
        float* dst = kd.data() + (size_t)(kbase + tap * s.cin + ci) * cout;
        if (out_major_src)
          for (int co = 0; co < cout; ++co) dst[co] = s.w[((size_t)co * s.cin + ci) * s.taps + tap];
        else
          for (int co = 0; co < cout; ++co) dst[co] = s.w[(size_t)ci * cout + co];
      }
    kbase += s.taps * s.cin;
  }
  const bool f16 = act_dtype(e.cfg) == DT_F16;
  if (!f16) {
    cw.w_direct = upload(e, kd.data(), kd.size() * 4);
    if (e.cfg.mode == SGMSE_B200_MODE_TF32_TC && cout % 64 == 0 && ktot % 32 == 0) {
      // [Cout][ktot] TF32 values (round to nearest, ties away); no identity tail: the residual stays out of the TF32
      // operands and is added in fp32 by the epilogue
      std::vector<float> ht((size_t)cout * ktot);
      for (int k = 0; k < ktot; ++k)
        for (int co = 0; co < cout; ++co) ht[(size_t)co * ktot + k] = tf32_rna(kd[(size_t)k * cout + co]);
      cw.w_tc = upload(e, ht.data(), ht.size() * 4);
      cw.w_tc_ld = ktot;
    }
  } else {
    std::vector<__half> hd(kd.size());
    for (size_t i = 0; i < kd.size(); ++i) hd[i] = __float2half_rn(kd[i]);
    cw.w_direct = upload(e, hd.data(), hd.size() * 2);
    if (e.cfg.mode == SGMSE_B200_MODE_FP16_TC && cout % 64 == 0 && ktot % 64 == 0) {
      // [Cout][ld]; with `identity_tail` an extra Cout x Cout identity block follows the real K columns so that the
      // tensor-core kernel can take the residual `x` as one more 1x1 K segment (acc += x * I, exact in fp32)
      // instead of re-reading it in the epilogue.
      const int ld = ktot + (identity_tail ? cout : 0);
      std::vector<__half> ht((size_t)cout * ld, __float2half_rn(0.f));
      for (int k = 0; k < ktot; ++k)
        for (int co = 0; co < cout; ++co) ht[(size_t)co * ld + k] = hd[(size_t)k * cout + co];
      if (identity_tail)
        for (int co = 0; co < cout; ++co) ht[(size_t)co * ld + ktot + co] = __float2half_rn(1.f);
      cw.w_tc = upload(e, ht.data(), ht.size() * 2);
      cw.w_tc_ld = ld;
      cw.identity_tail = identity_tail;
    }
  }
}

void ensure_lanes(Engine& e, int want);
void clear_graphs(Engine& e);

void free_ode(Engine& e) {
  OdeBuffers& o = e.ode;
  cudaFree(o.y); cudaFree(o.y_new); cudaFree(o.stage); cudaFree(o.partial);
  for (int i = 0; i < 7; ++i) cudaFree(o.k[i]);
  if (o.partial_host) cudaFreeHost(o.partial_host);
  cudaFree(o.gpartial); cudaFree(o.rows_scale); cudaFree(o.raw);
  if (o.gpartial_host) cudaFreeHost(o.gpartial_host);
  o = OdeBuffers{};
}

void free_workspace(Engine& e) {
  for (auto& g : e.graphs) cudaGraphExecDestroy(g.second.exec);
  e.graphs.clear();
  for (auto& g : e.fwd_graphs) cudaGraphExecDestroy(g.second.exec);
  e.fwd_graphs.clear();
  for (auto& g : e.fwd_rows_graphs) cudaGraphExecDestroy(g.second.exec);
  e.fwd_rows_graphs.clear();
  free_ode(e);
  for (auto& p : e.fft_plans) cufftDestroy(p.second);
  e.fft_plans.clear();
  cudaFree(e.arena.base); e.arena = Arena{};
  cudaFree(e.state); cudaFree(e.xmean); cudaFree(e.temb_table); cudaFree(e.temb_scratch); cudaFree(e.t_dev);
  cudaFree(e.coef_dev); cudaFree(e.rng_dev); cudaFree(e.lv_scratch);
  e.state = nullptr; e.xmean = nullptr; e.temb_table = nullptr; e.temb_scratch = nullptr; e.t_dev = nullptr;
  e.coef_dev = nullptr; e.rng_dev = nullptr; e.lv_scratch = nullptr; e.dbg_flag = nullptr;
  e.persist_px = 0; e.persist_rows = 0;
  for (int i = 0; i < 4; ++i) { cudaFree(e.stft_buf[i]); e.stft_buf[i] = nullptr; e.stft_cap[i] = 0; }
  if (e.own_stream) { cudaStreamDestroy(e.own_stream); e.own_stream = nullptr; }
  for (auto& c : e.conv_events) { cudaEventDestroy(c.start); cudaEventDestroy(c.stop); }
  e.conv_events.clear();
}

void free_weights(Engine& e) {
  if (!e.owns_weights) return;
  if (e.lanes.size() > 1) ensure_lanes(e, 1);   // shadow engines hold pointers into the weights being freed
  clear_graphs(e);                              // ... and so do the kernel arguments baked into captured graphs
  for (void* p : e.dev_allocs) cudaFree(p);
  e.dev_allocs.clear();
  if (e.blob_dev) { cudaFree(e.blob_dev); e.blob_dev = nullptr; }
  e.weights_bytes = 0;
  e.loaded = false;
}

void load_weights(Engine& e, const float* blob) {
  free_weights(e);
  if (!e.range_flag) {                        // fp16 range detector word (gn.cu), shared with the lanes created later
    CUDA_OK(cudaMalloc((void**)&e.range_flag, sizeof(unsigned int)));
    CUDA_OK(cudaMemset(e.range_flag, 0, sizeof(unsigned int)));
  }
  const sgmse_b200_config& c = e.cfg;
  CUDA_OK(cudaMalloc(&e.blob_dev, (size_t)e.weights_numel * 4));
  CUDA_OK(cudaMemcpy(e.blob_dev, blob, (size_t)e.weights_numel * 4, cudaMemcpyHostToDevice));
  e.weights_bytes += (size_t)e.weights_numel * 4;
  const int nf = c.nf, D = 4 * nf;
  {  // input conv [nf][4][3][3] -> [36][nf]
    std::vector<float> p((size_t)36 * nf);
    for (int co = 0; co < nf; ++co)
      for (int ci = 0; ci < 4; ++ci)
        for (int tap = 0; tap < 9; ++tap) p[(size_t)(tap * 4 + ci) * nf + co] = blob[e.inconv_w + ((size_t)co * 4 + ci) * 9 + tap];
    e.inconv_w_packed = (float*)upload(e, p.data(), p.size() * 4);
  }
  std::vector<float> dw((size_t)e.total_temb_c * D), db(e.total_temb_c);
  for (Layer& l : e.layers) {
    if (l.kind == LK_RES) {
      pack_conv(e, {{blob + l.conv0_w, l.cin, 9}}, l.cout, true, l.c0);
      std::vector<PackSrc> s1{{blob + l.conv1_w, l.cout, 9}};
      if (l.shortcut) s1.push_back({blob + l.conv2_w, l.cin, 1});
      pack_conv(e, s1, l.cout, true, l.c1, /*identity_tail=*/!l.shortcut);
      std::vector<float> b1(blob + l.conv1_b, blob + l.conv1_b + l.cout);
      if (l.shortcut) for (int i = 0; i < l.cout; ++i) b1[i] += blob[l.conv2_b + i];
      l.c1.bias = (float*)upload(e, b1.data(), b1.size() * 4);
      memcpy(dw.data() + (size_t)l.temb_off * D, blob + l.dense_w, (size_t)l.cout * D * 4);
      for (int i = 0; i < l.cout; ++i) db[l.temb_off + i] = blob[l.dense_b + i] + blob[l.conv0_b + i];
    } else if (l.kind == LK_ATTN) {
      const int C = l.cin;
      // q|k|v as one 1x1 conv with 3C outputs: NIN weights are [in][out] (layers.py:549)
      std::vector<float> wq((size_t)C * 3 * C), bq(3 * C);
      for (int j = 0; j < 3; ++j) {
        for (int ci = 0; ci < C; ++ci)
          for (int co = 0; co < C; ++co) wq[(size_t)ci * 3 * C + j * C + co] = blob[l.nin_w[j] + (size_t)ci * C + co];
        for (int co = 0; co < C; ++co) bq[j * C + co] = blob[l.nin_b[j] + co];
      }
      pack_conv(e, {{wq.data(), C, 1}}, 3 * C, false, l.c0);
      l.c0.bias = (float*)upload(e, bq.data(), bq.size() * 4);
      pack_conv(e, {{blob + l.nin_w[3], C, 1}}, C, false, l.c1, /*identity_tail=*/true);
      l.c1.bias = e.blob_dev + l.nin_b[3];
    } else if (l.kind == LK_COMBINE) {
      const int C = l.cout;
      std::vector<float> p((size_t)4 * C);
      for (int co = 0; co < C; ++co)
        for (int ci = 0; ci < 4; ++ci) p[(size_t)ci * C + co] = blob[l.conv0_w + (size_t)co * 4 + ci];
      l.small_w = (float*)upload(e, p.data(), p.size() * 4);
      l.small_b = e.blob_dev + l.conv0_b;
    } else {  // LK_OUTCONV: [4][C][3][3] -> [9*C][4]
      const int C = l.cin;
      std::vector<float> p((size_t)9 * C * 4);
      for (int o = 0; o < 4; ++o)
        for (int ci = 0; ci < C; ++ci)
          for (int tap = 0; tap < 9; ++tap) p[((size_t)tap * C + ci) * 4 + o] = blob[l.conv0_w + ((size_t)o * C + ci) * 9 + tap];
      l.small_w = (float*)upload(e, p.data(), p.size() * 4);
      for (int o = 0; o < 4; ++o) l.out_bias_host[o] = blob[l.conv0_b + o];
      if (C % 16 == 0) {
        // B fragments of mma.sync m16n8k16 (k x n = 16 x 8, the 4 outputs in columns 0..3): lane (g, t) holds
        // b0 = (k = 2t, 2t+1 ; n = g), b1 = (k = 2t+8, 2t+9 ; n = g)
        const int KS = C / 16;
        std::vector<uint2> fr((size_t)9 * KS * 32, make_uint2(0u, 0u));
        auto h2 = [](float lo, float hi) {
          const __half2 v = __floats2half2_rn(lo, hi);
          uint32_t u; memcpy(&u, &v, 4); return u;
        };
        for (int tap = 0; tap < 9; ++tap)
          for (int kk = 0; kk < KS; ++kk)
            for (int ln = 0; ln < 32; ++ln) {
              const int gg = ln >> 2, tt = ln & 3;
              if (gg >= 4) continue;
              const float* wp = &p[((size_t)tap * C + kk * 16 + 2 * tt) * 4 + gg];
              fr[((size_t)tap * KS + kk) * 32 + ln] = make_uint2(h2(wp[0], wp[4]), h2(wp[32], wp[36]));
            }
        l.small_wfrag = (uint2*)upload(e, fr.data(), fr.size() * sizeof(uint2));
      }
    }
  }
  e.dense_w_stacked = (float*)upload(e, dw.data(), dw.size() * 4);
  e.dense_b_stacked = (float*)upload(e, db.data(), db.size() * 4);
  for (int o = 0; o < 2; ++o) {
    for (int i = 0; i < 4; ++i) e.out_layer.w[o][i] = blob[e.outl_w + o * 4 + i];
    e.out_layer.b[o] = blob[e.outl_b + o];
  }
  e.out_layer.scale_after = c.backbone == SGMSE_B200_BACKBONE_NCSNPP_48K ? 1 : 0;
  e.out_layer.scale_by_sigma = c.scale_by_sigma;
  for (auto& g : e.graphs) cudaGraphExecDestroy(g.second.exec);
  e.graphs.clear();
  e.loaded = true;
}

// The same packed state as load_weights(), produced on the device from a blob that already lives there (pack.cu): no 262 MB
// device -> host copy, no host loops, no re-upload.  Used by sgmse_b200_load_weights_device, i.e. by every refresh() of an
// installed model (EMA swap at the start of a validation epoch).  Mirrors load_weights() statement by statement.
void* dev_alloc(Engine& e, size_t bytes) {
  void* d = nullptr;
  CUDA_OK(cudaMalloc(&d, bytes));
  e.dev_allocs.push_back(d);
  e.weights_bytes += bytes;
  return d;
}
void pack_conv_dev(Engine& e, cudaStream_t st, const PackJob& job_in, ConvW& cw) {
  PackJob j = job_in;
  const bool f16 = act_dtype(e.cfg) == DT_F16;
  cw.ktot = j.ktot; cw.cout = j.cout;
  const size_t n = (size_t)j.ktot * j.cout;
  cw.w_direct = dev_alloc(e, n * (f16 ? 2 : 4));
  __half* ht = nullptr;
  j.ld = j.ktot;
  if (e.cfg.mode == SGMSE_B200_MODE_FP16_TC && j.cout % 64 == 0 && j.ktot % 64 == 0) {
    j.ld = j.ktot + (j.identity_tail ? j.cout : 0);
    ht = (__half*)dev_alloc(e, (size_t)j.cout * j.ld * 2);
    cw.w_tc = ht; cw.w_tc_ld = j.ld; cw.identity_tail = j.identity_tail != 0;
  }
  launch_pack_conv(st, e.blob_dev, j, cw.w_direct, f16, ht);
  if (e.cfg.mode == SGMSE_B200_MODE_TF32_TC && j.cout % 64 == 0 && j.ktot % 32 == 0) {   // as pack_conv: no identity tail
    cw.w_tc = dev_alloc(e, n * 4);
    cw.w_tc_ld = j.ktot;
    launch_pack_tc_tf32(st, (const float*)cw.w_direct, j.ktot, j.cout, j.ktot, (float*)cw.w_tc);
  }
}
PackJob conv_job(std::initializer_list<PackSeg> segs, int cout, int mode, bool identity_tail) {
  PackJob j{};
  int kb = 0;
  for (const PackSeg& sg : segs) {
    j.seg[j.nseg] = sg;
    j.seg[j.nseg].kbase = kb;
    kb += sg.taps * sg.cin;
    ++j.nseg;
  }
  j.cout = cout; j.ktot = kb; j.mode = mode; j.identity_tail = identity_tail ? 1 : 0;
  return j;
}

void load_weights_device(Engine& e, const float* blob_src, cudaStream_t st) {
  free_weights(e);
  if (!e.range_flag) {
    CUDA_OK(cudaMalloc((void**)&e.range_flag, sizeof(unsigned int)));
    CUDA_OK(cudaMemset(e.range_flag, 0, sizeof(unsigned int)));
  }
  const sgmse_b200_config& c = e.cfg;
  CUDA_OK(cudaMalloc(&e.blob_dev, (size_t)e.weights_numel * 4));
  CUDA_OK(cudaMemcpyAsync(e.blob_dev, blob_src, (size_t)e.weights_numel * 4, cudaMemcpyDeviceToDevice, st));
  e.weights_bytes += (size_t)e.weights_numel * 4;
  const float* blob = e.blob_dev;
  const int nf = c.nf, D = 4 * nf;
  e.inconv_w_packed = (float*)dev_alloc(e, (size_t)36 * nf * 4);
  launch_pack_inconv(st, blob + e.inconv_w, nf, e.inconv_w_packed);
  e.dense_w_stacked = (float*)dev_alloc(e, (size_t)e.total_temb_c * D * 4);
  e.dense_b_stacked = (float*)dev_alloc(e, (size_t)e.total_temb_c * 4);
  std::vector<std::pair<Layer*, long long>> out_bias;          // host copies of the 4-channel output biases (kernel arguments)
  for (Layer& l : e.layers) {
    if (l.kind == LK_RES) {
      pack_conv_dev(e, st, conv_job({{l.conv0_w, l.cin, 9, 0}}, l.cout, 0, false), l.c0);
      if (l.shortcut) pack_conv_dev(e, st, conv_job({{l.conv1_w, l.cout, 9, 0}, {l.conv2_w, l.cin, 1, 0}}, l.cout, 0, false), l.c1);
      else pack_conv_dev(e, st, conv_job({{l.conv1_w, l.cout, 9, 0}}, l.cout, 0, /*identity_tail=*/true), l.c1);
      l.c1.bias = (float*)dev_alloc(e, (size_t)l.cout * 4);
      launch_add_vec(st, blob + l.conv1_b, l.shortcut ? blob + l.conv2_b : nullptr, l.c1.bias, l.cout);
      CUDA_OK(cudaMemcpyAsync(e.dense_w_stacked + (size_t)l.temb_off * D, blob + l.dense_w, (size_t)l.cout * D * 4, cudaMemcpyDeviceToDevice, st));
      launch_add_vec(st, blob + l.dense_b, blob + l.conv0_b, e.dense_b_stacked + l.temb_off, l.cout);
    } else if (l.kind == LK_ATTN) {
      const int C = l.cin;
      PackJob q{};
      q.nseg = 3; q.cout = 3 * C; q.ktot = C; q.mode = 2; q.identity_tail = 0;
      for (int jx = 0; jx < 3; ++jx) q.seg[jx] = PackSeg{l.nin_w[jx], C, 1, 0};
      pack_conv_dev(e, st, q, l.c0);
      l.c0.bias = (float*)dev_alloc(e, (size_t)3 * C * 4);
      for (int jx = 0; jx < 3; ++jx)
        CUDA_OK(cudaMemcpyAsync(l.c0.bias + jx * C, blob + l.nin_b[jx], (size_t)C * 4, cudaMemcpyDeviceToDevice, st));
      pack_conv_dev(e, st, conv_job({{l.nin_w[3], C, 1, 0}}, C, 1, /*identity_tail=*/true), l.c1);
      l.c1.bias = e.blob_dev + l.nin_b[3];
    } else if (l.kind == LK_COMBINE) {
      const int C = l.cout;
      l.small_w = (float*)dev_alloc(e, (size_t)4 * C * 4);
      launch_pack_combine(st, blob + l.conv0_w, C, l.small_w);
      l.small_b = e.blob_dev + l.conv0_b;
    } else {  // LK_OUTCONV
      const int C = l.cin;
      l.small_w = (float*)dev_alloc(e, (size_t)9 * C * 4 * 4);
      l.small_wfrag = C % 16 == 0 ? (uint2*)dev_alloc(e, (size_t)9 * (C / 16) * 32 * sizeof(uint2)) : nullptr;
      launch_pack_outconv(st, blob + l.conv0_w, C, l.small_w, l.small_wfrag);
      out_bias.push_back({&l, l.conv0_b});
    }
  }
  // the few scalars the launch sequence passes by value
  for (auto& ob : out_bias) CUDA_OK(cudaMemcpyAsync(ob.first->out_bias_host, blob + ob.second, 4 * sizeof(float), cudaMemcpyDeviceToHost, st));
  float ol[10];
  CUDA_OK(cudaMemcpyAsync(ol, blob + e.outl_w, 8 * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaMemcpyAsync(ol + 8, blob + e.outl_b, 2 * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  for (int o = 0; o < 2; ++o) {
    for (int i = 0; i < 4; ++i) e.out_layer.w[o][i] = ol[o * 4 + i];
    e.out_layer.b[o] = ol[8 + o];
  }
  e.out_layer.scale_after = c.backbone == SGMSE_B200_BACKBONE_NCSNPP_48K ? 1 : 0;
  e.out_layer.scale_by_sigma = c.scale_by_sigma;
  for (auto& g : e.graphs) cudaGraphExecDestroy(g.second.exec);
  e.graphs.clear();
  e.loaded = true;
}

TembWeights temb_weights(const Engine& e) {
  TembWeights w{};
  w.gfp_w = e.blob_dev + e.gfp_w;
  w.l1_w = e.blob_dev + e.lin1_w; w.l1_b = e.blob_dev + e.lin1_b;
  w.l2_w = e.blob_dev + e.lin2_w; w.l2_b = e.blob_dev + e.lin2_b;
  w.dense_w = e.dense_w_stacked; w.dense_b = e.dense_b_stacked;
  w.nf = e.cfg.nf; w.totalC = e.total_temb_c;
  return w;
}

// ------------------------------------------------------------------------------------------------
// forward pass
// ------------------------------------------------------------------------------------------------
const WsPlan& ensure_arena(Engine& e, int B, int F, int T);

struct Fwd {
  Engine& e;
  cudaStream_t st;
  const float* temb;     // table row(s) for this evaluation
  int temb_stride;       // 0: one row for all samples; totalC: one row per sample
  bool dry;
  DType dt;
  float in_scale = 1.f;  // c_in of the preconditioned forward: multiplies the (x, y) state inside the input conv
  // the input pyramid's source when it differs from `state` (state already scaled by c_in per sample), and its
  // per-sample c_in, applied after the first FIR-down as in_scale is (device, nullable)
  const float4* pyr_state = nullptr;
  const float* pyr_scale_rows = nullptr;

  TensorDesc act(int N, int H, int W, int C, bool stats) {
    TensorDesc t;
    t.N = N; t.H = H; t.W = W; t.C = C; t.dt = dt;
    // element offsets are 64-bit, but several kernels index pixels x channels of one tensor in 32 bits
    SG_CHECK(t.numel() < ((size_t)1 << 31), "a [%d, %d, %d, %d] activation has 2^31 elements or more: the batch or clip is "
             "too long for one forward (16 kHz: T < 32768 frames per utterance, 48 kHz: T < 10923)", N, C, H, W);
    t.p = e.arena.alloc(t.bytes());
    if (stats) t.stats = (float*)e.arena.alloc(t.stats_capacity_floats() * 4);
    return t;
  }
  float4* act4(int N, int H, int W) { return (float4*)e.arena.alloc((size_t)N * H * W * 16); }
  void tap(const std::string& name, const TensorDesc& t) {
    if (!e.record_taps) return;
    if (dry) { e.arena.keep(t.p, true); e.arena.keep(t.stats, true); }
    else e.taps[name] = t;
  }
  void tap4(const std::string& name, const float4* p, int N, int H, int W) {
    if (!e.record_taps) return;
    if (dry) e.arena.keep(p, true);
    else e.taps4[name] = {p, {N, 4, H, W}};
  }

  // Lifetimes (planning run): every launch site ends with step(...) naming each arena buffer the launch reads or
  // writes, so a buffer's last step is the launch of its last reader.  Run mode: counts the launch and, with
  // workspace_poison, fills the buffers that launch was the last reader of.
  void mark(const void* p) { e.arena.use(p); }
  void mark(const TensorDesc& t) { mark(t.p); mark(t.stats); }
  void mark(const TensorDesc* t) { if (t) mark(*t); }
  void mark(const ConvArgs& a) {
    for (int i = 0; i < a.nseg; ++i) mark(a.seg[i].src);
    mark(a.residual);
    mark((const void*)a.gn_ab);
    if (a.gn_has_cat) mark(a.gn_cat);
  }
  template <typename... A> void step(const A&... bufs) {
    if (dry) { (mark(bufs), ...); ++e.arena.step; return; }
    e.kernel_launches += 1; e.launches_this_forward += 1;
    if (e.workspace_poison)
      for (int b : e.arena.plan->ends[e.arena.step]) {
        const WsBuf& w = e.arena.plan->bufs[b];
        CUDA_OK(cudaMemsetAsync(e.arena.base + w.off, 0xFF, w.bytes, st));
      }
    ++e.arena.step;
  }

  void conv(const ConvArgs& a, TensorDesc& out, int cls) {
    if (dry) { step(a, out); return; }
    const bool want_tc = tc_mode(e.cfg) && ((e.tc_mask >> cls) & 1);
    const bool tc = a.gn_ab != nullptr || (want_tc && conv_tc_supported(a, out));
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    if (e.time_convs) {
      CUDA_OK(cudaEventCreate(&ev0)); CUDA_OK(cudaEventCreate(&ev1));
      CUDA_OK(cudaEventRecord(ev0, st));
    }
    if (tc) { launch_conv_tc(st, a, out, e.dbg_flag); ++e.tc_convs; }
    else { launch_conv_direct(st, a, out); ++e.direct_convs; }
    if (e.time_convs) {
      CUDA_OK(cudaEventRecord(ev1, st));
      const double flops = 2.0 * (double)out.N * out.H * out.W * out.C * a.ktot();
      const double bytes = (double)out.bytes() + (a.residual ? (double)out.bytes() : 0.0) +
                           [&] { double b = 0; for (int i = 0; i < a.nseg; ++i) b += (double)a.seg[i].src.bytes(); return b; }();
      e.conv_events.push_back(ConvTiming{ev0, ev1, flops, bytes, tc});
    }
    step(a, out);
  }

  // `plain_consumer`: the only reader of (a, b) is apply_plain below -- with the gn_self candidate it rebuilds the
  // coefficients itself and the finalize launch is skipped (the table is still allocated: same workspace either way)
  float2* gn(const TensorDesc& x0, const TensorDesc* x1, long long g_off, long long b_off, bool plain_consumer = false) {
    const int Ct = x0.C + (x1 ? x1->C : 0);
    // (a, b) as float2 [N][Ct]
    float2* ab = (float2*)e.arena.alloc((size_t)x0.N * Ct * sizeof(float2));
    const int groups = gn_groups(Ct);
    if (plain_consumer && gn_self_applies(x0, x1)) return ab;
    if (!dry) launch_gn_finalize(st, x0, x1, e.blob_dev + g_off, e.blob_dev + b_off, groups, ab, e.range_flag);
    step(x0, x1, ab);
    return ab;
  }
  // y = [silu](a x + b) without resampling: gn_apply_plain on the finalized table, or (gn_self) finalize + apply in one kernel
  void apply_plain(const TensorDesc& x0, const TensorDesc* x1, const float2* ab, long long g_off, long long b_off, bool silu,
                   TensorDesc& out) {
    if (!dry) {
      if (gn_self_applies(x0, x1))
        launch_gn_norm_apply(st, x0, x1, e.blob_dev + g_off, e.blob_dev + b_off, gn_groups(x0.C + (x1 ? x1->C : 0)), silu, out, e.range_flag);
      else
        launch_gn_apply(st, x0, x1, ab, silu, RS_NONE, out, nullptr);
    }
    step(x0, x1, ab, out);
  }

  TensorDesc resblock(const Layer& l, const TensorDesc& x0, const TensorDesc* x1) {
    const int N = x0.N, Ct = x0.C + (x1 ? x1->C : 0);
    SG_CHECK(Ct == l.cin, "resblock %d: expected %d input channels, got %d", l.idx, l.cin, Ct);
    const Resample rs = l.up ? RS_UP : (l.down ? RS_DOWN : RS_NONE);
    const int Ho = l.up ? x0.H * 2 : (l.down ? x0.H / 2 : x0.H);
    const int Wo = l.up ? x0.W * 2 : (l.down ? x0.W / 2 : x0.W);
    // Fused path (conv_tc, opt-in tc_variant 5): the 3x3 convs read the RAW tensor and apply GroupNorm+SiLU on the way into
    // shared memory, so the gn_apply pass and its buffer disappear -- but its producer evaluates GroupNorm+SiLU once per tap
    // (9x the activation work): the benchmark step takes 3.2x longer than with TMA-fed operands and separate gn_apply passes.
    const bool fuse_ok = e.cfg.mode == SGMSE_B200_MODE_FP16_TC && g_tc_variant == 5;
    const bool fuse0 = fuse_ok && ((e.tc_mask >> 8) & 1) && rs == RS_NONE && l.c0.w_tc && conv_tc_fuse_shape_ok(Ho, Wo, x0.C, x1 ? x1->C : 0, l.cout);
    const bool fuse1 = fuse_ok && ((e.tc_mask >> 9) & 1) && l.c1.w_tc && conv_tc_fuse_shape_ok(Ho, Wo, l.cout, 0, l.cout);
    float2* ab0 = gn(x0, x1, l.gn0_w, l.gn0_b, rs == RS_NONE && !fuse0);
    TensorDesc h0;
    TensorDesc xr;                                 // FIR-resampled raw input (up/down blocks)
    if (rs != RS_NONE) {
      SG_CHECK(!x1, "resampling resblock with concatenated input");
      h0 = act(N, Ho, Wo, Ct, false);
      xr = act(N, Ho, Wo, Ct, false);
      if (!dry) launch_gn_apply(st, x0, nullptr, ab0, true, rs, h0, &xr);
      step(x0, ab0, h0, xr);
    } else if (!fuse0) {
      h0 = act(N, Ho, Wo, Ct, false);
      apply_plain(x0, x1, ab0, l.gn0_w, l.gn0_b, true, h0);
    }
    TensorDesc h1 = act(N, Ho, Wo, l.cout, true);
    {
      ConvArgs a;
      a.nseg = 1; a.seg[0].taps = 9;
      if (fuse0) {
        a.seg[0].src = x0; a.gn_ab = ab0;
        if (x1) { a.gn_has_cat = true; a.gn_cat = *x1; }
      } else {
        a.seg[0].src = h0;
      }
      a.w_direct = l.c0.w_direct; a.w_tc = l.c0.w_tc; a.w_tc_ld = l.c0.w_tc_ld;
      a.temb = temb + l.temb_off; a.temb_stride = temb_stride;   // Conv_0.bias is folded into the table
      conv(a, h1, 0);
    }
    float2* ab1 = gn(h1, nullptr, l.gn1_w, l.gn1_b, !fuse1);
    TensorDesc h2;
    if (!fuse1) {
      h2 = act(N, Ho, Wo, l.cout, false);
      apply_plain(h1, nullptr, ab1, l.gn1_w, l.gn1_b, true, h2);
    }
    TensorDesc out = act(N, Ho, Wo, l.cout, true);
    {
      ConvArgs a;
      a.nseg = 1; a.seg[0].taps = 9;
      if (fuse1) {
        a.seg[0].src = h1; a.gn_ab = ab1;
      } else { a.seg[0].src = h2; }
      if (l.shortcut) {
        if (rs != RS_NONE) { a.seg[a.nseg].src = xr; a.seg[a.nseg++].taps = 1; }
        else {
          a.seg[a.nseg].src = x0; a.seg[a.nseg++].taps = 1;
          if (x1) { a.seg[a.nseg].src = *x1; a.seg[a.nseg++].taps = 1; }
        }
      } else {
        a.residual = &x0;
      }
      a.w_direct = l.c1.w_direct; a.w_tc = l.c1.w_tc; a.w_tc_ld = l.c1.w_tc_ld; a.tc_identity_tail = l.c1.identity_tail;
      a.bias = l.c1.bias; a.scale = INV_SQRT2;
      conv(a, out, 1);
    }
    tap("m" + std::to_string(l.idx), out);
    return out;
  }

  TensorDesc attn(const Layer& l, const TensorDesc& x) {
    const int C = l.cin;
    SG_CHECK(x.C == C, "attention %d: channel mismatch", l.idx);
    float2* ab = gn(x, nullptr, l.gn0_w, l.gn0_b, true);
    TensorDesc hn = act(x.N, x.H, x.W, C, false);
    apply_plain(x, nullptr, ab, l.gn0_w, l.gn0_b, false, hn);
    TensorDesc qkv = act(x.N, x.H, x.W, 3 * C, false);
    {
      ConvArgs a;
      a.nseg = 1; a.seg[0].src = hn; a.seg[0].taps = 1;
      a.w_direct = l.c0.w_direct; a.w_tc = l.c0.w_tc; a.w_tc_ld = l.c0.w_tc_ld; a.bias = l.c0.bias;
      conv(a, qkv, 2);
    }
    TensorDesc av = act(x.N, x.H, x.W, C, false);
    if (!dry) launch_attention(st, qkv, av);
    step(qkv, av);
    TensorDesc out = act(x.N, x.H, x.W, C, true);
    {
      ConvArgs a;
      a.nseg = 1; a.seg[0].src = av; a.seg[0].taps = 1;
      a.w_direct = l.c1.w_direct; a.w_tc = l.c1.w_tc; a.w_tc_ld = l.c1.w_tc_ld; a.tc_identity_tail = l.c1.identity_tail;
      a.bias = l.c1.bias;
      a.residual = &x; a.scale = INV_SQRT2;
      conv(a, out, 3);
    }
    tap("m" + std::to_string(l.idx), out);
    return out;
  }

  const float4* outconv(const Layer& l, const TensorDesc& h, const float4* addend) {
    float2* ab = gn(h, nullptr, l.gn0_w, l.gn0_b, !out_conv_fuses_gn(h));
    if (out_conv_fuses_gn(h)) {                    // GroupNorm-apply + SiLU happen while the conv stages its tile
      float4* out = act4(h.N, h.H, h.W);
      if (!dry) launch_out_conv(st, h, l.small_w, l.out_bias_host, addend, out, ab, l.small_wfrag);
      step(h, ab, addend, out);
      return out;
    }
    TensorDesc a = act(h.N, h.H, h.W, h.C, false);
    apply_plain(h, nullptr, ab, l.gn0_w, l.gn0_b, true, a);
    float4* out = act4(h.N, h.H, h.W);
    if (!dry) launch_out_conv(st, a, l.small_w, l.out_bias_host, addend, out, nullptr, l.small_wfrag);
    step(a, addend, out);
    return out;
  }

  // returns the 4-channel tensor that feeds `/t` + output_layer
  const float4* run(const float4* state, int B, int H, int W) {
    const sgmse_b200_config& c = e.cfg;
    const int L = c.num_levels;
    SG_CHECK(H % (1 << (L - 1)) == 0 && W % (1 << (L - 1)) == 0, "F=%d, T=%d must be multiples of %d", H, W, 1 << (L - 1));
    if (c.num_attn_resolutions > 0 && c.backbone != SGMSE_B200_BACKBONE_NCSNPP_48K)
      SG_CHECK(H == c.image_size, "ncsnpp places attention for F == image_size == %d (got F=%d), see ncsnpp.py:84,308", c.image_size, H);
    if (dry) e.arena.begin(nullptr);
    else e.arena.begin(&ensure_arena(e, B, H, W));
    e.launches_this_forward = 0;
    e.tc_convs = e.direct_convs = 0;
    if (e.record_taps && !dry) { e.taps.clear(); e.taps4.clear(); }
    size_t it = 0;
    auto next = [&](LayerKind k) -> const Layer& {
      SG_CHECK(it < e.layers.size() && e.layers[it].kind == k, "internal: layer sequence mismatch at %zu", it);
      return e.layers[it++];
    };
    auto next_is = [&](LayerKind k) { return it < e.layers.size() && e.layers[it].kind == k; };

    std::vector<TensorDesc> hs;
    {
      TensorDesc h0 = act(B, H, W, c.nf, true);
      if (!dry) launch_input_conv(st, state, B, H, W, e.inconv_w_packed, e.blob_dev + e.inconv_b, h0, in_scale, c.not_centered != 0);
      step(h0);
      tap("in_conv", h0);
      hs.push_back(h0);
    }
    const float4* pyr_in = pyr_state ? pyr_state : state;
    const float4* const pyr0 = pyr_in;
    int ph = H, pw = W;
    for (int lvl = 0; lvl < L; ++lvl) {
      for (int b = 0; b < c.num_res_blocks; ++b) {
        TensorDesc h = resblock(next(LK_RES), hs.back(), nullptr);
        if (next_is(LK_ATTN)) h = attn(next(LK_ATTN), h);
        hs.push_back(h);
      }
      if (lvl != L - 1) {
        TensorDesc h = resblock(next(LK_RES), hs.back(), nullptr);
        if (c.progressive_input_skip) {
          const Layer& l = next(LK_COMBINE);
          float4* pd = act4(B, ph / 2, pw / 2);
          // the input pyramid starts at the network input c_in * (x, y) (ncsnpp.py:293-296), or 2 (x, y) - 1 when not centered
          // (ncsnpp.py:288-290): the first level carries c_in and the mapping
          if (!dry)
            launch_fir4(st, pyr_in, B, ph, pw, RS_DOWN, pd, pyr_in == pyr0 ? in_scale : 1.f, pyr_in == pyr0 ? pyr_scale_rows : nullptr,
                        pyr_in == pyr0 && c.not_centered != 0);
          step(pyr_in, pd);
          pyr_in = pd; ph /= 2; pw /= 2;
          TensorDesc o = act(B, h.H, h.W, h.C, true);
          if (!dry) launch_combine(st, pyr_in, l.small_w, l.small_b, h, o);
          step(pyr_in, h, o);
          tap("m" + std::to_string(l.idx), o);
          h = o;
        }
        hs.push_back(h);
      }
    }
    TensorDesc h = hs.back();
    h = resblock(next(LK_RES), h, nullptr);
    h = attn(next(LK_ATTN), h);
    h = resblock(next(LK_RES), h, nullptr);

    const float4* pyramid = nullptr;
    int qh = 0, qw = 0;
    for (int lvl = L - 1; lvl >= 0; --lvl) {
      for (int b = 0; b < c.num_res_blocks + 1; ++b) {
        TensorDesc skip = hs.back();
        hs.pop_back();
        h = resblock(next(LK_RES), h, &skip);
      }
      if (next_is(LK_ATTN)) h = attn(next(LK_ATTN), h);
      if (c.progressive_output_skip) {
        const Layer& l = next(LK_OUTCONV);
        const float4* add = nullptr;
        if (pyramid) {
          float4* up = act4(B, qh * 2, qw * 2);
          if (!dry) launch_fir4(st, pyramid, B, qh, qw, RS_UP, up);
          step(pyramid, up);
          add = up;
        }
        pyramid = outconv(l, h, add);
        qh = h.H; qw = h.W;
        tap4("pyr" + std::to_string(lvl), pyramid, B, qh, qw);
      }
      if (lvl != 0) h = resblock(next(LK_RES), h, nullptr);
    }
    SG_CHECK(hs.empty(), "internal: skip stack not empty after the up path");
    if (!c.progressive_output_skip) {
      pyramid = outconv(next(LK_OUTCONV), h, nullptr);
      tap4("pyr0", pyramid, B, h.H, h.W);
    }
    SG_CHECK(it == e.layers.size(), "internal: %zu of %zu layers consumed", it, e.layers.size());
    if (dry) e.arena.keep(pyramid, false);   // read by the output layer / sampler update after the forward
    else SG_CHECK(e.arena.step == e.arena.plan->steps && e.arena.next == e.arena.plan->bufs.size(),
                  "internal: the forward departed from its workspace plan");
    return pyramid;
  }
};

// Interval packing of one forward's buffers (planning run in e.arena.rec).  Largest buffers first (ties: earlier
// allocation first), each at the lowest 256-B aligned offset that overlaps no placed buffer whose lifetime
// intersects its own.  Deterministic: the layout depends on the shapes and the launch sequence alone.
//
// Reuse is safe because every launch of one forward is enqueued on one stream (each lane has its own arena and
// stream): a buffer placed over a dead one is first written by a launch that follows, in stream order, the dead
// buffer's last reader.  With programmatic dependent launch every kernel waits for its predecessor's completion
// before its first global access (common.cuh), which keeps that order.
WsPlan pack_workspace(std::vector<WsBuf> bufs, int steps) {
  WsPlan p;
  p.steps = steps;
  p.ends.assign(steps, {});
  for (WsBuf& b : bufs) {
    p.bump = ((p.bump + 255) & ~(size_t)255) + b.bytes;
    if (b.last == INT_MAX) b.last = steps;
  }
  std::vector<int> order(bufs.size());
  for (size_t i = 0; i < order.size(); ++i) order[i] = (int)i;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return bufs[a].bytes > bufs[b].bytes; });
  std::vector<int> placed, conflicts;
  for (int i : order) {
    WsBuf& b = bufs[i];
    conflicts.clear();
    for (int j : placed)
      if (bufs[j].first <= b.last && b.first <= bufs[j].last) conflicts.push_back(j);
    std::sort(conflicts.begin(), conflicts.end(), [&](int x, int y) { return bufs[x].off < bufs[y].off; });
    size_t off = 0;
    for (int j : conflicts) {
      if (off + b.bytes <= bufs[j].off) break;
      off = std::max(off, (bufs[j].off + bufs[j].bytes + 255) & ~(size_t)255);
    }
    b.off = off;
    p.bytes = std::max(p.bytes, off + b.bytes);
    placed.push_back(i);
    if (b.last < steps) p.ends[b.last].push_back(i);
  }
  p.bytes += 4096;
  p.bufs = std::move(bufs);
  return p;
}

// The workspace layout of one forward of (B, F, T) with the engine's current options: planned once by a host-only
// run of the launch sequence, then cached.
const WsPlan& workspace_plan(Engine& e, int B, int F, int T) {
  const auto key = std::make_tuple(B, F, T, e.record_taps);
  auto it = e.ws_plans.find(key);
  if (it != e.ws_plans.end()) return it->second;
  Arena saved = e.arena;
  e.arena = Arena{};
  e.arena.dry = true;
  Fwd f{e, nullptr, nullptr, 0, true, act_dtype(e.cfg)};
  try { f.run(nullptr, B, F, T); } catch (...) { e.arena = saved; throw; }
  WsPlan p = pack_workspace(std::move(e.arena.rec), e.arena.step);
  e.arena = saved;
  return e.ws_plans.emplace(key, std::move(p)).first->second;
}

void clear_graphs(Engine& e) {
  for (auto& g : e.graphs) cudaGraphExecDestroy(g.second.exec);
  e.graphs.clear();
  for (auto& g : e.fwd_graphs) cudaGraphExecDestroy(g.second.exec);
  e.fwd_graphs.clear();
  for (auto& g : e.fwd_rows_graphs) cudaGraphExecDestroy(g.second.exec);
  e.fwd_rows_graphs.clear();
  ++e.generation;
}

void free_workspace(Engine& e);

// Shadow engines for concurrent lanes (see engine.h): same weights, private workspace.
void ensure_lanes(Engine& e, int want) {
  if (e.lanes.empty()) { e.lanes.push_back(&e); e.lane_streams.push_back(nullptr); }
  if ((int)e.lanes.size() > want) {          // shrink
    CUDA_OK(cudaDeviceSynchronize());
    clear_graphs(e);
    while ((int)e.lanes.size() > want) {
      Engine* l = e.lanes.back();
      free_workspace(*l);
      delete l;
      cudaStreamDestroy(e.lane_streams.back());
      e.lanes.pop_back(); e.lane_streams.pop_back();
    }
  }
  while ((int)e.lanes.size() < want) {
    Engine* l = new Engine(e);               // copies config, layer table and (shared) weight pointers
    l->owns_weights = false;
    l->dev_allocs.clear();
    l->arena = Arena{};
    l->state = nullptr; l->xmean = nullptr; l->temb_table = nullptr; l->temb_scratch = nullptr; l->t_dev = nullptr;
    l->coef_dev = nullptr; l->rng_dev = nullptr; l->lv_scratch = nullptr; l->dbg_flag = nullptr;
    l->persist_px = 0; l->persist_rows = 0;
    l->graphs.clear(); l->fwd_graphs.clear(); l->fwd_rows_graphs.clear(); l->fft_plans.clear();
    l->ode = OdeBuffers{};
    for (int i = 0; i < 4; ++i) { l->stft_buf[i] = nullptr; l->stft_cap[i] = 0; }
    l->own_stream = nullptr;
    l->lanes.clear(); l->lane_streams.clear(); l->lane_events.clear();
    l->taps.clear(); l->taps4.clear(); l->conv_events.clear();
    l->record_taps = false; l->time_convs = false;
    l->kernel_launches = 0; l->graph_launches = 0; l->generation = 0;
    cudaStream_t s = nullptr;
    CUDA_OK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    e.lanes.push_back(l);
    e.lane_streams.push_back(s);
  }
  while ((int)e.lane_events.size() < want + 1) {
    cudaEvent_t ev;
    CUDA_OK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    e.lane_events.push_back(ev);
  }
}

// Workspace for one forward pass of (B, F, T).  Every forward of a shape follows the same cached plan, so buffer
// addresses (and with them captured graphs) stay valid as long as the arena itself is not re-allocated.
const WsPlan& ensure_arena(Engine& e, int B, int F, int T) {
  const WsPlan& p = workspace_plan(e, B, F, T);
  if (p.bytes > e.arena.cap) {
    clear_graphs(e);
    if (e.arena.base) { CUDA_OK(cudaDeviceSynchronize()); cudaFree(e.arena.base); e.arena.base = nullptr; e.arena.cap = 0; }
    CUDA_OK(cudaMalloc((void**)&e.arena.base, p.bytes));
    e.arena.cap = p.bytes;
  }
  e.arena.dry = false;
  return p;
}

template <typename T>
void ensure_buf(T*& p, size_t& cap_elems, size_t need_elems) {
  if (need_elems <= cap_elems) return;
  if (p) { CUDA_OK(cudaDeviceSynchronize()); cudaFree(p); p = nullptr; }
  CUDA_OK(cudaMalloc((void**)&p, need_elems * sizeof(T)));
  cap_elems = need_elems;
}

void ensure_persistent(Engine& e, size_t px, int rows) {
  if (px > e.persist_px) {
    if (e.state) { CUDA_OK(cudaDeviceSynchronize()); cudaFree(e.state); cudaFree(e.xmean); }
    CUDA_OK(cudaMalloc((void**)&e.state, px * sizeof(float4)));
    CUDA_OK(cudaMalloc((void**)&e.xmean, px * sizeof(float2)));
    e.persist_px = px;
    clear_graphs(e);
  }
  if (rows > e.persist_rows) {
    if (e.temb_table) { CUDA_OK(cudaDeviceSynchronize()); cudaFree(e.temb_table); cudaFree(e.temb_scratch); cudaFree(e.t_dev); cudaFree(e.coef_dev); }
    CUDA_OK(cudaMalloc((void**)&e.temb_table, (size_t)rows * e.total_temb_c * 4));
    CUDA_OK(cudaMalloc((void**)&e.temb_scratch, (size_t)rows * 4 * e.cfg.nf * 4));
    CUDA_OK(cudaMalloc((void**)&e.t_dev, (size_t)rows * 4));
    CUDA_OK(cudaMalloc((void**)&e.coef_dev, (size_t)rows * 4 * sizeof(UpdateCoef)));
    e.persist_rows = rows;
    clear_graphs(e);
  }
  if (!e.rng_dev) {
    CUDA_OK(cudaMalloc((void**)&e.rng_dev, sizeof(RngParams)));
    CUDA_OK(cudaMalloc((void**)&e.lv_scratch, (size_t)std::max(e.cfg.max_batch, 1) * 64 * 2 * 4));
    if (!g_wait_code_host) {
      int* h = nullptr;
      CUDA_OK(cudaHostAlloc((void**)&h, 4, cudaHostAllocMapped));
      *h = 0;
      g_wait_code_host = h;
    }
    e.dbg_flag = const_cast<int*>(g_wait_code_host);      // one process-wide word (UVA: same pointer on the device)
  }
}

__global__ void extract_x_kernel(const float4* __restrict__ state, size_t total, float2* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) { const float4 s = state[i]; out[i] = make_float2(s.x, s.y); }
}
__global__ void nhwc_to_nchw_kernel(const void* __restrict__ src, int is_half, int C, int HW, size_t total, float* __restrict__ dst) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;   // index into NCHW output
  if (i >= total) return;
  const int p = (int)(i % HW);
  const int c = (int)((i / HW) % C);
  const size_t n = i / ((size_t)HW * C);
  const size_t s = (n * HW + p) * C + c;
  dst[i] = is_half ? __half2float(((const __half*)src)[s]) : ((const float*)src)[s];
}

// ------------------------------------------------------------------------------------------------
// network evaluation with per-sample times (backbone contract / score)
// ------------------------------------------------------------------------------------------------
void dnn_forward(Engine& e, const float2* x, const float2* y, const float* t, float2* out, int B, int F, int T,
                 bool negate, cudaStream_t st) {
  SG_CHECK(e.loaded, "weights not loaded");
  const int mb = std::max(1, e.cfg.max_batch);
  ensure_arena(e, std::min(B, mb), F, T);
  ensure_persistent(e, (size_t)std::min(B, mb) * F * T, std::max(mb, 64));
  const size_t px1 = (size_t)F * T;
  for (int b0 = 0; b0 < B; b0 += mb) {
    const int Bc = std::min(mb, B - b0);
    launch_pack_state(st, x + b0 * px1, y + b0 * px1, Bc, F, T, e.state); ++e.kernel_launches;
    launch_temb(st, temb_weights(e), t + b0, Bc, e.temb_scratch, e.temb_table); e.kernel_launches += 2;
    Fwd f{e, st, e.temb_table, e.total_temb_c, false, act_dtype(e.cfg)};
    const float4* p = f.run(e.state, Bc, F, T);
    launch_out_layer(st, p, Bc, F, T, e.out_layer, t + b0, out + b0 * px1, negate); ++e.kernel_launches;
  }
}

// ------------------------------------------------------------------------------------------------
// predictor-corrector sampler
// ------------------------------------------------------------------------------------------------
std::vector<float> linspace_f32(float start, float end, int steps) {
  // torch.linspace (CPU, fp32): step = (end-start)/(steps-1); first half from start, second half from end
  std::vector<float> v(steps);
  if (steps == 1) { v[0] = start; return v; }
  const float step = (end - start) / (float)(steps - 1);
  const int half = steps / 2;
  for (int i = 0; i < steps; ++i) v[i] = i < half ? start + step * (float)i : end - step * (float)(steps - 1 - i);
  return v;
}

int noise_draws(const sgmse_b200_sampler& s) {
  if (s.kind == SGMSE_B200_SAMPLER_SB_SDE) return s.N;   // one draw per step, the last one with weight 0 (sampling/__init__.py:176-179)
  if (s.kind == SGMSE_B200_SAMPLER_SB_ODE) return 0;
  const int c = s.corrector != SGMSE_B200_CORR_NONE ? s.corrector_steps : 0;
  const int p = s.predictor != SGMSE_B200_PRED_NONE ? 1 : 0;
  return 1 + s.N * (c + p);
}

// ---- SDE scalars (double on the host; the reference evaluates them on fp32 tensors) ----
double ouve_std(const sgmse_b200_config& c, double t) {          // sdes.py:206-219
  const double th = c.theta, smin = c.sigma_min, ls = log((double)c.sigma_max / c.sigma_min);
  return sqrt(smin * smin * exp(-2 * th * t) * (exp(2 * (th + ls) * t) - 1) * ls / (th + ls));
}
struct SbSigmas { double sigma_t, sigma_T, sigma_bar; };           // alpha_t = alpha_T = 1 (sdes.py:277-278)
SbSigmas sb_sigmas(const sgmse_b200_config& c, double t) {         // sdes.py:276-287
  const double k = c.sb_k, logk2 = 2 * log(k);
  SbSigmas r;
  r.sigma_t = sqrt(c.sb_c * (pow(k, 2 * t) - 1.0) / logk2);
  r.sigma_T = sqrt(c.sb_c * (pow(k, 2.0) - 1.0) / logk2);
  r.sigma_bar = sqrt(r.sigma_T * r.sigma_T - r.sigma_t * r.sigma_t + c.sb_eps);
  return r;
}
double sde_std(const sgmse_b200_config& c, double t) {
  if (c.sde_kind == SGMSE_B200_SDE_OUVE) return ouve_std(c, t);
  const SbSigmas g = sb_sigmas(c, t);                              // sdes.py:298-302
  return g.sigma_bar * g.sigma_t / (g.sigma_T + c.sb_eps);
}
// ScoreModel.forward of the 'ncsnpp_v2' branch as  M(x_t, y, t) = a * x_t + b * dnn(c_in x_t, c_in y, t)  (model.py:283-341)
struct Precond { double c_in, a, b; };
Precond precond(const sgmse_b200_config& c, double t) {
  const double sig = sde_std(c, t), sd2 = (double)c.sigma_data * c.sigma_data;
  Precond p;
  p.c_in = c.c_in == SGMSE_B200_CIN_ONE ? 1.0 : 1.0 / sqrt(sig * sig + sd2);
  const double c_out = c.c_out == SGMSE_B200_COUT_ONE ? 1.0 : c.c_out == SGMSE_B200_COUT_SIGMA ? sig :
                       c.c_out == SGMSE_B200_COUT_INV_SIGMA ? 1.0 / sig : sig * c.sigma_data / sqrt(sd2 + sig * sig);
  const double c_skip = c.c_skip == SGMSE_B200_CSKIP_ZERO ? 0.0 : sd2 / (sig * sig + sd2);
  const double ns = c.network_scaling == SGMSE_B200_NETSCALE_INV_SIGMA ? 1.0 / sig :
                    c.network_scaling == SGMSE_B200_NETSCALE_INV_T ? 1.0 / t : 1.0;
  if (c.loss_type == SGMSE_B200_LOSS_DENOISER) { p.a = -1.0 / (sig * sig); p.b = ns / (sig * sig); }
  else { p.a = c_skip; p.b = c_out * ns; }
  return p;
}
bool is_v2(const Engine& e) { return e.cfg.backbone == SGMSE_B200_BACKBONE_NCSNPP_V2; }

struct SamplerTables {
  std::vector<float> ts;
  std::vector<UpdateCoef> coef;    // one per update, in execution order (langevin entries filled on device)
  // general path (SB samplers; every sampler on the preconditioned v2 model): x_mean = cx x + cF F + cy y, x = x_mean + cz z
  bool affine = false;
  std::vector<AffineCoef> acoef;   // one per update
  std::vector<float> in_scale;     // c_in(t_i), one per time step
  std::vector<float> sb_raw;       // SB kinds: (weight_prev, weight_estimate, weight_z | weight_prior_mean) per step, as the reference names them
};

SamplerTables make_tables(const Engine& e, const sgmse_b200_sampler& s) {
  // sdes.py:188-219, predictors.py:41-65, correctors.py:69-81, sampling/__init__.py:56-62
  SamplerTables tb;
  const sgmse_b200_config& c = e.cfg;
  if (s.kind != SGMSE_B200_SAMPLER_PC) {
    // Schroedinger-bridge samplers (sampling/__init__.py:145-249): N steps over linspace(T, eps, N+1)[1:]
    SG_CHECK(c.sde_kind == SGMSE_B200_SDE_SBVE, "the SB samplers need the 'sbve' SDE");
    SG_CHECK(is_v2(e), "the SB samplers are driven by ScoreModel.forward(x_t, y, t) of backbone 'ncsnpp_v2'");
    const std::vector<float> all = linspace_f32(1.0f, s.sb_eps, s.N + 1);
    tb.ts.assign(all.begin() + 1, all.end());
    tb.affine = true;
    SbSigmas prev = sb_sigmas(c, all[0]);
    const double eps = c.sb_eps;
    for (int i = 0; i < s.N; ++i) {
      const double t = tb.ts[i];
      const SbSigmas cur = sb_sigmas(c, t);
      double w_prev, w_est, w_third;
      if (s.kind == SGMSE_B200_SAMPLER_SB_SDE) {                     // :165-179
        w_prev = cur.sigma_t * cur.sigma_t / (prev.sigma_t * prev.sigma_t + eps);
        const double tmp = 1 - cur.sigma_t * cur.sigma_t / (prev.sigma_t * prev.sigma_t + eps);
        w_est = tmp;
        w_third = i == s.N - 1 ? 0.0 : cur.sigma_t * sqrt(tmp);      // weight_z
      } else {                                                       // :211-231
        w_prev = cur.sigma_t * cur.sigma_bar / (prev.sigma_t * prev.sigma_bar + eps);
        w_est = 1.0 / (cur.sigma_T * cur.sigma_T + eps) *
                (cur.sigma_bar * cur.sigma_bar - prev.sigma_bar * cur.sigma_t * cur.sigma_bar / (prev.sigma_t + eps));
        w_third = 1.0 / (cur.sigma_T * cur.sigma_T + eps) *
                  (cur.sigma_t * cur.sigma_t - prev.sigma_t * cur.sigma_t * cur.sigma_bar / (prev.sigma_bar + eps));   // weight_prior_mean
      }
      tb.sb_raw.push_back((float)w_prev); tb.sb_raw.push_back((float)w_est); tb.sb_raw.push_back((float)w_third);
      const Precond pc = precond(c, t);
      tb.in_scale.push_back((float)pc.c_in);
      // x' = w_prev x + w_est (a x + b F) + [w_y y | w_z z]
      AffineCoef a;
      a.cx = (float)(w_prev + w_est * pc.a);
      a.cF = (float)(w_est * pc.b);
      a.cy = s.kind == SGMSE_B200_SAMPLER_SB_ODE ? (float)w_third : 0.f;
      a.cz = s.kind == SGMSE_B200_SAMPLER_SB_SDE ? (float)w_third : 0.f;
      tb.acoef.push_back(a);
      prev = cur;
    }
    return tb;
  }
  SG_CHECK(c.sde_kind == SGMSE_B200_SDE_OUVE, "the predictor-corrector sampler is implemented for the 'ouve' SDE");
  tb.ts = linspace_f32(1.0f, c.t_eps, s.N);
  const double th = c.theta, smin = c.sigma_min, smax = c.sigma_max, ls = log(smax / smin);
  const double pf = s.probability_flow ? 0.5 : 1.0;
  for (int i = 0; i < s.N; ++i) {
    const double t = tb.ts[i];
    const double std = sqrt(smin * smin * exp(-2 * th * t) * (exp(2 * (th + ls) * t) - 1) * ls / (th + ls));
    const double g = smin * pow(smax / smin, t) * sqrt(2 * ls);
    if (s.corrector != SGMSE_B200_CORR_NONE)
      for (int k = 0; k < s.corrector_steps; ++k) {
        const double eps = 2.0 * (s.snr * std) * (s.snr * std);
        tb.coef.push_back(UpdateCoef{0.f, (float)eps, (float)sqrt(2 * eps)});
      }
    if (s.predictor == SGMSE_B200_PRED_REVERSE_DIFFUSION) {
      const float dtf = i != s.N - 1 ? tb.ts[i] - tb.ts[i + 1] : tb.ts[s.N - 1];
      const double dt = dtf, G = g * sqrt(dt);
      tb.coef.push_back(UpdateCoef{(float)(-th * dt), (float)(G * G * pf), s.probability_flow ? 0.f : (float)G});
    } else if (s.predictor == SGMSE_B200_PRED_EULER_MARUYAMA) {
      // x + (theta (y-x) - g^2 score) * dt + g sqrt(-dt) z,  dt = -1/N   (predictors.py:46-52, as intended;
      // the reference's call site forwards `stepsize` into OUVESDE.sde() and raises TypeError)
      const double dt = -1.0 / s.N;
      tb.coef.push_back(UpdateCoef{(float)(th * dt), (float)(-g * g * pf * dt), s.probability_flow ? 0.f : (float)(g * sqrt(-dt))});
    }
  }
  if (is_v2(e)) {
    // the same updates driven by the preconditioned model: score = a x + b F  ->
    // x_mean = x + cy (y - x) + cs score = (1 - cy + cs a) x + cs b F + cy y
    SG_CHECK(s.corrector != SGMSE_B200_CORR_LANGEVIN, "the Langevin corrector (data-dependent step) is not available on 'ncsnpp_v2'");
    SG_CHECK(c.loss_type != SGMSE_B200_LOSS_DATA_PREDICTION, "the predictor-corrector sampler needs a score model (loss_type)");
    tb.affine = true;
    const int per_step = (int)tb.coef.size() / s.N;
    for (size_t u = 0; u < tb.coef.size(); ++u) {
      const int i = per_step ? (int)u / per_step : 0;
      const Precond pc = precond(c, tb.ts[i]);
      const UpdateCoef& k = tb.coef[u];
      tb.acoef.push_back(AffineCoef{(float)(1.0 - k.cy + k.cs * pc.a), (float)(k.cs * pc.b), k.cy, k.cz});
    }
    for (int i = 0; i < s.N; ++i) tb.in_scale.push_back((float)precond(c, tb.ts[i]).c_in);
  }
  return tb;
}

// One micro-batch.  y/out: [Bc][F*T] float2; noise: nullptr or base of [draws][Btot][F*T] with chunk offset applied.
void sample_chunk(Engine& e, const float2* y, int Bc, int F, int T, const sgmse_b200_sampler& s, const float2* noise,
                  size_t noise_draw_stride, float2* out, cudaStream_t st, bool inside_capture) {
  const SamplerTables tb = make_tables(e, s);
  const size_t px = (size_t)Bc * F * T;
  const RngParams* rng = e.rng_dev;
  auto nz = [&](int draw) { return noise ? noise + (size_t)draw * noise_draw_stride : nullptr; };
  const sgmse_b200_config& c = e.cfg;
  if (tb.affine) {
    // general update path: Schroedinger-bridge samplers, and the predictor-corrector sampler on the preconditioned
    // 'ncsnpp_v2' model.  Coefficient rows live in coef_dev (reinterpreted), one per update in execution order.
    const AffineCoef* ac = reinterpret_cast<const AffineCoef*>(e.coef_dev);
    launch_pack_state(st, y, y, Bc, F, T, e.state); ++e.kernel_launches;       // x = y (SB: sampling/__init__.py:150,193)
    int draw = 0, ci = 0;
    const bool pc = s.kind == SGMSE_B200_SAMPLER_PC;
    if (pc) {                                                                    // x = y + std(1) z (sdes.py:224-229)
      launch_prior(st, e.state, Bc, F, T, (float)ouve_std(c, 1.0), nz(draw), rng, draw); ++e.kernel_launches;
      ++draw;
    }
    Fwd f{e, st, nullptr, 0, false, act_dtype(e.cfg)};
    bool have_mean = false;
    for (int i = 0; i < s.N; ++i) {
      f.temb = e.temb_table + (size_t)i * e.total_temb_c;
      f.in_scale = tb.in_scale[i];
      const int ncorr = pc && s.corrector != SGMSE_B200_CORR_NONE ? s.corrector_steps : 0;
      const int npred = pc ? (s.predictor != SGMSE_B200_PRED_NONE ? 1 : 0) : 1;
      for (int u = 0; u < ncorr + npred; ++u) {
        const float4* p = f.run(e.state, Bc, F, T);
        const bool is_pred = u >= ncorr;
        const bool last = pc && is_pred && i == s.N - 1;
        const bool use_noise = pc || s.kind == SGMSE_B200_SAMPLER_SB_SDE;
        launch_affine_update(st, e.state, p, Bc, F, T, e.out_layer, ac + ci, use_noise ? nz(draw) : nullptr, rng, draw, use_noise,
                             (last && s.denoise) ? e.xmean : nullptr);
        ++e.kernel_launches; ++ci;
        if (use_noise) ++draw;
        have_mean = last && s.denoise;
      }
    }
    if (have_mean) {
      CUDA_OK(cudaMemcpyAsync(out, e.xmean, px * sizeof(float2), cudaMemcpyDeviceToDevice, st));
    } else {
      extract_x_kernel<<<(unsigned)((px + 255) / 256), 256, 0, st>>>(e.state, px, out);
      CUDA_OK(cudaGetLastError()); ++e.kernel_launches;
    }
    return;
  }
  const double th = c.theta, smin = c.sigma_min, smax = c.sigma_max, ls = log(smax / smin);
  const float std1 = (float)sqrt(smin * smin * exp(-2 * th) * (exp(2 * (th + ls)) - 1) * ls / (th + ls));

  launch_pack_state(st, y, y, Bc, F, T, e.state); ++e.kernel_launches;
  int draw = 0;
  launch_prior(st, e.state, Bc, F, T, std1, nz(draw), rng, draw); ++e.kernel_launches;
  ++draw;
  int ci = 0;
  bool have_mean = false;
  Fwd f{e, st, nullptr, 0, false, act_dtype(e.cfg)};
  for (int i = 0; i < s.N; ++i) {
    const float inv_t = 1.0f / tb.ts[i];
    f.temb = e.temb_table + (size_t)i * e.total_temb_c;
    if (s.corrector != SGMSE_B200_CORR_NONE)
      for (int k = 0; k < s.corrector_steps; ++k) {
        const float4* p = f.run(e.state, Bc, F, T);
        if (s.corrector == SGMSE_B200_CORR_LANGEVIN) {
          launch_langevin_coef(st, p, Bc, F, T, e.out_layer, inv_t, nz(draw), rng, draw, s.snr, e.lv_scratch, e.coef_dev + ci);
          e.kernel_launches += 2;
        }
        launch_pc_update(st, e.state, p, Bc, F, T, e.out_layer, nullptr, inv_t, e.coef_dev + ci, nz(draw), rng, draw, nullptr);
        ++e.kernel_launches; ++draw; ++ci;
        have_mean = false;
      }
    if (s.predictor != SGMSE_B200_PRED_NONE) {
      const float4* p = f.run(e.state, Bc, F, T);
      const bool last = i == s.N - 1;
      launch_pc_update(st, e.state, p, Bc, F, T, e.out_layer, nullptr, inv_t, e.coef_dev + ci, nz(draw), rng, draw,
                       (last && s.denoise) ? e.xmean : nullptr);
      ++e.kernel_launches; ++draw; ++ci;
      have_mean = last && s.denoise;
    }
  }
  if (have_mean) {
    CUDA_OK(cudaMemcpyAsync(out, e.xmean, px * sizeof(float2), cudaMemcpyDeviceToDevice, st));
  } else {
    // NonePredictor returns (x, x): x_mean == x  (predictors.py:75-76)
    extract_x_kernel<<<(unsigned)((px + 255) / 256), 256, 0, st>>>(e.state, px, out);
    CUDA_OK(cudaGetLastError()); ++e.kernel_launches;
  }
  (void)inside_capture;
}

void ensure_stft_buf(Engine& e, int slot, size_t bytes);

void prepare_tables(Engine& e, const sgmse_b200_sampler& s, cudaStream_t st) {
  const SamplerTables tb = make_tables(e, s);
  CUDA_OK(cudaMemcpyAsync(e.t_dev, tb.ts.data(), tb.ts.size() * 4, cudaMemcpyHostToDevice, st));
  if (tb.affine) {
    if (!tb.acoef.empty())
      CUDA_OK(cudaMemcpyAsync(e.coef_dev, tb.acoef.data(), tb.acoef.size() * sizeof(AffineCoef), cudaMemcpyHostToDevice, st));
  } else if (!tb.coef.empty())
    CUDA_OK(cudaMemcpyAsync(e.coef_dev, tb.coef.data(), tb.coef.size() * sizeof(UpdateCoef), cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaStreamSynchronize(st));   // tb is a temporary; keep the host buffers alive until copied
  launch_temb(st, temb_weights(e), e.t_dev, s.N, e.temb_scratch, e.temb_table); e.kernel_launches += 2;
}

void pc_sample(Engine& e, const float2* y, int B, int F, int T, const sgmse_b200_sampler& s, const float2* noise,
               float2* out, int* nfe, cudaStream_t st_in) {
  SG_CHECK(e.loaded, "weights not loaded");
  // stream capture is illegal on the legacy default stream: run on an engine-owned (blocking) stream instead
  cudaStream_t st = st_in;
  if (!st) {
    if (!e.own_stream) CUDA_OK(cudaStreamCreate(&e.own_stream));
    st = e.own_stream;
  }
  struct SyncOnExit { cudaStream_t s; bool on; ~SyncOnExit() { if (on) cudaStreamSynchronize(s); } } sync_guard{st, st_in == nullptr};
  SG_CHECK(s.N >= 1 && s.corrector_steps >= 0, "bad sampler settings");
  SG_CHECK(s.kind >= SGMSE_B200_SAMPLER_PC && s.kind <= SGMSE_B200_SAMPLER_SB_SDE, "Invalid type. Choose 'ode' or 'sde'.");
  SG_CHECK(s.predictor >= 0 && s.predictor <= 2, "Predictor with id %d unknown.", s.predictor);
  SG_CHECK(s.corrector >= 0 && s.corrector <= 2, "Corrector with id %d unknown.", s.corrector);
  const int mb = std::max(1, e.cfg.max_batch);
  const int csteps = s.corrector != SGMSE_B200_CORR_NONE ? s.corrector_steps : 0;
  const bool coupled = s.kind == SGMSE_B200_SAMPLER_PC && s.corrector == SGMSE_B200_CORR_LANGEVIN && csteps > 0;
  SG_CHECK(!coupled || B <= mb,
           "the Langevin corrector couples the utterances of a batch through batch-mean norms (correctors.py:50-52): B=%d "
           "must not exceed max_batch=%d (it would be sampled in independent micro-batches)", B, mb);
  ensure_arena(e, std::min(B, mb), F, T);
  ensure_persistent(e, (size_t)std::min(B, mb) * F * T, std::max({mb, 64, s.N * (csteps + 1) + 1}));
  prepare_tables(e, s, st);
  const size_t px1 = (size_t)F * T;
  for (int b0 = 0; b0 < B; b0 += mb) {
    const int Bc = std::min(mb, B - b0);
    RngParams rp{s.seed, s.utt_offset + b0, 0};
    CUDA_OK(cudaMemcpyAsync(e.rng_dev, &rp, sizeof(rp), cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaStreamSynchronize(st));
    const float2* nchunk = noise ? noise + b0 * px1 : nullptr;
    const bool graph_ok = e.cfg.use_graphs && !noise && !e.time_convs;
    if (!graph_ok) {
      sample_chunk(e, y + b0 * px1, Bc, F, T, s, nchunk, (size_t)B * px1, out + b0 * px1, st, false);
      continue;
    }
    // graph path: the micro-batch is split over concurrent lanes; every lane's launch sequence works on
    // lane-owned staging (pointer-stable), forked from / joined into the caller's stream inside ONE graph.
    // the Langevin corrector couples the utterances of a batch (batch-mean norms, correctors.py:50-52): one launch sequence
    const int L = coupled ? 1 : std::max(1, std::min(e.num_lanes, Bc));
    ensure_lanes(e, std::max(L, (int)e.lanes.size()));
    const int per = (Bc + L - 1) / L;
    int lb[16], ln[16];
    for (int i = 0; i < L; ++i) { lb[i] = std::min(Bc, i * per); ln[i] = std::min(Bc, lb[i] + per) - lb[i]; }
    for (int i = 0; i < L; ++i) {
      if (ln[i] <= 0) continue;
      Engine& le = *e.lanes[i];
      ensure_arena(le, ln[i], F, T);
      ensure_persistent(le, (size_t)per * px1, std::max({mb, 64, s.N * (csteps + 1) + 1}));
      ensure_stft_buf(le, 3, (size_t)per * px1 * 8);
      if (i > 0) prepare_tables(le, s, st);                       // lane 0's tables were prepared above
      RngParams lrp{s.seed, s.utt_offset + b0 + lb[i], 0};
      CUDA_OK(cudaMemcpyAsync(le.rng_dev, &lrp, sizeof(lrp), cudaMemcpyHostToDevice, st));
      CUDA_OK(cudaStreamSynchronize(st));
      CUDA_OK(cudaMemcpyAsync(le.stft_buf[3], y + (b0 + lb[i]) * px1, ln[i] * px1 * sizeof(float2), cudaMemcpyDeviceToDevice, st));
    }
    // generations of ALL existing lanes, not of the first L: calls that alternate between L = 1 and L = 2 (bucket
    // remainders of the batched service, the last micro-batch of B % max_batch == 1) would otherwise see a different
    // sum every time and throw every captured graph away
    long long gen = 0;
    for (size_t i = 0; i < e.lanes.size(); ++i) gen += e.lanes[i]->generation;
    if (gen != e.lanes_generation_seen) {          // some lane re-allocated a buffer a captured graph points to
      for (auto& g : e.graphs) cudaGraphExecDestroy(g.second.exec);
      e.graphs.clear();
      e.lanes_generation_seen = gen;
    }
    GraphKey key{Bc * 64 + L, F, T, s.N, s.predictor, s.corrector, csteps, s.denoise, s.probability_flow, s.snr, s.kind, s.sb_eps};
    auto it = e.graphs.find(key);
    if (it == e.graphs.end()) {
      // one eager network evaluation first: sets function attributes and surfaces launch errors early
      {
        launch_pack_state(st, y + b0 * px1, y + b0 * px1, ln[0], F, T, e.state);
        Fwd f{e, st, e.temb_table, 0, false, act_dtype(e.cfg)};
        f.run(e.state, ln[0], F, T);
        CUDA_OK(cudaStreamSynchronize(st));
      }
      cudaGraph_t g = nullptr;
      long long before = 0;
      for (int i = 0; i < L; ++i) before += e.lanes[i]->kernel_launches;
      std::vector<long long> saved(L);
      for (int i = 0; i < L; ++i) saved[i] = e.lanes[i]->kernel_launches;
      CUDA_OK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
      try {
        CUDA_OK(cudaEventRecord(e.lane_events[0], st));
        for (int i = 1; i < L; ++i) if (ln[i] > 0) CUDA_OK(cudaStreamWaitEvent(e.lane_streams[i], e.lane_events[0], 0));
        for (int i = 0; i < L; ++i) {
          if (ln[i] <= 0) continue;
          Engine& le = *e.lanes[i];
          cudaStream_t ls = i == 0 ? st : e.lane_streams[i];
          sample_chunk(le, (const float2*)le.stft_buf[3], ln[i], F, T, s, nullptr, 0, (float2*)le.stft_buf[3], ls, true);
          if (i > 0) CUDA_OK(cudaEventRecord(e.lane_events[i], ls));
        }
        for (int i = 1; i < L; ++i) if (ln[i] > 0) CUDA_OK(cudaStreamWaitEvent(st, e.lane_events[i], 0));
      } catch (...) {
        cudaStreamEndCapture(st, &g);
        if (g) cudaGraphDestroy(g);
        throw;
      }
      CUDA_OK(cudaStreamEndCapture(st, &g));
      cudaGraphExec_t ge = nullptr;
      CUDA_OK(cudaGraphInstantiate(&ge, g, 0));
      cudaGraphDestroy(g);
      long long after = 0;
      for (int i = 0; i < L; ++i) { after += e.lanes[i]->kernel_launches; e.lanes[i]->kernel_launches = saved[i]; }
      if ((int)e.graphs.size() >= std::max(1, e.max_graphs)) {           // evict the least recently launched executable
        auto victim = e.graphs.begin();
        for (auto g2 = e.graphs.begin(); g2 != e.graphs.end(); ++g2)
          if (g2->second.last_used < victim->second.last_used) victim = g2;
        cudaGraphExecDestroy(victim->second.exec);                        // deferred by the runtime if still in flight
        e.graphs.erase(victim);
      }
      it = e.graphs.emplace(key, GraphEntry{ge, after - before, 0}).first;   // kernels recorded, not executed
    }
    it->second.last_used = ++e.graph_clock;
    CUDA_OK(cudaGraphLaunch(it->second.exec, st));
    ++e.graph_launches;
    e.kernel_launches += it->second.kernel_nodes;
    for (int i = 0; i < L; ++i)
      if (ln[i] > 0)
        CUDA_OK(cudaMemcpyAsync(out + (b0 + lb[i]) * px1, e.lanes[i]->stft_buf[3], ln[i] * px1 * sizeof(float2), cudaMemcpyDeviceToDevice, st));
  }
  if (nfe) *nfe = s.kind == SGMSE_B200_SAMPLER_PC ? s.N * (csteps + 1) : s.sb_n_steps;   // the SB samplers report their n_steps argument
}

// ------------------------------------------------------------------------------------------------
// probability-flow ODE sampler (SURVEY.md §8f-4): sampling/__init__.py:72-143 without the host round trips
// ------------------------------------------------------------------------------------------------
__global__ void set_float_kernel(float* dst, float v) { *dst = v; }

void ensure_ode(Engine& e, size_t px) {
  OdeBuffers& o = e.ode;
  if (!o.partial) {
    CUDA_OK(cudaMalloc((void**)&o.partial, kOdeNormBlocks * sizeof(double)));
    CUDA_OK(cudaHostAlloc((void**)&o.partial_host, kOdeNormBlocks * sizeof(double), cudaHostAllocDefault));
  }
  if (px <= o.cap_px) return;
  if (o.y) {
    CUDA_OK(cudaDeviceSynchronize());
    cudaFree(o.y); cudaFree(o.y_new); cudaFree(o.stage);
    for (int i = 0; i < 7; ++i) { cudaFree(o.k[i]); o.k[i] = nullptr; }
    o.y = nullptr; o.y_new = nullptr; o.stage = nullptr; o.cap_px = 0;
  }
  CUDA_OK(cudaMalloc((void**)&o.y, px * sizeof(double2)));
  CUDA_OK(cudaMalloc((void**)&o.y_new, px * sizeof(double2)));
  CUDA_OK(cudaMalloc((void**)&o.stage, px * sizeof(float2)));
  for (int i = 0; i < 7; ++i) CUDA_OK(cudaMalloc((void**)&o.k[i], px * sizeof(float2)));
  o.cap_px = px;
}

// One score-network evaluation on e.state with the time-embedding row e.temb_table[0].  The launch sequence of a
// shape is captured the first time it runs (that first evaluation itself is eager) and replayed afterwards: an ODE
// solve is hundreds of evaluations of the same sequence with nothing but t changing, and t lives in device memory
// (temb row, drift coefficients are kernel arguments of the un-captured drift kernel).
template <class Key>
const float4* run_graphed(Engine& e, std::map<Key, FwdGraph>& graphs, const Key& key, Fwd& f, const float4* state, int Bc,
                          int F, int T, cudaStream_t st, bool graph_ok) {
  if (!graph_ok) return f.run(state, Bc, F, T);
  auto it = graphs.find(key);
  if (it != graphs.end()) {
    CUDA_OK(cudaGraphLaunch(it->second.exec, st));
    ++e.graph_launches;
    e.kernel_launches += it->second.kernel_nodes;
    e.launches_this_forward = it->second.kernel_nodes;
    e.tc_convs = it->second.tc_convs; e.direct_convs = it->second.direct_convs;
    return it->second.out;
  }
  const float4* p = f.run(state, Bc, F, T);                     // eager: sets function attributes, surfaces launch errors
  const long long saved = e.kernel_launches;
  cudaGraph_t g = nullptr;
  CUDA_OK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  const float4* pc = nullptr;
  try {
    pc = f.run(state, Bc, F, T);
  } catch (...) {
    cudaStreamEndCapture(st, &g);
    if (g) cudaGraphDestroy(g);
    throw;
  }
  CUDA_OK(cudaStreamEndCapture(st, &g));
  cudaGraphExec_t ge = nullptr;
  const cudaError_t ierr = cudaGraphInstantiate(&ge, g, 0);
  cudaGraphDestroy(g);
  CUDA_OK(ierr);
  const long long nodes = e.kernel_launches - saved;
  e.kernel_launches = saved;                                    // recorded, not executed
  if (pc != p) { cudaGraphExecDestroy(ge); SG_CHECK(false, "internal: workspace replay moved the network output"); }
  graphs.emplace(key, FwdGraph{ge, p, nodes, e.tc_convs, e.direct_convs});
  return p;
}

const float4* forward_on_state(Engine& e, int Bc, int F, int T, cudaStream_t st, float in_scale = 1.f) {
  Fwd f{e, st, e.temb_table, 0, false, act_dtype(e.cfg)};
  f.in_scale = in_scale;                                       // c_in(t) of a preconditioned model: a kernel argument, so
  const bool graph_ok = e.cfg.use_graphs && !e.time_convs && !e.record_taps && st != nullptr && in_scale == 1.f;   // not graphed
  return run_graphed(e, e.fwd_graphs, std::make_tuple(Bc, F, T), f, e.state, Bc, F, T, st, graph_ok);
}

// One score-network evaluation of Bc rows with their own times: e.temb_table holds one row per sample.  With
// `scaled` (per-sample c_in of a preconditioned model) e.state holds c_in (x, y) and e.ode.raw the unscaled rows, from
// which the input pyramid starts; c_in lives in device memory, so this family is captured too.
const float4* forward_rows(Engine& e, int Bc, int F, int T, cudaStream_t st, bool scaled) {
  Fwd f{e, st, e.temb_table, e.total_temb_c, false, act_dtype(e.cfg)};
  if (scaled) { f.pyr_state = e.ode.raw; f.pyr_scale_rows = e.ode.rows_scale; }
  const bool graph_ok = e.cfg.use_graphs && !e.time_convs && !e.record_taps && st != nullptr;
  return run_graphed(e, e.fwd_rows_graphs, std::make_tuple(Bc, F, T, scaled), f, e.state, Bc, F, T, st, graph_ok);
}

// Drift coefficients at t (float, as the reference's vec_t), computed in double and rounded to float
struct OdeDriftCoefs { float inv_t, cs, c_in, cx, cF; };
OdeDriftCoefs ode_drift_coefs(const Engine& e, float tf) {
  const sgmse_b200_config& c = e.cfg;
  const double ls = log((double)c.sigma_max / c.sigma_min);
  const double g = c.sigma_min * pow((double)c.sigma_max / c.sigma_min, (double)tf) * sqrt(2 * ls);   // sdes.py:188-196
  const Precond pc = is_v2(e) ? precond(c, (double)tf) : Precond{1.0, 0.0, 0.0};   // score = a x + b F(c_in x, c_in y, t)
  OdeDriftCoefs d;
  d.cs = (float)(0.5 * g * g);                                  // -g^2 * score * 0.5 with score = -dnn (sdes.py:116-117)
  d.inv_t = 1.0f / tf;
  d.c_in = (float)pc.c_in;
  d.cx = (float)(-(double)c.theta - 0.5 * g * g * pc.a);
  d.cF = (float)(-0.5 * g * g * pc.b);
  return d;
}

struct OdeDeviceOps {
  Engine& e;
  const float2* Y;
  int B, F, T;
  cudaStream_t st;
  size_t px1, total;
  double2 *y, *y_new;
  float2* k[7];

  size_t size() const { return total; }
  OdeK kk() const { OdeK K; for (int i = 0; i < 7; ++i) K.k[i] = k[i]; return K; }
  void combine(int s, const double* a, double h, bool to_new) {
    OdeCoefs c{};
    for (int j = 0; j < s; ++j) c.a[j] = a[j];
    launch_ode_combine(st, y, kk(), s, c, h, total, e.ode.stage, to_new ? y_new : nullptr);
    ++e.kernel_launches;
  }
  void eval(double t, int slot) {
    const sgmse_b200_config& c = e.cfg;
    const float tf = (float)t;                                  // vec_t = torch.ones(B) * t (sampling/__init__.py:122)
    set_float_kernel<<<1, 1, 0, st>>>(e.t_dev, tf);
    CUDA_OK(cudaGetLastError());
    launch_temb(st, temb_weights(e), e.t_dev, 1, e.temb_scratch, e.temb_table);
    e.kernel_launches += 3;
    const OdeDriftCoefs d = ode_drift_coefs(e, tf);
    const bool v2 = is_v2(e);
    const int mb = std::max(1, c.max_batch);
    for (int b0 = 0; b0 < B; b0 += mb) {
      const int Bc = std::min(mb, B - b0);
      launch_pack_state(st, e.ode.stage + b0 * px1, Y + b0 * px1, Bc, F, T, e.state); ++e.kernel_launches;
      const float4* p = forward_on_state(e, Bc, F, T, st, d.c_in);
      if (v2) launch_ode_drift_affine(st, e.state, p, Bc, F, T, e.out_layer, d.cx, c.theta, d.cF, k[slot] + b0 * px1);
      else launch_ode_drift(st, e.state, p, Bc, F, T, e.out_layer, d.inv_t, c.theta, d.cs, k[slot] + b0 * px1);
      ++e.kernel_launches;
    }
  }
  double finish_norm() {
    CUDA_OK(cudaMemcpyAsync(e.ode.partial_host, e.ode.partial, kOdeNormBlocks * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    double s = 0.0;
    for (int i = 0; i < kOdeNormBlocks; ++i) s += e.ode.partial_host[i];
    return sqrt(s / (double)total);
  }
  double norm_init(int which, double rtol, double atol) {
    launch_ode_norm(st, which, y, y_new, kk(), OdeCoefs{}, 0.0, rtol, atol, total, e.ode.partial); ++e.kernel_launches;
    return finish_norm();
  }
  double norm_err(const double* E, double h, double rtol, double atol) {
    OdeCoefs c{};
    for (int j = 0; j < 7; ++j) c.a[j] = E[j];
    launch_ode_norm(st, 3, y, y_new, kk(), c, h, rtol, atol, total, e.ode.partial); ++e.kernel_launches;
    return finish_norm();
  }
  void accept() { std::swap(y, y_new); std::swap(k[0], k[6]); }
};

void ode_sample(Engine& e, const float2* Y, int B, int F, int T, const sgmse_b200_ode& o, const float2* prior_noise,
                float2* out, int* nfe, int* stats, cudaStream_t st_in) {
  SG_CHECK(e.loaded, "weights not loaded");
  SG_CHECK(e.cfg.sde_kind == SGMSE_B200_SDE_OUVE, "the probability-flow ODE sampler is implemented for the 'ouve' SDE");
  SG_CHECK(!is_v2(e) || e.cfg.loss_type != SGMSE_B200_LOSS_DATA_PREDICTION,
           "the probability-flow ODE sampler needs a score model (loss_type 'score_matching' or 'denoiser')");
  SG_CHECK(o.atol >= 0 && o.rtol >= 0, "`atol` must be positive.");                      // scipy validate_tol
  SG_CHECK(o.eps > 0 && o.eps <= 1, "eps must lie in (0, T=1]");
  cudaStream_t st = st_in;
  if (!st) {                                        // stream capture is illegal on the legacy default stream
    if (!e.own_stream) CUDA_OK(cudaStreamCreate(&e.own_stream));
    st = e.own_stream;
  }
  struct SyncOnExit { cudaStream_t s; bool on; ~SyncOnExit() { if (on) cudaStreamSynchronize(s); } } sync_guard{st, st_in == nullptr};
  const int mb = std::max(1, e.cfg.max_batch);
  const size_t px1 = (size_t)F * T, total = (size_t)B * px1;
  ensure_arena(e, std::min(B, mb), F, T);
  ensure_persistent(e, (size_t)std::min(B, mb) * px1, std::max(mb, 64));
  ensure_ode(e, total);
  const float std1 = (float)ouve_std(e.cfg, 1.0);
  for (int b0 = 0; b0 < B; b0 += mb) {              // x(T) = y + z * std(1)  (sdes.py:224-229), fp32 like the reference
    const int Bc = std::min(mb, B - b0);
    RngParams rp{o.seed, o.utt_offset + b0, 0};
    CUDA_OK(cudaMemcpyAsync(e.rng_dev, &rp, sizeof(rp), cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaStreamSynchronize(st));
    launch_pack_state(st, Y + b0 * px1, Y + b0 * px1, Bc, F, T, e.state);
    launch_prior(st, e.state, Bc, F, T, std1, prior_noise ? prior_noise + b0 * px1 : nullptr, e.rng_dev, 0);
    launch_ode_init(st, e.state, (size_t)Bc * px1, e.ode.y + b0 * px1);
    e.kernel_launches += 3;
    CUDA_OK(cudaStreamSynchronize(st));             // rng_dev is rewritten by the next chunk
  }
  OdeDeviceOps ops{e, Y, B, F, T, st, px1, total, e.ode.y, e.ode.y_new,
                   {e.ode.k[0], e.ode.k[1], e.ode.k[2], e.ode.k[3], e.ode.k[4], e.ode.k[5], e.ode.k[6]}};
  const rk45::Result r = rk45::solve(ops, 1.0, o.eps, o.rtol, o.atol, o.max_attempts > 0 ? o.max_attempts : 100000);
  launch_ode_finish(st, ops.y, total, out); ++e.kernel_launches;
  if (nfe) *nfe = r.nfev;
  if (stats) { stats[0] = r.steps; stats[1] = r.rejected; stats[2] = r.status; stats[3] = 0; }
}

// ode_sample_groups: ceil(B / group) independent ODE systems of `group` consecutive utterances each, every system
// with its own RK45 controller (rk45::solve_groups).  At most max_batch utterances are in flight: slot k of the
// max_batch / group slots owns region k of the y / y_new / stage / K buffers.  Per round, the norms of all systems
// in flight are one launch per kOdeSysPerLaunch systems and ONE device-to-host copy and sync; their evaluations are
// one combine launch, one network forward over all their utterances (one time-embedding row and c_in per utterance)
// and one drift launch.  Every kernel does, per system, what ode_sample's kernels do for that system alone, and the
// forward is bit-identical under any batch composition, so each system's result equals ode_sample on it alone.
struct OdeGroupOps {
  Engine& e;
  const float2* Y;
  int B, group, F, T;
  cudaStream_t st;
  size_t px1;
  const sgmse_b200_ode& o;
  const float2* prior_noise;
  float2* out;
  float std1;
  bool v2;
  struct Slot { double2 *y, *y_new; float2* k[7]; float2* stage; size_t total; };
  std::vector<Slot> slots;
  long long syncs = 0, evaluated_rows = 0, forwards = 0;

  int first(int sys) const { return sys * group; }
  int count(int sys) const { return std::min(group, B - sys * group); }
  size_t size(int sys) const { return (size_t)count(sys) * px1; }
  static OdeK kk(const Slot& s) { OdeK K; for (int i = 0; i < 7; ++i) K.k[i] = s.k[i]; return K; }

  void start(int sys, int k) {                       // x(T) = y + z * std(1) of the system's utterances, as ode_sample
    const int b0 = first(sys), n = count(sys);
    RngParams rp{o.seed, o.utt_offset + b0, 0};
    CUDA_OK(cudaMemcpyAsync(e.rng_dev, &rp, sizeof(rp), cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaStreamSynchronize(st));
    launch_pack_state(st, Y + b0 * px1, Y + b0 * px1, n, F, T, e.state);
    launch_prior(st, e.state, n, F, T, std1, prior_noise ? prior_noise + b0 * px1 : nullptr, e.rng_dev, 0);
    launch_ode_init(st, e.state, (size_t)n * px1, slots[k].y);
    e.kernel_launches += 3;
    CUDA_OK(cudaStreamSynchronize(st));             // rng_dev is rewritten by the next start
    syncs += 2;
    slots[k].total = size(sys);
  }
  void norms(int n, const int* sl, const rk45::Request* q, double rtol, double atol, double* v) {
    for (int i0 = 0; i0 < n; i0 += kOdeSysPerLaunch) {
      const int m = std::min(kOdeSysPerLaunch, n - i0);
      OdeSysTable tab{};
      for (int i = 0; i < m; ++i) {
        const Slot& s = slots[sl[i0 + i]];
        const rk45::Request& r = q[i0 + i];
        OdeSys& d = tab.sys[i];
        d.y = s.y; d.y_new = s.y_new; d.K = kk(s); d.total = s.total; d.s = r.s;
        if (r.s == 3) { for (int j = 0; j < 7; ++j) d.c.a[j] = r.a[j]; d.h = r.h; }
      }
      launch_ode_norm_groups(st, tab, m, rtol, atol, e.ode.gpartial + (size_t)i0 * kOdeNormBlocks); ++e.kernel_launches;
    }
    CUDA_OK(cudaMemcpyAsync(e.ode.gpartial_host, e.ode.gpartial, (size_t)n * kOdeNormBlocks * sizeof(double),
                            cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    ++syncs;
    for (int i = 0; i < n; ++i) {
      double acc = 0.0;
      for (int b = 0; b < kOdeNormBlocks; ++b) acc += e.ode.gpartial_host[(size_t)i * kOdeNormBlocks + b];
      v[i] = sqrt(acc / (double)slots[sl[i]].total);
    }
  }
  void evals(int n, const int* sys, const int* sl, const rk45::Request* q) {
    for (int i0 = 0; i0 < n; i0 += kOdeSysPerLaunch) {
      const int m = std::min(kOdeSysPerLaunch, n - i0);
      OdeSysTable tab{};
      for (int i = 0; i < m; ++i) {
        const Slot& s = slots[sl[i0 + i]];
        const rk45::Request& r = q[i0 + i];
        OdeSys& d = tab.sys[i];
        d.y = s.y; d.y_new = r.to_new ? s.y_new : nullptr; d.K = kk(s); d.total = s.total; d.stage = s.stage; d.s = r.s; d.h = r.h;
        for (int j = 0; j < r.s; ++j) d.c.a[j] = r.a[j];
      }
      launch_ode_combine_groups(st, tab, m); ++e.kernel_launches;
    }
    std::vector<OdeRows> tabs;
    int R = 0;
    for (int i = 0; i < n; ++i) {
      const Slot& s = slots[sl[i]];
      const float tf = (float)q[i].t;                             // vec_t = torch.ones(B) * t (sampling/__init__.py:122)
      const OdeDriftCoefs d = ode_drift_coefs(e, tf);
      for (int u = 0; u < count(sys[i]); ++u, ++R) {
        if (R % kOdeRowsPerLaunch == 0) tabs.emplace_back();
        OdeRows& t = tabs.back();
        const int r = R % kOdeRowsPerLaunch;
        t.x[r] = s.stage + u * px1;
        t.y[r] = Y + (first(sys[i]) + u) * px1;
        t.k_out[r] = s.k[q[i].s] + u * px1;
        t.t[r] = tf;
        t.c_in[r] = d.c_in;
        t.c0[r] = v2 ? d.cx : d.inv_t;
        t.c1[r] = v2 ? d.cF : d.cs;
      }
    }
    for (size_t c = 0; c < tabs.size(); ++c) {
      const int r0 = (int)c * kOdeRowsPerLaunch, m = std::min(kOdeRowsPerLaunch, R - r0);
      launch_ode_rows_pack(st, tabs[c], m, px1, e.state + r0 * px1, v2 ? e.ode.raw + r0 * px1 : nullptr, e.t_dev + r0,
                           e.ode.rows_scale + r0);
      ++e.kernel_launches;
    }
    launch_temb(st, temb_weights(e), e.t_dev, R, e.temb_scratch, e.temb_table); e.kernel_launches += 2;
    const float4* p = forward_rows(e, R, F, T, st, v2);
    for (size_t c = 0; c < tabs.size(); ++c) {
      const int r0 = (int)c * kOdeRowsPerLaunch, m = std::min(kOdeRowsPerLaunch, R - r0);
      launch_ode_rows_drift(st, tabs[c], m, px1, (v2 ? e.ode.raw : e.state) + r0 * px1, p + r0 * px1, e.out_layer,
                            e.cfg.theta, v2);
      ++e.kernel_launches;
    }
    evaluated_rows += R;
    ++forwards;
  }
  void accept(int k) { std::swap(slots[k].y, slots[k].y_new); std::swap(slots[k].k[0], slots[k].k[6]); }
  void finish(int sys, int k, const rk45::Result&) {
    launch_ode_finish(st, slots[k].y, slots[k].total, out + first(sys) * px1); ++e.kernel_launches;
  }
};

// nfe[systems], stats[systems][4] = {accepted steps, rejected attempts, status, 0} (both nullable); info (nullable):
// {rounds, host syncs, network forwards, utterance evaluations}
void ode_sample_groups(Engine& e, const float2* Y, int B, int F, int T, int group, const sgmse_b200_ode& o,
                       const float2* prior_noise, float2* out, int* nfe, int* stats, long long* info, cudaStream_t st_in) {
  SG_CHECK(e.loaded, "weights not loaded");
  SG_CHECK(e.cfg.sde_kind == SGMSE_B200_SDE_OUVE, "the probability-flow ODE sampler is implemented for the 'ouve' SDE");
  SG_CHECK(!is_v2(e) || e.cfg.loss_type != SGMSE_B200_LOSS_DATA_PREDICTION,
           "the probability-flow ODE sampler needs a score model (loss_type 'score_matching' or 'denoiser')");
  SG_CHECK(o.atol >= 0 && o.rtol >= 0, "`atol` must be positive.");                      // scipy validate_tol
  SG_CHECK(o.eps > 0 && o.eps <= 1, "eps must lie in (0, T=1]");
  const int mb = std::max(1, e.cfg.max_batch);
  SG_CHECK(group >= 1 && group <= mb, "group=%d: a system must fit one network evaluation (1 <= group <= max_batch=%d)", group, mb);
  cudaStream_t st = st_in;
  if (!st) {                                        // stream capture is illegal on the legacy default stream
    if (!e.own_stream) CUDA_OK(cudaStreamCreate(&e.own_stream));
    st = e.own_stream;
  }
  struct SyncOnExit { cudaStream_t s; bool on; ~SyncOnExit() { if (on) cudaStreamSynchronize(s); } } sync_guard{st, st_in == nullptr};
  const int systems = (B + group - 1) / group;
  const int nslots = std::min(mb / group, systems);
  const size_t px1 = (size_t)F * T, slot_px = (size_t)group * px1;
  const int rows = std::min(B, nslots * group);
  ensure_arena(e, rows, F, T);
  ensure_persistent(e, (size_t)rows * px1, std::max(mb, 64));
  ensure_ode(e, (size_t)nslots * slot_px);
  OdeBuffers& ob = e.ode;
  if (nslots > ob.cap_slots) {
    if (ob.gpartial) { CUDA_OK(cudaDeviceSynchronize()); cudaFree(ob.gpartial); cudaFreeHost(ob.gpartial_host); }
    CUDA_OK(cudaMalloc((void**)&ob.gpartial, (size_t)nslots * kOdeNormBlocks * sizeof(double)));
    CUDA_OK(cudaHostAlloc((void**)&ob.gpartial_host, (size_t)nslots * kOdeNormBlocks * sizeof(double), cudaHostAllocDefault));
    ob.cap_slots = nslots;
  }
  if (!ob.rows_scale) CUDA_OK(cudaMalloc((void**)&ob.rows_scale, (size_t)std::max(mb, 64) * sizeof(float)));
  if (is_v2(e) && (size_t)rows * px1 > ob.cap_raw_px) {   // read inside captured forwards
    if (ob.raw) { CUDA_OK(cudaDeviceSynchronize()); cudaFree(ob.raw); }
    CUDA_OK(cudaMalloc((void**)&ob.raw, (size_t)rows * px1 * sizeof(float4)));
    ob.cap_raw_px = (size_t)rows * px1;
    clear_graphs(e);
  }
  OdeGroupOps ops{e, Y, B, group, F, T, st, px1, o, prior_noise, out, (float)ouve_std(e.cfg, 1.0), is_v2(e), {}};
  for (int k = 0; k < nslots; ++k) {
    OdeGroupOps::Slot s{};
    s.y = ob.y + k * slot_px; s.y_new = ob.y_new + k * slot_px; s.stage = ob.stage + k * slot_px;
    for (int j = 0; j < 7; ++j) s.k[j] = ob.k[j] + k * slot_px;
    ops.slots.push_back(s);
  }
  std::vector<rk45::Result> res((size_t)systems);
  const long long rounds = rk45::solve_groups(ops, systems, nslots, 1.0, o.eps, o.rtol, o.atol,
                                              o.max_attempts > 0 ? o.max_attempts : 100000, res.data());
  for (int i = 0; i < systems; ++i) {
    if (nfe) nfe[i] = res[i].nfev;
    if (stats) { stats[4 * i] = res[i].steps; stats[4 * i + 1] = res[i].rejected; stats[4 * i + 2] = res[i].status; stats[4 * i + 3] = 0; }
  }
  if (info) { info[0] = rounds; info[1] = ops.syncs; info[2] = ops.forwards; info[3] = ops.evaluated_rows; }
}

// The same controller on a host callback (test hook: pins rk45.h against scipy without a GPU).
struct OdeHostOps {
  sgmse_b200_ode_rhs rhs;
  void* user;
  long long n;
  std::vector<double> y, y_new, stage, k[7];
  size_t size() const { return (size_t)n; }
  void combine(int s, const double* a, double h, bool to_new) {
    for (long long i = 0; i < 2 * n; ++i) {
      double d = 0.0;
      for (int j = 0; j < s; ++j) d += a[j] * k[j][i];
      stage[i] = y[i] + d * h;
    }
    if (to_new) y_new = stage;
  }
  void eval(double t, int slot) { rhs(t, stage.data(), k[slot].data(), n, user); }
  double rms(const std::vector<double>& v, const std::vector<double>* other_for_scale, double rtol, double atol) const {
    double s = 0.0;
    for (long long i = 0; i < n; ++i) {
      double ay = hypot(y[2 * i], y[2 * i + 1]);
      if (other_for_scale) ay = fmax(ay, hypot((*other_for_scale)[2 * i], (*other_for_scale)[2 * i + 1]));
      const double sc = atol + ay * rtol, a = v[2 * i] / sc, b = v[2 * i + 1] / sc;
      s += a * a + b * b;
    }
    return sqrt(s / (double)n);
  }
  double norm_init(int which, double rtol, double atol) {
    if (which == 0) return rms(y, nullptr, rtol, atol);
    if (which == 1) return rms(k[0], nullptr, rtol, atol);
    std::vector<double> d((size_t)2 * n);
    for (long long i = 0; i < 2 * n; ++i) d[i] = k[1][i] - k[0][i];
    return rms(d, nullptr, rtol, atol);
  }
  double norm_err(const double* E, double h, double rtol, double atol) {
    std::vector<double> d((size_t)2 * n);
    for (long long i = 0; i < 2 * n; ++i) {
      double v = 0.0;
      for (int j = 0; j < 7; ++j) v += E[j] * k[j][i];
      d[i] = v * h;
    }
    return rms(d, &y_new, rtol, atol);
  }
  void accept() { y.swap(y_new); k[0].swap(k[6]); }
};

// rk45::solve_groups on a host callback: each slot is an OdeHostOps, and one callback evaluates every system in flight.
struct OdeHostGroupOps {
  sgmse_b200_ode_rhs_groups rhs;
  void* user;
  const long long* n;
  const std::vector<long long>& off;    // offset of each system's values in y (complex units)
  double* y;
  std::vector<OdeHostOps> slots;
  size_t size(int sys) const { return (size_t)n[sys]; }
  void start(int sys, int k) {
    OdeHostOps& s = slots[k];
    s.n = n[sys];
    s.y.assign(y + 2 * off[sys], y + 2 * (off[sys] + n[sys]));
    s.y_new.assign((size_t)2 * s.n, 0.0);
    s.stage.assign((size_t)2 * s.n, 0.0);
    for (auto& v : s.k) v.assign((size_t)2 * s.n, 0.0);
  }
  void norms(int m, const int* sl, const rk45::Request* q, double rtol, double atol, double* v) {
    for (int i = 0; i < m; ++i)
      v[i] = q[i].s == 3 ? slots[sl[i]].norm_err(q[i].a, q[i].h, rtol, atol) : slots[sl[i]].norm_init(q[i].s, rtol, atol);
  }
  void evals(int m, const int* sys, const int* sl, const rk45::Request* q) {
    std::vector<double> t((size_t)m);
    std::vector<const double*> in((size_t)m);
    std::vector<double*> outp((size_t)m);
    std::vector<long long> nn((size_t)m);
    for (int i = 0; i < m; ++i) {
      OdeHostOps& s = slots[sl[i]];
      s.combine(q[i].s, q[i].a, q[i].h, q[i].to_new);
      t[i] = q[i].t; in[i] = s.stage.data(); outp[i] = s.k[q[i].s].data(); nn[i] = s.n;
    }
    rhs(m, sys, t.data(), in.data(), outp.data(), nn.data(), user);
  }
  void accept(int k) { slots[k].accept(); }
  void finish(int sys, int k, const rk45::Result&) { std::copy(slots[k].y.begin(), slots[k].y.end(), y + 2 * off[sys]); }
};

// ------------------------------------------------------------------------------------------------
// STFT front / back end
// ------------------------------------------------------------------------------------------------
void ensure_stft_buf(Engine& e, int slot, size_t bytes) {
  if (bytes <= e.stft_cap[slot]) return;
  if (e.stft_buf[slot]) { CUDA_OK(cudaDeviceSynchronize()); cudaFree(e.stft_buf[slot]); e.stft_buf[slot] = nullptr; }
  CUDA_OK(cudaMalloc(&e.stft_buf[slot], bytes));
  e.stft_cap[slot] = bytes;
  if (slot == 3) clear_graphs(e);
}

cufftHandle fft_plan(Engine& e, bool inverse, int n_fft, int batch) {
  const std::pair<int, int> key{(inverse ? 1 << 28 : 0) | n_fft, batch};
  auto it = e.fft_plans.find(key);
  if (it != e.fft_plans.end()) return it->second;
  cufftHandle h;
  int n[1] = {n_fft};
  const cufftResult r = cufftPlanMany(&h, 1, n, nullptr, 1, n_fft, nullptr, 1, n_fft / 2 + 1, inverse ? CUFFT_C2R : CUFFT_R2C, batch);
  SG_CHECK(r == CUFFT_SUCCESS, "cufftPlanMany(n=%d, batch=%d) failed: %d", n_fft, batch, (int)r);
  e.fft_plans[key] = h;
  return h;
}

int frames_of(const Engine& e, int L) { return 1 + L / e.cfg.hop_length; }
int padded_frames(const Engine& e, int L) { const int nT = frames_of(e, L); return (nT + 63) / 64 * 64; }

void analysis(Engine& e, const float* wav, int B, int L, int pad_mode, float2* Y, float* norm, cudaStream_t st) {
  const sgmse_b200_config& c = e.cfg;
  const int nT = frames_of(e, L), Tpad = padded_frames(e, L), F = c.n_fft / 2 + 1;
  SG_CHECK(L > c.n_fft / 2, "waveform too short for reflect padding");
  SG_CHECK(pad_mode != SGMSE_B200_PAD_REFLECTION || Tpad - nT < nT,
           "reflection padding of %d frames needs more than %d input frames (torch ReflectionPad2d contract)", Tpad - nT, nT);
  ensure_stft_buf(e, 0, (size_t)B * nT * c.n_fft * 4);
  ensure_stft_buf(e, 1, (size_t)B * nT * F * 8);
  launch_absmax(st, wav, B, L, norm);
  launch_frame(st, wav, norm, B, L, c.n_fft, c.hop_length, nT, c.sqrt_window, (float*)e.stft_buf[0]);
  cufftHandle h = fft_plan(e, false, c.n_fft, B * nT);
  SG_CHECK(cufftSetStream(h, st) == CUFFT_SUCCESS, "cufftSetStream failed");
  SG_CHECK(cufftExecR2C(h, (cufftReal*)e.stft_buf[0], (cufftComplex*)e.stft_buf[1]) == CUFFT_SUCCESS, "cufftExecR2C failed");
  launch_spec_fwd(st, (const float2*)e.stft_buf[1], B, nT, F, F, Tpad, c.spec_factor, c.spec_abs_exponent, c.transform_type,
                  pad_mode == SGMSE_B200_PAD_REFLECTION, Y);
  e.kernel_launches += 4;
}

void synthesis(Engine& e, const float2* X, const float* norm, int B, int Tpad, int L, float* wav, cudaStream_t st) {
  const sgmse_b200_config& c = e.cfg;
  const int F = c.n_fft / 2 + 1;
  ensure_stft_buf(e, 0, (size_t)B * Tpad * c.n_fft * 4);
  ensure_stft_buf(e, 1, (size_t)B * Tpad * F * 8);
  launch_spec_back(st, X, B, F, Tpad, F, c.spec_factor, c.spec_abs_exponent, c.transform_type, (float2*)e.stft_buf[1]);
  cufftHandle h = fft_plan(e, true, c.n_fft, B * Tpad);
  SG_CHECK(cufftSetStream(h, st) == CUFFT_SUCCESS, "cufftSetStream failed");
  SG_CHECK(cufftExecC2R(h, (cufftComplex*)e.stft_buf[1], (cufftReal*)e.stft_buf[0]) == CUFFT_SUCCESS, "cufftExecC2R failed");
  launch_overlap_add(st, (const float*)e.stft_buf[0], norm, B, Tpad, c.n_fft, c.hop_length, c.sqrt_window, L, wav);
  e.kernel_launches += 3;
}

// Host-buffer entry points end with a stream synchronisation anyway: read the fp16 range detector with it and refuse to hand
// out a waveform that went through an overflowed (inf -> NaN) activation.  fp32 mode cannot trip it below 3.4e38.
void check_range(Engine& e, cudaStream_t st) {
  unsigned int v = 0;
  if (!e.range_flag) { CUDA_OK(cudaStreamSynchronize(st)); return; }
  CUDA_OK(cudaMemcpyAsync(&v, e.range_flag, sizeof(v), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  if (v) {
    CUDA_OK(cudaMemsetAsync(e.range_flag, 0, sizeof(unsigned int), st));
    SG_CHECK(false, "fp16 activation range exceeded: %u GroupNorm input group(s) held values beyond +-65504 (stored as inf); "
                    "the result is not usable -- run this model in mode tf32_tc (fp32 activations on tensor cores)", v);
  }
}

void enhance(Engine& e, const float* wav, int B, int L, const sgmse_b200_sampler& s, const float2* noise, float* out,
             bool host, cudaStream_t st) {
  const int Tpad = padded_frames(e, L), F = e.cfg.n_fft / 2 + 1;
  const size_t px = (size_t)B * F * Tpad;
  // slot 2: [wav in | wav out | norm | Y | X]
  const size_t wav_bytes = ((size_t)B * L * 4 + 255) & ~(size_t)255;
  ensure_stft_buf(e, 2, 2 * wav_bytes + 256 + ((size_t)B * 4 + 255) / 256 * 256 + 2 * px * 8);
  uint8_t* base = (uint8_t*)e.stft_buf[2];
  float* wav_d = (float*)base;
  float* out_d = (float*)(base + wav_bytes);
  float* norm = (float*)(base + 2 * wav_bytes);
  float2* Y = (float2*)(base + 2 * wav_bytes + ((size_t)B * 4 + 255) / 256 * 256);
  float2* X = Y + px;
  const int mb = std::max(1, e.cfg.max_batch);
  ensure_stft_buf(e, 3, (size_t)std::min(B, mb) * F * Tpad * 8);
  const float* wsrc = wav;
  if (host) { CUDA_OK(cudaMemcpyAsync(wav_d, wav, (size_t)B * L * 4, cudaMemcpyHostToDevice, st)); wsrc = wav_d; }
  analysis(e, wsrc, B, L, s.pad_mode, Y, norm, st);
  pc_sample(e, Y, B, F, Tpad, s, noise, X, nullptr, st);
  float* odst = host ? out_d : out;
  synthesis(e, X, norm, B, Tpad, L, odst, st);
  if (host) {
    CUDA_OK(cudaMemcpyAsync(out, out_d, (size_t)B * L * 4, cudaMemcpyDeviceToHost, st));
    check_range(e, st);                          // synchronises; device-resident callers poll counter "fp16_range_events"
  }
}

// ScoreModel.enhance with sde.sampler_type == 'ode' (model.py:446-447): every utterance is its own ODE system, as
// enhance() is called per file in the reference; the systems share each batched network evaluation (group = 1).
void enhance_ode(Engine& e, const float* wav, int B, int L, const sgmse_b200_ode& o, int pad_mode, const float2* prior_noise,
                 float* out, bool host, int* nfe, cudaStream_t st) {
  const int Tpad = padded_frames(e, L), F = e.cfg.n_fft / 2 + 1;
  const size_t px1 = (size_t)F * Tpad, px = (size_t)B * px1;
  const size_t wav_bytes = ((size_t)B * L * 4 + 255) & ~(size_t)255;
  ensure_stft_buf(e, 2, 2 * wav_bytes + 256 + ((size_t)B * 4 + 255) / 256 * 256 + 2 * px * 8);
  uint8_t* base = (uint8_t*)e.stft_buf[2];
  float* wav_d = (float*)base;
  float* out_d = (float*)(base + wav_bytes);
  float* norm = (float*)(base + 2 * wav_bytes);
  float2* Y = (float2*)(base + 2 * wav_bytes + ((size_t)B * 4 + 255) / 256 * 256);
  float2* X = Y + px;
  const float* wsrc = wav;
  if (host) { CUDA_OK(cudaMemcpyAsync(wav_d, wav, (size_t)B * L * 4, cudaMemcpyHostToDevice, st)); wsrc = wav_d; }
  analysis(e, wsrc, B, L, pad_mode, Y, norm, st);
  ode_sample_groups(e, Y, B, F, Tpad, 1, o, prior_noise, X, nfe, nullptr, nullptr, st);
  float* odst = host ? out_d : out;
  synthesis(e, X, norm, B, Tpad, L, odst, st);
  if (host) {
    CUDA_OK(cudaMemcpyAsync(out, out_d, (size_t)B * L * 4, cudaMemcpyDeviceToHost, st));
    check_range(e, st);
  }
}

}  // namespace

// ================================================================================================
// C-ABI
// ================================================================================================
// Install the calling engine's kernel selection into the thread-local switches the launch helpers read.
// Option value 0 always means "the current default kernel".  Round 2 made the gated round-2 candidates the defaults (bit-identical
// to the round-1 kernels except fir_variant: half2 FIR-up, rel-L2 8e-4 per forward); the round-1 kernels stay selectable under a
// new number.  The launch helpers keep their internal numbering, the translation lives here:
//   fir_variant     0 = all loads in flight + half2 FIR-up (internal 2) | 1 = expf silu, fp32 FIR | 3 = round-1 kernel
//   outconv_variant 0 = cp.async staging (internal 3) | 1 = CUDA-core | 2 = fused GroupNorm | 4 = round-1 kernel
//   inconv_variant  0 = prefetched A fragments (internal 2) | 1 = CUDA-core | 3 = round-1 kernel
//   combine_variant 0 = thread per 8-channel vector (internal 1) | 2 = round-1 kernel
//   tc1_narrow / gn_self / gnfin_variant   0 = on (internal 1) | 2 = off (round 1)
static int xl(int v, int new_default, int old_number) { return v == 0 ? new_default : (v == old_number ? 0 : v); }
static void activate(const sgmse_b200_engine& e) {
  const auto& o = e.opts;
  sgmse::g_tc_variant = o.tc_variant; sgmse::g_attn_variant = o.attn_variant;
  sgmse::g_fir_variant = xl(o.fir_variant, 2, 3);
  sgmse::g_outconv_variant = xl(o.outconv_variant, 3, 4);
  sgmse::g_inconv_variant = xl(o.inconv_variant, 2, 3);
  sgmse::g_combine_variant = xl(o.combine_variant, 1, 2);
  sgmse::g_tc1_narrow = xl(o.tc1_narrow, 1, 2);
  sgmse::g_gn_self = xl(o.gn_self, 1, 2);
  sgmse::g_gnfin_variant = xl(o.gnfin_variant, 1, 2);
  sgmse::g_pdl = o.pdl;
}

#define API_BEGIN try {
#define API_END                                                          \
  return 0;                                                              \
  }                                                                      \
  catch (const sgmse::Error& err) { sgmse::set_last_error(err.msg); return 1; } \
  catch (const std::exception& ex) { sgmse::set_last_error(ex.what()); return 2; } \
  catch (...) { sgmse::set_last_error("unknown error"); return 3; }

extern "C" {

const char* sgmse_b200_last_error(void) { return sgmse::get_last_error(); }
const char* sgmse_b200_version(void) { return "sgmse_b200 0.1 (sm_90a)"; }

int sgmse_b200_create(const sgmse_b200_config* cfg, sgmse_b200_engine** out) {
  API_BEGIN
  SG_CHECK(cfg && out, "null argument");
  std::unique_ptr<Engine> e(new Engine());
  e->cfg = *cfg;
  if (e->cfg.max_batch <= 0) e->cfg.max_batch = 8;
  SG_CHECK(cfg->mode >= 0 && cfg->mode <= 3, "unknown mode %d", cfg->mode);
  SG_CHECK(cfg->transform_type >= SGMSE_B200_TRANSFORM_EXPONENT && cfg->transform_type <= SGMSE_B200_TRANSFORM_NONE,
           "unknown transform_type %d (0 exponent, 1 log, 2 none)", cfg->transform_type);
  SG_CHECK(cfg->not_centered == 0 || cfg->not_centered == 1, "not_centered must be 0 or 1, got %d", cfg->not_centered);
  SG_CHECK(!cfg->not_centered || cfg->backbone != SGMSE_B200_BACKBONE_NCSNPP_V2,
           "not_centered: backbone 'ncsnpp_v2' has no --no-centered option");
  build_network(*e);                          // host only: no CUDA call before the first weights arrive
  *out = e.release();
  API_END
}

void sgmse_b200_destroy(sgmse_b200_engine* e) {
  if (!e) return;
  cudaDeviceSynchronize();
  try { if (e->lanes.size() > 1) ensure_lanes(*e, 1); } catch (...) {}
  for (cudaEvent_t ev : e->lane_events) cudaEventDestroy(ev);
  try { free_weights(*e); free_workspace(*e); } catch (...) {}   // a dead context must not terminate the host process
  cudaFree(e->range_flag);
  delete e;
}

int sgmse_b200_manifest_count(const sgmse_b200_engine* e) { return e ? (int)e->manifest.size() : -1; }
int sgmse_b200_manifest_entry(const sgmse_b200_engine* e, int i, char* name, int name_cap, long long* numel) {
  API_BEGIN
  SG_CHECK(e && i >= 0 && i < (int)e->manifest.size(), "manifest index out of range");
  activate(*e);
  if (name && name_cap > 0) { strncpy(name, e->manifest[i].name.c_str(), name_cap - 1); name[name_cap - 1] = 0; }
  if (numel) *numel = e->manifest[i].numel;
  API_END
}
long long sgmse_b200_weights_numel(const sgmse_b200_engine* e) { return e ? e->weights_numel : -1; }

int sgmse_b200_load_weights(sgmse_b200_engine* e, const float* blob, long long numel) {
  API_BEGIN
  SG_CHECK(e && blob, "null argument");
  activate(*e);
  SG_CHECK(numel == e->weights_numel, "weight blob has %lld floats, the network needs %lld", numel, e->weights_numel);
  load_weights(*e, blob);
  API_END
}
int sgmse_b200_load_weights_device(sgmse_b200_engine* e, const float* blob_dev, long long numel, void* stream) {
  API_BEGIN
  SG_CHECK(e && blob_dev, "null argument");
  activate(*e);
  SG_CHECK(numel == e->weights_numel, "weight blob has %lld floats, the network needs %lld", numel, e->weights_numel);
  load_weights_device(*e, blob_dev, (cudaStream_t)stream);      // packed on the device (pack.cu): no host round trip
  API_END
}

int sgmse_b200_dnn_forward(sgmse_b200_engine* e, const void* x, const float* t, void* out, int B, int F, int T, void* stream) {
  API_BEGIN
  SG_CHECK(e && x && t && out && B > 0, "bad argument");
  activate(*e);
  const float2* xx = (const float2*)x;   // [B][2][F*T]: channel 0 = x_t, channel 1 = y
  // the two channels of one sample are F*T apart; re-pack through pack_state per sample pair
  const size_t px1 = (size_t)F * T;
  ensure_stft_buf(*e, 3, (size_t)2 * B * px1 * 8);
  float2* xs = (float2*)e->stft_buf[3];
  float2* ys = xs + (size_t)B * px1;
  for (int b = 0; b < B; ++b) {
    CUDA_OK(cudaMemcpyAsync(xs + b * px1, xx + (size_t)(2 * b) * px1, px1 * 8, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    CUDA_OK(cudaMemcpyAsync(ys + b * px1, xx + (size_t)(2 * b + 1) * px1, px1 * 8, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  }
  dnn_forward(*e, xs, ys, t, (float2*)out, B, F, T, false, (cudaStream_t)stream);
  API_END
}
int sgmse_b200_score(sgmse_b200_engine* e, const void* x_t, const void* y, const float* t, void* out, int B, int F, int T, void* stream) {
  API_BEGIN
  SG_CHECK(e && x_t && y && t && out && B > 0, "bad argument");
  activate(*e);
  dnn_forward(*e, (const float2*)x_t, (const float2*)y, t, (float2*)out, B, F, T, true, (cudaStream_t)stream);
  API_END
}

int sgmse_b200_noise_draws(const sgmse_b200_sampler* s) { return s ? noise_draws(*s) : -1; }

int sgmse_b200_model_forward(sgmse_b200_engine* e, const void* x_t, const void* y, const float* t, void* out, int B, int F,
                             int T, void* stream) {
  API_BEGIN
  SG_CHECK(e && x_t && y && t && out && B > 0, "bad argument");
  activate(*e);
  cudaStream_t st = (cudaStream_t)stream;
  if (!is_v2(*e)) {                                  // legacy branch (model.py:307-310)
    dnn_forward(*e, (const float2*)x_t, (const float2*)y, t, (float2*)out, B, F, T, true, st);
  } else {
    // per-sample scalars of model.py:283-304 on the host (this is the parity entry point, not the sampler's hot path)
    SG_CHECK(e->loaded, "weights not loaded");
    std::vector<float> th(B);
    CUDA_OK(cudaMemcpyAsync(th.data(), t, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    const int mb = std::max(1, e->cfg.max_batch);
    ensure_arena(*e, std::min(B, mb), F, T);
    ensure_persistent(*e, (size_t)std::min(B, mb) * F * T, std::max(mb, 64));
    const size_t px1 = (size_t)F * T;
    for (int b0 = 0; b0 < B; b0 += mb) {
      const int Bc = std::min(mb, B - b0);
      std::vector<float> sc(3 * (size_t)Bc);
      for (int i = 0; i < Bc; ++i) {
        const Precond p = precond(e->cfg, th[b0 + i]);
        sc[i] = (float)p.c_in; sc[Bc + i] = (float)p.a; sc[2 * Bc + i] = (float)p.b;
      }
      // the three per-sample vectors (c_in, a, b) are staged in coef_dev (capacity: rows x 48 B >= 3 x Bc floats)
      float* vec = reinterpret_cast<float*>(e->coef_dev);
      CUDA_OK(cudaMemcpyAsync(vec, sc.data(), sc.size() * 4, cudaMemcpyHostToDevice, st));
      CUDA_OK(cudaStreamSynchronize(st));
      launch_pack_state_scaled(st, (const float2*)x_t + b0 * px1, (const float2*)y + b0 * px1, vec, Bc, F, T, e->state);
      ++e->kernel_launches;
      launch_temb(st, temb_weights(*e), t + b0, Bc, e->temb_scratch, e->temb_table); e->kernel_launches += 2;
      Fwd f{*e, st, e->temb_table, e->total_temb_c, false, act_dtype(e->cfg)};
      const float4* p = f.run(e->state, Bc, F, T);
      launch_precond_out(st, (const float2*)x_t + b0 * px1, p, Bc, F, T, e->out_layer, vec + Bc, vec + 2 * Bc,
                         (float2*)out + b0 * px1);
      ++e->kernel_launches;
    }
  }
  API_END
}

int sgmse_b200_sampler_schedule(const sgmse_b200_engine* e, const sgmse_b200_sampler* s, float* ts, float* prior_std,
                                float* coef, int cap_updates, int* n_updates) {
  API_BEGIN
  SG_CHECK(e && s && s->N >= 1, "bad argument");
  activate(*e);
  const SamplerTables tb = make_tables(*e, *s);
  if (ts) for (int i = 0; i < s->N; ++i) ts[i] = tb.ts[i];
  if (s->kind != SGMSE_B200_SAMPLER_PC) {
    if (prior_std) *prior_std = 0.f;
    if (n_updates) *n_updates = s->N;
    if (coef) {
      SG_CHECK(cap_updates >= s->N, "coef buffer holds %d rows, the schedule has %d", cap_updates, s->N);
      for (int i = 0; i < 3 * s->N; ++i) coef[i] = tb.sb_raw[i];
    }
    return 0;
  }
  if (prior_std) {
    const sgmse_b200_config& c = e->cfg;
    const double th = c.theta, smin = c.sigma_min, smax = c.sigma_max, ls = log(smax / smin);
    *prior_std = (float)sqrt(smin * smin * exp(-2 * th) * (exp(2 * (th + ls)) - 1) * ls / (th + ls));
  }
  if (n_updates) *n_updates = (int)tb.coef.size();
  if (coef) {
    SG_CHECK(cap_updates >= (int)tb.coef.size(), "coef buffer holds %d rows, the schedule has %zu", cap_updates, tb.coef.size());
    const int ncorr = s->corrector != SGMSE_B200_CORR_NONE ? s->corrector_steps : 0;
    const int per_step = ncorr + (s->predictor != SGMSE_B200_PRED_NONE ? 1 : 0);
    for (size_t i = 0; i < tb.coef.size(); ++i) {
      const bool on_device = s->corrector == SGMSE_B200_CORR_LANGEVIN && per_step > 0 && (int)(i % per_step) < ncorr;
      coef[3 * i] = on_device ? 0.f : tb.coef[i].cy;
      coef[3 * i + 1] = on_device ? 0.f : tb.coef[i].cs;
      coef[3 * i + 2] = on_device ? 0.f : tb.coef[i].cz;
    }
  }
  API_END
}

int sgmse_b200_pc_sample(sgmse_b200_engine* e, const void* y, int B, int F, int T, const sgmse_b200_sampler* s,
                         const void* noise, void* out, int* nfe, void* stream) {
  API_BEGIN
  SG_CHECK(e && y && s && out && B > 0, "bad argument");
  activate(*e);
  const int mb = std::max(1, e->cfg.max_batch);
  ensure_stft_buf(*e, 3, (size_t)std::min(B, mb) * F * T * 8);
  pc_sample(*e, (const float2*)y, B, F, T, *s, (const float2*)noise, (float2*)out, nfe, (cudaStream_t)stream);
  API_END
}

int sgmse_b200_ode_sample(sgmse_b200_engine* e, const void* y, int B, int F, int T, const sgmse_b200_ode* o,
                          const void* prior_noise, void* out, int* nfe, int stats[4], void* stream) {
  API_BEGIN
  SG_CHECK(e && y && o && out && B > 0, "bad argument");
  activate(*e);
  ode_sample(*e, (const float2*)y, B, F, T, *o, (const float2*)prior_noise, (float2*)out, nfe, stats, (cudaStream_t)stream);
  API_END
}

int sgmse_b200_rk45_host(sgmse_b200_ode_rhs rhs, void* user, double t0, double t_bound, double* y, long long n,
                         double rtol, double atol, int max_attempts, int* nfev, int stats[4]) {
  API_BEGIN
  SG_CHECK(rhs && (y || n == 0) && n >= 0, "bad argument");
  SG_CHECK(atol >= 0, "`atol` must be positive.");
  OdeHostOps ops{rhs, user, n, {}, {}, {}, {}};
  ops.y.assign(y, y + 2 * n);
  ops.y_new.assign((size_t)2 * n, 0.0);
  ops.stage.assign((size_t)2 * n, 0.0);
  for (auto& k : ops.k) k.assign((size_t)2 * n, 0.0);
  const rk45::Result r = rk45::solve(ops, t0, t_bound, rtol, atol, max_attempts > 0 ? max_attempts : 100000);
  for (long long i = 0; i < 2 * n; ++i) y[i] = ops.y[i];
  if (nfev) *nfev = r.nfev;
  if (stats) { stats[0] = r.steps; stats[1] = r.rejected; stats[2] = r.status; stats[3] = 0; }
  API_END
}

int sgmse_b200_ode_sample_groups(sgmse_b200_engine* e, const void* y, int B, int F, int T, int group, const sgmse_b200_ode* o,
                                 const void* prior_noise, void* out, int* nfe, int* stats, long long info[4], void* stream) {
  API_BEGIN
  SG_CHECK(e && y && o && out && B > 0, "bad argument");
  activate(*e);
  ode_sample_groups(*e, (const float2*)y, B, F, T, group, *o, (const float2*)prior_noise, (float2*)out, nfe, stats, info,
                    (cudaStream_t)stream);
  API_END
}

int sgmse_b200_rk45_host_groups(sgmse_b200_ode_rhs_groups rhs, void* user, int systems, int slots, const long long* n,
                                double t0, double t_bound, double* y, double rtol, double atol, int max_attempts, int* nfev,
                                int* stats, long long* rounds) {
  API_BEGIN
  SG_CHECK(rhs && n && systems > 0 && slots > 0, "bad argument");
  SG_CHECK(atol >= 0, "`atol` must be positive.");
  std::vector<long long> off((size_t)systems + 1, 0);
  for (int i = 0; i < systems; ++i) { SG_CHECK(n[i] >= 0, "bad argument"); off[i + 1] = off[i] + n[i]; }
  SG_CHECK(y || off[systems] == 0, "bad argument");
  OdeHostGroupOps ops{rhs, user, n, off, y, {}};
  ops.slots.resize((size_t)std::min(slots, systems), OdeHostOps{nullptr, nullptr, 0, {}, {}, {}, {}});
  std::vector<rk45::Result> res((size_t)systems);
  const long long r = rk45::solve_groups(ops, systems, slots, t0, t_bound, rtol, atol, max_attempts > 0 ? max_attempts : 100000,
                                         res.data());
  for (int i = 0; i < systems; ++i) {
    if (nfev) nfev[i] = res[i].nfev;
    if (stats) { stats[4 * i] = res[i].steps; stats[4 * i + 1] = res[i].rejected; stats[4 * i + 2] = res[i].status; stats[4 * i + 3] = 0; }
  }
  if (rounds) *rounds = r;
  API_END
}

int sgmse_b200_padded_frames(const sgmse_b200_engine* e, int L) { return e ? padded_frames(*e, L) : -1; }

int sgmse_b200_analysis(sgmse_b200_engine* e, const float* wav, int B, int L, int pad_mode, void* Y, float* norm, void* stream) {
  API_BEGIN
  SG_CHECK(e && wav && Y && norm, "bad argument");
  activate(*e);
  analysis(*e, wav, B, L, pad_mode, (float2*)Y, norm, (cudaStream_t)stream);
  API_END
}
int sgmse_b200_synthesis(sgmse_b200_engine* e, const void* X, const float* norm, int B, int Tpad, int L, float* wav, void* stream) {
  API_BEGIN
  SG_CHECK(e && X && norm && wav, "bad argument");
  activate(*e);
  synthesis(*e, (const float2*)X, norm, B, Tpad, L, wav, (cudaStream_t)stream);
  API_END
}
int sgmse_b200_enhance(sgmse_b200_engine* e, const float* wav, int B, int L, const sgmse_b200_sampler* s,
                       const void* noise, float* out, int host_buffers, void* stream) {
  API_BEGIN
  SG_CHECK(e && wav && s && out && B > 0 && L > 0, "bad argument");
  activate(*e);
  enhance(*e, wav, B, L, *s, (const float2*)noise, out, host_buffers != 0, (cudaStream_t)stream);
  API_END
}

int sgmse_b200_enhance_ode(sgmse_b200_engine* e, const float* wav, int B, int L, const sgmse_b200_ode* o, int pad_mode,
                           const void* prior_noise, float* out, int host_buffers, int* nfe, void* stream) {
  API_BEGIN
  SG_CHECK(e && wav && o && out && B > 0 && L > 0, "bad argument");
  activate(*e);
  enhance_ode(*e, wav, B, L, *o, pad_mode, (const float2*)prior_noise, out, host_buffers != 0, nfe, (cudaStream_t)stream);
  API_END
}

int sgmse_b200_get_tap(sgmse_b200_engine* e, const char* name, float* out_host, long long cap, int shape[4]) {
  API_BEGIN
  SG_CHECK(e && name, "bad argument");
  activate(*e);
  CUDA_OK(cudaDeviceSynchronize());
  auto it = e->taps.find(name);
  if (it != e->taps.end()) {
    const TensorDesc& t = it->second;
    if (shape) { shape[0] = t.N; shape[1] = t.C; shape[2] = t.H; shape[3] = t.W; }
    if (!out_host) return 0;
    SG_CHECK((long long)t.numel() <= cap, "tap buffer too small");
    float* tmp = nullptr;
    CUDA_OK(cudaMalloc((void**)&tmp, t.numel() * 4));
    nhwc_to_nchw_kernel<<<(unsigned)((t.numel() + 255) / 256), 256>>>(t.p, t.dt == DT_F16, t.C, t.H * t.W, t.numel(), tmp);
    cudaError_t err = cudaMemcpy(out_host, tmp, t.numel() * 4, cudaMemcpyDeviceToHost);
    cudaFree(tmp);
    CUDA_OK(err);
    return 0;
  }
  auto it4 = e->taps4.find(name);
  SG_CHECK(it4 != e->taps4.end(), "no recorded activation named '%s'", name);
  const std::vector<int>& s4 = it4->second.second;
  const size_t numel = (size_t)s4[0] * 4 * s4[2] * s4[3];
  if (shape) for (int i = 0; i < 4; ++i) shape[i] = s4[i];
  if (!out_host) return 0;
  SG_CHECK((long long)numel <= cap, "tap buffer too small");
  float* tmp = nullptr;
  CUDA_OK(cudaMalloc((void**)&tmp, numel * 4));
  nhwc_to_nchw_kernel<<<(unsigned)((numel + 255) / 256), 256>>>(it4->second.first, 0, 4, s4[2] * s4[3], numel, tmp);
  cudaError_t err = cudaMemcpy(out_host, tmp, numel * 4, cudaMemcpyDeviceToHost);
  cudaFree(tmp);
  CUDA_OK(err);
  API_END
}

long long sgmse_b200_workspace_bytes(sgmse_b200_engine* e, int B, int F, int T) {
  // host-only planning run of the launch sequence (no CUDA call): exercises the whole layer walk
  try {
    SG_CHECK(e && B > 0, "bad argument");
    activate(*e);
    return (long long)workspace_plan(*e, B, F, T).bump + 4096;
  } catch (const sgmse::Error& err) { sgmse::set_last_error(err.msg); return -1; }
  catch (...) { sgmse::set_last_error("unknown error"); return -1; }
}

long long sgmse_b200_workspace_plan(sgmse_b200_engine* e, int B, int F, int T, long long* rows, long long cap,
                                    long long* n_bufs, int* n_steps) {
  try {
    SG_CHECK(e && B > 0, "bad argument");
    activate(*e);
    const WsPlan& p = workspace_plan(*e, B, F, T);
    if (n_bufs) *n_bufs = (long long)p.bufs.size();
    if (n_steps) *n_steps = p.steps;
    if (rows) {
      SG_CHECK(cap >= (long long)p.bufs.size(), "plan buffer holds %lld rows, the plan has %zu", cap, p.bufs.size());
      for (size_t i = 0; i < p.bufs.size(); ++i) {
        const WsBuf& b = p.bufs[i];
        long long* r = rows + 5 * i;
        r[0] = (long long)b.off; r[1] = (long long)b.bytes; r[2] = b.first; r[3] = b.last; r[4] = b.tapped;
      }
    }
    return (long long)p.bytes;
  } catch (const sgmse::Error& err) { sgmse::set_last_error(err.msg); return -1; }
  catch (...) { sgmse::set_last_error("unknown error"); return -1; }
}

int sgmse_b200_set_option(sgmse_b200_engine* e, const char* key, long long value) {
  API_BEGIN
  SG_CHECK(e && key, "bad argument");
  activate(*e);
  const std::string k = key;
  if (k == "record_taps") e->record_taps = value != 0;
  else if (k == "time_convs") {
    // per-launch CUDA-event timing of the convolution kernels (eager launches only; see bench.py)
    CUDA_OK(cudaDeviceSynchronize());
    for (auto& c : e->conv_events) { cudaEventDestroy(c.start); cudaEventDestroy(c.stop); }
    e->conv_events.clear();
    e->time_convs = value != 0;
  }
  else if (k == "use_graphs") e->cfg.use_graphs = value != 0;
  else if (k == "reset_range_events") {
    if (e->range_flag) { CUDA_OK(cudaDeviceSynchronize()); CUDA_OK(cudaMemset(e->range_flag, 0, sizeof(unsigned int))); }
  }
  else if (k == "tc_variant") {
    // changes which intermediate buffers a forward needs: drop cached workspace sizes, graphs and shadow lanes
    SG_CHECK(value == 0 || value == 5, "tc_variant %lld: 0 (TMA-fed convolutions, separate GroupNorm passes) or 5 (GroupNorm+SiLU fused into the convolutions)", value);
    e->opts.tc_variant = (int)value;
    if (e->lanes.size() > 1) ensure_lanes(*e, 1);
    e->ws_plans.clear();
    clear_graphs(*e);
  }
  else if (k == "attn_variant") { e->opts.attn_variant = (int)value; clear_graphs(*e); }
  else if (k == "fir_variant") { e->opts.fir_variant = (int)value; clear_graphs(*e); }
  else if (k == "inconv_variant") { e->opts.inconv_variant = (int)value; clear_graphs(*e); }
  else if (k == "combine_variant") { e->opts.combine_variant = (int)value; clear_graphs(*e); }
  else if (k == "tc1_narrow") { e->opts.tc1_narrow = (int)value; clear_graphs(*e); }
  else if (k == "gn_self") {
    e->opts.gn_self = (int)value;               // skips or keeps the finalize launches: changes the plan's steps
    if (e->lanes.size() > 1) ensure_lanes(*e, 1);
    e->ws_plans.clear();
    clear_graphs(*e);
  }
  else if (k == "workspace_poison") {
    // test option: fill each buffer with 0xFF bytes (NaN in fp16 and fp32) right after its last reader is enqueued, so
    // that a read past a buffer's planned lifetime shows up as NaN; captured graphs are re-captured with the fills
    e->workspace_poison = value != 0;
    for (Engine* l : e->lanes) l->workspace_poison = e->workspace_poison;
    clear_graphs(*e);
  }
  else if (k == "gnfin_variant") { e->opts.gnfin_variant = (int)value; clear_graphs(*e); }
  else if (k == "outconv_variant") {
    e->opts.outconv_variant = (int)value;       // changes the buffers a forward needs (fused GroupNorm or not)
    if (e->lanes.size() > 1) ensure_lanes(*e, 1);
    e->ws_plans.clear();
    clear_graphs(*e);
  }
  else if (k == "pdl") {
    // programmatic dependent launch between the kernels of the launch sequence
    SG_CHECK(value == 0 || sgmse::pdl_compiled(),
             "option 'pdl' needs the library built with -DSGMSE_B200_PDL (python -m sgmse_b200.build --pdl, SGMSE_B200_LIB=...)");
    e->opts.pdl = value != 0;
    clear_graphs(*e);
  }
  else if (k == "max_graphs") {
    SG_CHECK(value >= 1 && value <= 1024, "max_graphs must be in 1..1024");
    e->max_graphs = (int)value;
  }
  else if (k == "lanes") {
    SG_CHECK(value >= 1 && value <= 8, "lanes must be in 1..8");
    e->num_lanes = (int)value;
    clear_graphs(*e);
  }
  else if (k == "tc_mask") {
    e->tc_mask = value;
    if (e->lanes.size() > 1) ensure_lanes(*e, 1);
    e->ws_plans.clear();
    clear_graphs(*e);
  }
  else SG_CHECK(false, "unknown option '%s'", key);
  API_END
}

long long sgmse_b200_get_counter(const sgmse_b200_engine* e, const char* key) {
  if (!e || !key) return -1;
  const std::string k = key;
  if (k == "kernel_launches") return e->kernel_launches;
  if (k == "graph_launches") return e->graph_launches;
  if (k == "cached_graphs") return (long long)e->graphs.size();
  if (k == "pdl_compiled") return sgmse::pdl_compiled() ? 1 : 0;
  if (k == "pdl") return e->opts.pdl;
  if (k == "workspace_bytes") return (long long)e->arena.cap;
  if (k == "weights_bytes") return (long long)e->weights_bytes;
  if (k == "tc_convs_last_forward") return e->tc_convs;
  if (k == "direct_convs_last_forward") return e->direct_convs;
  if (k == "launches_last_forward") return e->launches_this_forward;
  if (k == "fp16_range_events") {               // GroupNorm inputs with non-finite statistics since the last reset (synchronises)
    unsigned int v = 0;
    if (!e->range_flag || cudaDeviceSynchronize() != cudaSuccess ||
        cudaMemcpy(&v, e->range_flag, sizeof(v), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    return (long long)v;
  }
  if (k == "barrier_wait_code") return sgmse::g_wait_code_host ? (long long)*sgmse::g_wait_code_host : 0;   // readable after a trap
  if (k == "timed_conv_tc_us" || k == "timed_conv_tc_mflop" || k == "timed_conv_tc_count" || k == "timed_conv_tc_kbytes" ||
      k == "timed_conv_direct_us") {
    cudaDeviceSynchronize();
    double us = 0, mflop = 0, n = 0, kb = 0, dus = 0;
    for (const auto& c : e->conv_events) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, c.start, c.stop) != cudaSuccess) continue;
      if (c.tc) { us += ms * 1e3; mflop += c.flops * 1e-6; kb += c.bytes * 1e-3; n += 1; } else dus += ms * 1e3;
    }
    if (k == "timed_conv_tc_us") return (long long)us;
    if (k == "timed_conv_tc_mflop") return (long long)mflop;
    if (k == "timed_conv_tc_kbytes") return (long long)kb;
    if (k == "timed_conv_direct_us") return (long long)dus;
    return (long long)n;
  }
  return -1;
}

}  // extern "C"
