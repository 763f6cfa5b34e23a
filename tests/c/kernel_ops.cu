// Op-level harness of tests/test_gpu_kernel_ops.py: extern "C" entry points that wrap raw device pointers in TensorDesc /
// ConvArgs and call the product launchers (conv_tc, gn_finalize, gn_norm_apply, gn_apply, attention) on the caller's
// stream.  It is linked against the objects sgmse_b200.build compiles for the engine library, so the kernels under test
// are the product's object code; the kernel-selection switches the engine installs per call (engine.cu: activate()) are
// set here from explicit arguments.  A launcher error returns a non-zero code; kops_last_error() has the message.
#include <string>

#include "kernels.h"

using namespace sgmse;

namespace {

thread_local std::string g_err;

TensorDesc f16(const void* p, int N, int H, int W, int C, const float* stats = nullptr, int slots = 0) {
  TensorDesc t;
  t.p = const_cast<void*>(p);
  t.N = N; t.H = H; t.W = W; t.C = C;
  t.dt = DT_F16;
  t.stats = const_cast<float*>(stats);
  t.slots = slots;
  return t;
}

void put_plan(const TcPlan& p, int* plan) {
  const int v[9] = {p.bw, p.bh, p.bn, p.block_n, p.stages, p.tiles, p.grid, p.min_local, p.max_local};
  for (int i = 0; i < 9; ++i) plan[i] = v[i];
}

}  // namespace

#define KOPS_TRY try {
#define KOPS_END                                                 \
  return 0;                                                      \
  }                                                              \
  catch (const sgmse::Error& e) { g_err = e.msg; return 1; }     \
  catch (const std::exception& e) { g_err = e.what(); return 2; }

extern "C" {

// one convolution: out[N,H,W,Cout] = (sum over segments of conv(seg) + bias + temb + residual) * scale (see ConvArgs)
struct KopsConv {
  int N, H, W, Cout;
  void* out;
  float* stats;                 // [N][slots][Cout][2] or null
  int nseg;
  const void* seg[3];
  int seg_c[3], seg_taps[3];
  const void* w;                // [Cout][w_ld] fp16
  int w_ld;
  const float* bias;
  const float* temb;
  int temb_stride;
  const void* residual;         // [N,H,W,Cout] fp16 or null
  float scale;
  const void* gn_ab;            // float2 [N][seg_c[0] + gn_cat_c]: GroupNorm+SiLU fused into segment 0, or null
  const void* gn_cat;
  int gn_cat_c;
};

const char* kops_last_error(void) { return g_err.c_str(); }

// plan[9] = bw, bh, bn, block_n, stages, tiles, grid, min_local, max_local
int kops_conv_plan(int N, int H, int W, int Cout, int sms, int narrow, int* plan) {
  KOPS_TRY
  put_plan(conv_tc_plan(f16(nullptr, N, H, W, Cout), sms, narrow != 0), plan);
  KOPS_END
}

// narrow: g_tc1_narrow.  plan[9] receives the plan of this launch, *slots the stats slots per sample.
int kops_conv_tc(void* stream, const KopsConv* c, int narrow, int* plan, int* slots) {
  KOPS_TRY
  g_tc1_narrow = narrow;
  ConvArgs a;
  a.nseg = c->nseg;
  for (int i = 0; i < c->nseg; ++i) {
    a.seg[i].src = f16(c->seg[i], c->N, c->H, c->W, c->seg_c[i]);
    a.seg[i].taps = c->seg_taps[i];
  }
  a.w_tc = static_cast<const __half*>(c->w);
  a.w_tc_ld = c->w_ld;
  a.bias = c->bias;
  a.temb = c->temb;
  a.temb_stride = c->temb_stride;
  const TensorDesc res = f16(c->residual, c->N, c->H, c->W, c->Cout);
  a.residual = c->residual ? &res : nullptr;
  a.scale = c->scale;
  if (c->gn_ab) {
    a.gn_ab = static_cast<const float2*>(c->gn_ab);
    a.gn_has_cat = c->gn_cat != nullptr;
    if (a.gn_has_cat) a.gn_cat = f16(c->gn_cat, c->N, c->H, c->W, c->gn_cat_c);
  }
  TensorDesc out = f16(c->out, c->N, c->H, c->W, c->Cout, c->stats);
  launch_conv_tc(static_cast<cudaStream_t>(stream), a, out, nullptr);
  int dev = 0, sms = 0;
  CUDA_OK(cudaGetDevice(&dev));
  CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  put_plan(conv_tc_plan(out, sms, narrow != 0), plan);
  *slots = out.slots;
  KOPS_END
}

// ab[N][C0 + C1] from the [N][slots][C][2] partials of one or two (concatenated) tensors; variant: g_gnfin_variant
int kops_gn_finalize(void* stream, int N, int H, int W, const float* stats0, int C0, int slots0, const float* stats1, int C1,
                     int slots1, const float* gamma, const float* beta, int groups, void* ab, int variant) {
  KOPS_TRY
  g_gnfin_variant = variant;
  const TensorDesc s0 = f16(nullptr, N, H, W, C0, stats0, slots0), s1 = f16(nullptr, N, H, W, C1, stats1, slots1);
  launch_gn_finalize(static_cast<cudaStream_t>(stream), s0, stats1 ? &s1 : nullptr, gamma, beta, groups,
                     static_cast<float2*>(ab));
  KOPS_END
}

// out = [silu](GroupNorm(x0 | x1)) with the statistics finalized in the same kernel (the gn_self path)
int kops_gn_norm_apply(void* stream, int N, int H, int W, const void* x0, int C0, const float* stats0, int slots0, const void* x1,
                       int C1, const float* stats1, int slots1, const float* gamma, const float* beta, int groups, int silu,
                       void* out, int gn_self) {
  KOPS_TRY
  g_gn_self = gn_self;
  const TensorDesc t0 = f16(x0, N, H, W, C0, stats0, slots0), t1 = f16(x1, N, H, W, C1, stats1, slots1);
  TensorDesc o = f16(out, N, H, W, C0 + C1);
  launch_gn_norm_apply(static_cast<cudaStream_t>(stream), t0, x1 ? &t1 : nullptr, gamma, beta, groups, silu != 0, o);
  KOPS_END
}

// out = [silu](a * (x0 | x1) + b), (a, b) = ab[n][channel]; no resampling
int kops_gn_apply(void* stream, int N, int H, int W, const void* x0, int C0, const void* x1, int C1, const void* ab, int silu,
                  void* out) {
  KOPS_TRY
  const TensorDesc t0 = f16(x0, N, H, W, C0), t1 = f16(x1, N, H, W, C1);
  TensorDesc o = f16(out, N, H, W, C0 + C1);
  launch_gn_apply(static_cast<cudaStream_t>(stream), t0, x1 ? &t1 : nullptr, static_cast<const float2*>(ab), silu != 0, RS_NONE,
                  o, nullptr);
  KOPS_END
}

// out[N][S][C] = softmax(q k^T / sqrt(C)) v over the S tokens of qkv[N][S][3C] (q | k | v); variant: g_attn_variant
int kops_attention(void* stream, int N, int S, int C, const void* qkv, void* out, int variant) {
  KOPS_TRY
  g_attn_variant = variant;
  const TensorDesc q = f16(qkv, N, 1, S, 3 * C);
  TensorDesc o = f16(out, N, 1, S, C);
  launch_attention(static_cast<cudaStream_t>(stream), q, o);
  KOPS_END
}

}  // extern "C"
