// Op-level harness of tests/test_gpu_kernel_ops_tf32.py: extern "C" entry points that wrap raw device pointers in fp32
// TensorDesc / ConvArgs and call the product launcher of the wgmma convolution with TF32 operands (conv_tc with fp32
// activations, mode tf32_tc).  Linked, like kernel_ops.cu, against the objects sgmse_b200.build compiles for the engine
// library, so the kernel under test is the product's object code.  A launcher error returns a non-zero code;
// kops_tf32_last_error() has the message.
#include <string>

#include "kernels.h"

using namespace sgmse;

namespace {

thread_local std::string g_err;

TensorDesc f32(const void* p, int N, int H, int W, int C, const float* stats = nullptr) {
  TensorDesc t;
  t.p = const_cast<void*>(p);
  t.N = N; t.H = H; t.W = W; t.C = C;
  t.dt = DT_F32;
  t.stats = const_cast<float*>(stats);
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

// one convolution: out[N,H,W,Cout] fp32 = (sum over segments of conv(seg) + bias + temb + residual) * scale (see ConvArgs)
struct KopsConvTf32 {
  int N, H, W, Cout;
  float* out;
  float* stats;                 // [N][slots][Cout][2] or null
  int nseg;
  const float* seg[3];          // fp32 NHWC, read by the tensor cores as TF32 (upper 19 bits)
  int seg_c[3], seg_taps[3];
  const float* w;               // [Cout][w_ld] fp32 holding TF32 values
  int w_ld;
  const float* bias;
  const float* temb;
  int temb_stride;
  const float* residual;        // [N,H,W,Cout] fp32 or null
  float scale;
};

const char* kops_tf32_last_error(void) { return g_err.c_str(); }

// plan[9] = bw, bh, bn, block_n, stages, tiles, grid, min_local, max_local
int kops_tf32_conv_plan(int N, int H, int W, int Cout, int sms, int* plan) {
  KOPS_TRY
  put_plan(conv_tc_plan(f32(nullptr, N, H, W, Cout), sms, true), plan);
  KOPS_END
}

// plan[9] receives the plan of this launch, *slots the stats slots per sample
int kops_tf32_conv_tc(void* stream, const KopsConvTf32* c, int* plan, int* slots) {
  KOPS_TRY
  ConvArgs a;
  a.nseg = c->nseg;
  for (int i = 0; i < c->nseg; ++i) {
    a.seg[i].src = f32(c->seg[i], c->N, c->H, c->W, c->seg_c[i]);
    a.seg[i].taps = c->seg_taps[i];
  }
  a.w_tc = c->w;
  a.w_tc_ld = c->w_ld;
  a.bias = c->bias;
  a.temb = c->temb;
  a.temb_stride = c->temb_stride;
  const TensorDesc res = f32(c->residual, c->N, c->H, c->W, c->Cout);
  a.residual = c->residual ? &res : nullptr;
  a.scale = c->scale;
  TensorDesc out = f32(c->out, c->N, c->H, c->W, c->Cout, c->stats);
  launch_conv_tc(static_cast<cudaStream_t>(stream), a, out, nullptr);
  int dev = 0, sms = 0;
  CUDA_OK(cudaGetDevice(&dev));
  CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  put_plan(conv_tc_plan(out, sms, true), plan);
  *slots = out.slots;
  KOPS_END
}

// the host packer's rounding: out[i] = tf32_rna(in[i])
int kops_tf32_rna(const float* in, float* out, long long n) {
  KOPS_TRY
  for (long long i = 0; i < n; ++i) out[i] = tf32_rna(in[i]);
  KOPS_END
}

}  // extern "C"
