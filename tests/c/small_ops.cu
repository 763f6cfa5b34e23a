// Op-level harness of tests/test_gpu_small_ops.py: extern "C" entry points over the product launchers of the resampling
// gn_apply (FIR up / down), channel_stats, the input conv, Combine, the 4-channel FIR and the output conv, plus the device
// weight packers of the last three, on the caller's stream.  Linked against the objects sgmse_b200.build compiles for the
// engine library (see tests/c/kernel_ops.cu); the kernel-selection switches the engine installs per call (engine.cu:
// activate()) are set here from explicit arguments.  dt: 0 = fp32, 1 = fp16 activations (DType).  A launcher error
// returns a non-zero code; sops_last_error() has the message.
#include <string>

#include "kernels.h"

using namespace sgmse;

namespace {

thread_local std::string g_err;

TensorDesc desc(const void* p, int dt, int N, int H, int W, int C, float* stats = nullptr) {
  TensorDesc t;
  t.p = const_cast<void*>(p);
  t.N = N; t.H = H; t.W = W; t.C = C;
  t.dt = dt ? DT_F16 : DT_F32;
  t.stats = stats;
  return t;
}

}  // namespace

#define SOPS_TRY try {
#define SOPS_END                                                 \
  return 0;                                                      \
  }                                                              \
  catch (const sgmse::Error& e) { g_err = e.msg; return 1; }     \
  catch (const std::exception& e) { g_err = e.what(); return 2; }

extern "C" {

const char* sops_last_error(void) { return g_err.c_str(); }

// out0 = FIR(silu(a * x + b)), out1 = FIR(x); x [N][Hi][Wi][C], ab float2 [N][C]; rs: RS_DOWN (1) or RS_UP (2);
// fir_variant: g_fir_variant
int sops_gn_apply_rs(void* stream, int dt, int N, int Hi, int Wi, int C, const void* x, const void* ab, int rs, void* out0,
                     void* out1, int fir_variant) {
  SOPS_TRY
  g_fir_variant = fir_variant;
  const int Ho = rs == RS_DOWN ? Hi / 2 : Hi * 2, Wo = rs == RS_DOWN ? Wi / 2 : Wi * 2;
  const TensorDesc in = desc(x, dt, N, Hi, Wi, C);
  TensorDesc o0 = desc(out0, dt, N, Ho, Wo, C), o1 = desc(out1, dt, N, Ho, Wo, C);
  launch_gn_apply(static_cast<cudaStream_t>(stream), in, nullptr, static_cast<const float2*>(ab), true,
                  static_cast<Resample>(rs), o0, &o1);
  SOPS_END
}

// stats [N][1][C][2] of x [N][H][W][C]
int sops_channel_stats(void* stream, int dt, int N, int H, int W, int C, const void* x, float* stats, int* slots) {
  SOPS_TRY
  TensorDesc t = desc(x, dt, N, H, W, C, stats);
  launch_channel_stats(static_cast<cudaStream_t>(stream), t);
  *slots = t.slots;
  SOPS_END
}

// out [N][H][W][C] = conv3x3(in_scale * state) + bias; w: the packed [36][C] layout; stats [N][slots][C][2] (nullable)
int sops_input_conv(void* stream, int dt, int N, int H, int W, int C, const void* state, const float* w, const float* bias,
                    void* out, float* stats, float in_scale, int inconv_variant, int* slots) {
  SOPS_TRY
  g_inconv_variant = inconv_variant;
  TensorDesc o = desc(out, dt, N, H, W, C, stats);
  launch_input_conv(static_cast<cudaStream_t>(stream), static_cast<const float4*>(state), N, H, W, w, bias, o, in_scale);
  *slots = o.slots;
  SOPS_END
}

// out = conv1x1(pyr) + bias + h; w: the packed [4][C] layout; stats [N][slots][C][2] (nullable)
int sops_combine(void* stream, int dt, int N, int H, int W, int C, const void* pyr, const float* w, const float* bias,
                 const void* h, void* out, float* stats, int combine_variant, int* slots) {
  SOPS_TRY
  g_combine_variant = combine_variant;
  const TensorDesc hd = desc(h, dt, N, H, W, C);
  TensorDesc o = desc(out, dt, N, H, W, C, stats);
  launch_combine(static_cast<cudaStream_t>(stream), static_cast<const float4*>(pyr), w, bias, hd, o);
  *slots = o.slots;
  SOPS_END
}

// 4-channel FIR of in [N][H][W] float4 (H, W: the input's), times scale
int sops_fir4(void* stream, int N, int H, int W, int rs, const void* in, void* out, float scale) {
  SOPS_TRY
  launch_fir4(static_cast<cudaStream_t>(stream), static_cast<const float4*>(in), N, H, W, static_cast<Resample>(rs),
              static_cast<float4*>(out), scale);
  SOPS_END
}

// out float4 [N][H][W] = conv3x3(act) + bias (+ addend); w: the packed [9C][4] layout, wfrag: its packed B fragments or
// null; bias: 4 host floats
int sops_out_conv(void* stream, int dt, int N, int H, int W, int C, const void* act, const float* w, const float* bias,
                  const void* addend, void* out, const void* wfrag, int outconv_variant) {
  SOPS_TRY
  g_outconv_variant = outconv_variant;
  const TensorDesc a = desc(act, dt, N, H, W, C);
  launch_out_conv(static_cast<cudaStream_t>(stream), a, w, bias, static_cast<const float4*>(addend), static_cast<float4*>(out),
                  nullptr, static_cast<const uint2*>(wfrag));
  SOPS_END
}

// torch layouts -> the engine's: [nf][4][3][3] -> [36][nf]; [C][4] -> [4][C]; [4][C][3][3] -> [9C][4] (+ fragments)
int sops_pack_inconv(void* stream, const float* w, int nf, float* out) {
  SOPS_TRY
  launch_pack_inconv(static_cast<cudaStream_t>(stream), w, nf, out);
  SOPS_END
}

int sops_pack_combine(void* stream, const float* w, int C, float* out) {
  SOPS_TRY
  launch_pack_combine(static_cast<cudaStream_t>(stream), w, C, out);
  SOPS_END
}

int sops_pack_outconv(void* stream, const float* w, int C, float* out, void* frag) {
  SOPS_TRY
  launch_pack_outconv(static_cast<cudaStream_t>(stream), w, C, out, static_cast<uint2*>(frag));
  SOPS_END
}

}  // extern "C"
