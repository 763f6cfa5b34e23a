// Op-level harness of tests/test_gpu_sampler_ops.py: extern "C" entry points over the product launchers of the time
// embedding, the predictor / corrector updates with their in-kernel Philox noise, the prior, the Langevin step size,
// the preconditioned-model epilogues and the probability-flow ODE vector kernels, on the caller's stream.  Linked
// against the objects sgmse_b200.build compiles for the engine library (see tests/c/kernel_ops.cu).  RngParams,
// UpdateCoef and AffineCoef are device pointers, as the engine keeps them.  OutLayer travels as w[8] (row-major
// [2][4]) + b[2] and its two flags.  A launcher error returns a non-zero code; samp_last_error() has the message.
#include <string>

#include "kernels.h"

using namespace sgmse;

namespace {

thread_local std::string g_err;

OutLayer out_layer(const float* w8, const float* b2, int scale_after, int scale_by_sigma) {
  OutLayer ol;
  for (int i = 0; i < 8; ++i) ol.w[i / 4][i % 4] = w8[i];
  ol.b[0] = b2[0];
  ol.b[1] = b2[1];
  ol.scale_after = scale_after;
  ol.scale_by_sigma = scale_by_sigma;
  return ol;
}

OdeK odek(void* const* k) {
  OdeK K;
  for (int i = 0; i < 7; ++i) K.k[i] = static_cast<const float2*>(k[i]);
  return K;
}

OdeCoefs coefs(const double* a) {
  OdeCoefs c{};
  for (int i = 0; i < 7; ++i) c.a[i] = a[i];
  return c;
}

cudaStream_t S(void* s) { return static_cast<cudaStream_t>(s); }

}  // namespace

#define SAMP_TRY try {
#define SAMP_END                                                 \
  return 0;                                                      \
  }                                                              \
  catch (const sgmse::Error& e) { g_err = e.msg; return 1; }     \
  catch (const std::exception& e) { g_err = e.what(); return 2; }

extern "C" {

const char* samp_last_error(void) { return g_err.c_str(); }

// out[i] = logf(t[i]) on the device: the same libdevice logf, compiled with the library's flags, that temb_mlp_kernel
// applies to its time, so the test knows the exact fp32 log t the kernel read (the CUDA guide bounds logf only to 1 ulp)
__global__ void logf_kernel(const float* t, float* out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = logf(t[i]);
}

int samp_logf(void* stream, const float* t, float* out, int n) {
  SAMP_TRY
  logf_kernel<<<(n + 255) / 256, 256, 0, S(stream)>>>(t, out, n);
  CUDA_OK(cudaGetLastError());
  SAMP_END
}

// table [R][totalC] from t [R]; scratch >= R * 4 nf floats
int samp_temb(void* stream, const float* gfp_w, const float* l1_w, const float* l1_b, const float* l2_w, const float* l2_b,
              const float* dense_w, const float* dense_b, int nf, int totalC, const float* t, int R, float* scratch,
              float* table) {
  SAMP_TRY
  const TembWeights w{gfp_w, l1_w, l1_b, l2_w, l2_b, dense_w, dense_b, nf, totalC};
  launch_temb(S(stream), w, t, R, scratch, table);
  SAMP_END
}

int samp_pc_update(void* stream, void* state, const void* pyr, int N, int H, int W, const float* ol_w, const float* ol_b,
                   int scale_after, int scale_by_sigma, const float* inv_t, float inv_t_scalar, const void* coef_dev,
                   const void* noise, const void* rng, int draw, void* x_mean_out) {
  SAMP_TRY
  launch_pc_update(S(stream), static_cast<float4*>(state), static_cast<const float4*>(pyr), N, H, W,
                   out_layer(ol_w, ol_b, scale_after, scale_by_sigma), inv_t, inv_t_scalar,
                   static_cast<const UpdateCoef*>(coef_dev), static_cast<const float2*>(noise),
                   static_cast<const RngParams*>(rng), draw, static_cast<float2*>(x_mean_out));
  SAMP_END
}

int samp_affine_update(void* stream, void* state, const void* pyr, int N, int H, int W, const float* ol_w, const float* ol_b,
                       int scale_after, int scale_by_sigma, const void* coef_dev, const void* noise, const void* rng, int draw,
                       int use_noise, void* x_mean_out) {
  SAMP_TRY
  launch_affine_update(S(stream), static_cast<float4*>(state), static_cast<const float4*>(pyr), N, H, W,
                       out_layer(ol_w, ol_b, scale_after, scale_by_sigma), static_cast<const AffineCoef*>(coef_dev),
                       static_cast<const float2*>(noise), static_cast<const RngParams*>(rng), draw, use_noise != 0,
                       static_cast<float2*>(x_mean_out));
  SAMP_END
}

int samp_prior(void* stream, void* state, int N, int H, int W, float std1, const void* noise, const void* rng, int draw) {
  SAMP_TRY
  launch_prior(S(stream), static_cast<float4*>(state), N, H, W, std1, static_cast<const float2*>(noise),
               static_cast<const RngParams*>(rng), draw);
  SAMP_END
}

// scratch >= N * 64 * 2 floats
int samp_langevin_coef(void* stream, const void* pyr, int N, int H, int W, const float* ol_w, const float* ol_b,
                       int scale_after, int scale_by_sigma, float inv_t, const void* noise, const void* rng, int draw,
                       float snr, float* scratch, void* coef_out) {
  SAMP_TRY
  launch_langevin_coef(S(stream), static_cast<const float4*>(pyr), N, H, W, out_layer(ol_w, ol_b, scale_after, scale_by_sigma),
                       inv_t, static_cast<const float2*>(noise), static_cast<const RngParams*>(rng), draw, snr, scratch,
                       static_cast<UpdateCoef*>(coef_out));
  SAMP_END
}

int samp_precond_out(void* stream, const void* x_t, const void* pyr, int N, int H, int W, const float* ol_w, const float* ol_b,
                     int scale_after, int scale_by_sigma, const float* a_dev, const float* b_dev, void* out) {
  SAMP_TRY
  launch_precond_out(S(stream), static_cast<const float2*>(x_t), static_cast<const float4*>(pyr), N, H, W,
                     out_layer(ol_w, ol_b, scale_after, scale_by_sigma), a_dev, b_dev, static_cast<float2*>(out));
  SAMP_END
}

int samp_out_layer(void* stream, const void* pyr, int N, int H, int W, const float* ol_w, const float* ol_b, int scale_after,
                   int scale_by_sigma, const float* t_dev, void* out, int negate) {
  SAMP_TRY
  launch_out_layer(S(stream), static_cast<const float4*>(pyr), N, H, W, out_layer(ol_w, ol_b, scale_after, scale_by_sigma),
                   t_dev, static_cast<float2*>(out), negate != 0);
  SAMP_END
}

int samp_pack_state(void* stream, const void* x, const void* y, int N, int H, int W, void* state) {
  SAMP_TRY
  launch_pack_state(S(stream), static_cast<const float2*>(x), static_cast<const float2*>(y), N, H, W,
                    static_cast<float4*>(state));
  SAMP_END
}

int samp_pack_state_scaled(void* stream, const void* x, const void* y, const float* scale_dev, int N, int H, int W,
                           void* state) {
  SAMP_TRY
  launch_pack_state_scaled(S(stream), static_cast<const float2*>(x), static_cast<const float2*>(y), scale_dev, N, H, W,
                           static_cast<float4*>(state));
  SAMP_END
}

// ---- probability-flow ODE: k[7] device pointers (unused ones may be null), a[7] host coefficients ----
int samp_ode_combine(void* stream, const void* y, void* const* k, int s, const double* a, double h, long long total,
                     void* stage, void* y_new) {
  SAMP_TRY
  launch_ode_combine(S(stream), static_cast<const double2*>(y), odek(k), s, coefs(a), h, (size_t)total,
                     static_cast<float2*>(stage), static_cast<double2*>(y_new));
  SAMP_END
}

int samp_ode_norm(void* stream, int kind, const void* y, const void* y_new, void* const* k, const double* a, double h,
                  double rtol, double atol, long long total, double* partial) {
  SAMP_TRY
  launch_ode_norm(S(stream), kind, static_cast<const double2*>(y), static_cast<const double2*>(y_new), odek(k), coefs(a), h,
                  rtol, atol, (size_t)total, partial);
  SAMP_END
}

int samp_ode_norm_blocks(void) { return kOdeNormBlocks; }

int samp_ode_drift(void* stream, const void* state, const void* pyr, int N, int H, int W, const float* ol_w, const float* ol_b,
                   int scale_after, int scale_by_sigma, float inv_t, float theta, float cs, void* k_out) {
  SAMP_TRY
  launch_ode_drift(S(stream), static_cast<const float4*>(state), static_cast<const float4*>(pyr), N, H, W,
                   out_layer(ol_w, ol_b, scale_after, scale_by_sigma), inv_t, theta, cs, static_cast<float2*>(k_out));
  SAMP_END
}

int samp_ode_drift_affine(void* stream, const void* state, const void* pyr, int N, int H, int W, const float* ol_w,
                          const float* ol_b, int scale_after, int scale_by_sigma, float cx, float cy, float cF, void* k_out) {
  SAMP_TRY
  launch_ode_drift_affine(S(stream), static_cast<const float4*>(state), static_cast<const float4*>(pyr), N, H, W,
                          out_layer(ol_w, ol_b, scale_after, scale_by_sigma), cx, cy, cF, static_cast<float2*>(k_out));
  SAMP_END
}

int samp_ode_init(void* stream, const void* state, long long total, void* y) {
  SAMP_TRY
  launch_ode_init(S(stream), static_cast<const float4*>(state), (size_t)total, static_cast<double2*>(y));
  SAMP_END
}

int samp_ode_finish(void* stream, const void* y, long long total, void* out) {
  SAMP_TRY
  launch_ode_finish(S(stream), static_cast<const double2*>(y), (size_t)total, static_cast<float2*>(out));
  SAMP_END
}

// n systems: y[i], y_new[i] (nullable), stage[i] (combine), k[i * 7 + j], a[i * 7 + j], h[i], total[i], s[i] (combine:
// stage count; norm: kind)
static OdeSysTable sys_table(int n, void* const* y, void* const* y_new, void* const* stage, void* const* k, const double* a,
                             const double* h, const long long* total, const int* s) {
  SG_CHECK(n >= 1 && n <= kOdeSysPerLaunch, "ode groups: 1 .. kOdeSysPerLaunch systems");
  OdeSysTable tab{};
  for (int i = 0; i < n; ++i) {
    OdeSys& q = tab.sys[i];
    q.y = static_cast<const double2*>(y[i]);
    q.y_new = static_cast<double2*>(y_new[i]);
    q.K = odek(k + 7 * i);
    q.c = coefs(a + 7 * i);
    q.h = h[i];
    q.total = (size_t)total[i];
    q.stage = stage ? static_cast<float2*>(stage[i]) : nullptr;
    q.s = s[i];
  }
  return tab;
}

int samp_ode_combine_groups(void* stream, int n, void* const* y, void* const* y_new, void* const* stage, void* const* k,
                            const double* a, const double* h, const long long* total, const int* s) {
  SAMP_TRY
  launch_ode_combine_groups(S(stream), sys_table(n, y, y_new, stage, k, a, h, total, s), n);
  SAMP_END
}

int samp_ode_norm_groups(void* stream, int n, void* const* y, void* const* y_new, void* const* k, const double* a,
                         const double* h, const long long* total, const int* kind, double rtol, double atol, double* partial) {
  SAMP_TRY
  launch_ode_norm_groups(S(stream), sys_table(n, y, y_new, nullptr, k, a, h, total, kind), n, rtol, atol, partial);
  SAMP_END
}

// n rows: x[r], y[r], k_out[r] device pointers; t, c_in, c0, c1 host floats [n]
static OdeRows rows_table(int n, void* const* x, void* const* y, void* const* k_out, const float* t, const float* c_in,
                          const float* c0, const float* c1) {
  SG_CHECK(n >= 1 && n <= kOdeRowsPerLaunch, "ode rows: 1 .. kOdeRowsPerLaunch rows");
  OdeRows rows{};
  for (int r = 0; r < n; ++r) {
    rows.x[r] = static_cast<const float2*>(x[r]);
    rows.y[r] = static_cast<const float2*>(y[r]);
    rows.k_out[r] = k_out ? static_cast<float2*>(k_out[r]) : nullptr;
    rows.t[r] = t[r];
    rows.c_in[r] = c_in[r];
    rows.c0[r] = c0[r];
    rows.c1[r] = c1[r];
  }
  return rows;
}

int samp_ode_rows_pack(void* stream, int n, void* const* x, void* const* y, const float* t, const float* c_in, long long px1,
                       void* state, void* raw, float* t_dev, float* scale_dev) {
  SAMP_TRY
  const OdeRows rows = rows_table(n, x, y, nullptr, t, c_in, c_in, c_in);
  launch_ode_rows_pack(S(stream), rows, n, (size_t)px1, static_cast<float4*>(state), static_cast<float4*>(raw), t_dev,
                       scale_dev);
  SAMP_END
}

int samp_ode_rows_drift(void* stream, int n, void* const* k_out, const float* c0, const float* c1, long long px1,
                        const void* state, const void* pyr, const float* ol_w, const float* ol_b, int scale_after,
                        int scale_by_sigma, float theta, int affine) {
  SAMP_TRY
  const OdeRows rows = rows_table(n, k_out, k_out, k_out, c0, c0, c0, c1);
  launch_ode_rows_drift(S(stream), rows, n, (size_t)px1, static_cast<const float4*>(state), static_cast<const float4*>(pyr),
                        out_layer(ol_w, ol_b, scale_after, scale_by_sigma), theta, affine != 0);
  SAMP_END
}

}  // extern "C"
