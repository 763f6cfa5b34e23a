// Host-side launcher interface of the sgmse_b200 CUDA kernels (internal; the public boundary is
// include/sgmse_b200.h).  All activations are NHWC; "stats" are per-(sample, slot, channel)
// partial (sum, sum of squares) written by the producer of a tensor and consumed by gn_finalize.
#pragma once
#include <algorithm>
#include <cstring>

#include "common.cuh"

namespace sgmse {

enum DType { DT_F32 = 0, DT_F16 = 1 };
static inline size_t dt_size(DType d) { return d == DT_F32 ? 4 : 2; }

struct TensorDesc {
  void* p = nullptr;
  int N = 0, H = 0, W = 0, C = 0;
  DType dt = DT_F32;
  float* stats = nullptr;  // [N][slots][C][2]; capacity = N * (H*W/32) * C * 2 floats
  int slots = 0;           // set by the producing launcher
  size_t numel() const { return (size_t)N * H * W * C; }
  size_t bytes() const { return numel() * dt_size(dt); }
  size_t stats_capacity_floats() const { return (size_t)N * std::max<size_t>(1, (size_t)H * W / 32) * C * 2; }
};

// ---- GroupNorm ----
// ab[n][c] = (a, b) with y = a*x + b  (a = gamma*rstd, b = beta - mean*rstd*gamma), eps = 1e-6
void launch_gn_finalize(cudaStream_t st, const TensorDesc& s0, const TensorDesc* s1, const float* gamma,
                        const float* beta, int groups, float2* ab, unsigned int* range_flag = nullptr);   // += 1 per (sample, group) whose fp16 input overflowed (non-finite sums)
// stand-alone per-(sample, channel) statistics (slots = 1) for levels too small for per-tile partials
void launch_channel_stats(cudaStream_t st, TensorDesc& t);
enum Resample { RS_NONE = 0, RS_DOWN = 1, RS_UP = 2 };
// out0 = [silu](a*x+b) (concat of x0,x1), optionally FIR-resampled; out1 (optional) = FIR-resampled raw x0
void launch_gn_apply(cudaStream_t st, const TensorDesc& x0, const TensorDesc* x1, const float2* ab, bool silu,
                     Resample rs, TensorDesc& out0, TensorDesc* out1);

// gn_self (round 2, on by default since): GroupNorm finalize folded into the plain apply for tensors with H*W <= 512 (see gn.cu)
extern thread_local int g_gnfin_variant;   // 1: gn_finalize with its partial loads batched eight at a time (round 2, the default since; bit-identical)
extern thread_local int g_gn_self;
bool gn_self_applies(const TensorDesc& x0, const TensorDesc* x1);
void launch_gn_norm_apply(cudaStream_t st, const TensorDesc& x0, const TensorDesc* x1, const float* gamma, const float* beta,
                          int groups, bool silu, TensorDesc& out, unsigned int* range_flag = nullptr);
extern thread_local int g_fir_variant;   // 0: one-MUFU (tanh-form) silu + half2 FIR-down arithmetic in the tiled fp16 kernels; 1: expf silu, fp32 FIR
                            // 2: 0 + phase-1 loads in flight at once + half2 quad FIR-up (round 2, the default since; see gn.cu)

// ---- convolutions ----
struct ConvSeg {
  TensorDesc src;
  int taps = 9;  // 9 (3x3, pad 1) or 1 (1x1)
};
struct ConvArgs {
  int nseg = 0;
  ConvSeg seg[3];
  const void* w_direct = nullptr;  // [Ktot][Cout], element type of the activations
  const void* w_tc = nullptr;      // [Cout][w_tc_ld] (K-major rows): fp16, or fp32 holding TF32 values (tf32_rna) for fp32 activations
  int w_tc_ld = 0;                 // row length in elements (>= ktot())
  bool tc_identity_tail = false;   // columns [ktot, ktot+Cout) hold I: the residual may be fed as a K segment
  const float* bias = nullptr;     // [Cout] (nullable)
  const float* temb = nullptr;     // per-(row, channel) additive bias table (nullable)
  int temb_stride = 0;             // floats between consecutive samples' rows (0: all samples share)
  const TensorDesc* residual = nullptr;
  float scale = 1.f;               // out = (acc + bias + temb + residual) * scale
  // Fused GroupNorm-apply + SiLU (conv_tc only): seg[0] (3x3) reads RAW tensors -- seg[0].src, concatenated with
  // gn_cat when gn_has_cat -- and applies silu(a*x+b) with (a, b) = gn_ab[n][channel] on the way into shared memory.
  const float2* gn_ab = nullptr;
  bool gn_has_cat = false;
  TensorDesc gn_cat;
  int ktot() const {
    int k = 0;
    for (int i = 0; i < nseg; ++i) k += seg[i].taps * (seg[i].src.C + (i == 0 && gn_has_cat ? gn_cat.C : 0));
    return k;
  }
};
void launch_conv_direct(cudaStream_t st, const ConvArgs& a, TensorDesc& out);
// wgmma implicit GEMM (conv_tc.cu); requires Cout % 64 == 0 and either fp16 activations with every segment C % 64 == 0, or
// fp32 activations (TF32 operands) with every segment C % 32 == 0
bool conv_tc_supported(const ConvArgs& a, const TensorDesc& out);
// shape test of the fused GroupNorm-apply/SiLU form (3x3 over c0 [+ c1] raw channels), usable before the tensors exist
bool conv_tc_fuse_shape_ok(int H, int W, int c0, int c1, int cout);
void launch_conv_tc(cudaStream_t st, const ConvArgs& a, TensorDesc& out, int* dbg_flag);
// Launch plan of conv_tc for an output tensor: the host-side decision launch_conv_tc acts on.
struct TcPlan {
  int bw = 0, bh = 0, bn = 0;          // pixel box of one 128-row tile (bw * bh * bn = 128); bw == 0: no box fits H x W
  int block_n = 0, stages = 0;         // channel tile width, shared-memory ring depth
  int tiles = 0, grid = 0;             // output tiles, persistent CTAs
  int min_local = 0, max_local = 0;    // tiles per CTA
};
// sms: multiprocessors the grid is sized for; narrow: g_tc1_narrow
TcPlan conv_tc_plan(const TensorDesc& out, int sms, bool narrow);
extern thread_local int g_tc1_narrow;   // 1: 64-wide channel tiles when 128-wide ones fill less than half the SMs (the default)
extern thread_local int g_tc_variant;   // 0: TMA-fed convolutions, separate gn_apply launches; 5: GroupNorm+SiLU fused into the 3x3
                                        // convolutions where the shape allows (its producer re-evaluates every tap: 3.2x slower per benchmark step on H100)

// input layer: state float4 (x.re,x.im,y.re,y.im) -> conv3x3(4->C); w [36][C] (k = tap*4+cin), bias [C]
// in_scale multiplies the state on the way in (c_in of the preconditioned 'ncsnpp_v2' forward, model.py:284,312-319);
// not_centered maps every in-bounds input value x to 2x - 1 first (--no-centered, ncsnpp.py:288-290), padding stays zero
void launch_input_conv(cudaStream_t st, const float4* state, int N, int H, int W, const float* w,
                       const float* bias, TensorDesc& out, float in_scale = 1.f, bool not_centered = false);
// Combine('sum'): out = conv1x1_{4->C}(pyr) + bias + h ; pyr float4 [N,H,W]; w [4][C]
void launch_combine(cudaStream_t st, const float4* pyr, const float* w, const float* bias, const TensorDesc& h,
                    TensorDesc& out);
// 4-channel FIR resample of the input/output pyramids
// `scale` multiplies the result (the input pyramid of a c_in-scaled network input starts from the unscaled state)
void launch_fir4(cudaStream_t st, const float4* in, int N, int H, int W, Resample rs, float4* out, float scale = 1.f,
                 const float* scale_rows = nullptr,    // scale_rows (device, nullable): one scale per sample instead
                 bool not_centered = false);           // RS_DOWN only: taps read 2x - 1 for x (the input pyramid's first level)
// out4 = conv3x3_{C->4}(act) + bias (+ addend);  w [9*C][4] (device), bias: HOST pointer to 4 floats
// gn_ab != nullptr: `act` is the RAW tensor and silu(a*x+b) is applied while staging (only when out_conv_fuses_gn(act))
bool out_conv_fuses_gn(const TensorDesc& act);
// wfrag (optional): the fp16 mma.sync B fragments of w packed at load time ([9][C/16][32] uint2), else built per block
void launch_out_conv(cudaStream_t st, const TensorDesc& act, const float* w, const float* bias,
                     const float4* addend, float4* out, const float2* gn_ab = nullptr, const uint2* wfrag = nullptr);
extern thread_local int g_outconv_variant;   // 0: mma.sync kernel for fp16 C in {128, 256}; 1: CUDA-core kernels; 2: mma.sync kernel with
                                // GroupNorm+SiLU fused into its staging
                                // 3: the mma.sync kernel with its tile staged by cp.async (round 2, the default since; see small.cu)
extern thread_local int g_combine_variant;   // 0: thread per channel (2-byte accesses); 1: thread per 8-channel vector (round 2, the default since; bit-identical)
extern thread_local int g_inconv_variant;    // 0: mma.sync input conv for fp16 C in {32, 64, 128}; 1: CUDA-core kernel; 2: 0 with prefetched A fragments (round 2, the default since)

// ---- attention: qkv [N,H,W,3C] (q|k|v), out [N,H,W,C] = softmax(q k^T / sqrt(C)) v over H*W tokens
void launch_attention(cudaStream_t st, const TensorDesc& qkv, TensorDesc& out);
extern thread_local int g_attn_variant;   // 0 (= 2): fp16 mma.sync flash kernel with cp.async tile staging (C in {128,256}); 1: fp32 CUDA-core
                                          // kernel; 3: the mma.sync kernel with plain (LDG/STS) tile staging

// ---- time embedding ----
struct TembWeights {
  const float* gfp_w;   // [nf]
  const float* l1_w;    // [4nf][2nf]
  const float* l1_b;    // [4nf]
  const float* l2_w;    // [4nf][4nf]
  const float* l2_b;
  const float* dense_w; // [totalC][4nf]  (all Dense_0 stacked)
  const float* dense_b; // [totalC]       (Dense_0.bias + Conv_0.bias)
  int nf, totalC;
};
// table[r][totalC] for r < R, from t[r]; scratch >= R*4nf floats
void launch_temb(cudaStream_t st, const TembWeights& w, const float* t, int R, float* scratch, float* table);

// ---- SDE / sampler ----
struct OutLayer {  // output_layer conv1x1(4->2) (+ the /t ordering of the backbone)
  float w[2][4];
  float b[2];
  int scale_after;  // 0: conv(p/t) (ncsnpp)   1: conv(p)/t (ncsnpp_48k)
  int scale_by_sigma;
};
struct RngParams {  // lives in device memory so that CUDA graphs can be re-launched with a new seed
  unsigned long long seed;
  int utt0;
  int pad;
};
struct UpdateCoef {  // x_mean = x + cy*(y-x) + cs*score ; x' = x_mean + cz*z
  float cy, cs, cz;
};
// state <- state with x replaced; score = -out_layer(pyr, 1/t).  coef read from device memory.
// noise: injected complex normals [N,H,W] (float2) or nullptr -> Philox(rng->seed, rng->utt0+n, draw).
void launch_pc_update(cudaStream_t st, float4* state, const float4* pyr, int N, int H, int W, const OutLayer& ol,
                      const float* inv_t /*device [N] or nullptr->use inv_t_scalar*/, float inv_t_scalar,
                      const UpdateCoef* coef_dev, const float2* noise, const RngParams* rng, int draw,
                      float2* x_mean_out /*nullable*/);
// dnn forward output only: out[n,h,w] = out_layer(pyr, 1/t[n])  (complex64)
void launch_out_layer(cudaStream_t st, const float4* pyr, int N, int H, int W, const OutLayer& ol, const float* t_dev,
                      float2* out, bool negate);
void launch_pack_state(cudaStream_t st, const float2* x, const float2* y, int N, int H, int W, float4* state);
// state = scale[n] * (x, y)   (per-sample c_in of ScoreModel.forward with a vector of times)
void launch_pack_state_scaled(cudaStream_t st, const float2* x, const float2* y, const float* scale_dev, int N, int H, int W,
                              float4* state);
// General one-step update (Schroedinger-bridge samplers, sampling/__init__.py:165-181,211-233, and every sampler on the
// preconditioned 'ncsnpp_v2' model): with F = output_layer(pyr) (no in-network scaling),
//   x_mean = cx * x + cF * F + cy * y ;  x = x_mean + cz * z     (z drawn only when use_noise)
struct AffineCoef {
  float cx, cF, cy, cz;
};
void launch_affine_update(cudaStream_t st, float4* state, const float4* pyr, int N, int H, int W, const OutLayer& ol,
                          const AffineCoef* coef_dev, const float2* noise, const RngParams* rng, int draw, bool use_noise,
                          float2* x_mean_out /*nullable*/);
// out[n] = a[n] * x_t + b[n] * output_layer(pyr)   (ScoreModel.forward of the 'ncsnpp_v2' branch, model.py:296-304)
void launch_precond_out(cudaStream_t st, const float2* x_t, const float4* pyr, int N, int H, int W, const OutLayer& ol,
                        const float* a_dev, const float* b_dev, float2* out);
// state.x = y + std1 * z
void launch_prior(cudaStream_t st, float4* state, int N, int H, int W, float std1, const float2* noise,
                  const RngParams* rng, int draw);
// Langevin corrector step size from batch-mean norms: coef = (0, eps, sqrt(2 eps)), eps = 2 (snr*|z|/|g|)^2
void launch_langevin_coef(cudaStream_t st, const float4* pyr, int N, int H, int W, const OutLayer& ol, float inv_t,
                          const float2* noise, const RngParams* rng, int draw, float snr, float* scratch,
                          UpdateCoef* coef_out);

// ---- probability-flow ODE sampler (SURVEY.md §8f-4; ode.cu, controller in rk45.h) ----
struct OdeK { const float2* k[7]; };   // stage derivatives K_0..K_6, complex64 like the reference's drift_fn output
struct OdeCoefs { double a[7]; };
constexpr int kOdeNormBlocks = 528;    // 4 x 132 SMs; one fp64 partial per block, summed on the host in block order
// stage = (complex64)(y + (sum_{j<s} a_j K_j) * h); y_new (nullable) receives the fp64 value
void launch_ode_combine(cudaStream_t st, const double2* y, const OdeK& K, int s, const OdeCoefs& c, double h, size_t total,
                        float2* stage, double2* y_new);
// k_out = theta (y - x) + cs * out_layer(pyr, inv_t)   [= theta (y - x) - 0.5 g^2 score, score = -dnn]; state = (x, y)
void launch_ode_drift(cudaStream_t st, const float4* state, const float4* pyr, int N, int H, int W, const OutLayer& ol,
                      float inv_t, float theta, float cs, float2* k_out);
// k_out = cx x + cy y + cF * output_layer(pyr)   (score of a preconditioned 'ncsnpp_v2' model folded in, see ode.cu)
void launch_ode_drift_affine(cudaStream_t st, const float4* state, const float4* pyr, int N, int H, int W, const OutLayer& ol,
                             float cx, float cy, float cF, float2* k_out);
void launch_ode_init(cudaStream_t st, const float4* state, size_t total, double2* y);     // y = (complex128) state.x
void launch_ode_finish(cudaStream_t st, const double2* y, size_t total, float2* out);     // out = (complex64) y
// partial[kOdeNormBlocks]: per-block sums of |v/scale|^2, see ode.cu for the four kinds
void launch_ode_norm(cudaStream_t st, int kind, const double2* y, const double2* y_new, const OdeK& K, const OdeCoefs& c, double h,
                     double rtol, double atol, size_t total, double* partial);
// Independent systems side by side (ode_sample_groups).  A launch covers up to kOdeSysPerLaunch systems; each system's
// blocks do the single-system kernels' arithmetic over its own bins (the norm in kOdeNormBlocks blocks per system).
constexpr int kOdeSysPerLaunch = 16;
struct OdeSys {              // combine: stage = y + (sum_{j<s} c_j K_j) h, y_new nullable;  norm: kind s, E = c
  const double2* y;
  double2* y_new;
  OdeK K;
  OdeCoefs c;
  double h;
  size_t total;              // bins of this system
  float2* stage;
  int s;
};
struct OdeSysTable { OdeSys sys[kOdeSysPerLaunch]; };
void launch_ode_combine_groups(cudaStream_t st, const OdeSysTable& tab, int n);
// partial[i * kOdeNormBlocks + b]: block b's sum of system i, as launch_ode_norm writes it for that system alone
void launch_ode_norm_groups(cudaStream_t st, const OdeSysTable& tab, int n, double rtol, double atol, double* partial);
// The rows (utterances) of one batched network evaluation: each row's stage x and conditioning y, where its drift
// goes, its time, its c_in, and its drift coefficients (inv_t, cs) or, affine, (cx, cF).
constexpr int kOdeRowsPerLaunch = 32;
struct OdeRows {
  const float2* x[kOdeRowsPerLaunch];
  const float2* y[kOdeRowsPerLaunch];
  float2* k_out[kOdeRowsPerLaunch];
  float t[kOdeRowsPerLaunch], c_in[kOdeRowsPerLaunch], c0[kOdeRowsPerLaunch], c1[kOdeRowsPerLaunch];
};
// state[r] = c_in (x, y) and raw[r] = (x, y) with raw != NULL, else state[r] = (x, y); t_dev / scale_dev (nullable) get t, c_in
void launch_ode_rows_pack(cudaStream_t st, const OdeRows& rows, int n, size_t px1, float4* state, float4* raw, float* t_dev,
                          float* scale_dev);
// launch_ode_drift (affine: launch_ode_drift_affine) per row, state unscaled
void launch_ode_rows_drift(cudaStream_t st, const OdeRows& rows, int n, size_t px1, const float4* state, const float4* pyr,
                           const OutLayer& ol, float theta, bool affine);

// ---- STFT front/back end (cuFFT plans live in the engine) ----
void launch_absmax(cudaStream_t st, const float* wav, int B, int L, float* norm);
void launch_frame(cudaStream_t st, const float* wav, const float* norm, int B, int L, int n_fft, int hop, int nT,
                  int sqrt_window, float* frames);
void launch_spec_fwd(cudaStream_t st, const float2* spec /*[B*nT][fstride]*/, int B, int nT, int F, int fstride,
                     int Tpad, float factor, float expo, int transform /* SGMSE_B200_TRANSFORM_* */, int reflect_pad,
                     float2* Y /*[B][F][Tpad]*/);
void launch_spec_back(cudaStream_t st, const float2* X /*[B][F][Tpad]*/, int B, int F, int Tpad, int fstride,
                          float factor, float expo, int transform, float2* spec /*[B*Tpad][fstride]*/);
void launch_overlap_add(cudaStream_t st, const float* frames, const float* norm, int B, int Tpad, int n_fft, int hop,
                        int sqrt_window, int L, float* wav);

// ---- device-side weight packing (pack.cu; engine.cu: load_weights_device) ----
struct PackSeg { long long w; int cin, taps, kbase; };
struct PackJob { PackSeg seg[4]; int nseg, cout, ktot, ld, mode, identity_tail; };
void launch_pack_conv(cudaStream_t st, const float* blob, const PackJob& j, void* kd, bool kd_half, __half* ht);
// conv_tc's TF32 weight operand: wt[co][ld] = tf32_rna(kd[k][co]) for k < ktot, from the fp32 [ktot][cout] direct layout
void launch_pack_tc_tf32(cudaStream_t st, const float* kd, int ktot, int cout, int ld, float* wt);
// fp32 -> the nearest TF32 value (10 mantissa bits), ties away from zero (the rounding of cvt.rna.tf32.f32); the same
// integer arithmetic on host and device, so both weight packers agree bit for bit
__host__ __device__ inline float tf32_rna(float v) {
  uint32_t u;
  memcpy(&u, &v, 4);
  if ((u & 0x7F800000u) != 0x7F800000u) u = (u + 0x1000u) & 0xFFFFE000u;   // Inf and NaN pass through
  memcpy(&v, &u, 4);
  return v;
}
void launch_pack_inconv(cudaStream_t st, const float* w, int nf, float* out);
void launch_pack_combine(cudaStream_t st, const float* w, int C, float* out);
void launch_pack_outconv(cudaStream_t st, const float* w, int C, float* out, uint2* frag);
void launch_add_vec(cudaStream_t st, const float* a, const float* b, float* out, int n);

}  // namespace sgmse
