// Vector kernels of the probability-flow ODE sampler (SURVEY.md §8f-4): what scipy's RK45 does on host numpy arrays
// in the reference (/root/reference/sgmse/sampling/__init__.py:117-141: flatten -> D2H -> numpy -> H2D per evaluation)
// stays in HBM here.  The integrator state is complex128 like scipy's (`y0.astype(complex)`), the stage derivatives
// are the complex64 values the reference's drift function returns (promoted on use), every network input is the
// complex64 rounding of the fp64 stage (`.type(torch.complex64)`, :121).  All kernels are HBM-bound elementwise /
// reduction passes over [B, F, T] bins (16-32 B per bin), negligible next to one score-network evaluation.
#include "kernels.h"

namespace sgmse {

namespace {

__device__ __forceinline__ double2 lin_comb(const OdeK& K, const OdeCoefs& c, int s, size_t i) {
  double re = 0.0, im = 0.0;
#pragma unroll
  for (int j = 0; j < 7; ++j)
    if (j < s) {
      const float2 k = K.k[j][i];
      re += c.a[j] * (double)k.x;
      im += c.a[j] * (double)k.y;
    }
  return make_double2(re, im);
}

__device__ __forceinline__ double block_sum(double v, double* sh) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sh[w];
  return t;   // valid in thread 0
}

// stage = (complex64)(y + (sum_{j<s} a_j K_j) * h); y_new (optional) keeps the fp64 value (rk_step: `y + dy`,
// `y_new = y + h * np.dot(K[:-1].T, B)`)
__global__ void ode_combine_kernel(const double2* __restrict__ y, OdeK K, int s, OdeCoefs c, double h, size_t total,
                                   float2* __restrict__ stage, double2* __restrict__ y_new) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const double2 yy = y[i];
    const double2 d = lin_comb(K, c, s, i);
    const double re = yy.x + d.x * h, im = yy.y + d.y * h;
    stage[i] = make_float2((float)re, (float)im);
    if (y_new) y_new[i] = make_double2(re, im);
  }
}

__device__ __forceinline__ float2 out_layer_ode(const OutLayer& ol, float4 p, float inv_t) {
  if (!ol.scale_by_sigma) inv_t = 1.f;
  if (!ol.scale_after) { p.x *= inv_t; p.y *= inv_t; p.z *= inv_t; p.w *= inv_t; }
  float re = ol.b[0] + ol.w[0][0] * p.x + ol.w[0][1] * p.y + ol.w[0][2] * p.z + ol.w[0][3] * p.w;
  float im = ol.b[1] + ol.w[1][0] * p.x + ol.w[1][1] * p.y + ol.w[1][2] * p.z + ol.w[1][3] * p.w;
  if (ol.scale_after) { re *= inv_t; im *= inv_t; }
  return make_float2(re, im);
}

// total_drift of RSDE.sde with probability_flow=True (sdes.py:113-127): theta (y - x) - 0.5 g(t)^2 score,
// score = -dnn(cat[x, y], t) = -out_layer(pyr)  ->  k = theta (y - x) + cs * out_layer(pyr),  cs = 0.5 g(t)^2
__global__ void ode_drift_kernel(const float4* __restrict__ state, const float4* __restrict__ pyr, size_t total, OutLayer ol,
                                 float inv_t, float theta, float cs, float2* __restrict__ k_out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float4 s = state[i];
  const float2 d = out_layer_ode(ol, pyr[i], inv_t);
  k_out[i] = make_float2(theta * (s.z - s.x) + cs * d.x, theta * (s.w - s.y) + cs * d.y);
}

// The same drift with the score of a preconditioned 'ncsnpp_v2' model, score = a x + b F, F = output_layer(pyr) of the
// network evaluated on c_in (x, y) (model.py:283-304):  k = cx x + cy y + cF F  with the host-folded coefficients
// cx = -theta - 0.5 g^2 a,  cy = theta,  cF = -0.5 g^2 b.
__global__ void ode_drift_affine_kernel(const float4* __restrict__ state, const float4* __restrict__ pyr, size_t total, OutLayer ol,
                                        float cx, float cy, float cF, float2* __restrict__ k_out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float4 s = state[i];
  const float2 d = out_layer_ode(ol, pyr[i], 1.0f);
  k_out[i] = make_float2(cx * s.x + cy * s.z + cF * d.x, cx * s.y + cy * s.w + cF * d.y);
}

__global__ void ode_init_kernel(const float4* __restrict__ state, size_t total, double2* __restrict__ y) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float4 s = state[i];
  y[i] = make_double2((double)s.x, (double)s.y);
}

__global__ void ode_finish_kernel(const double2* __restrict__ y, size_t total, float2* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const double2 v = y[i];
  out[i] = make_float2((float)v.x, (float)v.y);
}

// partial[block] = sum |v / scale|^2 over the block's bins (common.norm without the final sqrt(./n)):
//   kind 0: v = y            scale = atol + |y| rtol                      (select_initial_step d0)
//   kind 1: v = K0           same scale                                    (d1)
//   kind 2: v = K1 - K0      same scale                                    (d2 * h0)
//   kind 3: v = (sum_j E_j K_j) h,  scale = atol + max(|y|, |y_new|) rtol  (_estimate_error_norm)
__global__ void ode_norm_kernel(int kind, const double2* __restrict__ y, const double2* __restrict__ y_new, OdeK K, OdeCoefs c,
                                double h, double rtol, double atol, size_t total, double* __restrict__ partial) {
  __shared__ double sh[32];
  double acc = 0.0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const double2 yy = y[i];
    double ay = hypot(yy.x, yy.y);
    double2 v;
    if (kind == 0) v = yy;
    else if (kind == 1) { const float2 k = K.k[0][i]; v = make_double2((double)k.x, (double)k.y); }
    else if (kind == 2) {
      const float2 k0 = K.k[0][i], k1 = K.k[1][i];
      v = make_double2((double)k1.x - (double)k0.x, (double)k1.y - (double)k0.y);
    } else {
      const double2 d = lin_comb(K, c, 7, i);
      v = make_double2(d.x * h, d.y * h);
      const double2 yn = y_new[i];
      ay = fmax(ay, hypot(yn.x, yn.y));
    }
    const double scale = atol + ay * rtol;
    const double a = v.x / scale, b = v.y / scale;
    acc += a * a + b * b;
  }
  const double t = block_sum(acc, sh);
  if (threadIdx.x == 0) partial[blockIdx.x] = t;
}

}  // namespace

static unsigned grid_for(size_t total, unsigned cap) {
  const size_t b = (total + 255) / 256;
  return (unsigned)std::max<size_t>(1, std::min<size_t>(b, cap));
}

void launch_ode_combine(cudaStream_t st, const double2* y, const OdeK& K, int s, const OdeCoefs& c, double h, size_t total,
                        float2* stage, double2* y_new) {
  ode_combine_kernel<<<grid_for(total, 132 * 16), 256, 0, st>>>(y, K, s, c, h, total, stage, y_new);
  CUDA_OK(cudaGetLastError());
}
void launch_ode_drift(cudaStream_t st, const float4* state, const float4* pyr, int N, int H, int W, const OutLayer& ol,
                      float inv_t, float theta, float cs, float2* k_out) {
  const size_t total = (size_t)N * H * W;
  ode_drift_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(state, pyr, total, ol, inv_t, theta, cs, k_out);
  CUDA_OK(cudaGetLastError());
}
void launch_ode_drift_affine(cudaStream_t st, const float4* state, const float4* pyr, int N, int H, int W, const OutLayer& ol,
                             float cx, float cy, float cF, float2* k_out) {
  const size_t total = (size_t)N * H * W;
  ode_drift_affine_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(state, pyr, total, ol, cx, cy, cF, k_out);
  CUDA_OK(cudaGetLastError());
}
void launch_ode_init(cudaStream_t st, const float4* state, size_t total, double2* y) {
  ode_init_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(state, total, y);
  CUDA_OK(cudaGetLastError());
}
void launch_ode_finish(cudaStream_t st, const double2* y, size_t total, float2* out) {
  ode_finish_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(y, total, out);
  CUDA_OK(cudaGetLastError());
}
void launch_ode_norm(cudaStream_t st, int kind, const double2* y, const double2* y_new, const OdeK& K, const OdeCoefs& c, double h,
                     double rtol, double atol, size_t total, double* partial) {
  ode_norm_kernel<<<kOdeNormBlocks, 256, 0, st>>>(kind, y, y_new, K, c, h, rtol, atol, total, partial);
  CUDA_OK(cudaGetLastError());
}

}  // namespace sgmse
