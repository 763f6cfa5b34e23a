// Time embedding tables, the fused predictor/corrector update (with the network's final
// /t + conv1x1(4->2) folded in), in-kernel Philox noise, and the STFT/iSTFT pre/post kernels.
//
// Reference: layerspp.py:32-41 + ncsnpp.py:267-284 (time embedding), ncsnpp.py:411-418 /
// ncsnpp_48k.py:414-424 (output layer), sdes.py:188-229, predictors.py:41-76,
// correctors.py:37-94 (update rules), data_module.py:162-218 (STFT chain), util/other.py:76-90.
#include "../../include/sgmse_b200.h"
#include "kernels.h"

namespace sgmse {

thread_local int g_pdl = 0;                 // see common.cuh
bool pdl_compiled() {
#ifdef SGMSE_B200_PDL
  return true;
#else
  return false;
#endif
}

// ================================================================================================
// time embedding
// ================================================================================================
__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// grid R, block 256.  scratch[r][4nf] = silu(Linear2(silu(Linear1(gfp(log t_r)))))
__global__ void temb_mlp_kernel(TembWeights w, const float* __restrict__ t, float* __restrict__ scratch) {
  extern __shared__ float sm[];
  const int nf = w.nf, E = 2 * nf, D = 4 * nf;
  float* emb = sm;       // [2nf]
  float* h1 = emb + E;   // [4nf]
  const int r = blockIdx.x;
  const float lt = logf(t[r]);
  for (int j = threadIdx.x; j < nf; j += blockDim.x) {
    // x_proj = x[:, None] * W[None, :] * 2 * np.pi  (layerspp.py:40), evaluated left to right in fp32
    const float pr = ((lt * w.gfp_w[j]) * 2.0f) * 3.14159265358979323846f;
    emb[j] = sinf(pr);
    emb[nf + j] = cosf(pr);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int o = warp; o < D; o += nw) {
    const float* row = w.l1_w + (size_t)o * E;
    float s = 0.f;
    for (int j = lane; j < E; j += 32) s = fmaf(row[j], emb[j], s);
    s = warp_sum(s);
    if (lane == 0) h1[o] = silu_f(s + w.l1_b[o]);
  }
  __syncthreads();
  for (int o = warp; o < D; o += nw) {
    const float* row = w.l2_w + (size_t)o * D;
    float s = 0.f;
    for (int j = lane; j < D; j += 32) s = fmaf(row[j], h1[j], s);
    s = warp_sum(s);
    if (lane == 0) scratch[(size_t)r * D + o] = silu_f(s + w.l2_b[o]);
  }
}

// grid (ceil(totalC/8), R), block 256 (warp per output column)
__global__ void temb_dense_kernel(TembWeights w, const float* __restrict__ scratch, float* __restrict__ table) {
  const int D = 4 * w.nf;
  const int col = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31, r = blockIdx.y;
  if (col >= w.totalC) return;
  const float* row = w.dense_w + (size_t)col * D;
  const float* s = scratch + (size_t)r * D;
  float acc = 0.f;
  for (int j = lane; j < D; j += 32) acc = fmaf(row[j], s[j], acc);
  acc = warp_sum(acc);
  if (lane == 0) table[(size_t)r * w.totalC + col] = acc + w.dense_b[col];
}

void launch_temb(cudaStream_t st, const TembWeights& w, const float* t, int R, float* scratch, float* table) {
  const size_t smem = (size_t)(6 * w.nf) * sizeof(float);
  temb_mlp_kernel<<<R, 256, smem, st>>>(w, t, scratch);
  CUDA_OK(cudaGetLastError());
  dim3 grid(cdiv(w.totalC, 8), R);
  temb_dense_kernel<<<grid, 256, 0, st>>>(w, scratch, table);
  CUDA_OK(cudaGetLastError());
}

// ================================================================================================
// Philox4x32-10 -> complex normal CN(0,1) (real, imag ~ N(0, 1/2)), keyed by
// (seed, global utterance id, draw index, pixel index): invariant to how the batch is sharded.
// ================================================================================================
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    const uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0; key.y += W1;
  }
  return ctr;
}
__device__ __forceinline__ float2 complex_normal(uint64_t seed, uint32_t utt, uint32_t draw, uint32_t pix) {
  const uint4 r = philox4x32_10(make_uint4(pix, draw, utt, 0x5347u), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  const float u1 = ((float)r.x + 1.0f) * 2.3283064365386963e-10f;  // (0, 1]
  const float u2 = (float)r.y * 2.3283064365386963e-10f;
  const float rad = sqrtf(-logf(u1));  // sqrt(-2 ln u1) * sqrt(1/2)
  float s, c;
  sincospif(2.0f * u2, &s, &c);
  return make_float2(rad * c, rad * s);
}
__device__ __forceinline__ float2 draw_noise(const float2* noise, size_t idx, const RngParams* rng, int n, int draw, uint32_t pix) {
  return noise ? noise[idx] : complex_normal(rng->seed, (uint32_t)(rng->utt0 + n), (uint32_t)draw, pix);
}

__device__ __forceinline__ float2 out_layer(const OutLayer& ol, float4 p, float inv_t) {
  if (!ol.scale_by_sigma) inv_t = 1.f;
  if (!ol.scale_after) { p.x *= inv_t; p.y *= inv_t; p.z *= inv_t; p.w *= inv_t; }
  float re = ol.b[0] + ol.w[0][0] * p.x + ol.w[0][1] * p.y + ol.w[0][2] * p.z + ol.w[0][3] * p.w;
  float im = ol.b[1] + ol.w[1][0] * p.x + ol.w[1][1] * p.y + ol.w[1][2] * p.z + ol.w[1][3] * p.w;
  if (ol.scale_after) { re *= inv_t; im *= inv_t; }
  return make_float2(re, im);
}

__global__ void pc_update_kernel(float4* __restrict__ state, const float4* __restrict__ pyr, int HW, size_t total,
                                 OutLayer ol, const float* __restrict__ inv_t_dev, float inv_t_scalar,
                                 const UpdateCoef* __restrict__ coef_dev, const float2* __restrict__ noise,
                                 const RngParams* rng, int draw, float2* __restrict__ x_mean_out) {
  pdl_trigger(); pdl_wait();
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int n = (int)(idx / HW);
  const uint32_t pix = (uint32_t)(idx - (size_t)n * HW);
  const UpdateCoef cf = *coef_dev;
  const float inv_t = inv_t_dev ? inv_t_dev[n] : inv_t_scalar;
  const float2 d = out_layer(ol, pyr[idx], inv_t);   // dnn output; score = -d
  float4 s = state[idx];
  const float2 z = draw_noise(noise, idx, rng, n, draw, pix);
  const float mre = s.x + cf.cy * (s.z - s.x) - cf.cs * d.x;
  const float mim = s.y + cf.cy * (s.w - s.y) - cf.cs * d.y;
  s.x = mre + cf.cz * z.x;
  s.y = mim + cf.cz * z.y;
  state[idx] = s;
  if (x_mean_out) x_mean_out[idx] = make_float2(mre, mim);
}

void launch_pc_update(cudaStream_t st, float4* state, const float4* pyr, int N, int H, int W, const OutLayer& ol,
                      const float* inv_t, float inv_t_scalar, const UpdateCoef* coef_dev, const float2* noise,
                      const RngParams* rng, int draw, float2* x_mean_out) {
  const size_t total = (size_t)N * H * W;
  launch_k(pc_update_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, st, state, pyr, H * W, total, ol, inv_t, inv_t_scalar,
                                                                    coef_dev, noise, rng, draw, x_mean_out);
  CUDA_OK(cudaGetLastError());
}

__global__ void affine_update_kernel(float4* __restrict__ state, const float4* __restrict__ pyr, int HW, size_t total,
                                     OutLayer ol, const AffineCoef* __restrict__ coef_dev, const float2* __restrict__ noise,
                                     const RngParams* rng, int draw, int use_noise, float2* __restrict__ x_mean_out) {
  pdl_trigger(); pdl_wait();
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int n = (int)(idx / HW);
  const AffineCoef cf = *coef_dev;
  const float2 d = out_layer(ol, pyr[idx], 1.0f);
  float4 s = state[idx];
  const float mre = cf.cx * s.x + cf.cF * d.x + cf.cy * s.z;
  const float mim = cf.cx * s.y + cf.cF * d.y + cf.cy * s.w;
  float2 z = make_float2(0.f, 0.f);
  if (use_noise) z = draw_noise(noise, idx, rng, n, draw, (uint32_t)(idx - (size_t)n * HW));
  s.x = mre + cf.cz * z.x;
  s.y = mim + cf.cz * z.y;
  state[idx] = s;
  if (x_mean_out) x_mean_out[idx] = make_float2(mre, mim);
}
void launch_affine_update(cudaStream_t st, float4* state, const float4* pyr, int N, int H, int W, const OutLayer& ol,
                          const AffineCoef* coef_dev, const float2* noise, const RngParams* rng, int draw, bool use_noise,
                          float2* x_mean_out) {
  const size_t total = (size_t)N * H * W;
  launch_k(affine_update_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, st, state, pyr, H * W, total, ol, coef_dev, noise, rng,
                                                                        draw, use_noise ? 1 : 0, x_mean_out);
  CUDA_OK(cudaGetLastError());
}

__global__ void precond_out_kernel(const float2* __restrict__ x_t, const float4* __restrict__ pyr, int HW, size_t total,
                                   OutLayer ol, const float* __restrict__ a_dev, const float* __restrict__ b_dev,
                                   float2* __restrict__ out) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int n = (int)(idx / HW);
  const float2 d = out_layer(ol, pyr[idx], 1.0f);
  const float2 x = x_t[idx];
  const float a = a_dev[n], b = b_dev[n];
  out[idx] = make_float2(a * x.x + b * d.x, a * x.y + b * d.y);
}
void launch_precond_out(cudaStream_t st, const float2* x_t, const float4* pyr, int N, int H, int W, const OutLayer& ol,
                        const float* a_dev, const float* b_dev, float2* out) {
  const size_t total = (size_t)N * H * W;
  precond_out_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x_t, pyr, H * W, total, ol, a_dev, b_dev, out);
  CUDA_OK(cudaGetLastError());
}

__global__ void out_layer_kernel(const float4* __restrict__ pyr, int HW, size_t total, OutLayer ol,
                                 const float* __restrict__ t_dev, float2* __restrict__ out, float sign) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int n = (int)(idx / HW);
  const float2 d = out_layer(ol, pyr[idx], 1.0f / t_dev[n]);
  out[idx] = make_float2(sign * d.x, sign * d.y);
}
void launch_out_layer(cudaStream_t st, const float4* pyr, int N, int H, int W, const OutLayer& ol, const float* t_dev,
                      float2* out, bool negate) {
  const size_t total = (size_t)N * H * W;
  out_layer_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(pyr, H * W, total, ol, t_dev, out, negate ? -1.f : 1.f);
  CUDA_OK(cudaGetLastError());
}

__global__ void pack_state_kernel(const float2* __restrict__ x, const float2* __restrict__ y, size_t total,
                                  float4* __restrict__ state) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const float2 a = x[idx], b = y[idx];
  state[idx] = make_float4(a.x, a.y, b.x, b.y);
}
void launch_pack_state(cudaStream_t st, const float2* x, const float2* y, int N, int H, int W, float4* state) {
  const size_t total = (size_t)N * H * W;
  pack_state_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, y, total, state);
  CUDA_OK(cudaGetLastError());
}

__global__ void pack_state_scaled_kernel(const float2* __restrict__ x, const float2* __restrict__ y,
                                         const float* __restrict__ scale, int HW, size_t total, float4* __restrict__ state) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const float c = scale[idx / HW];
  const float2 a = x[idx], b = y[idx];
  state[idx] = make_float4(c * a.x, c * a.y, c * b.x, c * b.y);
}
void launch_pack_state_scaled(cudaStream_t st, const float2* x, const float2* y, const float* scale_dev, int N, int H, int W,
                              float4* state) {
  const size_t total = (size_t)N * H * W;
  pack_state_scaled_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, y, scale_dev, H * W, total, state);
  CUDA_OK(cudaGetLastError());
}

__global__ void prior_kernel(float4* __restrict__ state, int HW, size_t total, float std1,
                             const float2* __restrict__ noise, const RngParams* rng, int draw) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int n = (int)(idx / HW);
  float4 s = state[idx];
  const float2 z = draw_noise(noise, idx, rng, n, draw, (uint32_t)(idx - (size_t)n * HW));
  s.x = s.z + z.x * std1;
  s.y = s.w + z.y * std1;
  state[idx] = s;
}
void launch_prior(cudaStream_t st, float4* state, int N, int H, int W, float std1, const float2* noise,
                  const RngParams* rng, int draw) {
  const size_t total = (size_t)N * H * W;
  prior_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(state, H * W, total, std1, noise, rng, draw);
  CUDA_OK(cudaGetLastError());
}

// ---- Langevin corrector step size (correctors.py:45-56): batch-mean norms of grad and noise ----
constexpr int LV_BLOCKS = 64;
__global__ void langevin_norm_kernel(const float4* __restrict__ pyr, int HW, OutLayer ol, float inv_t,
                                     const float2* __restrict__ noise, const RngParams* rng, int draw,
                                     float* __restrict__ partial /*[N][LV_BLOCKS][2]*/) {
  const int n = blockIdx.y;
  float g2 = 0.f, z2 = 0.f;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += gridDim.x * blockDim.x) {
    const size_t idx = (size_t)n * HW + p;
    const float2 d = out_layer(ol, pyr[idx], inv_t);
    const float2 z = draw_noise(noise, idx, rng, n, draw, (uint32_t)p);
    g2 += d.x * d.x + d.y * d.y;
    z2 += z.x * z.x + z.y * z.y;
  }
  __shared__ float sg[8], sz[8];
  g2 = warp_sum(g2); z2 = warp_sum(z2);
  if ((threadIdx.x & 31) == 0) { sg[threadIdx.x >> 5] = g2; sz[threadIdx.x >> 5] = z2; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { a += sg[i]; b += sz[i]; }
    partial[((size_t)n * LV_BLOCKS + blockIdx.x) * 2 + 0] = a;
    partial[((size_t)n * LV_BLOCKS + blockIdx.x) * 2 + 1] = b;
  }
}
__global__ void langevin_coef_kernel(const float* __restrict__ partial, int N, float snr, UpdateCoef* __restrict__ coef) {
  if (threadIdx.x != 0) return;
  double gn = 0.0, zn = 0.0;
  for (int n = 0; n < N; ++n) {
    double a = 0.0, b = 0.0;
    for (int i = 0; i < LV_BLOCKS; ++i) { a += partial[((size_t)n * LV_BLOCKS + i) * 2]; b += partial[((size_t)n * LV_BLOCKS + i) * 2 + 1]; }
    gn += sqrt(a); zn += sqrt(b);
  }
  gn /= N; zn /= N;
  const double r = snr * zn / gn;
  const float eps = (float)(r * r * 2.0);
  coef->cy = 0.f; coef->cs = eps; coef->cz = sqrtf(eps * 2.f);
}
void launch_langevin_coef(cudaStream_t st, const float4* pyr, int N, int H, int W, const OutLayer& ol, float inv_t,
                          const float2* noise, const RngParams* rng, int draw, float snr, float* scratch,
                          UpdateCoef* coef_out) {
  dim3 grid(LV_BLOCKS, N);
  langevin_norm_kernel<<<grid, 256, 0, st>>>(pyr, H * W, ol, inv_t, noise, rng, draw, scratch);
  CUDA_OK(cudaGetLastError());
  langevin_coef_kernel<<<1, 32, 0, st>>>(scratch, N, snr, coef_out);
  CUDA_OK(cudaGetLastError());
}

// ================================================================================================
// STFT / iSTFT glue around cuFFT
// ================================================================================================
__global__ void absmax_kernel(const float* __restrict__ wav, int L, float* __restrict__ norm) {
  const float* y = wav + (size_t)blockIdx.x * L;
  float m = 0.f;
  for (int i = threadIdx.x; i < L; i += blockDim.x) m = fmaxf(m, fabsf(y[i]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ float s[32];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) m = fmaxf(m, s[i]);
    norm[blockIdx.x] = m;
  }
}
void launch_absmax(cudaStream_t st, const float* wav, int B, int L, float* norm) {
  absmax_kernel<<<B, 1024, 0, st>>>(wav, L, norm);
  CUDA_OK(cudaGetLastError());
}

__device__ __forceinline__ float hann_periodic(int i, int n, int sqrt_window) {
  const float w = 0.5f - 0.5f * cospif(2.0f * (float)i / (float)n);
  return sqrt_window ? sqrtf(w) : w;
}

// frames[(b*nT+t)][i] = window[i] * (y_b / norm_b)[reflect(t*hop + i - n_fft/2)]
__global__ void frame_kernel(const float* __restrict__ wav, const float* __restrict__ norm, int L, int n_fft, int hop,
                             int nT, int sqrt_window, float* __restrict__ frames) {
  const int t = blockIdx.x, b = blockIdx.y;
  const float nb = norm[b];
  const float* y = wav + (size_t)b * L;
  float* f = frames + ((size_t)b * nT + t) * n_fft;
  for (int i = threadIdx.x; i < n_fft; i += blockDim.x) {
    int j = t * hop + i - n_fft / 2;
    if (j < 0) j = -j;
    if (j >= L) j = 2 * (L - 1) - j;
    f[i] = hann_periodic(i, n_fft, sqrt_window) * (y[j] / nb);
  }
}
void launch_frame(cudaStream_t st, const float* wav, const float* norm, int B, int L, int n_fft, int hop, int nT,
                  int sqrt_window, float* frames) {
  dim3 grid(nT, B);
  frame_kernel<<<grid, 256, 0, st>>>(wav, norm, L, n_fft, hop, nT, sqrt_window, frames);
  CUDA_OK(cudaGetLastError());
}

// spec_fwd, transpose [b][t][f] -> Y[b][f][t], pad T.  transform (SGMSE_B200_TRANSFORM_*, data_module.py:162-175):
// exponent |z|^e e^{j arg z} * factor, log log(1 + |z|) e^{j arg z} * factor, none z.  The phase factor is z / |z| in both
// magnitude maps, and log(1 + a) is evaluated as the reference writes it, not as log1p.
__global__ void spec_fwd_kernel(const float2* __restrict__ spec, int nT, int F, int fstride, int Tpad,
                                     float factor, float expo, int transform, int reflect_pad, float2* __restrict__ Y) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int f = blockIdx.y, b = blockIdx.z;
  if (t >= Tpad) return;
  int ts = t;
  float2 z = make_float2(0.f, 0.f);
  if (t >= nT) ts = reflect_pad ? (2 * nT - 2 - t) : -1;
  if (ts >= 0) {
    z = spec[((size_t)b * nT + ts) * fstride + f];
    if (transform == SGMSE_B200_TRANSFORM_EXPONENT) {
      if (expo != 1.0f) {
        const float mag = hypotf(z.x, z.y);
        const float g = mag > 0.f ? powf(mag, expo) / mag : 0.f;
        z.x *= g; z.y *= g;
      }
      z.x *= factor; z.y *= factor;
    } else if (transform == SGMSE_B200_TRANSFORM_LOG) {
      const float mag = hypotf(z.x, z.y);
      const float g = mag > 0.f ? logf(1.0f + mag) / mag : 0.f;
      z.x *= g; z.y *= g;
      z.x *= factor; z.y *= factor;
    }
  }
  Y[((size_t)b * F + f) * Tpad + t] = z;
}
void launch_spec_fwd(cudaStream_t st, const float2* spec, int B, int nT, int F, int fstride, int Tpad,
                     float factor, float expo, int transform, int reflect_pad, float2* Y) {
  dim3 grid(cdiv(Tpad, 128), F, B);
  spec_fwd_kernel<<<grid, 128, 0, st>>>(spec, nT, F, fstride, Tpad, factor, expo, transform, reflect_pad, Y);
  CUDA_OK(cudaGetLastError());
}

// spec_back, transpose X[b][f][t] -> spec[(b*Tpad+t)][f].  transform (data_module.py:177-188): exponent
// (|z|/factor)^(1/e) e^{j arg z}, log (exp(|z/factor|) - 1) e^{j arg z} (exp(a) - 1 as written, not expm1), none z
__global__ void spec_back_kernel(const float2* __restrict__ X, int F, int Tpad, int fstride, float factor,
                                     float expo, int transform, float2* __restrict__ spec) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  const int t = blockIdx.y, b = blockIdx.z;
  if (f >= fstride) return;
  float2 z = make_float2(0.f, 0.f);
  if (f < F) {
    z = X[((size_t)b * F + f) * Tpad + t];
    if (transform == SGMSE_B200_TRANSFORM_EXPONENT) {
      z.x /= factor; z.y /= factor;
      if (expo != 1.0f) {
        const float mag = hypotf(z.x, z.y);
        const float g = mag > 0.f ? powf(mag, 1.0f / expo) / mag : 0.f;
        z.x *= g; z.y *= g;
      }
    } else if (transform == SGMSE_B200_TRANSFORM_LOG) {
      z.x /= factor; z.y /= factor;
      const float mag = hypotf(z.x, z.y);
      const float g = mag > 0.f ? (expf(mag) - 1.0f) / mag : 0.f;
      z.x *= g; z.y *= g;
    }
  }
  spec[((size_t)b * Tpad + t) * fstride + f] = z;
}
void launch_spec_back(cudaStream_t st, const float2* X, int B, int F, int Tpad, int fstride, float factor,
                          float expo, int transform, float2* spec) {
  dim3 grid(cdiv(fstride, 128), Tpad, B);
  spec_back_kernel<<<grid, 128, 0, st>>>(X, F, Tpad, fstride, factor, expo, transform, spec);
  CUDA_OK(cudaGetLastError());
}

// overlap-add of the windowed inverse frames with window-envelope normalisation, centre trim,
// 1/n_fft (cuFFT C2R is unnormalised) and the per-utterance renormalisation.
__global__ void overlap_add_kernel(const float* __restrict__ frames, const float* __restrict__ norm, int Tpad,
                                   int n_fft, int hop, int sqrt_window, int L, float* __restrict__ wav) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (s >= L) return;
  const int pos = s + n_fft / 2;
  int t_hi = pos / hop;
  if (t_hi > Tpad - 1) t_hi = Tpad - 1;
  float acc = 0.f, env = 0.f;
  for (int t = t_hi; t >= 0; --t) {
    const int i = pos - t * hop;
    if (i >= n_fft) break;
    const float w = hann_periodic(i, n_fft, sqrt_window);
    acc = fmaf(frames[((size_t)b * Tpad + t) * n_fft + i], w, acc);
    env = fmaf(w, w, env);
  }
  wav[(size_t)b * L + s] = env > 1e-11f ? (acc / (float)n_fft) / env * norm[b] : 0.f;
}
void launch_overlap_add(cudaStream_t st, const float* frames, const float* norm, int B, int Tpad, int n_fft, int hop,
                        int sqrt_window, int L, float* wav) {
  dim3 grid(cdiv(L, 256), B);
  overlap_add_kernel<<<grid, 256, 0, st>>>(frames, norm, Tpad, n_fft, hop, sqrt_window, L, wav);
  CUDA_OK(cudaGetLastError());
}

}  // namespace sgmse
