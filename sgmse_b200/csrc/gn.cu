// GroupNorm statistics finalisation and the fused GroupNorm-apply + SiLU (+ FIR up/down) pass.
//
// Reference semantics: nn.GroupNorm(min(C/4,32), eps=1e-6) + SiLU of
// ResnetBlockBigGANpp.forward (/root/reference/sgmse/backbones/ncsnpp_utils/layerspp.py:242-258)
// and the FIR resamplers upsample_2d / downsample_2d (up_or_down_sampling.py:195-257).
// HBM-bound elementwise work: 128-bit accesses, one read of x, one write per output.
#include <type_traits>

#include "kernels.h"

namespace sgmse {

// ------------------------------------------------------------------------------------------------
// gn_finalize: grid (groups, N).  Sums the producer's per-slot partials in double, fixed order.
// ------------------------------------------------------------------------------------------------
// BATCH (gnfin_variant 1; round 2, the default since -- bit-identical): the partials of a thread are loaded eight at a time before
// they are added, in the same order (the plain loop is load -> add -> branch: 8 serialized round trips per thread at the 512-slot
// levels, most of the kernel's time); bit-identical.
thread_local int g_gnfin_variant = 0;

template <bool BATCH>
__global__ void gn_finalize_kernel(const float* __restrict__ st0, int C0, int slots0,
                                   const float* __restrict__ st1, int C1, int slots1,
                                   const float* __restrict__ gamma, const float* __restrict__ beta,
                                   int cpg, double inv_count, float2* __restrict__ ab,
                                   unsigned int* __restrict__ range_flag) {
  pdl_trigger(); pdl_wait();
  const int g = blockIdx.x, n = blockIdx.y;
  const int Ct = C0 + C1;
  const int max_slots = slots0 > slots1 ? slots0 : slots1;
  double s = 0.0, q = 0.0;
  if (BATCH) {
    const int items = cpg * max_slots;
    for (int j0 = threadIdx.x; j0 < items; j0 += 8 * blockDim.x) {
      float2 v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int j = j0 + u * blockDim.x;
        v[u] = make_float2(0.f, 0.f);
        if (j < items) {
          const int cl = j % cpg, slot = j / cpg;
          const int ch = g * cpg + cl;
          if (ch < C0) {
            if (slot < slots0) v[u] = *reinterpret_cast<const float2*>(st0 + (((size_t)n * slots0 + slot) * C0 + ch) * 2);
          } else {
            if (slot < slots1) v[u] = *reinterpret_cast<const float2*>(st1 + (((size_t)n * slots1 + slot) * C1 + (ch - C0)) * 2);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) { s += v[u].x; q += v[u].y; }   // an absent item adds +0.0: the sum is unchanged
    }
  } else
  for (int j = threadIdx.x; j < cpg * max_slots; j += blockDim.x) {
    const int cl = j % cpg, slot = j / cpg;
    const int ch = g * cpg + cl;
    if (ch < C0) {
      if (slot < slots0) {
        const float2 v = *reinterpret_cast<const float2*>(st0 + (((size_t)n * slots0 + slot) * C0 + ch) * 2);
        s += v.x; q += v.y;
      }
    } else {
      if (slot < slots1) {
        const float2 v = *reinterpret_cast<const float2*>(st1 + (((size_t)n * slots1 + slot) * C1 + (ch - C0)) * 2);
        s += v.x; q += v.y;
      }
    }
  }
  __shared__ double sh_s[32], sh_q[32];
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { sh_s[warp] = s; sh_q[warp] = q; }
  __syncthreads();
  if (warp == 0) {
    const int nw = blockDim.x >> 5;
    s = lane < nw ? sh_s[lane] : 0.0;
    q = lane < nw ? sh_q[lane] : 0.0;
    for (int o = 16; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      q += __shfl_xor_sync(0xffffffffu, q, o);
    }
    if (lane == 0) { sh_s[0] = s; sh_q[0] = q; }
  }
  __syncthreads();
  // fp16 range detector: the producers' partial sums are taken over the ROUNDED fp16 values they store, so an activation
  // beyond +-65504 (stored as inf) makes the sums non-finite -- and every later result NaN.  Count it instead of staying silent.
  if (range_flag && threadIdx.x == 0 && !(isfinite(sh_s[0]) && isfinite(sh_q[0]))) atomicAdd(range_flag, 1u);
  const double mean = sh_s[0] * inv_count;
  double var = sh_q[0] * inv_count - mean * mean;
  if (var < 0.0) var = 0.0;
  const float rstd = (float)(1.0 / sqrt(var + 1e-6));
  for (int cl = threadIdx.x; cl < cpg; cl += blockDim.x) {
    const int ch = g * cpg + cl;
    const float a = gamma[ch] * rstd;
    ab[(size_t)n * Ct + ch] = make_float2(a, beta[ch] - (float)mean * a);
  }
}

void launch_gn_finalize(cudaStream_t st, const TensorDesc& s0, const TensorDesc* s1, const float* gamma,
                        const float* beta, int groups, float2* ab, unsigned int* range_flag) {
  const int C1 = s1 ? s1->C : 0;
  const int Ct = s0.C + C1;
  SG_CHECK(Ct % groups == 0, "GroupNorm: %d channels not divisible by %d groups", Ct, groups);
  SG_CHECK(s0.stats && s0.slots > 0 && (!s1 || (s1->stats && s1->slots > 0)), "GroupNorm input has no statistics");
  if (s1) SG_CHECK(s1->N == s0.N && s1->H == s0.H && s1->W == s0.W, "concat shape mismatch");
  const int cpg = Ct / groups;
  const double inv_count = 1.0 / ((double)s0.H * s0.W * cpg);
  dim3 grid(groups, s0.N);
  if (g_gnfin_variant == 1) {
    launch_k(gn_finalize_kernel<true>, grid, dim3(256), 0, st, s0.stats, s0.C, s0.slots, s1 ? s1->stats : nullptr, C1,
             s1 ? s1->slots : 0, gamma, beta, cpg, inv_count, ab, range_flag);
    CUDA_OK(cudaGetLastError());
    return;
  }
  launch_k(gn_finalize_kernel<false>, grid, dim3(256), 0, st, s0.stats, s0.C, s0.slots, s1 ? s1->stats : nullptr, C1,
                                           s1 ? s1->slots : 0, gamma, beta, cpg, inv_count, ab, range_flag);
  CUDA_OK(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------
// channel_stats: stand-alone (sum, sum^2) per (sample, channel) for tiny levels whose producers cannot
// emit per-tile partials (H*W not a multiple of the tile).  grid (ceil(C/32), N), block (32, 8).
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void channel_stats_kernel(const T* __restrict__ x, int HW, int C, float* __restrict__ stats) {
  pdl_trigger(); pdl_wait();
  const int c = blockIdx.x * 32 + threadIdx.x, n = blockIdx.y;
  float s = 0.f, q = 0.f;
  if (c < C)
    for (int p = threadIdx.y; p < HW; p += 8) { const float v = Act<T>::ld(x + ((size_t)n * HW + p) * C + c); s += v; q += v * v; }
  __shared__ float sh[8][32][2];
  sh[threadIdx.y][threadIdx.x][0] = s; sh[threadIdx.y][threadIdx.x][1] = q;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    for (int r = 1; r < 8; ++r) { s += sh[r][threadIdx.x][0]; q += sh[r][threadIdx.x][1]; }
    stats[((size_t)n * C + c) * 2] = s; stats[((size_t)n * C + c) * 2 + 1] = q;
  }
}
void launch_channel_stats(cudaStream_t st, TensorDesc& t) {
  SG_CHECK(t.stats != nullptr, "channel_stats: tensor has no statistics buffer");
  t.slots = 1;
  dim3 grid(cdiv(t.C, 32), t.N), block(32, 8);
  if (t.dt == DT_F16) launch_k(channel_stats_kernel<__half>, grid, block, 0, st, (const __half*)t.p, t.H * t.W, t.C, t.stats);
  else launch_k(channel_stats_kernel<float>, grid, block, 0, st, (const float*)t.p, t.H * t.W, t.C, t.stats);
  CUDA_OK(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------
// gn_apply (no resampling): y = [silu](a*x + b), optional channel concat of two sources.
// grid (blocks, N); a thread owns one fixed group of 8 channels (its a/b live in registers) and walks pixels,
// so the inner loop is 128-bit load -> 8 x (fma, silu) -> 128-bit store with no index arithmetic.
// ------------------------------------------------------------------------------------------------
template <typename T, bool SILU>
__global__ void __launch_bounds__(256)
gn_apply_plain_kernel(const T* __restrict__ x0, int C0, const T* __restrict__ x1, int C1,
                      const float2* __restrict__ ab, int HW, T* __restrict__ out) {
  pdl_trigger(); pdl_wait();
  const int Ct = C0 + C1, cvpp = Ct >> 3;
  const int ppb = blockDim.x / cvpp;
  const int cv = threadIdx.x % cvpp, pl = threadIdx.x / cvpp;
  if (pl >= ppb) return;
  const int n = blockIdx.y;
  const int c = cv << 3;
  const T* src; int Cs, cs;
  if (c < C0) { src = x0; Cs = C0; cs = c; } else { src = x1; Cs = C1; cs = c - C0; }
  float a[8], b[8];
  {
    const float4* p = reinterpret_cast<const float4*>(ab + (size_t)n * Ct + c);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float4 v = p[i]; a[2 * i] = v.x; b[2 * i] = v.y; a[2 * i + 1] = v.z; b[2 * i + 1] = v.w; }
  }
  const T* sp = src + (size_t)n * HW * Cs + cs;
  T* op = out + (size_t)n * HW * Ct + c;
  // 4 independent 128-bit loads in flight per thread (grid is sized for 4 pixels per thread)
  const int stride = gridDim.x * ppb;
  int p = blockIdx.x * ppb + pl;
  for (; p + 3 * stride < HW; p += 4 * stride) {
    Vec8<T> v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u].load(sp + (size_t)(p + u * stride) * Cs);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      float f[8];
      v[u].get(f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float h = fmaf(a[i], f[i], b[i]);
        if (SILU) h = silu_f(h);
        f[i] = h;
      }
      v[u].set(f);
      v[u].store(op + (size_t)(p + u * stride) * Ct);
    }
  }
  for (; p < HW; p += stride) {
    Vec8<T> v; float f[8];
    v.load(sp + (size_t)p * Cs);
    v.get(f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float h = fmaf(a[i], f[i], b[i]);
      if (SILU) h = silu_f(h);
      f[i] = h;
    }
    v.set(f);
    v.store(op + (size_t)p * Ct);
  }
}

// ------------------------------------------------------------------------------------------------
// gn_self (round 2, on by default since -- bit-identical): gn_finalize folded into the gn_apply_plain that
// consumes it, for the small tensors of the levels below 32 rows (H*W <= 512), where a forward spends ~46 launches
// on finalizing statistics that fit in a few hundred bytes.  Every block first rebuilds (a, b) of ITS sample in
// shared memory -- warp w reduces groups w, w+8, ...: lane j adds the group's (channel, slot) items j, j+32, ... in
// double and the warp combines them with the same xor tree gn_finalize uses, so for channels-per-group x slots <= 32
// (one item per lane) the coefficients are bit-identical by construction; beyond that (a Combine output has 16 slots of 32
// pixels at 16x32) the association differs, but these are fp64 sums of <= 512 fp32 partials, which do not round unless the
// partials span more than ~2^20 in magnitude -- and then applies them exactly like gn_apply_plain.
// ------------------------------------------------------------------------------------------------
thread_local int g_gn_self = 0;

template <typename T, bool SILU>
__global__ void __launch_bounds__(256)
gn_norm_apply_kernel(const T* __restrict__ x0, int C0, const float* __restrict__ st0, int slots0,
                     const T* __restrict__ x1, int C1, const float* __restrict__ st1, int slots1,
                     const float* __restrict__ gamma, const float* __restrict__ beta, int cpg, double inv_count,
                     int HW, int ppb, T* __restrict__ out, unsigned int* __restrict__ range_flag) {
  pdl_trigger(); pdl_wait();
  extern __shared__ float2 ab_s[];                        // [Ct]
  const int Ct = C0 + C1, groups = Ct / cpg, n = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int max_slots = slots0 > slots1 ? slots0 : slots1;
  for (int g = warp; g < groups; g += (int)(blockDim.x >> 5)) {
    double s = 0.0, q = 0.0;
    for (int j = lane; j < cpg * max_slots; j += 32) {
      const int cl = j % cpg, slot = j / cpg;
      const int ch = g * cpg + cl;
      if (ch < C0) {
        if (slot < slots0) {
          const float2 v = *reinterpret_cast<const float2*>(st0 + (((size_t)n * slots0 + slot) * C0 + ch) * 2);
          s += v.x; q += v.y;
        }
      } else {
        if (slot < slots1) {
          const float2 v = *reinterpret_cast<const float2*>(st1 + (((size_t)n * slots1 + slot) * C1 + (ch - C0)) * 2);
          s += v.x; q += v.y;
        }
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      q += __shfl_xor_sync(0xffffffffu, q, o);
    }
    if (range_flag && blockIdx.x == 0 && lane == 0 && !(isfinite(s) && isfinite(q))) atomicAdd(range_flag, 1u);   // see gn_finalize
    const double mean = s * inv_count;
    double var = q * inv_count - mean * mean;
    if (var < 0.0) var = 0.0;
    const float rstd = (float)(1.0 / sqrt(var + 1e-6));
    for (int cl = lane; cl < cpg; cl += 32) {
      const int ch = g * cpg + cl;
      const float a = gamma[ch] * rstd;
      ab_s[ch] = make_float2(a, beta[ch] - (float)mean * a);
    }
  }
  __syncthreads();
  const int cvpp = Ct >> 3;
  const int cv = threadIdx.x % cvpp, pl = threadIdx.x / cvpp;
  if (pl >= ppb) return;
  const int c = cv << 3;
  const T* src; int Cs, cs;
  if (c < C0) { src = x0; Cs = C0; cs = c; } else { src = x1; Cs = C1; cs = c - C0; }
  float a[8], b[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { const float2 v = ab_s[c + i]; a[i] = v.x; b[i] = v.y; }
  const T* sp = src + (size_t)n * HW * Cs + cs;
  T* op = out + (size_t)n * HW * Ct + c;
  const int stride = gridDim.x * ppb;
  for (int p = blockIdx.x * ppb + pl; p < HW; p += stride) {
    Vec8<T> v; float f[8];
    v.load(sp + (size_t)p * Cs);
    v.get(f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float h = fmaf(a[i], f[i], b[i]);
      if (SILU) h = silu_f(h);
      f[i] = h;
    }
    v.set(f);
    v.store(op + (size_t)p * Ct);
  }
}

bool gn_self_applies(const TensorDesc& x0, const TensorDesc* x1) {
  const int Ct = x0.C + (x1 ? x1->C : 0);
  return g_gn_self != 0 && x0.H * x0.W <= 512 && Ct % 8 == 0 && Ct / 8 <= 256;
}

void launch_gn_norm_apply(cudaStream_t st, const TensorDesc& x0, const TensorDesc* x1, const float* gamma, const float* beta,
                          int groups, bool silu, TensorDesc& out, unsigned int* range_flag) {
  const int C1 = x1 ? x1->C : 0;
  const int Ct = x0.C + C1, cvpp = Ct / 8;
  SG_CHECK(Ct % groups == 0 && out.C == Ct && out.N == x0.N && out.H == x0.H && out.W == x0.W, "gn_norm_apply: shape mismatch");
  SG_CHECK(x0.stats && x0.slots > 0 && (!x1 || (x1->stats && x1->slots > 0)), "GroupNorm input has no statistics");
  const int cpg = Ct / groups;
  const double inv_count = 1.0 / ((double)x0.H * x0.W * cpg);
  const int ppb = 256 / cvpp, HW = x0.H * x0.W;
  int gx = cdiv(HW, ppb * 4);
  if (gx < 1) gx = 1;
  dim3 grid(gx, x0.N);
  const size_t smem = (size_t)Ct * sizeof(float2);
#define GO(T, S) launch_k(gn_norm_apply_kernel<T, S>, grid, dim3(256), smem, st, (const T*)x0.p, x0.C, x0.stats, x0.slots, \
                          x1 ? (const T*)x1->p : (const T*)nullptr, C1, x1 ? x1->stats : (const float*)nullptr, x1 ? x1->slots : 0, gamma, beta, cpg, inv_count, HW, ppb, (T*)out.p, range_flag)
  if (x0.dt == DT_F16) { if (silu) GO(__half, true); else GO(__half, false); }
  else { if (silu) GO(float, true); else GO(float, false); }
#undef GO
  CUDA_OK(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------
// gn_apply + FIR up/down: one thread = one output pixel x 8 channels; grid (blocks, N).
// out0 = FIR(silu(a*x+b)), out1 = FIR(x) (the ResBlock shortcut input), one read of x.
// ------------------------------------------------------------------------------------------------
template <typename T, int RS>
__global__ void __launch_bounds__(256)
gn_apply_fir_kernel(const T* __restrict__ x0, int C, const float2* __restrict__ ab, int Hi, int Wi,
                    T* __restrict__ out0, T* __restrict__ out1) {
  pdl_trigger(); pdl_wait();
  const int cvpp = C >> 3;
  const int Ho = RS == RS_DOWN ? Hi / 2 : Hi * 2;
  const int Wo = RS == RS_DOWN ? Wi / 2 : Wi * 2;
  const int n = blockIdx.y;
  const unsigned total = (unsigned)Ho * Wo * cvpp;
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cv = idx % cvpp;
  const unsigned pix = idx / cvpp;
  const int X = pix % Wo, Y = pix / Wo;
  const int c = cv << 3;
  float a[8], b[8];
  {
    const float4* p = reinterpret_cast<const float4*>(ab + (size_t)n * C + c);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float4 v = p[i]; a[2 * i] = v.x; b[2 * i] = v.y; a[2 * i + 1] = v.z; b[2 * i + 1] = v.w; }
  }
  const T* src = x0 + (size_t)n * Hi * Wi * C + c;
  float acc[8], raw[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { acc[i] = 0.f; raw[i] = 0.f; }
  auto tap = [&](int y, int x, float w) {
    if ((unsigned)y >= (unsigned)Hi || (unsigned)x >= (unsigned)Wi) return;
    Vec8<T> v; float f[8];
    v.load(src + ((size_t)y * Wi + x) * C);
    v.get(f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float h = silu_f(fmaf(a[i], f[i], b[i]));
      acc[i] = fmaf(w, h, acc[i]);
      raw[i] = fmaf(w, f[i], raw[i]);
    }
  };
  if (RS == RS_DOWN) {
    // out[Y,X] = sum_{i,j} k[i]k[j] h[2Y+i-1, 2X+j-1], k = [1,3,3,1]/8, zero outside
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) tap(2 * Y + i - 1, 2 * X + j - 1, fir_tap(i) * fir_tap(j));
  } else {
    // zero-insert x2, pad (2,1), FIR [1,3,3,1]/4 per axis:
    //   even Y=2y: 3/4 h[y] + 1/4 h[y-1];  odd Y=2y+1: 3/4 h[y] + 1/4 h[y+1]
    const int y0 = Y >> 1, x0i = X >> 1;
    const int y1 = (Y & 1) ? y0 + 1 : y0 - 1;
    const int x1i = (X & 1) ? x0i + 1 : x0i - 1;
    tap(y0, x0i, 0.5625f);
    tap(y0, x1i, 0.1875f);
    tap(y1, x0i, 0.1875f);
    tap(y1, x1i, 0.0625f);
  }
  const size_t o = ((size_t)n * Ho * Wo + pix) * C + c;
  Vec8<T> ov;
  ov.set(acc); ov.store(out0 + o);
  ov.set(raw); ov.store(out1 + o);
}

// ------------------------------------------------------------------------------------------------
// Shared-memory tiled FIR variants: silu(gn(x)) is evaluated ONCE per input element (the generic kernel above
// re-evaluates it per tap: 4x for up-, 16x for down-sampling, which makes it MUFU-bound instead of HBM-bound).
// Phase 1 stages h = silu(a*x+b) and the raw x of an input tile (+1 pixel halo) in smem as fp32->half pairs;
// phase 2 applies the separable [1,3,3,1] FIR from smem and writes both outputs with 128-bit stores.
// ------------------------------------------------------------------------------------------------
thread_local int g_fir_variant = 0;   // 0: one-MUFU silu (tanh form) + half2 FIR-down arithmetic; 1: expf/divide silu, fp32 FIR;
                         // 2 (round 2, the default since: FIR-down bit-identical, half2 FIR-up rel-L2 8e-4): 0 + all global loads of phase 1 in flight at once
                         //    (the SASS of 0 has ONE LDG.128 per loop trip in front of 8 MUFU: 4-6 serialized memory
                         //    round trips per thread) + half2 FIR-up over 2x2 output quads (9 instead of 16 LDS.128 and
                         //    ~50 instead of ~150 instructions per output vector)

// silu(z) = hz*tanh(hz) + hz with hz = z/2: one MUFU instead of two (ex2 + rcp)
__device__ __forceinline__ float silu_tanh_half_arg(float hz) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(hz));
  return fmaf(hz, t, hz);
}
__device__ __forceinline__ uint32_t h2_add(uint32_t a, uint32_t b) { uint32_t d; asm("add.rn.f16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b)); return d; }
__device__ __forceinline__ uint32_t h2_mul(uint32_t a, uint32_t b) { uint32_t d; asm("mul.rn.f16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b)); return d; }
__device__ __forceinline__ uint32_t h2_fma(uint32_t a, uint32_t b, uint32_t c) { uint32_t d; asm("fma.rn.f16x2 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }

template <typename T, int RS, int TIN, int CV, int MODE>   // TIN: input tile edge incl. halo; CV: 8-channel vectors per block; MODE = g_fir_variant
__global__ void __launch_bounds__(256)
gn_apply_fir_tiled_kernel(const T* __restrict__ x0, int C, const float2* __restrict__ ab, int Hi, int Wi,
                          T* __restrict__ out0, T* __restrict__ out1) {
  pdl_trigger(); pdl_wait();
  constexpr bool FAST = MODE != 1;
  constexpr int TOUT = RS == RS_UP ? (TIN - 2) * 2 : (TIN - 2) / 2;   // output tile edge
  __shared__ __align__(16) __half hs[TIN * TIN][CV * 8];
  __shared__ __align__(16) __half xs[TIN * TIN][CV * 8];
  const int Ho = RS == RS_DOWN ? Hi / 2 : Hi * 2, Wo = RS == RS_DOWN ? Wi / 2 : Wi * 2;
  const int cblocks = C / (CV * 8);
  const int n = blockIdx.z / cblocks, cb = blockIdx.z % cblocks;
  const int cv = threadIdx.x % CV;
  const int c = (cb * CV + cv) * 8;
  // input tile origin (top-left halo pixel)
  const int iy0 = RS == RS_UP ? blockIdx.y * (TIN - 2) - 1 : blockIdx.y * (TIN - 2) - 1;
  const int ix0 = RS == RS_UP ? blockIdx.x * (TIN - 2) - 1 : blockIdx.x * (TIN - 2) - 1;
  float a[8], b[8];
  {
    const float4* p = reinterpret_cast<const float4*>(ab + (size_t)n * C + c);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float4 v = p[i]; a[2 * i] = v.x; b[2 * i] = v.y; a[2 * i + 1] = v.z; b[2 * i + 1] = v.w; }
    if (FAST) {
#pragma unroll
      for (int i = 0; i < 8; ++i) { a[i] *= 0.5f; b[i] *= 0.5f; }   // the tanh form takes z/2
    }
  }
  const T* src = x0 + (size_t)n * Hi * Wi * C + c;
  if constexpr (MODE == 2) {
    // same arithmetic as below, but the loads of this thread are issued in batches of up to four before their first use
    constexpr int ITEMS = TIN * TIN * CV, ROUNDS = (ITEMS + 255) / 256;
    constexpr int GROUP = ROUNDS > 4 ? (ROUNDS + 1) / 2 : ROUNDS;     // 6 rounds (FIR-down) -> 3 + 3: 64 instead of 80 registers
    static_assert(256 % CV == 0, "a thread must keep its channel vector across rounds");
#pragma unroll
    for (int r0 = 0; r0 < ROUNDS; r0 += GROUP) {
      Vec8<T> v[GROUP];
      bool inside[GROUP];
#pragma unroll
      for (int r = 0; r < GROUP; ++r) {
        const int item = threadIdx.x + (r0 + r) * 256;
        const int px = item / CV;
        const int y = iy0 + px / TIN, x = ix0 + px % TIN;
        inside[r] = r0 + r < ROUNDS && item < ITEMS && (unsigned)y < (unsigned)Hi && (unsigned)x < (unsigned)Wi;
        if (inside[r]) v[r].load(src + ((size_t)y * Wi + x) * C);
      }
#pragma unroll
      for (int r = 0; r < GROUP; ++r) {
        const int item = threadIdx.x + (r0 + r) * 256;
        if (r0 + r < ROUNDS && item < ITEMS) {
          const int px = item / CV;
          float f[8], h[8];
          if (inside[r]) {
            v[r].get(f);
#pragma unroll
            for (int i = 0; i < 8; ++i) h[i] = silu_tanh_half_arg(fmaf(a[i], f[i], b[i]));
          } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) { f[i] = 0.f; h[i] = 0.f; }
          }
          Vec8<__half> o;
          o.set(h); o.store(&hs[px][cv * 8]);
          o.set(f); o.store(&xs[px][cv * 8]);
        }
      }
    }
  } else
  for (int item = threadIdx.x; item < TIN * TIN * CV; item += 256) {
    const int px = item / CV;
    const int y = iy0 + px / TIN, x = ix0 + px % TIN;
    float f[8], h[8];
    if ((unsigned)y < (unsigned)Hi && (unsigned)x < (unsigned)Wi) {
      Vec8<T> v; v.load(src + ((size_t)y * Wi + x) * C); v.get(f);
#pragma unroll
      for (int i = 0; i < 8; ++i) h[i] = FAST ? silu_tanh_half_arg(fmaf(a[i], f[i], b[i])) : silu_f(fmaf(a[i], f[i], b[i]));
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) { f[i] = 0.f; h[i] = 0.f; }   // zero padding applies AFTER the activation
    }
    Vec8<__half> o;
    o.set(h); o.store(&hs[px][cv * 8]);
    o.set(f); o.store(&xs[px][cv * 8]);
  }
  __syncthreads();
  if constexpr (FAST && RS == RS_DOWN) {
    // half2 arithmetic, tree-shaped: row sums k0*(t0+t3) + k1*(t1+t2), then the same across the four rows
    // (4 rounding levels of 2^-11 instead of 16 sequential ones; x0.125 is exact)
    const uint32_t K0 = 0x30003000u, K1 = 0x36003600u;   // half2(0.125), half2(0.375)
    for (int item = threadIdx.x; item < TOUT * TOUT * CV; item += 256) {
      const int opx = item / CV;
      const int oy = opx / TOUT, ox = opx % TOUT;
      uint4 rh[4], rx[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int base = (2 * oy + i) * TIN + 2 * ox;
        uint4 th[4], tx[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          th[j] = *reinterpret_cast<const uint4*>(&hs[base + j][cv * 8]);
          tx[j] = *reinterpret_cast<const uint4*>(&xs[base + j][cv * 8]);
        }
        auto rowsum = [&](const uint4 (&tt)[4], uint4& r) {
          const uint32_t* t0 = reinterpret_cast<const uint32_t*>(&tt[0]);
          const uint32_t* t1 = reinterpret_cast<const uint32_t*>(&tt[1]);
          const uint32_t* t2 = reinterpret_cast<const uint32_t*>(&tt[2]);
          const uint32_t* t3 = reinterpret_cast<const uint32_t*>(&tt[3]);
          uint32_t* rr = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
          for (int q = 0; q < 4; ++q) rr[q] = h2_fma(K1, h2_add(t1[q], t2[q]), h2_mul(K0, h2_add(t0[q], t3[q])));
        };
        rowsum(th, rh[i]);
        rowsum(tx, rx[i]);
      }
      uint4 oh, oxr;
      auto colsum = [&](const uint4 (&r)[4], uint4& o) {
        const uint32_t* r0 = reinterpret_cast<const uint32_t*>(&r[0]);
        const uint32_t* r1 = reinterpret_cast<const uint32_t*>(&r[1]);
        const uint32_t* r2 = reinterpret_cast<const uint32_t*>(&r[2]);
        const uint32_t* r3 = reinterpret_cast<const uint32_t*>(&r[3]);
        uint32_t* oo = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
        for (int q = 0; q < 4; ++q) oo[q] = h2_fma(K1, h2_add(r1[q], r2[q]), h2_mul(K0, h2_add(r0[q], r3[q])));
      };
      colsum(rh, oh);
      colsum(rx, oxr);
      const int Y = blockIdx.y * TOUT + oy, X = blockIdx.x * TOUT + ox;
      const size_t o = (((size_t)n * Ho + Y) * Wo + X) * C + c;
      *reinterpret_cast<uint4*>(out0 + o) = oh;
      *reinterpret_cast<uint4*>(out1 + o) = oxr;
    }
  } else if constexpr (MODE == 2 && RS == RS_UP) {
    // One item = one input pixel (ly, lx) of the tile's interior and its 2x2 output quad.  Separable, in half2:
    //   e_r = 3/4 h[r][lx] + 1/4 h[r][lx-1],  o_r = 3/4 h[r][lx] + 1/4 h[r][lx+1]            (r = ly-1, ly, ly+1)
    //   out(2y, 2x) = 3/4 e_ly + 1/4 e_(ly-1)   out(2y, 2x+1) = 3/4 o_ly + 1/4 o_(ly-1)
    //   out(2y+1, 2x) = 3/4 e_ly + 1/4 e_(ly+1) out(2y+1, 2x+1) = 3/4 o_ly + 1/4 o_(ly+1)
    // (up_or_down_sampling.py:195-224: zero-insert x2, FIR [1,3,3,1]/4 per axis; x1/4 is exact, so two roundings of
    // 2^-11 per output on top of the fp16 store)
    const uint32_t K75 = 0x3A003A00u, K25 = 0x34003400u;   // half2(0.75), half2(0.25)
    constexpr int TI = TIN - 2;
    for (int item = threadIdx.x; item < TI * TI * CV; item += 256) {
      const int ipx = item / CV;
      const int ly = ipx / TI + 1, lx = ipx % TI + 1;
      const int Y = blockIdx.y * TOUT + 2 * (ly - 1), X = blockIdx.x * TOUT + 2 * (lx - 1);
#pragma unroll
      for (int tsr = 0; tsr < 2; ++tsr) {
        uint4 q[4];                                        // [dy*2+dx]
        uint4 e[3], o[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const int base = (ly - 1 + r) * TIN + lx;
          const __half* row = tsr == 0 ? &hs[0][0] : &xs[0][0];
          const uint4 vl = *reinterpret_cast<const uint4*>(row + (size_t)(base - 1) * (CV * 8) + cv * 8);
          const uint4 vc = *reinterpret_cast<const uint4*>(row + (size_t)base * (CV * 8) + cv * 8);
          const uint4 vr = *reinterpret_cast<const uint4*>(row + (size_t)(base + 1) * (CV * 8) + cv * 8);
          const uint32_t* wl = reinterpret_cast<const uint32_t*>(&vl);
          const uint32_t* wc = reinterpret_cast<const uint32_t*>(&vc);
          const uint32_t* wr = reinterpret_cast<const uint32_t*>(&vr);
          uint32_t* we = reinterpret_cast<uint32_t*>(&e[r]);
          uint32_t* wo = reinterpret_cast<uint32_t*>(&o[r]);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            we[k] = h2_fma(K75, wc[k], h2_mul(K25, wl[k]));
            wo[k] = h2_fma(K75, wc[k], h2_mul(K25, wr[k]));
          }
        }
        const uint32_t* e0 = reinterpret_cast<const uint32_t*>(&e[0]); const uint32_t* e1 = reinterpret_cast<const uint32_t*>(&e[1]);
        const uint32_t* e2 = reinterpret_cast<const uint32_t*>(&e[2]); const uint32_t* o0 = reinterpret_cast<const uint32_t*>(&o[0]);
        const uint32_t* o1 = reinterpret_cast<const uint32_t*>(&o[1]); const uint32_t* o2 = reinterpret_cast<const uint32_t*>(&o[2]);
        uint32_t* q00 = reinterpret_cast<uint32_t*>(&q[0]); uint32_t* q01 = reinterpret_cast<uint32_t*>(&q[1]);
        uint32_t* q10 = reinterpret_cast<uint32_t*>(&q[2]); uint32_t* q11 = reinterpret_cast<uint32_t*>(&q[3]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          q00[k] = h2_fma(K75, e1[k], h2_mul(K25, e0[k]));
          q01[k] = h2_fma(K75, o1[k], h2_mul(K25, o0[k]));
          q10[k] = h2_fma(K75, e1[k], h2_mul(K25, e2[k]));
          q11[k] = h2_fma(K75, o1[k], h2_mul(K25, o2[k]));
        }
        T* dst = tsr == 0 ? out0 : out1;
#pragma unroll
        for (int d = 0; d < 4; ++d) {
          const size_t o = (((size_t)n * Ho + Y + (d >> 1)) * Wo + X + (d & 1)) * C + c;
          *reinterpret_cast<uint4*>(dst + o) = q[d];
        }
      }
    }
  } else
  for (int item = threadIdx.x; item < TOUT * TOUT * CV; item += 256) {
    const int opx = item / CV;
    const int oy = opx / TOUT, ox = opx % TOUT;
    float acc[8], raw[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { acc[i] = 0.f; raw[i] = 0.f; }
    auto tap = [&](int ly, int lx, float w) {
      float fh[8], fx[8];
      Vec8<__half> v;
      v.load(&hs[ly * TIN + lx][cv * 8]); v.get(fh);
      v.load(&xs[ly * TIN + lx][cv * 8]); v.get(fx);
#pragma unroll
      for (int i = 0; i < 8; ++i) { acc[i] = fmaf(w, fh[i], acc[i]); raw[i] = fmaf(w, fx[i], raw[i]); }
    };
    if (RS == RS_UP) {
      // local input coords (incl. halo offset 1): even out 2y: 3/4 h[y] + 1/4 h[y-1]; odd 2y+1: 3/4 h[y] + 1/4 h[y+1]
      const int ly0 = (oy >> 1) + 1, lx0 = (ox >> 1) + 1;
      const int ly1 = (oy & 1) ? ly0 + 1 : ly0 - 1, lx1 = (ox & 1) ? lx0 + 1 : lx0 - 1;
      tap(ly0, lx0, 0.5625f); tap(ly0, lx1, 0.1875f); tap(ly1, lx0, 0.1875f); tap(ly1, lx1, 0.0625f);
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) tap(2 * oy + i, 2 * ox + j, fir_tap(i) * fir_tap(j));   // (2Y+i-1) - iy0
    }
    const int Y = blockIdx.y * TOUT + oy, X = blockIdx.x * TOUT + ox;
    const size_t o = (((size_t)n * Ho + Y) * Wo + X) * C + c;
    Vec8<T> ov;
    ov.set(acc); ov.store(out0 + o);
    ov.set(raw); ov.store(out1 + o);
  }
}

template <typename T>
static void gn_apply_dispatch(cudaStream_t st, const TensorDesc& x0, const TensorDesc* x1, const float2* ab, bool silu,
                              Resample rs, TensorDesc& out0, TensorDesc* out1) {
  const int C1 = x1 ? x1->C : 0;
  const int Ct = x0.C + C1, cvpp = Ct / 8;
  const T* p0 = (const T*)x0.p; const T* p1 = x1 ? (const T*)x1->p : nullptr;
  T* o0 = (T*)out0.p;
  if (rs == RS_NONE) {
    SG_CHECK(cvpp <= 256, "gn_apply: %d channels exceed one block", Ct);
    const int block = (256 / cvpp) * cvpp;
    const int ppb = block / cvpp;
    const int HW = x0.H * x0.W;
    int gx = cdiv(HW, ppb * 4);
    if (gx < 1) gx = 1;
    dim3 grid(gx, x0.N);
    if (silu) launch_k(gn_apply_plain_kernel<T, true>, grid, dim3(block), 0, st, p0, x0.C, p1, C1, ab, HW, o0);
    else launch_k(gn_apply_plain_kernel<T, false>, grid, dim3(block), 0, st, p0, x0.C, p1, C1, ab, HW, o0);
  } else {
    SG_CHECK(silu && out1 && !x1, "resampling gn_apply expects silu, a raw output and a single source");
    const size_t total = (size_t)out0.H * out0.W * cvpp;
    SG_CHECK(total < (1ull << 31), "gn_apply: tensor too large for 32-bit indexing");
    dim3 grid((unsigned)((total + 255) / 256), x0.N);
    T* o1 = (T*)out1->p;
    if (std::is_same<T, __half>::value && rs == RS_UP && x0.H % 8 == 0 && x0.W % 8 == 0 && x0.C % 64 == 0) {
      dim3 g(x0.W / 8, x0.H / 8, x0.N * (x0.C / 64));
      if (g_fir_variant == 0) launch_k(gn_apply_fir_tiled_kernel<T, RS_UP, 10, 8, 0>, g, dim3(256), 0, st, p0, x0.C, ab, x0.H, x0.W, o0, o1);
      else if (g_fir_variant == 2) launch_k(gn_apply_fir_tiled_kernel<T, RS_UP, 10, 8, 2>, g, dim3(256), 0, st, p0, x0.C, ab, x0.H, x0.W, o0, o1);
      else launch_k(gn_apply_fir_tiled_kernel<T, RS_UP, 10, 8, 1>, g, dim3(256), 0, st, p0, x0.C, ab, x0.H, x0.W, o0, o1);
    } else if (std::is_same<T, __half>::value && rs == RS_DOWN && out0.H % 8 == 0 && out0.W % 8 == 0 && x0.C % 32 == 0) {
      dim3 g(out0.W / 8, out0.H / 8, x0.N * (x0.C / 32));
      if (g_fir_variant == 0) launch_k(gn_apply_fir_tiled_kernel<T, RS_DOWN, 18, 4, 0>, g, dim3(256), 0, st, p0, x0.C, ab, x0.H, x0.W, o0, o1);
      else if (g_fir_variant == 2) launch_k(gn_apply_fir_tiled_kernel<T, RS_DOWN, 18, 4, 2>, g, dim3(256), 0, st, p0, x0.C, ab, x0.H, x0.W, o0, o1);
      else launch_k(gn_apply_fir_tiled_kernel<T, RS_DOWN, 18, 4, 1>, g, dim3(256), 0, st, p0, x0.C, ab, x0.H, x0.W, o0, o1);
    } else
    if (rs == RS_DOWN) launch_k(gn_apply_fir_kernel<T, RS_DOWN>, grid, dim3(256), 0, st, p0, x0.C, ab, x0.H, x0.W, o0, o1);
    else launch_k(gn_apply_fir_kernel<T, RS_UP>, grid, dim3(256), 0, st, p0, x0.C, ab, x0.H, x0.W, o0, o1);
  }
  CUDA_OK(cudaGetLastError());
}

void launch_gn_apply(cudaStream_t st, const TensorDesc& x0, const TensorDesc* x1, const float2* ab, bool silu,
                     Resample rs, TensorDesc& out0, TensorDesc* out1) {
  const int C1 = x1 ? x1->C : 0;
  SG_CHECK(x0.C % 8 == 0 && C1 % 8 == 0, "channel counts must be multiples of 8 (got %d, %d)", x0.C, C1);
  SG_CHECK(out0.C == x0.C + C1 && out0.N == x0.N, "gn_apply output shape mismatch");
  const int Ho = rs == RS_DOWN ? x0.H / 2 : (rs == RS_UP ? x0.H * 2 : x0.H);
  const int Wo = rs == RS_DOWN ? x0.W / 2 : (rs == RS_UP ? x0.W * 2 : x0.W);
  SG_CHECK(out0.H == Ho && out0.W == Wo, "gn_apply output resolution mismatch");
  if (x0.dt == DT_F16) gn_apply_dispatch<__half>(st, x0, x1, ab, silu, rs, out0, out1);
  else gn_apply_dispatch<float>(st, x0, x1, ab, silu, rs, out0, out1);
}

}  // namespace sgmse
