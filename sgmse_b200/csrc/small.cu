// The 4-channel ends of the network: input conv3x3(4->nf), Combine (conv1x1 4->C of the FIR-down
// input pyramid, summed into h), the progressive-output conv3x3(C->4), and 4-channel FIR resamplers.
// All of these are HBM-bound (N=4 or K=4 "GEMMs"): plain coalesced CUDA-core kernels.
//
// Reference: ncsnpp.py:293-298 (input conv), layerspp.py:44-59 (Combine), ncsnpp.py:358-379
// (output_skip pyramid), up_or_down_sampling.py:195-257 (FIR).
#include "kernels.h"

namespace sgmse {

// mma.sync helpers shared by the 4-channel ends
__device__ __forceinline__ void oc_ldsm_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void oc_mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// --no-centered backbones (ncsnpp.py:288-290): x -> 2x - 1 on the network input, in fp32 (2x is exact, so the fma rounds
// as the reference's two operations do).  Applied to in-bounds pixels only: the reference zero-pads after the mapping.
__device__ __forceinline__ float2 uncenter2(float2 v) { return make_float2(fmaf(2.f, v.x, -1.f), fmaf(2.f, v.y, -1.f)); }
__device__ __forceinline__ float4 uncenter4(float4 v) {
  return make_float4(fmaf(2.f, v.x, -1.f), fmaf(2.f, v.y, -1.f), fmaf(2.f, v.z, -1.f), fmaf(2.f, v.w, -1.f));
}

// ------------------------------------------------------------------------------------------------
// input conv: state float4 [N,H,W] -> T [N,H,W,C];   w[k][c], k = tap*4 + cin
// ------------------------------------------------------------------------------------------------
template <typename T, int TP>
__global__ void __launch_bounds__(128) input_conv_kernel(const float4* __restrict__ state, int H, int W, int C,
                                                         const float* __restrict__ w, const float* __restrict__ bias,
                                                         T* __restrict__ out, float* __restrict__ stats, int slots,
                                                         float in_scale, int not_centered) {
  __shared__ __align__(16) float in[TP][36];
  const int HW = H * W;
  const int m0 = blockIdx.x * TP;
  const int n = m0 / HW;
  const int r0 = m0 - n * HW;
  for (int i = threadIdx.x; i < TP * 9; i += blockDim.x) {
    const int p = i / 9, tap = i - p * 9;
    const int r = r0 + p;
    const int y = r / W + tap / 3 - 1, x = r % W + tap % 3 - 1;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if ((unsigned)y < (unsigned)H && (unsigned)x < (unsigned)W) {
      v = state[(size_t)n * HW + (size_t)y * W + x];
      if (not_centered) v = uncenter4(v);
    }
    in[p][tap * 4 + 0] = in_scale * v.x; in[p][tap * 4 + 1] = in_scale * v.y;
    in[p][tap * 4 + 2] = in_scale * v.z; in[p][tap * 4 + 3] = in_scale * v.w;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float wr[36];
#pragma unroll
    for (int k = 0; k < 36; ++k) wr[k] = w[k * C + c];
    const float b = bias[c];
    float s = 0.f, q = 0.f;
    for (int p = 0; p < TP; ++p) {
      float acc = b;
      const float4* ip = reinterpret_cast<const float4*>(&in[p][0]);   // warp-wide broadcast, 128-bit
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const float4 v = ip[k];
        acc = fmaf(wr[4 * k], v.x, acc); acc = fmaf(wr[4 * k + 1], v.y, acc);
        acc = fmaf(wr[4 * k + 2], v.z, acc); acc = fmaf(wr[4 * k + 3], v.w, acc);
      }
      Act<T>::st(out + (size_t)(m0 + p) * C + c, acc);
      const float r = Act<T>::rnd(acc);
      s += r; q += r * r;
    }
    if (stats) {
      float* d = stats + (((size_t)n * slots + r0 / TP) * C + c) * 2;
      d[0] = s; d[1] = q;
    }
  }
}

// fp16 tensor-core variant (mma.sync m16n8k16): the 36-deep contraction (9 taps x 4 state components) is padded to
// K = 48 = 3 k-steps; a warp owns 32 pixels x all C output channels (2 m-tiles x NT n-tiles).  The CUDA-core kernel
// above needs 36 FMA per output element (FMA-bound);
// here the arithmetic is 3 HMMA per 16x8 outputs and the kernel is bound by the 256 B/pixel it writes.
//   A fragment (pixels x k): k = tap*4 + component, so the k pair (2t, 2t+1) of k-step s is the (.xy | .zw) half of the
//   state float4 of neighbour tap 4s + (t >> 1) [a0/a1] and 4s + 2 + (t >> 1) [a2/a3]: straight from global/L1.
//   B fragments (k x channels) are built once per block in shared memory; the block then walks tiles of 128 pixels.
//   Output goes through a per-warp padded smem tile so that global stores are 128-bit and row-contiguous.
thread_local int g_inconv_variant = 0;   // 0: tensor-core kernel for fp16 output where it applies, 1: CUDA-core kernel,
                            // 2 (round 2, the default since -- bit-identical): 0 with the A fragments of the NEXT 16-pixel m-tile
                            //   loaded before the 48 MMAs of the current one (today every m-tile starts with an exposed
                            //   L1/L2 round trip at 16 warps per SM); same arithmetic, bit-identical

template <int NT>   // NT = C / 8
__global__ void __launch_bounds__(128) input_conv_mma_kernel(const float4* __restrict__ state, int H, int W,
                                                             const float* __restrict__ w, const float* __restrict__ bias,
                                                             __half* __restrict__ out, float* __restrict__ stats, int slots,
                                                             int num_tiles, float in_scale, int not_centered) {
  constexpr int C = NT * 8;
  constexpr int PITCH = C + 8;                       // halfs per staged row: conflict-free 32-bit writes, 16-B aligned rows
  pdl_trigger();                                     // weights / bias are constant: staged before pdl_wait()
  extern __shared__ __align__(16) uint8_t ic_smem[];
  uint2* wfrag = reinterpret_cast<uint2*>(ic_smem);                                   // [3][NT][32]
  __half* stage = reinterpret_cast<__half*>(ic_smem + (size_t)3 * NT * 32 * sizeof(uint2));   // [4 warps][32][PITCH]
  float* red = reinterpret_cast<float*>(stage + (size_t)4 * 32 * PITCH);              // [4 warps][C][2]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  for (int i = tid; i < 3 * NT * 32; i += 128) {
    const int l = i & 31, j = (i >> 5) % NT, s = i / (32 * NT);
    const int gg = l >> 2, tt = l & 3;
    const int c = j * 8 + gg;
    const int k0 = 16 * s + 2 * tt;
    auto wk = [&](int k) { return k < 36 ? w[k * C + c] : 0.f; };
    const __half2 b0 = __floats2half2_rn(wk(k0), wk(k0 + 1));
    const __half2 b1 = __floats2half2_rn(wk(k0 + 8), wk(k0 + 9));
    wfrag[i] = make_uint2(*reinterpret_cast<const uint32_t*>(&b0), *reinterpret_cast<const uint32_t*>(&b1));
  }
  float bia[NT][2];
#pragma unroll
  for (int j = 0; j < NT; ++j) { bia[j][0] = bias[j * 8 + 2 * t]; bia[j][1] = bias[j * 8 + 2 * t + 1]; }
  __syncthreads();
  pdl_wait();
  const int HW = H * W;
  __half* wstage = stage + (size_t)warp * 32 * PITCH;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m0 = tile * 128;
    const int n = m0 / HW, r0 = m0 - n * HW;
    const float4* sp = state + (size_t)n * HW;
    float ssum[NT][2], ssq[NT][2];
#pragma unroll
    for (int j = 0; j < NT; ++j) { ssum[j][0] = ssum[j][1] = ssq[j][0] = ssq[j][1] = 0.f; }
#pragma unroll 1
    for (int mt = 0; mt < 2; ++mt) {
      // A fragments of this m-tile: rows g and g + 8
      uint32_t af[3][4];
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int r = r0 + warp * 32 + mt * 16 + g + hr * 8;
        const int py = r / W, px = r - py * W;
#pragma unroll
        for (int q = 0; q < 6; ++q) {                 // q-th k-octet: tap 2q + (t >> 1)
          const int tap = 2 * q + (t >> 1);
          float2 v = make_float2(0.f, 0.f);
          if (tap < 9) {
            const int y = py + tap / 3 - 1, x = px + tap % 3 - 1;
            if ((unsigned)y < (unsigned)H && (unsigned)x < (unsigned)W) {
              v = reinterpret_cast<const float2*>(sp + (size_t)y * W + x)[t & 1];
              if (not_centered) v = uncenter2(v);
            }
          }
          const __half2 hv = __floats2half2_rn(in_scale * v.x, in_scale * v.y);
          af[q >> 1][(q & 1) * 2 + hr] = *reinterpret_cast<const uint32_t*>(&hv);
        }
      }
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const uint2 b = wfrag[(s * NT + j) * 32 + lane];
          oc_mma(acc, af[s], b.x, b.y);
        }
        // rows g (acc[0..1]) and g + 8 (acc[2..3]), channels 8j + 2t, +1
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const __half2 hv = __floats2half2_rn(acc[2 * hr] + bia[j][0], acc[2 * hr + 1] + bia[j][1]);
          const float2 f = __half22float2(hv);
          ssum[j][0] += f.x; ssq[j][0] = fmaf(f.x, f.x, ssq[j][0]);
          ssum[j][1] += f.y; ssq[j][1] = fmaf(f.y, f.y, ssq[j][1]);
          *reinterpret_cast<__half2*>(wstage + (size_t)(mt * 16 + g + hr * 8) * PITCH + j * 8 + 2 * t) = hv;
        }
      }
    }
    __syncwarp();
    // 32 rows x C halfs -> global, 128-bit, row-contiguous
    {
      __half* op = out + (size_t)(m0 + warp * 32) * C;
      constexpr int VPR = C / 8;                       // 16-B vectors per row
      for (int i = lane; i < 32 * VPR; i += 32) {
        const int row = i / VPR, cvv = i - row * VPR;
        *reinterpret_cast<uint4*>(op + (size_t)row * C + cvv * 8) =
            *reinterpret_cast<const uint4*>(wstage + (size_t)row * PITCH + cvv * 8);
      }
    }
    if (stats) {
      // per-channel partials of the 128-pixel tile: rows across lanes (fixed xor tree), then the 4 warps in order
#pragma unroll
      for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float s1 = ssum[j][e], s2 = ssq[j][e];
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
          if (g == 0) { red[(warp * C + j * 8 + 2 * t + e) * 2] = s1; red[(warp * C + j * 8 + 2 * t + e) * 2 + 1] = s2; }
        }
      __syncthreads();
      for (int c = tid; c < C; c += 128) {
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int wv = 0; wv < 4; ++wv) { s1 += red[(wv * C + c) * 2]; s2 += red[(wv * C + c) * 2 + 1]; }
        float* d = stats + (((size_t)n * slots + r0 / 128) * C + c) * 2;
        d[0] = s1; d[1] = s2;
      }
      __syncthreads();
    }
    __syncwarp();
  }
}

template <int NT, bool PREFETCH>   // NT = C / 8; the separate copy keeps the verified kernel above untouched
__global__ void __launch_bounds__(128) input_conv_mma_pf_kernel(const float4* __restrict__ state, int H, int W,
                                                             const float* __restrict__ w, const float* __restrict__ bias,
                                                             __half* __restrict__ out, float* __restrict__ stats, int slots,
                                                             int num_tiles, float in_scale, int not_centered) {
  constexpr int C = NT * 8;
  constexpr int PITCH = C + 8;                       // halfs per staged row: conflict-free 32-bit writes, 16-B aligned rows
  pdl_trigger();                                     // weights / bias are constant: staged before pdl_wait()
  extern __shared__ __align__(16) uint8_t ic_smem[];
  uint2* wfrag = reinterpret_cast<uint2*>(ic_smem);                                   // [3][NT][32]
  __half* stage = reinterpret_cast<__half*>(ic_smem + (size_t)3 * NT * 32 * sizeof(uint2));   // [4 warps][32][PITCH]
  float* red = reinterpret_cast<float*>(stage + (size_t)4 * 32 * PITCH);              // [4 warps][C][2]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  for (int i = tid; i < 3 * NT * 32; i += 128) {
    const int l = i & 31, j = (i >> 5) % NT, s = i / (32 * NT);
    const int gg = l >> 2, tt = l & 3;
    const int c = j * 8 + gg;
    const int k0 = 16 * s + 2 * tt;
    auto wk = [&](int k) { return k < 36 ? w[k * C + c] : 0.f; };
    const __half2 b0 = __floats2half2_rn(wk(k0), wk(k0 + 1));
    const __half2 b1 = __floats2half2_rn(wk(k0 + 8), wk(k0 + 9));
    wfrag[i] = make_uint2(*reinterpret_cast<const uint32_t*>(&b0), *reinterpret_cast<const uint32_t*>(&b1));
  }
  float bia[NT][2];
#pragma unroll
  for (int j = 0; j < NT; ++j) { bia[j][0] = bias[j * 8 + 2 * t]; bia[j][1] = bias[j * 8 + 2 * t + 1]; }
  __syncthreads();
  pdl_wait();
  const int HW = H * W;
  __half* wstage = stage + (size_t)warp * 32 * PITCH;
  // A fragments of m-tile `mt` of `tile`: rows g and g + 8.  Loads (raw fp32 pairs) and the conversion to fp16 fragments
  // are separate steps so that the prefetching variant converts only after the current m-tile's MMAs were issued.
  auto load_raw = [&](int tile, int mt, float2 (&raw)[12]) {
    const int m0 = tile * 128;
    const int n = m0 / HW, r0 = m0 - n * HW;
    const float4* sp = state + (size_t)n * HW;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int r = r0 + warp * 32 + mt * 16 + g + hr * 8;
      const int py = r / W, px = r - py * W;
#pragma unroll
      for (int q = 0; q < 6; ++q) {                 // q-th k-octet: tap 2q + (t >> 1)
        const int tap = 2 * q + (t >> 1);
        float2 v = make_float2(0.f, 0.f);
        if (tap < 9) {
          const int y = py + tap / 3 - 1, x = px + tap % 3 - 1;
          if ((unsigned)y < (unsigned)H && (unsigned)x < (unsigned)W) {
            v = reinterpret_cast<const float2*>(sp + (size_t)y * W + x)[t & 1];
            if (not_centered) v = uncenter2(v);
          }
        }
        raw[hr * 6 + q] = v;
      }
    }
  };
  auto convert = [&](const float2 (&raw)[12], uint32_t (&af)[3][4]) {
#pragma unroll
    for (int hr = 0; hr < 2; ++hr)
#pragma unroll
      for (int q = 0; q < 6; ++q) {
        const __half2 hv = __floats2half2_rn(in_scale * raw[hr * 6 + q].x, in_scale * raw[hr * 6 + q].y);
        af[q >> 1][(q & 1) * 2 + hr] = *reinterpret_cast<const uint32_t*>(&hv);
      }
  };
  uint32_t af[3][4];
  float2 raw[12];
  if (PREFETCH && (int)blockIdx.x < num_tiles) { load_raw(blockIdx.x, 0, raw); convert(raw, af); }
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m0 = tile * 128;
    const int n = m0 / HW, r0 = m0 - n * HW;
    float ssum[NT][2], ssq[NT][2];
#pragma unroll
    for (int j = 0; j < NT; ++j) { ssum[j][0] = ssum[j][1] = ssq[j][0] = ssq[j][1] = 0.f; }
#pragma unroll 1
    for (int mt = 0; mt < 2; ++mt) {
      if (PREFETCH) {                                 // next m-tile's loads fly during this one's MMAs
        if (mt == 0) load_raw(tile, 1, raw);
        else if (tile + (int)gridDim.x < num_tiles) load_raw(tile + gridDim.x, 0, raw);
      } else {
        load_raw(tile, mt, raw);
        convert(raw, af);
      }
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const uint2 b = wfrag[(s * NT + j) * 32 + lane];
          oc_mma(acc, af[s], b.x, b.y);
        }
        // rows g (acc[0..1]) and g + 8 (acc[2..3]), channels 8j + 2t, +1
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const __half2 hv = __floats2half2_rn(acc[2 * hr] + bia[j][0], acc[2 * hr + 1] + bia[j][1]);
          const float2 f = __half22float2(hv);
          ssum[j][0] += f.x; ssq[j][0] = fmaf(f.x, f.x, ssq[j][0]);
          ssum[j][1] += f.y; ssq[j][1] = fmaf(f.y, f.y, ssq[j][1]);
          *reinterpret_cast<__half2*>(wstage + (size_t)(mt * 16 + g + hr * 8) * PITCH + j * 8 + 2 * t) = hv;
        }
      }
      if (PREFETCH) convert(raw, af);
    }
    __syncwarp();
    // 32 rows x C halfs -> global, 128-bit, row-contiguous
    {
      __half* op = out + (size_t)(m0 + warp * 32) * C;
      constexpr int VPR = C / 8;                       // 16-B vectors per row
      for (int i = lane; i < 32 * VPR; i += 32) {
        const int row = i / VPR, cvv = i - row * VPR;
        *reinterpret_cast<uint4*>(op + (size_t)row * C + cvv * 8) =
            *reinterpret_cast<const uint4*>(wstage + (size_t)row * PITCH + cvv * 8);
      }
    }
    if (stats) {
      // per-channel partials of the 128-pixel tile: rows across lanes (fixed xor tree), then the 4 warps in order
#pragma unroll
      for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float s1 = ssum[j][e], s2 = ssq[j][e];
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
          if (g == 0) { red[(warp * C + j * 8 + 2 * t + e) * 2] = s1; red[(warp * C + j * 8 + 2 * t + e) * 2 + 1] = s2; }
        }
      __syncthreads();
      for (int c = tid; c < C; c += 128) {
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int wv = 0; wv < 4; ++wv) { s1 += red[(wv * C + c) * 2]; s2 += red[(wv * C + c) * 2 + 1]; }
        float* d = stats + (((size_t)n * slots + r0 / 128) * C + c) * 2;
        d[0] = s1; d[1] = s2;
      }
      __syncthreads();
    }
    __syncwarp();
  }
}

template <int NT, bool PREFETCH = false>
static void input_conv_mma_launch(cudaStream_t st, const float4* state, int N, int H, int W, const float* w,
                                  const float* bias, TensorDesc& out, float in_scale, int not_centered) {
  constexpr int C = NT * 8;
  const int num_tiles = N * H * W / 128;
  const size_t smem = (size_t)3 * NT * 32 * sizeof(uint2) + (size_t)4 * 32 * (C + 8) * 2 + (size_t)4 * C * 2 * 4;
  auto k = PREFETCH ? input_conv_mma_pf_kernel<NT, true> : input_conv_mma_kernel<NT>;
  CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = std::min(num_tiles, 132 * 4);
  launch_k(k, dim3(grid), dim3(128), smem, st, state, H, W, w, bias, (__half*)out.p, out.stats, out.slots, num_tiles, in_scale, not_centered);
  CUDA_OK(cudaGetLastError());
}

void launch_input_conv(cudaStream_t st, const float4* state, int N, int H, int W, const float* w,
                       const float* bias, TensorDesc& out, float in_scale, bool not_centered) {
  const int nc = not_centered ? 1 : 0;
  const int HW = H * W;
  SG_CHECK(HW % 32 == 0, "input conv: H*W must be a multiple of 32");
  if (out.dt == DT_F16 && g_inconv_variant == 2 && HW % 128 == 0 && (out.C == 128 || out.C == 64 || out.C == 32)) {
    out.slots = HW / 128;
    if (out.C == 128) input_conv_mma_launch<16, true>(st, state, N, H, W, w, bias, out, in_scale, nc);
    else if (out.C == 64) input_conv_mma_launch<8, true>(st, state, N, H, W, w, bias, out, in_scale, nc);
    else input_conv_mma_launch<4, true>(st, state, N, H, W, w, bias, out, in_scale, nc);
    return;
  }
  if (out.dt == DT_F16 && g_inconv_variant == 0 && HW % 128 == 0 && (out.C == 128 || out.C == 64 || out.C == 32)) {
    out.slots = HW / 128;
    if (out.C == 128) input_conv_mma_launch<16>(st, state, N, H, W, w, bias, out, in_scale, nc);
    else if (out.C == 64) input_conv_mma_launch<8>(st, state, N, H, W, w, bias, out, in_scale, nc);
    else input_conv_mma_launch<4>(st, state, N, H, W, w, bias, out, in_scale, nc);
    return;
  }
  const int TP = (HW % 128 == 0) ? 128 : 32;
  out.slots = HW / TP;
  const int grid = N * HW / TP;
#define GO(T, TP_) input_conv_kernel<T, TP_><<<grid, 128, 0, st>>>(state, H, W, out.C, w, bias, (T*)out.p, out.stats, out.slots, in_scale, nc)
  if (out.dt == DT_F16) { if (TP == 128) GO(__half, 128); else GO(__half, 32); }
  else { if (TP == 128) GO(float, 128); else GO(float, 32); }
#undef GO
  CUDA_OK(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------
// Combine: out = W^T pyr + b + h ;  32 pixels per block, thread owns channels
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(128) combine_kernel(const float4* __restrict__ pyr, const float* __restrict__ w,
                                                      const float* __restrict__ bias, const T* __restrict__ h, int HW, int M,
                                                      int C, T* __restrict__ out, float* __restrict__ stats, int slots) {
  pdl_trigger(); pdl_wait();
  __shared__ float4 pin[32];
  const int m0 = blockIdx.x * 32;
  const int n = m0 / HW, r0 = m0 - n * HW;
  if (threadIdx.x < 32) pin[threadIdx.x] = m0 + threadIdx.x < M ? pyr[m0 + threadIdx.x] : make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float w0 = w[c], w1 = w[C + c], w2 = w[2 * C + c], w3 = w[3 * C + c], b = bias[c];
    float s = 0.f, q = 0.f;
    for (int p = 0; p < 32 && m0 + p < M; ++p) {
      const float4 v = pin[p];
      const size_t o = (size_t)(m0 + p) * C + c;
      float acc = b + w0 * v.x + w1 * v.y + w2 * v.z + w3 * v.w + Act<T>::ld(h + o);
      Act<T>::st(out + o, acc);
      const float r = Act<T>::rnd(acc);
      s += r; q += r * r;
    }
    if (stats) {
      float* d = stats + (((size_t)n * slots + r0 / 32) * C + c) * 2;
      d[0] = s; d[1] = q;
    }
  }
}

// combine_variant 1 (round 2, the default since -- bit-identical): a thread owns 8 channels (one 128-bit vector) of one
// 32-pixel tile and walks the tile's pixels in order -- the same per-channel expression and the same summation order as
// the kernel above, so results and statistics are bit-identical -- with 8 vector loads in flight per thread instead of
// four 2-byte ones (the scalar kernel keeps too few bytes in flight per SM to reach HBM bandwidth).
thread_local int g_combine_variant = 0;

template <int CV>   // CV = C / 8 vectors per pixel (16 or 32); block = 128 threads = 128 / CV tiles
__global__ void __launch_bounds__(128) combine_vec_kernel(const float4* __restrict__ pyr, const float* __restrict__ w,
                                                          const float* __restrict__ bias, const __half* __restrict__ h, int HW,
                                                          int M, __half* __restrict__ out, float* __restrict__ stats, int slots) {
  pdl_trigger(); pdl_wait();
  constexpr int C = CV * 8, TPB = 128 / CV;
  const int cv = threadIdx.x % CV, tl = threadIdx.x / CV;
  const int tile = blockIdx.x * TPB + tl;
  const int m0 = tile * 32;
  if (m0 >= M) return;
  const int n = m0 / HW, r0 = m0 - n * HW;
  const int c0 = cv * 8;
  float w0[8], w1[8], w2[8], w3[8], bb[8], s[8], q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    w0[i] = w[c0 + i]; w1[i] = w[C + c0 + i]; w2[i] = w[2 * C + c0 + i]; w3[i] = w[3 * C + c0 + i]; bb[i] = bias[c0 + i];
    s[i] = 0.f; q[i] = 0.f;
  }
#pragma unroll 1
  for (int pb = 0; pb < 32; pb += 8) {
    uint4 hv[8];
    float4 pv[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int m = m0 + pb + u;
      if (m < M) {
        hv[u] = *reinterpret_cast<const uint4*>(h + (size_t)m * C + c0);
        pv[u] = __ldg(pyr + m);
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int m = m0 + pb + u;
      if (m < M) {
        const float4 v = pv[u];
        const __half* hh = reinterpret_cast<const __half*>(&hv[u]);
        uint4 ov;
        __half* oh = reinterpret_cast<__half*>(&ov);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float acc = bb[i] + w0[i] * v.x + w1[i] * v.y + w2[i] * v.z + w3[i] * v.w + __half2float(hh[i]);
          oh[i] = __float2half_rn(acc);
          const float r = __half2float(oh[i]);
          s[i] += r; q[i] += r * r;
        }
        *reinterpret_cast<uint4*>(out + (size_t)m * C + c0) = ov;
      }
    }
  }
  if (stats) {
    float* d = stats + (((size_t)n * slots + r0 / 32) * C + c0) * 2;
#pragma unroll
    for (int i = 0; i < 8; i += 2) *reinterpret_cast<float4*>(d + 2 * i) = make_float4(s[i], q[i], s[i + 1], q[i + 1]);
  }
}

void launch_combine(cudaStream_t st, const float4* pyr, const float* w, const float* bias, const TensorDesc& h,
                    TensorDesc& out) {
  const int HW = h.H * h.W;
  const int M = h.N * HW;
  const bool tile_stats = out.stats && HW % 32 == 0;
  out.slots = tile_stats ? HW / 32 : 0;
  float* stp = tile_stats ? out.stats : nullptr;
  const int grid = cdiv(M, 32);
  if (h.dt == DT_F16 && g_combine_variant == 1 && (h.C == 128 || h.C == 256) && HW % 32 == 0) {
    if (h.C == 128)
      launch_k(combine_vec_kernel<16>, dim3(cdiv(grid, 8)), dim3(128), 0, st, pyr, w, bias, (const __half*)h.p, HW, M, (__half*)out.p, stp, out.slots);
    else
      launch_k(combine_vec_kernel<32>, dim3(cdiv(grid, 4)), dim3(128), 0, st, pyr, w, bias, (const __half*)h.p, HW, M, (__half*)out.p, stp, out.slots);
    CUDA_OK(cudaGetLastError());
    if (out.stats && !tile_stats) launch_channel_stats(st, out);
    return;
  }
  if (h.dt == DT_F16)
    launch_k(combine_kernel<__half>, dim3(grid), dim3(128), 0, st, pyr, w, bias, (const __half*)h.p, HW, M, h.C, (__half*)out.p, stp, out.slots);
  else
    launch_k(combine_kernel<float>, dim3(grid), dim3(128), 0, st, pyr, w, bias, (const float*)h.p, HW, M, h.C, (float*)out.p, stp, out.slots);
  CUDA_OK(cudaGetLastError());
  if (out.stats && !tile_stats) launch_channel_stats(st, out);
}

// ------------------------------------------------------------------------------------------------
// 4-channel FIR resample (pyramids, fp32)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void fma4(float4& a, float w, const float4& v) {
  a.x = fmaf(w, v.x, a.x); a.y = fmaf(w, v.y, a.y); a.z = fmaf(w, v.z, a.z); a.w = fmaf(w, v.w, a.w);
}

template <int RS>
__global__ void fir4_kernel(const float4* __restrict__ in, int N, int Hi, int Wi, float4* __restrict__ out, float scale,
                            const float* __restrict__ scale_rows, int not_centered) {
  pdl_trigger(); pdl_wait();
  const int Ho = RS == RS_DOWN ? Hi / 2 : Hi * 2, Wo = RS == RS_DOWN ? Wi / 2 : Wi * 2;
  const size_t total = (size_t)N * Ho * Wo;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int X = (int)(idx % Wo), Y = (int)((idx / Wo) % Ho), n = (int)(idx / ((size_t)Wo * Ho));
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  auto tap = [&](int y, int x, float w) {
    if ((unsigned)y < (unsigned)Hi && (unsigned)x < (unsigned)Wi) {
      const float4 v = in[((size_t)n * Hi + y) * Wi + x];
      fma4(acc, w, not_centered ? uncenter4(v) : v);
    }
  };
  if (RS == RS_DOWN) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) tap(2 * Y + i - 1, 2 * X + j - 1, fir_tap(i) * fir_tap(j));
  } else {
    const int y0 = Y >> 1, x0 = X >> 1;
    const int y1 = (Y & 1) ? y0 + 1 : y0 - 1, x1 = (X & 1) ? x0 + 1 : x0 - 1;
    tap(y0, x0, 0.5625f); tap(y0, x1, 0.1875f); tap(y1, x0, 0.1875f); tap(y1, x1, 0.0625f);
  }
  if (scale_rows) scale = scale_rows[n];
  if (scale != 1.f) { acc.x *= scale; acc.y *= scale; acc.z *= scale; acc.w *= scale; }
  out[idx] = acc;
}

void launch_fir4(cudaStream_t st, const float4* in, int N, int H, int W, Resample rs, float4* out, float scale,
                 const float* scale_rows, bool not_centered) {
  SG_CHECK(rs != RS_NONE, "fir4: nothing to do");
  SG_CHECK(!not_centered || rs == RS_DOWN, "fir4: the input mapping belongs to the input pyramid's FIR-down");
  const size_t total = rs == RS_DOWN ? (size_t)N * (H / 2) * (W / 2) : (size_t)N * H * 2 * W * 2;
  const int grid = (int)((total + 255) / 256);
  if (rs == RS_DOWN) launch_k(fir4_kernel<RS_DOWN>, dim3(grid), dim3(256), 0, st, in, N, H, W, out, scale, scale_rows,
                                 not_centered ? 1 : 0);
  else launch_k(fir4_kernel<RS_UP>, dim3(grid), dim3(256), 0, st, in, N, H, W, out, scale, scale_rows, 0);
  CUDA_OK(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------
// progressive output conv3x3 (C -> 4) + bias (+ FIR-up'ed pyramid).  N=4 "GEMM": CUDA cores.
// One thread per output pixel (16x16 pixel tile per block), the [9*C] x 4 weights live in shared memory as
// float4 rows and are read as warp-wide broadcasts (1 LDS.128 per 4 FMA); activations stream through L1 with
// 128-bit loads.  w [9*C][4] (k = tap*C + cin).
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) out_conv_kernel(const T* __restrict__ act, int H, int W, int C,
                                                       const float4* __restrict__ w, float4 bias,
                                                       const float4* __restrict__ addend, float4* __restrict__ out) {
  extern __shared__ float4 wsm[];          // [9*C]
  for (int i = threadIdx.x; i < 9 * C; i += blockDim.x) wsm[i] = w[i];
  __syncthreads();
  const int x = blockIdx.x * 16 + (threadIdx.x & 15);
  const int y = blockIdx.y * 16 + (threadIdx.x >> 4);
  const int n = blockIdx.z;
  if (x >= W || y >= H) return;
  float4 acc = bias;
#pragma unroll 1
  for (int tap = 0; tap < 9; ++tap) {
    const int yy = y + tap / 3 - 1, xx = x + tap % 3 - 1;
    if ((unsigned)yy >= (unsigned)H || (unsigned)xx >= (unsigned)W) continue;
    const T* row = act + (((size_t)n * H + yy) * W + xx) * C;
    const float4* wr = wsm + tap * C;
#pragma unroll 2
    for (int c = 0; c < C; c += 8) {
      Vec8<T> v; float f[8];
      v.load(row + c); v.get(f);
#pragma unroll
      for (int i = 0; i < 8; ++i) fma4(acc, f[i], wr[c + i]);
    }
  }
  const size_t o = ((size_t)n * H + y) * W + x;
  if (addend) { const float4 a = addend[o]; acc.x += a.x; acc.y += a.y; acc.z += a.z; acc.w += a.w; }
  out[o] = acc;
}

// Warp-cooperative variant for C = 8*LP (LP = lanes per pixel, a power of two <= 32): a warp owns a strip of 16
// pixels of one row; the LP lanes of a pixel split its channels (one fully coalesced 128-bit load each), keep the
// tap's 8x4 weights in registers across the strip, and shuffle-reduce the 4 outputs at the end.
template <typename T, int LP>
__global__ void __launch_bounds__(256) out_conv_coop_kernel(const T* __restrict__ act, int H, int W,
                                                            const float4* __restrict__ w, float4 bias,
                                                            const float4* __restrict__ addend, float4* __restrict__ out) {
  constexpr int C = LP * 8;
  constexpr int PPL = 32 / LP;       // pixels per warp-wide load
  constexpr int P = 16 / PPL;        // loads per 16-pixel strip
  extern __shared__ float4 wsm[];    // [9][8][LP]: conflict-free when lanes read consecutive float4
  for (int i = threadIdx.x; i < 9 * C; i += blockDim.x) {
    const int tap = i / C, c = i % C;
    wsm[(tap * 8 + (c & 7)) * LP + (c >> 3)] = w[i];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sub = lane / LP, cl = lane % LP;
  const int x0 = blockIdx.x * 16, y = blockIdx.y * 8 + warp, n = blockIdx.z;
  if (y >= H) return;
  float4 acc[P];
#pragma unroll
  for (int p = 0; p < P; ++p) acc[p] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
  for (int tap = 0; tap < 9; ++tap) {
    const int yy = y + tap / 3 - 1, dx = tap % 3 - 1;
    if ((unsigned)yy >= (unsigned)H) continue;
    float4 wr[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) wr[i] = wsm[(tap * 8 + i) * LP + cl];
    const T* rowp = act + ((size_t)n * H + yy) * W * C + cl * 8;
#pragma unroll
    for (int p = 0; p < P; ++p) {
      const int xx = x0 + p * PPL + sub + dx;
      if ((unsigned)xx < (unsigned)W) {
        Vec8<T> v; float f[8];
        v.load(rowp + (size_t)xx * C); v.get(f);
#pragma unroll
        for (int i = 0; i < 8; ++i) fma4(acc[p], f[i], wr[i]);
      }
    }
  }
#pragma unroll
  for (int p = 0; p < P; ++p) {
#pragma unroll
    for (int o = LP / 2; o > 0; o >>= 1) {
      acc[p].x += __shfl_xor_sync(0xffffffffu, acc[p].x, o);
      acc[p].y += __shfl_xor_sync(0xffffffffu, acc[p].y, o);
      acc[p].z += __shfl_xor_sync(0xffffffffu, acc[p].z, o);
      acc[p].w += __shfl_xor_sync(0xffffffffu, acc[p].w, o);
    }
    const int x = x0 + p * PPL + sub;
    if (cl == 0 && x < W) {
      float4 r = acc[p];
      r.x += bias.x; r.y += bias.y; r.z += bias.z; r.w += bias.w;
      const size_t o = ((size_t)n * H + y) * W + x;
      if (addend) { const float4 a = addend[o]; r.x += a.x; r.y += a.y; r.z += a.z; r.w += a.w; }
      out[o] = r;
    }
  }
}

// fp16 tensor-core variant (mma.sync m16n8k16, N = 8 with the 4 real outputs in columns 0..3): a block stages a
// 16x16 pixel tile (+1 halo) of the activation in shared memory once, every warp computes two 16-pixel rows with
// 9 taps x C/16 MMAs each.  ~15x fewer instructions than the CUDA-core kernels above; HBM/L2-bound.
// ASYNC (outconv_variant 3; round 2, the default since -- bit-identical): the 18x18-pixel tile is staged with cp.async
// (16 B each, zero-filled outside the image), i.e. all ~20 (C = 128) / ~40 (C = 256) loads of a thread are in flight at
// once.  The SASS of the plain staging loop is LDG.128 -> STS.128 -> branch: one memory round trip per loop trip, which
// is why the plain form stays well below HBM bandwidth.  Same bytes in shared memory, same arithmetic: bit-identical.
template <int C, bool ASYNC = false>
__global__ void __launch_bounds__(256) out_conv_mma_kernel(const __half* __restrict__ act, int H, int W,
                                                           const float* __restrict__ w, float4 bias,
                                                           const float4* __restrict__ addend, float4* __restrict__ out,
                                                           const float2* __restrict__ gn_ab, const uint2* __restrict__ wfrag_g) {
  constexpr int LD = C + 8;            // halfs per staged pixel (16-byte aligned, conflict-free ldmatrix rows)
  constexpr int KS = C / 16;
  pdl_trigger();                       // weight fragments are constant: staged before pdl_wait()
  extern __shared__ __align__(16) uint8_t oc_smem[];
  __half* tile = reinterpret_cast<__half*>(oc_smem);                       // [18*18][LD]
  uint2* wfrag = reinterpret_cast<uint2*>(oc_smem + (size_t)18 * 18 * LD * 2);   // [9*KS][32] B fragments
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int x0 = blockIdx.x * 16, y0 = blockIdx.y * 16, n = blockIdx.z;
  // B fragments: b0 = (k = 2t, 2t+1 ; n = g), b1 = (k = 2t+8, 2t+9 ; n = g); output columns >= 4 are zero padding
  if (wfrag_g) {                                   // packed at load time: a plain 128-bit copy
    const uint4* src = reinterpret_cast<const uint4*>(wfrag_g);
    for (int i = tid; i < 9 * KS * 16; i += 256) reinterpret_cast<uint4*>(wfrag)[i] = __ldg(src + i);
  } else
  for (int i = tid; i < 9 * KS * 32; i += 256) {
    const int l = i & 31, blk = i >> 5;
    const int tap = blk / KS, kk = blk % KS, gg = l >> 2, tt = l & 3;
    uint2 v = make_uint2(0u, 0u);
    if (gg < 4) {
      const float* wp = w + ((size_t)tap * C + kk * 16 + 2 * tt) * 4 + gg;
      const __half2 b0 = __floats2half2_rn(wp[0], wp[4]);
      const __half2 b1 = __floats2half2_rn(wp[32], wp[36]);
      v.x = *reinterpret_cast<const uint32_t*>(&b0);
      v.y = *reinterpret_cast<const uint32_t*>(&b1);
    }
    wfrag[i] = v;
  }
  // optional fused GroupNorm-apply + SiLU of the RAW tensor while staging (256 % (C/8) == 0: a thread keeps one
  // 8-channel vector, so its (a, b) live in registers); out-of-image pixels stay zero (padding follows the activation)
  pdl_wait();
  float ga[8], gb[8];
  if (gn_ab) {
    const float4* q = reinterpret_cast<const float4*>(gn_ab + (size_t)n * C + (tid % (C / 8)) * 8);
#pragma unroll
    for (int k = 0; k < 4; ++k) { const float4 v = q[k]; ga[2 * k] = v.x; gb[2 * k] = v.y; ga[2 * k + 1] = v.z; gb[2 * k + 1] = v.w; }
  }
  if constexpr (ASYNC) {
    for (int i = tid; i < 18 * 18 * (C / 8); i += 256) {
      const int px = i / (C / 8), cv = i % (C / 8);
      const int y = y0 - 1 + px / 18, x = x0 - 1 + px % 18;
      const bool in = (unsigned)y < (unsigned)H && (unsigned)x < (unsigned)W;
      // src-size 0 -> the 16 destination bytes are zero-filled; the (unused) source address stays inside the tensor
      const __half* src = act + (((size_t)n * H + (in ? y : 0)) * W + (in ? x : 0)) * C + cv * 8;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;"
                   ::"r"(smem_u32(tile + (size_t)px * LD + cv * 8)), "l"(src), "r"(in ? 16 : 0) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
  } else
  for (int i = tid; i < 18 * 18 * (C / 8); i += 256) {
    const int px = i / (C / 8), cv = i % (C / 8);
    const int y = y0 - 1 + px / 18, x = x0 - 1 + px % 18;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if ((unsigned)y < (unsigned)H && (unsigned)x < (unsigned)W) {
      v = *reinterpret_cast<const uint4*>(act + (((size_t)n * H + y) * W + x) * C + cv * 8);
      if (gn_ab) {
        Vec8<__half> vv; vv.raw = v;
        float f[8];
        vv.get(f);
#pragma unroll
        for (int k = 0; k < 8; ++k) f[k] = silu_f(fmaf(ga[k], f[k], gb[k]));
        vv.set(f);
        v = vv.raw;
      }
    }
    *reinterpret_cast<uint4*>(tile + (size_t)px * LD + cv * 8) = v;
  }
  __syncthreads();
#pragma unroll 1
  for (int rr = 0; rr < 2; ++rr) {
    const int ly = warp * 2 + rr;                 // row inside the 16x16 tile
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
    for (int tap = 0; tap < 9; ++tap) {
      // A fragment rows = the 16 pixels (ly + dy, 0..15 + dx) of the staged tile (halo offset 1)
      const __half* arow = tile + (size_t)((ly + tap / 3) * 18 + (tap % 3) + (lane & 15)) * LD + (lane >> 4) * 8;
      const uint2* wf = wfrag + (size_t)tap * KS * 32 + lane;
#pragma unroll 4
      for (int kk = 0; kk < KS; ++kk) {
        uint32_t a[4];
        oc_ldsm_x4(a, arow + kk * 16);
        const uint2 b = wf[kk * 32];
        oc_mma(acc, a, b.x, b.y);
      }
    }
    // C fragment: (row g, cols 2t, 2t+1) and (row g+8, same cols); real outputs are columns 0..3 -> lanes with t < 2
    if (t < 2) {
      const int y = y0 + ly;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int x = x0 + g + h * 8;
        if (y < H && x < W) {
          const size_t o = ((size_t)n * H + y) * W + x;
          float2 r = make_float2(acc[2 * h] + (t == 0 ? bias.x : bias.z), acc[2 * h + 1] + (t == 0 ? bias.y : bias.w));
          if (addend) { const float2 ad = reinterpret_cast<const float2*>(addend + o)[t]; r.x += ad.x; r.y += ad.y; }
          reinterpret_cast<float2*>(out + o)[t] = r;
        }
      }
    }
  }
}

template <int C, bool ASYNC = false>
static void out_conv_mma_launch(cudaStream_t st, const TensorDesc& act, const float* w, float4 b, const float4* addend,
                                float4* out, const float2* gn_ab, const uint2* wfrag) {
  const size_t smem = (size_t)18 * 18 * (C + 8) * 2 + (size_t)9 * (C / 16) * 32 * sizeof(uint2);
  auto k = out_conv_mma_kernel<C, ASYNC>;
  CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(cdiv(act.W, 16), cdiv(act.H, 16), act.N);
  launch_k(k, grid, dim3(256), smem, st, (const __half*)act.p, act.H, act.W, w, b, addend, out, gn_ab, wfrag);
  CUDA_OK(cudaGetLastError());
}

thread_local int g_outconv_variant = 0;   // see kernels.h

template <typename T>
static void out_conv_dispatch(cudaStream_t st, const TensorDesc& act, const float4* w, float4 b, const float4* addend,
                              float4* out) {
  const size_t smem = (size_t)9 * act.C * sizeof(float4);
  const T* ap = (const T*)act.p;
  const int LP = act.C / 8;
  dim3 gridc(cdiv(act.W, 16), cdiv(act.H, 8), act.N);
#define COOP(LP_) \
  do { auto k = out_conv_coop_kernel<T, LP_>; \
       if (smem > 48 * 1024) CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
       k<<<gridc, 256, smem, st>>>(ap, act.H, act.W, w, b, addend, out); } while (0)
  if (LP == 32) COOP(32);
  else if (LP == 16) COOP(16);
  else if (LP == 8) COOP(8);
  else if (LP == 4) COOP(4);
  else if (LP == 2) COOP(2);
  else {
    auto k = out_conv_kernel<T>;
    if (smem > 48 * 1024) CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(cdiv(act.W, 16), cdiv(act.H, 16), act.N);
    k<<<grid, 256, smem, st>>>(ap, act.H, act.W, act.C, w, b, addend, out);
  }
#undef COOP
  CUDA_OK(cudaGetLastError());
}

bool out_conv_fuses_gn(const TensorDesc& act) {
  return act.dt == DT_F16 && g_outconv_variant == 2 && (act.C == 128 || act.C == 256);
}

void launch_out_conv(cudaStream_t st, const TensorDesc& act, const float* w, const float* bias,
                     const float4* addend, float4* out, const float2* gn_ab, const uint2* wfrag) {
  SG_CHECK(!gn_ab || out_conv_fuses_gn(act), "out conv: fused GroupNorm is only available in the tensor-core kernel");
  SG_CHECK(act.C % 8 == 0, "out conv: C must be a multiple of 8");
  SG_CHECK((size_t)9 * act.C * sizeof(float4) <= 96 * 1024, "out conv: %d channels exceed the shared-memory weight buffer", act.C);
  // `bias` is a HOST pointer to 4 floats (kept with the layer description)
  const float4 b = make_float4(bias[0], bias[1], bias[2], bias[3]);
  if (act.dt == DT_F16 && g_outconv_variant != 1 && (act.C == 128 || act.C == 256)) {
    if (g_outconv_variant == 3 && !gn_ab) {
      if (act.C == 128) out_conv_mma_launch<128, true>(st, act, w, b, addend, out, gn_ab, wfrag);
      else out_conv_mma_launch<256, true>(st, act, w, b, addend, out, gn_ab, wfrag);
      return;
    }
    if (act.C == 128) out_conv_mma_launch<128>(st, act, w, b, addend, out, gn_ab, wfrag);
    else out_conv_mma_launch<256>(st, act, w, b, addend, out, gn_ab, wfrag);
    return;
  }
  if (act.dt == DT_F16) out_conv_dispatch<__half>(st, act, (const float4*)w, b, addend, out);
  else out_conv_dispatch<float>(st, act, (const float4*)w, b, addend, out);
}

}  // namespace sgmse
