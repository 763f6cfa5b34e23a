// CUDA-core implicit-GEMM convolution (3x3 pad 1 / 1x1, multi-segment K, fused epilogue).
//
// This is the *validation* convolution: fp32 (or fp16-storage) arithmetic with fp32 accumulation,
// any channel count that is a multiple of 16.  It implements exactly the same contract as the
// wgmma kernel in conv_tc.cu (same K ordering, same epilogue, same statistics side-output), so
// that (a) the engine has an fp32-accurate mode to separate algorithmic from precision error and
// (b) the tensor-core kernel can be checked against it on the device.
//
// Reference semantics: F.conv2d in ResnetBlockBigGANpp (layerspp.py:260-269), NIN (layers.py:546-555).
#include "kernels.h"

namespace sgmse {

namespace {
constexpr int TM = 32;   // pixels per block
constexpr int TN = 64;   // output channels per block
constexpr int KC = 16;   // K chunk

struct SegDev {
  const void* p;
  int C;
  int taps;
};
struct DirectParams {
  SegDev seg[3];
  int nseg;
  int N, H, W, Cout, M;
  const void* w;       // [Ktot][Cout]
  const float* bias;
  const float* temb;
  int temb_stride;
  const void* residual;
  float scale;
  void* out;
  float* stats;        // [N][slots][Cout][2]
  int slots;
};

template <typename T>
__global__ void __launch_bounds__(128) conv_direct_kernel(const DirectParams P) {
  __shared__ __align__(16) float As[KC][TM + 4];
  __shared__ __align__(16) float Bs[KC][TN];
  __shared__ float red[8][TN][2];

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.x * TM;
  const int n0c = blockIdx.y * TN;
  const int HW = P.H * P.W;

  // the pixel this thread loads for the A tile
  const int lp = tid >> 2;          // 0..31
  const int lc = (tid & 3) * 4;     // cin offset inside the chunk
  const int lm = m0 + lp;
  const int ln = lm / HW;
  const int lrem = lm - ln * HW;
  const int ly = lrem / P.W, lx = lrem - ly * P.W;
  // B tile load coordinates
  const int bk = tid >> 3;          // 0..15
  const int bc = (tid & 7) * 8;     // 0..56

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  int kbase = 0;
  for (int s = 0; s < P.nseg; ++s) {
    const T* src = (const T*)P.seg[s].p;
    const int Cs = P.seg[s].C;
    const int taps = P.seg[s].taps;
    for (int tap = 0; tap < taps; ++tap) {
      const int dy = taps == 9 ? tap / 3 - 1 : 0;
      const int dx = taps == 9 ? tap % 3 - 1 : 0;
      const int yy = ly + dy, xx = lx + dx;
      const bool inb = lm < P.M && (unsigned)yy < (unsigned)P.H && (unsigned)xx < (unsigned)P.W;
      const T* arow = src + (((size_t)ln * P.H + yy) * P.W + xx) * Cs + lc;
      for (int c0 = 0; c0 < Cs; c0 += KC) {
        // ---- stage A (transposed) and B ----
        float av[4] = {0.f, 0.f, 0.f, 0.f};
        if (inb) {
#pragma unroll
          for (int i = 0; i < 4; ++i) av[i] = Act<T>::ld(arow + c0 + i);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) As[lc + i][lp] = av[i];
        {
          const int krow = kbase + tap * Cs + c0 + bk;
          const T* wrow = (const T*)P.w + (size_t)krow * P.Cout + n0c + bc;
          if (n0c + bc < P.Cout) {
            Vec8<T> v; float f[8];
            v.load(wrow); v.get(f);
#pragma unroll
            for (int i = 0; i < 8; ++i) Bs[bk][bc + i] = f[i];
          } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) Bs[bk][bc + i] = 0.f;
          }
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < KC; ++k) {
          const float4 a4 = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
          const float4 b4 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
          const float a[4] = {a4.x, a4.y, a4.z, a4.w};
          const float b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
      }
    }
    kbase += taps * Cs;
  }

  // ---- epilogue ----
  float ssum[4] = {0.f, 0.f, 0.f, 0.f}, ssq[4] = {0.f, 0.f, 0.f, 0.f};
  const int cbase = n0c + tx * 4;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    const int n = m / HW;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = cbase + j;
      if (c < P.Cout && m < P.M) {
        float v = acc[i][j];
        if (P.bias) v += P.bias[c];
        if (P.temb) v += P.temb[(size_t)n * P.temb_stride + c];
        if (P.residual) v += Act<T>::ld((const T*)P.residual + (size_t)m * P.Cout + c);
        v *= P.scale;
        T* op = (T*)P.out + (size_t)m * P.Cout + c;
        Act<T>::st(op, v);
        const float r = Act<T>::rnd(v);
        ssum[j] += r; ssq[j] += r * r;
      }
    }
  }
  if (P.stats) {
#pragma unroll
    for (int j = 0; j < 4; ++j) { red[ty][tx * 4 + j][0] = ssum[j]; red[ty][tx * 4 + j][1] = ssq[j]; }
    __syncthreads();
    if (tid < TN && n0c + tid < P.Cout) {
      float s = 0.f, q = 0.f;
#pragma unroll
      for (int r = 0; r < 8; ++r) { s += red[r][tid][0]; q += red[r][tid][1]; }
      const int n = m0 / HW;
      const int slot = (m0 - n * HW) / TM;
      float* dst = P.stats + (((size_t)n * P.slots + slot) * P.Cout + n0c + tid) * 2;
      dst[0] = s; dst[1] = q;
    }
  }
}
}  // namespace

void launch_conv_direct(cudaStream_t st, const ConvArgs& a, TensorDesc& out) {
  SG_CHECK(a.nseg >= 1 && a.nseg <= 3, "conv: bad segment count %d", a.nseg);
  DirectParams P{};
  P.nseg = a.nseg;
  for (int i = 0; i < a.nseg; ++i) {
    const TensorDesc& s = a.seg[i].src;
    SG_CHECK(s.N == out.N && s.H == out.H && s.W == out.W, "conv: segment %d shape mismatch", i);
    SG_CHECK(s.dt == out.dt, "conv: dtype mismatch");
    SG_CHECK(s.C % KC == 0, "conv_direct: Cin=%d must be a multiple of %d", s.C, KC);
    SG_CHECK(a.seg[i].taps == 9 || a.seg[i].taps == 1, "conv: taps must be 9 or 1");
    P.seg[i] = SegDev{s.p, s.C, a.seg[i].taps};
  }
  SG_CHECK(out.C % 8 == 0, "conv_direct: Cout=%d must be a multiple of 8", out.C);
  P.N = out.N; P.H = out.H; P.W = out.W; P.Cout = out.C; P.M = out.N * out.H * out.W;
  P.w = a.w_direct; P.bias = a.bias; P.temb = a.temb; P.temb_stride = a.temb_stride;
  P.residual = a.residual ? a.residual->p : nullptr;
  if (a.residual) SG_CHECK(a.residual->C == out.C && a.residual->dt == out.dt, "conv: residual mismatch");
  P.scale = a.scale; P.out = out.p;
  // per-tile statistics need tiles that do not straddle samples; tiny levels use a separate pass instead
  const bool tile_stats = out.stats && (out.H * out.W) % TM == 0;
  out.slots = tile_stats ? out.H * out.W / TM : 0;
  P.stats = tile_stats ? out.stats : nullptr; P.slots = out.slots;
  SG_CHECK(a.w_direct != nullptr, "conv_direct: missing weights");
  dim3 grid((unsigned)cdiv(P.M, TM), (unsigned)cdiv(out.C, TN));
  if (out.dt == DT_F16) conv_direct_kernel<__half><<<grid, 128, 0, st>>>(P);
  else conv_direct_kernel<float><<<grid, 128, 0, st>>>(P);
  CUDA_OK(cudaGetLastError());
  if (out.stats && !tile_stats) launch_channel_stats(st, out);
}

}  // namespace sgmse
