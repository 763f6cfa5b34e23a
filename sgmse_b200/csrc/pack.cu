// Device-side weight packing: the layouts of engine.cu: load_weights() produced from the fp32 state_dict blob where it already
// lives -- in HBM.  sgmse_b200_load_weights_device (a re-snapshot of model.dnn after an EMA swap, SURVEY.md section 8f-3) used to
// copy the 262 MB blob to the host, repack it there and upload ~400 MB again; these kernels read the blob once and write the
// packed tensors directly.  Every element is the same fp32 value, rounded at the same point, as on the host path
// (tests/test_gpu_parity.py::test_device_side_weight_packing_equals_the_host_path: bit-identical network outputs).
#include "kernels.h"

namespace sgmse {

// [k][cout] (fp32 or fp16) and, optionally, [cout][ld] fp16 (K-major, conv_tc) of up to four K segments.
//   mode 0: Conv2d weights [cout][cin][taps];  mode 1: NIN weights [cin][cout];
//   mode 2: three NIN weights [cin][cout/3] side by side (q | k | v of the attention block; seg[0..2].w hold the three offsets)
template <typename T>
__global__ void pack_conv_kernel(const float* __restrict__ blob, PackJob j, T* __restrict__ kd, __half* __restrict__ ht) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)j.ktot * j.cout) return;
  const int k = (int)(idx / j.cout), co = (int)(idx - (long long)k * j.cout);
  float v;
  if (j.mode == 2) {
    const int C = j.cout / 3, part = co / C;
    v = blob[j.seg[part].w + (long long)k * C + (co - part * C)];
  } else {
    int s = 0;
    while (s + 1 < j.nseg && k >= j.seg[s + 1].kbase) ++s;
    const int kk = k - j.seg[s].kbase, cin = j.seg[s].cin, taps = j.seg[s].taps;
    const int tap = kk / cin, ci = kk - tap * cin;
    v = j.mode == 0 ? blob[j.seg[s].w + ((long long)co * cin + ci) * taps + tap] : blob[j.seg[s].w + (long long)ci * j.cout + co];
  }
  if (sizeof(T) == 2) reinterpret_cast<__half*>(kd)[idx] = __float2half_rn(v);
  else reinterpret_cast<float*>(kd)[idx] = v;
  if (ht) ht[(long long)co * j.ld + k] = __float2half_rn(v);
}
__global__ void identity_tail_kernel(__half* __restrict__ ht, int cout, int ld, int ktot) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;           // over cout * cout: zeros off the diagonal, ones on it
  if (idx >= cout * cout) return;
  const int co = idx / cout, c2 = idx - co * cout;
  ht[(long long)co * ld + ktot + c2] = __float2half_rn(co == c2 ? 1.f : 0.f);
}
// input conv [nf][4][3][3] -> [36][nf]
__global__ void pack_inconv_kernel(const float* __restrict__ w, int nf, float* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= 36 * nf) return;
  const int k = idx / nf, co = idx - k * nf, tap = k / 4, ci = k - tap * 4;
  out[idx] = w[((long long)co * 4 + ci) * 9 + tap];
}
// Combine conv1x1 [C][4] -> [4][C]
__global__ void pack_combine_kernel(const float* __restrict__ w, int C, float* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= 4 * C) return;
  const int ci = idx / C, co = idx - ci * C;
  out[idx] = w[(long long)co * 4 + ci];
}
// progressive-output conv [4][C][3][3] -> [9 C][4]
__global__ void pack_outconv_kernel(const float* __restrict__ w, int C, float* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= 9 * C * 4) return;
  const int o = idx & 3, r = idx >> 2, tap = r / C, ci = r - tap * C;
  out[idx] = w[((long long)o * C + ci) * 9 + tap];
}
// ... and its mma.sync B fragments [9][C/16][32] (see engine.cu: load_weights)
__global__ void pack_outconv_frag_kernel(const float* __restrict__ p, int C, uint2* __restrict__ fr) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int KS = C / 16;
  if (idx >= 9 * KS * 32) return;
  const int ln = idx & 31, kk = (idx >> 5) % KS, tap = idx / (32 * KS);
  const int gg = ln >> 2, tt = ln & 3;
  uint2 v = make_uint2(0u, 0u);
  if (gg < 4) {
    const float* wp = p + ((long long)tap * C + kk * 16 + 2 * tt) * 4 + gg;
    const __half2 a = __floats2half2_rn(wp[0], wp[4]), b = __floats2half2_rn(wp[32], wp[36]);
    v = make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
  }
  fr[idx] = v;
}
__global__ void add_vec_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = a[i] + (b ? b[i] : 0.f);
}

static inline unsigned blocks(long long n) { return (unsigned)((n + 255) / 256); }

void launch_pack_conv(cudaStream_t st, const float* blob, const PackJob& j, void* kd, bool kd_half, __half* ht) {
  const long long n = (long long)j.ktot * j.cout;
  if (kd_half) pack_conv_kernel<__half><<<blocks(n), 256, 0, st>>>(blob, j, (__half*)kd, ht);
  else pack_conv_kernel<float><<<blocks(n), 256, 0, st>>>(blob, j, (float*)kd, ht);
  CUDA_OK(cudaGetLastError());
  if (ht && j.identity_tail) {
    identity_tail_kernel<<<blocks((long long)j.cout * j.cout), 256, 0, st>>>(ht, j.cout, j.ld, j.ktot);
    CUDA_OK(cudaGetLastError());
  }
}
void launch_pack_inconv(cudaStream_t st, const float* w, int nf, float* out) {
  pack_inconv_kernel<<<blocks(36LL * nf), 256, 0, st>>>(w, nf, out);
  CUDA_OK(cudaGetLastError());
}
void launch_pack_combine(cudaStream_t st, const float* w, int C, float* out) {
  pack_combine_kernel<<<blocks(4LL * C), 256, 0, st>>>(w, C, out);
  CUDA_OK(cudaGetLastError());
}
void launch_pack_outconv(cudaStream_t st, const float* w, int C, float* out, uint2* frag) {
  pack_outconv_kernel<<<blocks(36LL * C), 256, 0, st>>>(w, C, out);
  CUDA_OK(cudaGetLastError());
  if (frag) {
    pack_outconv_frag_kernel<<<blocks(9LL * (C / 16) * 32), 256, 0, st>>>(out, C, frag);
    CUDA_OK(cudaGetLastError());
  }
}
void launch_add_vec(cudaStream_t st, const float* a, const float* b, float* out, int n) {
  add_vec_kernel<<<blocks(n), 256, 0, st>>>(a, b, out, n);
  CUDA_OK(cudaGetLastError());
}

}  // namespace sgmse
