// Single-head global self-attention over the H*W tokens of one utterance (AttnBlockpp core).
//
// Reference: sgmse/backbones/ncsnpp_utils/layerspp.py:82-86
//   w = softmax_k( sum_c q[c,tok] k[c,key] / sqrt(C) );  h[tok] = sum_key w v[key]
// 0.16 % of the network FLOPs (SURVEY.md §8a) -> fp32 CUDA-core kernel, smem-tiled; the q/k/v
// projections and the output projection run through the convolution kernels as 1x1 convs.
#include "kernels.h"

namespace sgmse {

namespace {
constexpr int KT = 64;  // keys per tile

template <typename T, int QT>
__global__ void __launch_bounds__(128) attention_kernel(const T* __restrict__ qkv, int S, int C, float scale,
                                                        T* __restrict__ out) {
  extern __shared__ float sm[];
  const int ldq = C + 1;
  const int lds = S + 1;
  float* Qs = sm;                    // [QT][C+1]
  float* KVs = Qs + QT * ldq;        // [KT][C+1]
  float* Ss = KVs + KT * ldq;        // [QT][S+1]
  const int n = blockIdx.y;
  const int q0 = blockIdx.x * QT;
  const int tid = threadIdx.x;
  const T* base = qkv + (size_t)n * S * 3 * C;
  constexpr int QG = QT / 4;         // query groups of 4
  constexpr int NT = 128 / QG;       // threads along keys / channels
  const int tq = tid / NT, tk = tid % NT;

  // ---- load Q tile ----
  for (int i = tid; i < QT * (C / 8); i += 128) {
    const int q = i / (C / 8), cv = i % (C / 8);
    float f[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (q0 + q < S) { Vec8<T> v; v.load(base + (size_t)(q0 + q) * 3 * C + cv * 8); v.get(f); }
#pragma unroll
    for (int j = 0; j < 8; ++j) Qs[q * ldq + cv * 8 + j] = f[j];
  }
  // ---- scores ----
  for (int k0 = 0; k0 < S; k0 += KT) {
    __syncthreads();
    for (int i = tid; i < KT * (C / 8); i += 128) {
      const int k = i / (C / 8), cv = i % (C / 8);
      float f[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (k0 + k < S) { Vec8<T> v; v.load(base + (size_t)(k0 + k) * 3 * C + C + cv * 8); v.get(f); }
#pragma unroll
      for (int j = 0; j < 8; ++j) KVs[k * ldq + cv * 8 + j] = f[j];
    }
    __syncthreads();
    // each thread: 4 queries x (KT/NT) keys, keys interleaved by NT
    constexpr int KPT = KT / NT;
    float acc[4][KPT];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < KPT; ++j) acc[i][j] = 0.f;
    for (int c = 0; c < C; ++c) {
      float qv[4], kv[KPT];
#pragma unroll
      for (int i = 0; i < 4; ++i) qv[i] = Qs[(tq * 4 + i) * ldq + c];
#pragma unroll
      for (int j = 0; j < KPT; ++j) kv[j] = KVs[(tk + j * NT) * ldq + c];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < KPT; ++j) acc[i][j] = fmaf(qv[i], kv[j], acc[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < KPT; ++j) {
        const int k = k0 + tk + j * NT;
        if (k < S) Ss[(tq * 4 + i) * lds + k] = acc[i][j] * scale;
      }
  }
  __syncthreads();
  // ---- softmax rows (one warp per row, round robin) ----
  {
    const int warp = tid >> 5, lane = tid & 31;
    for (int q = warp; q < QT; q += 4) {
      float* row = Ss + q * lds;
      float mx = -INFINITY;
      for (int k = lane; k < S; k += 32) mx = fmaxf(mx, row[k]);
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      float sum = 0.f;
      for (int k = lane; k < S; k += 32) { const float e = __expf(row[k] - mx); row[k] = e; sum += e; }
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      const float inv = 1.f / sum;
      for (int k = lane; k < S; k += 32) row[k] *= inv;
    }
  }
  // ---- O = P V ; thread: 4 queries x channels {tk, tk+NT, ...} handled in passes of 16 channels ----
  for (int cb = 0; cb < C; cb += 16 * NT) {
    float o[4][16];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 16; ++j) o[i][j] = 0.f;
    for (int k0 = 0; k0 < S; k0 += KT) {
      __syncthreads();
      for (int i = tid; i < KT * (C / 8); i += 128) {
        const int k = i / (C / 8), cv = i % (C / 8);
        float f[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (k0 + k < S) { Vec8<T> v; v.load(base + (size_t)(k0 + k) * 3 * C + 2 * C + cv * 8); v.get(f); }
#pragma unroll
        for (int j = 0; j < 8; ++j) KVs[k * ldq + cv * 8 + j] = f[j];
      }
      __syncthreads();
      const int kmax = (S - k0) < KT ? (S - k0) : KT;
      for (int k = 0; k < kmax; ++k) {
        float p[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) p[i] = Ss[(tq * 4 + i) * lds + k0 + k];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int c = cb + tk + j * NT;
          const float v = c < C ? KVs[k * ldq + c] : 0.f;
#pragma unroll
          for (int i = 0; i < 4; ++i) o[i][j] = fmaf(p[i], v, o[i][j]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int q = q0 + tq * 4 + i;
      if (q >= S) continue;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = cb + tk + j * NT;
        if (c < C) Act<T>::st(out + ((size_t)n * S + q) * C + c, o[i][j]);
      }
    }
  }
}

template <typename T, int QT>
static void run(cudaStream_t st, const TensorDesc& qkv, TensorDesc& out, int S, int C, size_t smem) {
  auto kern = attention_kernel<T, QT>;
  CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(cdiv(S, QT), qkv.N);
  kern<<<grid, 128, smem, st>>>((const T*)qkv.p, S, C, 1.0f / sqrtf((float)C), (T*)out.p);
  CUDA_OK(cudaGetLastError());
}

// fp32 storage at any token count: the full score row of attention_kernel outgrows shared memory past S ~ 4 700
// (C = 256).  Flash-style instead: a block keeps 32 queries resident, streams keys and values through shared memory in
// tiles of KT and keeps a running max and sum per query (online softmax).  fp32 CUDA-core FMAs throughout, as every
// non-convolution kernel of the fp32 and tf32_tc modes.  Thread (tq, tk): queries 4 tq .. 4 tq + 3; keys tk + 16 j of a
// tile for the scores, channels tk + 16 j of the output.
constexpr int SQT = 32;
template <int C>
size_t stream_smem() { return ((size_t)(SQT + KT) * (C + 1) + SQT * (KT + 1) + 2 * SQT) * sizeof(float); }

template <int C>
__global__ void __launch_bounds__(128) attention_stream_kernel(const float* __restrict__ qkv, int S, float scale_log2e,
                                                               float* __restrict__ out) {
  constexpr int LD = C + 1, LDP = KT + 1, CPT = C / 16;
  extern __shared__ float sm[];
  float* Qs = sm;                    // [SQT][LD]
  float* KVs = Qs + SQT * LD;        // [KT][LD]: the key tile, then the value tile
  float* Ps = KVs + KT * LD;         // [SQT][LDP]: scores, then probabilities (log2 domain)
  float* alpha = Ps + SQT * LDP;     // [SQT]: rescale factor of the running output for this tile
  float* lsum = alpha + SQT;         // [SQT]: final softmax denominators
  const int n = blockIdx.y, q0 = blockIdx.x * SQT;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tq = tid / 16, tk = tid % 16;
  const float* base = qkv + (size_t)n * S * 3 * C;

  auto load_tile = [&](float* dst, int rows, int row0, int col0) {
    for (int i = tid; i < rows * (C / 4); i += 128) {
      const int r = i / (C / 4), cv = i % (C / 4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row0 + r < S) v = *reinterpret_cast<const float4*>(base + (size_t)(row0 + r) * 3 * C + col0 + cv * 4);
      float* d = dst + r * LD + cv * 4;
      d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
    }
  };
  load_tile(Qs, SQT, q0, 0);

  float o[4][CPT];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < CPT; ++j) o[i][j] = 0.f;
  float mrow[SQT / 4], lrow[SQT / 4];          // rows warp * 8 + r, replicated over the warp's lanes
#pragma unroll
  for (int r = 0; r < SQT / 4; ++r) { mrow[r] = -INFINITY; lrow[r] = 0.f; }

  for (int k0 = 0; k0 < S; k0 += KT) {
    __syncthreads();                           // previous tile's P V done with KVs and Ps
    load_tile(KVs, KT, k0, C);
    __syncthreads();
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int c = 0; c < C; ++c) {
      float qv[4], kv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) qv[i] = Qs[(tq * 4 + i) * LD + c];
#pragma unroll
      for (int j = 0; j < 4; ++j) kv[j] = KVs[(tk + 16 * j) * LD + c];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(qv[i], kv[j], acc[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j)
        Ps[(tq * 4 + i) * LDP + tk + 16 * j] = k0 + tk + 16 * j < S ? acc[i][j] * scale_log2e : -INFINITY;
    __syncthreads();                           // scores complete; the key tile is no longer read
    // online softmax: warp w owns rows 8 w .. 8 w + 7, two keys per lane
#pragma unroll
    for (int r = 0; r < SQT / 4; ++r) {
      float* row = Ps + (warp * (SQT / 4) + r) * LDP;
      const float s0 = row[lane], s1 = row[lane + 32];
      float mx = fmaxf(s0, s1);
      for (int of = 16; of > 0; of >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, of));
      mx = fmaxf(mx, mrow[r]);                 // finite: key k0 of the first tile is always a real token
      const float p0 = exp2f(s0 - mx), p1 = exp2f(s1 - mx);
      row[lane] = p0; row[lane + 32] = p1;
      float sum = p0 + p1;
      for (int of = 16; of > 0; of >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, of);
      const float a = exp2f(mrow[r] - mx);
      lrow[r] = lrow[r] * a + sum;
      mrow[r] = mx;
      if (lane == 0) alpha[warp * (SQT / 4) + r] = a;
    }
    load_tile(KVs, KT, k0, 2 * C);             // value tile (zero past S, where p = 0 as well)
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float a = alpha[tq * 4 + i];
#pragma unroll
      for (int j = 0; j < CPT; ++j) o[i][j] *= a;
    }
    for (int k = 0; k < KT; ++k) {
      float p[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) p[i] = Ps[(tq * 4 + i) * LDP + k];
#pragma unroll
      for (int j = 0; j < CPT; ++j) {
        const float v = KVs[k * LD + tk + 16 * j];
#pragma unroll
        for (int i = 0; i < 4; ++i) o[i][j] = fmaf(p[i], v, o[i][j]);
      }
    }
  }
  if (lane == 0)
#pragma unroll
    for (int r = 0; r < SQT / 4; ++r) lsum[warp * (SQT / 4) + r] = lrow[r];
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int q = q0 + tq * 4 + i;
    if (q >= S) continue;
    const float inv = 1.f / lsum[tq * 4 + i];
#pragma unroll
    for (int j = 0; j < CPT; ++j) out[((size_t)n * S + q) * C + tk + 16 * j] = o[i][j] * inv;
  }
}

template <int C>
void run_stream(cudaStream_t st, const TensorDesc& qkv, TensorDesc& out, int S) {
  auto kern = attention_stream_kernel<C>;
  CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)stream_smem<C>()));
  dim3 grid(cdiv(S, SQT), qkv.N);
  kern<<<grid, 128, stream_smem<C>(), st>>>((const float*)qkv.p, S, 1.4426950408889634f / sqrtf((float)C), (float*)out.p);
  CUDA_OK(cudaGetLastError());
}
}  // namespace

// ------------------------------------------------------------------------------------------------
// fp16 tensor-core path (mma.sync m16n8k16, fp32 accumulate), flash-style online softmax.
// One block = 64 queries of one utterance (4 warps x 16 queries); keys/values stream through smem in tiles of 64.
// mma.sync rather than wgmma on purpose: attention is 0.16 % of the network FLOPs and its tiles (S <= 512 tokens,
// head dim 128/256) are too small to amortise a warpgroup pipeline; the convolutions own the wgmma kernels.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}

namespace {
// ASYNC (the default; attn_variant 3 selects the plain staging, bit-identical): Q/K/V tiles are staged with cp.async (zero-fill past the
// last token).  The SASS of the plain load_tile loop is LDG.128 -> STS.128 -> branch, 16 (C = 128) / 32 (C = 256) serialized
// round trips per tile and two tiles per key block, i.e. the plain form is latency-bound on its loads.  Same bytes in
// shared memory, same arithmetic: bit-identical.
template <int C, bool ASYNC = false>
__global__ void __launch_bounds__(128) attention_tc_kernel(const __half* __restrict__ qkv, int S, float scale_log2e,
                                                           __half* __restrict__ out) {
  pdl_trigger(); pdl_wait();
  constexpr int LD = C + 8;                       // padded row (halfs): 16-byte aligned rows, conflict-free fragments
  extern __shared__ __align__(16) __half smh[];
  __half* Qs = smh;                               // [64][LD]
  __half* Ks = Qs + 64 * LD;
  __half* Vs = Ks + 64 * LD;
  const int n = blockIdx.y, q0 = blockIdx.x * 64;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const __half* base = qkv + (size_t)n * S * 3 * C;

  auto load_tile = [&](__half* dst, int row0, int col0) {
    for (int i = tid; i < 64 * (C / 8); i += 128) {
      const int r = i / (C / 8), cv = i % (C / 8);
      if constexpr (ASYNC) {
        const bool in = row0 + r < S;             // src-size 0 -> zero fill; the unused address stays inside the tensor
        const __half* src = base + (size_t)(in ? row0 + r : 0) * 3 * C + col0 + cv * 8;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;"
                     ::"r"((uint32_t)__cvta_generic_to_shared(dst + r * LD + cv * 8)), "l"(src), "r"(in ? 16 : 0) : "memory");
      } else {
        uint4 v = make_uint4(0, 0, 0, 0);
        if (row0 + r < S) v = *reinterpret_cast<const uint4*>(base + (size_t)(row0 + r) * 3 * C + col0 + cv * 8);
        *reinterpret_cast<uint4*>(dst + r * LD + cv * 8) = v;
      }
    }
  };
  auto tiles_landed = [&]() {
    if constexpr (ASYNC) {
      asm volatile("cp.async.commit_group;" ::: "memory");
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
  };
  load_tile(Qs, q0, 0);

  float oacc[C / 8][4];
#pragma unroll
  for (int j = 0; j < C / 8; ++j) { oacc[j][0] = oacc[j][1] = oacc[j][2] = oacc[j][3] = 0.f; }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;     // rows g and g+8 of this warp's 16 queries

  for (int k0 = 0; k0 < S; k0 += 64) {
    __syncthreads();
    load_tile(Ks, k0, C);
    load_tile(Vs, k0, 2 * C);
    tiles_landed();
    __syncthreads();
    float sacc[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { sacc[j][0] = sacc[j][1] = sacc[j][2] = sacc[j][3] = 0.f; }
#pragma unroll 4
    for (int kk = 0; kk < C / 16; ++kk) {
      uint32_t a[4];
      ldsm_x4(a, Qs + (warp * 16 + (lane & 15)) * LD + kk * 16 + (lane >> 4) * 8);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const __half* kr = Ks + (j * 8 + g) * LD + kk * 16 + 2 * t;
        mma_16816(sacc[j], a, *reinterpret_cast<const uint32_t*>(kr), *reinterpret_cast<const uint32_t*>(kr + 8));
      }
    }
    // online softmax in the log2 domain
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int key = k0 + j * 8 + 2 * t + (i & 1);
        sacc[j][i] = key < S ? sacc[j][i] * scale_log2e : -INFINITY;
      }
      mx0 = fmaxf(mx0, fmaxf(sacc[j][0], sacc[j][1]));
      mx1 = fmaxf(mx1, fmaxf(sacc[j][2], sacc[j][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float al0 = exp2f(m0 - mx0), al1 = exp2f(m1 - mx1);
    m0 = mx0; m1 = mx1;
    l0 *= al0; l1 *= al1;
#pragma unroll
    for (int j = 0; j < C / 8; ++j) { oacc[j][0] *= al0; oacc[j][1] *= al0; oacc[j][2] *= al1; oacc[j][3] *= al1; }
    uint32_t pa[4][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float p0 = exp2f(sacc[j][0] - m0), p1 = exp2f(sacc[j][1] - m0);
      const float p2 = exp2f(sacc[j][2] - m1), p3 = exp2f(sacc[j][3] - m1);
      l0 += p0 + p1; l1 += p2 + p3;
      // S accumulator tiles 2kk, 2kk+1 -> A fragment of the P V product (k = keys)
      pa[j >> 1][(j & 1) * 2 + 0] = pack_half2(p0, p1);
      pa[j >> 1][(j & 1) * 2 + 1] = pack_half2(p2, p3);
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int jn = 0; jn < C / 8; jn += 2) {
        uint32_t b[4];
        // V tile is [key][channel]: transposed 8x8 loads give the k-major B fragments of two channel octets
        ldsm_x4_trans(b, Vs + (kk * 16 + (lane & 15)) * LD + (jn + (lane >> 4)) * 8);
        mma_16816(oacc[jn], pa[kk], b[0], b[1]);
        mma_16816(oacc[jn + 1], pa[kk], b[2], b[3]);
      }
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.f / l0, i1 = 1.f / l1;
  const int qa = q0 + warp * 16 + g, qb = qa + 8;
#pragma unroll
  for (int j = 0; j < C / 8; ++j) {
    const int c = j * 8 + 2 * t;
    if (qa < S) *reinterpret_cast<__half2*>(out + ((size_t)n * S + qa) * C + c) = __floats2half2_rn(oacc[j][0] * i0, oacc[j][1] * i0);
    if (qb < S) *reinterpret_cast<__half2*>(out + ((size_t)n * S + qb) * C + c) = __floats2half2_rn(oacc[j][2] * i1, oacc[j][3] * i1);
  }
}

template <int C, bool ASYNC = false>
void run_tc(cudaStream_t st, const TensorDesc& qkv, TensorDesc& out, int S) {
  const size_t smem = (size_t)3 * 64 * (C + 8) * sizeof(__half);
  auto kern = attention_tc_kernel<C, ASYNC>;
  CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(cdiv(S, 64), qkv.N);
  launch_k(kern, grid, dim3(128), smem, st, (const __half*)qkv.p, S, 1.4426950408889634f / sqrtf((float)C), (__half*)out.p);
  CUDA_OK(cudaGetLastError());
}
}  // namespace

thread_local int g_attn_variant = 0;   // see kernels.h

void launch_attention(cudaStream_t st, const TensorDesc& qkv, TensorDesc& out) {
  const int C = out.C, S = qkv.H * qkv.W;
  SG_CHECK(qkv.C == 3 * C && C % 8 == 0, "attention: qkv must have 3C channels");
  if (qkv.dt == DT_F16 && (g_attn_variant == 0 || g_attn_variant == 2)) {
    if (C == 256) { run_tc<256, true>(st, qkv, out, S); return; }
    if (C == 128) { run_tc<128, true>(st, qkv, out, S); return; }
  }
  if (qkv.dt == DT_F16 && g_attn_variant == 3) {
    if (C == 256) { run_tc<256>(st, qkv, out, S); return; }
    if (C == 128) { run_tc<128>(st, qkv, out, S); return; }
  }
  auto smem_for = [&](int QT) { return (size_t)((QT + KT) * (C + 1) + QT * (S + 1)) * sizeof(float); };
  const size_t lim = 220 * 1024;
  int QT = 32;
  if (smem_for(32) > lim) QT = 16;
  if (QT == 16 && smem_for(16) > lim) QT = 8;
  if (smem_for(QT) > lim && qkv.dt == DT_F32) {  // the full score row does not fit: stream the keys
    if (C == 256) { run_stream<256>(st, qkv, out, S); return; }
    if (C == 128) { run_stream<128>(st, qkv, out, S); return; }
  }
  SG_CHECK(smem_for(QT) <= lim, "attention: %d tokens x %d channels does not fit the v1 kernel", S, C);
#define GO(T) \
  do { if (QT == 32) run<T, 32>(st, qkv, out, S, C, smem_for(32)); \
       else if (QT == 16) run<T, 16>(st, qkv, out, S, C, smem_for(16)); \
       else run<T, 8>(st, qkv, out, S, C, smem_for(8)); } while (0)
  if (qkv.dt == DT_F16) GO(__half); else GO(float);
#undef GO
}

}  // namespace sgmse
