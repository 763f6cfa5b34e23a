// wgmma implicit-GEMM convolution for sm_90a (3x3 pad-1 / 1x1, NHWC fp16 -> fp16, fp32 accumulate in registers).
//
//   D[pixel, cout] = sum_{segment, tap, cin} A_seg[pixel + tap offset, cin] * W[cout, (segment, tap, cin)]
//
// GEMM view: M = N*H*W pixels (tiles of 128 = one TMA box bw x bh x bn of pixels), N = Cout (tiles of
// BLOCK_N), K = sum over segments of taps*Cin (blocks of 64 channels of one tap).  There is no im2col
// buffer: for each (tap, 64-channel chunk) the producer issues ONE 4-D TMA box load of the activation
// tensor at the tap-shifted pixel coordinates; TMA zero-fills out-of-bounds pixels, which is exactly
// the conv's zero padding, and lands the box as a 128-row K-major SWIZZLE_128B operand tile.  Several
// K segments let one accumulator take  conv3x3(h) + conv1x1(x_a) + conv1x1(x_b)  (ResnetBlockBigGANpp's
// Conv_1 plus the Conv_2 shortcut over a concatenated skip input) without materialising the concat.
//
// Persistent, warp-specialised CTA (384 threads = 3 warpgroups, 1 CTA/SM):
//   warpgroup 0   producer: one thread issues the TMA loads into an smem ring of NUM_STAGES x {A 16 KB,
//                 B BLOCK_N*128 B}.  With FUSED (GroupNorm-apply + SiLU of the 3x3 input, see below) all 128
//                 threads build the segment-0 A tiles from the RAW tensor instead.
//   warpgroups 1, 2   wgmma m64nBLOCK_Nk16 on rows [64 wg, 64 wg + 64) of the tile, then the epilogue straight from
//                 the accumulator registers: +bias +time-embedding bias +residual, *scale -> fp16 -> swizzled smem
//                 staging -> TMA store; per-channel (sum, sum^2) partials for the next GroupNorm are reduced from
//                 the staged tile (deterministic, no atomics).  The producer runs ahead into the next tile's
//                 stages while the epilogue drains.
//
// FUSED: out = conv3x3(silu(a * x + b)) with (a, b) = gn_ab[n][channel] (launch_gn_finalize) over the raw input x
// (seg[0].src, concatenated with gn_cat), so the gn_apply pass and its buffer disappear.  Out-of-image taps read 0
// (the padding of the ACTIVATED tensor, as in F.conv2d after the activation).
//
// Reference semantics: F.conv2d calls of ResnetBlockBigGANpp.forward (layerspp.py:260-269) and NIN
// (layers.py:546-555); the epilogue fuses `h += Dense_0(act(temb))[:, :, None, None]`, the Conv_2
// shortcut add and `(x + h) / sqrt(2)` (layerspp.py:262-274).
#include "kernels.h"

#include <mutex>

namespace sgmse {

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;     // fp16 elements = 128 B = one swizzle row
constexpr int WG_K = 16;
constexpr int NUM_THREADS = 384;
constexpr int NUM_CONS = 256;   // the two MMA/epilogue warpgroups
constexpr int A_TILE_BYTES = BLOCK_M * BLOCK_K * 2;   // 16 KB

struct TcParams {
  int tiles_w, tiles_h, tiles_n;
  int bw, bh, bn;
  int n_tiles_n, num_m_tiles, num_tiles;
  int N, H, W, Cout;
  int nseg;
  int seg_chunks[3];
  int seg_taps[3];
  int num_k_blocks;
  const float* bias;
  const float* temb;
  int temb_stride;
  int has_residual;
  float scale;
  float* stats;
  int slots;
  // FUSED producer: raw segment-0 input (c0 channels) [+ concatenated raw input (c1 channels)], coefficients [N][c0+c1]
  const __half* raw0;
  const __half* raw1;
  int c0, c1;
  const float2* gn_ab;
  int* dbg;
};

template <int BLOCK_N, int NUM_STAGES>
struct SmemLayout {
  static constexpr int B_TILE_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_TILE_BYTES + B_TILE_BYTES;
  static constexpr int N_CHUNKS = BLOCK_N / 64;
  static constexpr int STAGING_BYTES = N_CHUNKS * A_TILE_BYTES;
  static constexpr int OFF_STAGING = NUM_STAGES * STAGE_BYTES;
  static constexpr int OFF_STATS = OFF_STAGING + STAGING_BYTES;         // float [4][BLOCK_N][2]
  static constexpr int OFF_BARS = OFF_STATS + 4 * BLOCK_N * 2 * 4;
  static constexpr int NUM_BARS = 2 * NUM_STAGES + 1;
  static constexpr int TOTAL = OFF_BARS + NUM_BARS * 8;
  static constexpr int DYN_BYTES = TOTAL + 1024;                        // slack for 1024 B alignment
};

// wgmma shared-memory matrix descriptor: K-major, SWIZZLE_128B canonical layout (8-row x 128 B atoms, 1024 B apart)
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);      // start address
  d |= (uint64_t)1 << 16;                          // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;                // stride byte offset
  d |= (uint64_t)1 << 62;                          // SWIZZLE_128B
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D (+)= A[smem desc] * B[smem desc]^T, fp16 inputs (both K-major), fp32 accumulators in registers
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(accumulate));
}
template <int BLOCK_N>
__device__ __forceinline__ void wgmma_tile(float (&d)[BLOCK_N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (BLOCK_N == 128) wgmma_m64n128k16(d, da, db, accumulate);
  else wgmma_m64n64k16(d, da, db, accumulate);
}

// FUSED producer, one thread per pixel row r of the box: silu(a*x+b) of 64 raw channels at the tap-shifted pixel,
// written as row r of a SWIZZLE_128B K-major tile (16-byte unit u lands at unit u ^ (r & 7), as TMA would put it)
__device__ __forceinline__ void fused_a_row(uint8_t* tile, int r, const TcParams& P, int x0, int y0, int n0, int dx, int dy,
                                            int chunk) {
  const int px = r % P.bw, py = (r / P.bw) % P.bh, pn = r / (P.bw * P.bh);
  const int x = x0 + px + dx, y = y0 + py + dy, n = n0 + pn;
  uint4* row = reinterpret_cast<uint4*>(tile + r * 128);
  const bool in = x >= 0 && x < P.W && y >= 0 && y < P.H && n < P.N;
  const int cbase = chunk * BLOCK_K;
  const bool cat = cbase >= P.c0;
  const __half* src = nullptr;
  if (in) {
    const size_t pix = ((size_t)n * P.H + y) * P.W + x;
    src = cat ? P.raw1 + pix * P.c1 + (cbase - P.c0) : P.raw0 + pix * P.c0 + cbase;
  }
  const float2* ab = P.gn_ab + (size_t)(in ? n : 0) * (P.c0 + P.c1) + cbase;
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    uint4 v = make_uint4(0, 0, 0, 0);
    if (in) {
      const uint4 raw = __ldg(reinterpret_cast<const uint4*>(src) + u);
      const __half2* h = reinterpret_cast<const __half2*>(&raw);
      __half2* o = reinterpret_cast<__half2*>(&v);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = __half22float2(h[i]);
        const float2 c0 = __ldg(ab + u * 8 + 2 * i), c1 = __ldg(ab + u * 8 + 2 * i + 1);
        o[i] = __floats2half2_rn(silu_f(c0.x * f.x + c0.y), silu_f(c1.x * f.y + c1.y));
      }
    }
    row[u ^ (r & 7)] = v;
  }
}

template <int BLOCK_N, int NUM_STAGES, bool FUSED>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap map_a0, const __grid_constant__ CUtensorMap map_a1,
               const __grid_constant__ CUtensorMap map_a2, const __grid_constant__ CUtensorMap map_b,
               const __grid_constant__ CUtensorMap map_d, const __grid_constant__ CUtensorMap map_r,
               const TcParams P) {
  using L = SmemLayout<BLOCK_N, NUM_STAGES>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::OFF_BARS);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + NUM_STAGES;
  uint64_t* res_full = bars + 2 * NUM_STAGES;
  uint8_t* staging = smem + L::OFF_STAGING;
  float* stats_sm = reinterpret_cast<float*>(smem + L::OFF_STATS);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_trigger();

  // full: the TMA transaction arrival (+ the 128 producer threads' arrivals when FUSED); empty: one arrival per consumer warp
  constexpr uint32_t FULL_COUNT = FUSED ? 1 + 128 : 1;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a0);
    tma_prefetch_desc(&map_b);
    tma_prefetch_desc(&map_d);
    if (P.nseg > 1) tma_prefetch_desc(&map_a1);
    if (P.nseg > 2) tma_prefetch_desc(&map_a2);
    if (P.has_residual) tma_prefetch_desc(&map_r);
    for (int i = 0; i < NUM_STAGES; ++i) { mbar_init(&full_bar[i], FULL_COUNT); mbar_init(&empty_bar[i], NUM_CONS / 32); }
    mbar_init(res_full, 1);
    mbar_fence_init();
  }
  __syncthreads();
  pdl_wait();                    // everything above is on-chip set-up; global memory is first touched below

  if (warp < 4) {
    // =========================== producer (warpgroup 0) ===========================
    const int pt = threadIdx.x;                 // 0..127
    if (!FUSED && pt != 0) return;
    int stage = 0; uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < P.num_tiles; tile += gridDim.x) {
      const int m_tile = tile % P.num_m_tiles, n_tile = tile / P.num_m_tiles;
      const int tx = m_tile % P.tiles_w, ty = (m_tile / P.tiles_w) % P.tiles_h, tn = m_tile / (P.tiles_w * P.tiles_h);
      const int x0 = tx * P.bw, y0 = ty * P.bh, n0 = tn * P.bn;
      int kb = 0;
      for (int s = 0; s < P.nseg; ++s) {
        const CUtensorMap* ma = s == 0 ? &map_a0 : (s == 1 ? &map_a1 : &map_a2);
        const int taps = P.seg_taps[s];
        for (int tap = 0; tap < taps; ++tap) {
          const int dy = taps == 9 ? tap / 3 - 1 : 0, dx = taps == 9 ? tap % 3 - 1 : 0;
          for (int ch = 0; ch < P.seg_chunks[s]; ++ch, ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1, P.dbg, 100 + stage);
            uint8_t* sa = smem + stage * L::STAGE_BYTES;
            const bool build_a = FUSED && s == 0;
            if (pt == 0) {
              mbar_arrive_expect_tx(&full_bar[stage], build_a ? L::B_TILE_BYTES : L::STAGE_BYTES);
              if (!build_a) tma_load_4d(sa, ma, &full_bar[stage], ch * BLOCK_K, x0 + dx, y0 + dy, n0);
              tma_load_2d(sa + A_TILE_BYTES, &map_b, &full_bar[stage], kb * BLOCK_K, n_tile * BLOCK_N);
            }
            if (FUSED) {
              if (build_a) {
                fused_a_row(sa, pt, P, x0, y0, n0, dx, dy, ch);
                fence_proxy_async_smem();          // generic-proxy smem writes -> visible to wgmma (async proxy)
              }
              mbar_arrive(&full_bar[stage]);
            }
            if (++stage == NUM_STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // =========================== MMA + epilogue (warpgroups 1, 2) ===========================
  const int ct = threadIdx.x - 128;            // 0..255
  const int wg = ct >> 7;                      // rows [64 wg, 64 wg + 64) of the tile
  const int wt = ct & 127;
  const int rps = P.bw * P.bh;                 // rows per sample inside a tile
  int stage = 0; uint32_t phase = 0; uint32_t res_phase = 0;
  float acc[BLOCK_N / 2];
  for (int tile = blockIdx.x; tile < P.num_tiles; tile += gridDim.x) {
    const int m_tile = tile % P.num_m_tiles, n_tile = tile / P.num_m_tiles;
    const int tx = m_tile % P.tiles_w, ty = (m_tile / P.tiles_w) % P.tiles_h, tn = m_tile / (P.tiles_w * P.tiles_h);
    const int x0 = tx * P.bw, y0 = ty * P.bh, n0 = tn * P.bn;
    const int c_tile = n_tile * BLOCK_N;

    // staging buffer must be free: the previous tile's TMA store has finished reading it, every thread is done with it
    if (ct == 0) tma_store_wait_read0();
    named_bar_sync(1, NUM_CONS);
    if (P.has_residual && ct == 0) {           // the residual tile lands in the staging buffer while the MMAs run
      fence_proxy_async_smem();
      mbar_arrive_expect_tx(res_full, L::STAGING_BYTES);
#pragma unroll
      for (int c = 0; c < L::N_CHUNKS; ++c)
        tma_load_4d(staging + c * A_TILE_BYTES, &map_r, res_full, c_tile + c * 64, x0, y0, n0);
    }

    int prev = -1;
    for (int kb = 0; kb < P.num_k_blocks; ++kb) {
      mbar_wait(&full_bar[stage], phase, P.dbg, 300 + stage);
      const uint32_t a_addr = smem_u32(smem + stage * L::STAGE_BYTES);
      const uint64_t adesc = make_smem_desc(a_addr + wg * 64 * 128);
      const uint64_t bdesc = make_smem_desc(a_addr + A_TILE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / WG_K; ++k)
        // advance 16 fp16 = 32 B along K inside the 128 B swizzle row: +2 in the (addr >> 4) field
        wgmma_tile<BLOCK_N>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (kb | k) != 0);
      wgmma_commit();
      wgmma_wait<1>();                         // the previous k-block's MMAs have retired: its stage is free
      if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
      prev = stage;
      if (++stage == NUM_STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[prev]);

    if (P.has_residual) {
      mbar_wait(res_full, res_phase, P.dbg, 400);
      res_phase ^= 1;
    }
    // accumulator fragment of m64nN: thread wt holds rows 16 (wt / 32) + (lane / 4) + {0, 8}, columns 8 j + 2 (lane % 4) + {0, 1}
    const float* bias_row = P.bias ? P.bias + c_tile : nullptr;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = wg * 64 + (wt >> 5) * 16 + (lane >> 2) + 8 * h;
      int n_s = n0 + row / rps;
      if (n_s >= P.N) n_s = P.N - 1;            // rows of a partially out-of-range box (never stored)
      const float* temb_row = P.temb ? P.temb + (size_t)n_s * P.temb_stride + c_tile : nullptr;
      uint8_t* my_row = staging + row * 128 + (lane & 3) * 4;
      const int sw = row & 7;
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int cb = j * 8 + (lane & 3) * 2;   // channel inside the tile
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (bias_row) { v0 += __ldg(bias_row + cb); v1 += __ldg(bias_row + cb + 1); }
        if (temb_row) { v0 += __ldg(temb_row + cb); v1 += __ldg(temb_row + cb + 1); }
        __half2* sp = reinterpret_cast<__half2*>(my_row + (j >> 3) * A_TILE_BYTES + (((j & 7) ^ sw) << 4));
        if (P.has_residual) {
          const float2 f = __half22float2(*sp);
          v0 += f.x; v1 += f.y;
        }
        *sp = __floats2half2_rn(v0 * P.scale, v1 * P.scale);
      }
    }

    fence_proxy_async_smem();
    named_bar_sync(1, NUM_CONS);
    if (ct == 0) {
#pragma unroll
      for (int c = 0; c < L::N_CHUNKS; ++c)
        tma_store_4d(&map_d, staging + c * A_TILE_BYTES, c_tile + c * 64, x0, y0, n0);
      tma_store_commit();
    }

    if (P.stats) {
      // per-channel (sum, sum^2) over each 32-row segment, from the fp16 values actually stored
      if (ct < 128) {
        const int seg = ct >> 5;
#pragma unroll
        for (int c = 0; c < L::N_CHUNKS; ++c) {
          float s0 = 0.f, q0 = 0.f, s1 = 0.f, q1 = 0.f;
          const uint8_t* cbase = staging + c * A_TILE_BYTES;
#pragma unroll 8
          for (int rr = 0; rr < 32; ++rr) {
            const int r2 = seg * 32 + rr;
            const __half2 hv = *reinterpret_cast<const __half2*>(cbase + r2 * 128 + ((((lane >> 2) ^ (r2 & 7)) << 4) | ((lane & 3) << 2)));
            const float2 f = __half22float2(hv);
            s0 += f.x; q0 += f.x * f.x; s1 += f.y; q1 += f.y * f.y;
          }
          float* d = stats_sm + ((seg * BLOCK_N) + c * 64 + lane * 2) * 2;
          d[0] = s0; d[1] = q0; d[2] = s1; d[3] = q1;
        }
      }
      named_bar_sync(1, NUM_CONS);
      const int groups = rps >= 128 ? 1 : 128 / rps;       // samples covered by this tile
      const int spg = 4 / groups;                          // 32-row segments per sample
      const int slot = ty * P.tiles_w + tx;
      for (int c = ct; c < BLOCK_N; c += NUM_CONS) {
        for (int g = 0; g < groups; ++g) {
          const int n = n0 + g;
          if (n >= P.N) break;
          float s = 0.f, q = 0.f;
          for (int j = 0; j < spg; ++j) {
            s += stats_sm[(((g * spg + j) * BLOCK_N) + c) * 2];
            q += stats_sm[(((g * spg + j) * BLOCK_N) + c) * 2 + 1];
          }
          float* d = P.stats + (((size_t)n * P.slots + slot) * P.Cout + c_tile + c) * 2;
          d[0] = s; d[1] = q;
        }
      }
    }
  }
  if (ct == 0) tma_store_wait_all0();
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  SG_CHECK(fn != nullptr, "cuTensorMapEncodeTiled not available from the driver");
  return fn;
}

// NHWC fp16 tensor, box {64 channels, bw, bh, bn}
CUtensorMap make_act_map(const void* p, int N, int H, int W, int C, int bw, int bh, int bn) {
  CUtensorMap m;
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bn};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = get_encode()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(p), dims, strides, box, es,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SG_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(activation %dx%dx%dx%d box %dx%dx%d) failed: %d", N, H, W, C, bw, bh, bn, (int)r);
  return m;
}
// weights [Cout][Ktot] fp16, box {64, block_n}
CUtensorMap make_w_map(const void* p, int Cout, int Ktot, int block_n) {
  CUtensorMap m;
  cuuint64_t dims[2] = {(cuuint64_t)Ktot, (cuuint64_t)Cout};
  cuuint64_t strides[1] = {(cuuint64_t)Ktot * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)block_n};
  cuuint32_t es[2] = {1, 1};
  CUresult r = get_encode()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(p), dims, strides, box, es,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SG_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(weights %dx%d) failed: %d", Cout, Ktot, (int)r);
  return m;
}

// Pixel box (bw, bh, bn) with bw*bh*bn = 128, bw | W, bh | H, bn in {1,2,4}: prefer a single sample
// and a square-ish box (smallest halo when neighbouring tiles share L2 lines).
bool choose_box(int H, int W, int& bw, int& bh, int& bn) {
  int best = -1000000;
  bool found = false;
  for (int w = 1; w <= 128; w *= 2)
    for (int h = 1; w * h <= 128; h *= 2) {
      if (w * h < 32 || W % w || H % h) continue;
      const int n = 128 / (w * h);
      const int score = -n * 100 - (w > h ? w / h : h / w);
      if (score > best) { best = score; bw = w; bh = h; bn = n; found = true; }
    }
  return found;
}

int num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    CUDA_OK(cudaGetDevice(&dev));
    CUDA_OK(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  }
  return n;
}

namespace {

template <int BLOCK_N, int NUM_STAGES, bool FUSED>
void launch_impl(cudaStream_t st, const ConvArgs& a, TensorDesc& out, int* dbg) {
  using L = SmemLayout<BLOCK_N, NUM_STAGES>;
  int bw, bh, bn;
  SG_CHECK(choose_box(out.H, out.W, bw, bh, bn), "conv_tc: no 128-pixel box for %dx%d", out.H, out.W);
  TcParams P{};
  P.bw = bw; P.bh = bh; P.bn = bn;
  P.tiles_w = out.W / bw; P.tiles_h = out.H / bh; P.tiles_n = cdiv(out.N, bn);
  P.n_tiles_n = out.C / BLOCK_N;
  P.num_m_tiles = P.tiles_w * P.tiles_h * P.tiles_n;
  P.num_tiles = P.num_m_tiles * P.n_tiles_n;
  P.N = out.N; P.H = out.H; P.W = out.W; P.Cout = out.C;
  P.nseg = a.nseg;
  CUtensorMap ma[3];
  int kblocks = 0;
  for (int i = 0; i < 3; ++i) {
    const TensorDesc& s = a.seg[i < a.nseg ? i : 0].src;
    ma[i] = make_act_map(s.p, s.N, s.H, s.W, s.C, bw, bh, bn);
    if (i < a.nseg) {
      const int cin = s.C + (i == 0 && FUSED && a.gn_has_cat ? a.gn_cat.C : 0);
      P.seg_chunks[i] = cin / 64; P.seg_taps[i] = a.seg[i].taps;
      kblocks += a.seg[i].taps * (cin / 64);
    }
  }
  P.num_k_blocks = kblocks;
  if (FUSED) {
    P.raw0 = static_cast<const __half*>(a.seg[0].src.p); P.c0 = a.seg[0].src.C;
    P.raw1 = a.gn_has_cat ? static_cast<const __half*>(a.gn_cat.p) : nullptr; P.c1 = a.gn_has_cat ? a.gn_cat.C : 0;
    P.gn_ab = a.gn_ab;
  }
  const CUtensorMap mb = make_w_map(a.w_tc, out.C, a.w_tc_ld ? a.w_tc_ld : a.ktot(), BLOCK_N);
  const CUtensorMap md = make_act_map(out.p, out.N, out.H, out.W, out.C, bw, bh, bn);
  const TensorDesc& rs = a.residual ? *a.residual : out;
  const CUtensorMap mr = make_act_map(rs.p, rs.N, rs.H, rs.W, rs.C, bw, bh, bn);
  P.bias = a.bias; P.temb = a.temb; P.temb_stride = a.temb_stride;
  P.has_residual = a.residual ? 1 : 0;
  P.scale = a.scale;
  out.slots = P.tiles_w * P.tiles_h;
  P.stats = out.stats; P.slots = out.slots;
  P.dbg = dbg;
  auto kern = conv_tc_kernel<BLOCK_N, NUM_STAGES, FUSED>;
  static unsigned long long attr_devs = 0;
  if (first_use_on_device(attr_devs)) {
    CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::DYN_BYTES));
  }
  const int grid = P.num_tiles < num_sms() ? P.num_tiles : num_sms();
  launch_k(kern, dim3(grid), dim3(NUM_THREADS), (size_t)L::DYN_BYTES, st, ma[0], ma[1], ma[2], mb, md, mr, P);
  CUDA_OK(cudaGetLastError());
}

template <bool FUSED>
void launch_width(cudaStream_t st, const ConvArgs& a, TensorDesc& out, int* dbg) {
  // tc1_narrow: when 128-wide channel tiles would fill less than half the SMs, 64-wide tiles double the CTAs.  The
  // accumulation order of an output element does not depend on the tile width: bit-identical.
  if (out.C % 128 == 0 && g_tc1_narrow) {
    int bw, bh, bn;
    choose_box(out.H, out.W, bw, bh, bn);
    const int tiles128 = (out.W / bw) * (out.H / bh) * cdiv(out.N, bn) * (out.C / 128);
    if (tiles128 * 2 <= num_sms()) { launch_impl<64, 6, FUSED>(st, a, out, dbg); return; }
  }
  if (out.C % 128 == 0) launch_impl<128, 5, FUSED>(st, a, out, dbg);
  else launch_impl<64, 6, FUSED>(st, a, out, dbg);
}

}  // namespace

thread_local int g_tc_variant = 0;   // see kernels.h
thread_local int g_tc1_narrow = 0;   // see launch_width
volatile int* g_wait_code_host = nullptr;

bool conv_tc_supported(const ConvArgs& a, const TensorDesc& out) {
  if (out.dt != DT_F16 || out.C % 64 != 0 || a.w_tc == nullptr) return false;
  for (int i = 0; i < a.nseg; ++i)
    if (a.seg[i].src.C % 64 != 0 || a.seg[i].src.dt != DT_F16) return false;
  int bw, bh, bn;
  return choose_box(out.H, out.W, bw, bh, bn);
}

// Shape test usable before the tensors exist (fused GroupNorm 3x3 over c0 [+ c1] raw channels).
bool conv_tc_fuse_shape_ok(int H, int W, int c0, int c1, int cout) {
  int bw, bh, bn;
  return c0 % 64 == 0 && c1 % 64 == 0 && cout % 64 == 0 && choose_box(H, W, bw, bh, bn);
}

void launch_conv_tc(cudaStream_t st, const ConvArgs& a, TensorDesc& out, int* dbg) {
  SG_CHECK(conv_tc_supported(a, out), "conv_tc: unsupported shape (Cout=%d)", out.C);
  for (int i = 0; i < a.nseg; ++i) {
    const TensorDesc& s = a.seg[i].src;
    SG_CHECK(s.N == out.N && s.H == out.H && s.W == out.W, "conv_tc: segment %d shape mismatch", i);
  }
  if (a.residual) SG_CHECK(a.residual->C == out.C && a.residual->dt == DT_F16, "conv_tc: residual mismatch");
  if (a.gn_ab) {                                                      // the engine only asks for fusion when it applies
    SG_CHECK(a.seg[0].taps == 9 && conv_tc_fuse_shape_ok(out.H, out.W, a.seg[0].src.C, a.gn_has_cat ? a.gn_cat.C : 0, out.C) &&
                 (!a.gn_has_cat || (a.gn_cat.dt == DT_F16 && a.gn_cat.N == out.N && a.gn_cat.H == out.H && a.gn_cat.W == out.W)),
             "conv_tc: unsupported fused shape");
    launch_width<true>(st, a, out, dbg);
    return;
  }
  launch_width<false>(st, a, out, dbg);
}

}  // namespace sgmse
