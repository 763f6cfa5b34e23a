// Ring schedule of conv_tc_kernel (conv_tc.cu): which shared-memory stage, and which mbarrier phase, each role uses for
// each (tile, k-block) of the B ring and each (tile, A fill) of the A ring.  Plain host/device code so that
// tests/test_conv_tc_schedule.py and tests/test_conv_tc_strips_host.py can replay the same sequences on the CPU.
//
// A CTA takes the global tiles blockIdx.x + j * gridDim.x, j = 0, 1, ... (its "local" tiles).  The producer fills the
// ring in that order, k-block after k-block: local tile j, k-block kb is fill number j * k_blocks + kb, which lands in
// stage fill % stages during the ring's round fill / stages.  Consumer warpgroup j & 1 takes local tile j, so each
// consumer skips over the other warpgroup's k-blocks; the MMA turn passes from one warpgroup to the other once per
// tile, which keeps the consumers' waits in the producer's order.
#pragma once

#ifndef __CUDACC__
#define __host__
#define __device__
#endif

namespace sgmse {

struct TcSlot {
  int stage;
  unsigned phase;   // parity of the ring round: full_bar waits on it, empty_bar waits on phase ^ 1
};

// consumer warpgroup (0 or 1) of the CTA's local tile j
__host__ __device__ inline int tc_consumer_of(int j) { return j & 1; }

// ring slot of local tile j, k-block kb (the same for the producer that fills it and the consumer that reads it)
__host__ __device__ inline TcSlot tc_slot(int j, int kb, int k_blocks, int stages) {
  const int fill = j * k_blocks + kb;
  return TcSlot{fill % stages, (unsigned)(fill / stages) & 1u};
}

// number of local tiles of CTA cta in a grid of `grid` CTAs over num_tiles tiles
__host__ __device__ inline int tc_local_tiles(int cta, int grid, int num_tiles) {
  return cta < num_tiles ? (num_tiles - cta + grid - 1) / grid : 0;
}

// ---- dy-halo strips of a 3x3 segment ----
// The A operand (activations) has a ring of its own, apart from the B (weights) ring.  A 3x3 segment over a single-sample
// pixel box bw x bh can take its A tiles from strips: one TMA box of bw x (bh + 2) pixels at (x0 + dx, y0 - 1) per (dx,
// 64-channel chunk).  Tap (dy, dx)'s 128-row tile then starts (dy + 1) * bw rows into the strip, which is a whole number
// of 1024 B SWIZZLE_128B atoms when bw % 8 == 0, so one strip serves three k-blocks.  Anywhere else every k-block has an
// A box of its own at the tap-shifted coordinates.
constexpr int TC_STRIP_MAX_ROWS = 160;   // the A ring's slots hold this many 128 B rows

// rows of segment 0's strips for pixel box (bw, bh, bn) and a segment of `taps` taps; 0: per-tap boxes.  It depends on
// the box alone (that is on H and W), never on the batch or the tile width, so both keep the accumulation order.
__host__ __device__ inline int tc_strip_rows(int bw, int bh, int bn, int taps) {
  const int rows = (bh + 2) * bw;
  return taps == 9 && bn == 1 && bw % 8 == 0 && rows <= TC_STRIP_MAX_ROWS ? rows : 0;
}

// A-ring fills of one tile of k_blocks k-blocks whose 3x3 segment 0 of strip_chunks channel chunks is fed from strips
// (strip_chunks = 0: no strips): 3 per strip chunk, one per other k-block
__host__ __device__ inline int tc_a_fills(int k_blocks, int strip_chunks) { return k_blocks - 6 * strip_chunks; }

// What k-block i (in issue order) of a tile reads from the A ring.  The strip segment is issued dx-major: for dx, for
// chunk, for dy; it reads packed k-block (3 (dy + 1) + (dx + 1)) * strip_chunks + chunk (tc_strip_column).  The k-blocks
// after it are issued in packed order.
struct TcAUse {
  int fill;    // A-ring fill of the tile (tc_slot(j, fill, tc_a_fills(...), a_stages))
  int dy1;     // strip: dy + 1 (the tile starts dy1 * bw rows into the strip); box: 0
  bool last;   // the last k-block that reads this fill: its slot is released once this k-block's MMAs retire
};
__host__ __device__ inline TcAUse tc_a_use(int i, int strip_chunks) {
  if (i < 9 * strip_chunks) return TcAUse{i / 3, i % 3, i % 3 == 2};
  return TcAUse{i - 6 * strip_chunks, 0, true};
}

// packed k-block (B column / 128 B) that strip k-block (dx, chunk, dy) reads
__host__ __device__ inline int tc_strip_column(int dx, int dy, int chunk, int strip_chunks) {
  return (3 * (dy + 1) + (dx + 1)) * strip_chunks + chunk;
}

}  // namespace sgmse
