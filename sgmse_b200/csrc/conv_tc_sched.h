// Ring schedule of conv_tc_kernel (conv_tc.cu): which shared-memory stage, and which mbarrier phase, each role uses for
// each (tile, k-block).  Plain host/device code so that tests/test_conv_tc_schedule.py can replay the same sequence
// on the CPU.
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

}  // namespace sgmse
