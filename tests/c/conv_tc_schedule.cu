// Host replay of conv_tc_kernel's ring schedule (sgmse_b200/csrc/conv_tc_sched.h): the same loops as the kernel's
// producer and consumer warpgroups, printing what each role would wait on.  Reads "num_tiles grid k_blocks stages"
// lines from stdin; for each CTA prints
//   P j kb stage phase          one line per fill, in the producer's order
//   C wg j kb stage phase       one line per k-block a consumer warpgroup reads, in its own order
// and "E" after each case.  tests/test_conv_tc_schedule.py simulates the mbarriers over these sequences.
#include <cstdio>

#include "conv_tc_sched.h"

using namespace sgmse;

int main() {
  int num_tiles, grid, k_blocks, stages;
  while (std::scanf("%d %d %d %d", &num_tiles, &grid, &k_blocks, &stages) == 4) {
    for (int cta = 0; cta < grid; ++cta) {
      std::printf("B %d\n", cta);
      const int n_local = tc_local_tiles(cta, grid, num_tiles);
      for (int j = 0; j < n_local; ++j)
        for (int kb = 0; kb < k_blocks; ++kb) {
          const TcSlot s = tc_slot(j, kb, k_blocks, stages);
          std::printf("P %d %d %d %u\n", j, kb, s.stage, s.phase);
        }
      for (int wg = 0; wg < 2; ++wg)
        for (int j = 0; j < n_local; ++j) {
          if (tc_consumer_of(j) != wg) continue;
          for (int kb = 0; kb < k_blocks; ++kb) {
            const TcSlot s = tc_slot(j, kb, k_blocks, stages);
            std::printf("C %d %d %d %d %u\n", wg, j, kb, s.stage, s.phase);
          }
        }
    }
    std::printf("E\n");
  }
  return 0;
}
