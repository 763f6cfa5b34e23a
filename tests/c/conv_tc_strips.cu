// Host replay of conv_tc_kernel's two operand rings (sgmse_b200/csrc/conv_tc.cu, conv_tc_sched.h): the same loops as
// the kernel's producer and consumer warpgroups, printing what each role fills, waits on and reads.  conv_tc.cu is
// included whole so that the ring depths and the shared-memory layout are the kernel's own; nothing here touches a GPU.
//
// stdin, one request per line:
//   S bw bh bn taps                        -> "R rows": tc_strip_rows
//   P num_tiles grid bw bh bn fused block_n esize nseg taps0 chunks0 taps1 chunks1 taps2 chunks2 stages a_stages
//                                          (ring depths, 0 0: the kernel's) -> for each CTA "B cta", then
//        PA j f stage phase seg chunk dx y rows     an A fill (box at x0 + dx, y0 + y, `rows` 128 B rows)
//        PB j kb stage phase col                    a B fill (packed k-block col), both in the producer's order
//        C wg j kb bstage bphase astage aphase fill dy1 last      one line per k-block a consumer warpgroup reads
//      and "E" after the case
// and first, once: "L block_n stages esize a_stages dyn_bytes" for each kernel instantiation.
#include <cstdio>

#include "conv_tc.cu"

namespace sgmse {
thread_local int g_pdl = 0;   // defined with the engine (common.cuh); the launchers are never called here
}

using namespace sgmse;

namespace {

template <int BLOCK_N, int NUM_STAGES, int ESIZE>
void print_layout() {
  using L = SmemLayout<BLOCK_N, NUM_STAGES, ESIZE>;
  std::printf("L %d %d %d %d %d\n", BLOCK_N, NUM_STAGES, ESIZE, L::A_STAGES, L::DYN_BYTES);
}

struct Case {
  int num_tiles, grid, bw, bh, bn, fused, block_n, esize, nseg, taps[3], chunks[3];
};

void replay(const Case& c, int stages, int a_stages) {
  int k_blocks = 0;
  for (int s = 0; s < c.nseg; ++s) k_blocks += c.taps[s] * c.chunks[s];
  const int rows = c.fused ? 0 : tc_strip_rows(c.bw, c.bh, c.bn, c.taps[0]);
  const int sc = rows ? c.chunks[0] : 0;
  const int a_fills = tc_a_fills(k_blocks, sc);
  for (int cta = 0; cta < c.grid; ++cta) {
    std::printf("B %d\n", cta);
    const int n_local = tc_local_tiles(cta, c.grid, c.num_tiles);
    // producer (conv_tc_kernel, warpgroup 0)
    for (int j = 0; j < n_local; ++j) {
      auto fill_b = [&](int kb, int col) {
        const TcSlot sl = tc_slot(j, kb, k_blocks, stages);
        std::printf("PB %d %d %d %u %d\n", j, kb, sl.stage, sl.phase, col);
      };
      for (int dx = -1; dx <= 1; ++dx)
        for (int ch = 0; ch < sc; ++ch) {
          const int f = (dx + 1) * sc + ch;
          const TcSlot sl = tc_slot(j, f, a_fills, a_stages);
          std::printf("PA %d %d %d %u %d %d %d %d %d\n", j, f, sl.stage, sl.phase, 0, ch, dx, -1, rows);
          for (int dy = -1; dy <= 1; ++dy) fill_b(3 * f + dy + 1, tc_strip_column(dx, dy, ch, sc));
        }
      int kb = 9 * sc;
      for (int s = sc ? 1 : 0; s < c.nseg; ++s) {
        const int taps = c.taps[s];
        for (int tap = 0; tap < taps; ++tap) {
          const int dy = taps == 9 ? tap / 3 - 1 : 0, dx = taps == 9 ? tap % 3 - 1 : 0;
          for (int ch = 0; ch < c.chunks[s]; ++ch, ++kb) {
            const TcSlot sl = tc_slot(j, kb - 6 * sc, a_fills, a_stages);
            std::printf("PA %d %d %d %u %d %d %d %d %d\n", j, kb - 6 * sc, sl.stage, sl.phase, s, ch, dx, dy, 128);
            fill_b(kb, kb);
          }
        }
      }
    }
    // consumers (warpgroups 1, 2)
    for (int wg = 0; wg < 2; ++wg)
      for (int j = 0; j < n_local; ++j) {
        if (tc_consumer_of(j) != wg) continue;
        for (int kb = 0; kb < k_blocks; ++kb) {
          const TcSlot sb = tc_slot(j, kb, k_blocks, stages);
          const TcAUse u = tc_a_use(kb, sc);
          const TcSlot sa = tc_slot(j, u.fill, a_fills, a_stages);
          std::printf("C %d %d %d %d %u %d %u %d %d %d\n", wg, j, kb, sb.stage, sb.phase, sa.stage, sa.phase, u.fill, u.dy1,
                      (int)u.last);
        }
      }
  }
  std::printf("E\n");
}

}  // namespace

int main() {
  print_layout<128, STAGES_N128, 2>();
  print_layout<64, STAGES_N64, 2>();
  print_layout<64, STAGES_TF32, 4>();
  char kind[4];
  while (std::scanf("%3s", kind) == 1) {
    if (kind[0] == 'S') {
      int bw, bh, bn, taps;
      if (std::scanf("%d %d %d %d", &bw, &bh, &bn, &taps) != 4) return 1;
      std::printf("R %d\n", tc_strip_rows(bw, bh, bn, taps));
    } else {
      Case c;
      if (std::scanf("%d %d %d %d %d %d %d %d %d %d %d %d %d %d %d", &c.num_tiles, &c.grid, &c.bw, &c.bh, &c.bn, &c.fused,
                     &c.block_n, &c.esize, &c.nseg, &c.taps[0], &c.chunks[0], &c.taps[1], &c.chunks[1], &c.taps[2],
                     &c.chunks[2]) != 15)
        return 1;
      int stages, a_stages;   // ring depths; 0 0: those of the instantiation launch_width / launch_tf32 pick
      if (std::scanf("%d %d", &stages, &a_stages) != 2) return 1;
      if (stages) replay(c, stages, a_stages);
      else if (c.esize == 4) replay(c, STAGES_TF32, SmemLayout<64, STAGES_TF32, 4>::A_STAGES);
      else if (c.block_n == 128) replay(c, STAGES_N128, SmemLayout<128, STAGES_N128, 2>::A_STAGES);
      else replay(c, STAGES_N64, SmemLayout<64, STAGES_N64, 2>::A_STAGES);
    }
  }
  return 0;
}
