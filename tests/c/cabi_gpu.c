/* Plain-C client of the PRODUCT path: host waveforms in, enhanced host waveforms out, through sgmse_b200_enhance with
 * host_buffers = 1 -- the client calls no CUDA API itself.  Small NCSN++ (nf 64, 3 levels, F = 64), fp16 wgmma mode,
 * pseudo-random weights, N = 2 predictor-corrector steps.  Checks: finite output, different from the input, bit-identical
 * for the same (seed, utterance id), different for another seed.  Needs a GPU: run by the -m gpu test
 * tests/test_gpu_zz_next_rows.py::test_plain_c_client_on_the_product_path. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "sgmse_b200.h"

#define CHECK(cond, msg)                                                        \
  do {                                                                          \
    if (!(cond)) { fprintf(stderr, "FAIL %s:%d %s (%s)\n", __FILE__, __LINE__, msg, sgmse_b200_last_error()); return 1; } \
  } while (0)

static unsigned long long g_state = 88172645463325252ULL;
static float uniform(void) {                      /* xorshift64*, (-1, 1) */
  g_state ^= g_state >> 12; g_state ^= g_state << 25; g_state ^= g_state >> 27;
  return (float)((double)((g_state * 2685821657736338717ULL) >> 11) / 9007199254740992.0 * 2.0 - 1.0);
}

int main(void) {
  sgmse_b200_config cfg;
  sgmse_b200_engine* e = NULL;
  sgmse_b200_sampler s;
  enum { B = 2, L = 4000 };
  static float wav[B * L], out1[B * L], out2[B * L], out3[B * L];
  float* blob;
  long long total, off = 0, numel = 0, j;
  int i, n;
  char name[160];
  double diff = 0.0, diff_seed = 0.0;

  memset(&cfg, 0, sizeof cfg);
  cfg.backbone = SGMSE_B200_BACKBONE_NCSNPP;
  cfg.nf = 64; cfg.num_levels = 3; cfg.ch_mult[0] = 1; cfg.ch_mult[1] = 2; cfg.ch_mult[2] = 2;
  cfg.num_res_blocks = 1; cfg.num_attn_resolutions = 1; cfg.attn_resolutions[0] = 16; cfg.image_size = 64;
  cfg.progressive_output_skip = 1; cfg.progressive_input_skip = 1; cfg.scale_by_sigma = 1;
  cfg.theta = 1.5f; cfg.sigma_min = 0.05f; cfg.sigma_max = 0.5f; cfg.t_eps = 0.03f;
  cfg.n_fft = 126; cfg.hop_length = 32; cfg.spec_factor = 0.15f; cfg.spec_abs_exponent = 0.5f; cfg.sample_rate = 16000;
  cfg.mode = SGMSE_B200_MODE_FP16_TC; cfg.max_batch = 2; cfg.use_graphs = 1;
  cfg.sde_kind = SGMSE_B200_SDE_OUVE; cfg.sigma_data = 0.1f;
  CHECK(sgmse_b200_create(&cfg, &e) == 0, "create");

  total = sgmse_b200_weights_numel(e);
  blob = (float*)malloc((size_t)total * sizeof(float));
  CHECK(blob != NULL, "malloc");
  n = sgmse_b200_manifest_count(e);
  for (i = 0; i < n; ++i) {
    size_t len;
    int affine_scale;
    CHECK(sgmse_b200_manifest_entry(e, i, name, (int)sizeof name, &numel) == 0, "manifest");
    len = strlen(name);
    /* 1-D '.weight' entries are GroupNorm scales (and the 8-element output layer): around 1; everything else small */
    affine_scale = len > 7 && strcmp(name + len - 7, ".weight") == 0 && numel <= 1024;
    for (j = 0; j < numel; ++j) blob[off + j] = affine_scale ? 1.0f + 0.1f * uniform() : 0.05f * uniform();
    off += numel;
  }
  CHECK(off == total, "manifest covers the blob");
  CHECK(sgmse_b200_load_weights(e, blob, total) == 0, "load_weights");
  free(blob);

  for (i = 0; i < B * L; ++i) wav[i] = 0.1f * uniform();
  memset(&s, 0, sizeof s);
  s.N = 2; s.predictor = SGMSE_B200_PRED_REVERSE_DIFFUSION; s.corrector = SGMSE_B200_CORR_ALD; s.corrector_steps = 1;
  s.snr = 0.5f; s.denoise = 1; s.kind = SGMSE_B200_SAMPLER_PC; s.pad_mode = SGMSE_B200_PAD_ZERO;
  s.seed = 1234; s.utt_offset = 0;
  CHECK(sgmse_b200_enhance(e, wav, B, L, &s, NULL, out1, 1, NULL) == 0, "enhance #1");
  CHECK(sgmse_b200_enhance(e, wav, B, L, &s, NULL, out2, 1, NULL) == 0, "enhance #2 (graph replay)");
  s.seed = 99;
  CHECK(sgmse_b200_enhance(e, wav, B, L, &s, NULL, out3, 1, NULL) == 0, "enhance #3 (other seed)");
  for (i = 0; i < B * L; ++i) {
    CHECK(isfinite(out1[i]), "finite output");
    diff += fabs((double)out1[i] - (double)wav[i]);
    diff_seed += fabs((double)out1[i] - (double)out3[i]);
  }
  CHECK(memcmp(out1, out2, sizeof out1) == 0, "same (seed, utterance id) -> bit-identical");
  CHECK(diff > 0.0 && diff_seed > 0.0, "the sampler did something, the seed matters");
  CHECK(sgmse_b200_get_counter(e, "tc_convs_last_forward") > 0, "wgmma convolutions ran");
  CHECK(sgmse_b200_get_counter(e, "graph_launches") >= 2, "CUDA graph replay");
  printf("cabi_gpu ok: %lld parameters, mean |out - in| %.4f, kernels launched %lld\n", total, diff / (B * L),
         sgmse_b200_get_counter(e, "kernel_launches"));
  sgmse_b200_destroy(e);
  return 0;
}
