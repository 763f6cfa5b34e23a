/* Plain-C client of include/sgmse_b200.h: proves that the boundary is a C ABI (this file is compiled with gcc -std=c99,
 * no C++ and no Python in the process) and exercises the host-only entry points, which work without a GPU.
 * Built and run by tests/test_cabi_host.py::test_plain_c_client. */
#include <math.h>
#include <stdio.h>
#include <string.h>

#include "sgmse_b200.h"

#define CHECK(cond, msg)                                                        \
  do {                                                                          \
    if (!(cond)) { fprintf(stderr, "FAIL %s:%d %s (%s)\n", __FILE__, __LINE__, msg, sgmse_b200_last_error()); return 1; } \
  } while (0)

/* dy/dt = -k y (complex scalar per unknown): y(t) = y0 exp(-k (t - t0)) */
static int g_calls = 0;
static void decay(double t, const double* y, double* dydt, long long n, void* user) {
  const double k = *(const double*)user;
  long long i;
  (void)t;
  for (i = 0; i < 2 * n; ++i) dydt[i] = -k * y[i];
  ++g_calls;
}

int main(void) {
  sgmse_b200_config cfg;
  sgmse_b200_engine* e = NULL;
  sgmse_b200_sampler s;
  float ts[30], coef[60 * 3], prior_std = 0.f;
  int n_updates = 0, i, nfev = 0, stats[4];
  long long numel = 0, total = 0;
  char name[128];
  double y[4] = {1.0, 0.5, -2.0, 0.25}, k = 3.0;

  memset(&cfg, 0, sizeof cfg);
  cfg.backbone = SGMSE_B200_BACKBONE_NCSNPP;
  cfg.nf = 128;
  cfg.num_levels = 7;
  { const int m[7] = {1, 1, 2, 2, 2, 2, 2}; for (i = 0; i < 7; ++i) cfg.ch_mult[i] = m[i]; }
  cfg.num_res_blocks = 2;
  cfg.num_attn_resolutions = 1;
  cfg.attn_resolutions[0] = 16;
  cfg.image_size = 256;
  cfg.progressive_output_skip = 1;
  cfg.progressive_input_skip = 1;
  cfg.scale_by_sigma = 1;
  cfg.theta = 1.5f; cfg.sigma_min = 0.05f; cfg.sigma_max = 0.5f; cfg.t_eps = 0.03f;
  cfg.n_fft = 510; cfg.hop_length = 128; cfg.spec_factor = 0.15f; cfg.spec_abs_exponent = 0.5f; cfg.sample_rate = 16000;
  cfg.mode = SGMSE_B200_MODE_FP16_TC; cfg.max_batch = 16; cfg.use_graphs = 1;
  cfg.sde_kind = SGMSE_B200_SDE_OUVE; cfg.sigma_data = 0.1f;

  CHECK(strstr(sgmse_b200_version(), "sm_90a") != NULL, "version string");
  CHECK(sgmse_b200_create(&cfg, &e) == 0 && e != NULL, "create");
  /* the weight manifest is the reference's state_dict() layout: 65.6 M parameters for the 16 kHz NCSN++ */
  CHECK(sgmse_b200_manifest_count(e) > 400, "manifest count");
  for (i = 0; i < sgmse_b200_manifest_count(e); ++i) {
    CHECK(sgmse_b200_manifest_entry(e, i, name, (int)sizeof name, &numel) == 0, "manifest entry");
    total += numel;
  }
  CHECK(total == sgmse_b200_weights_numel(e) && total > 65000000LL && total < 66000000LL, "parameter count");
  CHECK(sgmse_b200_manifest_entry(e, -1, name, (int)sizeof name, &numel) != 0, "out-of-range index must fail");
  CHECK(strlen(sgmse_b200_last_error()) > 0, "error message");
  CHECK(sgmse_b200_padded_frames(e, 64000) == 512, "4-s clip -> 501 frames -> 512");
  CHECK(sgmse_b200_workspace_bytes(e, 1, 256, 512) > (1LL << 30), "workspace of one utterance");

  memset(&s, 0, sizeof s);
  s.N = 30; s.predictor = SGMSE_B200_PRED_REVERSE_DIFFUSION; s.corrector = SGMSE_B200_CORR_ALD; s.corrector_steps = 1;
  s.snr = 0.5f; s.denoise = 1; s.kind = SGMSE_B200_SAMPLER_PC;
  CHECK(sgmse_b200_noise_draws(&s) == 61, "1 prior + 2 draws per step");
  CHECK(sgmse_b200_sampler_schedule(e, &s, ts, &prior_std, coef, 60, &n_updates) == 0, "schedule");
  CHECK(n_updates == 60 && fabs(prior_std - 0.38898) < 1e-4 && ts[0] == 1.0f && fabs(ts[29] - 0.03) < 1e-6, "SURVEY 8a scalars");
  CHECK(fabs(coef[1] - 7.565e-2) < 1e-4 && fabs(coef[3 * 1 + 2] - 0.19624) < 1e-4, "step 0: eps of ald, G of the predictor");

  /* the ODE sampler's RK45 controller on a C right-hand side */
  CHECK(sgmse_b200_rk45_host(decay, &k, 1.0, 0.03, y, 2, 1e-8, 1e-10, 0, &nfev, stats) == 0, "rk45");
  CHECK(stats[2] == 0 && nfev == g_calls && nfev == 2 + 6 * (stats[0] + stats[1]), "nfev bookkeeping");
  CHECK(fabs(y[0] - exp(-k * (0.03 - 1.0))) < 1e-5 * exp(-k * (0.03 - 1.0)), "solution of dy/dt = -k y");
  CHECK(sgmse_b200_rk45_host(NULL, NULL, 0, 1, y, 2, 1e-3, 1e-6, 0, &nfev, stats) != 0, "null callback must fail");

  sgmse_b200_destroy(e);
  printf("cabi_host ok: %lld parameters, %d updates, rk45 nfev %d\n", total, n_updates, nfev);
  return 0;
}
