/* sgmse_b200 — C-ABI of the H100-native reverse-SDE enhancement engine.
 *
 * Drop-in boundary for the hot path of sp-uhh/sgmse (SURVEY.md §8b).  Plain C: opaque handle, raw
 * device/host pointers and sizes, int return codes (0 = ok, non-zero = error; the message is available
 * from sgmse_b200_last_error()).  Nothing here throws and no torch type crosses the boundary; the Python
 * shim (sgmse_b200/_lib.py) binds these with ctypes and forwards `tensor.data_ptr()` and the current
 * CUDA stream.
 *
 * The only native/FFI boundary the reference itself has is the pybind11 module `upfirdn2d`
 * (/root/reference/sgmse/backbones/ncsnpp_utils/op/upfirdn2d.cpp:12-23, upfirdn2d_kernel.cu:209-369); the
 * engine replaces that op together with the Python call stack above it:
 *
 *   entry point                      replaces (reference file:line)
 *   ------------------------------   ---------------------------------------------------------------
 *   sgmse_b200_dnn_forward           NCSNpp.forward / NCSNpp_48k.forward   sgmse/backbones/ncsnpp.py:256-419,
 *                                    ncsnpp_48k.py:259-424 (incl. upfirdn2d, op/upfirdn2d.py:148-159)
 *   sgmse_b200_score                 ScoreModel.forward (legacy branch)    sgmse/model.py:307-310
 *   sgmse_b200_model_forward         ScoreModel.forward, all branches      sgmse/model.py:261-341 (preconditioned
 *                                    'ncsnpp_v2' branch :283-304 incl. _c_in/_c_out/_c_skip)
 *   sgmse_b200_pc_sample             sampling.get_pc_sampler()/pc_sampler  sgmse/sampling/__init__.py:26-70,
 *                                    predictors.py:41-76, correctors.py:37-94, sdes.py:72-137,188-229,
 *                                    ScoreModel.get_pc_sampler (minibatch loop) sgmse/model.py:348-368;
 *                                    with sampler.kind = SB_ODE / SB_SDE: sampling.get_sb_sampler()
 *                                    sgmse/sampling/__init__.py:145-249, SBVESDE sdes.py:235-312,
 *                                    ScoreModel.get_sb_sampler model.py:392-397
 *   sgmse_b200_ode_sample            sampling.get_ode_sampler()/ode_sampler sgmse/sampling/__init__.py:72-143 (probability-flow
 *                                    ODE, RSDE.sde sdes.py:113-127; the scipy RK45 loop with its per-evaluation host numpy
 *                                    round trips :117-141), ScoreModel.get_ode_sampler model.py:370-390
 *   sgmse_b200_rk45_host             scipy.integrate.solve_ivp(method='RK45') as called at sampling/__init__.py:127-130
 *                                    (the controller sgmse_b200_ode_sample runs, on a host callback; test hook)
 *   sgmse_b200_analysis              _stft + _forward_transform + pad_spec sgmse/data_module.py:162-175,212-214,
 *                                    sgmse/util/other.py:76-90, model.py:435-438
 *   sgmse_b200_synthesis             to_audio (spec_back + istft) + renorm sgmse/data_module.py:177-188,216-218,
 *                                    model.py:411-412,457-458
 *   sgmse_b200_enhance               ScoreModel.enhance                    sgmse/model.py:426-465
 *                                    (= enhancement.py:75-96 per file)
 *   sgmse_b200_enhance_ode           ScoreModel.enhance, sde.sampler_type == 'ode'   sgmse/model.py:446-447
 *   sgmse_b200_load_weights          model.dnn.state_dict() after eval()   sgmse/model.py:111-125 (EMA swap)
 *
 * Threading: one engine per (device, caller); an engine is not thread-safe.  All work is enqueued on the
 * `stream` argument (a cudaStream_t passed as void*; NULL = legacy default stream).
 * Ownership: the caller owns every buffer it passes; the engine owns weights, workspace, cuFFT plans and
 * CUDA graph executables.
 */
#ifndef SGMSE_B200_H
#define SGMSE_B200_H

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sgmse_b200_engine sgmse_b200_engine;

enum { SGMSE_B200_BACKBONE_NCSNPP = 0, SGMSE_B200_BACKBONE_NCSNPP_48K = 1, SGMSE_B200_BACKBONE_NCSNPP_V2 = 2 };
/* arithmetic mode: 0 = fp32 activations, CUDA-core convolutions (validation);
 *                  1 = fp16 activations, CUDA-core convolutions (debug);
 *                  2 = fp16 activations, wgmma tensor-core convolutions (product path) */
enum { SGMSE_B200_MODE_FP32 = 0, SGMSE_B200_MODE_FP16_DIRECT = 1, SGMSE_B200_MODE_FP16_TC = 2 };
enum { SGMSE_B200_PRED_REVERSE_DIFFUSION = 0, SGMSE_B200_PRED_EULER_MARUYAMA = 1, SGMSE_B200_PRED_NONE = 2 };
enum { SGMSE_B200_CORR_ALD = 0, SGMSE_B200_CORR_LANGEVIN = 1, SGMSE_B200_CORR_NONE = 2 };
enum { SGMSE_B200_PAD_ZERO = 0, SGMSE_B200_PAD_REFLECTION = 1 };
/* SDE (sdes.py:144 'ouve', :235 'sbve') and the preconditioning of ScoreModel.forward for backbone 'ncsnpp_v2'
 * (model.py:283-341) */
enum { SGMSE_B200_SDE_OUVE = 0, SGMSE_B200_SDE_SBVE = 1 };
enum { SGMSE_B200_LOSS_SCORE_MATCHING = 0, SGMSE_B200_LOSS_DENOISER = 1, SGMSE_B200_LOSS_DATA_PREDICTION = 2 };
enum { SGMSE_B200_NETSCALE_NONE = 0, SGMSE_B200_NETSCALE_INV_SIGMA = 1, SGMSE_B200_NETSCALE_INV_T = 2 };
enum { SGMSE_B200_CIN_ONE = 0, SGMSE_B200_CIN_EDM = 1 };
enum { SGMSE_B200_COUT_ONE = 0, SGMSE_B200_COUT_SIGMA = 1, SGMSE_B200_COUT_INV_SIGMA = 2, SGMSE_B200_COUT_EDM = 3 };
enum { SGMSE_B200_CSKIP_ZERO = 0, SGMSE_B200_CSKIP_EDM = 1 };
/* sampler kind: predictor-corrector (sampling/__init__.py:26-70) or the Schroedinger-bridge samplers (:145-249) */
enum { SGMSE_B200_SAMPLER_PC = 0, SGMSE_B200_SAMPLER_SB_ODE = 1, SGMSE_B200_SAMPLER_SB_SDE = 2 };

typedef struct sgmse_b200_config {
  /* backbone (kwargs of NCSNpp.__init__, ncsnpp.py:50-74) */
  int backbone;
  int nf;
  int num_levels;            /* len(ch_mult) */
  int ch_mult[8];
  int num_res_blocks;
  int num_attn_resolutions;
  int attn_resolutions[8];
  int image_size;            /* 256 */
  int progressive_output_skip;   /* progressive == 'output_skip' (else 'none') */
  int progressive_input_skip;    /* progressive_input == 'input_skip' (else 'none') */
  int scale_by_sigma;
  /* OUVESDE (sdes.py:148-166) + ScoreModel.t_eps (model.py:29) */
  float theta, sigma_min, sigma_max, t_eps;
  /* SpecsDataModule (data_module.py:121-147) */
  int n_fft, hop_length, sqrt_window;
  float spec_factor, spec_abs_exponent;
  int sample_rate;
  /* engine */
  int mode;                  /* SGMSE_B200_MODE_* */
  int max_batch;             /* utterances processed together (micro-batch); larger batches are looped */
  int use_graphs;            /* capture the N-step sampler loop as one CUDA graph */
  /* SDE kind + SBVESDE parameters (sdes.py:246-263) */
  int sde_kind;              /* SGMSE_B200_SDE_* */
  float sb_k, sb_c, sb_eps;  /* 2.6, 0.4, 1e-8 */
  /* ScoreModel attributes used by the 'ncsnpp_v2' branch of forward (model.py:52-60); ignored by the other backbones */
  int loss_type, network_scaling, c_in, c_out, c_skip;
  float sigma_data;          /* 0.1 */
} sgmse_b200_config;

typedef struct sgmse_b200_sampler {
  int N;                     /* reverse steps (30) */
  int predictor;             /* SGMSE_B200_PRED_* */
  int corrector;             /* SGMSE_B200_CORR_* */
  int corrector_steps;       /* 1 */
  float snr;                 /* 0.5 */
  int denoise;               /* 1: return x_mean of the last predictor step */
  int probability_flow;      /* 0 */
  unsigned long long seed;   /* Philox seed (ignored with injected noise) */
  int utt_offset;            /* global index of utterance 0 (noise is keyed by global utterance id) */
  int pad_mode;              /* SGMSE_B200_PAD_* (enhance/analysis only) */
  int kind;                  /* SGMSE_B200_SAMPLER_*; the SB kinds use N, seed, utt_offset and the two fields below */
  float sb_eps;              /* end time of the SB samplers (1e-4, sampling/__init__.py:145) */
  int sb_n_steps;            /* value the SB samplers report as their second return value (50) */
} sgmse_b200_sampler;

const char* sgmse_b200_last_error(void);
const char* sgmse_b200_version(void);

int sgmse_b200_create(const sgmse_b200_config* cfg, sgmse_b200_engine** out);
void sgmse_b200_destroy(sgmse_b200_engine* e);

/* Weight manifest = the backbone's state_dict() in order: (key, numel).  Host-only; works without a GPU. */
int sgmse_b200_manifest_count(const sgmse_b200_engine* e);
int sgmse_b200_manifest_entry(const sgmse_b200_engine* e, int i, char* name, int name_cap, long long* numel);
long long sgmse_b200_weights_numel(const sgmse_b200_engine* e);
/* blob: fp32, all state_dict() tensors flattened and concatenated in manifest order (host memory). */
int sgmse_b200_load_weights(sgmse_b200_engine* e, const float* blob_host, long long numel);
/* same blob, already resident on this device (e.g. after an NCCL broadcast from rank 0) */
int sgmse_b200_load_weights_device(sgmse_b200_engine* e, const float* blob_dev, long long numel, void* stream);

/* Backbone contract: x c64 [B,2,F,T], t f32 [B] -> out c64 [B,1,F,T]  (device pointers). */
int sgmse_b200_dnn_forward(sgmse_b200_engine* e, const void* x, const float* t, void* out, int B, int F, int T,
                           void* stream);
/* score = -dnn(cat[x_t, y], t); x_t, y, out: c64 [B,1,F,T] */
int sgmse_b200_score(sgmse_b200_engine* e, const void* x_t, const void* y, const float* t, void* out, int B, int F,
                     int T, void* stream);
/* PC sampler.  y, out: c64 [B,1,F,T] (device).  noise: NULL (in-kernel Philox keyed by seed / global utterance
 * id / draw index) or device c64 [n_draws,B,1,F,T] consumed in the order prior, then per step the corrector
 * draws and the predictor draw (the order torch.randn_like is called in the reference).  *nfe receives
 * N * (corrector_steps + 1). */
int sgmse_b200_pc_sample(sgmse_b200_engine* e, const void* y, int B, int F, int T, const sgmse_b200_sampler* s,
                         const void* noise, void* out, int* nfe, void* stream);
int sgmse_b200_noise_draws(const sgmse_b200_sampler* s);
/* ScoreModel.forward(x_t, y, t) for the configured backbone: the legacy branch returns the score -dnn(cat[x_t, y], t);
 * the 'ncsnpp_v2' branch applies c_in / network_scaling / c_skip / c_out and returns the score (score_matching,
 * denoiser) or the data prediction, exactly as model.py:283-304.  x_t, y, out: c64 [B,1,F,T] (device), t: f32 [B]. */
int sgmse_b200_model_forward(sgmse_b200_engine* e, const void* x_t, const void* y, const float* t, void* out, int B,
                             int F, int T, void* stream);
/* Probability-flow ODE sampler (sampling/__init__.py:72-143 with denoise=False; the reference's default denoise=True
 * raises TypeError at predictors.py:60, the host mirror reproduces that).  x(1) = y + std(1) z, then
 * dx/dt = theta (y - x) - 0.5 g(t)^2 score(x, y, t) from t = 1 to t = eps with scipy's RK45 (Dormand-Prince 5(4), rtol /
 * atol error control, RMS norm over ALL bins of the batch: the utterances of one call share one adaptive step sequence,
 * as in the reference).  The integrator state is complex128 and stays in HBM; one double per norm crosses to the host.
 * OUVE SDE; backbones 'ncsnpp' / 'ncsnpp_48k', and 'ncsnpp_v2' with loss_type score_matching / denoiser (the drift calls
 * ScoreModel.forward, model.py:283-304). */
typedef struct sgmse_b200_ode {
  double rtol, atol;         /* 1e-5, 1e-5 (sampling/__init__.py:74) */
  double eps;                /* end time; ScoreModel.get_ode_sampler passes t_eps = 0.03 (model.py:375) */
  int max_attempts;          /* bound on Runge-Kutta step attempts, accepted + rejected (<= 0: 100000) */
  unsigned long long seed;   /* Philox seed of the prior draw (ignored with injected noise) */
  int utt_offset;            /* global index of utterance 0 */
} sgmse_b200_ode;
/* y, out: c64 [B,1,F,T] (device).  prior_noise: NULL (Philox) or device c64 [B,1,F,T], the one draw of prior_sampling
 * (sdes.py:224-229).  *nfe = number of network evaluations (scipy's nfev).  stats (nullable) receives
 * {accepted steps, rejected attempts, status (0 reached eps, -1 step size underflow = scipy "failed", whose last state
 * the reference silently returns, -2 max_attempts exhausted), 0}. */
int sgmse_b200_ode_sample(sgmse_b200_engine* e, const void* y, int B, int F, int T, const sgmse_b200_ode* o,
                          const void* prior_noise, void* out, int* nfe, int stats[4], void* stream);
/* The same controller on a host right-hand side (host-only; works without a GPU).  y: n complex128 values,
 * interleaved (re, im), in/out.  rhs(t, y, dydt, n, user) fills dydt.  Mirrors
 * solve_ivp(rhs, (t0, t_bound), y, method='RK45', rtol=rtol, atol=atol): y receives solution.y[:, -1]. */
typedef void (*sgmse_b200_ode_rhs)(double t, const double* y, double* dydt, long long n, void* user);
int sgmse_b200_rk45_host(sgmse_b200_ode_rhs rhs, void* user, double t0, double t_bound, double* y, long long n,
                         double rtol, double atol, int max_attempts, int* nfev, int stats[4]);

/* The sampler's host-computed schedule, exactly as the captured launch sequence uses it (host-only; works without a
 * GPU): ts[N] = torch.linspace(1, t_eps, N) in fp32 (sampling/__init__.py:56), prior_std = OUVESDE._std(1)
 * (sdes.py:206-229), and one (cy, cs, cz) row per state update in execution order -- per step the corrector steps, then
 * the predictor: x_mean = x + cy (y - x) + cs * score ; x = x_mean + cz * z  (correctors.py:69-81: cy = 0,
 * cs = eps = 2 (snr std(t))^2, cz = sqrt(2 eps); predictors.py:60-65 + sdes.py:72-137: cy = -theta dt, cs = G^2,
 * cz = G = g(t) sqrt(dt)).  The Langevin corrector's data-dependent rows are returned as zeros (filled on the device).
 * coef: [cap_updates][3] floats; *n_updates receives the number of rows (also when coef is NULL).
 * SB kinds: ts[N] = torch.linspace(1, sb_eps, N+1)[1:], prior_std = 0 and one row per step
 * (weight_prev, weight_estimate, weight_z | weight_prior_mean) of sampling/__init__.py:165-179 / :211-231. */
int sgmse_b200_sampler_schedule(const sgmse_b200_engine* e, const sgmse_b200_sampler* s, float* ts, float* prior_std,
                                float* coef, int cap_updates, int* n_updates);

/* padded frame count for a waveform of L samples */
int sgmse_b200_padded_frames(const sgmse_b200_engine* e, int L);
/* wav f32 [B,L] (device) -> Y c64 [B,1,F,Tpad], norm f32 [B] (device) */
int sgmse_b200_analysis(sgmse_b200_engine* e, const float* wav, int B, int L, int pad_mode, void* Y, float* norm,
                        void* stream);
/* X c64 [B,1,F,Tpad], norm f32 [B] -> wav f32 [B,L] (device) */
int sgmse_b200_synthesis(sgmse_b200_engine* e, const void* X, const float* norm, int B, int Tpad, int L, float* wav,
                         void* stream);
/* One call: wav [B,L] -> enhanced wav [B,L].  host_buffers != 0: wav/out are host pointers (pinned memory
 * recommended); the H2D / D2H copies are part of the call and it returns after the result is in `out`.
 * fp16 range: in the fp16 modes a raw convolution output beyond +-65504 is stored as inf; GroupNorm's statistics pass counts
 * every such event (counter "fp16_range_events").  With host buffers the call checks the counter before returning and FAILS
 * (non-zero code, message in sgmse_b200_last_error, counter reset) rather than hand out a NaN waveform; device-resident
 * callers read the counter themselves (it synchronises) and clear it with option "reset_range_events". */
int sgmse_b200_enhance(sgmse_b200_engine* e, const float* wav, int B, int L, const sgmse_b200_sampler* s,
                       const void* noise, float* out, int host_buffers, void* stream);

/* The same with the probability-flow ODE sampler (ScoreModel.enhance with sde.sampler_type == 'ode', model.py:446-447):
 * every utterance is its own ODE system (the reference calls enhance() per file); nfe (nullable) receives B counts.
 * prior_noise: NULL or device c64 [B,1,F,Tpad]. */
int sgmse_b200_enhance_ode(sgmse_b200_engine* e, const float* wav, int B, int L, const sgmse_b200_ode* o, int pad_mode,
                           const void* prior_noise, float* out, int host_buffers, int* nfe, void* stream);

/* Introspection / debugging */
/* bytes of activation workspace one forward pass of (B, F, T) needs; host-only (no CUDA call); -1 on error */
long long sgmse_b200_workspace_bytes(sgmse_b200_engine* e, int B, int F, int T);
/* copy a recorded intermediate activation (see sgmse_b200_set_option "record_taps") as fp32 NCHW to host */
int sgmse_b200_get_tap(sgmse_b200_engine* e, const char* name, float* out_host, long long cap, int shape[4]);
/* options: "record_taps" (0/1), "use_graphs" (0/1), "tc_mask" (bit i set = conv class i may use the wgmma kernel),
 * "time_convs" (0/1: bracket every convolution launch with CUDA events; disables graph replay),
 * "lanes" (1..8 concurrent launch sequences inside a captured sampler graph), "max_graphs" (captured sampler graphs kept,
 * least recently used evicted; default 16).  The kernel A/B switches the tools use ("tc_variant", "attn_variant",
 * "fir_variant", "inconv_variant", "outconv_variant", "combine_variant", "tc1_narrow", "gn_self", "gnfin_variant") are
 * state of THIS engine: every entry point installs the calling engine's selection before it launches anything, so another
 * engine of the same process (another device, another host thread) never sees them, and a captured sampler graph keeps
 * the selection it was captured with.  Value 0 always selects the current default kernel (TMA-fed wgmma convolutions,
 * cp.async / prefetched small-end kernels, half2 FIR-up, folded gn_finalize), and the alternatives keep a number of their
 * own: tc_variant 5 (GroupNorm+SiLU fused into the convolutions), fir_variant 3, outconv_variant 4, inconv_variant 3,
 * combine_variant 2, tc1_narrow / gn_self / gnfin_variant 2, attn_variant 3 (plain tile staging)
 * (tests/test_gpu_zz_next_rows.py::test_round1_kernels_agree_with_the_defaults).  No environment variable changes kernel
 * selection.  "pdl" (0/1: programmatic dependent launch between the kernels of the launch sequence) exists only in the
 * twin library built with -DSGMSE_B200_PDL (libsgmse_b200_pdl.so, counter "pdl_compiled" = 1); the product library
 * refuses it. */
int sgmse_b200_set_option(sgmse_b200_engine* e, const char* key, long long value);
/* counters: "kernel_launches" (since creation), "graph_launches", "cached_graphs", "workspace_bytes", "weights_bytes",
 * "tc_convs_last_forward", "direct_convs_last_forward", "launches_last_forward",
 * "timed_conv_tc_us" / "timed_conv_tc_mflop" / "timed_conv_tc_kbytes" / "timed_conv_tc_count" /
 * "timed_conv_direct_us" (sums over the launches timed since "time_convs" was switched on), "pdl_compiled", "pdl",
 * "fp16_range_events" (see sgmse_b200_enhance; synchronises the device) */
long long sgmse_b200_get_counter(const sgmse_b200_engine* e, const char* key);

#ifdef __cplusplus
}
#endif
#endif /* SGMSE_B200_H */
