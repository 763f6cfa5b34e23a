"""Pins the oracle (oracle/) to outputs of the unmodified reference (tests/golden/*.npz,
produced by oracle/make_golden.py).  CPU only."""
import os

import numpy as np
import pytest
import torch

from oracle import ncsnpp, sde as sde_mod, spec as spec_mod, pipeline
from oracle.arch import NetConfig, state_dict_manifest

SMALL = dict(nf=16, ch_mult=(1, 2, 2), image_size=64, num_res_blocks=2)
CASES = {
    "ncsnpp_small": NetConfig.ncsnpp(attn_resolutions=(16,), **SMALL),
    "ncsnpp48k_small": NetConfig.ncsnpp_48k(**SMALL),
}


def _load(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    sd = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w/")}
    return z, sd


def _rel(a, b):
    a, b = torch.as_tensor(a), torch.as_tensor(b)
    return ((a - b).abs().max() / b.abs().max()).item()


@pytest.mark.parametrize("name", list(CASES))
def test_manifest_matches_reference_state_dict(golden_dir, name):
    z, sd = _load(golden_dir, name)
    man = state_dict_manifest(CASES[name])
    assert [k for k, _ in man] == list(sd.keys())
    for k, s in man:
        assert tuple(sd[k].shape) == s


@pytest.mark.parametrize("name", list(CASES))
def test_forward_and_score(golden_dir, name):
    z, sd = _load(golden_dir, name)
    cfg = CASES[name]
    x, y, t = (torch.from_numpy(z[k]) for k in ("x", "y", "t"))
    out = ncsnpp.forward(sd, cfg, torch.cat([x, y], 1), t)
    assert _rel(out, z["dnn_out"]) < 1e-5
    assert _rel(ncsnpp.score(sd, cfg, x, y, t), z["score"]) < 1e-5


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("pred,corr", [("reverse_diffusion", "ald"), ("reverse_diffusion", "langevin"),
                                       ("none", "ald"), ("reverse_diffusion", "none")])
def test_pc_sampler(golden_dir, name, pred, corr):
    z, sd = _load(golden_dir, name)
    cfg = CASES[name]
    y = torch.from_numpy(z["y"])
    N = 3
    draws = sde_mod.make_noise(tuple(y.shape), sde_mod.n_noise_draws(N, pred, corr, 1), seed=7)
    with torch.no_grad():
        smp, nfe = sde_mod.pc_sample(lambda a, b, c: ncsnpp.score(sd, cfg, a, b, c), y, sde_mod.OUVE(), N=N,
                                     predictor=pred, corrector=corr, corrector_steps=1, snr=0.5, noise=draws)
    assert nfe == int(z[f"nfe_{pred}_{corr}"])
    assert _rel(smp, z[f"pc_{pred}_{corr}"]) < 2e-4


@pytest.mark.parametrize("name", list(CASES))
def test_enhance_chain(golden_dir, name):
    z, sd = _load(golden_dir, name)
    cfg = CASES[name]
    scfg = spec_mod.SpecConfig(n_fft=126, hop_length=32)
    wav = torch.from_numpy(z["wav"])
    B, N = wav.shape[0], 3
    draws = sde_mod.make_noise((B, 1, 64, 64), sde_mod.n_noise_draws(N, "reverse_diffusion", "ald", 1), seed=11)
    xh, X, Y = pipeline.enhance(sd, cfg, scfg, sde_mod.OUVE(), wav, draws, N=N, return_spec=True)
    assert _rel(Y, z["Y"]) < 1e-4
    assert _rel(xh, z["enh"]) < 1e-3


def test_fir_and_stft_ops(golden_dir):
    z = np.load(os.path.join(golden_dir, "ops.npz"))
    x = torch.from_numpy(z["fir_x"])
    assert _rel(ncsnpp.fir_down2(x), z["fir_down"]) < 1e-6
    assert _rel(ncsnpp.fir_up2(x), z["fir_up"]) < 1e-6
    scfg = spec_mod.SpecConfig(n_fft=126, hop_length=32)
    wav = torch.from_numpy(z["wav"])
    S = spec_mod.stft(wav, scfg)
    assert _rel(S, z["stft"]) < 1e-5
    assert _rel(spec_mod.spec_fwd(S, scfg), z["spec_fwd"]) < 1e-5
    assert _rel(spec_mod.spec_back(spec_mod.spec_fwd(S, scfg), scfg), z["spec_back"]) < 1e-4
    assert _rel(spec_mod.istft(torch.from_numpy(z["stft"]), scfg, 2000), z["istft"]) < 1e-5
    s48 = spec_mod.SpecConfig.cfg_48k()
    w48 = torch.from_numpy(z["wav48"])
    S48 = spec_mod.stft(w48, s48)
    assert _rel(S48, z["stft48"]) < 1e-5
    assert _rel(spec_mod.spec_fwd(S48, s48), z["spec_fwd48"]) < 1e-5
    assert _rel(spec_mod.istft(torch.from_numpy(z["stft48"]), s48, 6000), z["istft48"]) < 1e-5


# ---- SURVEY.md §8f-1: ncsnpp_v2 + preconditioned forward + Schroedinger-bridge samplers ----
V2_CFG = NetConfig.ncsnpp_v2(attn_resolutions=(16,), **SMALL)
PRECOND = {
    "plain": dict(loss_type="data_prediction", network_scaling=None, c_in="1", c_out="1", c_skip="0", sigma_data=0.1),
    "edm": dict(loss_type="data_prediction", network_scaling="1/sigma", c_in="edm", c_out="edm", c_skip="edm", sigma_data=0.1),
}


def test_v2_forward_and_preconditioning(golden_dir):
    z, sd = _load(golden_dir, "ncsnpp_v2_small")
    assert [k for k, _ in state_dict_manifest(V2_CFG)] == list(sd.keys())
    x, y, t = (torch.from_numpy(z[k]) for k in ("x", "y", "t"))
    sb = sde_mod.SBVE(2.6, 0.4)
    assert _rel(ncsnpp.forward_v2(sd, V2_CFG, x, y, t), z["dnn_out"]) < 1e-5
    for tag, pre in PRECOND.items():
        assert _rel(ncsnpp.precond_forward(sd, V2_CFG, pre, sb.std, x, y, t), z[f"fwd_{tag}"]) < 1e-5
    ou = sde_mod.OUVE()
    pre = dict(loss_type="score_matching", network_scaling=None, c_in="1", c_out="1/sigma", c_skip="0", sigma_data=0.1)
    std = lambda tt: torch.tensor([ou.std(float(v)) for v in tt])
    assert _rel(ncsnpp.precond_forward(sd, V2_CFG, pre, std, x, y, t), z["fwd_ouve_score"]) < 1e-5


@pytest.mark.parametrize("tag", list(PRECOND))
@pytest.mark.parametrize("sampler_type", ["sde", "ode"])
def test_v2_sb_sampler(golden_dir, tag, sampler_type):
    z, sd = _load(golden_dir, "ncsnpp_v2_small")
    y = torch.from_numpy(z["y"])
    sb = sde_mod.SBVE(2.6, 0.4)
    draws = sde_mod.make_noise(tuple(y.shape), 3, seed=13)
    fn = lambda a, b, c: ncsnpp.precond_forward(sd, V2_CFG, PRECOND[tag], sb.std, a, b, c)
    with torch.no_grad():
        got, n = sde_mod.sb_sample(fn, y, sb, N=3, sampler_type=sampler_type, noise=draws)
    assert n == int(z[f"sb_n_{sampler_type}_{tag}"])
    assert _rel(got, z[f"sb_{sampler_type}_{tag}"]) < 1e-4


def test_v2_pc_sampler_on_ouve(golden_dir):
    z, sd = _load(golden_dir, "ncsnpp_v2_small")
    y = torch.from_numpy(z["y"])
    ou = sde_mod.OUVE()
    pre = dict(loss_type="score_matching", network_scaling=None, c_in="1", c_out="1/sigma", c_skip="0", sigma_data=0.1)
    std = lambda tt: torch.tensor([ou.std(float(v)) for v in tt])
    fn = lambda a, b, c: ncsnpp.precond_forward(sd, V2_CFG, pre, std, a, b, c)
    draws = sde_mod.make_noise(tuple(y.shape), sde_mod.n_noise_draws(3, "reverse_diffusion", "ald", 1), seed=7)
    with torch.no_grad():
        got, nfe = sde_mod.pc_sample(fn, y, ou, N=3, noise=draws)
    assert nfe == 6 and _rel(got, z["pc_ouve_score"]) < 1e-4


# ---- SURVEY.md §8f-4: probability-flow ODE sampler ------------------------------------------------------------
def test_rk45_restatement_equals_scipy():
    """The integrator is third-party (scipy.integrate.solve_ivp, method RK45): the oracle's restatement of its
    published algorithm takes the same steps, the same number of evaluations and returns the same state, bit for bit,
    on a complex system whose right-hand side is rounded to complex64 like the sampler's."""
    from scipy.integrate import solve_ivp
    from oracle import ode
    rng = np.random.default_rng(0)
    n = 200
    M = (rng.standard_normal((n, n)) + 1j * rng.standard_normal((n, n))) * 0.3 / np.sqrt(n)
    b = rng.standard_normal(n) + 1j * rng.standard_normal(n)

    def fun(t, y):
        return (-1.5 * y + M @ np.tanh(y.real) + 1j * np.sin(3 * t) * b).astype(np.complex64)

    y0 = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    for rtol, atol, tb in [(1e-5, 1e-5, 0.03), (1e-3, 1e-6, 0.03), (1e-8, 1e-10, 0.5), (1e-5, 1e-5, 2.0), (1e-5, 1e-5, 1.0)]:
        s = solve_ivp(fun, (1.0, tb), y0, rtol=rtol, atol=atol, method="RK45")
        r = ode.rk45_solve(fun, 1.0, y0, tb, rtol=rtol, atol=atol)
        assert (s.nfev, s.status) == (r.nfev, r.status)
        assert np.array_equal(s.y[:, -1], r.y)
        if tb != 1.0:                                   # (an empty interval is reported by scipy as one zero-length step)
            assert np.array_equal(np.diff(s.t), np.asarray(r.hs))


@pytest.mark.parametrize("name,src", [("ode_small", "ncsnpp_small"), ("ode48k_small", "ncsnpp48k_small")])
def test_ode_sampler(golden_dir, name, src):
    """oracle/ode.py against get_ode_sampler() of the unmodified reference (denoise=False, prior draw injected):
    same number of function evaluations, same state."""
    from oracle import ode
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    _, sd = _load(golden_dir, src)
    cfg = CASES[src]
    y = torch.from_numpy(z["y"])
    prior = sde_mod.make_noise(tuple(y.shape), 1, seed=int(z["prior_seed"]))[0]
    tol = float(z["tol_loose"])
    x, nfe = ode.ode_sample(lambda a, b, c: ncsnpp.score(sd, cfg, a, b, c), y, sde_mod.OUVE(), eps=0.03, rtol=tol,
                            atol=tol, prior_noise=prior)
    assert nfe == int(z["nfe_loose"])
    assert _rel(x, z["x_loose"]) < 1e-6
    assert int(z["denoise_default_raises"]) == 1        # the reference's default denoise=True is a TypeError
    with pytest.raises(TypeError):
        ode.ode_sample(lambda a, b, c: None, y, sde_mod.OUVE(), prior_noise=prior, denoise=True)


@pytest.mark.slow
@pytest.mark.skipif(not os.environ.get("SGMSE_B200_SLOW"), reason="~3 minutes of CPU: set SGMSE_B200_SLOW=1")
def test_full_size_n30_oracle_equals_reference_run(golden_dir):
    """BASELINE.json configs[0]: the oracle repeats the unmodified reference's full-size N = 30 enhancement of one 4-s clip
    (tests/golden/full_n30.npz) from the same seeds."""
    from oracle import weights as o_w
    from sgmse_b200.synth import synthetic_speech
    z = np.load(os.path.join(golden_dir, "full_n30.npz"))
    cfg = NetConfig.ncsnpp()
    sd = o_w.make_state_dict(cfg, seed=int(z["weight_seed"]))
    wav = synthetic_speech(1, int(z["L"]), seed=int(z["wav_seed"]))
    N = int(z["N"])
    draws = sde_mod.make_noise((1, 1, 256, 512), sde_mod.n_noise_draws(N, "reverse_diffusion", "ald", 1), seed=int(z["noise_seed"]))
    x_hat, X, _ = pipeline.enhance(sd, cfg, spec_mod.SpecConfig(), sde_mod.OUVE(), wav, draws, N=N, snr=float(z["snr"]), return_spec=True)
    assert _rel(X[0, 0], z["sample"]) < 1e-4 and _rel(x_hat[0], z["enh"]) < 1e-4


V2_ODE_PRECOND = {
    "score": dict(loss_type="score_matching", network_scaling=None, c_in="1", c_out="1/sigma", c_skip="0", sigma_data=0.1),
    "denoiser_edm_in": dict(loss_type="denoiser", network_scaling="1/t", c_in="edm", c_out="1", c_skip="0", sigma_data=0.1),
}


@pytest.mark.parametrize("tag", list(V2_ODE_PRECOND))
def test_ode_sampler_on_v2_score_models(golden_dir, tag):
    """get_ode_sampler on preconditioned 'ncsnpp_v2' score models with the OUVE SDE (the drift calls ScoreModel.forward,
    model.py:283-304) against the unmodified reference: same number of evaluations, same state."""
    from oracle import ode
    z = np.load(os.path.join(golden_dir, "ode_v2_small.npz"))
    _, sd = _load(golden_dir, "ncsnpp_v2_small")
    y = torch.from_numpy(z["y"])
    prior = sde_mod.make_noise(tuple(y.shape), 1, seed=int(z["prior_seed"]))[0]
    ou = sde_mod.OUVE()
    pre = V2_ODE_PRECOND[tag]
    tol = float(z["tol"])
    x, nfe = ode.ode_sample(lambda a, b, c: ncsnpp.precond_forward(sd, V2_CFG, pre, ou.std_tensor, a, b, c), y, ou, eps=0.03,
                            rtol=tol, atol=tol, prior_noise=prior)
    assert nfe == int(z[f"nfe_{tag}"])
    assert _rel(x, z[f"x_{tag}"]) < 1e-5


MID = dict(nf=64, ch_mult=(1, 2, 2), image_size=64, attn_resolutions=(16,), num_res_blocks=1)
MID_PAIRS = [("reverse_diffusion", "ald", 3), ("reverse_diffusion", "langevin", 3), ("none", "ald", 3),
             ("reverse_diffusion", "none", 3), ("reverse_diffusion", "ald", 12)]


def test_mid_size_fixture_is_reproduced_by_the_oracle(golden_dir):
    """tests/golden/ncsnpp_mid.npz (oracle/make_golden.py: golden_mid_tc): reference outputs on the tensor-core-tileable
    mid-size config, weights from oracle/weights.py seed 5 -- the pin of the product-mode GPU tests."""
    from oracle import weights as o_w
    z = np.load(os.path.join(golden_dir, "ncsnpp_mid.npz"))
    cfg = NetConfig.ncsnpp(**MID)
    sd = o_w.make_state_dict(cfg, seed=int(z["weight_seed"]))
    x, y, t = (torch.from_numpy(z[k]) for k in ("x", "y", "t"))
    with torch.no_grad():
        assert _rel(ncsnpp.score(sd, cfg, x, y, t), z["score"]) < 1e-5
        for pred, corr, N in MID_PAIRS:
            draws = sde_mod.make_noise(tuple(y.shape), sde_mod.n_noise_draws(N, pred, corr, 1), seed=7)
            smp, nfe = sde_mod.pc_sample(lambda a, b, c: ncsnpp.score(sd, cfg, a, b, c), y, sde_mod.OUVE(), N=N,
                                         predictor=pred, corrector=corr, corrector_steps=1, snr=0.5, noise=draws)
            assert nfe == int(z[f"nfe_{pred}_{corr}_N{N}"])
            assert _rel(smp, z[f"pc_{pred}_{corr}_N{N}"]) < 5e-4, (pred, corr, N)
        # BASELINE config 4 sampler settings (N = 50, snr 0.33)
        draws = sde_mod.make_noise(tuple(y.shape), sde_mod.n_noise_draws(50, "reverse_diffusion", "ald", 1), seed=9)
        smp, nfe = sde_mod.pc_sample(lambda a, b, c: ncsnpp.score(sd, cfg, a, b, c), y, sde_mod.OUVE(), N=50,
                                     predictor="reverse_diffusion", corrector="ald", corrector_steps=1, snr=0.33, noise=draws)
        assert nfe == int(z["nfe_dereverb_N50_snr033"]) == 100
        assert _rel(smp, z["pc_dereverb_N50_snr033"]) < 5e-4
    wav = torch.from_numpy(z["wav"])
    draws = sde_mod.make_noise((2, 1, 64, 128), sde_mod.n_noise_draws(6, "reverse_diffusion", "ald", 1), seed=11)
    xh = pipeline.enhance(sd, cfg, spec_mod.SpecConfig(n_fft=126, hop_length=32), sde_mod.OUVE(), wav, draws, N=6)
    assert _rel(xh, z["enh"][:, 0] if z["enh"].ndim == 3 else z["enh"]) < 1e-3
