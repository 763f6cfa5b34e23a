"""Generate tests/golden/*.npz from the UNMODIFIED reference (build container only).

    python -m oracle.make_golden

Every array below is an output of the reference's own modules imported from
/root/reference (see oracle/refshim.py); the weights are the reference's own
random init (``torch.manual_seed``), stored so the fixtures travel to the GPU box.
Configs are reduced (nf=16, 3 levels, F=64) so that the fixtures stay small; the
full-size comparison against the live reference is tests/test_oracle_vs_reference.py.
TEST INFRASTRUCTURE – see oracle/__init__.py.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import refshim, sde as sde_mod
from .arch import NetConfig, state_dict_manifest

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

SMALL = dict(nf=16, ch_mult=(1, 2, 2), image_size=64, num_res_blocks=2)


def _np(t):
    return t.detach().cpu().numpy()


def golden_network(name, backbone, cfg: NetConfig, seed):
    model = refshim.make_score_model(backbone=backbone, seed=seed, nf=cfg.nf, ch_mult=cfg.ch_mult,
                                     image_size=cfg.image_size, attn_resolutions=cfg.attn_resolutions,
                                     n_fft=126, hop_length=32)
    sd = model.dnn.state_dict()
    assert [k for k, _ in state_dict_manifest(cfg)] == list(sd.keys())
    g = torch.Generator().manual_seed(seed + 100)
    B, F, T = 2, 64, 64
    x = torch.complex(torch.randn(B, 1, F, T, generator=g), torch.randn(B, 1, F, T, generator=g)) * 0.3
    y = torch.complex(torch.randn(B, 1, F, T, generator=g), torch.randn(B, 1, F, T, generator=g)) * 0.3
    t = torch.tensor([0.83, 0.11])
    with torch.no_grad():
        dnn_out = model.dnn(torch.cat([x, y], dim=1), t)
        score = model(x, y, t)

    # PC sampler with injected noise.  'euler_maruyama' is not reachable through pc_sampler in the
    # reference: predictors.py:49 forwards `stepsize` into OUVESDE.sde() -> TypeError.
    samples = {}
    N = 3
    for pred, corr in [("reverse_diffusion", "ald"), ("reverse_diffusion", "langevin"), ("none", "ald"),
                       ("reverse_diffusion", "none")]:
        nd = sde_mod.n_noise_draws(N, pred, corr, 1)
        draws = sde_mod.make_noise((B, 1, F, T), nd, seed=7)
        with refshim.injected_noise(draws):
            smp, nfe = model.get_pc_sampler(pred, corr, y, N=N, corrector_steps=1, snr=0.5)()
        samples[f"pc_{pred}_{corr}"] = _np(smp)
        samples[f"nfe_{pred}_{corr}"] = np.int64(nfe)

    # full enhancement chain (enhancement.py:75-96 sequence on CPU)
    from sgmse.util.other import pad_spec
    L = 2000
    wav = 0.1 * torch.randn(B, L, generator=g)
    outs, Ys = [], []
    for b in range(B):
        yb = wav[b:b + 1]
        norm = yb.abs().max()
        Y = torch.unsqueeze(model._forward_transform(model._stft(yb / norm)), 0)
        Y = pad_spec(Y)
        draws = [d[b:b + 1] for d in sde_mod.make_noise((B, 1, F, Y.shape[-1]), sde_mod.n_noise_draws(N, "reverse_diffusion", "ald", 1), seed=11)]
        with refshim.injected_noise(draws):
            smp, _ = model.get_pc_sampler("reverse_diffusion", "ald", Y, N=N, corrector_steps=1, snr=0.5)()
        xh = model.to_audio(smp.squeeze(), L) * norm
        outs.append(_np(xh)); Ys.append(_np(Y[0]))
    np.savez_compressed(
        os.path.join(OUT, f"{name}.npz"),
        **{"w/" + k: _np(v) for k, v in sd.items()},
        x=_np(x), y=_np(y), t=_np(t), dnn_out=_np(dnn_out), score=_np(score),
        wav=_np(wav), enh=np.stack(outs), Y=np.stack(Ys), **samples)
    print(name, "params", sum(v.numel() for v in sd.values()))


PRECOND = {
    "plain": dict(loss_type="data_prediction", network_scaling=None, c_in="1", c_out="1", c_skip="0", sigma_data=0.1),
    "edm": dict(loss_type="data_prediction", network_scaling="1/sigma", c_in="edm", c_out="edm", c_skip="edm", sigma_data=0.1),
}


def golden_v2(name, cfg: NetConfig, seed):
    """SURVEY.md §8f-1: backbone 'ncsnpp_v2' behind ScoreModel.forward's preconditioning (model.py:283-304) with the
    Schroedinger-bridge SDE and both SB samplers (sampling/__init__.py:145-249), plus the OUVE predictor-corrector
    sampler driven by a score-matching v2 model.  One set of weights, several ScoreModel wrappers."""
    kw = dict(nf=cfg.nf, ch_mult=cfg.ch_mult, image_size=cfg.image_size, attn_resolutions=cfg.attn_resolutions,
              n_fft=126, hop_length=32)
    base = refshim.make_score_model(backbone="ncsnpp_v2", seed=seed, sde="sbve", k=2.6, c=0.4, N=3, **kw, **PRECOND["plain"])
    sd = base.dnn.state_dict()
    assert [k for k, _ in state_dict_manifest(cfg)] == list(sd.keys())
    g = torch.Generator().manual_seed(seed + 100)
    B, F, T = 2, 64, 64
    x = torch.complex(torch.randn(B, 1, F, T, generator=g), torch.randn(B, 1, F, T, generator=g)) * 0.3
    y = torch.complex(torch.randn(B, 1, F, T, generator=g), torch.randn(B, 1, F, T, generator=g)) * 0.3
    t = torch.tensor([0.83, 0.11])
    out = {}
    with torch.no_grad():
        out["dnn_out"] = _np(base.dnn(x, y, t))
        for tag, pre in PRECOND.items():
            m = refshim.make_score_model(backbone="ncsnpp_v2", seed=seed, sde="sbve", k=2.6, c=0.4, N=3, **kw, **pre)
            m.dnn.load_state_dict(sd)
            out[f"fwd_{tag}"] = _np(m(x, y, t))
            for st in ("sde", "ode"):
                draws = sde_mod.make_noise((B, 1, F, T), 3, seed=13)
                with refshim.injected_noise(draws):
                    smp, n = m.get_sb_sampler(m.sde, y, sampler_type=st)()
                out[f"sb_{st}_{tag}"] = _np(smp)
                out[f"sb_n_{st}_{tag}"] = np.int64(n)
        # OUVE + PC sampler on a score-matching v2 model (c_skip = 0, c_out = 1/sigma, network output unscaled)
        pre = dict(loss_type="score_matching", network_scaling=None, c_in="1", c_out="1/sigma", c_skip="0", sigma_data=0.1)
        m = refshim.make_score_model(backbone="ncsnpp_v2", seed=seed, **kw, **pre)
        m.dnn.load_state_dict(sd)
        out["fwd_ouve_score"] = _np(m(x, y, t))
        N = 3
        draws = sde_mod.make_noise((B, 1, F, T), sde_mod.n_noise_draws(N, "reverse_diffusion", "ald", 1), seed=7)
        with refshim.injected_noise(draws):
            smp, nfe = m.get_pc_sampler("reverse_diffusion", "ald", y, N=N, corrector_steps=1, snr=0.5)()
        out["pc_ouve_score"] = _np(smp)
    np.savez_compressed(os.path.join(OUT, f"{name}.npz"), **{"w/" + k: _np(v) for k, v in sd.items()},
                        x=_np(x), y=_np(y), t=_np(t), **out)
    print(name, "params", sum(v.numel() for v in sd.values()))


def golden_ops():
    """Op-level outputs of the reference layer library (FIR resamplers, STFT chain)."""
    refshim.import_reference()
    from sgmse.backbones.ncsnpp_utils import up_or_down_sampling as uds
    from sgmse.data_module import SpecsDataModule
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 3, 8, 12, generator=g)
    dm = SpecsDataModule(base_dir="/nonexistent", n_fft=126, hop_length=32)
    dm48 = SpecsDataModule(base_dir="/nonexistent", n_fft=1534, hop_length=384, spec_factor=0.065,
                           spec_abs_exponent=0.667)
    wav = 0.1 * torch.randn(2, 2000, generator=g)
    wav48 = 0.1 * torch.randn(1, 6000, generator=g)
    S = dm.stft(wav)
    S48 = dm48.stft(wav48)
    np.savez_compressed(
        os.path.join(OUT, "ops.npz"),
        fir_x=_np(x), fir_down=_np(uds.downsample_2d(x, (1, 3, 3, 1), factor=2)),
        fir_up=_np(uds.upsample_2d(x, (1, 3, 3, 1), factor=2)),
        wav=_np(wav), stft=_np(S), spec_fwd=_np(dm.spec_fwd(S)), spec_back=_np(dm.spec_back(dm.spec_fwd(S))),
        istft=_np(dm.istft(S, 2000)),
        wav48=_np(wav48), stft48=_np(S48), spec_fwd48=_np(dm48.spec_fwd(S48)), istft48=_np(dm48.istft(S48, 6000)))


def golden_ode(name, src_name, backbone, cfg: NetConfig, seed):
    """SURVEY.md §8f-4: the probability-flow ODE sampler (sampling/__init__.py:72-143; scipy RK45 through host numpy
    round trips) of the unmodified reference, prior draw injected, ``denoise=False`` (``denoise=True`` raises TypeError in
    the reference, predictors.py:60).  The network is the one of ``src_name``.npz (same seed -> same init; asserted)."""
    model = refshim.make_score_model(backbone=backbone, seed=seed, nf=cfg.nf, ch_mult=cfg.ch_mult,
                                     image_size=cfg.image_size, attn_resolutions=cfg.attn_resolutions,
                                     n_fft=126, hop_length=32)
    z = np.load(os.path.join(OUT, src_name + ".npz"))
    for k, v in model.dnn.state_dict().items():
        assert np.array_equal(z["w/" + k], _np(v)), k
    y = torch.from_numpy(z["y"])
    out = {}
    for tag, tol in (("loose", 1e-3), ("default", 1e-5)):
        draws = sde_mod.make_noise(tuple(y.shape), 1, seed=17)
        with refshim.injected_noise(draws):
            smp, nfe = model.get_ode_sampler(y, denoise=False, device="cpu", rtol=tol, atol=tol)()
        out[f"x_{tag}"] = _np(smp)
        out[f"nfe_{tag}"] = np.int64(nfe)
        out[f"tol_{tag}"] = np.float64(tol)
        print(name, tag, "nfe", nfe)
    try:
        with refshim.injected_noise(sde_mod.make_noise(tuple(y.shape), 1, seed=17)):
            model.get_ode_sampler(y, device="cpu", rtol=1e-3, atol=1e-3)()
        out["denoise_default_raises"] = np.int64(0)
    except TypeError as exc:
        out["denoise_default_raises"] = np.int64(1)
        print("denoise=True ->", type(exc).__name__, exc)
    np.savez_compressed(os.path.join(OUT, f"{name}.npz"), y=_np(y), prior_seed=np.int64(17), **out)


def golden_full_n30(name="full_n30"):
    """BASELINE.json configs[0] through the UNMODIFIED reference: one 4-s 16 kHz clip, full-size NCSN++ (65.6 M
    parameters), OUVE SDE, predictor-corrector sampler reverse_diffusion + ald, N = 30, snr = 0.5 -- the sequence of
    model.enhance (model.py:433-459) / enhancement.py:75-96 on CPU, ~5 minutes on 8 cores.  The weights are the oracle's
    seeded init (oracle/weights.py, seed 0) loaded into the reference model, the clip is bench.py's synthetic utterance 0
    and the 61 noise draws come from seeds -- all three are regenerated on the GPU box, only the reference's OUTPUT is
    stored (enhanced waveform + final spectrogram, 1.3 MB)."""
    import time
    from . import weights as o_w
    from sgmse_b200.synth import synthetic_speech
    cfg = NetConfig.ncsnpp()
    model = refshim.make_score_model("ncsnpp", seed=0)
    from sgmse.util.other import pad_spec
    model.dnn.load_state_dict(o_w.make_state_dict(cfg, seed=0))
    L, N = 64000, 30
    wav = synthetic_speech(1, L)                                   # 0.1 * randn, torch.manual_seed(1000)
    t0 = time.time()
    norm = wav.abs().max()
    Y = torch.unsqueeze(model._forward_transform(model._stft(wav / norm)), 0)
    Y = pad_spec(Y)
    draws = sde_mod.make_noise(tuple(Y.shape), sde_mod.n_noise_draws(N, "reverse_diffusion", "ald", 1), seed=2000)
    with refshim.injected_noise(draws), torch.no_grad():
        sample, nfe = model.get_pc_sampler("reverse_diffusion", "ald", Y, N=N, corrector_steps=1, snr=0.5)()
    x_hat = model.to_audio(sample.squeeze(), L) * norm
    print(name, "reference CPU run", round(time.time() - t0, 1), "s, nfe", nfe, "threads", torch.get_num_threads())
    np.savez_compressed(os.path.join(OUT, f"{name}.npz"), enh=_np(x_hat.reshape(-1)), sample=_np(sample[0, 0]),
                        nfe=np.int64(nfe), N=np.int64(N), L=np.int64(L), wav_seed=np.int64(1000), weight_seed=np.int64(0),
                        noise_seed=np.int64(2000), snr=np.float64(0.5), cpu_seconds=np.float64(time.time() - t0),
                        cpu_threads=np.int64(torch.get_num_threads()))


V2_ODE_PRECOND = {
    "score": dict(loss_type="score_matching", network_scaling=None, c_in="1", c_out="1/sigma", c_skip="0", sigma_data=0.1),
    "denoiser_edm_in": dict(loss_type="denoiser", network_scaling="1/t", c_in="edm", c_out="1", c_skip="0", sigma_data=0.1),
}


def golden_ode_v2(name="ode_v2_small"):
    """The probability-flow ODE sampler on preconditioned 'ncsnpp_v2' score models with the OUVE SDE (get_ode_sampler calls
    ScoreModel.forward(x, y, t), i.e. model.py:283-304): the weights of ncsnpp_v2_small.npz under two ScoreModel wrappers --
    a plain score-matching model, and a 'denoiser' model with c_in = 'edm' and 1/t network scaling (every evaluation
    rescales the network input)."""
    cfg = NetConfig.ncsnpp_v2(attn_resolutions=(16,), **SMALL)
    kw = dict(nf=cfg.nf, ch_mult=cfg.ch_mult, image_size=cfg.image_size, attn_resolutions=cfg.attn_resolutions,
              n_fft=126, hop_length=32)
    z = np.load(os.path.join(OUT, "ncsnpp_v2_small.npz"))
    sd = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w/")}
    y = torch.from_numpy(z["y"])
    out = {}
    for tag, pre in V2_ODE_PRECOND.items():
        m = refshim.make_score_model(backbone="ncsnpp_v2", seed=3, **kw, **pre)
        m.dnn.load_state_dict(sd)
        with refshim.injected_noise(sde_mod.make_noise(tuple(y.shape), 1, seed=19)):
            smp, nfe = m.get_ode_sampler(y, denoise=False, device="cpu", rtol=1e-3, atol=1e-3)()
        out[f"x_{tag}"] = _np(smp)
        out[f"nfe_{tag}"] = np.int64(nfe)
        print(name, tag, "nfe", nfe, "finite", bool(torch.isfinite(torch.view_as_real(smp)).all()))
    np.savez_compressed(os.path.join(OUT, f"{name}.npz"), y=_np(y), prior_seed=np.int64(19), tol=np.float64(1e-3), **out)


MID = dict(nf=64, ch_mult=(1, 2, 2), image_size=64, attn_resolutions=(16,), num_res_blocks=1)


def golden_mid_tc(name="ncsnpp_mid"):
    """Reference-generated sampler / enhancement fixtures on a config whose layers are tensor-core-tileable (64..128 channels),
    so that the PRODUCT mode (fp16_tc) -- not only the fp32 validation mode -- is compared with outputs of the unmodified
    reference (VERDICT r1, weak #1).  Like full_n30: weights (oracle/weights.py seed 5, loaded into the reference model),
    inputs and noise are regenerated from seeds on the GPU box; only the reference's OUTPUTS are stored.
    Sampler: the four predictor/corrector pairs at N = 3, the default pair also at N = 12 (24 evaluations: drift over a
    longer chain); chain: enhancement.py:75-96 at N = 6 on two clips."""
    from . import weights as o_w
    cfg = NetConfig.ncsnpp(**MID)
    model = refshim.make_score_model("ncsnpp", seed=0, n_fft=126, hop_length=32, **MID)
    from sgmse.util.other import pad_spec
    model.dnn.load_state_dict(o_w.make_state_dict(cfg, seed=5))
    g = torch.Generator().manual_seed(105)
    B, F, T = 2, 64, 128
    y = torch.complex(torch.randn(B, 1, F, T, generator=g), torch.randn(B, 1, F, T, generator=g)) * 0.3
    x = y + 0.2 * torch.complex(torch.randn(B, 1, F, T, generator=g), torch.randn(B, 1, F, T, generator=g))
    t = torch.tensor([0.83, 0.11])
    out = {}
    with torch.no_grad():
        out["score"] = _np(model(x, y, t))
    for pred, corr, N in [("reverse_diffusion", "ald", 3), ("reverse_diffusion", "langevin", 3), ("none", "ald", 3),
                          ("reverse_diffusion", "none", 3), ("reverse_diffusion", "ald", 12)]:
        draws = sde_mod.make_noise((B, 1, F, T), sde_mod.n_noise_draws(N, pred, corr, 1), seed=7)
        with refshim.injected_noise(draws):
            smp, nfe = model.get_pc_sampler(pred, corr, y, N=N, corrector_steps=1, snr=0.5)()
        out[f"pc_{pred}_{corr}_N{N}"] = _np(smp)
        out[f"nfe_{pred}_{corr}_N{N}"] = np.int64(nfe)
    # BASELINE config 4 sampler settings (README.md:43: dereverberation checkpoint, --N 50 --snr 0.33): 100 evaluations
    draws = sde_mod.make_noise((B, 1, F, T), sde_mod.n_noise_draws(50, "reverse_diffusion", "ald", 1), seed=9)
    with refshim.injected_noise(draws):
        smp, nfe = model.get_pc_sampler("reverse_diffusion", "ald", y, N=50, corrector_steps=1, snr=0.33)()
    out["pc_dereverb_N50_snr033"] = _np(smp)
    out["nfe_dereverb_N50_snr033"] = np.int64(nfe)
    L, N = 4000, 6
    wav = 0.1 * torch.randn(B, L, generator=g)
    enh = []
    for b in range(B):
        yb = wav[b:b + 1]
        norm = yb.abs().max()
        Y = pad_spec(torch.unsqueeze(model._forward_transform(model._stft(yb / norm)), 0))
        draws = [d[b:b + 1] for d in sde_mod.make_noise((B, 1, F, Y.shape[-1]), sde_mod.n_noise_draws(N, "reverse_diffusion", "ald", 1), seed=11)]
        with refshim.injected_noise(draws):
            smp, _ = model.get_pc_sampler("reverse_diffusion", "ald", Y, N=N, corrector_steps=1, snr=0.5)()
        enh.append(_np(model.to_audio(smp.squeeze(), L) * norm))
    np.savez_compressed(os.path.join(OUT, f"{name}.npz"), x=_np(x), y=_np(y), t=_np(t), wav=_np(wav), enh=np.stack(enh),
                        weight_seed=np.int64(5), input_seed=np.int64(105), **out)
    print(name, "params", sum(v.numel() for v in model.dnn.state_dict().values()))


def main():
    os.makedirs(OUT, exist_ok=True)
    golden_ops()
    golden_network("ncsnpp_small", "ncsnpp", NetConfig.ncsnpp(attn_resolutions=(16,), **SMALL), seed=1)
    golden_network("ncsnpp48k_small", "ncsnpp_48k", NetConfig.ncsnpp_48k(**SMALL), seed=2)
    golden_v2("ncsnpp_v2_small", NetConfig.ncsnpp_v2(attn_resolutions=(16,), **SMALL), seed=3)
    golden_ode("ode_small", "ncsnpp_small", "ncsnpp", NetConfig.ncsnpp(attn_resolutions=(16,), **SMALL), seed=1)
    golden_ode("ode48k_small", "ncsnpp48k_small", "ncsnpp_48k", NetConfig.ncsnpp_48k(**SMALL), seed=2)
    golden_ode_v2()
    golden_mid_tc()
    golden_full_n30()            # ~2.5 minutes: the full-size reference run


if __name__ == "__main__":
    main()
