"""The spectrogram transforms 'log' / 'none' (SpecsDataModule --transform_type, data_module.py:118,162-188) and the
--no-centered backbones (ncsnpp.py:45-47,288-290): the oracle against tests/golden/transforms_small.npz (outputs of the
unmodified reference, oracle/transforms.py: golden_transforms), how the drop-in reads both options off a live
ScoreModel, and the C ABI's range checks.  CPU only."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import refshim, sde as sde_mod, spec as spec_mod, transforms as o_tr, weights as o_w
from oracle.transforms import TRANSFORM_CASES, TRANSFORMS_NET, transforms_net_config
from sgmse_b200 import EngineConfig, _lib


def _rel(a, b):
    a, b = torch.as_tensor(a), torch.as_tensor(b)
    return ((a - b).abs().max() / b.abs().max()).item()


def _case(tag):
    backbone, transform_type, spec_factor, centered, seed = TRANSFORM_CASES[tag]
    cfg = transforms_net_config(backbone)
    sd = o_w.make_state_dict(cfg, seed=seed)
    scfg = spec_mod.SpecConfig(n_fft=126, hop_length=32, spec_factor=spec_factor)
    return cfg, sd, scfg, transform_type, centered, seed


@pytest.fixture(scope="module")
def fixture(golden_dir):
    return np.load(os.path.join(golden_dir, "transforms_small.npz"))


@pytest.mark.parametrize("tag", list(TRANSFORM_CASES))
def test_oracle_reproduces_fixture(fixture, tag):
    z = fixture
    cfg, sd, scfg, transform_type, centered, seed = _case(tag)
    wav = 0.1 * torch.randn(2, 2000, generator=torch.Generator().manual_seed(int(z["wav_seed"])))
    B, L, N = wav.shape[0], wav.shape[1], 3
    Y, norm = o_tr.analysis(wav, scfg, transform_type)
    assert _rel(Y, z[f"{tag}/Y"]) < 1e-6
    S = o_tr.spec_fwd(spec_mod.stft(wav / norm[:, None], scfg), scfg, transform_type)
    assert _rel(o_tr.spec_back(S, scfg, transform_type), z[f"{tag}/back"]) < 1e-6
    F, T = Y.shape[-2:]
    gx = torch.Generator().manual_seed(seed + 100)
    x = Y + 0.2 * torch.complex(torch.randn(B, 1, F, T, generator=gx), torch.randn(B, 1, F, T, generator=gx))
    t = torch.tensor([0.83, 0.11])
    score_fn = lambda a, b, c: o_tr.score(sd, cfg, a, b, c, centered=centered)
    # max-abs errors relative to the largest value, measured: transforms <= 7.3e-7, score <= 2.0e-6, 3-step sampler
    # <= 1.2e-6, waveform <= 7.8e-6 (log: exp() amplifies) / 1.1e-6 (the others)
    with torch.no_grad():
        assert _rel(score_fn(x, Y, t), z[f"{tag}/score"]) < 1e-5
        # the other centering misses by O(1): the fixture pins the option, not only the transform
        assert _rel(o_tr.score(sd, cfg, x, Y, t, centered=not centered), z[f"{tag}/score"]) > 0.1
        for key, seed_n in (("pc", 7), ("enh", 11)):
            draws = sde_mod.make_noise((B, 1, F, T), sde_mod.n_noise_draws(N, "reverse_diffusion", "ald", 1), seed=seed_n)
            X, _ = sde_mod.pc_sample(score_fn, Y, sde_mod.OUVE(), N=N, predictor="reverse_diffusion", corrector="ald",
                                     corrector_steps=1, snr=0.5, noise=draws)
            if key == "pc":
                assert _rel(X, z[f"{tag}/pc"]) < 1e-5
            else:
                assert _rel(o_tr.synthesis(X, norm, scfg, transform_type, L), z[f"{tag}/enh"]) < 3e-5


def test_transforms_of_zero_and_round_trip():
    g = torch.Generator().manual_seed(3)
    S = torch.complex(torch.randn(2, 64, 40, generator=g), torch.randn(2, 64, 40, generator=g))
    S[0, 0, :5] = 0
    scfg = spec_mod.SpecConfig(n_fft=126, hop_length=32)
    for tt in ("log", "none"):
        Y = o_tr.spec_fwd(S, scfg, tt)
        assert torch.equal(Y[0, 0, :5], torch.zeros(5, dtype=Y.dtype))
        assert _rel(o_tr.spec_back(Y, scfg, tt), S) < 1e-5
    assert torch.equal(o_tr.spec_fwd(S, spec_mod.SpecConfig(spec_factor=0.3), "none"), S)
    assert torch.equal(o_tr.spec_fwd(S, scfg, "exponent"), spec_mod.spec_fwd(S, scfg))
    with pytest.raises(ValueError):
        o_tr.spec_fwd(S, scfg, "sqrt")


@pytest.mark.skipif(not refshim.reference_available(), reason="reference checkout not present")
@pytest.mark.parametrize("tag", list(TRANSFORM_CASES))
def test_config_from_score_model_reads_both_options(tag):
    from sgmse_b200.api import config_from_score_model
    backbone, transform_type, spec_factor, centered, _ = TRANSFORM_CASES[tag]
    cfg = transforms_net_config(backbone)
    model = refshim.make_score_model(backbone, seed=0, n_fft=126, hop_length=32, transform_type=transform_type,
                                     spec_factor=spec_factor, centered=centered, attn_resolutions=cfg.attn_resolutions,
                                     **TRANSFORMS_NET)
    ec = config_from_score_model(model, mode="fp32")
    assert (ec.backbone, ec.transform_type, ec.spec_factor, ec.centered) == (backbone, transform_type, spec_factor, centered)
    c = ec.to_c()
    assert c.transform_type == {"exponent": 0, "log": 1, "none": 2}[transform_type]
    assert c.not_centered == int(not centered)
    # the defaults map to the zero fields of a zero-initialised struct
    dflt = config_from_score_model(refshim.make_score_model(backbone, seed=0, n_fft=126, hop_length=32,
                                                             attn_resolutions=cfg.attn_resolutions, **TRANSFORMS_NET))
    assert (dflt.transform_type, dflt.centered) == ("exponent", True)
    assert (dflt.to_c().transform_type, dflt.to_c().not_centered) == (0, 0)


def _create(cfg):
    lib = _lib.load()
    h = C.c_void_p()
    rc = lib.sgmse_b200_create(C.byref(cfg), C.byref(h))
    if rc == 0:
        lib.sgmse_b200_destroy(h)
    return rc, lib.sgmse_b200_last_error().decode()


def test_c_abi_checks_the_new_fields():
    for tt in range(3):
        cfg = EngineConfig(nf=16, ch_mult=(1, 2, 2), image_size=64).to_c()
        cfg.transform_type = tt
        assert _create(cfg)[0] == 0
    cfg = EngineConfig(nf=16, ch_mult=(1, 2, 2), image_size=64).to_c()
    cfg.transform_type = 3
    rc, msg = _create(cfg)
    assert rc != 0 and "transform_type 3" in msg
    cfg = EngineConfig(nf=16, ch_mult=(1, 2, 2), image_size=64, centered=False).to_c()
    assert cfg.not_centered == 1 and _create(cfg)[0] == 0
    cfg.not_centered = 2
    rc, msg = _create(cfg)
    assert rc != 0 and "not_centered" in msg
    cfg = EngineConfig.ncsnpp_v2(nf=16, ch_mult=(1, 2, 2), image_size=64).to_c()
    cfg.not_centered = 1
    rc, msg = _create(cfg)
    assert rc != 0 and "ncsnpp_v2" in msg
    with pytest.raises(ValueError, match="Transform type with name 'sqrt' unknown."):
        EngineConfig(transform_type="sqrt").to_c()
    with pytest.raises(ValueError, match="no-centered"):
        EngineConfig.ncsnpp_v2(centered=False).to_c()
