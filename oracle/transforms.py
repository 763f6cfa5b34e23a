"""The two training options the default path leaves out (oracle), and the fixture that pins them.

* SpecsDataModule ``--transform_type {exponent,log,none}`` (sgmse/data_module.py:118, spec_fwd / spec_back :162-188):
  ``log`` is log(1 + |z|) e^{j arg z} * spec_factor, inverse (exp(|z / spec_factor|) - 1) e^{j arg z}; ``none`` is the
  identity both ways.  ``exponent`` is oracle/spec.py.
* ``--no-centered`` on NCSNpp / NCSNpp_48k (ncsnpp.py:45-47,288-290; ncsnpp_48k.py:46-47,291-293): the backbone maps its
  four real input channels to 2x - 1 before the input conv and the input pyramid.

``python -m oracle.transforms`` regenerates tests/golden/transforms_small.npz from the UNMODIFIED reference (build
container only), like oracle/make_golden.py does for the other fixtures.
TEST INFRASTRUCTURE – see oracle/__init__.py.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import ncsnpp, refshim, sde as sde_mod, spec as spec_mod
from .arch import NetConfig
from .make_golden import OUT, _np

def spec_fwd(spec: torch.Tensor, cfg: spec_mod.SpecConfig, transform_type: str = "exponent") -> torch.Tensor:
    if transform_type == "exponent":
        return spec_mod.spec_fwd(spec, cfg)
    if transform_type == "log":                            # data_module.py:170-172
        return torch.log(1 + spec.abs()) * torch.exp(1j * spec.angle()) * cfg.spec_factor
    if transform_type == "none":                           # data_module.py:173-174: spec_factor is ignored
        return spec
    raise ValueError(transform_type)


def spec_back(spec: torch.Tensor, cfg: spec_mod.SpecConfig, transform_type: str = "exponent") -> torch.Tensor:
    if transform_type == "exponent":
        return spec_mod.spec_back(spec, cfg)
    if transform_type == "log":                            # data_module.py:183-185
        spec = spec / cfg.spec_factor
        return (torch.exp(spec.abs()) - 1) * torch.exp(1j * spec.angle())
    if transform_type == "none":                           # data_module.py:186-187
        return spec
    raise ValueError(transform_type)


def analysis(y: torch.Tensor, cfg: spec_mod.SpecConfig, transform_type: str, pad_mode="zero_pad"):
    """oracle/pipeline.py: analysis with the given transform.  [B, L] -> (Y c64 [B,1,F,Tpad], norm [B])."""
    norm = y.abs().amax(dim=1)
    Y = spec_fwd(spec_mod.stft(y / norm[:, None], cfg), cfg, transform_type)[:, None]
    return spec_mod.pad_spec(Y, pad_mode), norm


def synthesis(X: torch.Tensor, norm: torch.Tensor, cfg: spec_mod.SpecConfig, transform_type: str, length: int):
    return spec_mod.istft(spec_back(X[:, 0], cfg, transform_type), cfg, length) * norm[:, None]


def score(sd, cfg: NetConfig, x_t, y, t, centered: bool = True, dtype=torch.float32):
    """ScoreModel.forward, legacy branch (model.py:307-310), of a backbone built with ``centered``.  The backbone splits
    its complex input into (Re, Im) channels (ncsnpp.py:262-263, ncsnpp_48k.py:265-266); 2x - 1 on both parts is
    2x - (1 + 1j) on the complex value, the same fp32 operations."""
    x = torch.cat([x_t, y], dim=1)
    if not centered:
        x = 2 * x - (1 + 1j)
    return -ncsnpp.forward(sd, cfg, x, t, dtype=dtype)


# ---- the fixture ------------------------------------------------------------------------------------------------
TRANSFORMS_NET = dict(nf=32, ch_mult=(1, 2, 2), image_size=64, num_res_blocks=1)
# tag -> (backbone, --transform_type, --spec_factor, centered, weight seed).  'log' with spec_factor 1: the inverse
# exp(|X / spec_factor|) - 1 of what an untrained network samples (|X| up to ~10) then stays finite and comparable; at
# 0.15 it reaches exp(67) ~ 1e29.  'none' ignores spec_factor (the default 0.15 is passed).
TRANSFORM_CASES = {
    "log": ("ncsnpp", "log", 1.0, True, 21),
    "none": ("ncsnpp", "none", 0.15, True, 22),
    "nc": ("ncsnpp", "exponent", 0.15, False, 23),
    "nc48k": ("ncsnpp_48k", "exponent", 0.15, False, 24),
}


def transforms_net_config(backbone) -> NetConfig:
    if backbone == "ncsnpp":
        return NetConfig.ncsnpp(attn_resolutions=(16,), **TRANSFORMS_NET)
    return NetConfig.ncsnpp_48k(**TRANSFORMS_NET)


def golden_transforms(name="transforms_small"):
    """Per case: STFT -> transform -> pad_spec of two clips, the inverse transform of the unpadded transform, one score
    forward, a 3-step PC sample with injected noise and the enhancement chain of enhancement.py:75-96.  nf = 32 so that the
    fp16 tensor-core input convolutions take part.  Like ncsnpp_mid: weights (oracle/weights.py), clips and noise are
    regenerated from seeds (clips: 205, score input x: weight seed + 100); only the reference's OUTPUTS are stored."""
    from . import weights as o_w
    refshim.import_reference()
    from sgmse.util.other import pad_spec
    g = torch.Generator().manual_seed(205)
    B, L, N = 2, 2000, 3
    wav = 0.1 * torch.randn(B, L, generator=g)
    t = torch.tensor([0.83, 0.11])
    out = {}
    for tag, (backbone, transform_type, spec_factor, centered, seed) in TRANSFORM_CASES.items():
        cfg = transforms_net_config(backbone)
        model = refshim.make_score_model(backbone, seed=0, n_fft=126, hop_length=32, transform_type=transform_type,
                                         spec_factor=spec_factor, centered=centered, attn_resolutions=cfg.attn_resolutions,
                                         **TRANSFORMS_NET)
        assert model.data_module.transform_type == transform_type and model.dnn.centered == centered
        model.dnn.load_state_dict(o_w.make_state_dict(cfg, seed=seed))
        norm = wav.abs().amax(dim=1, keepdim=True)
        S = model._forward_transform(model._stft(wav / norm))
        Y = pad_spec(S[:, None])
        F, T = Y.shape[-2:]
        gx = torch.Generator().manual_seed(seed + 100)
        x = Y + 0.2 * torch.complex(torch.randn(B, 1, F, T, generator=gx), torch.randn(B, 1, F, T, generator=gx))
        with torch.no_grad():
            out[f"{tag}/Y"] = _np(Y)
            out[f"{tag}/back"] = _np(model._backward_transform(S))
            out[f"{tag}/score"] = _np(model(x, Y, t))
        draws = sde_mod.make_noise((B, 1, F, T), sde_mod.n_noise_draws(N, "reverse_diffusion", "ald", 1), seed=7)
        with refshim.injected_noise(draws):
            smp, _ = model.get_pc_sampler("reverse_diffusion", "ald", Y, N=N, corrector_steps=1, snr=0.5)()
        out[f"{tag}/pc"] = _np(smp)
        enh = []
        draws = sde_mod.make_noise((B, 1, F, T), sde_mod.n_noise_draws(N, "reverse_diffusion", "ald", 1), seed=11)
        for b in range(B):
            yb = wav[b:b + 1]
            nb = yb.abs().max()
            Yb = pad_spec(torch.unsqueeze(model._forward_transform(model._stft(yb / nb)), 0))
            with refshim.injected_noise([d[b:b + 1] for d in draws]):
                smp, _ = model.get_pc_sampler("reverse_diffusion", "ald", Yb, N=N, corrector_steps=1, snr=0.5)()
            enh.append(_np(model.to_audio(smp.squeeze(), L) * nb))
        out[f"{tag}/enh"] = np.stack(enh)
        print(name, tag, "|Y| max", float(Y.abs().max()), "|X| max", float(smp.abs().max()),
              "enh max", float(np.abs(out[f"{tag}/enh"]).max()))
    np.savez_compressed(os.path.join(OUT, f"{name}.npz"), wav_seed=np.int64(205), **out)


if __name__ == "__main__":
    golden_transforms()
