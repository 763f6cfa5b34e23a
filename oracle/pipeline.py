"""End-to-end enhancement path (oracle): normalise -> STFT -> compress -> pad -> PC sample
-> decompress -> iSTFT -> renormalise.

Follows the sequence of sgmse/model.py:426-465 (``ScoreModel.enhance``)
resp. enhancement.py:75-96, batched over utterances.
TEST INFRASTRUCTURE – see oracle/__init__.py.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from . import ncsnpp, sde as sde_mod, spec as spec_mod
from .arch import NetConfig


def analysis(y: torch.Tensor, scfg: spec_mod.SpecConfig, pad_mode="zero_pad"):
    """[B, L] -> (Y c64 [B,1,F,Tpad], norm [B])."""
    norm = y.abs().amax(dim=1)
    Y = spec_mod.spec_fwd(spec_mod.stft(y / norm[:, None], scfg), scfg)[:, None]
    return spec_mod.pad_spec(Y, pad_mode), norm


def synthesis(X: torch.Tensor, norm: torch.Tensor, scfg: spec_mod.SpecConfig, length: int):
    x = spec_mod.istft(spec_mod.spec_back(X[:, 0], scfg), scfg, length)
    return x * norm[:, None]


def enhance(sd, cfg: NetConfig, scfg: spec_mod.SpecConfig, sde: sde_mod.OUVE, y: torch.Tensor,
            noise: List[torch.Tensor], N=30, eps=0.03, predictor="reverse_diffusion", corrector="ald",
            corrector_steps=1, snr=0.5, pad_mode="zero_pad", return_spec=False):
    Y, norm = analysis(y, scfg, pad_mode)

    def score_fn(x, yy, t):
        return ncsnpp.score(sd, cfg, x, yy, t)

    with torch.no_grad():
        X, nfe = sde_mod.pc_sample(score_fn, Y, sde, N=N, eps=eps, predictor=predictor, corrector=corrector,
                                   corrector_steps=corrector_steps, snr=snr, noise=noise)
    x_hat = synthesis(X, norm, scfg, y.shape[1])
    return (x_hat, X, Y) if return_spec else x_hat


def si_sdr(s, s_hat):
    """util/other.py:64-68."""
    import numpy as np
    alpha = np.dot(s_hat, s) / np.linalg.norm(s) ** 2
    return 10 * np.log10(np.linalg.norm(alpha * s) ** 2 / np.linalg.norm(alpha * s - s_hat) ** 2)
