"""OUVE SDE scalars and the predictor-corrector sampler (oracle).

Follows sgmse/sdes.py:72-89,130-135,188-229,
sampling/__init__.py:52-68, sampling/predictors.py:41-76 and
sampling/correctors.py:37-94.  Noise is *injected* (popped from a list of
pre-generated complex normals) instead of drawn from torch's global RNG, so that
the CUDA engine can be compared on identical noise (SURVEY.md §4).

TEST INFRASTRUCTURE – see oracle/__init__.py.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable, List, Optional

import torch


@dataclass
class OUVE:
    theta: float = 1.5
    sigma_min: float = 0.05
    sigma_max: float = 0.5

    @property
    def logsig(self):
        return math.log(self.sigma_max / self.sigma_min)

    def diffusion(self, t: float) -> float:
        # sdes.py:188-196
        return self.sigma_min * (self.sigma_max / self.sigma_min) ** t * math.sqrt(2 * self.logsig)

    def std(self, t: float) -> float:
        # sdes.py:206-219
        th, ls, smin = self.theta, self.logsig, self.sigma_min
        return math.sqrt(smin ** 2 * math.exp(-2 * th * t) * (math.exp(2 * (th + ls) * t) - 1) * ls / (th + ls))

    def std_tensor(self, t: torch.Tensor) -> torch.Tensor:
        # sdes.py:206-219 on an fp32 tensor, operation by operation (what ScoreModel.forward's v2 branch calls, model.py:284)
        sigma_min, theta, logsig = self.sigma_min, self.theta, self.logsig
        return torch.sqrt((sigma_min ** 2 * torch.exp(-2 * theta * t) * (torch.exp(2 * (theta + logsig) * t) - 1) * logsig)
                          / (theta + logsig))


def timesteps(N: int, eps: float, T: float = 1.0):
    """torch.linspace(T, eps, N) evaluated in fp32 like the reference (sampling/__init__.py:56)."""
    return [float(v) for v in torch.linspace(T, eps, N)]


def complex_normal(shape, seed: int) -> torch.Tensor:
    """CN(0,1) like torch.randn_like(complex64): real, imag ~ N(0, 1/2)."""
    g = torch.Generator().manual_seed(seed)
    re = torch.randn(shape, generator=g)
    im = torch.randn(shape, generator=g)
    return torch.complex(re, im) * math.sqrt(0.5)


def make_noise(shape, n_draws: int, seed: int) -> List[torch.Tensor]:
    return [complex_normal(shape, seed * 1000 + i) for i in range(n_draws)]


def n_noise_draws(N: int, predictor: str, corrector: str, corrector_steps: int) -> int:
    c = corrector_steps if corrector != "none" else 0
    p = 0 if predictor == "none" else 1
    return 1 + N * (c + p)


def pc_sample(score_fn: Callable, y: torch.Tensor, sde: OUVE, N: int = 30, eps: float = 0.03,
              predictor: str = "reverse_diffusion", corrector: str = "ald",
              corrector_steps: int = 1, snr: float = 0.5, noise: Optional[List[torch.Tensor]] = None,
              denoise: bool = True, probability_flow: bool = False):
    """pc_sampler() of sampling/__init__.py:52-68.  ``score_fn(x, y, t_vec) -> score``.
    ``noise`` is consumed in call order: prior, then per step corrector draws, predictor draw."""
    B = y.shape[0]
    noise = list(noise) if noise is not None else None
    if noise is None:
        raise ValueError("oracle sampler requires injected noise")
    it = iter(noise)

    xt = y + next(it) * sde.std(1.0)                                   # sdes.py:224-229
    ts = timesteps(N, eps)
    xt_mean = xt
    for i in range(N):
        t = ts[i]
        # reference computes `t - timesteps[i+1]` on fp32 tensors (sampling/__init__.py:59-62)
        stepsize = float(torch.tensor(ts[i], dtype=torch.float32) - torch.tensor(ts[i + 1], dtype=torch.float32)) \
            if i != N - 1 else ts[-1]
        vec_t = torch.full((B,), t, dtype=torch.float32)
        # ---- corrector (correctors.py) ----
        if corrector == "ald":
            std = sde.std(t)
            for _ in range(corrector_steps):
                grad = score_fn(xt, y, vec_t)
                z = next(it)
                step = (snr * std) ** 2 * 2
                xt_mean = xt + step * grad
                xt = xt_mean + z * math.sqrt(step * 2)
        elif corrector == "langevin":
            for _ in range(corrector_steps):
                grad = score_fn(xt, y, vec_t)
                z = next(it)
                gnorm = torch.linalg.vector_norm(grad.reshape(B, -1), dim=-1).mean()
                znorm = torch.linalg.vector_norm(z.reshape(B, -1), dim=-1).mean()
                step = (snr * znorm / gnorm) ** 2 * 2
                xt_mean = xt + step * grad
                xt = xt_mean + z * torch.sqrt(step * 2)
        elif corrector == "none":
            xt_mean = xt
        else:
            raise ValueError(f"Corrector with name '{corrector}' unknown.")
        # ---- predictor (predictors.py) ----
        if predictor == "reverse_diffusion":
            g = sde.diffusion(t)
            f = sde.theta * (y - xt) * stepsize                       # sdes.py:85-88
            G = g * math.sqrt(stepsize)
            sc = score_fn(xt, y, vec_t)
            rev_f = f - G ** 2 * sc * (0.5 if probability_flow else 1.0)
            rev_G = 0.0 if probability_flow else G
            z = next(it)
            xt_mean = xt - rev_f
            xt = xt_mean + rev_G * z
        elif predictor == "euler_maruyama":
            dt = -1.0 / N
            z = next(it)
            g = sde.diffusion(t)
            sc = score_fn(xt, y, vec_t)
            drift = sde.theta * (y - xt) - g ** 2 * sc * (0.5 if probability_flow else 1.0)
            gg = 0.0 if probability_flow else g
            xt_mean = xt + drift * dt
            xt = xt_mean + gg * math.sqrt(-dt) * z
        elif predictor == "none":
            xt_mean = xt
        else:
            raise ValueError(f"Predictor with name '{predictor}' unknown.")
    nfe = N * ((corrector_steps if corrector != "none" else 0) + 1)
    return (xt_mean if denoise else xt), nfe


# ---- Schroedinger bridge (SURVEY.md §8f-1) ---------------------------------------------------------------------
@dataclass
class SBVE:
    """SBVESDE (sdes.py:235-312).  ``eps`` is the stabiliser of ``_sigmas_alphas`` (1e-8), not the end time.  All
    scalars are evaluated on fp32 tensors like the reference does."""
    k: float = 2.6
    c: float = 0.4
    eps: float = 1e-8
    T: float = 1.0

    def sigmas_alphas(self, t: torch.Tensor):
        # sdes.py:276-287
        alpha_t = torch.ones_like(t)
        alpha_T = torch.ones_like(t)
        logk2 = 2 * torch.log(torch.tensor(self.k))
        sigma_t = torch.sqrt((self.c * (self.k ** (2 * t) - 1.0)) / logk2)
        sigma_T = torch.sqrt((self.c * (self.k ** (2 * self.T) - 1.0)) / logk2)
        alpha_bart = alpha_t / (alpha_T + self.eps)
        sigma_bart = torch.sqrt(sigma_T ** 2 - sigma_t ** 2 + self.eps)
        return sigma_t, sigma_T, sigma_bart, alpha_t, alpha_T, alpha_bart

    def std(self, t: torch.Tensor):
        # sdes.py:298-302
        sigma_t, sigma_T, sigma_bart, alpha_t, _, _ = self.sigmas_alphas(t)
        return (alpha_t * sigma_bart * sigma_t) / (sigma_T + self.eps)


def sb_weights(sde: SBVE, N: int, eps: float, sampler_type: str):
    """Per-step time and weights of the SB samplers, evaluated on fp32 tensors exactly as sampling/__init__.py:152-179
    (sde: weight_prev, weight_estimate, weight_z -- zero in the last step) and :195-231 (ode: weight_prev, weight_estimate,
    weight_prior_mean).  Returns ``(ts f32 [N], rows f32 [N, 3])``."""
    ts = torch.linspace(sde.T, eps, N + 1)
    one = torch.ones(1)
    sigma_prev, sigma_T, sigma_bar_prev, alpha_prev, alpha_T, _ = sde.sigmas_alphas(ts[0] * one)
    rows = []
    for t in ts[1:]:
        sigma_t, sigma_T, sigma_bart, alpha_t, alpha_T, _ = sde.sigmas_alphas(t * one)
        if sampler_type == "sde":
            w_prev = alpha_t * sigma_t ** 2 / (alpha_prev * sigma_prev ** 2 + sde.eps)
            tmp = 1 - sigma_t ** 2 / (sigma_prev ** 2 + sde.eps)
            w_est = alpha_t * tmp
            w_3 = alpha_t * sigma_t * torch.sqrt(tmp)
            if t == ts[-1]:
                w_3 = torch.zeros(1)
        elif sampler_type == "ode":
            w_prev = alpha_t * sigma_t * sigma_bart / (alpha_prev * sigma_prev * sigma_bar_prev + sde.eps)
            w_est = alpha_t / (sigma_T ** 2 + sde.eps) * (sigma_bart ** 2 - sigma_bar_prev * sigma_t * sigma_bart / (sigma_prev + sde.eps))
            w_3 = alpha_t / (alpha_T * sigma_T ** 2 + sde.eps) * (sigma_t ** 2 - sigma_prev * sigma_t * sigma_bart / (sigma_bar_prev + sde.eps))
        else:
            raise ValueError("Invalid type. Choose 'ode' or 'sde'.")
        rows.append(torch.cat([w_prev, w_est, w_3]))
        alpha_prev, sigma_prev, sigma_bar_prev = alpha_t, sigma_t, sigma_bart
    return ts[1:].clone(), torch.stack(rows)


def sb_sample(model_fn: Callable, y: torch.Tensor, sde: SBVE, N: int = 50, eps: float = 1e-4, sampler_type: str = "ode",
              noise: Optional[List[torch.Tensor]] = None, n_steps: int = 50):
    """get_sb_sampler() of sampling/__init__.py:145-249.  ``model_fn(x_t, y, t_vec) -> current estimate`` (the
    data-prediction output of ScoreModel.forward).  The SDE variant draws one complex normal per step (also in the
    last one, where its weight is zeroed, sampling/__init__.py:176-179); ``noise`` is consumed in that order.
    Returns ``(x, n_steps)`` -- the reference reports its ``n_steps`` argument, not the number of evaluations."""
    B = y.shape[0]
    xt = y[:, [0]] if sampler_type == "sde" else y
    ts, rows = sb_weights(sde, N, eps, sampler_type)
    it = iter(noise) if noise is not None else None
    for t, (w_prev, w_est, w_3) in zip(ts, rows):
        est = model_fn(xt, y, t * torch.ones(B))
        if sampler_type == "sde":
            if it is None:
                raise ValueError("oracle sampler requires injected noise")
            z = next(it)
            xt = w_prev * xt + w_est * est + (w_3 * z if float(w_3) != 0.0 else 0.0)
        else:
            xt = w_prev * xt + w_est * est + w_3 * y
    return xt, n_steps
