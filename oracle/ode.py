"""Probability-flow ODE sampler (oracle) -- SURVEY.md §8(f-4).

Follows sgmse/sampling/__init__.py:72-143 (``get_ode_sampler``), sdes.py:91-137
(``RSDE.sde`` with ``probability_flow=True``) and sdes.py:188-196 (``OUVESDE.sde``).

The integrator the reference calls is third-party: ``scipy.integrate.solve_ivp(method='RK45')`` (the reference pins
scipy==1.10.1, requirements_version.txt:14; this image has scipy 1.18.1).  It is not under /root/reference, so its
published algorithm is restated here -- Dormand-Prince 5(4) with the step-size controller of Hairer, Norsett & Wanner,
"Solving Ordinary Differential Equations I", Sec. II.4, as scipy implements it (scipy/integrate/_ivp/rk.py
``RungeKutta._step_impl`` / ``rk_step``, common.py ``select_initial_step`` / ``norm``, base.py ``OdeSolver.step``) --
and pinned against the installed scipy (tests/test_oracle_golden.py::test_rk45_restatement_equals_scipy) and against
the unmodified reference sampler (tests/golden/ode_small.npz, tests/test_oracle_vs_reference.py).  scipy 1.10.1's
``select_initial_step`` lacks the two ``interval_length`` clamps of 1.18.1; they only act when the first step would
overshoot the whole interval (never for T=1 -> eps=0.03 at the sampler's tolerances).

What the reference does, as executed (sampling/__init__.py:107-141):
  * x(T) = y + z * std(1)                       (prior_sampling, sdes.py:224-229; one complex normal)
  * the state is flattened to a complex128 numpy vector; every right-hand-side evaluation casts it back to complex64,
    evaluates ``drift = theta (y - x) - 0.5 g(t)^2 score(x, y, t)`` in fp32 and returns complex64 (promoted to
    complex128 inside scipy)
  * the error norm is the RMS over ALL elements of the batch: one ODE system per sampler call, the utterances of a
    batch share one adaptive step sequence
  * ``denoise=True`` (the default!) calls ``predictor.update_fn(x, y, vec_eps)`` without ``stepsize`` ->
    ``TypeError`` (predictors.py:60): only ``denoise=False`` returns a result.  The oracle mirrors that.

TEST INFRASTRUCTURE -- see oracle/__init__.py.
"""
from __future__ import annotations

import math
from typing import Callable, Optional

import numpy as np
import torch

from .sde import OUVE

# Dormand-Prince 5(4) tableau (Dormand & Prince 1980; the numbers scipy's RK45 class carries)
C = np.array([0, 1 / 5, 3 / 10, 4 / 5, 8 / 9, 1])
A = np.array([
    [0, 0, 0, 0, 0],
    [1 / 5, 0, 0, 0, 0],
    [3 / 40, 9 / 40, 0, 0, 0],
    [44 / 45, -56 / 15, 32 / 9, 0, 0],
    [19372 / 6561, -25360 / 2187, 64448 / 6561, -212 / 729, 0],
    [9017 / 3168, -355 / 33, 46732 / 5247, 49 / 176, -5103 / 18656],
])
B = np.array([35 / 384, 0, 500 / 1113, 125 / 192, -2187 / 6784, 11 / 84])
E = np.array([-71 / 57600, 0, 71 / 16695, -71 / 1920, 17253 / 339200, -22 / 525, 1 / 40])
ORDER = 5
ERROR_ESTIMATOR_ORDER = 4
N_STAGES = 6
SAFETY, MIN_FACTOR, MAX_FACTOR = 0.9, 0.2, 10.0


def rms_norm(x: np.ndarray) -> float:
    """scipy common.norm: ||x||_2 / sqrt(n) (complex modulus for complex x)."""
    return float(np.linalg.norm(x) / x.size ** 0.5)


def select_initial_step(fun, t0, y0, t_bound, f0, direction, rtol, atol):
    """common.select_initial_step (scipy 1.18.1), max_step = inf.  One extra evaluation of ``fun``."""
    if y0.size == 0:
        return math.inf
    interval_length = abs(t_bound - t0)
    if interval_length == 0.0:
        return 0.0
    scale = atol + np.abs(y0) * rtol
    d0 = rms_norm(y0 / scale)
    d1 = rms_norm(f0 / scale)
    h0 = 1e-6 if (d0 < 1e-5 or d1 < 1e-5) else 0.01 * d0 / d1
    h0 = min(h0, interval_length)
    y1 = y0 + h0 * direction * f0
    f1 = fun(t0 + h0 * direction, y1)
    d2 = rms_norm((f1 - f0) / scale) / h0
    if d1 <= 1e-15 and d2 <= 1e-15:
        h1 = max(1e-6, h0 * 1e-3)
    else:
        h1 = (0.01 / max(d1, d2)) ** (1 / (ERROR_ESTIMATOR_ORDER + 1))
    return min(100 * h0, h1, interval_length)


class Rk45Result:
    def __init__(self, t, y, nfev, steps, status, hs):
        self.t, self.y, self.nfev, self.steps, self.status, self.hs = t, y, nfev, steps, status, hs


def rk45_solve(fun: Callable, t0: float, y0: np.ndarray, t_bound: float, rtol: float = 1e-3, atol: float = 1e-6,
               max_steps: int = 100000) -> Rk45Result:
    """``solve_ivp(fun, (t0, t_bound), y0, method='RK45', rtol=rtol, atol=atol)`` restated: returns the state at
    ``t_bound`` (``solution.y[:, -1]``), ``nfev``, the accepted step sizes and ``status`` (0 finished, -1 step too
    small -- in which case y is the last accepted state, which is what the reference silently uses)."""
    y = np.asarray(y0).astype(complex if np.iscomplexobj(y0) else float)
    t = float(t0)
    t_bound = float(t_bound)
    direction = float(np.sign(t_bound - t0)) if t_bound != t0 else 1.0
    eps = np.finfo(float).eps
    if rtol < 100 * eps:                      # validate_tol
        rtol = 100 * eps
    nfev = 0

    def f(tt, yy):
        nonlocal nfev
        nfev += 1
        return np.asarray(fun(tt, yy), dtype=y.dtype)

    fcur = f(t, y)
    h_abs = select_initial_step(f, t, y, t_bound, fcur, direction, rtol, atol)
    n = y.size
    K = np.empty((N_STAGES + 1, n), dtype=y.dtype)
    error_exponent = -1 / (ERROR_ESTIMATOR_ORDER + 1)
    hs = []
    status = None
    steps = 0
    while status is None:
        if n == 0 or t == t_bound:            # OdeSolver.step
            t = t_bound
            status = 0
            break
        if steps >= max_steps:
            status = -2
            break
        min_step = 10 * abs(np.nextafter(t, direction * np.inf) - t)
        if h_abs < min_step:
            h_abs = min_step
        step_accepted = False
        step_rejected = False
        failed = False
        while not step_accepted:
            if h_abs < min_step:
                failed = True
                break
            h = h_abs * direction
            t_new = t + h
            if direction * (t_new - t_bound) > 0:
                t_new = t_bound
            h = t_new - t
            h_abs = abs(h)
            # rk_step
            K[0] = fcur
            for s in range(1, N_STAGES):
                dy = np.dot(K[:s].T, A[s, :s]) * h
                K[s] = f(t + C[s] * h, y + dy)
            y_new = y + h * np.dot(K[:-1].T, B)
            f_new = f(t + h, y_new)
            K[-1] = f_new
            scale = atol + np.maximum(np.abs(y), np.abs(y_new)) * rtol
            error_norm = rms_norm(np.dot(K.T, E) * h / scale)
            if error_norm < 1:
                factor = MAX_FACTOR if error_norm == 0 else min(MAX_FACTOR, SAFETY * error_norm ** error_exponent)
                if step_rejected:
                    factor = min(1, factor)
                h_abs *= factor
                step_accepted = True
            else:
                h_abs *= max(MIN_FACTOR, SAFETY * error_norm ** error_exponent)
                step_rejected = True
        if failed:
            status = -1
            break
        hs.append(h)
        steps += 1
        t, y, fcur = t_new, y_new, f_new
        if direction * (t - t_bound) >= 0:
            status = 0
    return Rk45Result(t, y, nfev, steps, status, hs)


def pf_drift(score_fn: Callable, sde: OUVE, x: torch.Tensor, y: torch.Tensor, t: float) -> torch.Tensor:
    """``rsde.sde(x, y, vec_t)[0]`` with probability_flow=True (sdes.py:113-127, :188-196): everything on fp32 /
    complex64 tensors, ``vec_t = torch.ones(B) * t`` (sampling/__init__.py:122)."""
    vec_t = torch.ones(y.shape[0]) * t
    sde_drift = sde.theta * (y - x)
    sigma = sde.sigma_min * (sde.sigma_max / sde.sigma_min) ** vec_t
    diffusion = sigma * np.sqrt(2 * sde.logsig)
    score = score_fn(x, y, vec_t)
    score_drift = -diffusion[:, None, None, None] ** 2 * score * 0.5
    return sde_drift + score_drift


def ode_sample(score_fn: Callable, y: torch.Tensor, sde: OUVE, eps: float = 0.03, rtol: float = 1e-5,
               atol: float = 1e-5, prior_noise: Optional[torch.Tensor] = None, denoise: bool = False):
    """``get_ode_sampler(sde, score_fn, y, denoise=..., rtol, atol, method='RK45', eps)()`` of
    sampling/__init__.py:72-143 with the prior draw injected.  Returns ``(x c64 [B,1,F,T], nfe)``."""
    if denoise:
        # sampling/__init__.py:99-102 -> predictors.py:60: update_fn() is called without `stepsize`
        raise TypeError("ReverseDiffusionPredictor.update_fn() missing 1 required positional argument: 'stepsize'")
    if prior_noise is None:
        raise ValueError("oracle sampler requires injected noise")
    x = y + prior_noise * sde.std(1.0)                                  # sdes.py:224-229

    def ode_func(t, xf):
        xt = torch.from_numpy(xf.reshape(y.shape)).type(torch.complex64)
        with torch.no_grad():
            d = pf_drift(score_fn, sde, xt, y, t)
        return d.detach().cpu().numpy().reshape((-1,))

    res = rk45_solve(ode_func, 1.0, x.detach().cpu().numpy().reshape((-1,)), eps, rtol=rtol, atol=atol)
    out = torch.tensor(res.y).reshape(y.shape).type(torch.complex64)
    return out, res.nfev
