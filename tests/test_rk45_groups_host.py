"""The lockstep driver of the ODE sampler's independent systems (csrc/rk45.h: solve_groups) on a host right-hand side,
and the ODE path of the batched file service with a stand-in engine.  No GPU."""
import numpy as np
import pytest
import torch

from sgmse_b200.engine import rk45_host, rk45_host_groups
from sgmse_b200.service import BatchedEnhancer

from test_service_host import FakeEngine


def _stiff(t, y):
    return -2000.0 * (y - np.cos(t)) + 0j


def _systems():
    """(fun, y0, rtol, atol-independent) per system: linear decays with rates over 10^3, an oscillator, the stiff case."""
    rng = np.random.default_rng(1)
    funs = []
    for rate in (0.5, 5.0, 50.0, 500.0):
        funs.append(lambda t, y, r=rate: (-r * y).astype(np.complex64).astype(np.complex128))
    M = (rng.standard_normal((6, 6)) + 1j * rng.standard_normal((6, 6))) * 0.5
    funs.append(lambda t, y: (M @ np.tanh(y.real) + 1j * np.sin(3 * t) - 0.3 * y).astype(np.complex64).astype(np.complex128))
    funs.append(_stiff)
    y0s = [rng.standard_normal(3) + 1j * rng.standard_normal(3) for _ in range(4)]
    y0s.append(rng.standard_normal(6) + 1j * rng.standard_normal(6))
    y0s.append(np.array([0 + 0j]))
    return funs, y0s


def _dispatch(funs, log=None):
    def fun(ids, ts, ys):
        if log is not None:
            log.append(list(ids))
        return [funs[i](t, y) for i, t, y in zip(ids, ts, ys)]
    return fun


@pytest.mark.parametrize("slots", [6, 2, 1])
def test_each_system_equals_its_solo_solve_and_scipy(slots):
    from scipy.integrate import solve_ivp
    funs, y0s = _systems()
    t_span, rtol, atol = (0.0, 0.5), 1e-4, 1e-7
    log = []
    ys, nfev, st, rounds = rk45_host_groups(_dispatch(funs, log), t_span, y0s, slots=slots, rtol=rtol, atol=atol)
    for i, (f, y0) in enumerate(zip(funs, y0s)):
        y1, n1, s1 = rk45_host(f, t_span, y0, rtol=rtol, atol=atol)
        assert np.array_equal(ys[i], y1), i                         # bit for bit
        assert (nfev[i], st[i]) == (n1, s1), i
        s = solve_ivp(f, t_span, y0, rtol=rtol, atol=atol, method="RK45")
        assert (nfev[i], st[i]["steps"], st[i]["status"]) == (s.nfev, len(s.t) - 1, 0), i
    assert st[5]["rejected"] > 10                                   # the stiff system rejects many steps
    assert len({n for n in nfev}) >= 3
    # the callback sees only systems in flight, each at most once per round, never more than `slots`
    assert all(len(c) == len(set(c)) and len(c) <= slots for c in log)
    if slots >= len(funs):
        # one request per system and round: rounds = the largest request count (evaluations + norms)
        assert rounds == max(_requests(n, s) for n, s in zip(nfev, st))
        assert rounds >= max(nfev)


def _requests(nfev, st):
    """Requests of a successful solve: its evaluations, the three norms of select_initial_step, one norm per attempt."""
    return nfev + 3 + st["steps"] + st["rejected"]


def test_refill_starts_the_next_system_in_the_round_after_one_finishes():
    funs = [lambda t, y, r=r: -r * y for r in (1.0, 100.0, 3.0)]
    y0s = [np.array([1 + 0j])] * 3
    log = []
    _, nfev, st, rounds = rk45_host_groups(_dispatch(funs, log), (0.0, 1.0), y0s, slots=2, rtol=1e-6, atol=1e-9)
    assert all(s["status"] == 0 for s in st)
    req = [_requests(n, s) for n, s in zip(nfev, st)]
    assert req[0] + req[2] < req[1]
    assert log[0] == [0, 1] and [sum(1 for c in log if i in c) for i in range(3)] == nfev
    # system 2 takes system 0's slot: never in flight together, and system 0's last request is followed directly
    # by system 2's first (rounds would exceed max(req[1], req[0] + req[2]) with an idle round in between)
    assert not any(0 in c and 2 in c for c in log)
    assert rounds == max(req[1], req[0] + req[2])
    _, nfev3, st3, rounds3 = rk45_host_groups(_dispatch(funs), (0.0, 1.0), y0s, slots=3, rtol=1e-6, atol=1e-9)
    assert (nfev3, st3) == (nfev, st) and rounds3 == max(req)


def test_failure_isolation():
    funs, y0s = _systems()
    funs = funs[:3] + [lambda t, y: y * np.nan] + funs[5:]
    y0s = y0s[:3] + [np.array([1 + 0j])] + y0s[5:]
    ys, nfev, st, _ = rk45_host_groups(_dispatch(funs), (0.0, 0.5), y0s, slots=3, rtol=1e-4, atol=1e-7)
    assert st[3]["status"] == -3 and nfev[3] <= 8
    for i in (0, 1, 2, 4):
        y1, n1, s1 = rk45_host(funs[i], (0.0, 0.5), y0s[i], rtol=1e-4, atol=1e-7)
        assert np.array_equal(ys[i], y1) and (nfev[i], st[i]) == (n1, s1)
    # a budget of step attempts that only the stiff system exhausts
    ys, nfev, st, _ = rk45_host_groups(_dispatch(funs[:3] + funs[4:]), (0.0, 0.5), y0s[:3] + y0s[4:], rtol=1e-4, atol=1e-7,
                                       max_attempts=30)
    assert st[3]["status"] == -2 and nfev[3] == 2 + 6 * 30
    for i in range(3):
        y1, n1, s1 = rk45_host(funs[i], (0.0, 0.5), y0s[i], rtol=1e-4, atol=1e-7, max_attempts=30)
        assert s1["status"] == 0 and np.array_equal(ys[i], y1) and nfev[i] == n1
    with pytest.raises(RuntimeError, match="atol"):
        rk45_host_groups(_dispatch(funs), (0, 0.5), y0s, atol=-1.0)


class FakeOdeEngine(FakeEngine):
    def ode_sample_groups(self, Y, group=1, seed=0, utt_offset=0, **kw):
        self.calls.append(("ode_sample_groups", tuple(Y.shape), group, seed, utt_offset, tuple(sorted(kw.items()))))
        return Y + utt_offset, [100] * Y.shape[0]


def test_batched_enhancer_ode_buckets_and_ids():
    eng = FakeOdeEngine(max_batch=2)
    lengths = [8000, 64000, 8100, 7000, 64100]
    waves = [torch.full((L,), 0.1 * (i + 1)) for i, L in enumerate(lengths)]
    outs, ids = BatchedEnhancer(eng, device="cpu")(waves, seed=5, utt_base=10, sampler_type="ode", denoise=False, rtol=1e-3)
    pc = BatchedEnhancer(FakeOdeEngine(max_batch=2), device="cpu")
    _, pc_ids = pc(waves, seed=5, utt_base=10)
    assert ids == pc_ids == [10, 13, 11, 12, 14]                   # the PC sampler's ids
    calls = [c for c in eng.calls if c[0] == "ode_sample_groups"]
    # one call per padded-length bucket, however many clips it holds, one system per clip
    assert [(c[1][0], c[2], c[3], c[4]) for c in calls] == [(3, 1, 5, 10), (2, 1, 5, 13)]
    assert all(dict(c[5]) == {"denoise": False, "rtol": 1e-3} for c in calls)
    for i, w in enumerate(waves):
        assert outs[i].shape == w.shape
        bucket_offset = 10 if lengths[i] < 10000 else 13              # the fake adds its call's utt_offset
        assert torch.allclose(outs[i], (w.sum() + bucket_offset) * w.abs().max() * torch.ones_like(w))
    with pytest.raises(TypeError):
        BatchedEnhancer(eng, device="cpu")(waves, sampler_type="ode")
    with pytest.raises(ValueError):
        BatchedEnhancer(eng, device="cpu")(waves, sampler_type="sde")
    assert not any(c[0] == "pc_sample" for c in eng.calls)
    assert any(c[0] == "pc_sample" for c in pc.engine.calls)        # the default is still the PC sampler
    assert not any(c[0] == "ode_sample_groups" for c in pc.engine.calls)


def test_batched_enhancer_ode_prior_noise_per_clip():
    eng = FakeOdeEngine()
    waves = [torch.ones(8000), torch.ones(7000)]
    BatchedEnhancer(eng, device="cpu")(waves, sampler_type="ode", denoise=False,
                                       noise_for=lambda i, tp: torch.full((1, 1, 1, 4, tp), float(i), dtype=torch.complex64))
    (call,) = [c for c in eng.calls if c[0] == "ode_sample_groups"]
    noise = dict(call[5])["prior_noise"]
    assert noise.shape == (2, 1, 4, 64) and noise[0].abs().max() == 0 and (noise[1] == 1).all()
