"""Independent probability-flow ODE systems solved side by side (Engine.ode_sample_groups): every system must equal
the single-system solve of its utterances alone (Engine.ode_sample), bit for bit -- the state, nfe, accepted and
rejected steps and status -- whatever else is in flight, in every mode and backbone.  Run on a GPU host."""
import os

import pytest
import torch

from oracle import weights as o_w
from oracle.arch import NetConfig
from sgmse_b200 import BatchedEnhancer, Engine, EngineConfig

from test_gpu_parity import MID_E, MID_N
from test_gpu_zz_next_rows import SMALL_E, V2_ODE_PRECOND, load_golden

pytestmark = pytest.mark.gpu

LEVELS = (1.0, 0.05, 3.0, 0.3, 10.0)          # input levels of the 5 utterances: different step sequences and nfe
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KW = dict(rtol=1e-2, atol=1e-2, denoise=False, seed=5)


def _inputs(F, T, seed=0):
    g = torch.Generator().manual_seed(seed)
    Y = torch.complex(torch.randn(len(LEVELS), 1, F, T, generator=g), torch.randn(len(LEVELS), 1, F, T, generator=g))
    return (0.5 * Y * torch.tensor(LEVELS).reshape(-1, 1, 1, 1)).to(torch.complex64).cuda()


def _solo(eng, Y, group=1, **kw):
    """ode_sample of each system alone: (outputs, nfe list, stats list)"""
    outs, nfes, sts = [], [], []
    for b0 in range(0, Y.shape[0], group):
        x, n, st = eng.ode_sample(Y[b0:b0 + group], utt_offset=b0, return_stats=True, **{**KW, **kw})
        outs.append(x)
        nfes.append(n)
        sts.append(st)
    return outs, nfes, sts


def _check(eng, Y, solo, group=1, **kw):
    x, nfes, sts = eng.ode_sample_groups(Y, group=group, return_stats=True, **{**KW, **kw})
    outs, n1, s1 = solo
    assert nfes == n1
    assert [{k: s[k] for k in ("steps", "rejected", "status")} for s in sts] == s1
    for i, o in enumerate(outs):
        assert torch.equal(x[i * group:i * group + o.shape[0]], o), f"system {i}"
    return sts[0]


def _engine(kind, mode, **kw):
    if kind == "ncsnpp_small":
        _, sd = load_golden(GOLDEN, "ncsnpp_small")
        eng = Engine(EngineConfig(attn_resolutions=(16,), mode=mode, **SMALL_E, **kw))
    elif kind == "ncsnpp48k_small":
        _, sd = load_golden(GOLDEN, "ncsnpp48k_small")
        eng = Engine(EngineConfig.ncsnpp_48k(mode=mode, theta=1.5, sigma_min=0.05, sigma_max=0.5, spec_factor=0.15,
                                             spec_abs_exponent=0.5, **SMALL_E, **kw))
    else:
        sd = o_w.make_state_dict(MID_N, seed=0)
        eng = Engine(EngineConfig(mode=mode, **MID_E, **kw))
    eng.load_state_dict(sd)
    return eng


@pytest.mark.parametrize("kind,mode", [("ncsnpp_small", "fp32"), ("ncsnpp48k_small", "fp32"), ("mid", "fp16_tc"),
                                       ("mid", "tf32_tc")])
def test_each_clip_equals_its_solo_solve(kind, mode):
    Y = _inputs(64, 64)
    ref = _engine(kind, mode, max_batch=2)
    solo = _solo(ref, Y)
    assert len(set(solo[1])) >= 2, solo[1]                          # the in-flight set changes during the solve
    solo2 = _solo(ref, Y, group=2)
    ref.close()
    for mb in (1, 2, 3, 8):
        for graphs in (True, False):
            eng = _engine(kind, mode, max_batch=mb, use_graphs=graphs)
            st = _check(eng, Y, solo)
            assert st["forwards"] <= st["rounds"] and st["rows"] == sum(solo[1])
            if mode != "fp32":
                assert eng.counter("tc_convs_last_forward") > 0
            if mb >= 2 and graphs:
                _check(eng, Y, solo2, group=2)
            eng.close()


@pytest.mark.parametrize("tag", list(V2_ODE_PRECOND))
def test_v2_score_models(tag):
    _, sd = load_golden(GOLDEN, "ncsnpp_v2_small")
    Y = _inputs(64, 64, seed=1)
    engs = [Engine(EngineConfig.ncsnpp_v2(attn_resolutions=(16,), mode="fp32", sde="ouve", max_batch=mb, **SMALL_E,
                                          **V2_ODE_PRECOND[tag])) for mb in (2, 3)]
    for e in engs:
        e.load_state_dict(sd)
    solo = _solo(engs[0], Y)
    assert len(set(solo[1])) >= 2
    for e in engs:
        _check(e, Y, solo)
    _check(engs[1], Y, _solo(engs[0], Y, group=2), group=2)
    with pytest.raises(RuntimeError, match="group"):
        engs[0].ode_sample_groups(Y, group=3, **KW)
    with pytest.raises(TypeError, match="stepsize"):
        engs[0].ode_sample_groups(Y)
    with pytest.raises(NotImplementedError):
        engs[0].ode_sample_groups(Y, method="RK23", **KW)
    for e in engs:
        e.close()


def test_batched_enhancer_ode_equals_enhance_ode_per_clip():
    eng = _engine("ncsnpp_small", "fp32", max_batch=3)
    g = torch.Generator().manual_seed(31)
    lengths = [2000, 4200, 1900, 2047, 4100, 1950]
    waves = [0.1 * torch.randn(L, generator=g) for L in lengths]
    kw = dict(rtol=1e-2, atol=1e-2, denoise=False)
    outs, ids = BatchedEnhancer(eng)(waves, seed=9, sampler_type="ode", **kw)
    assert sorted(ids) == list(range(len(waves)))
    for w, o, i in zip(waves, outs, ids):
        alone, _ = eng.enhance_ode(w[None].cuda(), seed=9, utt_offset=i, **kw)
        assert o.shape == w.shape and torch.equal(o, alone[0])
    eng.close()


def test_failure_isolation_max_attempts():
    eng = _engine("ncsnpp_small", "fp32", max_batch=3)
    Y = _inputs(64, 64)
    attempts = [s["steps"] + s["rejected"] for s in _solo(eng, Y)[2]]
    budget = max(attempts) - 1                                      # exhausted by the longest solves only
    assert min(attempts) <= budget, attempts
    solo = _solo(eng, Y, max_attempts=budget)
    status = [s["status"] for s in solo[2]]
    assert -2 in status and 0 in status, (attempts, budget)
    _check(eng, Y, solo, max_attempts=budget)
    eng.close()


def test_workspace_poison_keeps_the_bits():
    eng = _engine("mid", "fp16_tc", max_batch=3)
    Y = _inputs(64, 64)
    solo = _solo(eng, Y)
    eng.set_option("workspace_poison", 1)
    _check(eng, Y, solo)
    eng.close()


def test_full_size_fp16_tc():
    sd = o_w.make_state_dict(NetConfig.ncsnpp(), seed=0)
    eng = Engine(EngineConfig.ncsnpp_16k(mode="fp16_tc", max_batch=4))
    eng.load_state_dict(sd)
    g = torch.Generator().manual_seed(3)
    wav = torch.stack([lv * 0.1 * torch.randn(16000, generator=g) for lv in (1.0, 0.3, 2.0, 0.1)]).cuda()
    Y, _ = eng.analysis(wav)
    kw = dict(rtol=5e-2, atol=5e-2)
    solo = _solo(eng, Y, **kw)
    st = _check(eng, Y, solo, **kw)
    assert eng.counter("tc_convs_last_forward") > 0
    print(f"full size: nfe {solo[1]}, rounds {st['rounds']}, forwards {st['forwards']}, syncs {st['syncs']}")
    eng.close()
