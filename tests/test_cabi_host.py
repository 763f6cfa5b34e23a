"""Host-only checks of the C-ABI library: it loads, exports every symbol include/sgmse_b200.h declares,
and its architecture walk (weight manifest) equals the reference's state_dict layout.  No GPU needed."""
import os
import re

import numpy as np
import pytest
import torch

from oracle.arch import NetConfig, state_dict_manifest
from sgmse_b200 import _lib, Engine, EngineConfig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    header = open(os.path.join(ROOT, "include", "sgmse_b200.h")).read()
    declared = set(re.findall(r"\b(sgmse_b200_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    for name in declared:
        assert getattr(lib, name) is not None
    assert b"sm_90a" in lib.sgmse_b200_version()


CASES = [
    (NetConfig.ncsnpp(), EngineConfig.ncsnpp_16k()),
    (NetConfig.ncsnpp_48k(), EngineConfig.ncsnpp_48k()),
    (NetConfig.ncsnpp(nf=16, ch_mult=(1, 2, 2), image_size=64, attn_resolutions=(16,)),
     EngineConfig(nf=16, ch_mult=(1, 2, 2), image_size=64, attn_resolutions=(16,), n_fft=126, hop_length=32)),
    (NetConfig.ncsnpp_48k(nf=16, ch_mult=(1, 2, 2), image_size=64),
     EngineConfig.ncsnpp_48k(nf=16, ch_mult=(1, 2, 2), image_size=64, n_fft=126, hop_length=32)),
]


@pytest.mark.parametrize("ncfg,ecfg", CASES)
def test_manifest_equals_reference_state_dict_layout(ncfg, ecfg):
    eng = Engine(ecfg)
    man = eng.manifest()
    ref = [(k, int(np.prod(s))) for k, s in state_dict_manifest(ncfg)]
    assert man == ref
    assert eng.weights_numel() == sum(n for _, n in ref)
    eng.close()


def test_golden_state_dict_is_accepted(golden_dir):
    z = np.load(os.path.join(golden_dir, "ncsnpp_small.npz"))
    sd = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w/")}
    eng = Engine(CASES[2][1])
    blob = eng.flatten_state_dict(sd)
    assert blob.numel() == eng.weights_numel()
    with pytest.raises(KeyError):
        eng.flatten_state_dict({k: v for k, v in list(sd.items())[1:]})
    eng.close()


def test_errors_are_reported_not_thrown():
    lib = _lib.load()
    import ctypes as C
    cfg = EngineConfig(nf=12).to_c()          # nf must be a multiple of 8
    h = C.c_void_p()
    assert lib.sgmse_b200_create(C.byref(cfg), C.byref(h)) != 0
    assert b"nf=12" in lib.sgmse_b200_last_error()
    with pytest.raises(ValueError, match="Predictor with name 'bogus' unknown."):
        Engine(CASES[2][1]).sampler_struct(predictor="bogus")


def test_no_cpu_fallback():
    eng = Engine(CASES[2][1])
    with pytest.raises(RuntimeError, match="no CPU path"):
        eng.score(torch.zeros(1, 1, 64, 64, dtype=torch.complex64), torch.zeros(1, 1, 64, 64, dtype=torch.complex64),
                  torch.ones(1))
    eng.close()


@pytest.mark.parametrize("sampler_type", ["ode", "sde"])
@pytest.mark.parametrize("N,eps", [(50, 1e-4), (7, 1e-4), (30, 1e-3)])
def test_sb_schedule_matches_oracle(sampler_type, N, eps):
    """Host-computed Schroedinger-bridge schedule (engine.cu: make_tables, double precision) against the oracle's fp32
    restatement of sampling/__init__.py:152-231, which tests/test_oracle_golden.py pins to the reference's sampler
    outputs.  The reference evaluates k**(2t) - 1 in fp32, a cancellation that costs ~3e-4 relative at t = 1e-4;
    the weights it feeds stay within 1e-5 of the double-precision values."""
    from oracle import sde as o_sde
    eng = Engine(EngineConfig.ncsnpp_v2(sde="sbve", loss_type="data_prediction", sb_k=2.6, sb_c=0.4))
    ts, std1, rows = eng.sampler_schedule(N=N, kind="sb_" + sampler_type, sb_eps=eps)
    eng.close()
    ref_ts, ref_rows = o_sde.sb_weights(o_sde.SBVE(2.6, 0.4), N, eps, sampler_type)
    assert std1 == 0.0 and rows.shape == (N, 3)
    assert torch.allclose(ts, ref_ts, rtol=2.5e-7, atol=1e-9)
    # the first ODE step divides by sigma_bar(T) = sqrt(eps) = 1e-4: weight_prev and weight_prior_mean are +-2.25e3 and
    # cancel (x_0 = y); their fp32 evaluation in the reference carries a relative error of a few 1e-6
    assert ((rows - ref_rows).abs() / ref_rows.abs().clamp(min=1.0)).max().item() < 1e-5
    assert ((rows[:, 0] + rows[:, 2]) - (ref_rows[:, 0] + ref_rows[:, 2])).abs().max().item() < 6e-4 or sampler_type == "sde"   # 2 ulp of 2.8e3
    if sampler_type == "sde":
        assert rows[-1, 2].item() == 0.0          # weight_z of the last step (sampling/__init__.py:176-179)


# ---- SURVEY.md §8f-4: the RK45 controller of the device ODE sampler, driven by a host callback -----------------
def _ode_case(n=200, seed=0):
    rng = np.random.default_rng(seed)
    M = (rng.standard_normal((n, n)) + 1j * rng.standard_normal((n, n))) * 0.3 / np.sqrt(n)
    b = rng.standard_normal(n) + 1j * rng.standard_normal(n)

    def fun(t, y):                                   # rounded to complex64 like the sampler's drift
        return (-1.5 * y + M @ np.tanh(y.real) + 1j * np.sin(3 * t) * b).astype(np.complex64)

    y0 = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    return fun, y0


@pytest.mark.parametrize("rtol,atol,t_bound", [(1e-5, 1e-5, 0.03), (1e-3, 1e-6, 0.03), (1e-8, 1e-10, 0.5), (1e-5, 1e-5, 2.0),
                                                (1e-5, 1e-5, 1.0)])
def test_rk45_controller_equals_scipy(rtol, atol, t_bound):
    """csrc/rk45.h (what sgmse_b200_ode_sample runs) takes scipy's steps: same nfev, same accepted steps, same state
    up to the summation order of the stage combinations (np.dot vs a plain loop, amplified by the complex64 rounding
    of the right-hand side)."""
    from scipy.integrate import solve_ivp
    from sgmse_b200.engine import rk45_host
    fun, y0 = _ode_case()
    s = solve_ivp(fun, (1.0, t_bound), y0, rtol=rtol, atol=atol, method="RK45")
    y, nfev, st = rk45_host(fun, (1.0, t_bound), y0, rtol=rtol, atol=atol)
    assert (nfev, st["status"]) == (s.nfev, s.status)
    if t_bound != 1.0:
        assert st["steps"] == len(s.t) - 1
    assert np.abs(s.y[:, -1] - y).max() <= 1e-6 * np.abs(y).max()


def test_rk45_controller_rejected_steps_and_failure_modes():
    from scipy.integrate import solve_ivp
    from sgmse_b200.engine import rk45_host

    def stiff(t, y):
        return -2000.0 * (y - np.cos(t)) + 0j

    s = solve_ivp(stiff, (0, 0.5), np.array([0 + 0j]), rtol=1e-4, atol=1e-7, method="RK45")
    y, nfev, st = rk45_host(stiff, (0, 0.5), np.array([0 + 0j]), rtol=1e-4, atol=1e-7)
    assert st["rejected"] > 10 and (nfev, st["steps"], st["status"]) == (s.nfev, len(s.t) - 1, 0)
    assert abs(s.y[0, -1] - y[0]) < 1e-12
    # bounded: a budget of step attempts, and a NaN right-hand side stops instead of spinning (scipy never returns there)
    _, nfev, st = rk45_host(stiff, (0, 0.5), np.array([0 + 0j]), rtol=1e-4, atol=1e-7, max_attempts=7)
    assert st["status"] == -2 and nfev == 2 + 6 * 7
    _, nfev, st = rk45_host(lambda t, y: y * np.nan, (0, 1), np.array([1 + 0j]))
    assert st["status"] == -3 and nfev <= 8
    # empty system and errors through the C-ABI
    y, nfev, st = rk45_host(lambda t, y: y, (0, 1), np.zeros(0, dtype=complex))
    assert y.size == 0 and st["status"] == 0
    with pytest.raises(RuntimeError, match="atol"):
        rk45_host(stiff, (0, 0.5), np.array([0 + 0j]), atol=-1.0)


def test_ode_sampler_host_mirror_errors():
    """Engine.ode_sample mirrors get_ode_sampler's argument behaviour before anything touches the GPU: the default
    denoise=True is the reference's TypeError (predictors.py:60), other integrators are not implemented."""
    eng = Engine(CASES[2][1])
    y = torch.zeros(1, 1, 64, 64, dtype=torch.complex64)
    with pytest.raises(TypeError, match="stepsize"):
        eng.ode_sample(y)
    with pytest.raises(NotImplementedError):
        eng.ode_sample(y, denoise=False, method="RK23")
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        eng.ode_sample(y, denoise=False)
    eng.close()


def test_plain_c_client(tmp_path):
    """include/sgmse_b200.h is C: a gcc -std=c99 program (tests/c/cabi_host.c) links libsgmse_b200.so and drives the
    host-only entry points -- manifest, schedule, RK45 controller with a C callback -- with no Python or C++ around it."""
    import shutil
    import subprocess
    from sgmse_b200 import build
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    _lib.load()
    lib = build.lib_path()
    exe = str(tmp_path / "cabi_host")
    cmd = ["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "c", "cabi_host.c"), "-o", exe, lib, "-lm", "-Wl,-rpath," + os.path.dirname(lib)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "cabi_host ok" in r.stdout, r.stdout + r.stderr


def test_shape_contract_is_enforced_on_the_host():
    """The reference's shape contract (SURVEY.md §8b): F and T multiples of 2^(levels-1) (6 down-samplings: 64), and for
    'ncsnpp' F == image_size, or the build-time attention placement disagrees with the run-time trigger (ncsnpp.py:84,308)
    -- checked by the host-side walk of the launch sequence, no GPU involved."""
    eng = Engine(CASES[0][1])                                    # full-size 16 kHz NCSN++
    assert eng.workspace_bytes(1, 256, 512) > 1 << 30
    assert eng.workspace_bytes(2, 256, 512) > 1.9 * eng.workspace_bytes(1, 256, 512)
    with pytest.raises(RuntimeError, match="multiples of 64"):
        eng.workspace_bytes(1, 256, 500)                         # pad_spec (util/other.py:76-90) exists for this
    with pytest.raises(RuntimeError, match="image_size"):
        eng.workspace_bytes(1, 128, 512)
    with pytest.raises(RuntimeError, match="bad argument"):
        eng.workspace_bytes(0, 256, 512)                         # empty batch
    assert eng.padded_frames(64000) == 512 and eng.padded_frames(63 * 128) == 64 and eng.padded_frames(64 * 128) == 128
    eng.close()
    eng48 = Engine(CASES[1][1])                                  # ncsnpp_48k: attention only in the bottleneck, any F % 64 == 0
    assert eng48.workspace_bytes(1, 768, 512) > eng48.workspace_bytes(1, 256, 512) > 0
    eng48.close()
    # sampler settings the reference's registries reject
    lib = _lib.load()
    s = Engine(CASES[2][1]).sampler_struct()
    s.predictor = 7
    import ctypes as C
    assert lib.sgmse_b200_noise_draws(C.byref(s)) >= 0           # counting draws is host-only
    with pytest.raises(ValueError, match="Corrector with name 'x' unknown."):
        Engine(CASES[2][1]).sampler_struct(corrector="x")


def test_pdl_twin_library_is_opt_in():
    """Programmatic dependent launch is compiled into a SECOND library only (sgmse_b200/build.py --pdl, DESIGN.md §10): the
    default library refuses `pdl=1` (its kernels carry no griddepcontrol.wait, so a PDL launch would race), the twin exports
    the same C-ABI and accepts it.  Host-only: the option touches no CUDA state on an engine that has captured nothing."""
    import ctypes as C
    from sgmse_b200 import build
    eng = Engine(CASES[2][1])
    assert eng.counter("pdl_compiled") == 0 and eng.counter("pdl") == 0
    with pytest.raises(RuntimeError, match="SGMSE_B200_PDL"):
        eng.set_option("pdl", 1)
    eng.set_option("pdl", 0)                                  # switching it off is always legal
    eng.close()
    twin = C.CDLL(build.build(pdl=True))
    for name, (res, args) in _lib.SYMBOLS.items():
        fn = getattr(twin, name)
        fn.restype, fn.argtypes = res, args
    cfg = CASES[2][1].to_c()
    h = C.c_void_p()
    assert twin.sgmse_b200_create(C.byref(cfg), C.byref(h)) == 0
    assert twin.sgmse_b200_get_counter(h, b"pdl_compiled") == 1
    assert twin.sgmse_b200_set_option(h, b"pdl", 1) == 0 and twin.sgmse_b200_get_counter(h, b"pdl") == 1
    assert twin.sgmse_b200_set_option(h, b"pdl", 0) == 0
    twin.sgmse_b200_destroy(h)


def test_every_ab_switch_is_a_known_option():
    """The A/B switches named in kernels.h / DESIGN.md are accepted by sgmse_b200_set_option (value 0 = the verified default),
    anything else is reported as an error.  Host-only: none of these touches CUDA state on an engine that has run nothing."""
    eng = Engine(CASES[2][1])
    for key in ("tc_variant", "attn_variant", "fir_variant", "inconv_variant",
                "outconv_variant", "combine_variant", "tc1_narrow", "gn_self", "gnfin_variant", "pdl", "record_taps", "use_graphs"):
        eng.set_option(key, 0)
    eng.set_option("max_graphs", 16)
    eng.set_option("lanes", 1)
    with pytest.raises(RuntimeError, match="unknown option"):
        eng.set_option("no_such_switch", 1)
    with pytest.raises(RuntimeError, match="max_graphs"):
        eng.set_option("max_graphs", 0)
    eng.close()


def test_kernel_selection_is_per_engine_and_the_product_library_has_no_lab_kernels():
    """Options are engine state (host-only calls here): unknown convolution variants and programmatic dependent
    launch are refused by the product library, a selection made on one engine is invisible to another."""
    from sgmse_b200 import Engine, EngineConfig
    a, b = Engine(EngineConfig(max_batch=1)), Engine(EngineConfig(max_batch=1))
    for v in (1, 2, 3, 4, 6, 9, 10):
        with pytest.raises(RuntimeError, match="tc_variant"):
            a.set_option("tc_variant", v)
    if a.counter("pdl_compiled") == 0:
        with pytest.raises(RuntimeError, match="SGMSE_B200_PDL"):
            a.set_option("pdl", 1)
    a.set_option("tc_variant", 5)
    a.set_option("fir_variant", 1)
    with pytest.raises(RuntimeError, match="unknown option"):
        b.set_option("no_such_option", 1)
    assert a.counter("pdl") == 0 and b.counter("pdl") == 0
    a.close()
    b.close()
