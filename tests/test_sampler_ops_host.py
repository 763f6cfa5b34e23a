"""Host checks of tests/test_gpu_sampler_ops.py: the shim builds for sm_90a, the numpy Philox4x32-10 the GPU tests take as
the reference is the published generator (Random123 known-answer vectors) and CUDA's own (curand_Philox4x32_10 compiled
for the host), its mutations are visible, and the scipy harness of the device-ODE test sees stage times and rejects steps
at the tight tolerance.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import test_gpu_sampler_ops as T
from sgmse_b200 import build as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CURAND_SRC = os.path.join(ROOT, "tests", "c", "philox_curand_host.cu")


def test_shim_compiles_and_links_for_sm90a(tmp_path):
    ops = T.SamplerOps(T.build_shim(str(tmp_path), T.SHIM_SRC))
    for name in T.SIGNATURES:
        assert hasattr(ops.lib, name)
    assert ops.lib.samp_ode_norm_blocks() == T.NORM_BLOCKS
    with pytest.raises(RuntimeError, match="ode groups: 1 .. kOdeSysPerLaunch systems"):
        ops._check(ops.lib.samp_ode_combine_groups(None, 0, None, None, None, None, None, None, None, None))


# Random123 kat_vectors (philox4x32_10): counter, key -> output
KAT = [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


def numpy_philox(ctr, key, **kw):
    return [int(v) for v in T.philox4x32_10([np.uint32(c) for c in ctr], [np.uint32(k) for k in key], **kw)]


@pytest.mark.parametrize("ctr, key, want", KAT)
def test_numpy_philox_known_answers(ctr, key, want):
    assert tuple(numpy_philox(ctr, key)) == want
    # one round constant changed: the vector no longer matches
    assert tuple(numpy_philox(ctr, key, M=(T.PHILOX_M[0] + 2, T.PHILOX_M[1]))) != want
    assert tuple(numpy_philox(ctr, key, W=(T.PHILOX_W[0], T.PHILOX_W[1] ^ 1))) != want


@pytest.fixture(scope="module")
def curand_philox(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("curand_philox") / "libphilox_curand_host.so")
    r = subprocess.run([B.NVCC, *B.ARCH, "-Xcompiler", "-fPIC", "-shared", "-o", so, CURAND_SRC], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lib = C.CDLL(so, mode=os.RTLD_LOCAL)
    lib.curand_philox_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong]
    lib.curand_philox_batch.restype = None

    def run(ctr, key):
        ctr, key = np.ascontiguousarray(ctr, np.uint32), np.ascontiguousarray(key, np.uint32)
        out = np.zeros_like(ctr)
        lib.curand_philox_batch(ctr.ctypes.data, key.ctypes.data, out.ctypes.data, len(ctr))
        return out
    return run


def test_curand_philox_known_answers(curand_philox):
    for ctr, key, want in KAT:
        assert tuple(int(v) for v in curand_philox([ctr], [key])[0]) == want


def test_numpy_philox_equals_curand_on_random_pairs(curand_philox):
    g = np.random.default_rng(2024)
    ctr = g.integers(0, 2 ** 32, (10 ** 4, 4), dtype=np.uint64).astype(np.uint32)
    key = g.integers(0, 2 ** 32, (10 ** 4, 2), dtype=np.uint64).astype(np.uint32)
    want = curand_philox(ctr, key)
    got = np.stack(T.philox4x32_10(list(ctr.T), list(key.T)), 1)
    assert np.array_equal(got, want)


def test_complex_normal_reference_and_mutations():
    """The reference z has unit complex variance and every Philox mutation of the GPU test moves it far past its bound."""
    N, HW = 2, 4096
    z, b, _ = T.noise_ref(N, HW, 0x0123456789ABCDEF, 5, 2)
    assert abs((z ** 2).sum(-1).mean() - 1) < 0.05 and b.max() < 1e-6
    for m in T.PHILOX_MUTATIONS:
        zm = T.noise_ref(N, HW, 0x0123456789ABCDEF, 5, 2, m)[0]
        assert (np.abs(zm - z) / b).max() > 1e4, m


def test_fma32_rounds_once():
    g = np.random.default_rng(3)
    a, b, c = (g.standard_normal(10 ** 5).astype(np.float32) for _ in range(3))
    got = T.fma32(a, b, c)
    # exact reference with Python integers scaled to a common exponent (fractions are exact)
    from fractions import Fraction
    for i in range(0, 10 ** 5, 997):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        r = got[i]
        lo, hi = np.nextafter(r, np.float32(-np.inf)), np.nextafter(r, np.float32(np.inf))
        assert abs(Fraction(float(r)) - exact) <= min(abs(Fraction(float(lo)) - exact), abs(Fraction(float(hi)) - exact))
    # (1 + 2^-12) 2^-24 (1 - 2^-12 + 2^-24) + 1 = 1 + 2^-24 + 2^-60: a float64 sum drops 2^-60 and lands on the fp32
    # midpoint, which rounds to even (1); the single rounding gives 1 + 2^-23
    a1, b1, one = np.float32(1 + 2.0 ** -12), np.float32(2.0 ** -24 * (1 - 2.0 ** -12 + 2.0 ** -24)), np.float32(1)
    assert np.float32(np.float64(a1) * np.float64(b1) + 1.0) == one
    assert T.fma32(a1, b1, one) == np.nextafter(one, np.float32(2))


@pytest.mark.parametrize("case", T.ODE_CASES, ids=[c.name for c in T.ODE_CASES])
def test_scipy_harness_sees_stage_times(case):
    """The harness of test_device_ode_solve_matches_scipy on the CPU, at the GPU test's size: the stage-time mutation
    changes nfev or misses the state bound by 10x."""
    m = T.ODE_MODEL[case.kind]
    Y, Z = T.ode_inputs()
    b = np.complex64(complex(*case.bias))
    ref = T.scipy_ode(m, Y.numpy(), Z.numpy(), b, case.tol, case.tol, 0.03)
    mut = T.scipy_ode(m, Y.numpy(), Z.numpy(), b, case.tol, case.tol, 0.03, stage_at_step_start=True)
    bound = T.ode_state_bound(m, ref)
    err = float(np.abs(mut.x - ref.x).max())
    print(f"{case.name}: scipy nfev {ref.nfev}, accepted {ref.accepted}, rejected {ref.rejected}, status {ref.status}, "
          f"state bound {bound:.3g}; stage times at the step start: nfev {mut.nfev}, state {err / bound:.3g} x the bound")
    assert ref.status == 0 and mut.status == 0
    assert mut.nfev != ref.nfev or err >= 10 * bound
    if case.tol <= 1e-6:
        assert ref.rejected > 0
