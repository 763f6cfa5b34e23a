"""Op-level tests of the sampler and probability-flow ODE kernels (misc.cu, ode.cu): the time embedding, the predictor /
corrector updates and the Philox noise they draw, the prior, the Langevin step size, the preconditioned-model epilogues,
and the ODE vector kernels.  Each is compared with a float64 reference of the same formula, computed from the exact fp32
inputs the kernel read, and the device RK45 solve is compared with scipy through the real engine.

Network-level tests see these kernels only through a rel-L2 norm, and the ODE sampler only through nfe +-6: a wrong Philox
round constant, a swapped key word, a stage evaluated at the wrong time or a dropped norm partial would pass them.  Here
every output element has its own bound, derived from the kernel's rounding model (in the comment beside it), and each
kernel prints its worst err/bound and its weakest mutation ratio.  The mutation controls compare the same kernel output
with a deliberately wrong reference and require a miss by at least 10x the bound.

tests/c/sampler_ops.cu is an extern "C" shim over the product launchers, linked against the library objects like
tests/c/kernel_ops.cu.  The reference Philox4x32-10 is numpy; tests/test_sampler_ops_host.py pins it to the Random123
known-answer vectors and to CUDA's own curand_Philox4x32_10.
"""
import collections
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from test_gpu_kernel_ops import PAD, U32, ULP32, Guarded, build_shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM_SRC = os.path.join(ROOT, "tests", "c", "sampler_ops.cu")

U64 = 2.0 ** -53            # fp64 unit roundoff
NORM_BLOCKS = 528           # kOdeNormBlocks
LV_BLOCKS = 64              # misc.cu: the Langevin norm's blocks per sample
TWO_M32 = np.float32(2.3283064365386963e-10)

_I, _P, _F, _D, _L = C.c_int, C.c_void_p, C.c_float, C.c_double, C.c_longlong
_FP, _DP = C.POINTER(C.c_float), C.POINTER(C.c_double)
_OL = [_FP, _FP, _I, _I]          # OutLayer: w[8], b[2], scale_after, scale_by_sigma
SIGNATURES = {
    "samp_temb": [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _P, _I, _P, _P],
    "samp_pc_update": [_P, _P, _P, _I, _I, _I, *_OL, _P, _F, _P, _P, _P, _I, _P],
    "samp_affine_update": [_P, _P, _P, _I, _I, _I, *_OL, _P, _P, _P, _I, _I, _P],
    "samp_prior": [_P, _P, _I, _I, _I, _F, _P, _P, _I],
    "samp_langevin_coef": [_P, _P, _I, _I, _I, *_OL, _F, _P, _P, _I, _F, _P, _P],
    "samp_precond_out": [_P, _P, _P, _I, _I, _I, *_OL, _P, _P, _P],
    "samp_out_layer": [_P, _P, _I, _I, _I, *_OL, _P, _P, _I],
    "samp_pack_state": [_P, _P, _P, _I, _I, _I, _P],
    "samp_pack_state_scaled": [_P, _P, _P, _P, _I, _I, _I, _P],
    "samp_ode_combine": [_P, _P, _P, _I, _DP, _D, _L, _P, _P],
    "samp_ode_norm": [_P, _I, _P, _P, _P, _DP, _D, _D, _D, _L, _P],
    "samp_ode_drift": [_P, _P, _P, _I, _I, _I, *_OL, _F, _F, _F, _P],
    "samp_ode_drift_affine": [_P, _P, _P, _I, _I, _I, *_OL, _F, _F, _F, _P],
    "samp_ode_init": [_P, _P, _L, _P],
    "samp_ode_finish": [_P, _P, _L, _P],
    "samp_ode_combine_groups": [_P, _I, _P, _P, _P, _P, _DP, _DP, C.POINTER(_L), C.POINTER(_I)],
    "samp_ode_norm_groups": [_P, _I, _P, _P, _P, _DP, _DP, C.POINTER(_L), C.POINTER(_I), _D, _D, _P],
    "samp_ode_rows_pack": [_P, _I, _P, _P, _FP, _FP, _L, _P, _P, _P, _P],
    "samp_ode_rows_drift": [_P, _I, _P, _FP, _FP, _L, _P, _P, *_OL, _F, _I],
    "samp_logf": [_P, _P, _P, _I],         # the device logf the time embedding applies (not a product launcher)
}
LAUNCHERS = {n.replace("samp_", "launch_") for n in SIGNATURES if n != "samp_logf"}


def _stream():
    return torch.cuda.current_stream().cuda_stream if torch.cuda.is_available() else None


def _ptr(t):
    return None if t is None else t.data_ptr()


def _ptrs(ts, n=None):
    ts = list(ts) + [None] * ((n or len(ts)) - len(ts))
    return (C.c_void_p * len(ts))(*[_ptr(t) for t in ts])


def _floats(v):
    return (C.c_float * len(v))(*[float(x) for x in v])


def _doubles(v):
    return (C.c_double * len(v))(*[float(x) for x in v])


OutLayer = collections.namedtuple("OutLayer", "w b scale_after scale_by_sigma")   # w: 8 fp32 (row-major [2][4]), b: 2 fp32


def _ol(ol):
    return [_floats(ol.w), _floats(ol.b), int(ol.scale_after), int(ol.scale_by_sigma)]


class SamplerOps:
    def __init__(self, path):
        self.lib = C.CDLL(path, mode=os.RTLD_LOCAL)
        for name, args in SIGNATURES.items():
            fn = getattr(self.lib, name)
            fn.argtypes, fn.restype = args, C.c_int
        self.lib.samp_last_error.restype = C.c_char_p
        self.lib.samp_ode_norm_blocks.restype = C.c_int

    def _check(self, code):
        if code != 0:
            raise RuntimeError(f"sampler_ops: {self.lib.samp_last_error().decode()} (code {code})")

    def __getattr__(self, name):
        fn = getattr(self.lib, "samp_" + name)
        return lambda *a: self._check(fn(_stream(), *a))


@pytest.fixture(scope="module")
def samp(tmp_path_factory):
    return SamplerOps(build_shim(str(tmp_path_factory.mktemp("sampler_ops")), SHIM_SRC))


# ------------------------------------------------------------------------------------------------
# numpy Philox4x32-10 (Salmon et al., SC'11; the Random123 / curand constants) and the kernel's complex normal
# ------------------------------------------------------------------------------------------------
PHILOX_M = (0xD2511F53, 0xCD9E8D57)
PHILOX_W = (0x9E3779B9, 0xBB67AE85)
MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key, M=PHILOX_M, W=PHILOX_W):
    """ctr: 4 uint32 arrays (broadcastable), key: 2 -> 4 uint32 arrays."""
    c = [np.asarray(v, dtype=np.uint64) & MASK32 for v in ctr]
    k = [np.asarray(v, dtype=np.uint64) & MASK32 for v in key]
    m0, m1, w0, w1 = (np.uint64(v) for v in (*M, *W))
    for _ in range(10):
        p0, p1 = m0 * c[0], m1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k[0], p1 & MASK32, (p0 >> np.uint64(32)) ^ c[3] ^ k[1], p0 & MASK32]
        k = [(k[0] + w0) & MASK32, (k[1] + w1) & MASK32]
    return [v.astype(np.uint32) for v in c]


def philox_words(seed, utt, draw, pix, **kw):
    """The kernel's generator call (misc.cu: complex_normal): counter (pix, draw, utt, 0x5347), key (seed lo, seed hi)."""
    seed = int(seed)
    return philox4x32_10((pix, draw, utt, 0x5347), (seed & 0xFFFFFFFF, seed >> 32), **kw)


def ulp32(v):
    """Spacing of fp32 at magnitude v >= 0 (the subnormal spacing below 2^-126)."""
    v = np.asarray(v, dtype=np.float64)
    return np.exp2(np.floor(np.log2(np.maximum(v, 2.0 ** -126))) - 23)


def complex_normal_ref(seed, utt, draw, pix, **kw):
    """(re, im, bound) float64 of the kernel's Box-Muller z: the integer-to-uniform steps in float32 exactly as the kernel
    does them ((float)r + 1.0f, * 2^-32: two correctly rounded fp32 operations, and 2.0f * u2 exact), the rest in float64.
    Error model (CUDA C++ Programming Guide, single-precision mathematical functions): logf <= 1 ulp, sqrtf correctly
    rounded, sinpif / cospif <= 1 ulp each, then the product rad * c rounds once."""
    r = philox_words(seed, utt, draw, pix, **kw)
    u1 = (r[0].astype(np.float64).astype(np.float32) + np.float32(1.0)) * TWO_M32
    u2 = r[1].astype(np.float64).astype(np.float32) * TWO_M32
    L = -np.log(u1.astype(np.float64))
    rad = np.sqrt(L)
    a = np.pi * (2.0 * u2.astype(np.float64))
    c, s = np.cos(a), np.sin(a)
    # sqrtf(L (1 + d)) with |d| <= ulp(L) / L: relative error <= d / 2, then its own rounding (half an ulp)
    with np.errstate(divide="ignore", invalid="ignore"):
        e_rad = np.where(L > 0, rad * ulp32(L * (1 + 2 ** -20)) / np.where(L > 0, 2 * L, 1), 0.0)
    e_rad = 1.001 * e_rad + 0.5 * ulp32(rad * (1 + 2 ** -20)) * (L > 0)

    def bound(v):
        ev = ulp32(np.abs(v) * (1 + 2 ** -20)) + 4e-16      # sinpif / cospif (1 ulp) and float64 sin / cos of pi * x
        p = (rad + e_rad) * (np.abs(v) + ev)
        return e_rad * np.abs(v) + rad * ev + e_rad * ev + 0.5 * ulp32(p) + 1e-300
    return rad * c, rad * s, bound(c), bound(s), r


def noise_ref(N, HW, seed, utt0, draw, mutate=None):
    """[N, HW, 2] float64 z and bound of draw_noise for samples n = 0..N-1; mutate: one of PHILOX_MUTATIONS."""
    n = np.arange(N, dtype=np.uint64)[:, None]
    pix = np.arange(HW, dtype=np.uint64)[None, :]
    utt, d, sd = n + np.uint64(utt0), draw, int(seed)
    kw = {}
    if mutate == "draw + 1":
        d = draw + 1
    elif mutate == "utterance + 1":
        utt = utt + np.uint64(1)
    elif mutate == "seed words swapped":
        sd = ((sd & 0xFFFFFFFF) << 32) | (sd >> 32)
    elif mutate == "draw <-> utterance in the counter":
        utt, d = np.uint64(draw) + 0 * n, n + np.uint64(utt0)
    elif mutate == "round constant M0 + 2":
        kw["M"] = (PHILOX_M[0] + 2, PHILOX_M[1])
    re, im, bre, bim, r = complex_normal_ref(sd, utt, d, pix, **kw)
    z, b = np.stack([re, im], -1), np.stack([bre, bim], -1)
    if mutate == "re <-> im":
        z = z[..., ::-1]
    return z, b, r


PHILOX_MUTATIONS = ("draw + 1", "utterance + 1", "seed words swapped", "draw <-> utterance in the counter", "re <-> im",
                    "round constant M0 + 2")


# ------------------------------------------------------------------------------------------------
# device structs and buffers
# ------------------------------------------------------------------------------------------------
def rng_params(seed, utt0):
    """RngParams {u64 seed; int utt0; int pad} in device memory."""
    a = np.zeros(2, dtype=np.int64)
    a.view(np.uint64)[0] = np.uint64(seed)
    a.view(np.int32)[2] = utt0
    return torch.from_numpy(a).cuda()


def dev_f32(v):
    return torch.tensor(v, dtype=torch.float32, device="cuda")


CANARY64 = 0x7FF8DEADBEEFCAFE      # an fp64 NaN


class Guarded64(Guarded):
    """Guarded for float64 tensors."""

    def __init__(self, shape, dtype=torch.float64):
        numel = math.prod(shape)
        self.bits, self.int_dtype = CANARY64, torch.int64
        self.buf = torch.empty(numel + 2 * PAD, dtype=torch.float64, device="cuda")
        self.buf.view(torch.int64).fill_(CANARY64)
        self.t = self.buf[PAD:PAD + numel].view(shape)
        self.numel = numel


def guarded(shape, dtype=torch.float32, init=None):
    g = Guarded64(shape) if dtype == torch.float64 else Guarded(shape, dtype)
    if init is not None:
        g.t.copy_(init)
    return g


def bits(t):
    return t.view(torch.int64 if t.dtype == torch.float64 else torch.int32)


def ratio(got, ref, bound):
    """max |got - ref| / bound (NaN: infinitely wrong)."""
    got, ref, bound = (v.double().cpu() if torch.is_tensor(v) else torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64))
                       for v in (got, ref, bound))
    return torch.nan_to_num((got - ref).abs() / bound, nan=math.inf).max().item()


class Report:
    """Worst err/bound and weakest mutation ratio of one kernel family; failures collected, asserted at the end."""

    def __init__(self, name):
        self.name, self.worst, self.weakest, self.failures = name, 0.0, math.inf, []

    def err(self, what, r):
        self.worst = max(self.worst, r)
        if not r <= 1:
            self.failures.append(f"{what}: err/bound {r:.3g}")
        return r

    def mut(self, what, r):
        self.weakest = min(self.weakest, r)
        if not r >= 10:
            self.failures.append(f"{what}: mutation only {r:.3g} x the bound")
        return r

    def exact(self, what, ok):
        if not ok:
            self.failures.append(f"{what}: not bit-identical")

    def done(self):
        print(f"[{self.name}] worst err/bound {self.worst:.3g}; weakest mutation {self.weakest:.3g}")
        assert not self.failures, "\n".join(self.failures)


# ------------------------------------------------------------------------------------------------
# Philox: launch_prior with y = 0, std1 = 1 and no injected noise writes z itself
# ------------------------------------------------------------------------------------------------
PHILOX_CASES = [   # seed, utt0, draw, N, H, W
    (0x0123456789ABCDEF, 0, 0, 2, 64, 37),
    (0xFFFFFFFF00000001, 7, 3, 3, 50, 50),
    (0x9E3779B97F4A7C15, 123456, 1, 1, 1024, 1024),       # 2^20 pixels: r.x within 2^22 of 0 and of 2^32
    ((5 << 40) | 17, 2 ** 31 - 3, 60, 2, 8, 9),
]


@pytest.mark.gpu
def test_philox_noise_against_numpy_philox(samp):
    rep = Report("philox / complex_normal")
    for seed, utt0, draw, N, H, W in PHILOX_CASES:
        HW = H * W
        st = guarded((N, HW, 4), init=torch.zeros(N, HW, 4))
        rng = rng_params(seed, utt0)
        samp.prior(st.t.data_ptr(), N, H, W, 1.0, None, rng.data_ptr(), draw)
        again = guarded((N, HW, 4), init=torch.zeros(N, HW, 4))
        samp.prior(again.t.data_ptr(), N, H, W, 1.0, None, rng.data_ptr(), draw)
        torch.cuda.synchronize()
        name = f"seed {seed:#x} utt0 {utt0} draw {draw} N {N} {H}x{W}"
        st.check(name)
        rep.exact(name + " relaunch", torch.equal(bits(st.t), bits(again.t)))
        rep.exact(name + " y untouched", bool((bits(st.t[..., 2:]) == 0).all()))
        z, b, r = noise_ref(N, HW, seed, utt0, draw)
        got = st.t[..., :2].cpu().numpy()
        rep.err(name, ratio(got, z, b))
        if HW >= 2 ** 20:
            assert r[0].min() < 2 ** 22 and r[0].max() > 2 ** 32 - 2 ** 22, "u1 not exercised at both ends"
        for m in PHILOX_MUTATIONS:
            rep.mut(f"{name}: {m}", ratio(got, noise_ref(N, HW, seed, utt0, draw, m)[0], b))
    rep.done()


# ------------------------------------------------------------------------------------------------
# output layer and the elementwise epilogues
# ------------------------------------------------------------------------------------------------
def make_ol(g, scale_after, scale_by_sigma, b=(0.3, -0.2)):
    w = (0.5 * torch.randn(8, generator=g)).tolist()
    return OutLayer([float(np.float32(v)) for v in w], [float(np.float32(v)) for v in b], scale_after, scale_by_sigma)


def out_layer_ref(pyr, ol, inv_t):
    """float64 output layer of pyr [N, HW, 4] fp32 with inv_t [N] (fp32 values) and its bound.  Without scale_after the
    kernel scales p by inv_t first (four fp32 products, emulated exactly here); then b + w . p as a chain of four fmas
    (four roundings, each <= U32 of the running sum <= |b| + sum |w p|); with scale_after one more product rounds."""
    N = pyr.shape[0]
    inv = inv_t.float() if ol.scale_by_sigma else torch.ones(N, device=pyr.device)
    w = torch.tensor(ol.w, dtype=torch.float64, device=pyr.device).view(2, 4)
    b = torch.tensor(ol.b, dtype=torch.float64, device=pyr.device)
    p = pyr if ol.scale_after else pyr * inv[:, None, None]
    pd = p.double()
    re = pd @ w.t() + b
    A = pd.abs() @ w.abs().t() + b.abs()
    bound = 4 * U32 * A * (1 + 8 * U32)
    if ol.scale_after:
        s = inv.double()[:, None, None]
        re, bound = re * s, bound * s.abs() + U32 * (re * s).abs() + U32 * bound * s.abs()
    return re, bound + 1e-300


UpdCase = collections.namedtuple("UpdCase", "name N H W scale_after scale_by_sigma inv_t_dev noise use_noise x_mean")

# N H W: N * H * W never a multiple of 256.  noise: "philox" or "injected"
UPD_CASES = [
    UpdCase("ncsnpp, per-sample 1/t, philox, x_mean", 3, 20, 37, 0, 1, True, "philox", 1, True),
    UpdCase("ncsnpp, scalar 1/t, injected", 2, 33, 31, 0, 1, False, "injected", 1, False),
    UpdCase("48k, per-sample 1/t, injected, x_mean", 3, 16, 29, 1, 1, True, "injected", 1, True),
    UpdCase("48k, scalar 1/t, philox", 1, 24, 45, 1, 1, False, "philox", 1, True),
    UpdCase("v2 (no scaling), philox, no noise, x_mean", 2, 17, 23, 0, 0, True, "philox", 0, True),
    UpdCase("v2 (no scaling) after, injected", 2, 17, 23, 1, 0, False, "injected", 1, False),
]


def upd_inputs(case, seed):
    g = torch.Generator().manual_seed(seed)
    N, HW = case.N, case.H * case.W
    state = torch.randn(N, HW, 4, generator=g).cuda()
    pyr = torch.randn(N, HW, 4, generator=g).cuda()
    tn = np.float32([0.03, 0.5, 0.999, 0.2][:N])
    t, inv_t = torch.from_numpy(tn).cuda(), torch.from_numpy(np.float32(1) / tn).cuda()   # 1.0f / t, correctly rounded
    noise = torch.randn(N, HW, 2, generator=g).cuda() if case.noise == "injected" else None
    return g, state, pyr, t, inv_t, noise


def z_of(N, HW, noise, rng_seed, utt0, draw):
    if noise is not None:
        return noise.double(), torch.zeros_like(noise, dtype=torch.float64)
    z, b, _ = noise_ref(N, HW, rng_seed, utt0, draw)
    return torch.from_numpy(z.copy()).cuda(), torch.from_numpy(b).cuda()


def run_twice(launch, shapes):
    """launch(outs) into fresh guarded buffers twice; returns the first set after checking the canaries and that the
    relaunch is bit-identical.  shapes: [(shape, dtype, init or None)]."""
    res = []
    for _ in range(2):
        outs = [guarded(s, d, i) for s, d, i in shapes]
        launch(*[o.t for o in outs])
        res.append(outs)
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(*res)):
        a.check(f"output {i}")
        assert torch.equal(bits(a.t), bits(b.t)), f"output {i}: relaunch not bit-identical"
    return [o.t for o in res[0]]


@pytest.mark.gpu
def test_update_kernels_against_fp64(samp):
    """pc_update, affine_update, the prior with injected noise, precond_out, out_layer, ode_drift, ode_drift_affine and
    the two state packers, over both output-layer orderings, scale_by_sigma 0 / 1, per-sample and scalar 1/t, Philox and
    injected noise, use_noise 0 / 1 and x_mean_out null / non-null."""
    rep = Report("updates / epilogues")
    SEED, UTT0, DRAW = 0xA5A5A5A5DEADBEEF, 11, 2
    for i, case in enumerate(UPD_CASES):
        g, state, pyr, t, inv_t, noise = upd_inputs(case, 900 + i)
        N, H, W = case.N, case.H, case.W
        HW = H * W
        ol = make_ol(g, case.scale_after, case.scale_by_sigma)
        rng = rng_params(SEED, UTT0)
        z, ez = z_of(N, HW, noise, SEED, UTT0, DRAW)
        s = state.double()
        sx, sz = s[..., :2], s[..., 2:]
        inv_scalar = float(inv_t[0])
        inv_vec = inv_t if case.inv_t_dev else inv_t[:1].expand(N).contiguous()
        d, ed = out_layer_ref(pyr, ol, inv_vec)
        nm = case.name
        mut_ol = ol._replace(scale_after=1 - ol.scale_after)
        swap = [1, 0] + list(range(2, N))

        # ---- pc_update: x_mean = x + cy (y - x) - cs d; x' = x_mean + cz z.  Three roundings of x_mean (the subtraction,
        # two fmas; each <= U32 of A_m = |x| + |cy| (|y| + |x|) + |cs d|) plus |cs| times d's bound; x' one more fma.
        cy, cs, cz = (float(np.float32(v)) for v in (0.37, 0.021, 0.11))
        coef = dev_f32([cy, cs, cz])
        out = run_twice(lambda st, xm: samp.pc_update(st.data_ptr(), pyr.data_ptr(), N, H, W, *_ol(ol),
                                                      _ptr(inv_t) if case.inv_t_dev else None, inv_scalar,
                                                      coef.data_ptr(), _ptr(noise), rng.data_ptr(), DRAW,
                                                      xm.data_ptr() if case.x_mean else None),
                        [((N, HW, 4), torch.float32, state), ((N, HW, 2), torch.float32, None)])
        mre = sx + cy * (sz - sx) - cs * d
        A_m = sx.abs() + abs(cy) * (sz.abs() + sx.abs()) + abs(cs) * d.abs()
        b_m = abs(cs) * ed + 4 * U32 * A_m
        xref = mre + cz * z
        b_x = b_m + abs(cz) * ez + 2 * U32 * (A_m + abs(cz) * z.abs())
        rep.err(f"pc_update {nm}", ratio(out[0][..., :2], xref, b_x))
        rep.exact(f"pc_update {nm}: y untouched", torch.equal(bits(out[0][..., 2:]), bits(state[..., 2:])))
        if case.x_mean:
            rep.err(f"pc_update x_mean {nm}", ratio(out[1], mre, b_m))
        else:
            rep.exact(f"pc_update {nm}: null x_mean_out", bool(torch.isnan(out[1]).all()))
        if case.scale_by_sigma:
            dm = out_layer_ref(pyr, mut_ol, inv_vec)[0]
            rep.mut(f"pc_update {nm}: /t on the other side", ratio(out[0][..., :2], sx + cy * (sz - sx) - cs * dm + cz * z, b_x))
            if case.inv_t_dev and N > 1:
                dm = out_layer_ref(pyr, ol, inv_t[swap])[0]
                rep.mut(f"pc_update {nm}: inv_t of samples 0, 1 swapped", ratio(out[0][..., :2], sx + cy * (sz - sx) - cs * dm + cz * z, b_x))
        if noise is None:
            rep.mut(f"pc_update {nm}: z re <-> im", ratio(out[0][..., :2], mre + cz * z.flip(-1), b_x))

        # ---- affine_update: x_mean = cx x + cF d + cy y (a product and two fmas), x' = x_mean + cz z (use_noise)
        cx, cF, cy2, cz2 = (float(np.float32(v)) for v in (0.93, -0.047, 0.061, 0.13))
        acoef = dev_f32([cx, cF, cy2, cz2])
        out = run_twice(lambda st, xm: samp.affine_update(st.data_ptr(), pyr.data_ptr(), N, H, W, *_ol(ol), acoef.data_ptr(),
                                                          _ptr(noise), rng.data_ptr(), DRAW, case.use_noise,
                                                          xm.data_ptr() if case.x_mean else None),
                        [((N, HW, 4), torch.float32, state), ((N, HW, 2), torch.float32, None)])
        one = torch.ones(N, device="cuda")
        d1, ed1 = out_layer_ref(pyr, ol, one)
        mre = cx * sx + cF * d1 + cy2 * sz
        A_m = (cx * sx).abs() + abs(cF) * d1.abs() + (cy2 * sz).abs()
        b_m = abs(cF) * ed1 + 4 * U32 * A_m
        zz, ezz = (z, ez) if case.use_noise else (0 * z, 0 * ez)
        b_x = b_m + abs(cz2) * ezz + 2 * U32 * (A_m + abs(cz2) * zz.abs())
        rep.err(f"affine_update {nm}", ratio(out[0][..., :2], mre + cz2 * zz, b_x))
        if case.x_mean:
            rep.err(f"affine_update x_mean {nm}", ratio(out[1], mre, b_m))
            if not case.use_noise:
                rep.exact(f"affine_update {nm}: x' == x_mean without noise", torch.equal(bits(out[0][..., :2]), bits(out[1])))
        if case.use_noise and noise is None:
            rep.mut(f"affine_update {nm}: z re <-> im", ratio(out[0][..., :2], mre + cz2 * z.flip(-1), b_x))
        if not case.use_noise:
            rep.mut(f"affine_update {nm}: noise drawn despite use_noise 0", ratio(out[0][..., :2], mre + cz2 * z, b_x))

        # ---- prior with injected noise: x = y + z std1, one fma
        if noise is not None:
            std1 = float(np.float32(0.4137))
            out = run_twice(lambda st: samp.prior(st.data_ptr(), N, H, W, std1, noise.data_ptr(), None, 0),
                            [((N, HW, 4), torch.float32, state)])
            ref = sz + std1 * z
            rep.err(f"prior {nm}", ratio(out[0][..., :2], ref, U32 * ref.abs() + 1e-300))
            rep.mut(f"prior {nm}: x kept instead of y", ratio(out[0][..., :2], sx + std1 * z, U32 * ref.abs() + 1e-300))

        # ---- precond_out: a[n] x + b[n] d (a product and an fma)
        a_dev, b_dev = dev_f32([0.7, -1.3, 2.1][:N]), dev_f32([1.9, 0.45, -0.8][:N])
        xt = torch.randn(N, HW, 2, generator=g).cuda()
        out = run_twice(lambda o: samp.precond_out(xt.data_ptr(), pyr.data_ptr(), N, H, W, *_ol(ol), a_dev.data_ptr(),
                                                   b_dev.data_ptr(), o.data_ptr()), [((N, HW, 2), torch.float32, None)])

        def pre_ref(a, b):
            a, b = a.double()[:, None, None], b.double()[:, None, None]
            return a * xt.double() + b * d1, b.abs() * ed1 + 3 * U32 * ((a * xt.double()).abs() + (b * d1).abs())
        ref, bnd = pre_ref(a_dev, b_dev)
        rep.err(f"precond_out {nm}", ratio(out[0], ref, bnd))
        if N > 1:
            rep.mut(f"precond_out {nm}: (a, b) of samples 0, 1 swapped", ratio(out[0], pre_ref(a_dev[swap], b_dev[swap])[0], bnd))

        # ---- out_layer: sign * out_layer(pyr, 1 / t[n]) with 1 / t in fp32 (correctly rounded, emulated exactly)
        for neg in (0, 1):
            out = run_twice(lambda o: samp.out_layer(pyr.data_ptr(), N, H, W, *_ol(ol), t.data_ptr(), o.data_ptr(), neg),
                            [((N, HW, 2), torch.float32, None)])
            sign = -1.0 if neg else 1.0
            dt, edt = out_layer_ref(pyr, ol, inv_t)
            rep.err(f"out_layer {nm} negate {neg}", ratio(out[0], sign * dt, edt))
            if case.scale_by_sigma:
                rep.mut(f"out_layer {nm}: /t on the other side", ratio(out[0], sign * out_layer_ref(pyr, mut_ol, inv_t)[0],
                                                                       out_layer_ref(pyr, ol, inv_t)[1]))
                if N > 1:
                    rep.mut(f"out_layer {nm}: t of samples 0, 1 swapped", ratio(out[0], sign * out_layer_ref(pyr, ol, inv_t[swap])[0],
                                                                                out_layer_ref(pyr, ol, inv_t)[1]))

        # ---- ode_drift: theta (y - x) + cs d (a subtraction, a product, an fma); ode_drift_affine: cx x + cy y + cF d
        theta, cs3 = float(np.float32(1.5)), float(np.float32(0.77))
        out = run_twice(lambda o: samp.ode_drift(state.data_ptr(), pyr.data_ptr(), N, H, W, *_ol(ol), inv_scalar, theta, cs3,
                                                 o.data_ptr()), [((N, HW, 2), torch.float32, None)])
        dsc, edsc = out_layer_ref(pyr, ol, inv_t[:1].expand(N))
        ref = theta * (sz - sx) + cs3 * dsc
        bnd = cs3 * edsc + 4 * U32 * (theta * (sz.abs() + sx.abs()) + cs3 * dsc.abs())
        rep.err(f"ode_drift {nm}", ratio(out[0], ref, bnd))
        rep.mut(f"ode_drift {nm}: theta (x - y)", ratio(out[0], theta * (sx - sz) + cs3 * dsc, bnd))
        if case.scale_by_sigma:
            rep.mut(f"ode_drift {nm}: /t on the other side",
                    ratio(out[0], theta * (sz - sx) + cs3 * out_layer_ref(pyr, mut_ol, inv_t[:1].expand(N))[0], bnd))
        out = run_twice(lambda o: samp.ode_drift_affine(state.data_ptr(), pyr.data_ptr(), N, H, W, *_ol(ol), cx, cy2, cF,
                                                        o.data_ptr()), [((N, HW, 2), torch.float32, None)])
        ref = cx * sx + cy2 * sz + cF * d1
        bnd = abs(cF) * ed1 + 4 * U32 * ((cx * sx).abs() + (cy2 * sz).abs() + abs(cF) * d1.abs())
        rep.err(f"ode_drift_affine {nm}", ratio(out[0], ref, bnd))
        rep.mut(f"ode_drift_affine {nm}: cx and cy exchanged", ratio(out[0], cy2 * sx + cx * sz + cF * d1, bnd))

        # ---- pack_state (exact) and pack_state_scaled (one fp32 product per component, emulated exactly)
        x2, y2 = state[..., :2].contiguous(), state[..., 2:].contiguous()
        out = run_twice(lambda o: samp.pack_state(x2.data_ptr(), y2.data_ptr(), N, H, W, o.data_ptr()),
                        [((N, HW, 4), torch.float32, None)])
        rep.exact(f"pack_state {nm}", torch.equal(bits(out[0]), bits(state)))
        out = run_twice(lambda o: samp.pack_state_scaled(x2.data_ptr(), y2.data_ptr(), inv_t.data_ptr(), N, H, W, o.data_ptr()),
                        [((N, HW, 4), torch.float32, None)])
        rep.exact(f"pack_state_scaled {nm}", torch.equal(bits(out[0]), bits(state * inv_t[:, None, None])))
    rep.done()


# ------------------------------------------------------------------------------------------------
# Langevin step size (correctors.py:45-56): eps = 2 (snr mean_n |z_n| / mean_n |grad_n|)^2, batch means
# ------------------------------------------------------------------------------------------------
LV_CASES = [   # N, H, W, noise.  H * W = 5000 < 64 * 256: blocks run the grid-stride loop 0 or 1 times; 49252: 3 or 4
    (1, 50, 100, "philox"),
    (2, 50, 100, "injected"),
    (5, 50, 100, "philox"),
    (1, 196, 251, "injected"),
    (2, 196, 251, "philox"),
    (5, 196, 251, "injected"),
]


def langevin_ref(gn2, zn2, snr):
    """eps, cz from the per-sample squared norms (float64)."""
    gn, zn = np.sqrt(gn2).mean(), np.sqrt(zn2).mean()
    eps = 2 * (snr * zn / gn) ** 2
    return eps, math.sqrt(2 * eps)


@pytest.mark.gpu
def test_langevin_coef_against_fp64(samp):
    rep = Report("langevin_coef")
    SEED, UTT0, DRAW, snr = 0x1234_0000_5678, 3, 5, float(np.float32(0.5))
    for i, (N, H, W, kind) in enumerate(LV_CASES):
        g = torch.Generator().manual_seed(1000 + i)
        HW = H * W
        pyr = (torch.randn(N, HW, 4, generator=g) * (1 + torch.arange(N)).view(N, 1, 1) ** 2).cuda()   # unequal norms
        noise = torch.randn(N, HW, 2, generator=g).cuda() * 0.7 if kind == "injected" else None
        ol = make_ol(g, 0, 1)
        inv_t = float(np.float32(1) / np.float32(0.2))
        rng = rng_params(SEED, UTT0)
        out = run_twice(lambda sc, cf: samp.langevin_coef(pyr.data_ptr(), N, H, W, *_ol(ol), inv_t, _ptr(noise), rng.data_ptr(),
                                                          DRAW, snr, sc.data_ptr(), cf.data_ptr()),
                        [((N * LV_BLOCKS * 2,), torch.float32, None), ((3,), torch.float32, None)])
        coef = out[1].cpu().double().numpy()
        d, ed = out_layer_ref(pyr, ol, torch.full((N,), inv_t, device="cuda"))
        z, ez = z_of(N, HW, noise, SEED, UTT0, DRAW)
        d, ed, z, ez = (v.reshape(N, -1).cpu().numpy() for v in (d, ed, z, ez))
        # Each squared norm is an fp32 sum: per thread a chain of at most `it` elements (each |v|^2 an fma pair: two
        # roundings), a 5-level shuffle tree, 8 warp sums in thread 0: relative error <= (2 it + 13) U32 of sum |v|^2.
        # The elements' own errors e add 2 |v| e + e^2.  Then sqrt halves the relative error, the batch means keep it,
        # snr zn / gn adds both, squaring doubles it, and eps rounds to fp32; cz = sqrtf(2 eps): half of eps's + U32.
        it = -(-HW // (LV_BLOCKS * 256))
        depth = (2 * it + 13) * U32

        def rel(v, e):
            s2 = (v * v).sum(1)
            return ((2 * np.abs(v) * e + e * e).sum(1) + depth * s2 * 1.01) / (2 * s2)
        gn2, zn2 = (d * d).sum(1), (z * z).sum(1)
        eps, cz = langevin_ref(gn2, zn2, snr)
        r_eps = 2 * (rel(d, ed).max() + rel(z, ez).max()) * 1.01 + U32
        r_cz = r_eps / 2 + U32
        name = f"N {N} H*W {HW} {kind}"
        rep.exact(name + ": cy", coef[0] == 0.0)
        rep.err(name + ": eps", abs(coef[1] - eps) / (r_eps * eps))
        rep.err(name + ": cz", abs(coef[2] - cz) / (r_cz * cz))
        if N > 1:
            e0 = 2 * (snr * math.sqrt(zn2[0]) / math.sqrt(gn2[0])) ** 2
            rep.mut(name + ": per-sample step (sample 0)", abs(coef[1] - e0) / (r_eps * eps))
            e_rms = 2 * (snr * np.sqrt(zn2.mean()) / np.sqrt(gn2.mean())) ** 2
            rep.mut(name + ": norm of the whole batch", abs(coef[1] - e_rms) / (r_eps * eps))
        print(f"[langevin_coef] {name}: eps {coef[1]:.6g} err/bound {abs(coef[1] - eps) / (r_eps * eps):.3g}")
    rep.done()


# ------------------------------------------------------------------------------------------------
# time embedding: GaussianFourierProjection -> Linear -> SiLU -> Linear -> SiLU -> stacked Dense (oracle/ncsnpp.py)
# ------------------------------------------------------------------------------------------------
TEMB_CASES = [   # nf, totalC, R
    (32, 8 * 32 + 5, 1),
    (32, 8 * 32 + 5, 3),
    (128, 3 * 128 + 7, 32),
    (128, 3 * 128 + 7, 61),
]


def temb_times(R):
    """0.03, then down to 1e-4 and up to 1; rows 0 and 1 far apart (their swap is a mutation)."""
    base = [0.03, 1.0, 1e-4, 0.5]
    return np.float32(np.concatenate([base, np.geomspace(1e-4, 1.0, max(R - 4, 0))])[:R])


def silu_bound(z, ez):
    """silu(z) float64 and the bound of silu_f(z + ez) = __fdividef(z, 1 + __expf(-z)) (common.cuh): |silu'| <= 1.1
    carries the input error; __expf errs by 2 + floor(|1.173 z|) ulps, scaled by sigmoid(-z) through 1 / (1 + e); the sum
    and __fdividef (2 ulps) round (CUDA C++ Programming Guide, intrinsic functions)."""
    h = z * torch.sigmoid(z)
    rel = torch.sigmoid(-z) * (2 + 1.173 * z.abs()) * ULP32 + U32 + 2 * ULP32
    return h, 1.1 * ez + rel * h.abs() * (1 + 4 * rel)


def tf32(x):
    """x (fp32 values) rounded to TF32 (10 explicit mantissa bits, round to nearest, ties away: cvt.rna.tf32.f32)."""
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32).to(x.dtype)


def linear_ref(x, ex, w, b, tf32_operands=False, bias=True):
    """float64 x w^T + b and the bound of the kernels' warp-per-output dot product: a per-lane fma chain of K / 32
    terms, a 5-level shuffle tree and the bias add round at most K / 32 + 6 times, each <= U32 of sum |w x| + |b|; the
    input errors ex add sum |w| ex.  tf32_operands / bias: the mutations (TF32 operands, bias dropped)."""
    wd, bd = w.double(), b.double() * bias
    if tf32_operands:
        x, wd = tf32(x), tf32(wd)
    K = wd.shape[1]
    y = x @ wd.t() + bd
    A = x.abs() @ wd.abs().t() + bd.abs()
    return y, ex @ wd.abs().t() + (K // 32 + 6) * U32 * A * 1.01


def fourier_args(lt, W):
    """The kernel's fp32 argument ((logf(t) W) 2) pi_f32 (misc.cu: temb_mlp_kernel) from the exact fp32 log t it read.  SASS
    of misc.o: FMUL(lt, W), then the doubling contracted into FFMA(lt, W, that product), then FMUL by pi_f32; emulated
    with one rounding each."""
    lt, W = np.float32(lt)[:, None], np.float32(W)[None, :]
    p = lt * W
    return fma32(np.broadcast_to(lt, p.shape), np.broadcast_to(W, p.shape), p) * np.float32(math.pi)


def temb_mlp_ref(pr, l1w, l1b, l2w, l2b, swap_halves=False, tf32_operands=False, l1_bias=True):
    """float64 scratch = silu(Linear2(silu(Linear1([sin pr, cos pr])))) from the kernel's fp32 arguments pr, and its
    bound: sinf / cosf err by at most 2 ulps each (CUDA C++ Programming Guide), then linear_ref and silu_bound."""
    a = torch.from_numpy(pr.astype(np.float64)).cuda()
    sn, cs = torch.sin(a), torch.cos(a)
    ulp = lambda v: torch.from_numpy(ulp32(v.abs().cpu().numpy() * (1 + 2 ** -20))).cuda()
    emb = torch.cat([cs, sn] if swap_halves else [sn, cs], 1)
    e_emb = 2 * torch.cat([ulp(cs), ulp(sn)] if swap_halves else [ulp(sn), ulp(cs)], 1) + 1e-300
    h1, e1 = silu_bound(*linear_ref(emb, e_emb, l1w, l1b, tf32_operands, l1_bias))
    return silu_bound(*linear_ref(h1, e1, l2w, l2b, tf32_operands))


@pytest.mark.gpu
def test_time_embedding_against_fp64(samp):
    """Both kernels of launch_temb on their own.  temb_mlp_kernel's scratch against the float64 MLP of the fp32 Fourier
    arguments the kernel formed (its logf(t) is read back from the device's own logf, the arithmetic after it is emulated
    exactly); temb_dense_kernel's table against float64 dense_w @ scratch + dense_b of the scratch the kernel wrote.
    The distance of the fp32 arguments from the exact ones (|arg| up to 3e3, so up to ~5e-4 in the embedding) is the
    same in any fp32 implementation, the reference model's included; it is printed, not folded into the bounds, which
    stay tight enough to see TF32 operands or a dropped bias."""
    rep = Report("temb")
    for i, (nf, totalC, R) in enumerate(TEMB_CASES):
        g = torch.Generator().manual_seed(1100 + i)
        D = 4 * nf
        W = (16 * torch.randn(nf, generator=g)).cuda()                             # GaussianFourierProjection(scale=16)
        u = lambda *s, fan: ((torch.rand(*s, generator=g) * 2 - 1) / math.sqrt(fan)).cuda()
        l1w, l1b, l2w, l2b = u(D, 2 * nf, fan=2 * nf), u(D, fan=2 * nf), u(D, D, fan=D), u(D, fan=D)
        dw, db = u(totalC, D, fan=D), u(totalC, fan=D)
        tt = temb_times(R)
        t = torch.from_numpy(tt).cuda()
        out = run_twice(lambda sc, tb: samp.temb(W.data_ptr(), l1w.data_ptr(), l1b.data_ptr(), l2w.data_ptr(), l2b.data_ptr(),
                                                 dw.data_ptr(), db.data_ptr(), nf, totalC, t.data_ptr(), R, sc.data_ptr(),
                                                 tb.data_ptr()),
                        [((R, D), torch.float32, None), ((R, totalC), torch.float32, None)])
        scratch, table = out
        lt_dev = torch.empty(R, device="cuda")
        samp.logf(t.data_ptr(), lt_dev.data_ptr(), R)
        torch.cuda.synchronize()
        lt = lt_dev.cpu().numpy()
        name = f"nf {nf} totalC {totalC} R {R}"
        exact_lt = np.log(tt.astype(np.float64))
        assert (np.abs(lt - exact_lt) <= ulp32(np.abs(exact_lt) * (1 + 2 ** -20))).all(), "logf beyond 1 ulp"
        Wn = W.cpu().numpy()
        pr = fourier_args(lt, Wn)
        ref, bnd = temb_mlp_ref(pr, l1w, l1b, l2w, l2b)
        r_s = rep.err(name + ": scratch", ratio(scratch, ref, bnd))
        # TF32 operands in the two MLP Linears must fail the scratch check, but the margin is smaller than 10: the bound
        # carries Linear1's worst-case fp32 rounding through all 4 nf columns of Linear2 with aligned signs, while TF32's
        # errors (2^-11 per operand) partly cancel.  TF32 in the Dense is held to 10x by the table check below.
        m_tf32 = ratio(scratch, temb_mlp_ref(pr, l1w, l1b, l2w, l2b, tf32_operands=True)[0], bnd)
        if not m_tf32 > 1:
            rep.failures.append(f"{name}: scratch, TF32 Linears within the bound ({m_tf32:.3g})")
        rep.mut(name + ": scratch, Linear1 bias dropped", ratio(scratch, temb_mlp_ref(pr, l1w, l1b, l2w, l2b, l1_bias=False)[0], bnd))
        rep.mut(name + ": scratch, sin / cos halves swapped", ratio(scratch, temb_mlp_ref(pr, l1w, l1b, l2w, l2b, True)[0], bnd))
        if R > 1:
            rep.mut(name + ": scratch, times of rows 0, 1 swapped",
                    ratio(scratch, temb_mlp_ref(pr[[1, 0] + list(range(2, R))], l1w, l1b, l2w, l2b)[0], bnd))
        s64 = scratch.double()
        zero = torch.zeros_like(s64)
        tref, tbnd = linear_ref(s64, zero, dw, db)
        r_t = rep.err(name + ": table", ratio(table, tref, tbnd))
        rep.mut(name + ": table, TF32 Dense", ratio(table, linear_ref(s64, zero, dw, db, tf32_operands=True)[0], tbnd))
        rep.mut(name + ": table, Dense bias dropped", ratio(table, linear_ref(s64, zero, dw, db, bias=False)[0], tbnd))
        exact = temb_mlp_ref(np.outer(exact_lt, Wn.astype(np.float64)) * 2 * math.pi, l1w, l1b, l2w, l2b)[0]
        print(f"[temb] {name}: |Fourier arg| up to {float(np.abs(pr).max()):.3g}, max err/bound scratch {r_s:.3g} table "
              f"{r_t:.3g}; TF32 Linears miss the scratch by {m_tf32:.3g} x its bound; the fp32 arguments move the scratch "
              f"by up to {float((exact - ref).abs().max()):.2g} from the exact-argument MLP")
    rep.done()


# ------------------------------------------------------------------------------------------------
# ODE vector kernels
# ------------------------------------------------------------------------------------------------
DP_A = [[1 / 5], [3 / 40, 9 / 40], [44 / 45, -56 / 15, 32 / 9], [19372 / 6561, -25360 / 2187, 64448 / 6561, -212 / 729],
        [9017 / 3168, -355 / 33, 46732 / 5247, 49 / 176, -5103 / 18656]]
DP_B = [35 / 384, 0, 500 / 1113, 125 / 192, -2187 / 6784, 11 / 84]
DP_E = [-71 / 57600, 0, 71 / 16695, -71 / 1920, 17253 / 339200, -22 / 525, 1 / 40]


def combine_coefs(s):
    """s = 1..5: a Dormand-Prince stage row; 6: the 5th-order weights; 7: the error weights."""
    a = DP_A[s - 1] if s <= 5 else DP_B if s == 6 else DP_E
    return list(a) + [0.0] * (7 - len(a))


def ode_data(total, seed, scale_new=3.0):
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(total, 2, generator=g, dtype=torch.float64).cuda()
    K = [torch.randn(total, 2, generator=g).cuda() * (1 + j) for j in range(7)]
    y_new = y + scale_new * torch.randn(total, 2, generator=g, dtype=torch.float64).cuda()
    return y, K, y_new


def combine_ref(y, K, a, h, s):
    """y + (sum_{j<s} a_j K_j) h and its bound: the kernel's fp64 chain (s fmas, the product by h, the sum) and the
    reference's own, each <= (s + 2) U64 of |y| + |h| sum |a_j K_j|."""
    lin = sum(a[j] * K[j].double() for j in range(s))
    A = y.abs() + abs(h) * sum(abs(a[j]) * K[j].double().abs() for j in range(s))
    return y + lin * h, 2 * (s + 2) * U64 * A * 1.01 + 1e-300


COMBINE_TOTALS = (100, 1000 + 17, 2112 * 256 + 4321)     # the last: above the 2112-block cap, so the grid strides
NORM_TOTALS = (100, 1000 + 17, NORM_BLOCKS * 256 + 5000)


@pytest.mark.gpu
def test_ode_combine_against_fp64(samp):
    rep = Report("ode_combine")
    for total in COMBINE_TOTALS:
        y, K, _ = ode_data(total, total)
        h = -0.0371
        for s in range(1, 8):
            a = combine_coefs(s)
            ref, bnd = combine_ref(y, K, a, h, s)
            for with_new in (True, False):
                shapes = [((total, 2), torch.float32, None), ((total, 2), torch.float64, None)]
                out = run_twice(lambda st, yn: samp.ode_combine(y.data_ptr(), _ptrs(K), s, _doubles(a), h, total, st.data_ptr(),
                                                                yn.data_ptr() if with_new else None), shapes)
                name = f"total {total} s {s} y_new {with_new}"
                if with_new:
                    rep.exact(name + ": stage == (float2) y_new", torch.equal(bits(out[0]), bits(out[1].float())))
                    rep.err(name + ": y_new", ratio(out[1], ref, bnd))
                    drop = list(a)
                    drop[s - 1] = 0.0
                    if any(drop[:s]) or s == 1:
                        rep.mut(name + f": coefficient {s - 1} dropped", ratio(out[1], combine_ref(y, K, drop, h, s)[0], bnd))
                else:
                    rep.exact(name + ": null y_new", bool(torch.isnan(out[1]).all()))
                    rep.err(name + ": stage", ratio(out[0], ref, bnd + torch.from_numpy(ulp32(ref.abs().cpu().numpy() * 1.001)).cuda()))
    rep.done()


def norm_terms(kind, y, y_new, K, E, h, rtol, atol, scale_y_only=False):
    """float64 |v / scale|^2 per bin and the bound of each term as the kernel forms it (see ode.cu: norm_acc)."""
    ay = torch.sqrt((y * y).sum(1))
    ev = torch.zeros_like(ay)
    if kind == 0:
        v = y
    elif kind == 1:
        v = K[0].double()
    elif kind == 2:
        v = K[1].double() - K[0].double()
    else:
        v = sum(E[j] * K[j].double() for j in range(7)) * h
        ev = 9 * U64 * abs(h) * sum(abs(E[j]) * K[j].double().abs().sum(1) for j in range(7))
        if not scale_y_only:
            ay = torch.maximum(ay, torch.sqrt((y_new * y_new).sum(1)))
    scale = atol + ay * rtol
    t = (v * v).sum(1) / (scale * scale)
    q = ev / scale
    # hypot (2 ulps), the fma of the scale, the division, the squares and their sum: 16 U64 of the term; v's error
    # enters as 2 |v / scale| ev / scale + (ev / scale)^2.  The float64 reference errs as much again.
    return t, 2 * (16 * U64 * t + 2 * torch.sqrt(t) * q + q * q)


def scipy_rms_norm(x):
    """The error norm of scipy's RK45 controller, scipy.integrate._ivp.common.norm: ||x|| / sqrt(x.size) (scipy 1.18.1,
    and every release since solve_ivp appeared).  The module is private; where a release no longer has it, the same
    formula stands in."""
    try:
        from scipy.integrate._ivp.common import norm
    except ImportError:
        return float(np.linalg.norm(x) / x.size ** 0.5)
    return float(norm(x))


def block_partition_sums(x, total):
    """sums of x over each block's grid-stride bins: bin i belongs to block (i // 256) % 528."""
    blk = (torch.arange(total, device=x.device) // 256) % NORM_BLOCKS
    return torch.zeros(NORM_BLOCKS, dtype=torch.float64, device=x.device).index_add_(0, blk, x)


@pytest.mark.gpu
def test_ode_norm_against_fp64(samp):
    rep = Report("ode_norm")
    rtol, atol, h = 1e-3, 1e-4, -0.0213
    for total in NORM_TOTALS:
        y, K, y_new = ode_data(total, 7 * total)
        depth = -(-total // (NORM_BLOCKS * 256)) + 13     # a thread's chain, the shuffle tree, thread 0's 8 warp sums
        for kind in range(4):
            out = run_twice(lambda p: samp.ode_norm(kind, y.data_ptr(), y_new.data_ptr(), _ptrs(K), _doubles(DP_E), h, rtol,
                                                    atol, total, p.data_ptr()), [((NORM_BLOCKS,), torch.float64, None)])
            t, et = norm_terms(kind, y, y_new, K, DP_E, h, rtol, atol)
            ref = block_partition_sums(t, total)
            bnd = block_partition_sums(et + 2 * depth * U64 * t * 1.01, total) + 1e-300
            name = f"total {total} kind {kind}"
            rep.err(name + ": partials", ratio(out[0], ref, bnd))
            if kind == 3:
                rep.mut(name + ": scale from |y| only",
                        ratio(out[0], block_partition_sums(norm_terms(kind, y, y_new, K, DP_E, h, rtol, atol, True)[0], total), bnd))
            # the host's sqrt(sum / total) (engine.cu: finish_norm, block order) against scipy's common.norm
            part = out[0].cpu().numpy()
            got = math.sqrt(sum(part.tolist()) / total)
            yn, Kn, ynn = y.cpu().numpy(), [k.cpu().numpy().astype(np.float64) for k in K], y_new.cpu().numpy()
            c = lambda a: a[:, 0] + 1j * a[:, 1]
            v = [c(yn), c(Kn[0]), c(Kn[1]) - c(Kn[0]), sum(DP_E[j] * c(Kn[j]) for j in range(7)) * h][kind]
            sc = atol + (np.maximum(np.abs(c(yn)), np.abs(c(ynn))) if kind == 3 else np.abs(c(yn))) * rtol
            want = scipy_rms_norm(v / sc)
            # the partials' bounds (half: the sqrt), the host's 528-term sum and numpy's sum of `total` squares
            b_norm = want * (0.5 * float(bnd.sum()) / float(ref.sum()) + (NORM_BLOCKS + 2 * total + 4) * U64) + 1e-300
            rep.err(name + ": norm vs scipy", abs(got - want) / b_norm)
            rep.mut(name + ": partial of block 0 dropped", abs(math.sqrt(sum(part[1:].tolist()) / total) - want) / b_norm)
    rep.done()


@pytest.mark.gpu
def test_ode_init_finish_exact(samp):
    rep = Report("ode_init / ode_finish")
    for total in (100, 1000 + 17, 70001):
        g = torch.Generator().manual_seed(total)
        st = torch.randn(total, 4, generator=g).cuda()
        out = run_twice(lambda y: samp.ode_init(st.data_ptr(), total, y.data_ptr()), [((total, 2), torch.float64, None)])
        rep.exact(f"init {total}", torch.equal(out[0], st[:, :2].double()))
        y = torch.randn(total, 2, generator=g, dtype=torch.float64).cuda() * 10
        out = run_twice(lambda o: samp.ode_finish(y.data_ptr(), total, o.data_ptr()), [((total, 2), torch.float32, None)])
        rep.exact(f"finish {total}", torch.equal(bits(out[0]), bits(y.float())))
    rep.done()


GROUP_TOTALS = {1: [NORM_BLOCKS * 256 + 777], 16: [37 + 1013 * i + (NORM_BLOCKS * 256 + 99 if i == 5 else 0) for i in range(16)]}


@pytest.mark.gpu
def test_ode_groups_and_rows_equal_single_kernels(samp):
    """ode_combine_groups / ode_norm_groups: each system bit for bit what ode_combine / ode_norm write for it alone;
    ode_rows_pack / ode_rows_drift: each row what pack_state(_scaled) and ode_drift(_affine) write for it alone."""
    rep = Report("ode groups / rows")
    rtol, atol = 1e-3, 1e-4
    for n, totals in GROUP_TOTALS.items():
        data = [ode_data(tt, 31 * tt + i) for i, tt in enumerate(totals)]
        s = [1 + i % 7 for i in range(n)]
        a = [combine_coefs(k) for k in s]
        h = [-0.01 * (i + 1) for i in range(n)]
        with_new = [i % 3 != 1 for i in range(n)]
        stage = [guarded((tt, 2)) for tt in totals]
        ynew = [guarded((tt, 2), torch.float64) for tt in totals]
        flat = lambda xs: sum(xs, [])
        samp.ode_combine_groups(n, _ptrs([d[0] for d in data]), _ptrs([yn.t if w else None for yn, w in zip(ynew, with_new)]),
                                _ptrs([x.t for x in stage]), _ptrs(flat([d[1] for d in data])), _doubles(flat(a)),
                                _doubles(h), (C.c_longlong * n)(*totals), (C.c_int * n)(*s))
        for i in range(n):
            one = run_twice(lambda st, yn: samp.ode_combine(data[i][0].data_ptr(), _ptrs(data[i][1]), s[i], _doubles(a[i]), h[i],
                                                            totals[i], st.data_ptr(), yn.data_ptr() if with_new[i] else None),
                            [((totals[i], 2), torch.float32, None), ((totals[i], 2), torch.float64, None)])
            torch.cuda.synchronize()
            stage[i].check(f"combine_groups system {i}")
            ynew[i].check(f"combine_groups system {i}")
            rep.exact(f"n {n} system {i} (total {totals[i]}, s {s[i]}): combine stage", torch.equal(bits(stage[i].t), bits(one[0])))
            rep.exact(f"n {n} system {i}: combine y_new", torch.equal(bits(ynew[i].t), bits(one[1])))
        kinds = [i % 4 for i in range(n)]
        part = guarded((n * NORM_BLOCKS,), torch.float64)
        samp.ode_norm_groups(n, _ptrs([d[0] for d in data]), _ptrs([d[2] for d in data]), _ptrs(flat([d[1] for d in data])),
                             _doubles(flat([DP_E] * n)), _doubles(h), (C.c_longlong * n)(*totals), (C.c_int * n)(*kinds),
                             rtol, atol, part.t.data_ptr())
        torch.cuda.synchronize()
        part.check("norm_groups")
        for i in range(n):
            one = run_twice(lambda p: samp.ode_norm(kinds[i], data[i][0].data_ptr(), data[i][2].data_ptr(), _ptrs(data[i][1]),
                                                    _doubles(DP_E), h[i], rtol, atol, totals[i], p.data_ptr()),
                            [((NORM_BLOCKS,), torch.float64, None)])
            rep.exact(f"n {n} system {i} (kind {kinds[i]}): norm partials",
                      torch.equal(bits(part.t[i * NORM_BLOCKS:(i + 1) * NORM_BLOCKS]), bits(one[0])))
    for nrows in (1, 32):
        g = torch.Generator().manual_seed(1300 + nrows)
        px1 = 333
        xs = [torch.randn(px1, 2, generator=g).cuda() for _ in range(nrows)]
        ys = [torch.randn(px1, 2, generator=g).cuda() for _ in range(nrows)]
        t = [float(np.float32(0.03 + 0.97 * r / 32)) for r in range(nrows)]
        c_in = [float(np.float32(1 / (1 + r))) for r in range(nrows)]
        ol = make_ol(g, nrows % 2, 1)
        for raw in (True, False):
            st, rw, td, sd = guarded((nrows, px1, 4)), guarded((nrows, px1, 4)), guarded((nrows,)), guarded((nrows,))
            samp.ode_rows_pack(nrows, _ptrs(xs), _ptrs(ys), _floats(t), _floats(c_in), px1, st.t.data_ptr(),
                               rw.t.data_ptr() if raw else None, td.t.data_ptr(), sd.t.data_ptr())
            torch.cuda.synchronize()
            for b in (st, rw, td, sd):
                b.check("rows_pack")
            rep.exact(f"rows {nrows} raw {raw}: t, c_in", torch.equal(td.t.cpu(), torch.tensor(t)) and torch.equal(sd.t.cpu(), torch.tensor(c_in)))
            for r in range(nrows):
                sc = dev_f32([c_in[r]])
                if raw:
                    one = run_twice(lambda o: samp.pack_state_scaled(xs[r].data_ptr(), ys[r].data_ptr(), sc.data_ptr(), 1, 1, px1,
                                                                     o.data_ptr()), [((px1, 4), torch.float32, None)])
                    rep.exact(f"rows {nrows} row {r}: scaled state", torch.equal(bits(st.t[r]), bits(one[0])))
                    rep.exact(f"rows {nrows} row {r}: raw", torch.equal(bits(rw.t[r]), bits(torch.cat([xs[r], ys[r]], 1))))
                else:
                    rep.exact(f"rows {nrows} row {r}: state", torch.equal(bits(st.t[r]), bits(torch.cat([xs[r], ys[r]], 1))))
            if not raw:
                rep.exact(f"rows {nrows}: raw untouched", bool(torch.isnan(rw.t).all()))
        state = torch.randn(nrows, px1, 4, generator=g).cuda()
        pyr = torch.randn(nrows, px1, 4, generator=g).cuda()
        theta = float(np.float32(1.5))
        c0 = [float(np.float32(v)) for v in (torch.rand(nrows, generator=g) * 30 + 1).tolist()]
        c1 = [float(np.float32(v)) for v in (torch.rand(nrows, generator=g) - 0.5).tolist()]
        for affine in (0, 1):
            ks = [guarded((px1, 2)) for _ in range(nrows)]
            samp.ode_rows_drift(nrows, _ptrs([k.t for k in ks]), _floats(c0), _floats(c1), px1, state.data_ptr(), pyr.data_ptr(),
                                *_ol(ol), theta, affine)
            torch.cuda.synchronize()
            for r in range(nrows):
                ks[r].check("rows_drift")
                if affine:
                    one = run_twice(lambda o: samp.ode_drift_affine(state[r].data_ptr(), pyr[r].data_ptr(), 1, 1, px1, *_ol(ol), c0[r],
                                                                    theta, c1[r], o.data_ptr()), [((px1, 2), torch.float32, None)])
                else:
                    one = run_twice(lambda o: samp.ode_drift(state[r].data_ptr(), pyr[r].data_ptr(), 1, 1, px1, *_ol(ol), c0[r],
                                                             theta, c1[r], o.data_ptr()), [((px1, 2), torch.float32, None)])
                rep.exact(f"rows {nrows} row {r} affine {affine}: drift", torch.equal(bits(ks[r].t), bits(one[0])))
    rep.done()


# ------------------------------------------------------------------------------------------------
# the device ODE solve against scipy: a network whose output is exactly its output-layer bias
# ------------------------------------------------------------------------------------------------
# With output_layer.weight = 0 the network output is b (ncsnpp, ncsnpp_v2) or b / t (ncsnpp_48k, which scales after the
# layer) whatever the upstream weights do, in every mode.  The probability-flow drift is then a known function of (t, x):
#   ncsnpp:  theta (y - x) + cs(t) b                         cs = (float)(0.5 g(t)^2)            (ode.cu: ode_drift)
#   48k:     theta (y - x) + cs(t) (float)(b * inv_t)        inv_t = 1.0f / (float)t
#   v2:      cx(t) x + theta y + cF(t) b                     cx, cF: engine.cu ode_drift_coefs with a = c_skip, b = c_out
# SASS of ode.o: ode_drift forms FFMA(theta, FADD(y, -x), FMUL(cs, d)); ode_drift_affine FFMA(cF, d, FFMA(cx, x,
# FMUL(theta, y))); prior_kernel FFMA(z, std1, y).  The harness rounds those operations exactly (fma32), so it evaluates
# the same fp32 drift the device does from the same complex64 stage.
OdeModel = collections.namedtuple("OdeModel", "kind theta sigma_min sigma_max")


def fma32(a, b, c):
    """float32(a * b + c) with one rounding (a, b, c float32 arrays): the product is exact in float64, the sum is made
    exact with TwoSum, and a float64 sum that lands on an fp32 midpoint is resolved by the sign of its residual."""
    p = np.asarray(a, np.float64) * np.asarray(b, np.float64)
    c = np.asarray(c, np.float64)
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    toward = np.where(s > r64, np.float32(np.inf), np.float32(-np.inf))
    other = np.nextafter(r, toward)
    tie = (err != 0) & (2 * (s - r64) == other.astype(np.float64) - r64)
    up = np.sign(err) == np.sign(other.astype(np.float64) - r64)
    return np.where(tie & up, other, r).astype(np.float32)


def c64(re, im):
    out = np.empty(np.shape(re), np.complex64)
    out.real, out.imag = re, im
    return out


def ouve_std(m, t):
    """engine.cu: ouve_std, in the same double operations."""
    th, smin, ls = float(np.float32(m.theta)), float(np.float32(m.sigma_min)), math.log(float(np.float32(m.sigma_max)) / float(np.float32(m.sigma_min)))
    return math.sqrt(smin * smin * math.exp(-2 * th * t) * (math.exp(2 * (th + ls) * t) - 1) * ls / (th + ls))


def drift_coefs(m, t):
    """engine.cu: ode_drift_coefs at (float)t: (theta, cs, inv_t, cx, cF) as fp32."""
    tf = np.float32(t)
    smin, smax = float(np.float32(m.sigma_min)), float(np.float32(m.sigma_max))
    ls = math.log(smax / smin)
    g = smin * math.pow(smax / smin, float(tf)) * math.sqrt(2 * ls)
    th = float(np.float32(m.theta))
    cs = np.float32(0.5 * g * g)
    inv_t = np.float32(1.0) / tf
    pa, pb = (0.0, 1.0 / ouve_std(m, float(tf))) if m.kind == "v2" else (1.0, 0.0)   # V2 'score': c_skip 0, c_out 1/sigma
    cx = np.float32(-th - 0.5 * g * g * pa)
    cF = np.float32(-0.5 * g * g * pb)
    return np.float32(th), cs, inv_t, cx, cF


def pf_drift_f32(m, t, x, y, b):
    """The engine's complex64 drift at (t, x) with the network output b (complex64 bias pair)."""
    th, cs, inv_t, cx, cF = drift_coefs(m, t)
    out = []
    for xr, yr, br in ((x.real, y.real, np.float32(b.real)), (x.imag, y.imag, np.float32(b.imag))):
        if m.kind == "v2":
            out.append(fma32(cF, br, fma32(cx, xr, th * yr)))
        else:
            d = br * inv_t if m.kind == "48k" else br
            out.append(fma32(th, yr - xr, cs * np.float32(d)))
    return c64(*out)


def prior_f32(m, y, z):
    std1 = np.float32(ouve_std(m, 1.0))
    return c64(fma32(z.real, std1, y.real), fma32(z.imag, std1, y.imag))


OdeRef = collections.namedtuple("OdeRef", "x nfev accepted rejected status hs xmax kmax")


def scipy_ode(m, y, z, b, rtol, atol, eps, stage_at_step_start=False):
    """solve_ivp(RK45) from the prior y + z std(1) (complex64 inputs), as sampling/__init__.py calls it, on the drift
    above.  Every attempted step costs six evaluations after the two of the start (f0 and select_initial_step), so
    rejected = (nfev - 2) / 6 - accepted.  xmax, kmax: the largest |x| (and |y|) and |k| of any evaluation.
    stage_at_step_start: the mutation that evaluates every stage at the time the step starts from, driven through the
    public RK45 class (solve_ivp is a loop over RK45.step, so the arithmetic is the same)."""
    from scipy.integrate import RK45, solve_ivp
    x0 = prior_f32(m, y.reshape(-1), z.reshape(-1)).astype(np.complex128)
    yy = y.reshape(-1)
    big = [float(np.abs(yy).max()), 0.0]

    def fun(t, v):
        x = v.astype(np.complex64)
        k = pf_drift_f32(m, t, x, yy, b)
        big[0], big[1] = max(big[0], float(np.abs(x).max())), max(big[1], float(np.abs(k).max()))
        return k
    if not stage_at_step_start:
        sol = solve_ivp(fun, (1.0, eps), x0, method="RK45", rtol=rtol, atol=atol)
        ts, x, nfev, status = sol.t, sol.y[:, -1], sol.nfev, sol.status
    else:
        start = [1.0]
        solver = RK45(lambda t, v: fun(start[0], v), 1.0, x0, eps, rtol=rtol, atol=atol)
        ts = [solver.t]
        while solver.status == "running":
            solver.step()
            start[0] = solver.t
            ts.append(solver.t)
        x, nfev, status = solver.y, solver.nfev, 0 if solver.status == "finished" else -1
    hs = np.abs(np.diff(ts))
    acc = len(hs)
    return OdeRef(x, nfev, acc, (nfev - 2) // 6 - acc, status, hs, big[0], big[1])


def ode_state_bound(m, ref):
    """How far the device solve may be from scipy's when both take the same steps (the test requires the same nfev,
    accepted and rejected steps).  Both evaluate the identical fp32 drift of a complex64 stage and differ only in the fp64
    integrator arithmetic.  Let D be the difference of the states at a step's start and, over a step of size h, delta_i
    and d_i the differences of stage i's fp64 input and of its derivative K_i.

    * delta_i = D + h sum_j a_ij d_j + rho_i, with |rho_i| <= 16 U64 (xmax + h sum_j |a_ij| kmax): both sides round
      y + h sum_j a_ij K_j at most 8 times.
    * The drift is affine in x with slope exactly -theta (theta (y - x) + c on ncsnpp and 48k, cx x + ... with
      cx = (float)(-theta) on the v2 score model, whose c_skip is 0).  So d_i = -theta delta_i + eta_i, where eta_i
      collects what is not linear: the complex64 rounding of the stage landing on a different neighbour (<= ulp32(xmax),
      times theta) and the drift's fp32 roundings doing the same (<= 2 theta ulp32(2 xmax) + ulp32(kmax)).  With rho_i
      moved into eta_i: |eta_i| <= e_i = 3 theta ulp32(2 xmax) + ulp32(kmax) + theta |rho_i|.
    * Solving the stage equations, d = S (eta - theta D 1) with S = (I + theta h A)^-1, so the new difference is
      D' = R D + h w . eta + rho_y with R = 1 - theta h b . S 1, w = b S, |rho_y| <= 16 U64 (xmax + h sum |b_j| kmax):
      |D'| <= |R| |D| + h sum_j |w_j| e_j + |rho_y| + 1e-12 h kmax.  The last term is the step size itself: h is the
      controller's function of an error norm whose host and device fp64 sums agree to ~1e-13 relative, taken to the power
      -1/5.
    Rejected attempts leave D unchanged; the engine's complex64 output adds one ulp32(xmax)."""
    th = float(np.float32(m.theta))
    A = np.zeros((6, 6))
    for i, row in enumerate(DP_A, 1):
        A[i, :len(row)] = row
    b = np.array(DP_B[:6])
    base = 3 * th * float(ulp32(2 * ref.xmax)) + float(ulp32(ref.kmax))
    D = 0.0
    for h in ref.hs:
        S = np.linalg.inv(np.eye(6) + th * h * A)
        R = 1 - th * h * b @ S @ np.ones(6)
        w = b @ S
        e = base + th * 16 * U64 * (ref.xmax + h * np.abs(A).sum(1) * ref.kmax)
        rho_y = 16 * U64 * (ref.xmax + h * np.abs(b).sum() * ref.kmax)
        D = abs(R) * D + h * float(np.abs(w) @ e) + rho_y + 1e-12 * h * ref.kmax
    return D + float(ulp32(ref.xmax))


ODE_BIAS = (0.3, -0.2)
OdeCase = collections.namedtuple("OdeCase", "name kind modes tol bias")
ODE_CASES = [
    OdeCase("ncsnpp_small", "ncsnpp", ("fp32", "fp16_tc", "tf32_tc"), 1e-5, ODE_BIAS),
    OdeCase("ncsnpp48k_small", "48k", ("fp32",), 1e-5, ODE_BIAS),
    OdeCase("ncsnpp_v2_small score", "v2", ("fp32",), 1e-5, ODE_BIAS),
    OdeCase("ncsnpp_small tight tolerance", "ncsnpp", ("fp32",), 1e-6, (30.0, -21.0)),     # rejects steps
]
ODE_MODEL = {"ncsnpp": OdeModel("ncsnpp", 1.5, 0.05, 0.5), "48k": OdeModel("48k", 1.5, 0.05, 0.5),
             "v2": OdeModel("v2", 1.5, 0.05, 0.5)}


def ode_engine(kind, mode, bias, **kw):
    from sgmse_b200 import Engine, EngineConfig
    from test_gpu_zz_next_rows import SMALL_E, V2_ODE_PRECOND, load_golden
    golden = os.path.join(ROOT, "tests", "golden")
    if kind == "ncsnpp":
        _, sd = load_golden(golden, "ncsnpp_small")
        eng = Engine(EngineConfig(attn_resolutions=(16,), mode=mode, **SMALL_E, **kw))
    elif kind == "48k":
        _, sd = load_golden(golden, "ncsnpp48k_small")
        eng = Engine(EngineConfig.ncsnpp_48k(mode=mode, theta=1.5, sigma_min=0.05, sigma_max=0.5, spec_factor=0.15,
                                             spec_abs_exponent=0.5, **SMALL_E, **kw))
    else:
        _, sd = load_golden(golden, "ncsnpp_v2_small")
        eng = Engine(EngineConfig.ncsnpp_v2(attn_resolutions=(16,), mode=mode, sde="ouve", **SMALL_E, **V2_ODE_PRECOND["score"],
                                            **kw))
    sd = dict(sd)
    sd["output_layer.weight"] = torch.zeros_like(sd["output_layer.weight"])
    sd["output_layer.bias"] = torch.tensor(bias, dtype=sd["output_layer.bias"].dtype)
    eng.load_state_dict(sd)
    return eng


def ode_inputs(B=3, F=64, T=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    lv = torch.tensor([1.0, 0.05, 3.0][:B]).view(B, 1, 1, 1)
    Y = (0.5 * lv * torch.complex(torch.randn(B, 1, F, T, generator=g), torch.randn(B, 1, F, T, generator=g))).to(torch.complex64)
    Z = torch.complex(torch.randn(B, 1, F, T, generator=g), torch.randn(B, 1, F, T, generator=g)).to(torch.complex64) / math.sqrt(2)
    return Y, Z


@pytest.mark.gpu
@pytest.mark.parametrize("case", ODE_CASES, ids=[c.name for c in ODE_CASES])
def test_device_ode_solve_matches_scipy(case):
    """Engine.ode_sample (the batch as one system) and every system of ode_sample_groups (each utterance its own system,
    max_batch 1 and 3, graphs on and off) give scipy's nfev, accepted and rejected steps and status, and its final state
    within ode_state_bound."""
    m = ODE_MODEL[case.kind]
    Y, Z = ode_inputs()
    b = np.complex64(complex(*case.bias))
    eps = 0.03
    kw = dict(rtol=case.tol, atol=case.tol, eps=eps, denoise=False, return_stats=True)
    Yn, Zn = Y.numpy(), Z.numpy()
    whole = scipy_ode(m, Yn, Zn, b, case.tol, case.tol, eps)
    per = [scipy_ode(m, Yn[i], Zn[i], b, case.tol, case.tol, eps) for i in range(Y.shape[0])]
    mut = scipy_ode(m, Yn, Zn, b, case.tol, case.tol, eps, stage_at_step_start=True)
    failures, worst, outs = [], 0.0, {}

    def check(what, x, nfe, st, ref):
        nonlocal worst
        xr, want = ref.x, (ref.nfev, ref.accepted, ref.rejected, ref.status)
        got = (nfe, st["steps"], st["rejected"], st["status"])
        bound = ode_state_bound(m, ref)
        err = float(np.abs(x.cpu().numpy().reshape(-1).astype(np.complex128) - xr).max())
        worst = max(worst, err / bound)
        print(f"[ode vs scipy] {case.name} {what}: nfev / accepted / rejected / status {got} (scipy {want}), "
              f"max |x - scipy| {err:.3g} (bound {bound:.3g})")
        if got != want or not err <= bound:
            failures.append(f"{what}: {got} vs scipy {want}, err {err:.3g} bound {bound:.3g}")
    for mode in case.modes:
        eng = ode_engine(case.kind, mode, case.bias, max_batch=2)
        x, nfe, st = eng.ode_sample(Y.cuda(), prior_noise=Z.cuda(), **kw)
        eng.close()
        check(f"{mode} ode_sample", x, nfe, st, whole)
        outs[mode] = x
        for mb in (1, 3):
            for graphs in (True, False):
                if mode != case.modes[0] and (mb, graphs) != (3, True):
                    continue
                eng = ode_engine(case.kind, mode, case.bias, max_batch=mb, use_graphs=graphs)
                xg, nfes, sts = eng.ode_sample_groups(Y.cuda(), group=1, prior_noise=Z.cuda(), **kw)
                eng.close()
                for i in range(Y.shape[0]):
                    check(f"{mode} groups max_batch {mb} graphs {graphs} system {i}", xg[i:i + 1], nfes[i], sts[i], per[i])
    for mode in case.modes[1:]:
        if not torch.equal(outs[mode].view(torch.float32), outs[case.modes[0]].view(torch.float32)):
            failures.append(f"{mode} differs from {case.modes[0]}: a zero output layer must make the modes bit-identical")
    bound = ode_state_bound(m, whole)
    mut_err = float(np.abs(mut.x - whole.x).max())
    print(f"[ode vs scipy] {case.name}: worst err/bound {worst:.3g}; stage times at the step start: nfev {mut.nfev} "
          f"(scipy {whole.nfev}), state {mut_err / bound:.3g} x the bound")
    assert mut.nfev != whole.nfev or mut_err >= 10 * bound, "the check cannot see stage times"
    if case.tol <= 1e-6:
        assert whole.rejected > 0, "the tight-tolerance case rejects no step"
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------
# host: the cases reach every launcher and branch
# ------------------------------------------------------------------------------------------------
# out_layer's two flags change the result only where the kernel passes an inv_t other than 1; affine_update,
# precond_out and ode_drift_affine pass 1.0f, for which both orderings and both scalings compute the same thing
LAUNCHERS_WITH_INV_T = ("launch_pc_update", "launch_out_layer", "launch_ode_drift")
LAUNCHERS_AT_UNIT_SCALE = ("launch_affine_update", "launch_precond_out", "launch_ode_drift_affine")


def case_coverage():
    """(launcher, branch) pairs the case lists above reach."""
    got = set()
    for c in UPD_CASES:
        for k in LAUNCHERS_WITH_INV_T + LAUNCHERS_AT_UNIT_SCALE + ("launch_pack_state", "launch_pack_state_scaled"):
            got.add((k, "N*H*W % 256" if c.N * c.H * c.W % 256 else "N*H*W multiple of 256"))
        for k in LAUNCHERS_WITH_INV_T:           # the ordering and the scaling only matter where inv_t is not 1
            got |= {(k, f"scale_after {c.scale_after}"), (k, f"scale_by_sigma {c.scale_by_sigma}")}
        got |= {("launch_pc_update", "inv_t device" if c.inv_t_dev else "inv_t scalar"),
                ("launch_pc_update", f"noise {c.noise}"), ("launch_affine_update", f"noise {c.noise}"),
                ("launch_affine_update", f"use_noise {c.use_noise}"),
                ("launch_pc_update", f"x_mean {'set' if c.x_mean else 'null'}"),
                ("launch_affine_update", f"x_mean {'set' if c.x_mean else 'null'}")}
        if c.noise == "injected":
            got.add(("launch_prior", "noise injected"))
        if c.scale_by_sigma and c.inv_t_dev and c.N > 1:
            got.add(("launch_pc_update", "inv_t swap mutation"))
    for seed, utt0, draw, N, H, W in PHILOX_CASES:
        got |= {("launch_prior", "noise philox"), ("philox", "seed hi word" if seed >> 32 else "seed lo only")}
        if H * W >= 2 ** 20:
            got.add(("philox", "u1 at both ends"))
    for N, H, W, kind in LV_CASES:
        got |= {("launch_langevin_coef", f"N {N}"), ("launch_langevin_coef", f"noise {kind}"),
                ("launch_langevin_coef", "loop 0/1" if H * W < LV_BLOCKS * 256 else "loop several")}
    for nf, totalC, R in TEMB_CASES:
        got |= {("launch_temb", f"nf {nf}"), ("launch_temb", f"R {R}")}
        if totalC % 8:
            got.add(("launch_temb", "totalC % 8"))
    for tt in COMBINE_TOTALS:
        got |= {("launch_ode_combine", f"s {s}") for s in range(1, 8)} | {("launch_ode_combine", "y_new"),
                                                                           ("launch_ode_combine", "no y_new")}
        if tt > 2112 * 256:
            got.add(("launch_ode_combine", "grid stride"))
    for tt in NORM_TOTALS:
        got |= {("launch_ode_norm", f"kind {k}") for k in range(4)}
        got.add(("launch_ode_norm", "total < 256" if tt < 256 else "total > 528*256" if tt > NORM_BLOCKS * 256 else "total % 256"))
    got |= {("launch_ode_init", ""), ("launch_ode_finish", "")}
    for n, totals in GROUP_TOTALS.items():
        got |= {("launch_ode_combine_groups", f"n {n}"), ("launch_ode_norm_groups", f"n {n}")}
        if len(set(totals)) > 1:
            got.add(("launch_ode_norm_groups", "unequal totals"))
    got |= {("launch_ode_rows_pack", "rows 1"), ("launch_ode_rows_pack", "rows 32"), ("launch_ode_rows_drift", "affine 0"),
            ("launch_ode_rows_drift", "affine 1")}
    for c in ODE_CASES:
        got |= {("engine ode", c.kind)} | {("engine ode", m) for m in c.modes}
        if c.tol <= 1e-6:
            got.add(("engine ode", "rejected steps"))
    return got


REQUIRED_COVERAGE = {
    *{(k, v) for k in LAUNCHERS_WITH_INV_T for v in ("scale_after 0", "scale_after 1", "scale_by_sigma 0", "scale_by_sigma 1")},
    *{(k, "N*H*W % 256") for k in LAUNCHERS_WITH_INV_T + LAUNCHERS_AT_UNIT_SCALE},
    ("launch_pc_update", "inv_t device"), ("launch_pc_update", "inv_t scalar"), ("launch_pc_update", "noise philox"),
    ("launch_pc_update", "noise injected"), ("launch_affine_update", "use_noise 0"), ("launch_affine_update", "use_noise 1"),
    ("launch_affine_update", "noise philox"), ("launch_affine_update", "noise injected"),
    ("launch_pc_update", "x_mean set"), ("launch_pc_update", "x_mean null"), ("launch_affine_update", "x_mean set"),
    ("launch_affine_update", "x_mean null"), ("launch_pc_update", "inv_t swap mutation"),
    ("launch_pack_state", "N*H*W % 256"), ("launch_pack_state_scaled", "N*H*W % 256"),
    ("launch_prior", "noise philox"), ("launch_prior", "noise injected"), ("philox", "seed hi word"), ("philox", "u1 at both ends"),
    ("launch_langevin_coef", "N 1"), ("launch_langevin_coef", "N 2"), ("launch_langevin_coef", "N 5"),
    ("launch_langevin_coef", "noise philox"), ("launch_langevin_coef", "noise injected"),
    ("launch_langevin_coef", "loop 0/1"), ("launch_langevin_coef", "loop several"),
    ("launch_temb", "nf 32"), ("launch_temb", "nf 128"), ("launch_temb", "totalC % 8"),
    *{("launch_temb", f"R {r}") for r in (1, 3, 32, 61)},
    *{("launch_ode_combine", f"s {s}") for s in range(1, 8)}, ("launch_ode_combine", "y_new"), ("launch_ode_combine", "no y_new"),
    ("launch_ode_combine", "grid stride"),
    *{("launch_ode_norm", f"kind {k}") for k in range(4)}, ("launch_ode_norm", "total < 256"), ("launch_ode_norm", "total % 256"),
    ("launch_ode_norm", "total > 528*256"), ("launch_ode_init", ""), ("launch_ode_finish", ""),
    ("launch_ode_combine_groups", "n 1"), ("launch_ode_combine_groups", "n 16"), ("launch_ode_norm_groups", "n 1"),
    ("launch_ode_norm_groups", "n 16"), ("launch_ode_norm_groups", "unequal totals"),
    ("launch_ode_rows_pack", "rows 1"), ("launch_ode_rows_pack", "rows 32"), ("launch_ode_rows_drift", "affine 0"),
    ("launch_ode_rows_drift", "affine 1"),
    ("engine ode", "ncsnpp"), ("engine ode", "48k"), ("engine ode", "v2"), ("engine ode", "fp32"), ("engine ode", "fp16_tc"),
    ("engine ode", "tf32_tc"), ("engine ode", "rejected steps"),
}


def test_cases_reach_every_launcher_and_branch():
    got = case_coverage()
    assert not REQUIRED_COVERAGE - got, f"no case reaches {sorted(REQUIRED_COVERAGE - got)}"
    assert LAUNCHERS <= {k for k, _ in got}, f"no case reaches {sorted(LAUNCHERS - {k for k, _ in got})}"
