"""Op-level tests of the resampling GroupNorm-apply (FIR up / down), channel_stats, the input conv, Combine, the 4-channel
FIR and the output conv: each kernel elementwise against a float64 reference of the same operation.

These kernels run in every forward, and most make a deliberate approximation (an fp16 tanh-form SiLU, fp16 staging,
half2 FIR arithmetic, fp16 operands of an mma.sync).  At network level they are covered only by a rel-L2 norm, in which
an error confined to a border row, a tile seam or one sample's (a, b) row disappears.  Here every output element has its
own bound, derived from the kernel's rounding model, and each case prints max(err / bound).  The mutation controls compare
the same kernel output with a deliberately wrong reference and require a failure by at least 10x the bound.

tests/c/small_ops.cu is an extern "C" shim over the product launchers and the engine's device weight packers, linked
against the library objects like tests/c/kernel_ops.cu.  The tests start from torch-layout weights, pack them with the
engine's packers and take plain F.conv2d / upfirdn2d (oracle.ncsnpp.fir_down2 / fir_up2) as the reference, computed from
the exact fp16 / fp32 values the kernels read.

The cases include the levels a long recording reaches (Tpad = 4800 on the 16 kHz backbone: 32 x 600 down to 4 x 75) and
the 48 kHz backbone's 12-row level, where the launchers fall back from the tiled, vectorized and tile-statistics kernels
to their generic forms.  The *_branch functions predict each case's kernel from the launchers' conditions; a host test
checks that the cases reach every branch.
"""
import collections
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.ncsnpp import fir_down2, fir_kernel_2d, fir_up2
from test_gpu_kernel_ops import U32, ULP32, Guarded, build_shim, ratio, ulp16

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM_SRC = os.path.join(ROOT, "tests", "c", "small_ops.cu")

# Kernel selection of the product, installed per call by activate() (sgmse_b200/csrc/engine.cu) from option value 0;
# the switches default to 0 in the kernel sources, so the shim takes them as explicit arguments.
PRODUCT_FIR_VARIANT = 2
PRODUCT_OUTCONV_VARIANT = 3
PRODUCT_INCONV_VARIANT = 2
PRODUCT_COMBINE_VARIANT = 1

RS_DOWN, RS_UP = 1, 2
F16, F32 = 1, 0

U16 = 2.0 ** -11            # fp16 unit roundoff (round to nearest)
SUB16 = 2.0 ** -25          # half the fp16 subnormal spacing: the absolute rounding error below 2^-14
# tanh.approx.f32: the PTX ISA gives a maximum error of 2^-10.987.  The bound below uses |hz| * 2^-10.987 for the error of
# hz * tanh(hz), which holds whether that figure is read as relative (|t| <= 1) or as absolute.
TANH_APPROX_ERR = 2.0 ** -10.987


_I, _P, _F = C.c_int, C.c_void_p, C.c_float
_IP = C.POINTER(C.c_int)
SIGNATURES = {
    "sops_gn_apply_rs": [_P, _I, _I, _I, _I, _I, _P, _P, _I, _P, _P, _I],
    "sops_channel_stats": [_P, _I, _I, _I, _I, _I, _P, _P, _IP],
    "sops_input_conv": [_P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _F, _I, _IP],
    "sops_combine": [_P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _I, _IP],
    "sops_fir4": [_P, _I, _I, _I, _I, _P, _P, _F],
    "sops_out_conv": [_P, _I, _I, _I, _I, _I, _P, _P, C.POINTER(C.c_float), _P, _P, _P, _I],
    "sops_pack_inconv": [_P, _P, _I, _P],
    "sops_pack_combine": [_P, _P, _I, _P],
    "sops_pack_outconv": [_P, _P, _I, _P, _P],
}


def _stream():
    return torch.cuda.current_stream().cuda_stream if torch.cuda.is_available() else None


def _ptr(t):
    return None if t is None else t.data_ptr()


def _dt(t):
    """DType code of a tensor or a torch dtype."""
    return F16 if getattr(t, "dtype", t) == torch.float16 else F32


class SmallOps:
    def __init__(self, path):
        self.lib = C.CDLL(path, mode=os.RTLD_LOCAL)
        for name, args in SIGNATURES.items():
            fn = getattr(self.lib, name)
            fn.argtypes, fn.restype = args, C.c_int
        self.lib.sops_last_error.restype = C.c_char_p

    def _check(self, code):
        if code != 0:
            raise RuntimeError(f"small_ops: {self.lib.sops_last_error().decode()} (code {code})")

    def gn_apply_rs(self, x, ab, rs, out0, out1, variant=PRODUCT_FIR_VARIANT):
        N, H, W, Cc = x.shape
        self._check(self.lib.sops_gn_apply_rs(_stream(), _dt(x), N, H, W, Cc, x.data_ptr(), ab.data_ptr(), rs,
                                              out0.data_ptr(), out1.data_ptr(), variant))

    def channel_stats(self, x, stats):
        N, H, W, Cc = x.shape
        slots = C.c_int()
        self._check(self.lib.sops_channel_stats(_stream(), _dt(x), N, H, W, Cc, x.data_ptr(), stats.data_ptr(),
                                                C.byref(slots)))
        return slots.value

    def input_conv(self, state, w, bias, out, stats, in_scale, variant=PRODUCT_INCONV_VARIANT):
        N, H, W, Cc = out.shape
        slots = C.c_int()
        self._check(self.lib.sops_input_conv(_stream(), _dt(out), N, H, W, Cc, state.data_ptr(), w.data_ptr(),
                                             bias.data_ptr(), out.data_ptr(), _ptr(stats), in_scale, variant,
                                             C.byref(slots)))
        return slots.value

    def combine(self, pyr, w, bias, h, out, stats, variant=PRODUCT_COMBINE_VARIANT):
        N, H, W, Cc = h.shape
        slots = C.c_int()
        self._check(self.lib.sops_combine(_stream(), _dt(h), N, H, W, Cc, pyr.data_ptr(), w.data_ptr(), bias.data_ptr(),
                                          h.data_ptr(), out.data_ptr(), _ptr(stats), variant, C.byref(slots)))
        return slots.value

    def fir4(self, x, rs, out, scale=1.0):
        N, H, W, _ = x.shape
        self._check(self.lib.sops_fir4(_stream(), N, H, W, rs, x.data_ptr(), out.data_ptr(), scale))

    def out_conv(self, act, w, bias, addend, out, wfrag, variant=PRODUCT_OUTCONV_VARIANT):
        N, H, W, Cc = act.shape
        b = (C.c_float * 4)(*[float(v) for v in bias])
        self._check(self.lib.sops_out_conv(_stream(), _dt(act), N, H, W, Cc, act.data_ptr(), w.data_ptr(), b,
                                           _ptr(addend), out.data_ptr(), _ptr(wfrag), variant))

    def pack_inconv(self, w):
        out = torch.empty(36 * w.shape[0], dtype=torch.float32, device="cuda")
        self._check(self.lib.sops_pack_inconv(_stream(), w.data_ptr(), w.shape[0], out.data_ptr()))
        return out

    def pack_combine(self, w):
        out = torch.empty(4 * w.shape[0], dtype=torch.float32, device="cuda")
        self._check(self.lib.sops_pack_combine(_stream(), w.data_ptr(), w.shape[0], out.data_ptr()))
        return out

    def pack_outconv(self, w):
        Cc = w.shape[1]
        out = torch.empty(36 * Cc, dtype=torch.float32, device="cuda")
        frag = torch.empty(9 * (Cc // 16) * 32 * 2, dtype=torch.int32, device="cuda")
        self._check(self.lib.sops_pack_outconv(_stream(), w.data_ptr(), Cc, out.data_ptr(), frag.data_ptr()))
        return out, frag


@pytest.fixture(scope="module")
def sops(tmp_path_factory):
    return SmallOps(build_shim(str(tmp_path_factory.mktemp("small_ops")), SHIM_SRC))


# ------------------------------------------------------------------------------------------------
# dispatch: which kernel each launcher picks (gn.cu: gn_apply_dispatch; small.cu: launch_input_conv, launch_combine,
# launch_out_conv), with the product's kernel selection
# ------------------------------------------------------------------------------------------------
def gn_rs_branch(dt, rs, Hi, Wi, Cc):
    Ho, Wo = (Hi // 2, Wi // 2) if rs == RS_DOWN else (2 * Hi, 2 * Wi)
    if dt == F16 and rs == RS_UP and Hi % 8 == 0 and Wi % 8 == 0 and Cc % 64 == 0:
        return "gn_apply tiled up"
    if dt == F16 and rs == RS_DOWN and Ho % 8 == 0 and Wo % 8 == 0 and Cc % 32 == 0:
        return "gn_apply tiled down"
    return f"gn_apply generic {'down' if rs == RS_DOWN else 'up'} {'fp16' if dt == F16 else 'fp32'}"


def input_conv_branch(dt, H, W, Cc):
    if dt == F16 and PRODUCT_INCONV_VARIANT == 2 and H * W % 128 == 0 and Cc in (32, 64, 128):
        return f"input conv mma C{Cc}"
    return f"input conv CUDA cores {'fp16' if dt == F16 else 'fp32'} {128 if H * W % 128 == 0 else 32}-pixel tiles"


def combine_branch(dt, H, W, Cc):
    tile_stats = H * W % 32 == 0
    if dt == F16 and PRODUCT_COMBINE_VARIANT == 1 and Cc in (128, 256) and tile_stats:
        return f"combine vector C{Cc}"
    return f"combine scalar {'fp16' if dt == F16 else 'fp32'} + {'tile stats' if tile_stats else 'channel_stats'}"


def out_conv_branch(dt, Cc):
    if dt == F16 and PRODUCT_OUTCONV_VARIANT != 1 and Cc in (128, 256):
        return f"out conv mma{' cp.async' if PRODUCT_OUTCONV_VARIANT == 3 else ''} C{Cc}"
    return f"out conv {'coop' if Cc // 8 in (2, 4, 8, 16, 32) else 'plain'} {'fp16' if dt == F16 else 'fp32'} C{Cc}"


# ------------------------------------------------------------------------------------------------
# resampling gn_apply: rounding models
# ------------------------------------------------------------------------------------------------
FIR_DOWN_TAPS, FIR_UP_TAPS = 16, 4


def silu_tanh_form(z):
    """silu(z) in float64 and the error of the tiled kernel's staged fp16 h = fp16(fmaf(hz, tanh.approx(hz), hz)) with
    hz = fmaf(a / 2, x, b / 2) (a / 2, b / 2 exact): hz errs by |hz| u (through silu' <= 1.1: 1.1 |z| u), tanh.approx by
    the PTX figure (times |hz|), the fma rounds once, and the fp16 staging rounds to nearest."""
    h = z * torch.sigmoid(z)
    e = 1.1 * z.abs() * U32 + 0.5 * z.abs() * (1 + U32) * TANH_APPROX_ERR
    e = e + U32 * (h.abs() + e)
    return h, e + 0.5 * ulp16(h.abs() + e)


def silu_expf_form(z):
    """silu(z) in float64 and the error of silu_f(fmaf(a, x, b)) = __fdividef(z, 1 + __expf(-z)) in fp32.  CUDA C++
    Programming Guide, intrinsic functions: __expf(x) errs by at most 2 + floor(|1.173 x|) ulps, __fdividef(x, y) by 2 ulps
    for 2^-126 <= |y| <= 2^126.  The error of exp(-z) reaches 1 + exp(-z) scaled by sigmoid(-z); that sum rounds once."""
    h = z * torch.sigmoid(z)
    rel = torch.sigmoid(-z) * (2 + 1.173 * z.abs()) * ULP32 + U32 + 2 * ULP32
    return h, 1.1 * z.abs() * U32 + rel * h.abs() * (1 + 4 * rel)


def fir_nchw(t, rs):
    return fir_down2(t) if rs == RS_DOWN else fir_up2(t)


def f16x2_fir_bound(staged_err, absval, rs):
    """Error bound of the tiled kernel's separable half2 FIR of staged fp16 values (NCHW float64): the staged errors
    through the FIR (its taps are positive, sum 1 per axis), plus one fp16 rounding per half2 operation (2^-11 of the
    magnitudes it adds, at most the FIR of |value|, or 2^-25 below the normal range).  FIR-down: four operations per row
    and four per column (x0.125 is exact unless it underflows); FIR-up: two and two.  The last operation is the store."""
    n = 8 if rs == RS_DOWN else 4
    P = fir_nchw(staged_err, rs)
    A = fir_nchw(absval, rs) + P
    return P + n * U16 * A * (1 + n * U16) + n * SUB16


def fp32_fir_bound(err, absval, rs):
    """Error bound of the generic kernel's fp32 FIR: the input errors through the FIR, one fp32 fma rounding per tap of the
    running sum (at most the FIR of |value|)."""
    n = FIR_DOWN_TAPS if rs == RS_DOWN else FIR_UP_TAPS
    P = fir_nchw(err, rs)
    return P + n * U32 * (fir_nchw(absval, rs) + P)


def store_bound(pre, ref, dtype):
    return pre + 0.5 * ulp16(ref.abs() + pre) if dtype == torch.float16 else pre


def gn_rs_reference(x, ab, rs, dtype):
    """float64 FIR(silu(a x + b)) and FIR(x) (NHWC) with the elementwise bounds of the kernel the launcher picks."""
    N, H, W, Cc = x.shape
    branch = gn_rs_branch(_dt(x), rs, H, W, Cc)
    xd = x.double().permute(0, 3, 1, 2)
    z = ab[..., 0].double()[:, :, None, None] * xd + ab[..., 1].double()[:, :, None, None]
    if "tiled" in branch:
        h, herr = silu_tanh_form(z)
        bh = f16x2_fir_bound(herr, h.abs(), rs)
        bx = f16x2_fir_bound(torch.zeros_like(xd), xd.abs(), rs)
    else:
        h, herr = silu_expf_form(z)
        ref_h, ref_x = fir_nchw(h, rs), fir_nchw(xd, rs)
        bh = store_bound(fp32_fir_bound(herr, h.abs(), rs), ref_h, dtype)
        bx = store_bound(fp32_fir_bound(torch.zeros_like(xd), xd.abs(), rs), ref_x, dtype)
    nhwc = lambda t: t.permute(0, 2, 3, 1)
    return branch, nhwc(fir_nchw(h, rs)), nhwc(bh), nhwc(fir_nchw(xd, rs)), nhwc(bx), z


def fir_pad_before_activation(x, ab, rs):
    """Mutation: the zero padding applied to x before the activation, so the taps outside the image see silu(b), not 0."""
    xd = F.pad(x.double().permute(0, 3, 1, 2), (1, 1, 1, 1))
    z = ab[..., 0].double()[:, :, None, None] * xd + ab[..., 1].double()[:, :, None, None]
    hc = z * torch.sigmoid(z)
    B_, Cc, Hp, Wp = hc.shape
    k = fir_kernel_2d(torch.float64).to(hc.device).view(1, 1, 4, 4)
    if rs == RS_DOWN:
        y = F.conv2d(hc.reshape(B_ * Cc, 1, Hp, Wp), k, stride=2)
    else:                                   # the canvas pixel j lands at 2j of the zero-inserted grid: pad (2, 1) exactly
        zi = hc.new_zeros(B_ * Cc, 1, 2 * Hp, 2 * Wp)
        zi[:, :, ::2, ::2] = hc.reshape(B_ * Cc, 1, Hp, Wp)
        y = F.conv2d(zi[:, :, :2 * Hp - 1, :2 * Wp - 1], 4 * k)
    return y.view(B_, Cc, y.shape[-2], y.shape[-1]).permute(0, 2, 3, 1)


def fir_up_pad12(t):
    """Mutation: FIR-up with pad (1, 2) instead of (2, 1) (NCHW)."""
    B_, Cc, H, W = t.shape
    z = t.new_zeros(B_ * Cc, 1, 2 * H, 2 * W)
    z[:, :, ::2, ::2] = t.reshape(B_ * Cc, 1, H, W)
    k = (fir_kernel_2d(t.dtype).to(t.device) * 4).view(1, 1, 4, 4)
    return F.conv2d(F.pad(z, (1, 2, 1, 2)), k).view(B_, Cc, 2 * H, 2 * W)


def fir_down_shifted(t):
    """Mutation: FIR-down one pixel off (pad (0, 2) instead of (1, 1)) (NCHW)."""
    B_, Cc, H, W = t.shape
    k = fir_kernel_2d(t.dtype).to(t.device).view(1, 1, 4, 4)
    return F.conv2d(F.pad(t.reshape(B_ * Cc, 1, H, W), (0, 2, 0, 2)), k, stride=2).view(B_, Cc, H // 2, W // 2)


def fir_mutant(t_nhwc, rs):
    t = t_nhwc.permute(0, 3, 1, 2)
    return (fir_down_shifted(t) if rs == RS_DOWN else fir_up_pad12(t)).permute(0, 2, 3, 1)


GnCase = collections.namedtuple("GnCase", "name N H W C rs dtype kind")

# H, W: the input's.  Levels: the full-size network's 256 x T pyramid (C 128 above, 256 below 64 rows), the long-clip
# bottom levels at Tpad = 4800 (32 x 600 ... 4 x 75) and the 48 kHz backbone's 24 x 16 -> 12 x 8.
GN_CASES = [
    GnCase("256x512 -> 128x256 C128", 1, 256, 512, 128, RS_DOWN, torch.float16, "normal"),
    GnCase("128x256 -> 256x512 C128", 1, 128, 256, 128, RS_UP, torch.float16, "normal"),
    GnCase("16x32 -> 8x16 C256 N3", 3, 16, 32, 256, RS_DOWN, torch.float16, "normal"),
    GnCase("8x16 -> 4x8 C256 N3", 3, 8, 16, 256, RS_DOWN, torch.float16, "normal"),
    GnCase("4x8 -> 8x16 C256 N3", 3, 4, 8, 256, RS_UP, torch.float16, "normal"),
    GnCase("8x16 -> 16x32 C256 N3", 3, 8, 16, 256, RS_UP, torch.float16, "normal"),
    GnCase("32x600 -> 16x300 C256", 1, 32, 600, 256, RS_DOWN, torch.float16, "normal"),
    GnCase("16x300 -> 8x150 C256 N2", 2, 16, 300, 256, RS_DOWN, torch.float16, "normal"),
    GnCase("8x150 -> 4x75 C256 N3", 3, 8, 150, 256, RS_DOWN, torch.float16, "normal"),
    GnCase("4x75 -> 8x150 C256 N3", 3, 4, 75, 256, RS_UP, torch.float16, "normal"),
    GnCase("8x150 -> 16x300 C256 N2", 2, 8, 150, 256, RS_UP, torch.float16, "normal"),
    GnCase("16x300 -> 32x600 C256", 1, 16, 300, 256, RS_UP, torch.float16, "normal"),
    GnCase("48k 24x16 -> 12x8 C256 N2", 2, 24, 16, 256, RS_DOWN, torch.float16, "normal"),
    GnCase("48k 12x8 -> 24x16 C256 N2", 2, 12, 8, 256, RS_UP, torch.float16, "normal"),
    GnCase("64x48 -> 32x24 C128 N2 (4x3 tiles)", 2, 64, 48, 128, RS_DOWN, torch.float16, "normal"),
    GnCase("24x40 -> 48x80 C128 N2 (3x5 tiles)", 2, 24, 40, 128, RS_UP, torch.float16, "normal"),
    GnCase("fp32 32x64 -> 16x32 C128 N3", 3, 32, 64, 128, RS_DOWN, torch.float32, "normal"),
    GnCase("fp32 8x150 -> 4x75 C256 N2", 2, 8, 150, 256, RS_DOWN, torch.float32, "normal"),
    GnCase("fp32 8x16 -> 16x32 C256 N3", 3, 8, 16, 256, RS_UP, torch.float32, "normal"),
    GnCase("fp32 4x75 -> 8x150 C256 N2", 2, 4, 75, 256, RS_UP, torch.float32, "normal"),
    # in-range fp16 values above 32760: x of channel 0 in [33000, 60000], h of channel 1 in [38500, 55000]
    GnCase("overflow 16x32 -> 8x16 C64", 1, 16, 32, 64, RS_DOWN, torch.float16, "large"),
    GnCase("overflow 16x32 -> 32x64 C64", 1, 16, 32, 64, RS_UP, torch.float16, "large"),
    GnCase("overflow 16x24 -> 8x12 C64", 1, 16, 24, 64, RS_DOWN, torch.float16, "large"),
]


def make_gn_inputs(case, seed):
    """x and ab = (a, b) per (sample, channel), different in every sample, with z = a x + b over about [-12, 6]."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    N, H, W, Cc = case.N, case.H, case.W, case.C
    u = lambda *s: torch.rand(*s, generator=g, device="cuda", dtype=torch.float64)
    x = (-8 + 11 * u(N, H, W, Cc)).to(case.dtype)
    a, b = 1 + 0.3 * u(N, Cc), -1.5 + 4 * u(N, Cc)
    if case.kind == "large":
        x[..., 0] = (33000 + 27000 * u(N, H, W)).to(case.dtype)
        a[:, 0], b[:, 0] = 1e-4, 0.0
        x[..., 1] = (0.7 + 0.3 * u(N, H, W)).to(case.dtype)
        a[:, 1], b[:, 1] = 55000.0, 0.0
    return x.contiguous(), torch.stack([a, b], -1).float().contiguous()


@pytest.mark.gpu
def test_resampling_gn_apply_against_fp64(sops):
    """Both outputs of the resampling gn_apply, FIR(silu(a x + b)) and FIR(x), on every branch of its dispatch."""
    failures, worst, weakest = [], 0.0, math.inf
    for i, case in enumerate(GN_CASES):
        x, ab = make_gn_inputs(case, 300 + i)
        Ho, Wo = (case.H // 2, case.W // 2) if case.rs == RS_DOWN else (2 * case.H, 2 * case.W)
        out0, out1 = Guarded((case.N, Ho, Wo, case.C), case.dtype), Guarded((case.N, Ho, Wo, case.C), case.dtype)
        sops.gn_apply_rs(x, ab, case.rs, out0.t, out1.t)
        torch.cuda.synchronize()
        branch, ref_h, bh, ref_x, bx, z = gn_rs_reference(x, ab, case.rs, case.dtype)
        try:
            out0.check("gn_apply h")
            out1.check("gn_apply x")
            finite = bool(torch.isfinite(out0.t).all() and torch.isfinite(out1.t).all())
            rh, rx = ratio(out0.t, ref_h, bh).max().item(), ratio(out1.t, ref_x, bx).max().item()
            worst = max(worst, rh, rx)
            muts = {}
            if case.kind == "normal":
                # the FIR's geometry, where the image meets the zero padding, and which sample's (a, b) is used
                muts["FIR-down shifted" if case.rs == RS_DOWN else "FIR-up pad (1, 2)"] = \
                    ratio(out1.t, fir_mutant(x.double(), case.rs), bx).max().item()
                muts["padding before the activation"] = ratio(out0.t, fir_pad_before_activation(x, ab, case.rs), bh).max().item()
                if case.N > 1:
                    swapped = gn_rs_reference(x, ab[[1, 0] + list(range(2, case.N))], case.rs, case.dtype)[1]
                    muts["(a, b) rows of samples 0, 1 swapped"] = ratio(out0.t, swapped, bh).max().item()
            print(f"[gn_apply] {case.name}: {branch}: z in [{z.min().item():.3g}, {z.max().item():.3g}], max err/bound "
                  f"h {rh:.3g} x {rx:.3g}, mutations {({k: round(v, 1) for k, v in muts.items()})}")
            assert finite, "non-finite output"
            assert rh <= 1 and rx <= 1, f"err/bound h {rh:.3g}, x {rx:.3g}"
            for k, v in muts.items():
                weakest = min(weakest, v)
                assert v >= 10, f"mutation '{k}' only {v:.3g} x the bound"
        except AssertionError as e:
            failures.append(f"{case.name} ({branch}): {e}")
    print(f"[gn_apply] worst err/bound {worst:.3g}; weakest mutation {weakest:.3g}")
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------
# GroupNorm partials: [N][slots][C][2] (sum, sum of squares) over row-major runs of `run` pixels
# ------------------------------------------------------------------------------------------------
def run_sums(y, run):
    N, H, W, Cc = y.shape
    t = y.double().reshape(N, H * W // run, run, Cc)
    return torch.stack([t.sum(2), (t * t).sum(2)], -1)


def box_sums(y, bh, bw):
    """Mutation of run_sums(y, bh * bw): sums over bh x bw pixel boxes instead of row-major runs."""
    N, H, W, Cc = y.shape
    t = y.double().reshape(N, H // bh, bh, W // bw, bw, Cc)
    return torch.stack([t.sum((2, 4)), (t * t).sum((2, 4))], -1).reshape(N, -1, Cc, 2)


def check_partials(stats, out, slots, run, what):
    """The partials against float64 sums of the kernel's own stored output.  Each is an fp32 sum of `run` values in some
    order: at most `run` roundings of the running sum <= sum |v| (sum v^2, one more rounding for the square).  Returns the
    worst err/bound; nothing past [N][slots][C][2] is written."""
    N, H, W, Cc = out.shape
    assert slots * run == H * W, f"{what}: {slots} slots of {run} pixels for {H} x {W}"
    used = N * slots * Cc * 2
    assert bool(torch.isnan(stats.t[used:]).all()), f"{what}: stats written past [N][slots][C][2]"
    st = stats.t[:used].view(N, slots, Cc, 2)
    a = run_sums(out.abs(), run)
    bnd = torch.stack([(run + 1) * U32 * a[..., 0], (run + 2) * U32 * a[..., 1]], -1) + 1e-30
    return ratio(st, run_sums(out, run), bnd).max().item(), st, bnd


def stats_buffer(N, H, W, Cc):
    return Guarded((N * max(1, H * W // 32) * Cc * 2,), torch.float32)   # the engine's capacity


# ------------------------------------------------------------------------------------------------
# input conv
# ------------------------------------------------------------------------------------------------
InCase = collections.namedtuple("InCase", "name N H W C dtype in_scale")

IN_CASES = [
    InCase("256x64 C128 fp16 in_scale 1", 2, 256, 64, 128, torch.float16, 1.0),
    InCase("256x64 C128 fp16 in_scale 0.37", 2, 256, 64, 128, torch.float16, 0.37),
    InCase("64x128 C64 fp16 (ncsnpp_mid)", 2, 64, 128, 64, torch.float16, 1.0),
    InCase("64x64 C16 fp16 (the small configs)", 2, 64, 64, 16, torch.float16, 0.37),
    InCase("256x64 C128 fp32", 2, 256, 64, 128, torch.float32, 0.37),
]


@pytest.mark.gpu
def test_input_conv_against_fp64(sops):
    """conv3x3(in_scale * state) + bias from torch-layout weights packed by the engine's packer, and its GN partials."""
    failures = []
    for i, case in enumerate(IN_CASES):
        g = torch.Generator(device="cuda").manual_seed(400 + i)
        N, H, W, Cc = case.N, case.H, case.W, case.C
        state = torch.randn(N, H, W, 4, generator=g, device="cuda")
        w = (torch.randn(Cc, 4, 3, 3, generator=g, device="cuda") / 6).contiguous()
        bias = 0.1 * torch.randn(Cc, generator=g, device="cuda")
        packed = sops.pack_inconv(w)
        out, stats = Guarded((N, H, W, Cc), case.dtype), stats_buffer(N, H, W, Cc)
        slots = sops.input_conv(state, packed, bias, out.t, stats.t, case.in_scale)
        torch.cuda.synchronize()
        branch = input_conv_branch(_dt(out.t), H, W, Cc)
        try:
            assert torch.equal(packed.view(36, Cc), w.permute(2, 3, 1, 0).reshape(36, Cc)), "packed layout"
            out.check("input conv")
            a32 = torch.tensor(case.in_scale, dtype=torch.float32, device="cuda") * state     # fp32, as the kernel forms it
            mma = "mma" in branch
            A, Wt = (a32.half(), w.half()) if mma else (a32, w)

            def ref_of(wt):
                return F.conv2d(A.double().permute(0, 3, 1, 2), wt.double(), padding=1).permute(0, 2, 3, 1) + bias.double()
            ref = ref_of(Wt)
            absacc = F.conv2d(A.double().abs().permute(0, 3, 1, 2), Wt.double().abs(), padding=1).permute(0, 2, 3, 1)
            # mma.sync: 3 k16 steps (K padded to 48) into an fp32 accumulator: 17 * 48 / 16 ulps of sum |a w|, then + bias.
            # CUDA cores: an fmaf chain of 36 taps from the bias.
            pre = (51 * ULP32 * absacc + U32 * (absacc + bias.double().abs())) if mma else \
                36 * U32 * (absacc + bias.double().abs())
            bound = store_bound(pre, ref, case.dtype)
            r = ratio(out.t, ref, bound).max().item()
            m_tap = ratio(out.t, ref_of(Wt.transpose(2, 3)), bound).max().item()
            r_st, _, _ = check_partials(stats, out.t, slots, 128, "input conv")
            st = stats.t[:N * slots * Cc * 2].view(N, slots, Cc, 2)
            a = box_sums(out.t.abs(), 8, 16)
            bbox = torch.stack([129 * U32 * a[..., 0], 130 * U32 * a[..., 1]], -1) + 1e-30
            m_box = ratio(st, box_sums(out.t, 8, 16), bbox).max().item()
            print(f"[input conv] {case.name}: {branch}, slots {slots}: max err/bound {r:.3g}, partials {r_st:.3g}; "
                  f"mutations: taps dy<->dx {m_tap:.3g}, partials over 8x16 boxes {m_box:.3g}")
            assert r <= 1 and r_st <= 1, f"err/bound {r:.3g}, partials {r_st:.3g}"
            assert m_tap >= 10 and m_box >= 10, f"mutations only {m_tap:.3g}, {m_box:.3g} x the bound"
        except AssertionError as e:
            failures.append(f"{case.name} ({branch}): {e}")
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------
# Combine and channel_stats
# ------------------------------------------------------------------------------------------------
CbCase = collections.namedtuple("CbCase", "name N H W C dtype")

CB_CASES = [
    CbCase("128x32 C128 fp16", 2, 128, 32, 128, torch.float16),
    CbCase("16x32 C256 fp16 N3", 3, 16, 32, 256, torch.float16),
    CbCase("8x150 C256 fp16 (H*W 1200)", 2, 8, 150, 256, torch.float16),
    CbCase("4x75 C256 fp16 (H*W 300) N3", 3, 4, 75, 256, torch.float16),
    CbCase("32x64 C128 fp32", 2, 32, 64, 128, torch.float32),
    CbCase("4x75 C256 fp32 (H*W 300)", 2, 4, 75, 256, torch.float32),
]


@pytest.mark.gpu
def test_combine_and_channel_stats_against_fp64(sops):
    """conv1x1(pyr) + bias + h from torch-layout weights packed by the engine's packer, and its GN partials: 32-pixel
    tiles where H * W allows, else one slot from channel_stats."""
    failures = []
    for i, case in enumerate(CB_CASES):
        g = torch.Generator(device="cuda").manual_seed(500 + i)
        N, H, W, Cc = case.N, case.H, case.W, case.C
        pyr = torch.randn(N, H, W, 4, generator=g, device="cuda")
        w = torch.randn(Cc, 4, 1, 1, generator=g, device="cuda") / 2
        bias = 0.1 * torch.randn(Cc, generator=g, device="cuda")
        h = torch.randn(N, H, W, Cc, generator=g, device="cuda").to(case.dtype)
        packed = sops.pack_combine(w)
        out, stats = Guarded((N, H, W, Cc), case.dtype), stats_buffer(N, H, W, Cc)
        slots = sops.combine(pyr, packed, bias, h, out.t, stats.t)
        torch.cuda.synchronize()
        branch = combine_branch(_dt(h), H, W, Cc)
        try:
            assert torch.equal(packed.view(4, Cc), w.view(Cc, 4).t()), "packed layout"
            out.check("combine")
            wd = w.view(Cc, 4).double()

            def ref_of(p):
                return p.double() @ wd.t() + bias.double() + h.double()
            ref = ref_of(pyr)
            # b + w0 p0 + w1 p1 + w2 p2 + w3 p3 + h in fp32: at most nine roundings (products and sums) of the running sum
            pre = 9 * U32 * (pyr.double().abs() @ wd.abs().t() + bias.double().abs() + h.double().abs())
            r = ratio(out.t, ref, store_bound(pre, ref, case.dtype)).max().item()
            m = ratio(out.t, ref_of(pyr[..., [1, 0, 2, 3]]), store_bound(pre, ref, case.dtype)).max().item()
            expect_slots = H * W // 32 if H * W % 32 == 0 else 1
            assert slots == expect_slots, f"slots {slots}, expected {expect_slots}"
            r_st, st, _ = check_partials(stats, out.t, slots, H * W // slots, "combine")
            if slots == 1:                              # channel_stats on its own: the same partials
                again = stats_buffer(N, H, W, Cc)
                assert sops.channel_stats(out.t, again.t) == 1
                torch.cuda.synchronize()
                assert torch.equal(again.t[:st.numel()].view(torch.int32), st.reshape(-1).view(torch.int32))
            print(f"[combine] {case.name}: {branch}, slots {slots}: max err/bound {r:.3g}, partials {r_st:.3g}; "
                  f"mutation: pyramid components 0, 1 swapped {m:.3g}")
            assert r <= 1 and r_st <= 1, f"err/bound {r:.3g}, partials {r_st:.3g}"
            assert m >= 10, f"mutation only {m:.3g} x the bound"
        except AssertionError as e:
            failures.append(f"{case.name} ({branch}): {e}")
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------
# fir4 (the 4-channel input / output pyramids, fp32)
# ------------------------------------------------------------------------------------------------
FIR4_CASES = [
    ("256x512 down x0.37", 2, 256, 512, RS_DOWN, 0.37),
    ("16x300 down x0.37", 3, 16, 300, RS_DOWN, 0.37),
    ("8x150 down", 2, 8, 150, RS_DOWN, 1.0),
    ("48k 24x16 down x0.37", 2, 24, 16, RS_DOWN, 0.37),
    ("4x75 up", 3, 4, 75, RS_UP, 1.0),
    ("8x16 up", 2, 8, 16, RS_UP, 1.0),
    ("128x256 up", 2, 128, 256, RS_UP, 1.0),
]


@pytest.mark.gpu
def test_fir4_against_fp64(sops):
    failures = []
    for i, (name, N, H, W, rs, scale) in enumerate(FIR4_CASES):
        g = torch.Generator(device="cuda").manual_seed(600 + i)
        x = torch.randn(N, H, W, 4, generator=g, device="cuda")
        Ho, Wo = (H // 2, W // 2) if rs == RS_DOWN else (2 * H, 2 * W)
        out = Guarded((N, Ho, Wo, 4), torch.float32)
        sops.fir4(x, rs, out.t, scale)
        torch.cuda.synchronize()
        try:
            out.check("fir4")
            s = float(np.float32(scale))
            xd = x.double().permute(0, 3, 1, 2)
            ref = fir_nchw(xd, rs).permute(0, 2, 3, 1) * s
            pre = abs(s) * (FIR_DOWN_TAPS if rs == RS_DOWN else FIR_UP_TAPS) * U32 * fir_nchw(xd.abs(), rs).permute(0, 2, 3, 1)
            bound = pre + (U32 * (ref.abs() + pre) if scale != 1 else 0) + 1e-300
            r = ratio(out.t, ref, bound).max().item()
            m = ratio(out.t, fir_mutant(x.double(), rs) * s, bound).max().item()
            print(f"[fir4] {name}: max err/bound {r:.3g}; mutation {'FIR-down shifted' if rs == RS_DOWN else 'FIR-up pad (1, 2)'} {m:.3g}")
            assert r <= 1, f"err/bound {r:.3g}"
            assert m >= 10, f"mutation only {m:.3g} x the bound"
        except AssertionError as e:
            failures.append(f"{name}: {e}")
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------
# output conv
# ------------------------------------------------------------------------------------------------
OcCase = collections.namedtuple("OcCase", "name N H W C dtype addend")

OC_CASES = [
    OcCase("256x64 C128 + addend", 1, 256, 64, 128, torch.float16, True),
    OcCase("8x150 C128 + addend N2", 2, 8, 150, 128, torch.float16, True),
    OcCase("4x75 C128", 3, 4, 75, 128, torch.float16, False),
    OcCase("4x75 C256 + addend N2", 2, 4, 75, 256, torch.float16, True),
    OcCase("8x150 C256", 1, 8, 150, 256, torch.float16, False),
    OcCase("16x300 C256 + addend", 1, 16, 300, 256, torch.float16, True),
    OcCase("fp32 16x300 C128 + addend", 1, 16, 300, 128, torch.float32, True),
    OcCase("fp32 8x150 C256 N2", 2, 8, 150, 256, torch.float32, False),
]


@pytest.mark.gpu
def test_out_conv_against_fp64(sops):
    """conv3x3_{C->4}(act) + bias (+ addend) from torch-layout weights packed by the engine's packer; the mma kernel with
    its packed B fragments and with fragments built per block, which must agree bit for bit."""
    failures = []
    for i, case in enumerate(OC_CASES):
        g = torch.Generator(device="cuda").manual_seed(700 + i)
        N, H, W, Cc = case.N, case.H, case.W, case.C
        act = torch.randn(N, H, W, Cc, generator=g, device="cuda").to(case.dtype)
        w = (torch.randn(4, Cc, 3, 3, generator=g, device="cuda") / math.sqrt(9 * Cc)).contiguous()
        bias = [float(np.float32(v)) for v in (0.1 * torch.randn(4, generator=g, device="cuda")).tolist()]
        addend = torch.randn(N, H, W, 4, generator=g, device="cuda") if case.addend else None
        packed, frag = sops.pack_outconv(w)
        out = Guarded((N, H, W, 4), torch.float32)
        sops.out_conv(act, packed, bias, addend, out.t, frag)
        torch.cuda.synchronize()
        branch = out_conv_branch(_dt(act), Cc)
        try:
            assert torch.equal(packed.view(9, Cc, 4), w.permute(2, 3, 1, 0).reshape(9, Cc, 4)), "packed layout"
            out.check("out conv")
            mma = "mma" in branch
            if mma:
                out2 = Guarded((N, H, W, 4), torch.float32)
                sops.out_conv(act, packed, bias, addend, out2.t, None)
                torch.cuda.synchronize()
                out2.check("out conv (fragments built per block)")
                assert torch.equal(out.t.view(torch.int32), out2.t.view(torch.int32)), "packed fragments change the output"
            Wt = w.half() if mma else w
            b = torch.tensor(bias, dtype=torch.float64, device="cuda")
            add = addend.double() if case.addend else torch.zeros(N, H, W, 4, dtype=torch.float64, device="cuda")

            def ref_of(wt):
                return F.conv2d(act.double().permute(0, 3, 1, 2), wt.double(), padding=1).permute(0, 2, 3, 1) + b + add
            ref = ref_of(Wt)
            absacc = F.conv2d(act.double().abs().permute(0, 3, 1, 2), Wt.double().abs(), padding=1).permute(0, 2, 3, 1)
            # mma.sync over K = 9 C in k16 steps: 17 K / 16 ulps of sum |a w|; the coop kernel: a chain of 9 x 8 fmas per
            # lane, log2(C / 8) shuffle additions; then + bias and + addend in fp32
            chain = 17 * 9 * Cc / 16 * ULP32 if mma else (72 + math.log2(Cc // 8)) * U32
            bound = chain * absacc + 2 * U32 * (absacc + b.abs() + add.abs()) + 1e-300
            r = ratio(out.t, ref, bound).max().item()
            m = ratio(out.t, ref_of(Wt.transpose(2, 3)), bound).max().item()
            print(f"[out conv] {case.name}: {branch}: max err/bound {r:.3g}; mutation taps dy<->dx {m:.3g}"
                  f"{', packed and per-block fragments bit-identical' if mma else ''}")
            assert r <= 1, f"err/bound {r:.3g}"
            assert m >= 10, f"mutation only {m:.3g} x the bound"
        except AssertionError as e:
            failures.append(f"{case.name} ({branch}): {e}")
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------
# host: the cases reach every branch of the dispatchers
# ------------------------------------------------------------------------------------------------
REQUIRED_BRANCHES = {
    "gn_apply tiled up", "gn_apply tiled down", "gn_apply generic up fp16", "gn_apply generic down fp16",
    "gn_apply generic up fp32", "gn_apply generic down fp32",
    "input conv mma C128", "input conv mma C64", "input conv CUDA cores fp32 128-pixel tiles",
    "input conv CUDA cores fp16 128-pixel tiles",
    "combine vector C128", "combine vector C256", "combine scalar fp16 + channel_stats", "combine scalar fp32 + tile stats",
    "combine scalar fp32 + channel_stats",
    "out conv mma cp.async C128", "out conv mma cp.async C256", "out conv coop fp32 C128", "out conv coop fp32 C256",
}


def case_branches():
    b = [gn_rs_branch(_dt(c.dtype), c.rs, c.H, c.W, c.C) for c in GN_CASES]
    b += [input_conv_branch(_dt(c.dtype), c.H, c.W, c.C) for c in IN_CASES]
    b += [combine_branch(_dt(c.dtype), c.H, c.W, c.C) for c in CB_CASES]
    b += [out_conv_branch(_dt(c.dtype), c.C) for c in OC_CASES]
    return b


def test_cases_reach_every_dispatch_branch():
    got = collections.Counter(case_branches())
    assert not REQUIRED_BRANCHES - set(got), f"no case reaches {sorted(REQUIRED_BRANCHES - set(got))}"
    # the overflow cases run on both tiled kernels and the generic FIR-down
    large = {gn_rs_branch(F16, c.rs, c.H, c.W, c.C) for c in GN_CASES if c.kind == "large"}
    assert large == {"gn_apply tiled up", "gn_apply tiled down", "gn_apply generic down fp16"}
    # the long-clip bottom levels take the generic FIR in both directions, and the mma out conv runs partial tiles
    assert gn_rs_branch(F16, RS_DOWN, 8, 150, 256) == "gn_apply generic down fp16"
    assert gn_rs_branch(F16, RS_UP, 4, 75, 256) == "gn_apply generic up fp16"
    assert any(c.W % 16 and c.dtype == torch.float16 for c in OC_CASES)
    assert any(c.H < 16 and c.dtype == torch.float16 for c in OC_CASES)
