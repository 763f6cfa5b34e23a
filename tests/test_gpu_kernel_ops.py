"""Op-level tests of the wgmma convolution (conv_tc), the GroupNorm statistics it writes, and the attention kernel.
Each kernel is compared elementwise with a float64 reference of the same operation.

The network-level tests compare a whole forward with the CPU oracle through a rel-L2 bound.  An error confined to a few
tiles disappears in that norm: one sample of a multi-sample pixel box, one consumer warpgroup, one slot of the GroupNorm
partials.  Here every output element has its own bound, derived from the kernel's rounding model.

tests/c/kernel_ops.cu is a small extern "C" shim over the product launchers.  It is linked against the objects that
sgmse_b200.build compiles for the engine library, with the same flags, so the kernels under test are the product's
object code.  The shim is linked -Bsymbolic and loaded RTLD_LOCAL, so it never binds to the engine library's copies of
the same symbols.  It runs on torch's current stream and reports the launch plan conv_tc_plan() chose.

The float64 references run on the GPU (torch), from the exact fp16 inputs and weights the kernels read.  Each case prints
max(err / bound) and its plan.  The mutation controls compare the same kernel output with a deliberately wrong reference
and require a failure by at least 10x the bound, so the bounds are not vacuous.
"""
import collections
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from sgmse_b200 import build as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM_SRC = os.path.join(ROOT, "tests", "c", "kernel_ops.cu")

# Kernel selection of the product.  The engine installs these per call in activate() (sgmse_b200/csrc/engine.cu), where
# option value 0 maps to g_tc1_narrow = 1, g_gn_self = 1, g_gnfin_variant = 1 and g_attn_variant = 0.  The switches
# default to 0 in the kernel sources, so the shim takes them as explicit arguments, and these are the defaults.
PRODUCT_TC1_NARROW = 1
PRODUCT_GN_SELF = 1
PRODUCT_GNFIN_VARIANT = 1
PRODUCT_ATTN_VARIANT = 0

H100_SMS = 132

U32 = 2.0 ** -24     # fp32 unit roundoff, round to nearest (CUDA-core fadd / fmul / fma)
ULP32 = 2.0 ** -23   # one fp32 ulp, relative: also covers an adder that truncates (tensor-core accumulation)

Plan = collections.namedtuple("Plan", "bw bh bn block_n stages tiles grid min_local max_local")


class KopsConv(C.Structure):
    _fields_ = [("N", C.c_int), ("H", C.c_int), ("W", C.c_int), ("Cout", C.c_int), ("out", C.c_void_p),
                ("stats", C.c_void_p), ("nseg", C.c_int), ("seg", C.c_void_p * 3), ("seg_c", C.c_int * 3),
                ("seg_taps", C.c_int * 3), ("w", C.c_void_p), ("w_ld", C.c_int), ("bias", C.c_void_p),
                ("temb", C.c_void_p), ("temb_stride", C.c_int), ("residual", C.c_void_p), ("scale", C.c_float),
                ("gn_ab", C.c_void_p), ("gn_cat", C.c_void_p), ("gn_cat_c", C.c_int)]


_I, _P = C.c_int, C.c_void_p
SIGNATURES = {
    "kops_conv_plan": [_I, _I, _I, _I, _I, _I, C.POINTER(C.c_int)],
    "kops_conv_tc": [_P, C.POINTER(KopsConv), _I, C.POINTER(C.c_int), C.POINTER(C.c_int)],
    "kops_gn_finalize": [_P, _I, _I, _I, _P, _I, _I, _P, _I, _I, _P, _P, _I, _P, _I],
    "kops_gn_norm_apply": [_P, _I, _I, _I, _P, _I, _P, _I, _P, _I, _P, _I, _P, _P, _I, _I, _P, _I],
    "kops_gn_apply": [_P, _I, _I, _I, _P, _I, _P, _I, _P, _I, _P],
    "kops_attention": [_P, _I, _I, _I, _P, _P, _I],
}


class KernelOps:
    def __init__(self, path):
        self.lib = C.CDLL(path, mode=os.RTLD_LOCAL)
        for name, args in SIGNATURES.items():
            fn = getattr(self.lib, name)
            fn.argtypes, fn.restype = args, C.c_int
        self.lib.kops_last_error.restype = C.c_char_p

    def _check(self, code):
        if code != 0:
            raise RuntimeError(f"kernel_ops: {self.lib.kops_last_error().decode()} (code {code})")

    def plan(self, N, H, W, C_out, sms=H100_SMS, narrow=PRODUCT_TC1_NARROW):
        p = (C.c_int * 9)()
        self._check(self.lib.kops_conv_plan(N, H, W, C_out, sms, narrow, p))
        return Plan(*p)

    def conv(self, args, narrow=PRODUCT_TC1_NARROW):
        p, slots = (C.c_int * 9)(), C.c_int()
        self._check(self.lib.kops_conv_tc(_stream(), C.byref(args), narrow, p, C.byref(slots)))
        return Plan(*p), slots.value

    def gn_finalize(self, shape, stats, C0, slots, gamma, beta, groups, ab, variant=PRODUCT_GNFIN_VARIANT):
        N, H, W = shape
        self._check(self.lib.kops_gn_finalize(_stream(), N, H, W, stats.data_ptr(), C0, slots, None, 0, 0,
                                              gamma.data_ptr(), beta.data_ptr(), groups, ab.data_ptr(), variant))

    def gn_norm_apply(self, x, stats, slots, gamma, beta, groups, out, silu=True, gn_self=PRODUCT_GN_SELF):
        N, H, W, C0 = x.shape
        self._check(self.lib.kops_gn_norm_apply(_stream(), N, H, W, x.data_ptr(), C0, stats.data_ptr(), slots, None, 0,
                                                None, 0, gamma.data_ptr(), beta.data_ptr(), groups, int(silu),
                                                out.data_ptr(), gn_self))

    def gn_apply(self, x, ab, out, silu=True):
        N, H, W, C0 = x.shape
        self._check(self.lib.kops_gn_apply(_stream(), N, H, W, x.data_ptr(), C0, None, 0, ab.data_ptr(), int(silu),
                                           out.data_ptr()))

    def attention(self, qkv, out, variant=PRODUCT_ATTN_VARIANT):
        N, S, C3 = qkv.shape
        self._check(self.lib.kops_attention(_stream(), N, S, C3 // 3, qkv.data_ptr(), out.data_ptr(), variant))


def _stream():
    return torch.cuda.current_stream().cuda_stream if torch.cuda.is_available() else None


def build_shim(outdir, src=SHIM_SRC):
    """Compile a shim (tests/c/*.cu) with the library's ARCH / CFLAGS and link it against the library's own objects."""
    B.build()
    objs = [os.path.join(B.LIBDIR, "obj", s.replace(".cu", ".o")) for s in B.SOURCES]
    if not all(os.path.exists(o) for o in objs):
        B.build(force=True)
    name = os.path.splitext(os.path.basename(src))[0]
    shim_o, so = os.path.join(outdir, name + ".o"), os.path.join(outdir, f"lib{name}.so")
    for cmd in ([B.NVCC, *B.ARCH, *B.CFLAGS, *B.PRODUCT_DEFS, "-I", B.CSRC, "-c", src, "-o", shim_o],
                [B.NVCC, *B.ARCH, "-shared", "-cudart", "static", "-o", so, shim_o, *objs, "-L" + B.CUDA_LIB, "-lcufft",
                 "-Xlinker", "-Bsymbolic", "-Xlinker", "-rpath," + B.CUDA_LIB]):
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
    return so


@pytest.fixture(scope="module")
def ops(tmp_path_factory):
    return KernelOps(build_shim(str(tmp_path_factory.mktemp("kernel_ops"))))


# ------------------------------------------------------------------------------------------------
# layouts shared by the host and GPU tests
# ------------------------------------------------------------------------------------------------
def pack_weights(ws, identity_tail=True):
    """conv_tc's weight operand: [Cout][ld] fp16, K-major, K ordered (segment, tap = 3 (dy + 1) + (dx + 1), cin).  ld
    includes the Cout x Cout identity block the engine appends after the real K columns (engine.cu: pack_conv)."""
    cout = ws[0].shape[0]
    cols = [w.permute(0, 2, 3, 1).reshape(cout, -1) for w in ws]      # [co][ky][kx][ci]: ky = dy + 1, kx = dx + 1
    if identity_tail:
        cols.append(torch.eye(cout, dtype=ws[0].dtype, device=ws[0].device))
    packed = torch.cat(cols, 1).contiguous()
    return packed, packed.shape[1]


def slot_sums(y, plan):
    """[N][slots][C][2] (sum, sum of squares) of y [N, H, W, C] over each bw x bh pixel box; slot = ty * tiles_w + tx."""
    N, H, W, Cc = y.shape
    th, tw = H // plan.bh, W // plan.bw
    t = y.reshape(N, th, plan.bh, tw, plan.bw, Cc)
    return torch.stack([t.sum((2, 4)), (t * t).sum((2, 4))], -1).reshape(N, th * tw, Cc, 2)


def conv_ref(xs, ws, absolute=False):
    """sum over segments of F.conv2d (pad 1 for 3x3), NHWC in and out, float64; absolute: the same over |x| and |w|."""
    acc = 0
    for x, w in zip(xs, ws):
        xd, wd = x.permute(0, 3, 1, 2).double(), w.double()
        if absolute:
            xd, wd = xd.abs(), wd.abs()
        acc = acc + F.conv2d(xd, wd, padding=w.shape[-1] // 2)
    return acc.permute(0, 2, 3, 1)


def ulp16(x):
    """Spacing of fp16 at magnitude x >= 0; below the normal range, the subnormal spacing 2^-24."""
    return torch.exp2(torch.floor(torch.log2(torch.clamp(x, min=2.0 ** -14))) - 10)


def ratio(got, ref, bound):
    """Elementwise |got - ref| / bound; a NaN (a canary the kernel never overwrote) counts as infinitely wrong."""
    return torch.nan_to_num((got.double() - ref).abs() / bound, nan=math.inf)


# ------------------------------------------------------------------------------------------------
# host tests
# ------------------------------------------------------------------------------------------------
def test_shim_compiles_and_links_for_sm90a(ops):
    """Builds without a GPU; launcher errors come back as codes with the message."""
    for name in SIGNATURES:
        assert hasattr(ops.lib, name)
    a = KopsConv(N=1, H=16, W=8, Cout=96, nseg=1, scale=1.0)
    with pytest.raises(RuntimeError, match="conv_tc: unsupported shape"):
        ops.conv(a)


@pytest.mark.parametrize("shape, narrow, expect", [
    # 256 x 64 level, T = 64, three utterances: single-sample 8 x 16 box, 128-wide tiles, 384 tiles over 132 CTAs
    ((3, 256, 64, 128), 1, Plan(8, 16, 1, 128, 4, 384, 132, 2, 3)),
    # 16 x 4 (T = 64): 64 pixels per sample -> two samples per box, the third in a half-empty box; few tiles -> 64-wide
    ((3, 16, 4, 256), 1, Plan(4, 16, 2, 64, 7, 8, 8, 1, 1)),
    ((3, 16, 4, 256), 0, Plan(4, 16, 2, 128, 4, 4, 4, 1, 1)),
    # 4 x 8 (T = 512): four samples per box
    ((5, 4, 8, 256), 1, Plan(8, 4, 4, 64, 7, 8, 8, 1, 1)),
    # Cout = 3 * 64: 64-wide tiles whatever the narrow switch says
    ((5, 128, 32, 192), 0, Plan(8, 16, 1, 64, 7, 480, 132, 3, 4)),
    # 8 x 2: no 128-pixel box of at least 32 pixels per sample
    ((2, 8, 2, 128), 1, Plan(0, 0, 0, 0, 0, 0, 0, 0, 0)),
])
def test_plan_for_product_shapes(ops, shape, narrow, expect):
    assert ops.plan(*shape, narrow=narrow) == expect


def emulate_conv_tc(xs, taps, packed, plan, cout):
    """conv_tc's implicit GEMM in numpy float64: 128-row tiles of box pixels x packed K columns, plus its stats slots."""
    N, H, W = xs[0].shape[:3]
    bw, bh, bn = plan.bw, plan.bh, plan.bn
    tiles_w, tiles_h, tiles_n = W // bw, H // bh, -(-N // bn)
    rps = bw * bh
    r = np.arange(128)
    px, py, pn = r % bw, (r // bw) % bh, r // rps
    out = np.zeros((N, H, W, cout))
    stats = np.zeros((N, tiles_w * tiles_h, cout, 2))
    for m in range(tiles_w * tiles_h * tiles_n):
        tx, ty, tn = m % tiles_w, (m // tiles_w) % tiles_h, m // (tiles_w * tiles_h)
        x, y, n = tx * bw + px, ty * bh + py, tn * bn + pn
        cols = []
        for src, t in zip(xs, taps):
            for tap in range(t):
                dy, dx = (tap // 3 - 1, tap % 3 - 1) if t == 9 else (0, 0)
                yy, xx = y + dy, x + dx
                inside = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H) & (n < N)
                a = np.zeros((128, src.shape[3]))
                a[inside] = src[n[inside], yy[inside], xx[inside]]
                cols.append(a)
        A = np.concatenate(cols, 1)
        D = A @ packed[:, :A.shape[1]].T
        valid = n < N
        out[n[valid], y[valid], x[valid]] = D[valid]
        for g in range(128 // rps if rps < 128 else 1):
            if tn * bn + g < N:
                rows = D[g * rps:(g + 1) * rps]
                stats[tn * bn + g, ty * tiles_w + tx] = np.stack([rows.sum(0), (rows * rows).sum(0)], -1)
    return out, stats


@pytest.mark.parametrize("N, H, W, segs", [
    (3, 16, 4, [(64, 9), (64, 1), (128, 1)]),      # two samples per box, the last box half past the batch
    (5, 4, 8, [(64, 9)]),                          # four samples per box
    (1, 32, 16, [(128, 1)]),                       # one sample, 2 x 2 slots
])
def test_packer_tap_order_and_slots_on_host(ops, N, H, W, segs):
    """The packer, tap order and slot layout the GPU tests rely on, against F.conv2d and direct per-box sums."""
    g = torch.Generator().manual_seed(N * 1000 + H)
    cout = 64
    plan = ops.plan(N, H, W, cout)
    xs = [torch.randn(N, H, W, c, generator=g, dtype=torch.float64) for c, _ in segs]
    ws = [torch.randn(cout, c, 3 if t == 9 else 1, 3 if t == 9 else 1, generator=g, dtype=torch.float64) for c, t in segs]
    packed, ld = pack_weights(ws)
    assert ld == sum(c * t for c, t in segs) + cout
    assert torch.equal(packed[:, ld - cout:], torch.eye(cout, dtype=torch.float64))
    got, got_stats = emulate_conv_tc([x.numpy() for x in xs], [t for _, t in segs], packed.numpy(), plan, cout)
    ref = conv_ref(xs, ws)
    np.testing.assert_allclose(got, ref.numpy(), rtol=1e-12, atol=1e-10)
    np.testing.assert_allclose(got_stats, slot_sums(ref, plan).numpy(), rtol=1e-12, atol=1e-9)
    # the same emulation with the segments' tap order reversed must disagree: the check can see a wrong tap order
    flipped = [torch.flip(w, (2, 3)) for w in ws]
    bad, _ = emulate_conv_tc([x.numpy() for x in xs], [t for _, t in segs], pack_weights(flipped)[0].numpy(), plan, cout)
    assert segs[0][1] == 1 or not np.allclose(bad, ref.numpy(), rtol=1e-6)


# ------------------------------------------------------------------------------------------------
# GPU: conv_tc
# ------------------------------------------------------------------------------------------------
PAD = 4096                 # canary elements on each side of an output (a multiple of 8: keeps TMA's 16-byte alignment)
CANARY16 = 0x7E5A          # an fp16 NaN
CANARY32 = 0x7FC0BEEF      # an fp32 NaN


class Guarded:
    """A tensor inside a larger buffer filled with a NaN canary; check() asserts nothing outside the tensor changed."""

    def __init__(self, shape, dtype):
        numel = math.prod(shape)
        self.bits = CANARY16 if dtype == torch.float16 else CANARY32
        self.int_dtype = torch.int16 if dtype == torch.float16 else torch.int32
        self.buf = torch.empty(numel + 2 * PAD, dtype=dtype, device="cuda")
        self.buf.view(self.int_dtype).fill_(self.bits)
        self.t = self.buf[PAD:PAD + numel].view(shape)
        self.numel = numel

    def check(self, what):
        b = self.buf.view(self.int_dtype)
        outside = torch.cat([b[:PAD], b[PAD + self.numel:]])
        assert bool((outside == self.bits).all()), f"{what}: wrote outside the tensor"


ConvCase = collections.namedtuple("ConvCase", "name N H W cout segs bias temb residual fused_cat fused")


def _case(name, N, H, W, cout, segs, bias=True, temb=None, residual=False, fused=False, fused_cat=0):
    return ConvCase(name, N, H, W, cout, segs, bias, temb, residual, fused_cat, fused)


# Product level shapes (full-size network: 256 frequency rows, T frames, levels 256 x T ... 4 x T/64; C 128 / 256) at
# T in {64, 128, 192, 512} and B in {1, 2, 3, 5}.
CONV_CASES = [
    _case("L0 T64 B3 3x3 128->128", 3, 256, 64, 128, [(128, 9)], temb="per"),
    _case("L0 T128 B1 3x3 128->128", 1, 256, 128, 128, [(128, 9)], bias=False, temb="shared"),
    _case("L1 T64 B5 3x3 64->192", 5, 128, 32, 192, [(64, 9)], temb="per"),
    _case("L0 T64 B5 1x1 64->64 kb=1", 5, 256, 64, 64, [(64, 1)], bias=False, temb="shared", residual=True),
    _case("16x4 T64 B3 bn=2 3x3 256->256", 3, 16, 4, 256, [(256, 9)], temb="per"),
    _case("16x12 T192 B5 bn=2 3 segments", 5, 16, 12, 256, [(256, 9), (256, 1), (256, 1)]),
    _case("8x4 T128 B3 bn=4 3x3 256->256", 3, 8, 4, 256, [(256, 9)], temb="per"),
    _case("4x8 T512 B5 bn=4 residual", 5, 4, 8, 256, [(256, 9)], bias=False, residual=True),
    _case("16x8 T128 B3 qkv 1x1 256->768", 3, 16, 8, 768, [(256, 1)]),
    _case("64x32 T128 B2 2 segments 256+128", 2, 64, 32, 256, [(256, 9), (128, 1)]),
    _case("32x16 T128 B2 3x3 512->256", 2, 32, 16, 256, [(512, 9)], temb="per"),
    _case("32x16 T128 B2 fused GN", 2, 32, 16, 256, [(256, 9)], temb="per", fused=True),
    _case("16x12 T192 B3 bn=2 fused GN + cat", 3, 16, 12, 256, [(256, 9)], temb="per", fused=True, fused_cat=256),
]
INV_SQRT2 = float(np.float32(1 / math.sqrt(2)))


def fused_operand(x, ab):
    """Segment 0 of the fused producer: fp16(silu(a * x + b)), emulated in fp32 arithmetic, and the allowance of the operands
    whose fp16 rounding the kernel may take the other way.

    The kernel evaluates z = fmaf(a, x, b) (exact product: fp32 x fp16 fits fp64) and silu_f(z) = __fdividef(z, 1 +
    __expf(-z)).  __expf errs by up to 2 + 1.17 |z| fp32 ulps, __fdividef by 2, so for |z| < 8 its fp32 silu lies within
    ~16 ulps of the exactly rounded one.  Only an operand whose fp32 value lies within that distance (taken as 64 ulps) of
    an fp16 rounding boundary can round to a different fp16 value, and then by one fp16 ulp.  Those operands are found
    here; the allowance is one fp16 ulp at the operand for them and 0 elsewhere."""
    a, b = ab[..., 0].double()[:, None, None, :], ab[..., 1].double()[:, None, None, :]
    z = (a * x.double() + b).float().double()
    s = (z / (1 + torch.exp(-z))).float().double()
    d = 64 * ULP32 * s.abs() + 2.0 ** -40
    near = (s - d).half() != (s + d).half()
    assert z.abs().max() < 8
    return s.half(), torch.where(near, ulp16(s.abs() + d), torch.zeros_like(s)), near


def launch_conv(ops, case, inputs, narrow=PRODUCT_TC1_NARROW):
    N, H, W, cout = case.N, case.H, case.W, case.cout
    out = Guarded((N, H, W, cout), torch.float16)
    stats = Guarded((N * (H * W // 32) * cout * 2,), torch.float32)   # the engine's capacity: N * (H*W/32) * C * 2 floats
    a = KopsConv(N=N, H=H, W=W, Cout=cout, out=out.t.data_ptr(), stats=stats.t.data_ptr(), nseg=len(case.segs),
                 w=inputs["packed"].data_ptr(), w_ld=inputs["ld"], scale=inputs["scale"])
    for i, (cin, taps) in enumerate(case.segs):
        a.seg[i], a.seg_c[i], a.seg_taps[i] = inputs["x"][i].data_ptr(), cin, taps
    if case.bias:
        a.bias = inputs["bias"].data_ptr()
    if case.temb:
        a.temb, a.temb_stride = inputs["temb_ptr"], inputs["temb_stride"]
    if case.residual:
        a.residual = inputs["res"].data_ptr()
    if case.fused:
        a.gn_ab = inputs["ab"].data_ptr()
        if case.fused_cat:
            a.gn_cat, a.gn_cat_c = inputs["cat"].data_ptr(), case.fused_cat
    plan, slots = ops.conv(a, narrow)
    torch.cuda.synchronize()
    out.check("conv_tc output")
    stats.check("conv_tc stats")
    return out, stats, plan, slots


def make_conv_inputs(case, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    N, H, W, cout = case.N, case.H, case.W, case.cout

    def randn(*shape, scale=1.0):
        return torch.randn(*shape, generator=g, device="cuda") * scale

    xs = [randn(N, H, W, cin).half() for cin, _ in case.segs]
    cins = [cin + (case.fused_cat if i == 0 and case.fused else 0) for i, (cin, _) in enumerate(case.segs)]
    ktot = sum(c * t for c, (_, t) in zip(cins, case.segs))
    ws = [randn(cout, c, 3 if t == 9 else 1, 3 if t == 9 else 1, scale=2 / math.sqrt(ktot)).half()
          for c, (_, t) in zip(cins, case.segs)]
    packed, ld = pack_weights(ws)
    inp = {"x": xs, "ws": ws, "packed": packed, "ld": ld, "ktot": ktot,
           "scale": INV_SQRT2 if case.residual or len(case.segs) > 1 else 1.0}
    inp["bias"] = randn(cout, scale=0.5)
    stride = cout + 64                                  # a wider table, read at a column offset like the engine's
    inp["temb_table"] = randn(N, stride)
    inp["temb_ptr"] = inp["temb_table"].data_ptr() + 32 * 4
    inp["temb_stride"] = stride if case.temb == "per" else 0
    inp["temb"] = (inp["temb_table"][:, 32:32 + cout] if case.temb == "per"
                   else inp["temb_table"][:1, 32:32 + cout].expand(N, cout))
    inp["res"] = randn(N, H, W, cout).half()
    if case.fused:
        ct = case.segs[0][0] + case.fused_cat
        inp["ab"] = torch.stack([0.5 + 0.5 * torch.rand(N, ct, generator=g, device="cuda"), randn(N, ct, scale=0.5)],
                                -1).contiguous()
        if case.fused_cat:
            inp["cat"] = randn(N, H, W, case.fused_cat).half()
        raw = torch.cat([xs[0], inp["cat"]], -1) if case.fused_cat else xs[0]
        inp["h"], inp["allow"], inp["near"] = fused_operand(raw, inp["ab"])
    return inp


def conv_reference(case, inp, ws=None, temb=None):
    """float64 reference and the elementwise bound of conv_tc's output."""
    ws = inp["ws"] if ws is None else ws
    ops_in = [inp["h"] if case.fused else inp["x"][0]] + inp["x"][1:]
    ref = conv_ref(ops_in, ws)
    absacc = conv_ref(ops_in, ws, absolute=True)
    extra = torch.zeros_like(ref)
    if case.bias:
        ref = ref + inp["bias"].double()
        extra = extra + inp["bias"].double().abs()
    if case.temb:
        t = (inp["temb"] if temb is None else temb).double()[:, None, None, :]
        ref, extra = ref + t, extra + t.abs()
    if case.residual:
        ref, extra = ref + inp["res"].double(), extra + inp["res"].double().abs()
    scale = inp["scale"]
    ref = ref * scale
    # Bound.  The fp16 x fp16 products are exact in fp32.  Each wgmma k16 step adds 16 products to the fp32 accumulator;
    # modelled as one multi-term adder that aligns the 17 addends to the largest and truncates, a step loses < 17 ulps
    # of a magnitude <= sum |a_i w_i| (the second float64 convolution, over |x| and |w|): 17 K / 16 ulps over K = ktot.
    # The epilogue adds bias, time embedding and residual and multiplies by scale in fp32: four more roundings of at
    # most one ulp of the running magnitude.  The fused producer adds one fp16 ulp per operand that may round the other
    # way (fused_operand), times |w|.  The fp16 store then rounds to nearest: half an fp16 ulp at the value, which is
    # at most |ref| + the error before rounding.
    pre = (17 * inp["ktot"] / 16 * ULP32) * absacc + 4 * ULP32 * (absacc + extra)
    if case.fused:
        pre = pre + conv_ref([inp["allow"]], [ws[0]], absolute=True)
    pre = abs(scale) * pre
    bound = pre + 0.5 * ulp16(ref.abs() + pre)
    return ref, bound


def stats_bounds(out16, plan):
    """Each slot's (sum, sum^2) is an fp32 sum of the bw*bh stored values of one sample, summed 32 rows at a time and then
    across the tile's 32-row segments: at most bw*bh roundings of u each, of the running sum <= sum |v| (sum v^2, with
    one more rounding for the square)."""
    a = slot_sums(out16.double().abs(), plan)
    n = plan.bw * plan.bh
    return torch.stack([(n + 1) * U32 * a[..., 0], (n + 2) * U32 * a[..., 1]], -1) + 1e-30


def check_stats(stats, out16, plan, slots, report):
    N, H, W, cout = out16.shape
    assert slots == (H // plan.bh) * (W // plan.bw)
    used = N * slots * cout * 2
    rest = stats.t[used:]
    assert bool(torch.isnan(rest).all()), "stats written past [N][slots][C][2]"
    st = stats.t[:used].view(N, slots, cout, 2).double()
    ref = slot_sums(out16.double(), plan)
    bnd = stats_bounds(out16, plan)
    per_slot = ratio(st, ref, bnd).max().item()
    totals = ratio(st.sum(1), ref.sum(1), bnd.sum(1)).max().item()
    # mutation control: one slot dropped from the sum over slots
    dropped = ratio(st[:, 1:].sum(1), ref.sum(1), bnd.sum(1)).max().item()
    report["stats"] = max(report.get("stats", 0), per_slot, totals)
    report.setdefault("stats mutation", []).append(dropped)
    assert per_slot <= 1 and totals <= 1, f"stats err/bound per slot {per_slot:.3g}, summed over slots {totals:.3g}"
    assert dropped >= 10, f"stats mutation (slot dropped) only {dropped:.3g} x the bound"
    return st, bnd


def check_groupnorm(ops, out16, st, bnd, slots, seed, report):
    """gn_finalize's (a, b) and gn_norm_apply's output against float64 GroupNorm (eps 1e-6) of the stored conv output;
    gn_norm_apply against gn_finalize + gn_apply bitwise where its claim of bit-identity holds."""
    N, H, W, Cc = out16.shape
    groups = min(Cc // 4, 32)
    cpg = Cc // groups
    g = torch.Generator(device="cuda").manual_seed(seed)
    gamma = (1 + 0.1 * torch.randn(Cc, generator=g, device="cuda")).contiguous()
    beta = (0.1 * torch.randn(Cc, generator=g, device="cuda")).contiguous()
    stats_c = st.float().contiguous()
    ab = Guarded((N, Cc, 2), torch.float32)
    ops.gn_finalize((N, H, W), stats_c, Cc, slots, gamma, beta, groups, ab.t)
    y = Guarded((N, H, W, Cc), torch.float16)
    ops.gn_norm_apply(out16, stats_c, slots, gamma, beta, groups, y.t)
    y2 = Guarded((N, H, W, Cc), torch.float16)
    ops.gn_apply(out16, ab.t, y2.t)
    torch.cuda.synchronize()
    ab.check("gn_finalize")
    y.check("gn_norm_apply")
    y2.check("gn_apply")

    x = out16.double()
    xg = x.reshape(N, H * W, groups, cpg)
    cnt = H * W * cpg
    mean = xg.mean((1, 3))
    var = (xg * xg).mean((1, 3)) - mean * mean
    rstd = 1 / torch.sqrt(var + 1e-6)
    gam, bet = gamma.double(), beta.double()
    a_ref = gam * rstd.repeat_interleave(cpg, 1)
    m_c = mean.repeat_interleave(cpg, 1)
    b_ref = bet - m_c * a_ref
    # Bound of (a, b).  E_s, E_q: the summed stats bounds of the group (the fp64 sums of the partials add nothing
    # measurable).  mean = s / cnt and var = q / cnt - mean^2 in fp64 then err by dm = E_s / cnt and
    # dv = E_q / cnt + (2 |mean| + dm) dm.  1 / sqrt over [v - dv, v + dv] moves by at most dv / (2 (v - dv)) relative;
    # rstd's cast to fp32 and a = gamma * rstd add one rounding each.  b = beta - fp32(mean) * a: the roundings of mean,
    # of the product and of the difference, plus the propagated |mean| da + |a| dm.
    E = bnd.reshape(N, slots, groups, cpg, 2).sum((1, 3))
    dm = E[..., 0] / cnt
    dv = E[..., 1] / cnt + (2 * mean.abs() + dm) * dm
    v = var + 1e-6
    assert bool((dv < v / 2).all())
    rel = (dv / (2 * (v - dv)) + 2 * U32).repeat_interleave(cpg, 1)
    da = a_ref.abs() * rel
    db = m_c.abs() * da + a_ref.abs() * dm.repeat_interleave(cpg, 1) + 3 * U32 * ((m_c * a_ref).abs() + bet.abs())
    got = ab.t.double()
    r_ab = max(ratio(got[..., 0], a_ref, da).max().item(), ratio(got[..., 1], b_ref, db).max().item())
    # Bound of silu(a x + b).  z = fmaf(a, x, b) errs by |x| da + db plus one rounding; |silu'| <= 1.1; silu_f's
    # __expf / __fdividef add (2 + 1.17 |z|) + 2 fp32 ulps (relative, taken as 6 + 1.2 |z|); the fp16 store half an ulp.
    z = a_ref[:, None, None, :] * x + b_ref[:, None, None, :]
    y_ref = z * torch.sigmoid(z)
    dz = x.abs() * da[:, None, None, :] + db[:, None, None, :] + 2 * U32 * z.abs()
    pre = 1.1 * dz + (6 + 1.2 * z.abs()) * ULP32 * y_ref.abs()
    bound = pre + 0.5 * ulp16(y_ref.abs() + pre)
    r_y = max(ratio(y.t, y_ref, bound).max().item(), ratio(y2.t, y_ref, bound).max().item())
    report["groupnorm"] = max(report.get("groupnorm", 0), r_ab, r_y)
    assert r_ab <= 1 and r_y <= 1, f"GroupNorm err/bound: (a, b) {r_ab:.3g}, output {r_y:.3g}"
    bitwise = cpg * slots <= 32
    if bitwise:
        assert torch.equal(y.t.view(torch.int16), y2.t.view(torch.int16)), "gn_norm_apply != gn_finalize + gn_apply"
    return bitwise


@pytest.mark.gpu
def test_conv_tc_against_fp64(ops):
    """Every conv case elementwise against float64, with its stats, GroupNorm on its output, the mutation controls, the
    determinism and tile-width claims, and the canaries.  Then the coverage of the launch plans the cases reached."""
    report, plans, failures = {}, [], []
    narrow_differs = gn_bitwise = 0
    for i, case in enumerate(CONV_CASES):
        try:
            inp = make_conv_inputs(case, 100 + i)
            out, stats, plan, slots = launch_conv(ops, case, inp)
            kb = inp["ktot"] // 64
            plans.append((case, plan, kb))
            ref, bound = conv_reference(case, inp)
            r = ratio(out.t, ref, bound).max().item()
            report["conv"] = max(report.get("conv", 0), r)
            muts = {}
            if any(t == 9 for _, t in case.segs):              # tap (dy, dx) = (-1, -1) of the 3x3 segment dropped
                ws = [w.clone() for w in inp["ws"]]
                ws[0][:, :, 0, 0] = 0
                muts["tap dropped"] = ratio(out.t, conv_reference(case, inp, ws=ws)[0], bound).max().item()
            if case.temb == "per":                              # samples 0 and 1 take each other's time embedding
                muts["temb rows swapped"] = ratio(out.t, conv_reference(case, inp, temb=inp["temb"][[1, 0] + list(
                    range(2, case.N))])[0], bound).max().item()
            extra = f", fused operands near an fp16 boundary {inp['near'].float().mean().item():.2%}" if case.fused else ""
            print(f"[conv] {case.name}: plan {plan._asdict()} k_blocks {kb} slots {slots}: max err/bound {r:.3g}, "
                  f"mutations {({k: round(v, 1) for k, v in muts.items()})}{extra}")
            assert r <= 1, f"err/bound {r:.3g}"
            for k, v in muts.items():
                report.setdefault("conv mutation", []).append(v)
                assert v >= 10, f"mutation '{k}' only {v:.3g} x the bound"
            st, bnd = check_stats(stats, out.t, plan, slots, report)
            # two identical launches: bit-identical output and stats (deterministic: no atomics)
            out2, stats2, _, _ = launch_conv(ops, case, inp)
            assert torch.equal(out.buf.view(torch.int16), out2.buf.view(torch.int16)), "relaunch changed the output"
            assert torch.equal(stats.buf.view(torch.int32), stats2.buf.view(torch.int32)), "relaunch changed the stats"
            # 64- and 128-wide channel tiles: bit-identical output and stats
            if case.cout % 128 == 0:
                out3, stats3, plan3, _ = launch_conv(ops, case, inp, narrow=1 - PRODUCT_TC1_NARROW)
                if plan3.block_n != plan.block_n:
                    narrow_differs += 1
                    assert torch.equal(out.buf.view(torch.int16), out3.buf.view(torch.int16)), "tile width changed the output"
                    assert torch.equal(stats.buf.view(torch.int32), stats3.buf.view(torch.int32)), "tile width changed the stats"
            gn_bitwise += check_groupnorm(ops, out.t, st, bnd, slots, 200 + i, report)
        except AssertionError as e:
            failures.append(f"{case.name}: {e}")
    print(f"[conv] worst err/bound: conv {report.get('conv', 0):.3g}, stats {report.get('stats', 0):.3g}, "
          f"GroupNorm {report.get('groupnorm', 0):.3g}; weakest mutation: conv {min(report.get('conv mutation', [0])):.3g}, "
          f"stats {min(report.get('stats mutation', [0])):.3g}")
    assert not failures, "\n".join(failures)

    # coverage of the launch plans
    bns = {p.bn for _, p, _ in plans}
    partial = {p.bn for c, p, _ in plans if c.N % p.bn}
    widths = {(p.block_n, p.stages) for _, p, _ in plans}
    local = {p.max_local for _, p, _ in plans} | {p.min_local for _, p, _ in plans}
    missing = []
    if not ({1, 2, 4} <= bns and {2, 4} <= partial):
        missing.append(f"boxes of 1, 2, 4 samples with a partial 2- and 4-sample box (have {bns}, partial {partial})")
    if not {(64, 7), (128, 4)} <= widths:
        missing.append(f"64-wide tiles with 7 stages and 128-wide with 4 (have {widths})")
    if not ({1, 2} <= local and any(n >= 3 and n % 2 for n in local)):
        missing.append(f"1, 2 and an odd number >= 3 of local tiles per CTA (have {local})")
    if not any(p.block_n == 64 and p.max_local > 1 for _, p, _ in plans):
        missing.append("64-wide tiles with more than one tile per CTA")
    if not any(kb == 1 for _, _, kb in plans) or not any(kb < p.stages for _, p, kb in plans) or \
            not any(kb > p.stages and kb % p.stages for _, p, kb in plans):
        missing.append("k_blocks = 1, k_blocks < stages and k_blocks > stages not a multiple of it")
    if not any(len(c.segs) == 3 for c in CONV_CASES) or not any(c.fused and c.fused_cat for c in CONV_CASES):
        missing.append("three K segments and the fused producer with a concatenated input")
    if not narrow_differs or not gn_bitwise:
        missing.append(f"the tile-width ({narrow_differs}) and gn_norm_apply bit-identity ({gn_bitwise}) comparisons")
    assert not missing, "the conv cases no longer reach: " + "; ".join(missing)


# ------------------------------------------------------------------------------------------------
# GPU: attention
# ------------------------------------------------------------------------------------------------
def attention_reference(qkv, keys=None):
    """float64 softmax(q k^T / sqrt(C)) v and the elementwise bound of the mma.sync flash kernel."""
    N, S, C3 = qkv.shape
    Cc = C3 // 3
    q, k, v = (t.double() for t in qkv.split(Cc, -1))
    if keys is not None:
        k, v = k[:, :keys], v[:, :keys]
    s = q @ k.transpose(1, 2) / math.sqrt(Cc)
    w = torch.softmax(s, -1)
    ref = w @ v
    # Bound.  Scores: an fp32 tensor-core sum of C exact fp16 products (C ulps of sum |q_c k_c|) scaled by the fp32
    # constant log2(e) / sqrt(C) (two roundings).  A score error ds perturbs the softmax weights by a factor within
    # exp(+-2 ds) (numerator and normalizer), bounded by 2 ds + (2 ds)^2.  exp2f adds 2 ulps per weight.  P is rounded
    # to fp16 for the P V product (half an ulp, relative 2^-11, or 2^-25 absolute below the normal range), while l sums
    # the unrounded P.  The P V product and l are fp32 sums over S keys; the per-tile rescaling by exp2(m_old - m_new)
    # adds a rounding per key tile; the final 1 / l and product two more.  Then the fp16 store: half an ulp.
    ds = (Cc * ULP32 * (q.abs() @ k.abs().transpose(1, 2)) / math.sqrt(Cc) + 2 * U32 * s.abs()).amax(-1, keepdim=True)
    w1 = w @ v.abs()
    l = torch.exp(s - s.amax(-1, keepdim=True)).sum(-1, keepdim=True)
    S_eff = s.shape[-1]
    rel = 2 * ds + (2 * ds) ** 2 + 2 * ULP32 + 2.0 ** -11 + (S_eff + 2 * math.ceil(S_eff / 64) + 4) * ULP32
    pre = w1 * rel + 2.0 ** -25 * v.abs().sum(1, keepdim=True) / l
    return ref, pre + 0.5 * ulp16(ref.abs() + pre)


@pytest.mark.gpu
def test_attention_against_fp64(ops):
    worst, weakest, failures = 0.0, math.inf, []
    for S in (4, 12, 24, 32, 96, 128, 192, 512):
        for Cc in (128, 256):
            N = 3 if S in (12, 96) else 2
            g = torch.Generator(device="cuda").manual_seed(S * 1000 + Cc)
            qkv = (1.5 * torch.randn(N, S, 3 * Cc, generator=g, device="cuda")).half()
            out = Guarded((N, S, Cc), torch.float16)
            ops.attention(qkv, out.t)
            alt = Guarded((N, S, Cc), torch.float16)
            ops.attention(qkv, alt.t, variant=3)
            torch.cuda.synchronize()
            out.check("attention")
            alt.check("attention (plain staging)")
            ref, bound = attention_reference(qkv)
            r = ratio(out.t, ref, bound).max().item()
            worst = max(worst, r)
            msg = f"[attention] S {S} C {Cc} N {N}: max err/bound {r:.3g}"
            try:
                assert r <= 1, f"S {S} C {Cc}: err/bound {r:.3g}"
                assert torch.equal(out.t.view(torch.int16), alt.t.view(torch.int16)), f"S {S} C {Cc}: attn_variant 3 differs"
                if S > 64:                                       # mutation control: the last key tile dropped
                    m = ratio(out.t, attention_reference(qkv, keys=(S - 1) // 64 * 64)[0], bound).max().item()
                    weakest = min(weakest, m)
                    msg += f", last key tile dropped {m:.3g}"
                    assert m >= 10, f"S {S} C {Cc}: mutation only {m:.3g} x the bound"
            except AssertionError as e:
                failures.append(str(e))
            print(msg)
    print(f"[attention] worst err/bound {worst:.3g}; weakest mutation {weakest:.3g}")
    assert not failures, "\n".join(failures)
