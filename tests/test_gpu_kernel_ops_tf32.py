"""Op-level tests of the wgmma convolution with TF32 operands (conv_tc on fp32 activations, mode tf32_tc) and the GroupNorm
statistics it writes, element by element against a float64 reference.

tests/c/kernel_ops_tf32.cu is a small extern "C" shim over launch_conv_tc with fp32 tensor descriptors, linked against the
objects sgmse_b200.build compiles for the engine library (as tests/c/kernel_ops.cu is), so the kernel under test is the
product's object code.  The layouts, canaries and stats checks are those of tests/test_gpu_kernel_ops.py.

The reference is float64 F.conv2d of the operands the tensor cores actually multiply: the activations as TF32 (the upper
19 bits of the fp32 value: the hardware ignores the 13 low mantissa bits of an fp32 operand, i.e. truncates) and the
weights as packed (already TF32 values, rounded to nearest by the packer).  Each case prints max(err / bound), and also the
error against the same reference with round-to-nearest activations, so a run shows which operand model the hardware
follows.  The mutation controls compare the kernel output with a deliberately wrong reference and require a failure by at
least 10x the bound.
"""
import collections
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_kernel_ops import (H100_SMS, INV_SQRT2, ULP32, Guarded, Plan, build_shim, check_stats, conv_ref, emulate_conv_tc,
                                 ratio, slot_sums)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM_SRC = os.path.join(ROOT, "tests", "c", "kernel_ops_tf32.cu")


class KopsConvTf32(C.Structure):
    _fields_ = [("N", C.c_int), ("H", C.c_int), ("W", C.c_int), ("Cout", C.c_int), ("out", C.c_void_p),
                ("stats", C.c_void_p), ("nseg", C.c_int), ("seg", C.c_void_p * 3), ("seg_c", C.c_int * 3),
                ("seg_taps", C.c_int * 3), ("w", C.c_void_p), ("w_ld", C.c_int), ("bias", C.c_void_p),
                ("temb", C.c_void_p), ("temb_stride", C.c_int), ("residual", C.c_void_p), ("scale", C.c_float)]


_I, _P = C.c_int, C.c_void_p
SIGNATURES = {
    "kops_tf32_conv_plan": [_I, _I, _I, _I, _I, C.POINTER(C.c_int)],
    "kops_tf32_conv_tc": [_P, C.POINTER(KopsConvTf32), C.POINTER(C.c_int), C.POINTER(C.c_int)],
    "kops_tf32_rna": [_P, _P, C.c_longlong],
}


class KernelOpsTf32:
    def __init__(self, path):
        self.lib = C.CDLL(path, mode=os.RTLD_LOCAL)
        for name, args in SIGNATURES.items():
            fn = getattr(self.lib, name)
            fn.argtypes, fn.restype = args, C.c_int
        self.lib.kops_tf32_last_error.restype = C.c_char_p

    def _check(self, code):
        if code != 0:
            raise RuntimeError(f"kernel_ops_tf32: {self.lib.kops_tf32_last_error().decode()} (code {code})")

    def plan(self, N, H, W, C_out, sms=H100_SMS):
        p = (C.c_int * 9)()
        self._check(self.lib.kops_tf32_conv_plan(N, H, W, C_out, sms, p))
        return Plan(*p)

    def conv(self, args):
        p, slots = (C.c_int * 9)(), C.c_int()
        stream = torch.cuda.current_stream().cuda_stream if torch.cuda.is_available() else None
        self._check(self.lib.kops_tf32_conv_tc(stream, C.byref(args), p, C.byref(slots)))
        return Plan(*p), slots.value

    def host_rna(self, x):
        """The engine's host packer rounding (tf32_rna) of a float32 numpy array."""
        x = np.ascontiguousarray(x, dtype=np.float32)
        out = np.empty_like(x)
        self._check(self.lib.kops_tf32_rna(x.ctypes.data, out.ctypes.data, x.size))
        return out


@pytest.fixture(scope="module")
def ops32(tmp_path_factory):
    return KernelOpsTf32(build_shim(str(tmp_path_factory.mktemp("kernel_ops_tf32")), SHIM_SRC))


# ------------------------------------------------------------------------------------------------
# TF32 operand models (torch, any device)
# ------------------------------------------------------------------------------------------------
def tf32_trunc(x):
    """fp32 -> TF32 by dropping the 13 low mantissa bits (how the tensor cores read an fp32 activation)."""
    return (x.float().contiguous().view(torch.int32) & -8192).view(torch.float32)


def tf32_rna(x):
    """fp32 -> nearest TF32, ties away from zero (the packer's tf32_rna; finite inputs)."""
    return ((x.float().contiguous().view(torch.int32) + 4096) & -8192).view(torch.float32)


def pack_weights_tf32(ws):
    """conv_tc's TF32 weight operand: [Cout][ktot] fp32 TF32 values, K-major, K ordered (segment, tap, cin); no identity
    tail (the residual is added in fp32 by the epilogue)."""
    cout = ws[0].shape[0]
    packed = torch.cat([w.permute(0, 2, 3, 1).reshape(cout, -1) for w in ws], 1)
    return tf32_rna(packed).contiguous(), packed.shape[1]


def unpack_weights(packed, segs, cout):
    """The packed operand back to Conv2d weights [cout][cin][k][k] per segment."""
    ws, k0 = [], 0
    for cin, taps in segs:
        k = 3 if taps == 9 else 1
        ws.append(packed[:, k0:k0 + taps * cin].reshape(cout, k, k, cin).permute(0, 3, 1, 2).contiguous())
        k0 += taps * cin
    return ws


# ------------------------------------------------------------------------------------------------
# host tests
# ------------------------------------------------------------------------------------------------
def test_tf32_shim_builds_plans_and_rejects(ops32):
    for name in SIGNATURES:
        assert hasattr(ops32.lib, name)
    # fp32 tiles are 64 wide with a 6-stage ring whatever the channel count
    assert ops32.plan(3, 256, 64, 128) == Plan(8, 16, 1, 64, 6, 768, 132, 5, 6)
    assert ops32.plan(3, 16, 4, 256) == Plan(4, 16, 2, 64, 6, 8, 8, 1, 1)
    a = KopsConvTf32(N=1, H=16, W=8, Cout=96, nseg=1, scale=1.0)
    with pytest.raises(RuntimeError, match="conv_tc: unsupported shape"):
        ops32.conv(a)


def test_host_packer_rounding_is_rna():
    """tf32_rna (the engine's host and device packers) against an independent float64 round-half-away to 10 bits."""
    g = np.random.default_rng(5)
    x = np.concatenate([g.standard_normal(20000).astype(np.float32) * np.float32(10.0) ** g.integers(-30, 30, 20000),
                        np.float32([0.0, -0.0, 1.0, -1.0, 1 + 2.0 ** -11, -(1 + 2.0 ** -11), 1 + 3 * 2.0 ** -11,
                                    2.0 ** -130, 65504.0])]).astype(np.float32)
    m, e = np.frexp(x.astype(np.float64))                      # |m| in [0.5, 1): 11 significant bits = 2^11 m
    want = np.where(x == 0, x, np.ldexp(np.sign(m) * np.floor(np.abs(m) * 2.0 ** 11 + 0.5), e - 11)).astype(np.float32)
    sub = np.abs(x) < np.float32(2.0 ** -126)                    # subnormals: the integer rounding rounds the raw field
    got = tf32_rna(torch.from_numpy(x)).numpy()
    assert np.array_equal(got[~sub], want[~sub])
    assert np.array_equal(got.view(np.int32) & 8191, np.zeros_like(got.view(np.int32)))


def test_host_packer_matches_the_c_implementation(ops32):
    g = np.random.default_rng(7)
    x = (g.standard_normal(50000) * 3).astype(np.float32)
    assert np.array_equal(ops32.host_rna(x).view(np.int32), tf32_rna(torch.from_numpy(x)).numpy().view(np.int32))


@pytest.mark.parametrize("N, H, W, segs", [
    (3, 16, 4, [(64, 9), (32, 1), (128, 1)]),      # two samples per box, the last box half past the batch
    (5, 4, 8, [(32, 9)]),                          # four samples per box
    (1, 32, 16, [(96, 1)]),                        # one sample, 2 x 2 slots, K = 3 k-blocks of 32
])
def test_tf32_implicit_gemm_emulation_on_host(ops32, N, H, W, segs):
    """numpy float64 emulation of the TF32 implicit GEMM: truncated activations times the packed RNA weights over the
    packed [Cout][ktot] fp32 layout, against F.conv2d on the same TF32-reduced operands, with the stats slots."""
    g = torch.Generator().manual_seed(N * 100 + H)
    cout = 64
    plan = ops32.plan(N, H, W, cout)
    xs = [torch.randn(N, H, W, c, generator=g) for c, _ in segs]
    ws = [torch.randn(cout, c, 3 if t == 9 else 1, 3 if t == 9 else 1, generator=g) / math.sqrt(c * t) for c, t in segs]
    packed, ld = pack_weights_tf32(ws)
    assert ld == sum(c * t for c, t in segs) and packed.dtype == torch.float32
    assert bool(((packed.view(torch.int32) & 8191) == 0).all())
    xt = [tf32_trunc(x) for x in xs]
    got, got_stats = emulate_conv_tc([x.double().numpy() for x in xt], [t for _, t in segs], packed.double().numpy(), plan, cout)
    ref = conv_ref(xt, unpack_weights(packed, segs, cout))
    np.testing.assert_allclose(got, ref.numpy(), rtol=1e-12, atol=1e-10)
    np.testing.assert_allclose(got_stats, slot_sums(ref, plan).numpy(), rtol=1e-12, atol=1e-9)
    # the TF32 reduction is visible at this precision: full fp32 operands give a different result
    full = conv_ref(xs, ws).numpy()
    assert np.abs(full - got).max() > 1e-5


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
ConvCase = collections.namedtuple("ConvCase", "name N H W cout segs bias temb residual res_scale")


def _case(name, N, H, W, cout, segs, bias=True, temb=None, residual=False, res_scale=1.0):
    return ConvCase(name, N, H, W, cout, segs, bias, temb, residual, res_scale)


# Product level shapes of the full-size network (256 frequency rows, T frames; C 128 / 256) in fp32.  k_blocks = taps x
# cin / 32; the ring has 6 stages.
CONV_CASES = [
    _case("L0 T64 B3 3x3 128->128", 3, 256, 64, 128, [(128, 9)], temb="per"),                    # 5-6 tiles per CTA
    _case("L0 T128 B1 3x3 no bias", 1, 256, 128, 128, [(128, 9)], bias=False, temb="shared"),   # 3-4 tiles per CTA
    _case("L1 T64 B3 3x3 128->128", 3, 128, 32, 128, [(128, 9)], temb="per"),                    # 1-2 tiles per CTA
    _case("L0 T64 B5 1x1 64->64 kb=2 residual", 5, 256, 64, 64, [(64, 1)], bias=False, temb="shared", residual=True),
    _case("L0 T64 B2 1x1 32->64 kb=1", 2, 256, 64, 64, [(32, 1)], temb="per"),
    _case("16x4 T64 B3 bn=2 3x3 256->256", 3, 16, 4, 256, [(256, 9)], temb="per"),
    _case("16x12 T192 B5 bn=2 3 segments", 5, 16, 12, 256, [(256, 9), (256, 1), (256, 1)]),     # kb 88: 88 % 6 = 4
    _case("8x4 T128 B3 bn=4 3x3 256->256", 3, 8, 4, 256, [(256, 9)], temb="per"),
    _case("4x8 T512 B5 bn=4 residual", 5, 4, 8, 256, [(256, 9)], bias=False, residual=True),
    _case("16x8 T128 B3 qkv 1x1 256->768", 3, 16, 8, 768, [(256, 1)]),                           # kb 8
    _case("64x32 T128 B2 2 segments 256+128", 2, 64, 32, 256, [(256, 9), (128, 1)]),
    _case("64x32 T128 B2 residual x 1e4", 2, 64, 32, 128, [(128, 9)], temb="per", residual=True, res_scale=1e4),
]


def make_inputs(case, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    N, H, W, cout = case.N, case.H, case.W, case.cout

    def randn(*shape, scale=1.0):
        return torch.randn(*shape, generator=g, device="cuda") * scale

    xs = [randn(N, H, W, cin) for cin, _ in case.segs]                # full fp32: the kernel sees them as TF32
    ktot = sum(c * t for c, t in case.segs)
    ws = [randn(cout, c, 3 if t == 9 else 1, 3 if t == 9 else 1, scale=2 / math.sqrt(ktot)) for c, t in case.segs]
    packed, ld = pack_weights_tf32(ws)
    inp = {"x": xs, "xt": [tf32_trunc(x) for x in xs], "xr": [tf32_rna(x) for x in xs],
           "ws": unpack_weights(packed, case.segs, cout), "packed": packed, "ld": ld, "ktot": ktot,
           "scale": INV_SQRT2 if case.residual or len(case.segs) > 1 else 1.0}
    inp["bias"] = randn(cout, scale=0.5)
    stride = cout + 64
    inp["temb_table"] = randn(N, stride)
    inp["temb_ptr"] = inp["temb_table"].data_ptr() + 32 * 4
    inp["temb_stride"] = stride if case.temb == "per" else 0
    inp["temb"] = (inp["temb_table"][:, 32:32 + cout] if case.temb == "per"
                   else inp["temb_table"][:1, 32:32 + cout].expand(N, cout))
    inp["res"] = randn(N, H, W, cout, scale=case.res_scale)
    return inp


def launch(ops32, case, inp):
    N, H, W, cout = case.N, case.H, case.W, case.cout
    out = Guarded((N, H, W, cout), torch.float32)
    stats = Guarded((N * (H * W // 32) * cout * 2,), torch.float32)
    a = KopsConvTf32(N=N, H=H, W=W, Cout=cout, out=out.t.data_ptr(), stats=stats.t.data_ptr(), nseg=len(case.segs),
                     w=inp["packed"].data_ptr(), w_ld=inp["ld"], scale=inp["scale"])
    for i, (cin, taps) in enumerate(case.segs):
        a.seg[i], a.seg_c[i], a.seg_taps[i] = inp["x"][i].data_ptr(), cin, taps
    if case.bias:
        a.bias = inp["bias"].data_ptr()
    if case.temb:
        a.temb, a.temb_stride = inp["temb_ptr"], inp["temb_stride"]
    if case.residual:
        a.residual = inp["res"].data_ptr()
    plan, slots = ops32.conv(a)
    torch.cuda.synchronize()
    out.check("conv_tc (TF32) output")
    stats.check("conv_tc (TF32) stats")
    return out, stats, plan, slots


def reference(case, inp, xs=None, ws=None, temb=None, res=None):
    """float64 reference from the TF32 operands, and the elementwise bound of conv_tc's fp32 output."""
    xs = inp["xt"] if xs is None else xs
    ws = inp["ws"] if ws is None else ws
    ref = conv_ref(xs, ws)
    absacc = conv_ref(xs, ws, absolute=True)
    extra = torch.zeros_like(ref)
    if case.bias:
        ref, extra = ref + inp["bias"].double(), extra + inp["bias"].double().abs()
    if case.temb:
        t = (inp["temb"] if temb is None else temb).double()[:, None, None, :]
        ref, extra = ref + t, extra + t.abs()
    if case.residual:
        r = (inp["res"] if res is None else res).double()
        ref, extra = ref + r, extra + r.abs()
    scale = inp["scale"]
    ref = ref * scale
    # Bound.  TF32 x TF32 products (11-bit significands) are exact in fp32.  Each wgmma k8 step adds 8 products to the
    # fp32 accumulator; modelled as one multi-term adder that aligns the 9 addends to the largest and truncates, a step
    # loses < 9 ulps of a magnitude <= sum |a_i w_i| (the float64 convolution over |x| and |w|): 9 K / 8 ulps over
    # K = ktot.  The epilogue adds bias, time embedding and the fp32 residual and multiplies by scale in fp32: four more
    # roundings of at most one ulp of the running magnitude.  The output is stored as fp32: no further rounding.
    pre = (9 * inp["ktot"] / 8 * ULP32) * absacc + 4 * ULP32 * (absacc + extra)
    return ref, abs(scale) * pre + 1e-30


@pytest.mark.gpu
def test_conv_tc_tf32_against_fp64(ops32):
    report, plans, failures = {}, [], []
    for i, case in enumerate(CONV_CASES):
        try:
            inp = make_inputs(case, 300 + i)
            out, stats, plan, slots = launch(ops32, case, inp)
            kb = inp["ktot"] // 32
            plans.append((case, plan, kb))
            ref, bound = reference(case, inp)
            r = ratio(out.t, ref, bound).max().item()
            err_t = (out.t.double() - ref).abs().mean().item()
            err_r = (out.t.double() - reference(case, inp, xs=inp["xr"])[0]).abs().mean().item()
            report["conv"] = max(report.get("conv", 0), r)
            report.setdefault("operand model", []).append((err_t, err_r))
            muts = {}
            if any(t == 9 for _, t in case.segs):
                ws = [w.clone() for w in inp["ws"]]
                ws[0][:, :, 0, 0] = 0
                muts["tap dropped"] = ratio(out.t, reference(case, inp, ws=ws)[0], bound).max().item()
            if case.temb == "per" and case.N > 1:
                muts["temb rows swapped"] = ratio(out.t, reference(case, inp, temb=inp["temb"][[1, 0] + list(
                    range(2, case.N))])[0], bound).max().item()
            if case.residual and case.res_scale > 1:            # the residual through a TF32 operand
                muts["residual as TF32"] = ratio(out.t, reference(case, inp, res=tf32_trunc(inp["res"]))[0],
                                                 bound).max().item()
            print(f"[conv tf32] {case.name}: plan {plan._asdict()} k_blocks {kb} slots {slots}: max err/bound {r:.3g}, "
                  f"mean |err| truncated-operand model {err_t:.3g}, round-to-nearest model {err_r:.3g}, "
                  f"mutations {({k: round(v, 1) for k, v in muts.items()})}")
            assert r <= 1, f"err/bound {r:.3g}"
            for k, v in muts.items():
                report.setdefault("conv mutation", []).append(v)
                assert v >= 10, f"mutation '{k}' only {v:.3g} x the bound"
            check_stats(stats, out.t, plan, slots, report)
            out2, stats2, _, _ = launch(ops32, case, inp)
            assert torch.equal(out.buf.view(torch.int32), out2.buf.view(torch.int32)), "relaunch changed the output"
            assert torch.equal(stats.buf.view(torch.int32), stats2.buf.view(torch.int32)), "relaunch changed the stats"
        except AssertionError as e:
            failures.append(f"{case.name}: {e}")
    model = report.get("operand model", [])
    print(f"[conv tf32] worst err/bound: conv {report.get('conv', 0):.3g}, stats {report.get('stats', 0):.3g}; weakest "
          f"mutation: conv {min(report.get('conv mutation', [0])):.3g}, stats {min(report.get('stats mutation', [0])):.3g}; "
          f"cases closer to the truncated-operand model: {sum(t < r for t, r in model)} of {len(model)}")
    assert not failures, "\n".join(failures)
    # the activations enter the tensor cores truncated, as the reference above assumes
    assert all(t < r for t, r in model), f"the hardware does not follow the truncated-operand model: {model}"

    bns = {p.bn for _, p, _ in plans}
    partial = {p.bn for c, p, _ in plans if c.N % p.bn}
    local = {p.max_local for _, p, _ in plans} | {p.min_local for _, p, _ in plans}
    missing = []
    if not ({1, 2, 4} <= bns and {2, 4} <= partial):
        missing.append(f"boxes of 1, 2, 4 samples with a partial 2- and 4-sample box (have {bns}, partial {partial})")
    if {(p.block_n, p.stages) for _, p, _ in plans} != {(64, 6)}:
        missing.append("64-wide tiles with 6 stages only")
    if not ({1, 2} <= local and any(n >= 3 and n % 2 for n in local)):
        missing.append(f"1, 2 and an odd number >= 3 of local tiles per CTA (have {local})")
    if not any(kb == 1 for _, _, kb in plans) or not any(kb < p.stages for _, p, kb in plans) or \
            not any(kb > p.stages and kb % p.stages for _, p, kb in plans):
        missing.append("k_blocks = 1, k_blocks < stages and k_blocks > stages not a multiple of it")
    if not {1, 2, 3} <= {len(c.segs) for c in CONV_CASES}:
        missing.append("one, two and three K segments")
    if not ({"per", "shared"} <= {c.temb for c in CONV_CASES} and any(not c.bias for c in CONV_CASES)
            and any(c.residual and c.res_scale > 1 for c in CONV_CASES)):
        missing.append("shared and per-sample time embedding, no bias, a large residual")
    assert not missing, "the conv cases no longer reach: " + "; ".join(missing)
