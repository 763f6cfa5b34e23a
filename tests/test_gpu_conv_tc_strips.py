"""GPU tests of the wgmma convolution's dy-halo strips (conv_tc.cu, conv_tc_sched.h).

A 3x3 segment over a single-sample pixel box bw x bh with bw % 8 == 0 and (bh + 2) bw <= 160 takes its A operand from
one bw x (bh + 2) strip per (dx, channel chunk), which serves the three dy taps.  These cases add what the op-level
cases of tests/test_gpu_kernel_ops.py lack: the 16 x 8 box (20 KB strips), 3x3 inputs of 1, 3 and 6 channel chunks, a
strip segment followed by two 1x1 segments with a residual, and a TF32 strip case.  Every output element is checked
against the float64 bound of test_gpu_kernel_ops.conv_reference (test_gpu_kernel_ops_tf32.reference for TF32), relaunch
and 64- vs 128-wide tiles bit for bit, and a reference with dy = -1 and dy = +1 swapped in one column of taps must fail.
"""
import pytest
import torch

import test_gpu_kernel_ops_tf32 as k32
from test_gpu_kernel_ops import (PRODUCT_TC1_NARROW, _case, conv_reference, launch_conv, make_conv_inputs, ops,  # noqa: F401
                                 ratio)
from test_gpu_kernel_ops_tf32 import ops32  # noqa: F401
from test_conv_tc_strips_host import strip_rows

CASES = [
    _case("8x16 T128 B3 16x8 box 3x3 256->256", 3, 8, 16, 256, [(256, 9)], temb="per"),
    _case("L0 T64 B2 3x3 64->128 (1 chunk)", 2, 256, 64, 128, [(64, 9)], temb="shared"),
    _case("L1 T64 B2 3x3 192->128 (3 chunks)", 2, 128, 32, 128, [(192, 9)], temb="per"),
    _case("32x16 T128 B2 3x3 384->256 (6 chunks)", 2, 32, 16, 256, [(384, 9)], bias=False),
    _case("64x32 T128 B2 strip + 1x1 + 1x1 residual", 2, 64, 32, 128, [(128, 9), (128, 1), (64, 1)], residual=True),
    _case("16x4 T64 B3 bn=2 per-tap boxes", 3, 16, 4, 128, [(128, 9)], temb="per"),
]

TF32_CASES = [
    k32._case("8x16 T128 B2 TF32 16x8 box 3x3 128->128", 2, 8, 16, 128, [(128, 9)], temb="per"),
    k32._case("64x32 T128 B2 TF32 strip + 1x1 residual", 2, 64, 32, 128, [(128, 9), (64, 1)], residual=True),
]


def dy_swapped(ws, kx=0):
    """The 3x3 weights with taps dy = -1 and dy = +1 exchanged in column kx = dx + 1."""
    bad = [w.clone() for w in ws]
    bad[0][:, :, 0, kx], bad[0][:, :, 2, kx] = ws[0][:, :, 2, kx], ws[0][:, :, 0, kx]
    return bad


@pytest.mark.gpu
def test_strip_convolutions_against_fp64(ops):
    rows_seen, failures = [], []
    for i, case in enumerate(CASES):
        try:
            inp = make_conv_inputs(case, 700 + i)
            out, _, plan, _ = launch_conv(ops, case, inp)
            rows = strip_rows(plan.bw, plan.bh, plan.bn, case.segs[0][1])
            rows_seen.append(rows)
            ref, bound = conv_reference(case, inp)
            r = ratio(out.t, ref, bound).max().item()
            mut = ratio(out.t, conv_reference(case, inp, ws=dy_swapped(inp["ws"]))[0], bound).max().item()
            print(f"[strips] {case.name}: plan {plan._asdict()} strip rows {rows}: max err/bound {r:.3g}, "
                  f"dy swapped {mut:.3g}")
            assert r <= 1, f"err/bound {r:.3g}"
            assert mut >= 10, f"dy-swap mutation only {mut:.3g} x the bound"
            out2, _, _, _ = launch_conv(ops, case, inp)
            assert torch.equal(out.buf.view(torch.int16), out2.buf.view(torch.int16)), "relaunch changed the output"
            if case.cout % 128 == 0:
                out3, _, plan3, _ = launch_conv(ops, case, inp, narrow=1 - PRODUCT_TC1_NARROW)
                assert torch.equal(out.buf.view(torch.int16), out3.buf.view(torch.int16)), "tile width changed the output"
        except AssertionError as e:
            failures.append(f"{case.name}: {e}")
    assert not failures, "\n".join(failures)
    assert {144, 160} <= set(rows_seen) and 0 in rows_seen, f"cases reach strip rows {sorted(set(rows_seen))}"


@pytest.mark.gpu
def test_tf32_strip_convolutions_against_fp64(ops32):
    for i, case in enumerate(TF32_CASES):
        inp = k32.make_inputs(case, 800 + i)
        out, _, plan, _ = k32.launch(ops32, case, inp)
        assert strip_rows(plan.bw, plan.bh, plan.bn, case.segs[0][1]) > 0
        ref, bound = k32.reference(case, inp)
        r = ratio(out.t, ref, bound).max().item()
        mut = ratio(out.t, k32.reference(case, inp, ws=dy_swapped(inp["ws"]))[0], bound).max().item()
        print(f"[strips tf32] {case.name}: plan {plan._asdict()}: max err/bound {r:.3g}, dy swapped {mut:.3g}")
        assert r <= 1, f"{case.name}: err/bound {r:.3g}"
        assert mut >= 10, f"{case.name}: dy-swap mutation only {mut:.3g} x the bound"
        out2, _, _, _ = k32.launch(ops32, case, inp)
        assert torch.equal(out.buf.view(torch.int32), out2.buf.view(torch.int32)), "relaunch changed the output"
