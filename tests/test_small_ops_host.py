"""Host checks of tests/test_gpu_small_ops.py: the shim builds for sm_90a, the kernel selection the op tests assume is the
one the engine installs, and the tiled fp16 FIR-down's half2 arithmetic (emulated in float64 with an fp16 rounding per
operation) stays finite and inside the bound the GPU test uses.

The emulation evaluates the row and column expressions of gn.cu's FIR-down branch as they stand in the source, so it
follows the kernel.  The earlier form h2_fma(K1, h2_add(t1, t2), h2_mul(K0, h2_add(t0, t3))) added two taps before
weighting them: two in-range fp16 values of 32760 or more summed to inf, although the filtered value is at most the largest
tap.  test_adding_taps_before_weighting_overflows keeps that failure in view.
"""
import os
import re

import numpy as np
import pytest
import torch

import test_gpu_kernel_ops as kops
import test_gpu_small_ops as sops_t
from test_gpu_small_ops import RS_DOWN, SHIM_SRC, SIGNATURES, SmallOps, build_shim, f16x2_fir_bound

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "sgmse_b200", "csrc")


def test_shim_compiles_and_links_for_sm90a(tmp_path):
    ops = SmallOps(build_shim(str(tmp_path), SHIM_SRC))
    for name in SIGNATURES:
        assert hasattr(ops.lib, name)
    with pytest.raises(RuntimeError, match="fir4: nothing to do"):
        ops._check(ops.lib.sops_fir4(None, 1, 8, 8, 0, None, None, 1.0))


def test_product_kernel_selection_matches_activate():
    """The PRODUCT_* constants of the op tests against the defaults activate() installs for option value 0."""
    src = open(os.path.join(CSRC, "engine.cu")).read()
    body = re.search(r"static void activate\(.*?\n\}", src, re.S).group(0)
    defaults = {m.group(1): int(m.group(2)) for m in re.finditer(r"g_(\w+) = xl\(o\.\w+, (\d+), \d+\);", body)}
    assert defaults == {
        "fir_variant": sops_t.PRODUCT_FIR_VARIANT, "outconv_variant": sops_t.PRODUCT_OUTCONV_VARIANT,
        "inconv_variant": sops_t.PRODUCT_INCONV_VARIANT, "combine_variant": sops_t.PRODUCT_COMBINE_VARIANT,
        "tc1_narrow": kops.PRODUCT_TC1_NARROW, "gn_self": kops.PRODUCT_GN_SELF, "gnfin_variant": kops.PRODUCT_GNFIN_VARIANT,
    }
    # attn_variant passes through: option value 0 is kernel 0
    assert re.search(r"g_attn_variant = o\.attn_variant;", body) and kops.PRODUCT_ATTN_VARIANT == 0


# ------------------------------------------------------------------------------------------------
# emulation of the half2 FIR-down
# ------------------------------------------------------------------------------------------------
def h2_mul(a, b):
    return (a.astype(np.float64) * b).astype(np.float16)


def h2_add(a, b):
    return (a.astype(np.float64) + b).astype(np.float16)


def h2_fma(a, b, c):
    # one rounding to fp16: a * b (fp16 x fp16) is exact in float64, and where + c is not, c exceeds a * b by 2^40
    return (a.astype(np.float64) * b + c).astype(np.float16)


K0, K1 = np.float16(0.125), np.float16(0.375)
SHIPPED_ROW = "h2_fma(K1, h2_add(t1, t2), h2_mul(K0, h2_add(t0, t3)))"


def source_fir_down_forms():
    """The row and column expressions of gn.cu's half2 FIR-down, with the [q] lane index dropped."""
    src = open(os.path.join(CSRC, "gn.cu")).read()
    branch = src[src.index("if constexpr (FAST && RS == RS_DOWN)"):src.index("else if constexpr (MODE == 2 && RS == RS_UP)")]
    row = re.search(r"rr\[q\] = (.+);", branch).group(1)
    col = re.search(r"oo\[q\] = (.+);", branch).group(1)
    clean = lambda e: re.sub(r"(\w+)\[q\]", r"\1", e)
    return clean(row), clean(col).replace("r0", "t0").replace("r1", "t1").replace("r2", "t2").replace("r3", "t3")


def emulate_fir_down(x16, row, col):
    """The tiled kernel's FIR-down of a staged fp16 image x16 [..., H, W] (zero padding of one pixel): the row expression
    over the taps 2X-1 .. 2X+2 of every padded row, then the column expression over rows 2Y-1 .. 2Y+2."""
    p = np.pad(x16, [(0, 0)] * (x16.ndim - 2) + [(1, 1), (1, 1)])
    env = {"h2_fma": h2_fma, "h2_mul": h2_mul, "h2_add": h2_add, "K0": K0, "K1": K1}
    with np.errstate(over="ignore"):
        r = eval(row, env, {f"t{j}": p[..., :, j:p.shape[-1] - 3 + j:2] for j in range(4)})
        return eval(col, env, {f"t{i}": r[..., i:r.shape[-2] - 3 + i:2, :] for i in range(4)})


def ratio_to_bound(x16, y16):
    x = torch.from_numpy(x16.astype(np.float64))[None]
    ref = sops_t.fir_down2(x)[0].numpy()
    bound = f16x2_fir_bound(torch.zeros_like(x), x.abs(), RS_DOWN)[0].numpy()
    with np.errstate(invalid="ignore"):
        return np.nan_to_num(np.abs(y16.astype(np.float64) - ref) / bound, nan=np.inf)


def overflow_case():
    """One channel at [33000, 60000] among normal ones (the GPU test's overflow case)."""
    g = np.random.default_rng(11)
    x = (g.standard_normal((4, 16, 32)) * 3).astype(np.float16)
    x[0] = g.uniform(33000, 60000, (16, 32)).astype(np.float16)
    return x


def test_source_fir_down_is_finite_and_inside_the_bound_on_in_range_values():
    row, col = source_fir_down_forms()
    y = emulate_fir_down(overflow_case(), row, col)
    assert np.isfinite(y).all(), f"the FIR-down of gn.cu ({row}) overflows on in-range fp16 values"
    assert ratio_to_bound(overflow_case(), y).max() <= 1


def test_adding_taps_before_weighting_overflows():
    y = emulate_fir_down(overflow_case(), SHIPPED_ROW, SHIPPED_ROW)
    assert np.isinf(y[0]).any() and np.isfinite(y[1:]).all()


@pytest.mark.parametrize("seed", range(4))
def test_source_fir_down_inside_the_bound_on_random_values(seed):
    """Magnitudes from the fp16 subnormals to 6e4, both signs, ties and cancellation."""
    g = np.random.default_rng(seed)
    mag = 2.0 ** g.uniform(-26, 15.8, (8, 24, 40))
    x = (np.sign(g.standard_normal(mag.shape)) * mag).astype(np.float16)
    x[1] = g.integers(-4, 5, x[1].shape).astype(np.float16) * np.float16(0.25)
    x[2] = np.abs(x[2])
    row, col = source_fir_down_forms()
    r = ratio_to_bound(x, emulate_fir_down(x, row, col))
    print(f"seed {seed}: max err/bound {r.max():.3g}")
    assert r.max() <= 1
