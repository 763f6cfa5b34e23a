"""Host tests (no GPU) of the tf32_tc mode: fp32 activations with the convolutions on the wgmma kernel with TF32 operands.
The kernel-level numerics are in tests/test_gpu_kernel_ops_tf32.py, the network-level ones in tests/test_gpu_tf32.py."""
import os
import re
import subprocess

import pytest

from sgmse_b200 import Engine, EngineConfig, build as B


@pytest.fixture(scope="module")
def lib():
    return B.build()


def test_library_builds_with_the_tf32_wgmma_instruction(lib):
    assert os.path.exists(lib)
    obj = os.path.join(B.LIBDIR, "obj", "conv_tc.o")
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    fp32_kernel = [f for f in re.split(r"\s+Function : ", sass) if re.match(r"\S*conv_tc_kernel\S*Lb0EfEE", f)]
    assert len(fp32_kernel) == 1, "the TF32 instantiation of conv_tc_kernel is missing"
    assert "HGMMA.64x64x8.F32.TF32" in fp32_kernel[0]


def test_tf32_instantiation_does_not_spill():
    r = subprocess.run([B.NVCC, *B.ARCH, *B.CFLAGS, *B.PRODUCT_DEFS, "-Xptxas", "-v", "-c", os.path.join(B.CSRC, "conv_tc.cu"),
                        "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    # ptxas prints "Compiling entry function '<name>'", then its properties: stack frame and spills
    blocks = re.split(r"Compiling entry function ", r.stderr)
    tf32 = [b for b in blocks if re.match(r"'\S*conv_tc_kernel\S*Lb0EfEE", b)]
    assert len(tf32) == 1
    assert re.search(r"0 bytes spill stores, 0 bytes spill loads", tf32[0]), tf32[0]
    print(re.search(r"Used \d+ registers", tf32[0]).group(0))


def test_engine_accepts_tf32_tc_and_refuses_unknown_modes(lib):
    eng = Engine(EngineConfig(mode="tf32_tc", max_batch=2))
    assert eng.cfg.mode == "tf32_tc"
    with pytest.raises(ValueError):
        Engine(EngineConfig(mode="tf64_tc"))
    # an out-of-range enum value through the C ABI
    from sgmse_b200 import _lib
    cfg = EngineConfig(max_batch=2).to_c()
    cfg.mode = 4
    import ctypes as C
    h = C.c_void_p()
    assert _lib.load().sgmse_b200_create(C.byref(cfg), C.byref(h)) != 0
    assert b"unknown mode 4" in _lib.load().sgmse_b200_last_error()


@pytest.mark.parametrize("B_, T", [(1, 64), (4, 256), (2, 512)])
def test_workspace_equals_fp32_mode(lib, B_, T):
    """fp32 storage: the same activation workspace as fp32 mode (the TF32 weight copy is part of the weights)."""
    w = {m: Engine(EngineConfig(mode=m, max_batch=B_)).workspace_bytes(B_, 256, T) for m in ("fp32", "tf32_tc", "fp16_tc")}
    assert w["tf32_tc"] == w["fp32"]
    assert w["tf32_tc"] > 1.5 * w["fp16_tc"]
