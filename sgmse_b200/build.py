"""In-tree build of libsgmse_b200.so (nvcc, sm_90a only).

    python -m sgmse_b200.build [--force] [--pdl]

The shared library lands in ``sgmse_b200/lib/`` (git-ignored build product).  CUDA runtime is linked
statically; cuFFT dynamically (``libcufft.so.11`` from the toolkit, rpath'ed).
"""
from __future__ import annotations

import concurrent.futures
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIBNAME = "libsgmse_b200.so"
SOURCES = ["gn.cu", "conv_direct.cu", "conv_tc.cu", "small.cu", "attn.cu", "misc.cu", "pack.cu", "ode.cu", "engine.cu"]
HEADERS = ["common.cuh", "kernels.h", "conv_tc_sched.h", "engine.h", "rk45.h", os.path.join("..", "..", "include", "sgmse_b200.h")]

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUDA_LIB = os.environ.get("CUDA_LIB", "/usr/local/cuda/lib64")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
          "--expt-relaxed-constexpr", "-diag-suppress", "177"]


# the PDL twin: the product sources with -DSGMSE_B200_PDL (programmatic dependent launch); never loaded unless SGMSE_B200_PDL=1
PDL_LIBNAME = "libsgmse_b200_pdl.so"
PRODUCT_DEFS: list = []                # see DESIGN.md section 3 (programmatic dependent launch)


def lib_path(pdl: bool = False) -> str:
    return os.path.join(LIBDIR, PDL_LIBNAME if pdl else LIBNAME)


def _digest(extra: str = "") -> str:
    h = hashlib.sha256()
    h.update(extra.encode())
    for f in SOURCES + HEADERS:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(ARCH + CFLAGS + PRODUCT_DEFS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False, pdl: bool = False) -> str:
    """Default library: no PDL instruction in its SASS.  pdl=True builds the A/B twin libsgmse_b200_pdl.so
    (select it at run time with SGMSE_B200_PDL=1, then ``Engine.set_option("pdl", 1)``)."""
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, "build_pdl.stamp" if pdl else "build.stamp")
    dig = _digest("pdl" if pdl else "")
    out = lib_path(pdl)
    defs = ["-DSGMSE_B200_PDL"] if pdl else PRODUCT_DEFS
    if not force and os.path.exists(out) and os.path.exists(stamp) and open(stamp).read() == dig:
        return out
    objdir = os.path.join(LIBDIR, "obj_pdl" if pdl else "obj")
    os.makedirs(objdir, exist_ok=True)

    def compile_one(src):
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [NVCC, *ARCH, *CFLAGS, *defs, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose and (r.stdout or r.stderr):
            print(r.stdout, r.stderr, file=sys.stderr)
        return obj

    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [NVCC, *ARCH, "-shared", "-cudart", "static", "-o", out, *objs,
           "-L" + CUDA_LIB, "-lcufft", "-Xlinker", "-rpath," + CUDA_LIB]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as fh:
        fh.write(dig)
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True, pdl="--pdl" in sys.argv))
