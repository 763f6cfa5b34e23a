"""Import shim for the *live* reference (build container only).

``/root/reference`` is mounted read-only in the build container and does not
exist on the GPU box; there the byte-for-byte staged copy ``oracle/_ref/`` is used
(``oracle/build_ref.py``, run by ``__graft_entry__.build()``; git-ignored, ships with the
gpurun snapshot).  ``sgmse.model`` / ``sgmse.data_module`` / ``sgmse.util.other``
import six packages that are not installed (pytorch_lightning, torch_ema, librosa,
pesq, pystoi, torch_pesq); none carries hot-path arithmetic (SURVEY.md §8c), so
inert stand-ins are injected into ``sys.modules`` before import.

Used by oracle/make_golden.py, tests/test_oracle_vs_reference.py, the ``-m gpu`` drop-in tests and the
CPU arm of bench.py.
TEST INFRASTRUCTURE – see oracle/__init__.py.
"""
from __future__ import annotations

import contextlib
import os
import sys
import types
from typing import List

import torch

_STAGED = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")


def _resolve_root() -> str:
    env = os.environ.get("SGMSE_REFERENCE_ROOT")
    if env:
        return env
    for cand in ("/root/reference", _STAGED):
        if os.path.isdir(os.path.join(cand, "sgmse")):
            return cand
    return "/root/reference"


REFERENCE_ROOT = _resolve_root()


def reference_available() -> bool:
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "sgmse"))


def reference_kind() -> str:
    """'live' = /root/reference itself, 'staged' = the oracle/_ref copy, 'none'."""
    if not reference_available():
        return "none"
    return "staged" if os.path.abspath(REFERENCE_ROOT) == os.path.abspath(_STAGED) else "live"


def _install_stubs():
    if "pytorch_lightning" not in sys.modules:
        pl = types.ModuleType("pytorch_lightning")

        class LightningModule(torch.nn.Module):
            def save_hyperparameters(self, *a, **k):
                pass

            def log(self, *a, **k):
                pass

        class LightningDataModule:
            def __init__(self, *a, **k):
                pass

        pl.LightningModule = LightningModule
        pl.LightningDataModule = LightningDataModule
        sys.modules["pytorch_lightning"] = pl
    if "torch_ema" not in sys.modules:
        m = types.ModuleType("torch_ema")

        class ExponentialMovingAverage:
            def __init__(self, params, decay):
                self.collected_params = None

            def update(self, *a):
                pass

            def store(self, *a):
                pass

            def copy_to(self, *a):
                pass

            def restore(self, *a):
                pass

            def to(self, *a, **k):
                pass

            def state_dict(self):
                return {}

            def load_state_dict(self, *a):
                pass

        m.ExponentialMovingAverage = ExponentialMovingAverage
        sys.modules["torch_ema"] = m
    for name, attrs in (("librosa", ["resample"]), ("pesq", ["pesq"]), ("pystoi", ["stoi"]),
                        ("torch_pesq", ["PesqLoss"])):
        if name not in sys.modules:
            m = types.ModuleType(name)
            for a in attrs:
                setattr(m, a, lambda *args, **kw: (_ for _ in ()).throw(RuntimeError(f"{name} stub")))
            sys.modules[name] = m


def import_reference(cuda_op: bool = False):
    """Returns the reference's ``sgmse`` package (imported from REFERENCE_ROOT).

    cuda_op=False (default): the reference stays a CPU checker -- its upfirdn2d CUDA op is JIT-compiled by
    ``torch.utils.cpp_extension.load`` at import time wherever ``torch.cuda.is_available()``
    (op/upfirdn2d.py:11-20), a minute of nvcc on every fresh GPU box; CUDA is hidden for the duration of the
    first import so CPU tensors take ``upfirdn2d_native`` exactly as in the build container.  cuda_op=True
    lets the JIT happen (the reference's own GPU path)."""
    if not reference_available():
        raise RuntimeError("reference not available at " + REFERENCE_ROOT)
    _install_stubs()
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    orig = torch.cuda.is_available
    if not cuda_op and "sgmse.backbones.ncsnpp_utils.op.upfirdn2d" not in sys.modules:
        torch.cuda.is_available = lambda: False
    try:
        import sgmse  # noqa
        import sgmse.model, sgmse.data_module, sgmse.sdes, sgmse.sampling, sgmse.backbones  # noqa
        import sgmse.util.other  # noqa
    finally:
        torch.cuda.is_available = orig
    return sgmse


def make_score_model(backbone="ncsnpp", seed=0, **kw):
    """ScoreModel with ``init_scale=1.0`` by default, ``eval()``-ed (EMA swap is a no-op stub)."""
    sg = import_reference()
    from sgmse.model import ScoreModel
    from sgmse.data_module import SpecsDataModule
    args = dict(backbone=backbone, sde="ouve", data_module_cls=SpecsDataModule, base_dir="/nonexistent",
                theta=1.5, sigma_min=0.05, sigma_max=0.5, init_scale=1.0)
    args.update(kw)
    torch.manual_seed(seed)
    model = ScoreModel(**args)
    model.eval()
    return model


@contextlib.contextmanager
def injected_noise(draws: List[torch.Tensor]):
    """Monkeypatch ``torch.randn_like`` so the reference sampler consumes ``draws`` in call order."""
    it = iter(draws)
    orig = torch.randn_like

    def fake(x, *a, **k):
        z = next(it)
        assert z.shape == x.shape and z.dtype == x.dtype, (z.shape, x.shape, z.dtype, x.dtype)
        return z.to(x.device)

    torch.randn_like = fake
    try:
        yield
    finally:
        torch.randn_like = orig
