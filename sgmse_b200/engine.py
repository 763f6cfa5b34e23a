"""Python host side of the engine: a thin object over the C-ABI (sgmse_b200/_lib.py).

PyTorch is used here only as the owner of device memory and streams; all arithmetic happens in
libsgmse_b200.so.  Mirrors the argument names/meaning of the reference interfaces it stands behind
(``ScoreModel.get_pc_sampler`` /root/reference/sgmse/model.py:348-368, ``ScoreModel.enhance`` :426-465,
``NCSNpp.forward`` backbones/ncsnpp.py:256).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib

MODES = {"fp32": 0, "fp16_direct": 1, "fp16_tc": 2, "tf32_tc": 3}
PREDICTORS = {"reverse_diffusion": 0, "euler_maruyama": 1, "none": 2}
CORRECTORS = {"ald": 0, "langevin": 1, "none": 2}
PAD_MODES = {"zero_pad": 0, "reflection": 1}
BACKBONES = {"ncsnpp": 0, "ncsnpp_48k": 1, "ncsnpp_v2": 2}
SDES = {"ouve": 0, "sbve": 1}
LOSS_TYPES = {"score_matching": 0, "denoiser": 1, "data_prediction": 2}
NETWORK_SCALINGS = {None: 0, "1/sigma": 1, "1/t": 2}
C_IN = {"1": 0, "edm": 1}
C_OUT = {"1": 0, "sigma": 1, "1/sigma": 2, "edm": 3}
C_SKIP = {"0": 0, "edm": 1}
SAMPLER_KINDS = {"pc": 0, "sb_ode": 1, "sb_sde": 2}
TRANSFORMS = {"exponent": 0, "log": 1, "none": 2}


def _lookup(table: Dict[str, int], name: str, what: str) -> int:
    # same error behaviour as Registry.get_by_name (/root/reference/sgmse/util/registry.py:25-30)
    if name in table:
        return table[name]
    raise ValueError(f"{what} with name '{name}' unknown.")


@dataclass
class EngineConfig:
    backbone: str = "ncsnpp"                       # 'ncsnpp' | 'ncsnpp_48k' | 'ncsnpp_v2'
    nf: int = 128
    ch_mult: Sequence[int] = (1, 1, 2, 2, 2, 2, 2)
    num_res_blocks: int = 2
    attn_resolutions: Sequence[int] = (16,)
    image_size: int = 256
    progressive: str = "output_skip"
    progressive_input: str = "input_skip"
    scale_by_sigma: bool = True
    theta: float = 1.5
    sigma_min: float = 0.05
    sigma_max: float = 0.5
    t_eps: float = 0.03
    n_fft: int = 510
    hop_length: int = 128
    window: str = "hann"
    spec_factor: float = 0.15
    spec_abs_exponent: float = 0.5
    transform_type: str = "exponent"               # SpecsDataModule --transform_type (data_module.py:118): 'exponent' | 'log' | 'none'
    sr: int = 16000
    mode: str = "fp16_tc"
    max_batch: int = 8
    use_graphs: bool = True
    # SDE registry name (sdes.py:144 'ouve', :235 'sbve') + SBVESDE parameters
    sde: str = "ouve"
    sb_k: float = 2.6
    sb_c: float = 0.4
    sb_eps: float = 1e-8
    # ScoreModel attributes of the 'ncsnpp_v2' branch of forward (model.py:52-60, 283-341); argparse strings as in the reference
    loss_type: str = "score_matching"
    network_scaling: Optional[str] = None
    c_in: str = "1"
    c_out: str = "1"
    c_skip: str = "0"
    sigma_data: float = 0.1
    # NCSNpp / NCSNpp_48k --no-centered (ncsnpp.py:45-47): the network maps its input to 2x - 1 (ncsnpp.py:288-290)
    centered: bool = True

    @staticmethod
    def ncsnpp_v2(**kw) -> "EngineConfig":
        # same module list as 'ncsnpp', no in-network /t (ncsnpp_v2.py:241-395)
        base = dict(backbone="ncsnpp_v2", scale_by_sigma=False)
        base.update(kw)
        return EngineConfig(**base)

    @staticmethod
    def ncsnpp_16k(**kw) -> "EngineConfig":
        return EngineConfig(**kw)

    @staticmethod
    def ncsnpp_48k(**kw) -> "EngineConfig":
        # README.md:89 of the reference (EARS-WHAM): --backbone ncsnpp_48k --n_fft 1534 --hop_length 384 ...
        base = dict(backbone="ncsnpp_48k", attn_resolutions=(), progressive="none", progressive_input="none",
                    theta=2.0, sigma_min=0.1, sigma_max=1.0, n_fft=1534, hop_length=384, spec_factor=0.065,
                    spec_abs_exponent=0.667, sr=48000)
        base.update(kw)
        return EngineConfig(**base)

    def to_c(self) -> _lib.Config:
        if self.backbone not in BACKBONES:
            raise ValueError(f"Backbone with name '{self.backbone}' unknown.")
        if self.backbone == "ncsnpp_v2" and self.scale_by_sigma:
            raise ValueError("'ncsnpp_v2' has no in-network scaling (scale_by_sigma must be False)")
        if self.progressive not in ("output_skip", "none") or self.progressive_input not in ("input_skip", "none"):
            raise NotImplementedError("only progressive in {output_skip, none} / progressive_input in {input_skip, none}")
        if len(self.ch_mult) > 8 or len(self.attn_resolutions) > 8:
            raise ValueError("at most 8 levels / attention resolutions")
        c = _lib.Config()
        c.backbone = BACKBONES[self.backbone]
        c.nf = self.nf
        c.num_levels = len(self.ch_mult)
        for i, m in enumerate(self.ch_mult):
            c.ch_mult[i] = int(m)
        c.num_res_blocks = self.num_res_blocks
        c.num_attn_resolutions = len(self.attn_resolutions)
        for i, r in enumerate(self.attn_resolutions):
            c.attn_resolutions[i] = int(r)
        c.image_size = self.image_size
        c.progressive_output_skip = int(self.progressive == "output_skip")
        c.progressive_input_skip = int(self.progressive_input == "input_skip")
        c.scale_by_sigma = int(self.scale_by_sigma)
        c.theta, c.sigma_min, c.sigma_max, c.t_eps = self.theta, self.sigma_min, self.sigma_max, self.t_eps
        c.n_fft, c.hop_length = self.n_fft, self.hop_length
        c.sqrt_window = int(_lookup({"hann": 0, "sqrthann": 1}, self.window, "Window"))
        c.spec_factor, c.spec_abs_exponent, c.sample_rate = self.spec_factor, self.spec_abs_exponent, self.sr
        c.mode = _lookup(MODES, self.mode, "Mode")
        c.max_batch = self.max_batch
        c.use_graphs = int(self.use_graphs)
        c.sde_kind = _lookup(SDES, self.sde, "SDE")
        c.sb_k, c.sb_c, c.sb_eps = self.sb_k, self.sb_c, self.sb_eps
        c.loss_type = _lookup(LOSS_TYPES, self.loss_type, "Loss type")
        c.network_scaling = _lookup(NETWORK_SCALINGS, self.network_scaling, "Network scaling")
        c.c_in = _lookup(C_IN, self.c_in, "c_in type")
        c.c_out = _lookup(C_OUT, self.c_out, "c_out type")
        c.c_skip = _lookup(C_SKIP, self.c_skip, "c_skip type")
        c.sigma_data = self.sigma_data
        c.transform_type = _lookup(TRANSFORMS, self.transform_type, "Transform type")
        if not self.centered and self.backbone == "ncsnpp_v2":
            raise ValueError("'ncsnpp_v2' has no --no-centered option (centered must be True)")
        c.not_centered = int(not self.centered)
        return c


def rk45_host(fun, t_span, y0, rtol=1e-3, atol=1e-6, max_attempts=0):
    """``scipy.integrate.solve_ivp(fun, t_span, y0, method='RK45', rtol=rtol, atol=atol)`` on the controller the device
    ODE sampler runs (csrc/rk45.h) with ``fun`` as a host callback.  Host-only.  ``y0``: complex array [n].
    Returns ``(y(t_bound) complex128 [n], nfev, {"steps", "rejected", "status"})``."""
    import numpy as np
    lib = _lib.load()
    y = np.ascontiguousarray(np.asarray(y0).astype(np.complex128).reshape(-1))
    n = y.size

    def rhs(t, yp, dp, nn, _user):
        if nn == 0:
            return
        yy = np.ctypeslib.as_array(yp, shape=(2 * nn,)).view(np.complex128)
        d = np.ctypeslib.as_array(dp, shape=(2 * nn,)).view(np.complex128)
        d[:] = np.asarray(fun(t, yy.copy()), dtype=np.complex128)

    cb = _lib.ODE_RHS(rhs)
    nfev = C.c_int()
    stats = (C.c_int * 4)()
    _lib.check(lib.sgmse_b200_rk45_host(cb, None, float(t_span[0]), float(t_span[1]), y.ctypes.data, n, float(rtol),
                                        float(atol), int(max_attempts), C.byref(nfev), C.byref(stats)))
    return y, int(nfev.value), {"steps": stats[0], "rejected": stats[1], "status": stats[2]}


def rk45_host_groups(fun, t_span, y0s, slots=None, rtol=1e-3, atol=1e-6, max_attempts=0):
    """Independent ``solve_ivp(method='RK45')`` systems side by side on the lockstep driver of
    :meth:`Engine.ode_sample_groups` (csrc/rk45.h: solve_groups), host-only.  ``y0s``: one complex array per system;
    at most ``slots`` (default: all) systems are in flight.  ``fun(systems, ts, ys)`` evaluates, once per round, every
    system in flight that asks for an evaluation and returns one derivative per system.
    Returns ``(ys, nfev list, stats list of {"steps", "rejected", "status"}, rounds)``."""
    import numpy as np
    lib = _lib.load()
    y0s = [np.asarray(v).astype(np.complex128).reshape(-1) for v in y0s]
    S = len(y0s)
    n = np.array([v.size for v in y0s], dtype=np.int64)
    y = np.ascontiguousarray(np.concatenate(y0s) if S else np.zeros(0, np.complex128))

    def rhs(count, systems, ts, yp, dp, nn, _user):
        ids = [int(systems[i]) for i in range(count)]
        ys = [np.ctypeslib.as_array(yp[i], shape=(2 * nn[i],)).view(np.complex128).copy() if nn[i] else
              np.zeros(0, np.complex128) for i in range(count)]
        ds = fun(ids, [float(ts[i]) for i in range(count)], ys)
        for i in range(count):
            if nn[i]:
                np.ctypeslib.as_array(dp[i], shape=(2 * nn[i],)).view(np.complex128)[:] = np.asarray(ds[i], dtype=np.complex128)

    cb = _lib.ODE_RHS_GROUPS(rhs)
    nfev = (C.c_int * max(S, 1))()
    stats = (C.c_int * (4 * max(S, 1)))()
    rounds = C.c_longlong()
    _lib.check(lib.sgmse_b200_rk45_host_groups(cb, None, S, int(slots if slots else max(S, 1)), n.ctypes.data,
                                               float(t_span[0]), float(t_span[1]), y.ctypes.data, float(rtol), float(atol),
                                               int(max_attempts), nfev, stats, C.byref(rounds)))
    off = np.concatenate([[0], np.cumsum(n)])
    ys = [y[off[i]:off[i + 1]].copy() for i in range(S)]
    st = [{"steps": stats[4 * i], "rejected": stats[4 * i + 1], "status": stats[4 * i + 2]} for i in range(S)]
    return ys, [int(nfev[i]) for i in range(S)], st, int(rounds.value)


def _stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


class Engine:
    """One engine per (process, device)."""

    def __init__(self, cfg: EngineConfig, device: Optional[torch.device] = None):
        self.cfg = cfg
        self.lib = _lib.load()
        self.device = torch.device(device) if device is not None else None
        self._h = C.c_void_p()
        self._ccfg = cfg.to_c()
        _lib.check(self.lib.sgmse_b200_create(C.byref(self._ccfg), C.byref(self._h)))
        self.F = cfg.n_fft // 2 + 1

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self.lib.sgmse_b200_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- weights ---------------------------------------------------------------------------------
    def manifest(self) -> List[Tuple[str, int]]:
        n = self.lib.sgmse_b200_manifest_count(self._h)
        out = []
        buf = C.create_string_buffer(256)
        num = C.c_longlong()
        for i in range(n):
            _lib.check(self.lib.sgmse_b200_manifest_entry(self._h, i, buf, 256, C.byref(num)))
            out.append((buf.value.decode(), int(num.value)))
        return out

    def weights_numel(self) -> int:
        return int(self.lib.sgmse_b200_weights_numel(self._h))

    def flatten_state_dict(self, sd: Dict[str, torch.Tensor], device="cpu") -> torch.Tensor:
        """fp32 blob in manifest (= ``state_dict()``) order on ``device``; verifies names and sizes."""
        man = self.manifest()
        missing = [k for k, _ in man if k not in sd]
        if missing:
            raise KeyError(f"state dict lacks {len(missing)} keys the engine expects, e.g. {missing[:3]}")
        extra = [k for k in sd if k not in dict(man)]
        if extra:
            raise KeyError(f"state dict has {len(extra)} keys the engine does not know, e.g. {extra[:3]}")
        parts = []
        for k, n in man:
            t = sd[k]
            if t.numel() != n:
                raise ValueError(f"{k}: expected {n} elements, state dict has {tuple(t.shape)}")
            parts.append(t.detach().reshape(-1).to(dtype=torch.float32, device=device))
        return torch.cat(parts).contiguous()

    def _use_device(self):
        if self.device is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        torch.cuda.set_device(self.device)

    def load_blob(self, blob: torch.Tensor):
        self._use_device()
        blob = blob.contiguous()
        if blob.dtype != torch.float32:
            raise TypeError("weight blob must be float32")
        if blob.is_cuda:
            _lib.check(self.lib.sgmse_b200_load_weights_device(self._h, blob.data_ptr(), blob.numel(), _stream_ptr()))
        else:
            _lib.check(self.lib.sgmse_b200_load_weights(self._h, blob.data_ptr(), blob.numel()))

    def load_state_dict(self, sd: Dict[str, torch.Tensor], on_device: bool = False):
        """``on_device``: flatten where the parameters live; a CUDA blob is packed on the device
        (sgmse_b200_load_weights_device, csrc/pack.cu: no host round trip -- the path of every ``refresh()`` between
        training epochs), a host blob on the host (sgmse_b200_load_weights); both give bit-identical packed weights."""
        dev = next(iter(sd.values())).device if on_device else "cpu"
        self.load_blob(self.flatten_state_dict(sd, device=dev))

    # ---- network ---------------------------------------------------------------------------------
    @staticmethod
    def _c64(x: torch.Tensor) -> torch.Tensor:
        if not x.is_cuda:
            raise RuntimeError("sgmse_b200: expected a CUDA tensor (there is no CPU path)")
        return x.to(torch.complex64).contiguous()

    def dnn_forward(self, x: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        """Backbone contract: c64 [B,2,F,T], f32 [B] -> c64 [B,1,F,T]."""
        self._use_device()
        x = self._c64(x)
        B, two, F, T = x.shape
        assert two == 2
        t = t.to(device=x.device, dtype=torch.float32).contiguous()
        out = torch.empty((B, 1, F, T), dtype=torch.complex64, device=x.device)
        _lib.check(self.lib.sgmse_b200_dnn_forward(self._h, x.data_ptr(), t.data_ptr(), out.data_ptr(), B, F, T, _stream_ptr()))
        return out

    def score(self, x_t: torch.Tensor, y: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        """ScoreModel.forward (legacy branch): -dnn(cat[x_t, y], t)."""
        x_t, y = self._c64(x_t), self._c64(y)
        self._use_device()
        B, _, F, T = y.shape
        t = t.to(device=y.device, dtype=torch.float32).contiguous()
        out = torch.empty_like(y)
        _lib.check(self.lib.sgmse_b200_score(self._h, x_t.data_ptr(), y.data_ptr(), t.data_ptr(), out.data_ptr(), B, F, T, _stream_ptr()))
        return out

    def model_forward(self, x_t: torch.Tensor, y: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        """ScoreModel.forward for the configured backbone (model.py:261-341): the score, or for
        ``loss_type='data_prediction'`` the clean-speech estimate of the preconditioned 'ncsnpp_v2' network."""
        x_t, y = self._c64(x_t), self._c64(y)
        self._use_device()
        B, _, F, T = y.shape
        t = t.to(device=y.device, dtype=torch.float32).contiguous()
        out = torch.empty_like(y)
        _lib.check(self.lib.sgmse_b200_model_forward(self._h, x_t.data_ptr(), y.data_ptr(), t.data_ptr(), out.data_ptr(),
                                                     B, F, T, _stream_ptr()))
        return out

    def sb_sample(self, y: torch.Tensor, sampler_type: str = "ode", N: int = 50, eps: float = 1e-4, n_steps: int = 50,
                  noise: Optional[torch.Tensor] = None, **kw):
        """sampling.get_sb_sampler(sde, model, y, eps, n_steps, sampler_type)() (sampling/__init__.py:145-249):
        y c64 [B,1,F,T] -> (sample, n_steps).  ``noise``: optional c64 [N,B,1,F,T] for ``sampler_type='sde'``."""
        if sampler_type not in ("ode", "sde"):
            raise ValueError("Invalid type. Choose 'ode' or 'sde'.")
        return self.pc_sample(y, noise=noise, N=N, kind="sb_" + sampler_type, sb_eps=eps, sb_n_steps=n_steps, **kw)

    # ---- sampler ---------------------------------------------------------------------------------
    def sampler_struct(self, N=30, predictor="reverse_diffusion", corrector="ald", corrector_steps=1, snr=0.5,
                       denoise=True, probability_flow=False, seed=0, utt_offset=0, pad_mode="zero_pad",
                       kind="pc", sb_eps=1e-4, sb_n_steps=50) -> _lib.Sampler:
        s = _lib.Sampler()
        s.N = int(N)
        s.predictor = _lookup(PREDICTORS, predictor, "Predictor")
        s.corrector = _lookup(CORRECTORS, corrector, "Corrector")
        s.corrector_steps = int(corrector_steps)
        s.snr = float(snr)
        s.denoise = int(bool(denoise))
        s.probability_flow = int(bool(probability_flow))
        s.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        s.utt_offset = int(utt_offset)
        s.pad_mode = _lookup(PAD_MODES, pad_mode, "Pad mode")
        s.kind = _lookup(SAMPLER_KINDS, kind, "Sampler kind")
        s.sb_eps = float(sb_eps)
        s.sb_n_steps = int(sb_n_steps)
        return s

    def noise_draws(self, **kw) -> int:
        s = self.sampler_struct(**kw)
        return int(self.lib.sgmse_b200_noise_draws(C.byref(s)))

    def sampler_schedule(self, **kw):
        """Host-computed schedule of the PC sampler (no GPU needed): ``(ts f32 [N], prior_std, coef f32 [updates, 3])``
        with rows ``(cy, cs, cz)`` of ``x_mean = x + cy (y - x) + cs score; x = x_mean + cz z`` in execution order."""
        s = self.sampler_struct(**kw)
        n = C.c_int(0)
        _lib.check(self.lib.sgmse_b200_sampler_schedule(self._h, C.byref(s), None, None, None, 0, C.byref(n)))
        ts = torch.empty(s.N, dtype=torch.float32)
        coef = torch.empty(n.value, 3, dtype=torch.float32)
        std = C.c_float(0.0)
        _lib.check(self.lib.sgmse_b200_sampler_schedule(self._h, C.byref(s), C.c_void_p(ts.data_ptr()), C.byref(std),
                                                        C.c_void_p(coef.data_ptr()), n.value, C.byref(n)))
        return ts, float(std.value), coef

    def pc_sample(self, y: torch.Tensor, noise: Optional[torch.Tensor] = None, **kw):
        """y c64 [B,1,F,T] -> (sample c64 [B,1,F,T], nfe).  ``noise``: optional c64 [draws,B,1,F,T]."""
        self._use_device()
        y = self._c64(y)
        B, _, F, T = y.shape
        s = self.sampler_struct(**kw)
        nptr = None
        if noise is not None:
            noise = self._c64(noise)
            need = int(self.lib.sgmse_b200_noise_draws(C.byref(s)))
            if tuple(noise.shape) != (need, B, 1, F, T):
                raise ValueError(f"noise must have shape {(need, B, 1, F, T)}, got {tuple(noise.shape)}")
            nptr = noise.data_ptr()
        out = torch.empty_like(y)
        nfe = C.c_int()
        _lib.check(self.lib.sgmse_b200_pc_sample(self._h, y.data_ptr(), B, F, T, C.byref(s), nptr, out.data_ptr(),
                                                 C.byref(nfe), _stream_ptr()))
        return out, int(nfe.value)

    def ode_sample(self, y: torch.Tensor, prior_noise: Optional[torch.Tensor] = None, rtol: float = 1e-5, atol: float = 1e-5,
                   eps: Optional[float] = None, denoise: bool = True, method: str = "RK45", seed: int = 0, utt_offset: int = 0,
                   max_attempts: int = 0, return_stats: bool = False):
        """sampling.get_ode_sampler(sde, score_fn, y, denoise, rtol, atol, method, eps)() (sampling/__init__.py:72-143):
        y c64 [B,1,F,T] -> (sample, nfe), the probability-flow ODE integrated from T=1 to ``eps`` (default: ``t_eps``, as
        ``ScoreModel.get_ode_sampler`` passes it, model.py:375) with scipy's RK45 restated on the device.  The whole
        batch is one ODE system (one shared adaptive step sequence), as in the reference.

        ``denoise`` defaults to True like the reference -- where that default raises ``TypeError`` (the denoising step
        calls ``ReverseDiffusionPredictor.update_fn(x, y, t)`` without ``stepsize``, predictors.py:60); same here.
        ``prior_noise``: optional c64 [B,1,F,T], the draw of ``prior_sampling`` (sdes.py:224-229)."""
        if method != "RK45":
            raise NotImplementedError("only scipy's default method 'RK45' is implemented on the device")
        if denoise:
            raise TypeError("ReverseDiffusionPredictor.update_fn() missing 1 required positional argument: 'stepsize' "
                            "(the reference's get_ode_sampler(denoise=True) fails the same way; pass denoise=False)")
        y = self._c64(y)
        self._use_device()
        B, _, F, T = y.shape
        o = _lib.Ode()
        o.rtol, o.atol = float(rtol), float(atol)
        o.eps = float(self.cfg.t_eps if eps is None else eps)
        o.max_attempts = int(max_attempts)
        o.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        o.utt_offset = int(utt_offset)
        nptr = None
        if prior_noise is not None:
            prior_noise = self._c64(prior_noise)
            if tuple(prior_noise.shape) != (B, 1, F, T):
                raise ValueError(f"prior_noise must have shape {(B, 1, F, T)}, got {tuple(prior_noise.shape)}")
            nptr = prior_noise.data_ptr()
        out = torch.empty_like(y)
        nfe = C.c_int()
        stats = (C.c_int * 4)()
        _lib.check(self.lib.sgmse_b200_ode_sample(self._h, y.data_ptr(), B, F, T, C.byref(o), nptr, out.data_ptr(),
                                                  C.byref(nfe), C.byref(stats), _stream_ptr()))
        if return_stats:
            return out, int(nfe.value), {"steps": stats[0], "rejected": stats[1], "status": stats[2]}
        return out, int(nfe.value)

    def ode_sample_groups(self, y: torch.Tensor, group: int = 1, prior_noise: Optional[torch.Tensor] = None, rtol: float = 1e-5,
                          atol: float = 1e-5, eps: Optional[float] = None, denoise: bool = True, method: str = "RK45",
                          seed: int = 0, utt_offset: int = 0, max_attempts: int = 0, return_stats: bool = False):
        """y c64 [B,1,F,T] -> (sample, nfe list[, stats list]): ``ceil(B / group)`` independent probability-flow ODE
        systems of ``group`` consecutive utterances each, every one with its own RK45 controller, solved side by side
        with each network evaluation batched across the systems in flight (at most ``max_batch`` utterances).
        System i equals :meth:`ode_sample` of ``y[i*group:(i+1)*group]`` with ``utt_offset + i*group``, bit for bit.
        ``group=1`` is per-file ``enhance()``; ``group=k`` is ``get_ode_sampler(minibatch=k)``.  Arguments as in
        :meth:`ode_sample`; stats also carry ``"rounds"``, ``"syncs"``, ``"forwards"`` and ``"rows"`` (utterance
        evaluations) of the whole call."""
        if method != "RK45":
            raise NotImplementedError("only scipy's default method 'RK45' is implemented on the device")
        if denoise:
            raise TypeError("ReverseDiffusionPredictor.update_fn() missing 1 required positional argument: 'stepsize' "
                            "(the reference's get_ode_sampler(denoise=True) fails the same way; pass denoise=False)")
        y = self._c64(y)
        self._use_device()
        B, _, F, T = y.shape
        group = int(group)
        o = _lib.Ode()
        o.rtol, o.atol = float(rtol), float(atol)
        o.eps = float(self.cfg.t_eps if eps is None else eps)
        o.max_attempts = int(max_attempts)
        o.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        o.utt_offset = int(utt_offset)
        nptr = None
        if prior_noise is not None:
            prior_noise = self._c64(prior_noise)
            if tuple(prior_noise.shape) != (B, 1, F, T):
                raise ValueError(f"prior_noise must have shape {(B, 1, F, T)}, got {tuple(prior_noise.shape)}")
            nptr = prior_noise.data_ptr()
        S = -(-B // group) if group > 0 else 1
        out = torch.empty_like(y)
        nfe = (C.c_int * S)()
        stats = (C.c_int * (4 * S))()
        info = (C.c_longlong * 4)()
        _lib.check(self.lib.sgmse_b200_ode_sample_groups(self._h, y.data_ptr(), B, F, T, group, C.byref(o), nptr,
                                                         out.data_ptr(), nfe, stats, info, _stream_ptr()))
        nfes = [int(v) for v in nfe]
        if return_stats:
            st = [{"steps": stats[4 * i], "rejected": stats[4 * i + 1], "status": stats[4 * i + 2],
                   "rounds": int(info[0]), "syncs": int(info[1]), "forwards": int(info[2]), "rows": int(info[3])}
                  for i in range(S)]
            return out, nfes, st
        return out, nfes

    # ---- STFT chain ------------------------------------------------------------------------------
    def padded_frames(self, L: int) -> int:
        return int(self.lib.sgmse_b200_padded_frames(self._h, int(L)))

    def analysis(self, wav: torch.Tensor, pad_mode="zero_pad"):
        """wav f32 [B,L] (cuda) -> (Y c64 [B,1,F,Tpad], norm f32 [B])."""
        self._use_device()
        wav = wav.to(torch.float32).contiguous()
        B, L = wav.shape
        Tp = self.padded_frames(L)
        Y = torch.empty((B, 1, self.F, Tp), dtype=torch.complex64, device=wav.device)
        norm = torch.empty((B,), dtype=torch.float32, device=wav.device)
        _lib.check(self.lib.sgmse_b200_analysis(self._h, wav.data_ptr(), B, L, _lookup(PAD_MODES, pad_mode, "Pad mode"),
                                                Y.data_ptr(), norm.data_ptr(), _stream_ptr()))
        return Y, norm

    def synthesis(self, X: torch.Tensor, norm: torch.Tensor, length: int) -> torch.Tensor:
        self._use_device()
        X = self._c64(X)
        B, _, F, Tp = X.shape
        wav = torch.empty((B, length), dtype=torch.float32, device=X.device)
        _lib.check(self.lib.sgmse_b200_synthesis(self._h, X.data_ptr(), norm.contiguous().data_ptr(), B, Tp, int(length),
                                                 wav.data_ptr(), _stream_ptr()))
        return wav

    def enhance(self, wav: torch.Tensor, noise: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None, **kw):
        """One call: wav f32 [B,L] (host or device) -> enhanced wav [B,L] on the same side.
        Host tensors (ideally pinned) make the H2D/D2H copies part of the call (sgmse_b200_enhance)."""
        self._use_device()
        wav = wav.to(torch.float32).contiguous()
        B, L = wav.shape
        host = not wav.is_cuda
        if out is None:
            out = torch.empty_like(wav, pin_memory=True) if host else torch.empty_like(wav)
        s = self.sampler_struct(**kw)
        nptr = None
        if noise is not None:
            noise = self._c64(noise)
            need = (int(self.lib.sgmse_b200_noise_draws(C.byref(s))), B, 1, self.F, self.padded_frames(L))
            if tuple(noise.shape) != need:
                raise ValueError(f"noise must have shape {need}, got {tuple(noise.shape)}")
            nptr = noise.data_ptr()
        _lib.check(self.lib.sgmse_b200_enhance(self._h, wav.data_ptr(), B, L, C.byref(s), nptr, out.data_ptr(), int(host),
                                               _stream_ptr()))
        return out

    def enhance_ode(self, wav: torch.Tensor, prior_noise: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                    rtol: float = 1e-5, atol: float = 1e-5, eps: Optional[float] = None, denoise: bool = True,
                    method: str = "RK45", seed: int = 0, utt_offset: int = 0, pad_mode: str = "zero_pad", max_attempts: int = 0):
        """``ScoreModel.enhance`` with ``sde.sampler_type == 'ode'`` (model.py:446-447) in one call
        (sgmse_b200_enhance_ode): wav f32 [B,L] (host or device) -> (enhanced wav [B,L] on the same side, nfe list).
        Every utterance is its own ODE system.  ``denoise`` as in :meth:`ode_sample` (the reference default raises)."""
        if method != "RK45":
            raise NotImplementedError("only scipy's default method 'RK45' is implemented on the device")
        if denoise:
            raise TypeError("ReverseDiffusionPredictor.update_fn() missing 1 required positional argument: 'stepsize' "
                            "(the reference's get_ode_sampler(denoise=True) fails the same way; pass denoise=False)")
        self._use_device()
        wav = wav.to(torch.float32).contiguous()
        B, L = wav.shape
        host = not wav.is_cuda
        if out is None:
            out = torch.empty_like(wav, pin_memory=True) if host else torch.empty_like(wav)
        o = _lib.Ode()
        o.rtol, o.atol = float(rtol), float(atol)
        o.eps = float(self.cfg.t_eps if eps is None else eps)
        o.max_attempts = int(max_attempts)
        o.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        o.utt_offset = int(utt_offset)
        nptr = None
        if prior_noise is not None:
            prior_noise = self._c64(prior_noise)
            nptr = prior_noise.data_ptr()
        nfe = (C.c_int * B)()
        _lib.check(self.lib.sgmse_b200_enhance_ode(self._h, wav.data_ptr(), B, L, C.byref(o), _lookup(PAD_MODES, pad_mode, "Pad mode"),
                                                   nptr, out.data_ptr(), int(host), nfe, _stream_ptr()))
        return out, [int(v) for v in nfe]

    # ---- introspection ---------------------------------------------------------------------------
    def set_option(self, key: str, value: int):
        _lib.check(self.lib.sgmse_b200_set_option(self._h, key.encode(), int(value)))

    def workspace_bytes(self, B: int, F: int, T: int) -> int:
        """Bytes of all activation buffers of one forward of (B, F, T) without reuse.  The engine allocates
        ``workspace_plan(B, F, T)["bytes"]``."""
        n = int(self.lib.sgmse_b200_workspace_bytes(self._h, B, F, T))
        if n < 0:
            _lib.check(1)
        return n

    def workspace_plan(self, B: int, F: int, T: int) -> dict:
        """The activation workspace of one forward of (B, F, T) with the current options, host-only:
        ``{"bytes": allocated bytes, "steps": launches of the forward, "buffers": int64 [n, 5]}`` with one row
        (offset, bytes, first step, last step, tapped) per buffer in allocation order.  ``last == steps``: the buffer
        is read after the forward returns (the output pyramid, and with ``record_taps`` every tapped tensor)."""
        import numpy as np
        n, steps = C.c_longlong(), C.c_int()
        if self.lib.sgmse_b200_workspace_plan(self._h, B, F, T, None, 0, C.byref(n), C.byref(steps)) < 0:
            _lib.check(1)
        rows = np.zeros((n.value, 5), dtype=np.int64)
        nbytes = int(self.lib.sgmse_b200_workspace_plan(self._h, B, F, T, rows.ctypes.data, n.value, C.byref(n),
                                                        C.byref(steps)))
        if nbytes < 0:
            _lib.check(1)
        return {"bytes": nbytes, "steps": int(steps.value), "buffers": rows}

    def counter(self, key: str) -> int:
        return int(self.lib.sgmse_b200_get_counter(self._h, key.encode()))

    def tap(self, name: str) -> torch.Tensor:
        shape = (C.c_int * 4)()
        _lib.check(self.lib.sgmse_b200_get_tap(self._h, name.encode(), None, 0, C.byref(shape)))
        n = shape[0] * shape[1] * shape[2] * shape[3]
        out = torch.empty(tuple(shape), dtype=torch.float32)
        _lib.check(self.lib.sgmse_b200_get_tap(self._h, name.encode(), out.data_ptr(), n, C.byref(shape)))
        return out
