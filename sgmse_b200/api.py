"""Drop-in installation behind the reference's public API.

``install(model)`` snapshots the configuration and (EMA-swapped) weights of a live
``sgmse.model.ScoreModel`` and rebinds

* ``model.get_pc_sampler(predictor_name, corrector_name, y, N=None, minibatch=None, **kw)``
  (/root/reference/sgmse/model.py:348-368) -> callable returning ``(sample c64 [B,1,F,T], nfe)``
  (with ``minibatch`` the second element is a list, model.py:359-367),
* ``model.enhance(y, sampler_type, predictor, corrector, N, corrector_steps, snr, timeit, **kw)``
  (model.py:426-465) -> ``np.ndarray [T]`` or ``(x_hat, nfe, rtf)``,
* ``model.forward(x_t, y, t)`` (legacy branch, model.py:307-310),
* ``model.get_ode_sampler(y, N=None, minibatch=None, **kw)`` (model.py:370-390; OUVE SDE, score backbones) -> callable
  returning ``(sample, nfe)`` -- the probability-flow ODE with scipy's RK45 restated on the device,

to the GPU engine.  ``sgmse/model.py`` itself is untouched; ``uninstall(model)`` restores the
original bound methods.  The predictor / corrector names are the reference registry names
(sampling/predictors.py:41,55,68; correctors.py:37,59,84) and unknown names raise the same
``ValueError`` as ``Registry.get_by_name`` (util/registry.py:25-30).
"""
from __future__ import annotations

import time
import types
from math import ceil
from typing import Optional

import torch

from .engine import Engine, EngineConfig, PREDICTORS, CORRECTORS, _lookup


def config_from_score_model(model, mode="fp16_tc", max_batch=8, use_graphs=True) -> EngineConfig:
    """Read every hyper-parameter of the hot path from a live ScoreModel."""
    dnn = model.dnn
    backbone = getattr(model, "backbone", None) or type(dnn).__name__.lower()
    if backbone not in ("ncsnpp", "ncsnpp_48k", "ncsnpp_v2"):
        raise NotImplementedError(f"sgmse_b200 accelerates the 'ncsnpp', 'ncsnpp_48k' and 'ncsnpp_v2' backbones, not '{backbone}'")
    for attr, want in (("resblock_type", "biggan"), ("embedding_type", "fourier"), ("skip_rescale", True),
                       ("conditional", True), ("centered", True)):
        if getattr(dnn, attr, want) != want:
            raise NotImplementedError(f"NCSN++ option {attr}={getattr(dnn, attr)!r} is outside the accelerated path")
    nf = dnn.nf
    # ch_mult is not kept as an attribute (ncsnpp.py:79): recover it from the block list
    mods = list(dnn.all_modules)
    i, ch_mult = 4, []
    L = dnn.num_resolutions
    for lvl in range(L):
        seen = 0
        while seen < dnn.num_res_blocks:
            m = mods[i]
            i += 1
            if type(m).__name__ == "ResnetBlockBigGANpp":
                if seen == 0:
                    ch_mult.append(m.out_ch // nf)
                seen += 1
        while type(mods[i]).__name__ == "AttnBlockpp":
            i += 1
        if lvl != L - 1:
            i += 1                                         # down-sampling resblock
            if dnn.progressive_input == "input_skip":
                i += 1                                     # Combine
    dm = model.data_module
    if getattr(dm, "transform_type", "exponent") != "exponent":
        raise NotImplementedError("only transform_type='exponent' is accelerated")
    hann = torch.hann_window(dm.n_fft, periodic=True)
    window = "hann" if torch.allclose(dm.window.cpu().float(), hann, atol=1e-6) else "sqrthann"
    sde = model.sde
    sde_name = type(sde).__name__
    if sde_name == "OUVESDE":
        sde_kw = dict(sde="ouve", theta=float(sde.theta), sigma_min=float(sde.sigma_min), sigma_max=float(sde.sigma_max))
    elif sde_name == "SBVESDE":
        if backbone != "ncsnpp_v2":
            raise NotImplementedError("the Schroedinger-bridge SDE is driven by the preconditioned 'ncsnpp_v2' forward")
        # get_sb_sampler works on sde.copy() = SBVESDE(k, c, N) (sdes.py:265-266): the stabiliser eps falls back to 1e-8
        # ... while ScoreModel.forward evaluates self.sde._std(t) on the model's OWN sde with its configured --eps
        # (sdes.py:242,297-301).  The engine carries one stabiliser: refuse a checkpoint trained with another eps
        # rather than silently precondition with different c_in / c_out / c_skip.
        if abs(float(getattr(sde, "eps", 1e-8)) - 1e-8) > 1e-14:
            raise NotImplementedError(f"SBVESDE eps={sde.eps!r}: only the default stabiliser 1e-8 is accelerated "
                                      "(ScoreModel.forward preconditions with the model's own sde.eps, the samplers with sde.copy()'s 1e-8)")
        sde_kw = dict(sde="sbve", sb_k=float(sde.k), sb_c=float(sde.c), sb_eps=1e-8)
    else:
        raise NotImplementedError("only the OUVE and SBVE SDEs are accelerated")
    pre_kw = {}
    if backbone == "ncsnpp_v2":                          # ScoreModel attributes of model.py:52-60
        pre_kw = dict(loss_type=model.loss_type, network_scaling=model.network_scaling, c_in=model.c_in, c_out=model.c_out,
                      c_skip=model.c_skip, sigma_data=float(model.sigma_data))
    return EngineConfig(
        backbone=backbone, nf=nf, ch_mult=tuple(ch_mult), num_res_blocks=dnn.num_res_blocks,
        attn_resolutions=tuple(dnn.attn_resolutions), image_size=dnn.all_resolutions[0],
        progressive=dnn.progressive, progressive_input=dnn.progressive_input,
        scale_by_sigma=bool(getattr(dnn, "scale_by_sigma", False)) and backbone != "ncsnpp_v2",
        t_eps=float(model.t_eps),
        n_fft=dm.n_fft, hop_length=dm.hop_length, window=window, spec_factor=float(dm.spec_factor),
        spec_abs_exponent=float(dm.spec_abs_exponent), sr=int(getattr(model, "sr", 16000)),
        mode=mode, max_batch=max_batch, use_graphs=use_graphs, **sde_kw, **pre_kw)


def engine_from_score_model(model, load_weights=True, **kw) -> Engine:
    """``model`` should be in ``eval()`` mode so that the EMA weights are the ones in ``model.dnn``
    (model.py:111-122)."""
    eng = Engine(config_from_score_model(model, **kw))
    if load_weights:
        eng.load_state_dict(model.dnn.state_dict())
    return eng


def make_pc_sampler(engine: Engine, default_N: int):
    def get_pc_sampler(self, predictor_name, corrector_name, y, N=None, minibatch=None, **kwargs):
        N = default_N if N is None else N
        _lookup(PREDICTORS, predictor_name, "Predictor")
        _lookup(CORRECTORS, corrector_name, "Corrector")
        kw = dict(N=N, predictor=predictor_name, corrector=corrector_name,
                  corrector_steps=kwargs.get("corrector_steps", 1), snr=kwargs.get("snr", 0.1),
                  denoise=kwargs.get("denoise", True), probability_flow=kwargs.get("probability_flow", False),
                  seed=kwargs.get("seed", int(torch.randint(0, 2 ** 62, (1,)).item())))
        if "eps" in kwargs and abs(kwargs["eps"] - engine.cfg.t_eps) > 1e-12:
            raise NotImplementedError("eps other than ScoreModel.t_eps is baked into the engine configuration")
        noise = kwargs.get("noise", None)

        if minibatch is None:
            def pc_sampler():
                with torch.no_grad():
                    return engine.pc_sample(y, noise=noise, **kw)
            return pc_sampler

        M = y.shape[0]

        def batched_sampling_fn():
            samples, ns = [], []
            for i in range(int(ceil(M / minibatch))):
                sl = slice(i * minibatch, (i + 1) * minibatch)
                nz = noise[:, sl] if noise is not None else None
                smp, n = engine.pc_sample(y[sl], noise=nz, **{**kw, "utt_offset": i * minibatch})
                samples.append(smp)
                ns.append(n)
            return torch.cat(samples, dim=0), ns
        return batched_sampling_fn
    return get_pc_sampler


def make_ode_sampler(engine: Engine):
    def get_ode_sampler(self, y, N=None, minibatch=None, **kwargs):
        """ScoreModel.get_ode_sampler (model.py:370-390) -> sampling.get_ode_sampler (sampling/__init__.py:72-143).
        ``N`` only lands in the copied SDE (unused by the ODE solver); ``eps`` defaults to ``t_eps`` (model.py:375).
        Each minibatch is its own ODE system (own adaptive step sequence), as in the reference."""
        kw = dict(rtol=kwargs.get("rtol", 1e-5), atol=kwargs.get("atol", 1e-5), eps=kwargs.get("eps", engine.cfg.t_eps),
                  denoise=kwargs.get("denoise", True), method=kwargs.get("method", "RK45"),
                  seed=kwargs.get("seed", int(torch.randint(0, 2 ** 62, (1,)).item())))
        noise = kwargs.get("noise", None)               # c64 [B,1,F,T]: the prior draw

        if minibatch is None:
            def ode_sampler():
                with torch.no_grad():
                    return engine.ode_sample(y, prior_noise=noise, **kw)
            return ode_sampler

        M = y.shape[0]

        def batched_sampling_fn():
            samples, ns = [], []
            for i in range(int(ceil(M / minibatch))):
                sl = slice(i * minibatch, (i + 1) * minibatch)
                smp, n = engine.ode_sample(y[sl], prior_noise=noise[sl] if noise is not None else None,
                                           utt_offset=i * minibatch, **kw)
                samples.append(smp)
                ns.append(n)
            # (the reference returns `sample`, the LAST minibatch only, model.py:389 -- a typo for `samples`;
            #  the concatenation is what its PC twin returns, model.py:367)
            return torch.cat(samples, dim=0), ns
        return batched_sampling_fn
    return get_ode_sampler


def make_enhance(engine: Engine):
    def enhance(self, y, sampler_type="pc", predictor="reverse_diffusion", corrector="ald", N=30,
                corrector_steps=1, snr=0.5, timeit=False, **kwargs):
        """One-call speech enhancement of noisy speech `y` [1, T] (or [B, T])."""
        start = time.time()
        yy = y if y.dim() == 2 else y[None]
        # the reference forwards **kwargs to get_pc_sampler / get_ode_sampler (model.py:443-447): what the engine honours is
        # passed on, anything else is refused instead of being dropped silently
        known = {"seed", "pad_mode", "denoise", "probability_flow", "eps", "intermediate", "noise", "rtol", "atol", "method"}
        unknown = sorted(set(kwargs) - known)
        if unknown:
            raise NotImplementedError(f"enhance(): keyword(s) {unknown} are not supported by the sgmse_b200 engine")
        if kwargs.get("intermediate", False):
            raise NotImplementedError("enhance(): intermediate=True is not supported by the sgmse_b200 engine")
        common = dict(seed=kwargs.get("seed", int(torch.randint(0, 2 ** 62, (1,)).item())), pad_mode=kwargs.get("pad_mode", "zero_pad"))
        sde_name = type(self.sde).__name__
        if sde_name == "SBVESDE":                     # model.py:450-452: get_sb_sampler(sde, Y, sampler_type=sde.sampler_type)
            st = self.sde.sampler_type
            if st not in ("ode", "sde"):
                raise ValueError("Invalid type. Choose 'ode' or 'sde'.")
            x_hat = engine.enhance(yy.detach().cpu().float(), N=self.sde.N, kind="sb_" + st, sb_eps=1e-4, sb_n_steps=50, **common)
            sb_nfe = 50
        elif getattr(self.sde, "sampler_type", "pc") == "ode":      # model.py:446-447: get_ode_sampler(Y, N=N, **kwargs)
            ode_kw = {k: kwargs[k] for k in ("rtol", "atol", "eps", "method") if k in kwargs}
            x_hat, nfes = engine.enhance_ode(yy.detach().cpu().float(), denoise=kwargs.get("denoise", True), **ode_kw, **common)
            sb_nfe = nfes[-1]                                            # one ODE system per clip, as enhance() is per file
        else:
            if getattr(self.sde, "sampler_type", "pc") != "pc":
                raise ValueError("Invalid sampler type for SGMSE sampling: {}".format(sampler_type))   # model.py:448-449
            if "eps" in kwargs and abs(kwargs["eps"] - engine.cfg.t_eps) > 1e-12:
                raise NotImplementedError("eps other than ScoreModel.t_eps is baked into the engine configuration")
            x_hat = engine.enhance(yy.detach().cpu().float(), N=N, predictor=predictor, corrector=corrector,
                                   corrector_steps=corrector_steps, snr=snr, denoise=kwargs.get("denoise", True),
                                   probability_flow=kwargs.get("probability_flow", False), noise=kwargs.get("noise", None), **common)
            sb_nfe = None
        x_hat = x_hat.squeeze().numpy()
        end = time.time()
        nfe = sb_nfe if sb_nfe is not None else N * ((corrector_steps if corrector != "none" else 0) + 1)
        if timeit:
            rtf = (end - start) / (x_hat.shape[-1] / self.sr)
            return x_hat, nfe, rtf
        return x_hat
    return enhance


def refresh(model):
    """Re-snapshot the weights of an installed model (e.g. after a training epoch; call it with the model in ``eval()``
    so that the EMA weights are the ones in ``model.dnn``, model.py:111-122)."""
    eng = model.__dict__.get("_sgmse_b200_engine")
    if eng is None:
        raise RuntimeError("sgmse_b200 is not installed on this model")
    sd = model.dnn.state_dict()
    eng.load_state_dict(sd, on_device=next(iter(sd.values())).is_cuda)
    return eng


def install(model, engine: Optional[Engine] = None, rebind_forward=True, refresh_on_eval: bool = False, **kw) -> Engine:
    """Route ``model.get_pc_sampler`` / ``model.get_sb_sampler`` / ``model.enhance`` (and ``model.forward``) through the engine.

    In-training evaluation (SURVEY.md §8f-3: ``validation_step`` calls ``self.enhance`` per file, model.py:205-257;
    ``evaluate_model`` calls ``model.get_pc_sampler``, util/inference.py:16-63): install with
    ``rebind_forward=False`` -- training steps keep the differentiable torch forward -- and ``refresh_on_eval=True`` --
    every ``model.eval()`` (which swaps in the EMA weights) re-snapshots ``model.dnn`` into the engine.
    ``rebind_forward="no_grad"`` additionally sends every forward that runs with gradients disabled to the engine: the
    validation loss (``validation_step`` -> ``_step`` -> ``self(x_t, y, t)``, model.py:189-198,257-258) while
    ``training_step`` stays on autograd."""
    if getattr(model, "_sgmse_b200_saved", None) is not None:
        uninstall(model)                              # re-installing: start again from the model's own methods
    if engine is None:
        engine = engine_from_score_model(model, **kw)
    model._sgmse_b200_saved = {k: model.__dict__.get(k) for k in ("get_pc_sampler", "get_ode_sampler", "enhance", "forward", "train")}
    model._sgmse_b200_engine = engine
    model.get_pc_sampler = types.MethodType(make_pc_sampler(engine, default_N=model.sde.N), model)
    if type(model.sde).__name__ == "OUVESDE" and not (engine.cfg.backbone == "ncsnpp_v2" and
                                                      getattr(engine.cfg, "loss_type", "score_matching") == "data_prediction"):
        model.get_ode_sampler = types.MethodType(make_ode_sampler(engine), model)    # needs a score model
    model.enhance = types.MethodType(make_enhance(engine), model)

    if rebind_forward == "no_grad":
        # training keeps the differentiable torch forward; whatever runs under torch.no_grad() -- the `_step` of
        # validation_step (model.py:189-198,257-258: x_t = mean + std z -> self(x_t, y, t) -> loss) -- goes to the engine
        torch_forward = model.forward                 # bound method of the class (or whatever was installed before)

        def forward(self, x_t, y, t):
            if torch.is_grad_enabled():
                return torch_forward(x_t, y, t)
            return engine.model_forward(x_t, y, t)
        model.forward = types.MethodType(forward, model)
    elif rebind_forward:
        def forward(self, x_t, y, t):
            return engine.model_forward(x_t, y, t)    # legacy: score; 'ncsnpp_v2': model.py:283-304
        model.forward = types.MethodType(forward, model)

    if refresh_on_eval:
        # ScoreModel.train(mode, no_ema=False) is the ONE place the reference swaps EMA weights in and out
        # (model.py:111-122); ScoreModel.eval() delegates to it (:124-125), and so does everything that never calls
        # ScoreModel.eval: Lightning's on_validation_model_eval() calls trainer.model.eval() on the DDP wrapper
        # (train.py:104, strategy="ddp"), i.e. nn.Module.eval(wrapper) -> child.train(False).  Hooking the instance's
        # `train` covers both routes (`self.train` inside ScoreModel.eval resolves to the instance attribute).
        orig_train = model.train

        def train_and_refresh(self, mode=True, *a, **k):
            res = orig_train(mode, *a, **k)           # EMA store + copy_to when mode is False (model.py:113-117)
            if not mode:
                refresh(self)
            return res
        model.train = types.MethodType(train_and_refresh, model)

    def get_sb_sampler(self, sde, y, sampler_type="ode", N=None, **kwargs):
        # model.py:392-397 + sampling/__init__.py:145 (eps=1e-4, n_steps=50 defaults)
        N_ = sde.N if N is None else N
        kw = dict(sampler_type=sampler_type, N=N_, eps=kwargs.get("eps", 1e-4), n_steps=kwargs.get("n_steps", 50),
                  seed=kwargs.get("seed", int(torch.randint(0, 2 ** 62, (1,)).item())))
        noise = kwargs.get("noise", None)

        def sb_sampler():
            with torch.no_grad():
                return engine.sb_sample(y, noise=noise, **kw)
        return sb_sampler
    model._sgmse_b200_saved["get_sb_sampler"] = model.__dict__.get("get_sb_sampler")
    model.get_sb_sampler = types.MethodType(get_sb_sampler, model)
    return engine


def uninstall(model):
    saved = getattr(model, "_sgmse_b200_saved", None)
    if saved is None:
        return
    for k, v in saved.items():
        if v is None:
            model.__dict__.pop(k, None)
        else:
            model.__dict__[k] = v
    del model._sgmse_b200_saved
    del model._sgmse_b200_engine
