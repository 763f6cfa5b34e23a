"""Functional fp32/fp64 restatement of the NCSN++ forward pass (oracle).

Follows sgmse/backbones/ncsnpp.py:256-419 (and ncsnpp_48k.py:259-424
for the ``ncsnpp_48k`` ordering of ``/t`` and ``output_layer``), with the blocks of
ncsnpp_utils/layerspp.py and the FIR resamplers of up_or_down_sampling.py:195-257 /
op/upfirdn2d.py:162-203.  Operates on a plain ``{key: tensor}`` state dict in the
reference's key layout.  TEST INFRASTRUCTURE – see oracle/__init__.py.
"""
from __future__ import annotations

import math
from typing import Dict

import torch
import torch.nn.functional as F

from .arch import NetConfig, build_layers, gn_groups

SQRT2 = math.sqrt(2.0)
_FIR_1D = (1.0, 3.0, 3.0, 1.0)


def fir_kernel_2d(dtype=torch.float32):
    """outer([1,3,3,1]) / 64   (up_or_down_sampling.py:181-188)."""
    k = torch.tensor(_FIR_1D, dtype=dtype)
    k = torch.outer(k, k)
    return k / k.sum()


def fir_down2(x: torch.Tensor) -> torch.Tensor:
    """downsample_2d(x, (1,3,3,1), factor=2): pad 1/1, 4x4 FIR, keep every 2nd
    (up_or_down_sampling.py:227-257 -> upfirdn2d(down=2, pad=(1,1)))."""
    B, C, H, W = x.shape
    k = fir_kernel_2d(x.dtype).to(x.device).view(1, 1, 4, 4)
    y = F.conv2d(F.pad(x.reshape(B * C, 1, H, W), (1, 1, 1, 1)), k, stride=2)
    return y.view(B, C, H // 2, W // 2)


def fir_up2(x: torch.Tensor) -> torch.Tensor:
    """upsample_2d(x, (1,3,3,1), factor=2): zero-insert x2, pad 2/1, 4x4 FIR with
    gain 4 (up_or_down_sampling.py:195-224 -> upfirdn2d(up=2, pad=(2,1)))."""
    B, C, H, W = x.shape
    z = x.new_zeros(B * C, 1, 2 * H, 2 * W)
    z[:, :, ::2, ::2] = x.reshape(B * C, 1, H, W)
    k = (fir_kernel_2d(x.dtype) * 4.0).to(x.device).view(1, 1, 4, 4)   # symmetric: flip is a no-op
    y = F.conv2d(F.pad(z, (2, 1, 2, 1)), k)
    return y.view(B, C, 2 * H, 2 * W)


def _gn(x, w, b):
    return F.group_norm(x, gn_groups(x.shape[1]), w, b, eps=1e-6)


def _nin(x, W, b):
    # layers.py:546-555: y[b,o,h,w] = sum_c x[b,c,h,w] W[c,o] + b[o]
    return torch.einsum("bchw,co->bohw", x, W) + b.view(1, -1, 1, 1)


class _P:
    """Prefix view on the state dict."""

    def __init__(self, sd: Dict[str, torch.Tensor], prefix: str, dtype):
        self.sd, self.prefix, self.dtype = sd, prefix, dtype

    def __getitem__(self, k):
        return self.sd[self.prefix + k].to(self.dtype)

    def has(self, k):
        return (self.prefix + k) in self.sd


def resblock(p: _P, x, temb, up=False, down=False):
    """ResnetBlockBigGANpp.forward  (layerspp.py:242-274)."""
    h = F.silu(_gn(x, p["GroupNorm_0.weight"], p["GroupNorm_0.bias"]))
    if up:
        h, x = fir_up2(h), fir_up2(x)
    elif down:
        h, x = fir_down2(h), fir_down2(x)
    h = F.conv2d(h, p["Conv_0.weight"], p["Conv_0.bias"], padding=1)
    h = h + F.linear(F.silu(temb), p["Dense_0.weight"], p["Dense_0.bias"])[:, :, None, None]
    h = F.silu(_gn(h, p["GroupNorm_1.weight"], p["GroupNorm_1.bias"]))
    h = F.conv2d(h, p["Conv_1.weight"], p["Conv_1.bias"], padding=1)
    if p.has("Conv_2.weight"):
        x = F.conv2d(x, p["Conv_2.weight"], p["Conv_2.bias"])
    return (x + h) / SQRT2


def attnblock(p: _P, x):
    """AttnBlockpp.forward  (layerspp.py:75-91)."""
    B, C, H, W = x.shape
    h = _gn(x, p["GroupNorm_0.weight"], p["GroupNorm_0.bias"])
    q = _nin(h, p["NIN_0.W"], p["NIN_0.b"]).reshape(B, C, H * W)
    k = _nin(h, p["NIN_1.W"], p["NIN_1.b"]).reshape(B, C, H * W)
    v = _nin(h, p["NIN_2.W"], p["NIN_2.b"]).reshape(B, C, H * W)
    w = torch.einsum("bcq,bck->bqk", q, k) * (int(C) ** (-0.5))
    w = torch.softmax(w, dim=-1)
    h = torch.einsum("bqk,bck->bcq", w, v).reshape(B, C, H, W)
    h = _nin(h, p["NIN_3.W"], p["NIN_3.b"])
    return (x + h) / SQRT2


def time_embedding(sd, cfg: NetConfig, t: torch.Tensor, dtype=torch.float32):
    """GaussianFourierProjection(log t) -> Linear -> SiLU -> Linear
    (layerspp.py:39-41, ncsnpp.py:267-284)."""
    W = sd["all_modules.0.W"].to(dtype)
    proj = torch.log(t.to(dtype))[:, None] * W[None, :] * 2 * math.pi
    emb = torch.cat([torch.sin(proj), torch.cos(proj)], dim=-1)
    emb = F.linear(emb, sd["all_modules.1.weight"].to(dtype), sd["all_modules.1.bias"].to(dtype))
    emb = F.linear(F.silu(emb), sd["all_modules.2.weight"].to(dtype), sd["all_modules.2.bias"].to(dtype))
    return emb


def forward(sd: Dict[str, torch.Tensor], cfg: NetConfig, x: torch.Tensor, t: torch.Tensor,
            dtype=torch.float32, taps: dict | None = None) -> torch.Tensor:
    """Backbone contract: ``x`` c64 [B,2,F,T], ``t`` f32 [B]  ->  c64 [B,1,F,T].

    ``taps`` (optional dict) receives named intermediate activations for op-level parity.
    """
    layers = build_layers(cfg)
    it = iter(layers[:-1])
    cdt = torch.complex64 if dtype == torch.float32 else torch.complex128
    x = x.to(cdt)
    xin = torch.cat([x[:, [0]].real, x[:, [0]].imag, x[:, [1]].real, x[:, [1]].imag], dim=1)

    def P(layer):
        return _P(sd, f"all_modules.{layer.idx}.", dtype)

    def tap(name, v):
        if taps is not None:
            taps[name] = v.detach().clone()

    next(it), next(it), next(it)                       # gfp + 2 linear
    temb = time_embedding(sd, cfg, t, dtype)
    tap("temb", temb)
    L = len(cfg.ch_mult)

    l = next(it)                                       # input conv3x3(4->nf)
    p = P(l)
    hs = [F.conv2d(xin, p["weight"], p["bias"], padding=1)]
    tap("in_conv", hs[0])
    pyr_in = xin if cfg.progressive_input == "input_skip" else None

    for lvl in range(L):
        for _ in range(cfg.num_res_blocks):
            l = next(it)
            h = resblock(P(l), hs[-1], temb)
            tap(f"m{l.idx}", h)
            if h.shape[-2] in cfg.attn_resolutions:    # ncsnpp.py:308 (checks the F axis)
                l = next(it)
                h = attnblock(P(l), h)
                tap(f"m{l.idx}", h)
            hs.append(h)
        if lvl != L - 1:
            l = next(it)
            h = resblock(P(l), hs[-1], temb, down=True)
            tap(f"m{l.idx}", h)
            if cfg.progressive_input == "input_skip":
                l = next(it)
                p = P(l)
                pyr_in = fir_down2(pyr_in)
                h = F.conv2d(pyr_in, p["Conv_0.weight"], p["Conv_0.bias"]) + h   # Combine 'sum'
                tap(f"m{l.idx}", h)
            hs.append(h)

    h = hs[-1]
    l = next(it); h = resblock(P(l), h, temb); tap(f"m{l.idx}", h)
    l = next(it); h = attnblock(P(l), h); tap(f"m{l.idx}", h)
    l = next(it); h = resblock(P(l), h, temb); tap(f"m{l.idx}", h)

    pyramid = None
    for lvl in reversed(range(L)):
        for _ in range(cfg.num_res_blocks + 1):
            l = next(it)
            h = resblock(P(l), torch.cat([h, hs.pop()], dim=1), temb)
            tap(f"m{l.idx}", h)
        if h.shape[-2] in cfg.attn_resolutions:
            l = next(it)
            h = attnblock(P(l), h)
            tap(f"m{l.idx}", h)
        if cfg.progressive == "output_skip":
            lg, lc = next(it), next(it)
            pg, pc = P(lg), P(lc)
            ph = F.conv2d(F.silu(_gn(h, pg["weight"], pg["bias"])), pc["weight"], pc["bias"], padding=1)
            pyramid = ph if pyramid is None else fir_up2(pyramid) + ph
            tap(f"pyr{lvl}", pyramid)
        if lvl != 0:
            l = next(it)
            h = resblock(P(l), h, temb, up=True)
            tap(f"m{l.idx}", h)
    assert not hs

    if cfg.progressive == "output_skip":
        h = pyramid
    else:
        lg, lc = next(it), next(it)
        pg, pc = P(lg), P(lc)
        h = F.conv2d(F.silu(_gn(h, pg["weight"], pg["bias"])), pc["weight"], pc["bias"], padding=1)
    assert next(it, None) is None

    ow, ob = sd["output_layer.weight"].to(dtype), sd["output_layer.bias"].to(dtype)
    tt = t.to(dtype).view(-1, 1, 1, 1)
    if cfg.backbone == "ncsnpp_48k":                   # ncsnpp_48k.py:416-420: conv, then /t
        h = F.conv2d(h, ow, ob)
        if cfg.scale_by_sigma:
            h = h / tt
    else:                                              # ncsnpp.py:411-416: /t, then conv
        if cfg.scale_by_sigma:
            h = h / tt
        h = F.conv2d(h, ow, ob)
    h = h.permute(0, 2, 3, 1).contiguous()
    return torch.view_as_complex(h)[:, None]


def score(sd, cfg: NetConfig, x_t, y, t, dtype=torch.float32):
    """ScoreModel.forward, legacy branch (model.py:307-310): -dnn(cat[x_t, y], t)."""
    return -forward(sd, cfg, torch.cat([x_t, y], dim=1), t, dtype=dtype)


# ---- ncsnpp_v2 + preconditioned forward (SURVEY.md §8f-1) -----------------------------------------------------
def forward_v2(sd, cfg: NetConfig, x, y, t, dtype=torch.float32):
    """NCSNpp_v2.forward(x, y, t) (ncsnpp_v2.py:241-395): the ncsnpp network on cat[x, y] without the ``/t``."""
    assert cfg.backbone == "ncsnpp_v2" and not cfg.scale_by_sigma
    return forward(sd, cfg, torch.cat([x, y], dim=1), t, dtype=dtype)


def precond_forward(sd, cfg: NetConfig, pre, std_fn, x_t, y, t, dtype=torch.float32):
    """ScoreModel.forward for backbone == 'ncsnpp_v2' (model.py:283-304).

    ``pre``: dict(loss_type, network_scaling, c_in, c_out, c_skip, sigma_data) -- the ScoreModel attributes of the same
    names (model.py:52-60); ``std_fn(t: Tensor[B]) -> Tensor[B]`` = ``sde._std``."""
    sig = std_fn(t).to(dtype)
    v = lambda a: a.view(-1, 1, 1, 1)
    sd2 = pre.get("sigma_data", 0.1) ** 2

    def c_in():                                           # model.py:312-319
        return 1.0 if pre["c_in"] == "1" else v(1.0 / torch.sqrt(sig ** 2 + sd2))

    def c_out():                                          # model.py:321-332
        k = pre["c_out"]
        if k == "1":
            return 1.0
        if k == "sigma":
            return v(sig)
        if k == "1/sigma":
            return v(1.0 / sig)
        return v(sig * pre["sigma_data"] / torch.sqrt(sd2 + sig ** 2))

    def c_skip():                                         # model.py:334-341
        return 0.0 if pre["c_skip"] == "0" else v(sd2 / (sig ** 2 + sd2))

    Fo = forward_v2(sd, cfg, c_in() * x_t, c_in() * y, t, dtype=dtype)
    if pre.get("network_scaling") == "1/sigma":
        Fo = Fo / v(sig)
    elif pre.get("network_scaling") == "1/t":
        Fo = Fo / v(t.to(dtype))
    lt = pre["loss_type"]
    if lt in ("score_matching", "data_prediction"):
        return c_skip() * x_t + c_out() * Fo
    if lt == "denoiser":
        return (Fo - x_t) / v(sig) ** 2
    raise ValueError(lt)
