"""STFT / iSTFT / magnitude compression / padding (oracle).

Follows sgmse/data_module.py:13-19 (window), :162-188
(spec_fwd / spec_back, 'exponent' transform), :190-218 (stft / istft kwargs) and
sgmse/util/other.py:76-90 (pad_spec).  The STFT itself is
restated with an explicit frame matrix + rfft so that the oracle does not share
``torch.stft`` with the reference; both are compared in tests/.

TEST INFRASTRUCTURE – see oracle/__init__.py.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch


@dataclass
class SpecConfig:
    n_fft: int = 510
    hop_length: int = 128
    window: str = "hann"            # 'hann' | 'sqrthann' (periodic)
    spec_factor: float = 0.15
    spec_abs_exponent: float = 0.5
    sr: int = 16000

    @staticmethod
    def cfg_48k():
        # README.md:89
        return SpecConfig(n_fft=1534, hop_length=384, spec_factor=0.065, spec_abs_exponent=0.667, sr=48000)


def get_window(cfg: SpecConfig, dtype=torch.float32):
    n = torch.arange(cfg.n_fft, dtype=torch.float64)
    w = 0.5 - 0.5 * torch.cos(2 * math.pi * n / cfg.n_fft)      # periodic Hann
    if cfg.window == "sqrthann":
        w = torch.sqrt(w)
    return w.to(dtype)


def stft(sig: torch.Tensor, cfg: SpecConfig) -> torch.Tensor:
    """[B, L] real -> c64 [B, n_fft//2+1, 1 + L//hop]   (center=True, reflect pad)."""
    pad = cfg.n_fft // 2
    x = torch.nn.functional.pad(sig[:, None, :], (pad, pad), mode="reflect")[:, 0]
    frames = x.unfold(-1, cfg.n_fft, cfg.hop_length)               # [B, nT, n_fft]
    frames = frames * get_window(cfg, sig.dtype)
    return torch.fft.rfft(frames, dim=-1).transpose(1, 2).contiguous()


def istft(spec: torch.Tensor, cfg: SpecConfig, length: int) -> torch.Tensor:
    """c64 [B, F, nT] -> [B, length]; overlap-add with window-envelope normalisation."""
    B, Fq, nT = spec.shape
    w = get_window(cfg, torch.float32 if spec.dtype == torch.complex64 else torch.float64)
    frames = torch.fft.irfft(spec.transpose(1, 2), n=cfg.n_fft, dim=-1) * w    # [B, nT, n_fft]
    total = cfg.n_fft + cfg.hop_length * (nT - 1)
    out = frames.new_zeros(B, total)
    env = frames.new_zeros(total)
    for i in range(nT):
        s = i * cfg.hop_length
        out[:, s:s + cfg.n_fft] += frames[:, i]
        env[s:s + cfg.n_fft] += w * w
    pad = cfg.n_fft // 2
    out = out[:, pad:pad + length] / env[pad:pad + length]
    if out.shape[1] < length:
        out = torch.nn.functional.pad(out, (0, length - out.shape[1]))
    return out


def spec_fwd(spec: torch.Tensor, cfg: SpecConfig) -> torch.Tensor:
    e = cfg.spec_abs_exponent
    if e != 1:
        spec = spec.abs() ** e * torch.exp(1j * spec.angle())
    return spec * cfg.spec_factor


def spec_back(spec: torch.Tensor, cfg: SpecConfig) -> torch.Tensor:
    spec = spec / cfg.spec_factor
    e = cfg.spec_abs_exponent
    if e != 1:
        spec = spec.abs() ** (1 / e) * torch.exp(1j * spec.angle())
    return spec


def pad_spec(Y: torch.Tensor, mode: str = "zero_pad") -> torch.Tensor:
    T = Y.size(-1)
    num_pad = (64 - T % 64) % 64
    if num_pad == 0:
        return Y
    if mode == "zero_pad":
        return torch.nn.functional.pad(Y, (0, num_pad))
    if mode == "reflection":
        pad = (0, num_pad, 0, 0) if Y.dim() == 4 else (0, num_pad)
        re = torch.nn.functional.pad(Y.real, pad, mode="reflect")
        im = torch.nn.functional.pad(Y.imag, pad, mode="reflect")
        return torch.complex(re, im)
    raise NotImplementedError(mode)
