"""Batched enhancement of many clips of different lengths (SURVEY.md §8f-2).

The reference's ``enhancement.py`` (lines 58-103) walks the files one by one: load, resample to the model's rate,
normalise by the clip's own peak, STFT, ``pad_spec`` to a multiple of 64 frames, sample, iSTFT to the original length,
renormalise, write.  Utterances are independent, so clips whose PADDED frame count is equal can share one sampler
launch sequence: this module buckets clips by padded frames, runs the per-clip front end (``sgmse_b200_analysis`` with
the clip's own length and peak), stacks the padded spectrograms of a bucket into batches for ``sgmse_b200_pc_sample``
(PC or Schroedinger-bridge kind) and runs the per-clip back end (``sgmse_b200_synthesis``).  With
``sampler_type="ode"`` each bucket goes whole to ``sgmse_b200_ode_sample_groups`` with one ODE system per clip, as
the reference's per-file ``enhance()`` solves it; the clips' network evaluations are batched.  Every clip's result is
bit-identical to enhancing it alone with the same ``(seed, utterance id)``; the ids are assigned in processing order
and returned.  The one sampler this cannot hold for is ``corrector='langevin'``, whose step size is a batch mean
(correctors.py:50-52: the clips of a batch are coupled): with it every clip is sampled as a batch of its own, which
is what the reference's file loop does.

Resampling and file I/O stay outside the engine (enhancement.py:66-71,100-103): pass callables.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch


def default_pad_mode(backbone: str) -> str:
    """enhancement.py:45-54: reflection padding for 'ncsnpp_48k' and 'ncsnpp_v2', zero padding otherwise."""
    return "reflection" if backbone in ("ncsnpp_48k", "ncsnpp_v2") else "zero_pad"


@dataclass
class Plan:
    """Which clips go together: ``batches`` = list of (padded_frames, [clip indices]); ``utt_id[i]`` = noise id of clip i."""
    batches: List[Tuple[int, List[int]]]
    utt_id: List[int]


def plan_batches(lengths: Sequence[int], padded_frames: Callable[[int], int], max_batch: int) -> Plan:
    """Bucket by padded frame count (ascending), keep the input order inside a bucket, cut buckets into batches of at
    most ``max_batch`` clips.  Noise ids follow the processing order so that a batch is a contiguous id range."""
    if max_batch < 1:
        raise ValueError("max_batch must be >= 1")
    buckets: Dict[int, List[int]] = {}
    for i, L in enumerate(lengths):
        if L <= 0:
            raise ValueError(f"clip {i} is empty")
        buckets.setdefault(int(padded_frames(int(L))), []).append(i)
    batches: List[Tuple[int, List[int]]] = []
    utt_id = [-1] * len(lengths)
    nxt = 0
    for tp in sorted(buckets):
        idx = buckets[tp]
        for b0 in range(0, len(idx), max_batch):
            chunk = idx[b0:b0 + max_batch]
            batches.append((tp, chunk))
            for i in chunk:
                utt_id[i] = nxt
                nxt += 1
    return Plan(batches, utt_id)


class BatchedEnhancer:
    """``enhancer = BatchedEnhancer(engine); outs, ids = enhancer(waves, seed=...)``.

    ``engine``: a ``sgmse_b200.Engine`` (anything with ``padded_frames / analysis / pc_sample / synthesis`` works, which
    is how the host logic is unit-tested without a GPU).  ``waves``: 1-D float tensors (any device), already at the
    model's sampling rate unless ``resample`` is given."""

    def __init__(self, engine, max_batch: Optional[int] = None, pad_mode: Optional[str] = None, device="cuda"):
        self.engine = engine
        self.max_batch = int(max_batch if max_batch is not None else engine.cfg.max_batch)
        self.pad_mode = pad_mode if pad_mode is not None else default_pad_mode(engine.cfg.backbone)
        self.device = device

    def __call__(self, waves: Sequence[torch.Tensor], seed: int = 0, sr: Optional[int] = None,
                 resample: Optional[Callable[[torch.Tensor, int, int], torch.Tensor]] = None, utt_base: int = 0,
                 noise_for: Optional[Callable[[int, int], torch.Tensor]] = None, sampler_type: str = "pc", **sampler_kw):
        """``utt_base``: first noise id of this call (a pipeline that feeds several calls keeps the ids of a run distinct).
        ``noise_for(clip_index, padded_frames)`` -> c64 [draws, 1, 1, F, Tpad]: injected noise per clip instead of the
        in-kernel Philox generator (parity tests against the reference's file loop); with the ODE sampler the one
        prior draw, c64 [1, 1, F, Tpad].
        ``sampler_type``: "pc" (``pc_sample`` keywords) or "ode" (``ode_sample_groups`` keywords: rtol, atol, eps,
        denoise, method, max_attempts); every clip's result equals ``enhance_ode`` of the clip alone with its id."""
        if sampler_type not in ("pc", "ode"):
            raise ValueError(f"sampler_type must be 'pc' or 'ode', got {sampler_type!r}")
        ode = sampler_type == "ode"
        if ode and sampler_kw.get("denoise", True):
            raise TypeError("ReverseDiffusionPredictor.update_fn() missing 1 required positional argument: 'stepsize' "
                            "(the reference's get_ode_sampler(denoise=True) fails the same way; pass denoise=False)")
        eng = self.engine
        target_sr = int(eng.cfg.sr)
        clips = []
        for w in waves:
            w = torch.as_tensor(w, dtype=torch.float32).reshape(-1)
            if sr is not None and sr != target_sr:
                if resample is None:
                    raise ValueError(f"clips are at {sr} Hz, the model at {target_sr} Hz: pass resample=")
                w = torch.as_tensor(resample(w, sr, target_sr), dtype=torch.float32).reshape(-1)
            clips.append(w)
        # corrector 'langevin' couples the clips of a batch (correctors.py:50-52) -> batches of one clip, as enhancement.py runs them
        max_batch = 1 if sampler_kw.get("corrector", "ald") == "langevin" else self.max_batch
        if ode:                    # one call per bucket: a finished clip's place goes to the next one of the bucket
            max_batch = max(1, len(clips))
        plan = plan_batches([int(w.numel()) for w in clips], eng.padded_frames, max_batch)
        outs: List[Optional[torch.Tensor]] = [None] * len(clips)
        for tp, idx in plan.batches:
            specs, norms = [], []
            for i in idx:                                   # per-clip front end: own length, own peak (enhancement.py:73-80)
                Y, norm = eng.analysis(clips[i].to(self.device)[None], pad_mode=self.pad_mode)
                assert Y.shape[-1] == tp
                specs.append(Y)
                norms.append(norm)
            kw = dict(sampler_kw)
            Ys = torch.cat(specs, dim=0)
            if ode:
                if noise_for is not None:
                    kw["prior_noise"] = torch.cat([torch.as_tensor(noise_for(i, tp)).to(self.device).reshape(1, *Ys.shape[1:])
                                                   for i in idx], dim=0)
                X, _ = eng.ode_sample_groups(Ys, group=1, seed=seed, utt_offset=utt_base + plan.utt_id[idx[0]], **kw)
            else:
                if noise_for is not None:
                    kw["noise"] = torch.cat([torch.as_tensor(noise_for(i, tp)).to(self.device) for i in idx], dim=1)
                X, _ = eng.pc_sample(Ys, seed=seed, utt_offset=utt_base + plan.utt_id[idx[0]], **kw)
            for j, i in enumerate(idx):                     # per-clip back end (enhancement.py:95-98)
                outs[i] = eng.synthesis(X[j:j + 1], norms[j], int(clips[i].numel()))[0]
        return outs, [utt_base + i for i in plan.utt_id]
