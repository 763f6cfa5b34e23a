"""The reference's ``enhancement.py`` directory loop (lines 38-103) as a pipelined service (SURVEY.md §8f-2, second half).

enhancement.py walks the files one by one: ``load`` -> ``resample`` to the model's rate (16 kHz, 48 kHz for ``ncsnpp_48k``;
lines 46-54, 62-66) -> normalise -> STFT -> sample -> iSTFT -> renormalise -> ``write`` (lines 68-103); disk, resampler and GPU
take turns.  Here the three stages overlap:

    reader threads (load + resample, ``io_workers``)  ->  GPU (BatchedEnhancer: clips bucketed by padded length)  ->  writer threads

Files are processed in windows of ``window`` files: while window k is on the GPU, window k + 1 is being read and window k - 1
is being written.  Per-file arithmetic is the ``BatchedEnhancer``'s (own peak normalisation, own length, pad mode per backbone).
Every file gets a noise id (returned): its result is bit-identical to enhancing that file alone with the same ``(seed, id)``;
ids follow the processing order (window by window, inside a window by padded length), so a run is reproducible for a given
(file list, window, max_batch, seed).  For the batch-coupled 'langevin' corrector every file is its own batch, as in the reference.

Audio I/O: ``soundfile`` is what the reference uses (``torchaudio.load`` / ``soundfile.write``); when it is not importable (the
build image has neither soundfile nor librosa) WAV files go through ``scipy.io.wavfile`` (PCM16 / PCM32 / float32 read, float32
write) and FLAC files are reported as unreadable.  Resampling: the reference calls ``librosa.resample`` (soxr_hq); without
librosa the default is ``torchaudio.functional.resample`` (windowed-sinc) -- a different anti-aliasing filter, i.e. NOT
sample-identical to the reference for files that need resampling; pass ``resample=`` to plug in the exact one.
"""
from __future__ import annotations

import concurrent.futures as cf
import glob
import os
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .service import BatchedEnhancer


def list_audio_files(test_dir: str) -> List[str]:
    """enhancement.py:38-43: *.wav, **/*.wav, *.flac, **/*.flac, each group sorted (non-recursive glob: one directory level)."""
    files: List[str] = []
    for pat in ("*.wav", os.path.join("**", "*.wav"), "*.flac", os.path.join("**", "*.flac")):
        files += sorted(glob.glob(os.path.join(test_dir, pat)))
    return files


def read_audio(path: str) -> Tuple[torch.Tensor, int]:
    """-> (float32 [channels, T] in [-1, 1], sampling rate), like ``torchaudio.load`` (enhancement.py:62)."""
    try:
        import soundfile as sf                                  # the reference's backend
        data, sr = sf.read(path, dtype="float32", always_2d=True)
        return torch.from_numpy(np.ascontiguousarray(data.T)), int(sr)
    except ImportError:
        pass
    if not path.lower().endswith(".wav"):
        raise RuntimeError(f"{path}: only WAV files can be read without the 'soundfile' package")
    from scipy.io import wavfile
    sr, data = wavfile.read(path)
    if data.dtype == np.int16:
        x = data.astype(np.float32) / 32768.0
    elif data.dtype == np.int32:
        x = data.astype(np.float32) / 2147483648.0
    elif data.dtype == np.uint8:
        x = (data.astype(np.float32) - 128.0) / 128.0
    else:
        x = data.astype(np.float32)
    if x.ndim == 1:
        x = x[:, None]
    return torch.from_numpy(np.ascontiguousarray(x.T)), int(sr)


def write_audio(path: str, x: np.ndarray, sr: int) -> None:
    """enhancement.py:102-103: makedirs + soundfile.write(path, x_hat, target_sr)."""
    os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
    try:
        import soundfile as sf
        sf.write(path, x, sr)
        return
    except ImportError:
        pass
    from scipy.io import wavfile
    wavfile.write(path, sr, np.asarray(x, dtype=np.float32))


def default_resample(x: torch.Tensor, sr: int, target_sr: int) -> torch.Tensor:
    import torchaudio.functional as AF
    return AF.resample(x, sr, target_sr)


class DirectoryEnhancer:
    """``DirectoryEnhancer(engine)(test_dir, enhanced_dir, N=30, corrector="ald", snr=0.5, ...)`` -> (written paths, noise ids).

    ``engine``: ``sgmse_b200.Engine`` (or any object a ``BatchedEnhancer`` accepts: the host logic is unit-tested with a
    stand-in).  ``window``: files per pipeline window (default 4 x the engine's micro-batch).  Keywords go to
    ``BatchedEnhancer``: ``sampler_type="ode", denoise=False, rtol=..., atol=...`` enhances with the ODE sampler, one
    system per file as the reference's file loop solves it."""

    def __init__(self, engine, window: Optional[int] = None, io_workers: int = 4, max_batch: Optional[int] = None,
                 resample: Optional[Callable[[torch.Tensor, int, int], torch.Tensor]] = None, device="cuda",
                 reader: Callable[[str], Tuple[torch.Tensor, int]] = read_audio,
                 writer: Callable[[str, np.ndarray, int], None] = write_audio):
        self.engine = engine
        self.enhancer = BatchedEnhancer(engine, max_batch=max_batch, device=device)
        self.window = int(window if window is not None else 4 * self.enhancer.max_batch)
        if self.window < 1:
            raise ValueError("window must be >= 1")
        self.io_workers = max(1, int(io_workers))
        self.resample = resample or default_resample
        self.reader, self.writer = reader, writer

    def _load(self, path: str) -> torch.Tensor:
        y, sr = self.reader(path)                               # [channels, T]
        target = int(self.engine.cfg.sr)
        if sr != target:                                        # enhancement.py:65-66
            y = torch.as_tensor(self.resample(y, sr, target), dtype=torch.float32)
        # the reference feeds y [channels, T] into a model whose STFT treats dim 0 as batch and squeezes the sample for
        # to_audio (enhancement.py:75,96): it only works for mono files; channel 0 is what a mono file is
        if y.shape[0] != 1:
            raise ValueError(f"{path}: {y.shape[0]} channels; the reference's file loop handles mono files only")
        return y[0].contiguous()

    def __call__(self, test_dir: str, enhanced_dir: str, seed: int = 0, files: Optional[Sequence[str]] = None, **sampler_kw):
        files = list(files) if files is not None else list_audio_files(test_dir)
        target = int(self.engine.cfg.sr)
        outs: List[str] = []
        all_ids: List[int] = []
        windows = [files[i:i + self.window] for i in range(0, len(files), self.window)]
        with cf.ThreadPoolExecutor(self.io_workers) as readers, cf.ThreadPoolExecutor(self.io_workers) as writers:
            pending = [readers.submit(self._load, f) for f in windows[0]] if windows else []
            writes: List[cf.Future] = []
            done_files = 0
            for wi, win in enumerate(windows):
                clips = [p.result() for p in pending]           # window wi is in memory ...
                pending = [readers.submit(self._load, f) for f in windows[wi + 1]] if wi + 1 < len(windows) else []   # ... wi + 1 starts loading
                enhanced, ids = self.enhancer(clips, seed=seed, utt_base=done_files, **sampler_kw)   # ids continue across windows
                all_ids += ids
                for f, x in zip(win, enhanced):
                    rel = f.replace(test_dir, "")
                    rel = rel[1:] if rel.startswith(os.sep) else rel    # enhancement.py:59-60
                    dst = os.path.join(enhanced_dir, rel)
                    writes.append(writers.submit(self.writer, dst, x.detach().cpu().numpy(), target))   # D2H here, disk in the pool
                    outs.append(dst)
                done_files += len(win)
            for w in writes:
                w.result()
        return outs, all_ids
