"""Long recordings per backbone and mode: the planned activation workspace, one forward's time and the attention
kernels' share of it, and an N = 30 enhancement as seconds of audio per second.  Prints one line per (backbone, mode,
length) and a JSON summary; lengths that were not run are reported as not measured.

    python tools/long_clip.py --out DIR [--quick]

16 kHz lengths: 4.1 s (S = 512 attention tokens: the full-row fp32 kernel), 38.4 s (S = 4800: past its shared memory,
the streaming fp32 kernel), and 261.6 s, the longest clip the 2^31-element tensor limit admits.  48 kHz: 1.5, 12.8,
41.0 and 87.0 s (its only attention is in the bottleneck, far below the streaming kernel's range).
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from sgmse_b200 import Engine, EngineConfig
from sgmse_b200.synth import synthetic_blob

ap = argparse.ArgumentParser()
ap.add_argument("--out", default="long_clip_out")
ap.add_argument("--quick", action="store_true", help="skip the N = 30 enhancement past 40 s in fp32 mode")
ap.add_argument("--enhance-limit-s", type=float, default=300.0, help="longest clip timed end to end, per mode")
a = ap.parse_args()
os.makedirs(a.out, exist_ok=True)

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(f"card: {card}", flush=True)

BACKBONES = {"ncsnpp": (EngineConfig.ncsnpp_16k, 16000, [512, 4800, 32704]),
             "ncsnpp_48k": (EngineConfig.ncsnpp_48k, 48000, [192, 1600, 5120, 10880])}
rows = []


def timed(fn, reps=1):
    fn()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(reps):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / reps / 1e3


for name, (make, sr, lengths) in BACKBONES.items():
    for mode in ("fp16_tc", "tf32_tc", "fp32"):
        cfg = make(mode=mode, max_batch=1)
        eng = Engine(cfg)
        eng.load_blob(synthetic_blob(eng, 0))
        F = cfg.n_fft // 2 + 1
        for T in lengths:
            secs = T * cfg.hop_length / sr
            row = {"backbone": name, "mode": mode, "T": T, "seconds": round(secs, 2),
                   "planned_workspace_GB": eng.workspace_plan(1, F, T)["bytes"] / 1e9,
                   "workspace_without_reuse_GB": eng.workspace_bytes(1, F, T) / 1e9}
            try:
                g = torch.Generator().manual_seed(0)
                x = (torch.complex(torch.randn(1, 2, F, T, generator=g), torch.randn(1, 2, F, T, generator=g)) * 0.3).cuda()
                t = torch.full((1,), 0.5).cuda()
                row["forward_s"] = timed(lambda: eng.dnn_forward(x, t))
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    eng.dnn_forward(x, t)
                    torch.cuda.synchronize()
                ev = [e for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA]
                tot = sum(e.self_device_time_total for e in ev)
                att = sum(e.self_device_time_total for e in ev if "attention" in e.key)
                row["attention_share"] = att / tot if tot else None
                row["attention_kernels"] = sorted({e.key.split("<")[0] for e in ev if "attention" in e.key})
                free, total = torch.cuda.mem_get_info()
                row["device_used_GB"] = (total - free) / 1e9
                L = (T - 1) * cfg.hop_length          # frames 1 + L / hop, padded to T
                too_long = secs > a.enhance_limit_s or (a.quick and mode == "fp32" and secs > 40)
                if too_long:
                    row["enhance_audio_s_per_s"] = "not measured"
                else:
                    wav = (0.1 * torch.randn(1, L, generator=g)).cuda()
                    dt = timed(lambda: eng.enhance(wav, N=30, seed=1))
                    row["enhance_s"] = dt
                    row["enhance_audio_s_per_s"] = (L / sr) / dt
            except Exception as ex:                  # e.g. out of memory: reported, not hidden
                row["error"] = str(ex)[:200]
            print(json.dumps(row), flush=True)
            rows.append(row)
            torch.cuda.empty_cache()
        eng.close()

with open(os.path.join(a.out, "long_clip.json"), "w") as f:
    json.dump({"card": card, "rows": rows}, f, indent=1)
