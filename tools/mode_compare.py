"""fp32, tf32_tc and fp16_tc side by side at the config-2 shape [B,1,256,512] (full-size NCSN++, 4-s 16 kHz clips).

    python tools/mode_compare.py [--batch 4] [--steps 3] [--reps 3] [--out results.json]

For each mode: the graph-replayed network forward (CUDA events), the PC sampler's throughput over --steps reverse steps
(reverse_diffusion + ald: 2 evaluations per step), and the convolutions' TFLOP/s from the engine's per-convolution event
timing (counters timed_conv_tc_*, one eager forward).  The modes are measured in turn within each repetition, so clock and
power drift fall on all of them alike; the median over repetitions is reported.  The card name and power limit are printed
with the numbers.  Needs a CUDA device.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sgmse_b200 import Engine, EngineConfig          # noqa: E402
from sgmse_b200.synth import synthetic_blob           # noqa: E402

MODES = ("fp32", "tf32_tc", "fp16_tc")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timed(fn, n):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / n * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--T", type=int, default=512)
    ap.add_argument("--steps", type=int, default=3, help="PC sampler reverse steps per timed call")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--fwd-iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("mode_compare.py needs a CUDA device")
    B, T, F = a.batch, a.T, 256
    engines = {}
    for m in MODES:
        eng = Engine(EngineConfig(mode=m, max_batch=B, use_graphs=True))
        print(f"{m}: workspace {eng.workspace_bytes(B, F, T) / 2 ** 30:.2f} GiB at B={B}", flush=True)
        eng.load_blob(synthetic_blob(eng, 0))
        engines[m] = eng
    g = torch.Generator().manual_seed(0)
    x = (torch.complex(torch.randn(B, 2, F, T, generator=g), torch.randn(B, 2, F, T, generator=g)) * 0.3).cuda()
    y = x[:, 1:2].contiguous()
    t = torch.full((B,), 0.5).cuda()
    stream = torch.cuda.Stream()                      # a non-default stream: dnn_forward captures and replays a graph
    res = {m: {"fwd_s": [], "utt_per_s": [], "conv_tflops": []} for m in MODES}
    with torch.cuda.stream(stream):
        for m, eng in engines.items():                # warm-up: modules, workspaces, graphs
            eng.dnn_forward(x, t)
            eng.dnn_forward(x, t)
            eng.pc_sample(y, N=a.steps, seed=1)
        torch.cuda.synchronize()
        for _ in range(a.reps):
            for m, eng in engines.items():
                res[m]["fwd_s"].append(timed(lambda: eng.dnn_forward(x, t), a.fwd_iters))
                res[m]["utt_per_s"].append(B / timed(lambda: eng.pc_sample(y, N=a.steps, seed=1), 1))
                eng.set_option("time_convs", 1)
                eng.dnn_forward(x, t)
                us, mflop = eng.counter("timed_conv_tc_us"), eng.counter("timed_conv_tc_mflop")
                direct_us = eng.counter("timed_conv_direct_us")
                eng.set_option("time_convs", 0)
                res[m]["conv_tflops"].append(mflop / us if us > 0 else float("nan"))   # 1e6 flop / 1e-6 s = TFLOP/s
                res[m]["direct_conv_ms"] = direct_us * 1e-3
    gpu = card()
    out = {"gpu": gpu, "batch": B, "T": T, "pc_steps": a.steps, "reps": a.reps, "modes": {}}
    print(f"\n{gpu}  [B={B},1,{F},{T}]  median of {a.reps}, modes alternated")
    for m in MODES:
        r = res[m]
        med = {k: statistics.median(r[k]) for k in ("fwd_s", "utt_per_s", "conv_tflops")}
        out["modes"][m] = {**med, "runs": {k: r[k] for k in ("fwd_s", "utt_per_s", "conv_tflops")},
                           "direct_conv_ms": r.get("direct_conv_ms", 0.0)}
        tf = f"{med['conv_tflops']:.0f} TFLOP/s" if med["conv_tflops"] == med["conv_tflops"] else "no wgmma convolutions"
        print(f"  {m:8s} forward {med['fwd_s'] * 1e3:8.2f} ms  sampler {med['utt_per_s']:6.3f} utt/s ({a.steps} PC steps)  "
              f"convolutions: {tf}, CUDA-core {r.get('direct_conv_ms', 0.0):.1f} ms per forward")
    f32, t32 = out["modes"]["fp32"]["fwd_s"], out["modes"]["tf32_tc"]["fwd_s"]
    print(f"  tf32_tc forward speed-up over fp32: {f32 / t32:.2f}x; over fp16_tc: "
          f"{out['modes']['fp16_tc']['fwd_s'] / t32:.2f}x")
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(out, fh, indent=1)
    for eng in engines.values():
        eng.close()


if __name__ == "__main__":
    main()
