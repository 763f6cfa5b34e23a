"""A/B timing of one eager (un-graphed) score-network evaluation at the benchmark shape under option settings.

    python tools/ab_forward.py [--batch 16] [--reps 4] tc_variant=8 tc_variant=0 inconv_variant=1 ...

Each positional `key=value` is applied on top of the defaults (all variants 0) for one measurement, then reset.
Prints ms per forward (CUDA events around `reps` forwards) and the summed wgmma conv time of one forward.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from sgmse_b200 import Engine, EngineConfig
from sgmse_b200.synth import synthetic_blob

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=16)
ap.add_argument("--reps", type=int, default=4)
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--T", type=int, default=512)
ap.add_argument("settings", nargs="*")
a = ap.parse_args()

cfg = EngineConfig(mode="fp16_tc", max_batch=a.batch, use_graphs=False)
eng = Engine(cfg)
eng.load_blob(synthetic_blob(eng, 0))
F = cfg.n_fft // 2 + 1
g = torch.Generator().manual_seed(0)
x = (torch.complex(torch.randn(a.batch, 2, F, a.T, generator=g), torch.randn(a.batch, 2, F, a.T, generator=g)) * 0.3).cuda()
t = torch.full((a.batch,), 0.5).cuda()
DEFAULTS = {"tc_variant": 0, "inconv_variant": 0, "outconv_variant": 0, "fir_variant": 0, "attn_variant": 0, "combine_variant": 0, "tc1_narrow": 0, "gn_self": 0, "gnfin_variant": 0,
            "pdl": 0}     # pdl=1 needs SGMSE_B200_PDL=1 (libsgmse_b200_pdl.so, `python -m sgmse_b200.build --pdl`)
settings = ["default"] + a.settings
times = {k: [] for k in settings}
convs = {}
errs = {}
ref = None
# interleaved rounds: the chip sits at its power cap, clocks drift with temperature -- only A/B/A/B medians are comparable
for rnd in range(a.rounds):
    for setting in settings:
        opts = dict(DEFAULTS)
        if setting != "default":
            for kv in setting.split(","):
                k, v = kv.split("=")
                opts[k] = int(v)
        for k, v in opts.items():
            eng.set_option(k, v)
        out = eng.dnn_forward(x, t)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            out = eng.dnn_forward(x, t)
        e1.record()
        torch.cuda.synchronize()
        times[setting].append(e0.elapsed_time(e1) / a.reps)
        if rnd == 0:
            eng.set_option("time_convs", 1)
            eng.dnn_forward(x, t)
            torch.cuda.synchronize()
            convs[setting] = (eng.counter("timed_conv_tc_us"), eng.counter("timed_conv_tc_mflop"), eng.counter("timed_conv_tc_count"),
                              eng.counter("launches_last_forward"))
            eng.set_option("time_convs", 0)
            if ref is None:
                ref = out.clone()
            errs[setting] = (torch.linalg.vector_norm(torch.view_as_real(out - ref)) / torch.linalg.vector_norm(torch.view_as_real(ref))).item()
for setting in settings:
    ts = sorted(times[setting])
    us, mf, cnt, nl = convs[setting]
    print(f"{setting:34s} median {ts[len(ts) // 2]:7.3f}  min {ts[0]:7.3f}  max {ts[-1]:7.3f} ms/forward  launches {nl:4d}  "
          f"tc convs {cnt:4d}: {us / 1e3:7.3f} ms = {mf / max(us, 1):7.1f} TFLOP/s  rel-L2 vs default {errs[setting]:.2e}", flush=True)
eng.close()
