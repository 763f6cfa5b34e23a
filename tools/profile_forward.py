"""Run a few eager (un-graphed) score-network evaluations at the benchmark shape, for ncu.

    ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file /tmp/launches.csv \
        python tools/profile_forward.py --batch 16 --evals 2
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
ap.add_argument("--evals", type=int, default=2)
ap.add_argument("--T", type=int, default=512)
ap.add_argument("--mode", default="fp16_tc")
ap.add_argument("--backbone", default="ncsnpp")
ap.add_argument("--opt", action="append", default=[], metavar="KEY=VALUE", help="Engine.set_option before the evaluations")
a = ap.parse_args()

cfg = EngineConfig(mode=a.mode, max_batch=a.batch, use_graphs=False) if a.backbone == "ncsnpp" else \
    EngineConfig.ncsnpp_48k(mode=a.mode, max_batch=a.batch, use_graphs=False)
eng = Engine(cfg)
eng.load_blob(synthetic_blob(eng, 0))
for kv in a.opt:
    k, v = kv.split("=")
    eng.set_option(k, int(v))
F = cfg.n_fft // 2 + 1
g = torch.Generator().manual_seed(0)
x = (torch.complex(torch.randn(a.batch, 2, F, a.T, generator=g), torch.randn(a.batch, 2, F, a.T, generator=g)) * 0.3).cuda()
t = torch.full((a.batch,), 0.5).cuda()
for i in range(a.evals):
    out = eng.dnn_forward(x, t)
torch.cuda.synchronize()
print("launches per forward", eng.counter("launches_last_forward"), "tc", eng.counter("tc_convs_last_forward"),
      "direct", eng.counter("direct_convs_last_forward"), "finite", bool(torch.isfinite(torch.view_as_real(out)).all()))
