#!/usr/bin/env python
"""Probability-flow ODE sampler (SURVEY.md §8f-4) at the benchmark shape: wall/device time of one solve, evaluations
per second, and how much of the solve is NOT the score network (RK stage kernels, norm reductions, the one-double D2H
syncs).  Not a BASELINE.json metric -- a measuring tool for round 2.

    python tools/bench_ode.py --batch 16 --rtol 1e-2 --atol 1e-2 [--no-graphs]

With --groups G --clips B: B clips of 4 s (16 kHz, fp16_tc, max_batch 16) as ceil(B / G) independent systems, solved
in lockstep (Engine.ode_sample_groups) against one after another (Engine.ode_sample per system), alternated, at each
of --tols (rtol = atol).  Reports utterances/s, rounds, mean in-flight occupancy (utterance evaluations per network
forward), host syncs and the spread of nfe, and checks that both give the same bits.

    python tools/bench_ode.py --groups 1 --clips 16 --tols 1e-2,1e-5
"""
import argparse
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sgmse_b200 import Engine, EngineConfig          # noqa: E402
from sgmse_b200.synth import synthetic_blob, synthetic_speech   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--micro-batch", type=int, default=16)
    ap.add_argument("--rtol", type=float, default=1e-2)
    ap.add_argument("--atol", type=float, default=1e-2)
    ap.add_argument("--eps", type=float, default=0.03)
    ap.add_argument("--no-graphs", action="store_true")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--groups", type=int, default=0, help="utterances per ODE system: compare lockstep with one by one")
    ap.add_argument("--clips", type=int, default=16)
    ap.add_argument("--tols", default="1e-2,1e-5")
    a = ap.parse_args()
    if a.groups:
        return bench_groups(a)
    eng = Engine(EngineConfig(mode="fp16_tc", max_batch=a.micro_batch, use_graphs=not a.no_graphs))
    eng.load_blob(synthetic_blob(eng, seed=0))
    wav = synthetic_speech(a.batch, 64000).cuda()
    Y, _ = eng.analysis(wav)
    # one network evaluation alone, for the split
    x = torch.cat([Y, Y], dim=1)
    t = torch.full((a.batch,), 0.5, device="cuda")
    for _ in range(2):
        eng.dnn_forward(x, t)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(3):
        eng.dnn_forward(x, t)
    torch.cuda.synchronize()
    fwd_ms = (time.perf_counter() - t0) / 3 * 1e3
    for rep in range(a.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out, nfe, st = eng.ode_sample(Y, rtol=a.rtol, atol=a.atol, eps=a.eps, denoise=False, seed=1, return_stats=True)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        print(f"rep {rep}: {dt * 1e3:.1f} ms, nfe {nfe}, {st}, {nfe / dt:.1f} evaluations/s, {a.batch / dt:.2f} utterances/s; "
              f"network alone {fwd_ms:.2f} ms/eval -> {100 * (1 - nfe * fwd_ms * 1e-3 / dt):.1f} % of the solve is outside it; "
              f"the reference's host round trips would add 2 x {out.numel() * 8 / 1e6:.1f} MB of PCIe traffic per evaluation")
    assert torch.isfinite(torch.view_as_real(out)).all()
    eng.close()


def bench_groups(a):
    name = torch.cuda.get_device_name()
    eng = Engine(EngineConfig(mode="fp16_tc", max_batch=a.micro_batch, use_graphs=not a.no_graphs))
    eng.load_blob(synthetic_blob(eng, seed=0))
    wav = synthetic_speech(a.clips, 64000).cuda()
    Y, _ = eng.analysis(wav)
    G = a.groups
    # warm-up: one loose solve each way captures the forward graphs of the in-flight counts a solve's tail passes through
    eng.ode_sample_groups(Y, group=G, rtol=1e-1, atol=1e-1, eps=a.eps, denoise=False, seed=2)
    eng.ode_sample(Y[:G], rtol=1e-1, atol=1e-1, eps=a.eps, denoise=False, seed=2)
    for tol in (float(v) for v in a.tols.split(",")):
        kw = dict(rtol=tol, atol=tol, eps=a.eps, denoise=False, seed=1)
        times = {"lockstep": [], "one by one": []}
        for rep in range(a.reps):
            for arm in (("one by one", "lockstep") if rep % 2 == 0 else ("lockstep", "one by one")):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if arm == "lockstep":
                    out, nfes, st = eng.ode_sample_groups(Y, group=G, return_stats=True, **kw)
                else:
                    parts = [eng.ode_sample(Y[b:b + G], utt_offset=b, **kw) for b in range(0, a.clips, G)]
                    ref, ref_nfe = torch.cat([p[0] for p in parts]), [p[1] for p in parts]
                torch.cuda.synchronize()
                times[arm].append(time.perf_counter() - t0)
        assert torch.equal(out, ref) and nfes == ref_nfe, "lockstep and one-by-one solves differ"
        s0 = st[0]
        for arm, ts in times.items():
            print(f"{name}, tol {tol:g}, {arm}: " + ", ".join(f"{a.clips / t:.3f}" for t in ts) + " utterances/s")
        print(f"  nfe min/median/max {min(nfes)}/{sorted(nfes)[len(nfes) // 2]}/{max(nfes)}, total {sum(nfes)}; lockstep: "
              f"{s0['rounds']} rounds, {s0['forwards']} forwards, mean occupancy {s0['rows'] / max(1, s0['forwards']):.2f} "
              f"utterances per forward, {s0['syncs']} host syncs (one by one: {sum(nfes)} forwards at {G} utterance(s))")
    eng.close()


if __name__ == "__main__":
    main()
