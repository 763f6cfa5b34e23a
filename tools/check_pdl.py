"""A/B of programmatic dependent launch (PDL): correctness against the default library, then timing.

    python -m sgmse_b200.build --pdl                 # here (cross-compiles): sgmse_b200/lib/libsgmse_b200_pdl.so
    SGMSE_B200_PDL=1 python tools/check_pdl.py       # on the GPU: correctness first, then timing

The default library carries no PDL instruction (cuobjdump: 0 x ACQBULK / PREEXIT); the twin is the same sources with
-DSGMSE_B200_PDL, and even there the launches stay plain until `set_option("pdl", 1)`.  With PDL every kernel of the
launch sequence triggers its dependents at entry and waits (griddepcontrol.wait) after its on-chip prologue, so barrier
initialisation, tensor-map prefetch and weight-fragment staging of kernel k+1 overlap the tail of
kernel k -- inside the captured sampler graph as programmatic dependency edges.

Checks (bitwise): sampler output with pdl=1 == pdl=0, eager and graph-replayed, small config (fp32 + fp16_tc) and the
full-size network at [2, 256, 128]; then ms per 60-evaluation sampler call at the benchmark shape, interleaved A/B.
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
ap.add_argument("--N", type=int, default=30)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--skip-timing", action="store_true")
a = ap.parse_args()
assert os.environ.get("SGMSE_B200_PDL", "0") not in ("", "0"), "run with SGMSE_B200_PDL=1 (loads libsgmse_b200_pdl.so)"


def sample(eng, y, pdl, graphs, **kw):
    eng.set_option("pdl", pdl)
    eng.set_option("use_graphs", int(graphs))
    x, _ = eng.pc_sample(y, **kw)
    torch.cuda.synchronize()
    return x


def check(cfg, shape, label, **kw):
    eng = Engine(cfg)
    assert eng.counter("pdl_compiled") == 1
    eng.load_blob(synthetic_blob(eng, 0))
    g = torch.Generator().manual_seed(1)
    y = (torch.complex(torch.randn(*shape, generator=g), torch.randn(*shape, generator=g)) * 0.2).cuda()
    ref = sample(eng, y, 0, False, **kw)
    for pdl, graphs in ((1, False), (1, True), (0, True), (1, True)):
        got = sample(eng, y, pdl, graphs, **kw)
        ok = torch.equal(ref, got)
        print(f"{label}: pdl={pdl} graphs={graphs}: {'bit-identical' if ok else 'MISMATCH'}", flush=True)
        assert ok
    eng.close()


small = dict(nf=32, ch_mult=(1, 2, 2), image_size=64, num_res_blocks=1, attn_resolutions=(16,), n_fft=126, hop_length=32)
check(EngineConfig(mode="fp32", max_batch=2, **small), (2, 1, 64, 64), "small fp32", N=2, seed=3)
check(EngineConfig(mode="fp16_tc", max_batch=2, **small), (2, 1, 64, 64), "small fp16_tc", N=2, seed=3)
check(EngineConfig(mode="fp16_tc", max_batch=2), (2, 1, 256, 128), "full-size fp16_tc", N=2, seed=3)

if not a.skip_timing:
    cfg = EngineConfig(mode="fp16_tc", max_batch=a.batch, use_graphs=True)
    eng = Engine(cfg)
    eng.load_blob(synthetic_blob(eng, 0))
    g = torch.Generator().manual_seed(2)
    shape = (a.batch, 1, 256, 512)
    y = (torch.complex(torch.randn(*shape, generator=g), torch.randn(*shape, generator=g)) * 0.2).cuda()
    times = {0: [], 1: []}
    for rnd in range(a.rounds + 1):                       # round 0 = capture + warm-up
        for pdl in (0, 1):
            eng.set_option("pdl", pdl)
            eng.pc_sample(y, N=a.N, seed=rnd)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            eng.pc_sample(y, N=a.N, seed=rnd + 100)
            e1.record()
            torch.cuda.synchronize()
            if rnd:
                times[pdl].append(e0.elapsed_time(e1))
    for pdl in (0, 1):
        ts = sorted(times[pdl])
        print(f"pdl={pdl}: sampler call [{a.batch}, 256, 512] N={a.N}: median {ts[len(ts) // 2]:.1f} ms (min {ts[0]:.1f}, max {ts[-1]:.1f})")
    eng.close()
