"""Where the product mode's N = 30 error comes from: the full-size run of tests/golden/full_n30.npz (the unmodified reference's
own CPU enhancement of one 4-s clip) repeated under engine modes / A-B options that each remove ONE approximation.

    python tools/parity_decompose.py            # on the GPU; prints one line per setting (SI-SDR / rel-L2 vs the reference)

fp32            : CUDA-core validation mode (no approximation besides summation order)
fp16_direct     : CUDA-core convolutions, fp16 STORAGE of activations, exact expf SiLU -> what storage alone costs
fp16_tc         : the product mode (wgmma, fused GroupNorm+SiLU producers, fp16 FIR arithmetic, mma.sync ends)
fp16_tc + opts  : tc_variant=5 (GroupNorm+SiLU fused into the convolutions), fir_variant=1 (fp32 FIR), inconv_variant=1 /
                  outconv_variant=1 (CUDA-core fp32 4-channel ends)
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import pipeline as o_pipe, sde as o_sde, weights as o_w        # noqa: E402  (checker side of a measurement tool)
from oracle.arch import NetConfig                                          # noqa: E402
from sgmse_b200 import Engine, EngineConfig                                # noqa: E402
from sgmse_b200.synth import synthetic_speech                              # noqa: E402

z = np.load(os.path.join(ROOT, "tests", "golden", "full_n30.npz"))
L, N = int(z["L"]), int(z["N"])
sd = o_w.make_state_dict(NetConfig.ncsnpp(), seed=int(z["weight_seed"]))
wav = synthetic_speech(1, L, seed=int(z["wav_seed"]))
draws = o_sde.make_noise((1, 1, 256, 512), o_sde.n_noise_draws(N, "reverse_diffusion", "ald", 1), seed=int(z["noise_seed"]))
noise = torch.stack(draws).cuda()
ref = z["enh"]

SETTINGS = [("fp32", {}), ("fp16_direct", {}), ("fp16_tc", {}), ("fp16_tc", {"tc_variant": 5}), ("fp16_tc", {"fir_variant": 1}),
            ("fp16_tc", {"inconv_variant": 1}), ("fp16_tc", {"outconv_variant": 1}),
            ("fp16_tc", {"fir_variant": 1, "inconv_variant": 1, "outconv_variant": 1})]
outs = {}
for mode, opts in SETTINGS:
    eng = Engine(EngineConfig(mode=mode, max_batch=1))
    eng.load_state_dict(sd)
    for k, v in opts.items():
        eng.set_option(k, v)
    got = eng.enhance(wav.cuda(), noise=noise, N=N, predictor="reverse_diffusion", corrector="ald", corrector_steps=1,
                      snr=float(z["snr"]))[0].cpu().numpy()
    for k in opts:
        eng.set_option(k, 0)
    eng.close()
    name = mode + ("" if not opts else " " + ",".join(f"{k}={v}" for k, v in opts.items()))
    outs[name] = got
    sdr, rel = o_pipe.si_sdr(ref, got), float(np.linalg.norm(got - ref) / np.linalg.norm(ref))
    print(f"{name:80s} SI-SDR {sdr:6.1f} dB  rel-L2 {rel:.3e}", flush=True)
# how far apart two fp16 pipelines are from EACH OTHER (both carry storage rounding, in different places)
a, b = outs["fp16_tc"], outs["fp16_direct"]
print(f"fp16_tc vs fp16_direct: SI-SDR {o_pipe.si_sdr(b, a):.1f} dB, rel-L2 {np.linalg.norm(a - b) / np.linalg.norm(b):.3e}")
