"""GPU parity tests: the CUDA engine (through the C-ABI) against the CPU oracle and the committed
reference golden fixtures.  Run on a GPU host: ``pytest -m gpu``.

Tolerances: every bound below is about 2x the error measured (on an H100, values in the comments):
  * mode fp32 (CUDA-core validation path): rel-L2 of a few 1e-6 per forward, per sampler run and per waveform vs the
    fp32 CPU oracle / the reference fixtures;
  * mode fp16_tc (product path: fp16 activation storage, wgmma MMA with fp32 accumulation -- the same 10-bit mantissa as
    the TF32 cuDNN path the reference itself takes on a GPU): 1.9e-3 .. 2.5e-3 per forward, 0.5e-3 .. 1.7e-3 after 3 .. 12
    sampler steps on the mid-size network, 1.35e-2 (37.4 dB SI-SDR) after the full N = 30 run of the full-size network
    (tests/test_gpu_zz_next_rows.py; storage rounding random-walks through 60 evaluations).
"""
import math
import os

import numpy as np
import pytest
import torch

from oracle import ncsnpp as o_net, sde as o_sde, spec as o_spec, pipeline as o_pipe, weights as o_w
from oracle.arch import NetConfig
from sgmse_b200 import Engine, EngineConfig

pytestmark = pytest.mark.gpu

SMALL_N = dict(nf=16, ch_mult=(1, 2, 2), image_size=64, num_res_blocks=2)
SMALL_E = dict(nf=16, ch_mult=(1, 2, 2), image_size=64, num_res_blocks=2, n_fft=126, hop_length=32)


def rel_l2(a, b):
    a, b = torch.as_tensor(a).cpu(), torch.as_tensor(b).cpu()
    return (torch.linalg.vector_norm((a - b).reshape(-1)) / torch.linalg.vector_norm(b.reshape(-1))).item()


def load_golden(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    sd = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w/")}
    return z, sd


def small_engine(kind, mode, **kw):
    if kind == "ncsnpp_small":
        return Engine(EngineConfig(attn_resolutions=(16,), mode=mode, **SMALL_E, **kw))
    return Engine(EngineConfig.ncsnpp_48k(mode=mode, theta=1.5, sigma_min=0.05, sigma_max=0.5, spec_factor=0.15,
                                          spec_abs_exponent=0.5, **SMALL_E, **kw))


# ------------------------------------------------------------------------------------------------
# golden fixtures (outputs of the unmodified reference), small configs, every arithmetic mode that
# supports 16/32-channel layers
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["ncsnpp_small", "ncsnpp48k_small"])
# measured on an H100: fp32 1.8e-6 / 9.1e-7, fp16_direct 2.4e-3 / 1.1e-3 (ncsnpp_small / ncsnpp48k_small)
@pytest.mark.parametrize("mode,tol", [("fp32", 3.7e-6), ("fp16_direct", 4.9e-3)])
def test_golden_forward_and_score(golden_dir, name, mode, tol):
    z, sd = load_golden(golden_dir, name)
    eng = small_engine(name, mode)
    eng.load_state_dict(sd)
    x, y, t = (torch.from_numpy(z[k]).cuda() for k in ("x", "y", "t"))
    out = eng.dnn_forward(torch.cat([x, y], 1), t)
    e1, e2 = rel_l2(out, z["dnn_out"]), rel_l2(eng.score(x, y, t), z["score"])
    print(f"golden {name} {mode}: dnn rel-L2 {e1:.3e}, score rel-L2 {e2:.3e}")
    assert e1 < tol and e2 < tol
    eng.close()


@pytest.mark.parametrize("name", ["ncsnpp_small", "ncsnpp48k_small"])
@pytest.mark.parametrize("pred,corr", [("reverse_diffusion", "ald"), ("reverse_diffusion", "langevin"),
                                       ("none", "ald"), ("reverse_diffusion", "none")])
def test_golden_pc_sampler(golden_dir, name, pred, corr):
    z, sd = load_golden(golden_dir, name)
    eng = small_engine(name, "fp32")
    eng.load_state_dict(sd)
    y = torch.from_numpy(z["y"]).cuda()
    N = 3
    draws = o_sde.make_noise(tuple(y.shape), o_sde.n_noise_draws(N, pred, corr, 1), seed=7)
    noise = torch.stack(draws).cuda()
    smp, nfe = eng.pc_sample(y, noise=noise, N=N, predictor=pred, corrector=corr, corrector_steps=1, snr=0.5)
    assert nfe == int(z[f"nfe_{pred}_{corr}"])
    e = rel_l2(smp, z[f"pc_{pred}_{corr}"])
    print(f"golden {name} pc {pred}+{corr}: rel-L2 {e:.3e}")
    assert e < 1.9e-6                              # measured <= 9.4e-7 over the eight cases (H100)
    eng.close()


@pytest.mark.parametrize("name", ["ncsnpp_small", "ncsnpp48k_small"])
def test_golden_enhance_chain(golden_dir, name):
    z, sd = load_golden(golden_dir, name)
    eng = small_engine(name, "fp32")
    eng.load_state_dict(sd)
    wav = torch.from_numpy(z["wav"])
    B, N = wav.shape[0], 3
    draws = o_sde.make_noise((B, 1, 64, 64), o_sde.n_noise_draws(N, "reverse_diffusion", "ald", 1), seed=11)
    Y, norm = eng.analysis(wav.cuda())
    e_y = rel_l2(Y, z["Y"])
    xh = eng.enhance(wav.cuda(), noise=torch.stack(draws).cuda(), N=N)
    e_w = rel_l2(xh, z["enh"])
    print(f"golden {name} chain: spectrogram rel-L2 {e_y:.3e}, waveform rel-L2 {e_w:.3e}")
    assert e_y < 4.3e-7 and e_w < 1.3e-6            # measured 2.1e-7 / 6.3e-7 (H100)
    # host-buffer entry point (H2D/D2H inside the call) gives the same result
    xh2 = eng.enhance(wav.pin_memory(), noise=torch.stack(draws).cuda(), N=N)
    assert torch.equal(xh.cpu(), xh2)
    eng.close()


# ---- SURVEY.md §8f-1: ncsnpp_v2 behind ScoreModel.forward's preconditioning, Schroedinger-bridge samplers ----
V2_PRECOND = {
    "plain": dict(loss_type="data_prediction", network_scaling=None, c_in="1", c_out="1", c_skip="0", sigma_data=0.1),
    "edm": dict(loss_type="data_prediction", network_scaling="1/sigma", c_in="edm", c_out="edm", c_skip="edm", sigma_data=0.1),
}


def v2_engine(mode, sde="sbve", **pre):
    return Engine(EngineConfig.ncsnpp_v2(attn_resolutions=(16,), mode=mode, sde=sde, sb_k=2.6, sb_c=0.4, **SMALL_E, **pre))


@pytest.mark.parametrize("mode,tol", [("fp32", 2e-4), ("fp16_direct", 2e-2)])
def test_golden_v2_forward_and_preconditioning(golden_dir, mode, tol):
    z, sd = load_golden(golden_dir, "ncsnpp_v2_small")
    x, y, t = (torch.from_numpy(z[k]).cuda() for k in ("x", "y", "t"))
    for tag, pre in V2_PRECOND.items():
        eng = v2_engine(mode, **pre)
        eng.load_state_dict(sd)
        if tag == "plain":
            assert rel_l2(eng.dnn_forward(torch.cat([x, y], 1), t), z["dnn_out"]) < tol      # NCSNpp_v2.forward(x, y, t)
        assert rel_l2(eng.model_forward(x, y, t), z[f"fwd_{tag}"]) < tol
        eng.close()
    eng = v2_engine(mode, sde="ouve", loss_type="score_matching", c_out="1/sigma")
    eng.load_state_dict(sd)
    assert rel_l2(eng.model_forward(x, y, t), z["fwd_ouve_score"]) < tol
    eng.close()


@pytest.mark.parametrize("tag", list(V2_PRECOND))
@pytest.mark.parametrize("sampler_type", ["sde", "ode"])
def test_golden_v2_sb_sampler(golden_dir, tag, sampler_type):
    z, sd = load_golden(golden_dir, "ncsnpp_v2_small")
    eng = v2_engine("fp32", **V2_PRECOND[tag])
    eng.load_state_dict(sd)
    y = torch.from_numpy(z["y"]).cuda()
    noise = torch.stack(o_sde.make_noise(tuple(y.shape), 3, seed=13)).cuda() if sampler_type == "sde" else None
    smp, n = eng.sb_sample(y, sampler_type=sampler_type, N=3, noise=noise)
    assert n == int(z[f"sb_n_{sampler_type}_{tag}"])
    # the first ODE step multiplies x and y (equal at that point) by +-2.25e3: ~2e-4 of fp32 noise in the reference itself
    assert rel_l2(smp, z[f"sb_{sampler_type}_{tag}"]) < 1e-3
    # Philox noise + CUDA-graph replay: finite, reproducible, and independent of the micro-batch split
    a, _ = eng.sb_sample(y, sampler_type=sampler_type, N=3, seed=5)
    b, _ = eng.sb_sample(y, sampler_type=sampler_type, N=3, seed=5)
    assert torch.isfinite(torch.view_as_real(a)).all() and torch.equal(a, b)
    eng.close()


def test_golden_v2_pc_sampler_on_ouve(golden_dir):
    z, sd = load_golden(golden_dir, "ncsnpp_v2_small")
    eng = v2_engine("fp32", sde="ouve", loss_type="score_matching", c_out="1/sigma")
    eng.load_state_dict(sd)
    y = torch.from_numpy(z["y"]).cuda()
    draws = o_sde.make_noise(tuple(y.shape), o_sde.n_noise_draws(3, "reverse_diffusion", "ald", 1), seed=7)
    smp, nfe = eng.pc_sample(y, noise=torch.stack(draws).cuda(), N=3, predictor="reverse_diffusion", corrector="ald",
                             corrector_steps=1, snr=0.5)
    assert nfe == 6 and rel_l2(smp, z["pc_ouve_score"]) < 1e-3
    eng.close()




def test_golden_stft_ops(golden_dir):
    z = np.load(os.path.join(golden_dir, "ops.npz"))
    eng = Engine(EngineConfig(mode="fp32", **SMALL_E))
    wav = torch.from_numpy(z["wav"]).cuda()
    Y, norm = eng.analysis(wav)
    nrm = torch.from_numpy(z["wav"]).abs().amax(dim=1)
    assert torch.allclose(norm.cpu(), nrm)
    # reference chain on the normalised waveform
    scfg = o_spec.SpecConfig(n_fft=126, hop_length=32)
    Yo = o_spec.pad_spec(o_spec.spec_fwd(o_spec.stft(torch.from_numpy(z["wav"]) / nrm[:, None], scfg), scfg))[:, None]
    assert rel_l2(Y, Yo) < 1e-5
    # synthesis == to_audio of the *padded* spectrogram (like the reference, the zero-padded frames take part
    # in the overlap-add and its window envelope, model.py:457 / data_module.py:216-218)
    back = eng.synthesis(Y, norm, 2000)
    want = o_spec.istft(o_spec.spec_back(Yo[:, 0], scfg), scfg, 2000) * nrm[:, None]
    assert rel_l2(back, want) < 1e-4
    assert rel_l2(back[:, :1900], z["wav"][:, :1900]) < 1e-4      # away from the padded tail it is the identity
    eng.close()
    e48 = Engine(EngineConfig.ncsnpp_48k(mode="fp32"))
    w48 = torch.from_numpy(z["wav48"]).cuda()
    Y48, n48 = e48.analysis(w48)
    s48 = o_spec.SpecConfig.cfg_48k()
    nrm48 = torch.from_numpy(z["wav48"]).abs().amax(dim=1)
    Yo48 = o_spec.pad_spec(o_spec.spec_fwd(o_spec.stft(torch.from_numpy(z["wav48"]) / nrm48[:, None], s48), s48)[:, None])
    assert Y48.shape == Yo48.shape
    assert rel_l2(Y48, Yo48) < 1e-5
    want48 = o_spec.istft(o_spec.spec_back(Yo48[:, 0], s48), s48, 6000) * nrm48[:, None]
    assert rel_l2(e48.synthesis(Y48, n48, 6000), want48) < 1e-4
    # reflection padding (enhancement.py:46-54 uses it for ncsnpp_48k): 79 frames -> 128
    g = torch.Generator().manual_seed(9)
    wl = 0.1 * torch.randn(2, 30000, generator=g)
    Yr, nr = e48.analysis(wl.cuda(), pad_mode="reflection")
    nl = wl.abs().amax(dim=1)
    Yor = o_spec.pad_spec(o_spec.spec_fwd(o_spec.stft(wl / nl[:, None], s48), s48)[:, None], "reflection")
    assert Yr.shape == Yor.shape and rel_l2(Yr, Yor) < 1e-5
    # like ReflectionPad2d, padding by more than the signal has frames is an error, not garbage
    with pytest.raises(RuntimeError, match="reflection"):
        e48.analysis(w48, pad_mode="reflection")
    e48.close()


# ------------------------------------------------------------------------------------------------
# per-module parity (oracle taps) on a mid-size config that exercises the wgmma path (C = 64..256)
# ------------------------------------------------------------------------------------------------
MID_N = NetConfig.ncsnpp(nf=64, ch_mult=(1, 2, 2), image_size=64, attn_resolutions=(16,), num_res_blocks=1)
MID_E = dict(nf=64, ch_mult=(1, 2, 2), image_size=64, attn_resolutions=(16,), num_res_blocks=1, n_fft=126, hop_length=32)


# measured on an H100 (worst module, pyr2): 3.6e-6, 2.53e-3, 2.47e-3
@pytest.mark.parametrize("mode,tol", [("fp32", 7.2e-6), ("fp16_direct", 5.1e-3), ("fp16_tc", 5.1e-3)])
def test_per_module_taps_mid(mode, tol):
    sd = o_w.make_state_dict(MID_N, seed=5)
    eng = Engine(EngineConfig(mode=mode, **MID_E))
    eng.load_state_dict(sd)
    eng.set_option("record_taps", 1)
    g = torch.Generator().manual_seed(3)
    B, F, T = 3, 64, 128
    x = torch.complex(torch.randn(B, 2, F, T, generator=g), torch.randn(B, 2, F, T, generator=g)) * 0.4
    t = torch.tensor([0.9, 0.35, 0.05])
    taps = {}
    ref = o_net.forward(sd, MID_N, x, t, taps=taps)
    out = eng.dnn_forward(x.cuda(), t.cuda())
    if mode == "fp16_tc":
        assert eng.counter("tc_convs_last_forward") > 0
    worst = []
    for name, v in taps.items():
        if name == "temb":
            continue
        got = eng.tap(name)
        worst.append((rel_l2(got, v), name))
    worst.sort(reverse=True)
    e_out = rel_l2(out, ref)
    print(f"per-module taps {mode}: worst {worst[0][1]} rel-L2 {worst[0][0]:.3e}, output rel-L2 {e_out:.3e}")
    assert worst[0][0] < tol, worst[:5]
    assert e_out < tol
    eng.close()


# ------------------------------------------------------------------------------------------------
# full-size network (VoiceBank config, 65.6 M parameters): product path vs oracle
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full_sd():
    return o_w.make_state_dict(NetConfig.ncsnpp(), seed=0)


# measured on an H100: 3.92e-6, 2.34e-3, 1.88e-3
@pytest.mark.parametrize("mode,tol,T", [("fp32", 8e-6, 128), ("fp16_tc", 5.2e-3, 128), ("fp16_tc", 4.3e-3, 512)])
def test_full_size_forward(full_sd, mode, tol, T):
    """T=128 (1-s clip): the coarsest levels hold < 32 pixels and take the CUDA-core path even in fp16_tc mode;
    T=512 (the 4-s benchmark shape): every convolution must run on wgmma."""
    cfg = NetConfig.ncsnpp()
    eng = Engine(EngineConfig(mode=mode, max_batch=2))
    eng.load_state_dict(full_sd)
    g = torch.Generator().manual_seed(11)
    B, F = 1, 256
    x = torch.complex(torch.randn(B, 2, F, T, generator=g), torch.randn(B, 2, F, T, generator=g)) * 0.3
    t = torch.tensor([0.5])
    with torch.no_grad():
        ref = o_net.forward(full_sd, cfg, x, t)
    out = eng.dnn_forward(x.cuda(), t.cuda())
    err = rel_l2(out, ref)
    print(f"full-size forward {mode} T={T}: rel-L2 {err:.3e}")
    assert err < tol
    if mode == "fp16_tc":
        assert eng.counter("tc_convs_last_forward") > 0
        if T == 512:
            assert eng.counter("direct_convs_last_forward") == 0
    eng.close()




def test_full_size_48k_forward():
    """BASELINE config 3 backbone (ncsnpp_48k defaults: no progressive skips, attention only in the bottleneck,
    output_layer before /t), 64.7 M parameters, F = 768."""
    cfg = NetConfig.ncsnpp_48k()
    sd = o_w.make_state_dict(cfg, seed=4)
    eng = Engine(EngineConfig.ncsnpp_48k(mode="fp16_tc", max_batch=1))
    eng.load_state_dict(sd)
    g = torch.Generator().manual_seed(13)
    x = torch.complex(torch.randn(1, 2, 768, 128, generator=g), torch.randn(1, 2, 768, 128, generator=g)) * 0.3
    t = torch.tensor([0.31])
    with torch.no_grad():
        ref = o_net.forward(sd, cfg, x, t)
    out = eng.dnn_forward(x.cuda(), t.cuda())
    err = rel_l2(out, ref)
    print(f"full-size 48k forward fp16_tc: rel-L2 {err:.3e}")
    assert err < 4.8e-3 and eng.counter("tc_convs_last_forward") > 0          # measured 2.08e-3 (H100)
    eng.close()


def test_end_to_end_si_sdr(full_sd):
    """Waveform-level agreement of the product path with the oracle on the full-size network (N=2, injected noise):
    SI-SDR(oracle, engine) as defined in the reference (util/other.py:64-68).  PESQ is not installable offline."""
    cfg = NetConfig.ncsnpp()
    eng = Engine(EngineConfig(mode="fp16_tc", max_batch=1))
    eng.load_state_dict(full_sd)
    g = torch.Generator().manual_seed(21)
    L, N = 16000, 2                                  # 1-s clip -> 126 frames -> padded to 128
    wav = 0.1 * torch.randn(1, L, generator=g)
    Tp = eng.padded_frames(L)
    draws = o_sde.make_noise((1, 1, 256, Tp), o_sde.n_noise_draws(N, "reverse_diffusion", "ald", 1), seed=8)
    ref = o_pipe.enhance(full_sd, cfg, o_spec.SpecConfig(), o_sde.OUVE(), wav, draws, N=N)[0].numpy()
    got = eng.enhance(wav.cuda(), noise=torch.stack(draws).cuda(), N=N)[0].cpu().numpy()
    sdr = o_pipe.si_sdr(ref, got)
    print(f"end-to-end SI-SDR(oracle, engine) = {sdr:.1f} dB")
    assert sdr > 48.7                              # measured 55.6 dB on an H100; twice the error = -6 dB
    eng.close()


def test_tc_kernel_variants_agree(full_sd):
    """The wgmma convolution with TMA-fed operands and separate gn_apply launches (default) and with GroupNorm+SiLU fused
    into its operand producer (tc_variant 5) compute the same network."""
    eng = Engine(EngineConfig(mode="fp16_tc", max_batch=2))
    eng.load_state_dict(full_sd)
    g = torch.Generator().manual_seed(12)
    x = (torch.complex(torch.randn(2, 2, 256, 512, generator=g), torch.randn(2, 2, 256, 512, generator=g)) * 0.3).cuda()
    t = torch.tensor([0.7, 0.1]).cuda()
    outs = {}
    with pytest.raises(RuntimeError, match="tc_variant"):
        eng.set_option("tc_variant", 2)
    for variant in (5, 0):
        eng.set_option("tc_variant", variant)
        outs[variant] = eng.dnn_forward(x, t)
        assert eng.counter("direct_convs_last_forward") == 0
        assert torch.isfinite(torch.view_as_real(outs[variant])).all()
    err = rel_l2(outs[5], outs[0])
    print(f"tc variants: fused vs unfused rel-L2 {err:.3e}")
    assert err < 5e-3
    # attention: mma.sync with cp.async staging (default) vs plain staging (3) vs fp32 CUDA-core (1)
    eng.set_option("attn_variant", 3)
    o2 = eng.dnn_forward(x, t)
    eng.set_option("attn_variant", 1)
    o1 = eng.dnn_forward(x, t)
    eng.set_option("attn_variant", 0)
    print(f"attention kernels, network output: cp.async staging vs fp32 CUDA-core rel-L2 {rel_l2(outs[0], o1):.3e}, plain staging vs fp32 {rel_l2(o2, o1):.3e}")
    assert rel_l2(outs[0], o1) < 3e-3 and rel_l2(o2, o1) < 3e-3
    eng.set_option("tc_variant", 0)
    eng.close()


def test_small_end_kernel_variants_agree(full_sd):
    """The mma.sync input conv (state rounded to fp16, K padded 36 -> 48) against the fp32-FMA CUDA-core kernel; the
    progressive-output conv on mma.sync against the CUDA-core kernel with fp32 weights, and with GroupNorm+SiLU fused
    into its staging (opt-in variant 2: same expression, same rounding point -> bit-identical); the one-MUFU / half2
    FIR resamplers against the expf / fp32 ones."""
    eng = Engine(EngineConfig(mode="fp16_tc", max_batch=2))
    eng.load_state_dict(full_sd)
    g = torch.Generator().manual_seed(13)
    x = (torch.complex(torch.randn(2, 2, 256, 128, generator=g), torch.randn(2, 2, 256, 128, generator=g)) * 0.3).cuda()
    t = torch.tensor([0.6, 0.05]).cuda()
    eng.set_option("record_taps", 1)
    base = eng.dnn_forward(x, t)
    tap0 = eng.tap("in_conv")
    eng.set_option("outconv_variant", 1)
    cuda_core = eng.dnn_forward(x, t)
    eng.set_option("outconv_variant", 2)
    fused = eng.dnn_forward(x, t)
    eng.set_option("outconv_variant", 0)
    assert rel_l2(cuda_core, base) < 2e-3
    assert torch.equal(fused, base)
    eng.set_option("inconv_variant", 1)
    cc = eng.dnn_forward(x, t)
    tap1 = eng.tap("in_conv")
    eng.set_option("inconv_variant", 0)
    e_in = (torch.linalg.vector_norm(tap0 - tap1) / torch.linalg.vector_norm(tap1)).item()
    eng.set_option("fir_variant", 1)
    slow_fir = eng.dnn_forward(x, t)
    eng.set_option("fir_variant", 0)
    print(f"input conv mma vs CUDA-core: rel-L2 {e_in:.3e}; network output {rel_l2(cc, base):.3e}; "
          f"out conv mma vs CUDA-core {rel_l2(cuda_core, base):.3e}; FIR fast vs fp32 {rel_l2(slow_fir, base):.3e}")
    assert e_in < 2e-3 and rel_l2(cc, base) < 5e-3 and rel_l2(slow_fir, base) < 5e-3
    eng.close()


def test_full_size_sampler_properties(full_sd):
    """Size-independent properties at the benchmark shape [B,1,256,512]:
    graph replay == eager launch sequence (bitwise), outputs do not depend on how the batch is split into
    micro-batches (noise is keyed by global utterance id), and a different seed changes the result."""
    eng = Engine(EngineConfig(mode="fp16_tc", max_batch=2, use_graphs=True))
    eng.load_state_dict(full_sd)
    g = torch.Generator().manual_seed(1)
    B, F, T = 3, 256, 512
    y = (torch.complex(torch.randn(B, 1, F, T, generator=g), torch.randn(B, 1, F, T, generator=g)) * 0.1).cuda()
    a, nfe = eng.pc_sample(y, N=2, seed=1234)
    assert nfe == 4 and torch.isfinite(torch.view_as_real(a)).all()
    b, _ = eng.pc_sample(y, N=2, seed=1234)                  # graph replay
    assert torch.equal(a, b)
    eng.set_option("use_graphs", 0)
    c, _ = eng.pc_sample(y, N=2, seed=1234)                  # eager
    assert torch.equal(a, c)
    d, _ = eng.pc_sample(y[1:2], N=2, seed=1234, utt_offset=1)   # utterance 1 alone
    assert torch.equal(a[1:2], d)
    e, _ = eng.pc_sample(y, N=2, seed=99)
    assert not torch.equal(a, e)
    assert eng.counter("graph_launches") >= 2
    eng.close()


# ------------------------------------------------------------------------------------------------
# the PRODUCT mode (fp16_tc) against reference-generated fixtures (tests/golden/ncsnpp_mid.npz, oracle/make_golden.py:
# golden_mid_tc: outputs of the unmodified reference on a tensor-core-tileable config; weights / inputs / noise from seeds)
# ------------------------------------------------------------------------------------------------
MID_PAIRS = [("reverse_diffusion", "ald", 3), ("reverse_diffusion", "langevin", 3), ("none", "ald", 3),
             ("reverse_diffusion", "none", 3), ("reverse_diffusion", "ald", 12)]
# bounds about 2x the error of the worst pair, measured on an H100: fp32 score 3.2e-6, pc <= 2.2e-6, chain 2.0e-6;
# fp16_tc score 2.36e-3, pc <= 1.65e-3, chain 1.68e-3 (SI-SDR 54.4 dB)
MID_TOL = {"fp32": dict(score=6.4e-6, pc=4.4e-6, enh=4.1e-6, n50=1.9e-6), "fp16_tc": dict(score=5e-3, pc=3.4e-3, enh=3.6e-3, n50=1.9e-3)}   # N=50: measured 9.3e-7 / 9.8e-4


@pytest.mark.parametrize("mode", ["fp32", "fp16_tc"])
def test_golden_mid_sampler_and_chain(golden_dir, mode):
    z = np.load(os.path.join(golden_dir, "ncsnpp_mid.npz"))
    sd = o_w.make_state_dict(MID_N, seed=int(z["weight_seed"]))
    eng = Engine(EngineConfig(mode=mode, max_batch=2, **MID_E))
    eng.load_state_dict(sd)
    x, y, t = (torch.from_numpy(z[k]).cuda() for k in ("x", "y", "t"))
    tol = MID_TOL[mode]
    e_score = rel_l2(eng.score(x, y, t), z["score"])
    if mode == "fp16_tc":
        assert eng.counter("tc_convs_last_forward") > 0
    report = [f"score {e_score:.3e}"]
    assert e_score < tol["score"]
    for pred, corr, N in MID_PAIRS:
        draws = o_sde.make_noise(tuple(y.shape), o_sde.n_noise_draws(N, pred, corr, 1), seed=7)
        smp, nfe = eng.pc_sample(y, noise=torch.stack(draws).cuda(), N=N, predictor=pred, corrector=corr, corrector_steps=1, snr=0.5)
        assert nfe == int(z[f"nfe_{pred}_{corr}_N{N}"])
        e = rel_l2(smp, z[f"pc_{pred}_{corr}_N{N}"])
        report.append(f"{pred}+{corr} N={N} {e:.3e}")
        assert e < tol["pc"], report
    # BASELINE config 4 sampler settings (README.md:43: N = 50, snr 0.33 -> 100 evaluations)
    draws = o_sde.make_noise(tuple(y.shape), o_sde.n_noise_draws(50, "reverse_diffusion", "ald", 1), seed=9)
    smp, nfe = eng.pc_sample(y, noise=torch.stack(draws).cuda(), N=50, predictor="reverse_diffusion", corrector="ald", corrector_steps=1, snr=0.33)
    e50 = rel_l2(smp, z["pc_dereverb_N50_snr033"])
    report.append(f"dereverb settings N=50 snr 0.33 {e50:.3e}")
    assert nfe == int(z["nfe_dereverb_N50_snr033"]) == 100 and e50 < tol["n50"], report
    wav = torch.from_numpy(z["wav"])
    draws = o_sde.make_noise((2, 1, 64, 128), o_sde.n_noise_draws(6, "reverse_diffusion", "ald", 1), seed=11)
    xh = eng.enhance(wav.cuda(), noise=torch.stack(draws).cuda(), N=6).cpu()
    ref = torch.from_numpy(z["enh"]).reshape(xh.shape)
    e_enh = rel_l2(xh, ref)
    sdr = min(o_pipe.si_sdr(ref[b].numpy(), xh[b].numpy()) for b in range(2))
    report.append(f"enhance chain N=6 {e_enh:.3e} (SI-SDR {sdr:.1f} dB)")
    print(f"mid-size reference fixture, {mode}: " + "; ".join(report))
    assert e_enh < tol["enh"]
    eng.close()


# ------------------------------------------------------------------------------------------------
# fp16 activation range (the product mode stores raw convolution outputs and the residual stream as fp16 BEFORE
# GroupNorm): large-but-representable activations keep parity, an overflow is detected and refused, never silent
# ------------------------------------------------------------------------------------------------
def _scale_resblock_convs(sd, s):
    """Scale the input conv and every ResBlock's Conv_0 / Conv_1 (weights and biases) by s: pre-GroupNorm activations grow
    linearly with s (the tap maximum of this network and input is 4.29 s), the network function barely moves (GroupNorm
    is scale-invariant; only the temb bias and the unscaled 1x1 shortcuts shift weight)."""
    return {k: (v * s if (".Conv_0." in k or ".Conv_1." in k or k.startswith("all_modules.3.")) else v) for k, v in sd.items()}


def test_fp16_activation_range_is_kept_or_reported():
    base = o_w.make_state_dict(MID_N, seed=5)
    g = torch.Generator().manual_seed(3)
    x = torch.complex(torch.randn(2, 2, 64, 128, generator=g), torch.randn(2, 2, 64, 128, generator=g)) * 0.4
    t = torch.tensor([0.9, 0.05])
    # (1) residual stream up to ~2e4 (fp16 ulp 16 there): representable -> finite, no range event, parity holds
    sd = _scale_resblock_convs(base, 4660.0)
    taps = {}
    with torch.no_grad():
        ref = o_net.forward(sd, MID_N, x, t, taps=taps)
    peak = max(v.abs().max().item() for k, v in taps.items() if k != "temb")
    assert 1.5e4 < peak < 3e4
    eng = Engine(EngineConfig(mode="fp16_tc", max_batch=2, **MID_E))
    eng.load_state_dict(sd)
    out = eng.dnn_forward(x.cuda(), t.cuda())
    err = rel_l2(out, ref)
    print(f"fp16 range stress: block outputs up to {peak:.3g}, rel-L2 {err:.3e}, range events {eng.counter('fp16_range_events')}")
    assert torch.isfinite(torch.view_as_real(out)).all() and eng.counter("fp16_range_events") == 0 and err < 4.1e-3   # measured 1.98e-3 (H100)
    # (2) 8x more: block outputs ~1.6e5 > 65504 -> inf in storage; the statistics pass counts it, the host-buffer call refuses
    sd8 = _scale_resblock_convs(base, 8 * 4660.0)
    eng.load_state_dict(sd8)
    out8 = eng.dnn_forward(x.cuda(), t.cuda())
    ev = eng.counter("fp16_range_events")
    assert ev > 0 and not torch.isfinite(torch.view_as_real(out8)).all()
    eng.set_option("reset_range_events", 1)
    assert eng.counter("fp16_range_events") == 0
    wav = 0.1 * torch.randn(1, 4000, generator=g)
    with pytest.raises(RuntimeError, match="fp16 activation range"):
        eng.enhance(wav, N=1, seed=1)                      # host buffers: checked before the call returns
    assert eng.counter("fp16_range_events") == 0           # ... and cleared for the next call
    eng.close()
    # the fp32 validation mode carries the same weights without trouble
    e32 = Engine(EngineConfig(mode="fp32", max_batch=2, **MID_E))
    e32.load_state_dict(sd8)
    with torch.no_grad():
        ref8 = o_net.forward(sd8, MID_N, x, t)
    assert rel_l2(e32.dnn_forward(x.cuda(), t.cuda()), ref8) < 2e-4 and e32.counter("fp16_range_events") == 0
    e32.close()


def test_kernel_options_are_per_engine(full_sd):
    """The A/B switches select code paths per ENGINE (thread-local selection installed at every C-ABI entry): an option set
    on one engine must not leak into another engine of the same process -- neither into its eager launches nor into the
    graphs it captures."""
    a = Engine(EngineConfig(mode="fp16_tc", max_batch=1))
    b = Engine(EngineConfig(mode="fp16_tc", max_batch=1))
    a.load_state_dict(full_sd)
    b.load_state_dict(full_sd)
    g = torch.Generator().manual_seed(14)
    x = (torch.complex(torch.randn(1, 2, 256, 128, generator=g), torch.randn(1, 2, 256, 128, generator=g)) * 0.3).cuda()
    t = torch.tensor([0.4]).cuda()
    ref = b.dnn_forward(x, t)
    n_default = b.counter("launches_last_forward")
    a.set_option("tc_variant", 5)                      # fused convolutions: no separate gn_apply launches on engine a only
    a.set_option("fir_variant", 1)                     # ... and the fp32 FIR resampler (rounds differently: a different output)
    out_a = a.dnn_forward(x, t)
    n_a = a.counter("launches_last_forward")
    out_b = b.dnn_forward(x, t)                        # b runs AFTER a's call on the same thread: still its own defaults
    assert n_a < n_default and b.counter("launches_last_forward") == n_default
    assert torch.equal(out_b, ref) and not torch.equal(out_a, ref) and rel_l2(out_a, ref) < 5e-3
    y = x[:, 1:2].contiguous()
    sa, _ = a.pc_sample(y, N=1, seed=3)                # captured graphs keep the capturing engine's choices
    sb, _ = b.pc_sample(y, N=1, seed=3)
    sb2, _ = b.pc_sample(y, N=1, seed=3)
    assert torch.equal(sb, sb2) and not torch.equal(sa, sb)
    a.close()
    b.close()


@pytest.mark.parametrize("kind,mode", [("ncsnpp", "fp16_tc"), ("ncsnpp", "fp32"), ("ncsnpp_small", "fp16_direct"), ("v2", "fp16_tc")])
def test_device_side_weight_packing_equals_the_host_path(full_sd, kind, mode):
    """sgmse_b200_load_weights_device packs the state_dict blob where it lives (csrc/pack.cu) -- the path of refresh() after an
    EMA swap and of every CUDA blob (bench.py) -- instead of copying 262 MB to the host and back: the packed weights, hence the
    network outputs, must be bit-identical to the host packer's, for the wgmma layouts (K-major + identity tail, q|k|v
    concatenation, mma.sync fragments of the 4-channel ends) as well as the CUDA-core ones."""
    if kind == "ncsnpp":
        cfg, sd, shape = EngineConfig(mode=mode, max_batch=1), full_sd, (1, 2, 256, 128)
    elif kind == "v2":
        pre = dict(loss_type="data_prediction", network_scaling="1/sigma", c_in="edm", c_out="edm", c_skip="edm", sigma_data=0.1)
        cfg, sd, shape = EngineConfig.ncsnpp_v2(mode=mode, max_batch=1, sde="sbve", sb_k=2.6, sb_c=0.4, **pre), full_sd, (1, 2, 256, 128)
    else:
        ncfg = NetConfig.ncsnpp(attn_resolutions=(16,), **SMALL_N)
        cfg, sd, shape = EngineConfig(attn_resolutions=(16,), mode=mode, **SMALL_E), o_w.make_state_dict(ncfg, seed=2), (2, 2, 64, 64)
    g = torch.Generator().manual_seed(5)
    x = (torch.complex(torch.randn(*shape, generator=g), torch.randn(*shape, generator=g)) * 0.3).cuda()
    t = torch.full((shape[0],), 0.37).cuda()
    host, dev = Engine(cfg), Engine(cfg)
    host.load_state_dict(sd)                                   # CPU tensors -> host packer
    dev.load_state_dict({k: v.cuda() for k, v in sd.items()}, on_device=True)   # CUDA blob -> device packer
    fwd = (lambda e: e.model_forward(x[:, :1], x[:, 1:], t)) if kind == "v2" else (lambda e: e.dnn_forward(x, t))
    a, b = fwd(host), fwd(dev)
    assert torch.isfinite(torch.view_as_real(a)).all() and torch.equal(a, b)
    y = x[:, 1:2].contiguous()
    if kind != "v2":
        sa, _ = host.pc_sample(y, N=2, seed=11)
        sb, _ = dev.pc_sample(y, N=2, seed=11)
        assert torch.equal(sa, sb)
        dev.load_state_dict({k: (v * 1.01).cuda() for k, v in sd.items()}, on_device=True)      # a refresh: new weights, new result
        assert not torch.equal(fwd(dev), a)
    host.close()
    dev.close()
