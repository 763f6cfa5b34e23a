"""The spectrogram transforms 'log' / 'none' (SpecsDataModule --transform_type, data_module.py:118,162-188) and the
--no-centered backbones (ncsnpp.py:45-47,288-290; ncsnpp_48k.py:46-47,291-293) on the device, against
tests/golden/transforms_small.npz (outputs of the unmodified reference, oracle/transforms.py: golden_transforms; weights,
clips and noise regenerated from seeds).  Run on a GPU host: ``pytest -m gpu``.

Tolerances are rel-L2 bounds about 2x the error measured on an H100 (values in the comments)."""
import os

import numpy as np
import pytest
import torch

from oracle import refshim, sde as o_sde, spec as o_spec, transforms as o_tr, weights as o_w
from oracle.transforms import TRANSFORM_CASES, TRANSFORMS_NET, transforms_net_config
from sgmse_b200 import Engine, EngineConfig

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
B, L, N = 2, 2000, 3


def rel_l2(a, b):
    a, b = torch.as_tensor(a).detach().cpu(), torch.as_tensor(b).detach().cpu()
    if a.is_complex():
        a, b = torch.view_as_real(a), torch.view_as_real(b)
    a, b = a.double(), b.double()
    return (torch.linalg.vector_norm((a - b).reshape(-1)) / torch.linalg.vector_norm(b.reshape(-1))).item()


@pytest.fixture(scope="module")
def z():
    return np.load(os.path.join(GOLDEN, "transforms_small.npz"))


def _wav(z):
    return 0.1 * torch.randn(B, L, generator=torch.Generator().manual_seed(int(z["wav_seed"])))


def _engine(tag, mode, **kw):
    backbone, transform_type, spec_factor, centered, seed = TRANSFORM_CASES[tag]
    common = dict(n_fft=126, hop_length=32, transform_type=transform_type, spec_factor=spec_factor, centered=centered,
                  mode=mode, **TRANSFORMS_NET)
    common.update(kw)
    if backbone == "ncsnpp":
        eng = Engine(EngineConfig(attn_resolutions=(16,), **common))
    else:   # the OUVE parameters and the exponent the reference model of the fixture was built with
        eng = Engine(EngineConfig.ncsnpp_48k(theta=1.5, sigma_min=0.05, sigma_max=0.5, spec_abs_exponent=0.5, **common))
    eng.load_state_dict(o_w.make_state_dict(transforms_net_config(backbone), seed=seed))
    return eng


def _draws(F, T, seed):
    return torch.stack(o_sde.make_noise((B, 1, F, T), o_sde.n_noise_draws(N, "reverse_diffusion", "ald", 1), seed=seed)).cuda()


@pytest.mark.parametrize("tag", ["log", "none"])
def test_analysis_and_synthesis(z, tag):
    eng = _engine(tag, "fp32")
    wav = _wav(z)
    Y, norm = eng.analysis(wav.cuda())
    e_y = rel_l2(Y, z[f"{tag}/Y"])
    assert torch.allclose(norm.cpu(), wav.abs().amax(dim=1))
    scfg = o_spec.SpecConfig(n_fft=126, hop_length=32, spec_factor=TRANSFORM_CASES[tag][2])
    Yz = torch.from_numpy(z[f"{tag}/Y"])
    # synthesis of the reference's padded spectrogram == inverse transform + iSTFT of the oracle (pinned to the reference)
    back = eng.synthesis(Yz.cuda(), norm, L)
    e_s = rel_l2(back, o_tr.synthesis(Yz, norm.cpu(), scfg, tag, L))
    # round trip: away from the padded tail the chain is the identity
    rt = eng.synthesis(Y, norm, L)
    e_rt = rel_l2(rt[:, :1900], wav[:, :1900])
    print(f"transform {tag}: analysis rel-L2 {e_y:.3e}, synthesis {e_s:.3e}, round trip {e_rt:.3e}")
    assert e_y < 4e-7 and e_s < 3.2e-7 and e_rt < 3e-7       # measured <= 2.0e-7 / 1.6e-7 / 1.4e-7
    eng.close()


# measured on an H100, max over the four cases (and the three input-conv forms): fp32 forward 2.3e-6, sampler 9.5e-7,
# waveform 1.2e-6; fp16_tc 2.0e-3 / 9.3e-4 / 1.1e-3.  The 'log' waveform goes through exp(|X|), which turns the sample's
# error into a relative error |X| (up to 10) times larger: measured 4.5e-6 (fp32) and 4.2e-3 (fp16_tc).
TOL = {"fp32": dict(fwd=4.6e-6, pc=1.9e-6, enh=2.5e-6, enh_log=9e-6),
       "fp16_tc": dict(fwd=4.1e-3, pc=1.9e-3, enh=2.2e-3, enh_log=8.4e-3)}


@pytest.mark.parametrize("tag", list(TRANSFORM_CASES))
@pytest.mark.parametrize("mode", ["fp32", "fp16_tc"])
def test_forward_sampler_and_enhance_chain(z, tag, mode):
    eng = _engine(tag, mode)
    seed = TRANSFORM_CASES[tag][4]
    Y = torch.from_numpy(z[f"{tag}/Y"])
    F, T = Y.shape[-2:]
    gx = torch.Generator().manual_seed(seed + 100)
    x = Y + 0.2 * torch.complex(torch.randn(B, 1, F, T, generator=gx), torch.randn(B, 1, F, T, generator=gx))
    t = torch.tensor([0.83, 0.11])
    e_f = rel_l2(eng.score(x.cuda(), Y.cuda(), t.cuda()), z[f"{tag}/score"])
    e_v = []
    if mode == "fp16_tc":
        assert eng.counter("tc_convs_last_forward") > 0
        # the other two forms of the input convolution: the CUDA-core kernel (1) and the unprefetched mma.sync kernel (3)
        for v in (1, 3):
            eng.set_option("inconv_variant", v)
            e_v.append(rel_l2(eng.score(x.cuda(), Y.cuda(), t.cuda()), z[f"{tag}/score"]))
        eng.set_option("inconv_variant", 0)
    smp, nfe = eng.pc_sample(Y.cuda(), noise=_draws(F, T, 7), N=N, predictor="reverse_diffusion", corrector="ald",
                             corrector_steps=1, snr=0.5)
    assert nfe == 2 * N
    e_pc = rel_l2(smp, z[f"{tag}/pc"])
    xh = eng.enhance(_wav(z).cuda(), noise=_draws(F, T, 11), N=N)
    e_w = rel_l2(xh, z[f"{tag}/enh"])
    print(f"transforms {tag} {mode}: forward rel-L2 {e_f:.3e} (inconv variants {e_v}), sampler {e_pc:.3e}, waveform {e_w:.3e}")
    tol = TOL[mode]
    assert max([e_f] + e_v) < tol["fwd"] and e_pc < tol["pc"] and e_w < tol["enh_log" if tag == "log" else "enh"]
    eng.close()


@pytest.mark.skipif(not refshim.reference_available(), reason="reference not staged (oracle/_ref) and no live checkout")
@pytest.mark.parametrize("tag", list(TRANSFORM_CASES))
def test_install_on_a_live_reference_score_model(z, tag):
    """As tests/test_gpu_dropin.py for the defaults: install() reads the option off the model, and the model's own public
    calls then match the same model before installation."""
    import sgmse_b200
    backbone, transform_type, spec_factor, centered, seed = TRANSFORM_CASES[tag]
    cfg = transforms_net_config(backbone)
    model = refshim.make_score_model(backbone, seed=0, n_fft=126, hop_length=32, transform_type=transform_type,
                                     spec_factor=spec_factor, centered=centered, attn_resolutions=cfg.attn_resolutions,
                                     **TRANSFORMS_NET)
    from sgmse.util.other import pad_spec                  # importable once refshim has imported the reference
    model.dnn.load_state_dict(o_w.make_state_dict(cfg, seed=seed))
    wav = _wav(z)[:1]
    norm = wav.abs().max()
    Y = pad_spec(torch.unsqueeze(model._forward_transform(model._stft(wav / norm)), 0))
    draws = o_sde.make_noise(tuple(Y.shape), o_sde.n_noise_draws(N, "reverse_diffusion", "ald", 1), seed=17)
    with refshim.injected_noise(list(draws)):
        ref_sample, _ = model.get_pc_sampler("reverse_diffusion", "ald", Y, N=N, corrector_steps=1, snr=0.5)()
    ref_wav = (model.to_audio(ref_sample.squeeze(), L) * norm).squeeze().numpy()
    x_t, t = Y + 0.3 * draws[0], torch.tensor([0.6])
    with torch.no_grad():
        ref_score = model(x_t, Y, t)
    eng = sgmse_b200.install(model, mode="fp32", max_batch=2)
    try:
        assert (eng.cfg.transform_type, eng.cfg.centered) == (transform_type, centered)
        noise = torch.stack(draws).cuda()
        sample, _ = model.get_pc_sampler("reverse_diffusion", "ald", Y.cuda(), N=N, corrector_steps=1, snr=0.5, noise=noise)()
        x_hat = model.enhance(wav, N=N, noise=noise)
        with torch.no_grad():
            e_f = rel_l2(model(x_t.cuda(), Y.cuda(), t.cuda()), ref_score)
        e_s, e_w = rel_l2(sample, ref_sample), rel_l2(x_hat, ref_wav)
        print(f"drop-in {tag}: forward rel-L2 {e_f:.3e}, sampler {e_s:.3e}, waveform {e_w:.3e}")
        # measured <= 2.5e-6 / 1.1e-6 / 1.4e-6, 'log' waveform 5.4e-6
        assert e_f < 5e-6 and e_s < 2.3e-6 and e_w < (1.1e-5 if tag == "log" else 2.8e-6)
    finally:
        sgmse_b200.uninstall(model)
        eng.close()


@pytest.mark.parametrize("tag,mode", [("nc", "fp16_tc"), ("nc48k", "fp32")])
def test_not_centered_graphs_lanes_and_ode_groups(z, tag, mode):
    """Every path that runs the forward applies the mapping: captured sampler graphs and lanes equal the eager launch
    sequence, the ODE forward graphs equal eager, and ode_sample_groups (row-batched forward) equals each solo solve."""
    eng = _engine(tag, mode, max_batch=2, use_graphs=True)
    g = torch.Generator().manual_seed(4)
    Y = (0.3 * torch.complex(torch.randn(3, 1, 64, 64, generator=g), torch.randn(3, 1, 64, 64, generator=g))).cuda()
    a, _ = eng.pc_sample(Y, N=2, seed=11)
    b, _ = eng.pc_sample(Y, N=2, seed=11)                  # graph replay
    eng.set_option("lanes", 2)
    c, _ = eng.pc_sample(Y, N=2, seed=11)
    eng.set_option("lanes", 1)
    assert eng.counter("graph_launches") >= 2
    kw = dict(rtol=1e-2, atol=1e-2, denoise=False, seed=5)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                         # the ODE forward graphs are captured on a non-default stream
        g0 = eng.counter("graph_launches")
        o_graph = [eng.ode_sample(Y[i:i + 1], utt_offset=i, return_stats=True, **kw) for i in range(3)]
        assert eng.counter("graph_launches") > g0
        grouped, nfes, _ = eng.ode_sample_groups(Y, group=1, return_stats=True, **kw)
        eng.set_option("use_graphs", 0)
        d, _ = eng.pc_sample(Y, N=2, seed=11)              # eager
        o_eager = [eng.ode_sample(Y[i:i + 1], utt_offset=i, return_stats=True, **kw) for i in range(3)]
    side.synchronize()
    assert torch.isfinite(torch.view_as_real(a)).all()
    assert torch.equal(a, b) and torch.equal(a, c) and torch.equal(a, d)
    for i in range(3):
        assert torch.equal(o_graph[i][0], o_eager[i][0]) and o_graph[i][1] == o_eager[i][1]
        assert torch.equal(grouped[i:i + 1], o_graph[i][0]) and nfes[i] == o_graph[i][1], f"system {i}"
    eng.close()
    # the option is live: a centered engine on the same weights gives another sample
    cen = _engine(tag, mode, max_batch=2, centered=True)
    assert rel_l2(cen.pc_sample(Y, N=2, seed=11)[0], a) > 1e-2
    cen.close()
