"""GPU tests of long recordings: the streaming fp32 attention kernel, full-size forwards past the token count the
full-row attention kernel holds, clips the workspace only fits with buffer reuse, and the workspace plan checked by
poisoning every buffer after its last reader (option "workspace_poison": a read past a buffer's planned lifetime turns
into NaN).  Host-side checks of the plan are in tests/test_workspace_plan_host.py."""
import ctypes as C
import math
import os
import subprocess

import pytest
import torch

from oracle import ncsnpp as o_net, weights as o_w
from oracle.arch import NetConfig
from sgmse_b200 import Engine, EngineConfig, build as B
from test_gpu_kernel_ops import ULP32, Guarded, attention_reference, ratio

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel_l2(a, b):
    a, b = torch.as_tensor(a).cpu().reshape(-1), torch.as_tensor(b).cpu().reshape(-1)
    return (torch.linalg.vector_norm(a - b) / torch.linalg.vector_norm(b)).item()


@pytest.fixture(scope="module")
def aops(tmp_path_factory):
    B.build()
    out = str(tmp_path_factory.mktemp("attention_ops"))
    objs = [os.path.join(B.LIBDIR, "obj", s.replace(".cu", ".o")) for s in B.SOURCES]
    shim_o, so = os.path.join(out, "attention_ops.o"), os.path.join(out, "libattention_ops.so")
    for cmd in ([B.NVCC, *B.ARCH, *B.CFLAGS, *B.PRODUCT_DEFS, "-I", B.CSRC, "-c",
                 os.path.join(ROOT, "tests", "c", "attention_ops.cu"), "-o", shim_o],
                [B.NVCC, *B.ARCH, "-shared", "-cudart", "static", "-o", so, shim_o, *objs, "-L" + B.CUDA_LIB, "-lcufft",
                 "-Xlinker", "-Bsymbolic", "-Xlinker", "-rpath," + B.CUDA_LIB]):
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
    lib = C.CDLL(so, mode=os.RTLD_LOCAL)
    lib.aops_attention.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.aops_last_error.restype = C.c_char_p

    def run(qkv, out):
        N, S, C3 = qkv.shape
        code = lib.aops_attention(torch.cuda.current_stream().cuda_stream, N, S, C3 // 3, int(qkv.dtype == torch.float32),
                                  qkv.data_ptr(), out.data_ptr())
        assert code == 0, lib.aops_last_error().decode()
    return run


def attention_reference_fp32(qkv, keys=None):
    """float64 attention and the elementwise bound of the streaming fp32 kernel.  Scores: fp32 FMA sums of C products
    (C ulps of sum |q_c k_c|) scaled by the fp32 constant log2(e) / sqrt(C) (two roundings); a score error ds moves a
    softmax weight by a factor within exp(+-2 ds).  exp2f: 2 ulps per weight.  P V and the normaliser l are fp32 sums
    over S keys, rescaled once per key tile; the final 1 / l and product two roundings more.  No storage rounding."""
    N, S, C3 = qkv.shape
    Cc = C3 // 3
    q, k, v = (t.double() for t in qkv.split(Cc, -1))
    if keys is not None:
        k, v = k[:, :keys], v[:, :keys]
    s = q @ k.transpose(1, 2) / math.sqrt(Cc)
    w = torch.softmax(s, -1)
    ref = w @ v
    ds = (Cc * ULP32 * (q.abs() @ k.abs().transpose(1, 2)) / math.sqrt(Cc) + 2 * ULP32 * s.abs()).amax(-1, keepdim=True)
    S_eff = s.shape[-1]
    rel = 2 * ds + (2 * ds) ** 2 + 2 * ULP32 + (S_eff + 2 * math.ceil(S_eff / 64) + 4) * ULP32
    return ref, (w @ v.abs()) * rel + 1e-30


@pytest.mark.parametrize("S", [4800, 4801, 9600])
@pytest.mark.parametrize("Cc", [128, 256])
def test_long_attention_against_fp64(aops, S, Cc):
    """fp32 storage past the full-row kernel's shared memory (streaming kernel) and the fp16 flash kernel at the same S."""
    g = torch.Generator(device="cuda").manual_seed(S * 1000 + Cc)
    qkv = 1.5 * torch.randn(1, S, 3 * Cc, generator=g, device="cuda")
    report = []
    for dt, ref_fn in ((torch.float32, attention_reference_fp32), (torch.float16, attention_reference)):
        x = qkv.to(dt)
        out = Guarded((1, S, Cc), dt)
        aops(x, out.t)
        again = torch.empty_like(out.t)
        aops(x, again)
        torch.cuda.synchronize()
        out.check(f"attention {dt}")
        assert torch.equal(out.t, again), "relaunch differs"
        ref, bound = ref_fn(x)
        r = ratio(out.t, ref, bound).max().item()
        # mutation control: the last key tile dropped
        m = ratio(out.t, ref_fn(x, keys=(S - 1) // 64 * 64)[0], bound).max().item()
        report.append(f"{dt}: err/bound {r:.3g}, last key tile dropped {m:.3g}")
        del ref, bound
        assert r <= 1 and m >= 10, report
    print(f"[long attention] S {S} C {Cc}: " + "; ".join(report))


@pytest.fixture(scope="module")
def full_sd():
    return o_w.make_state_dict(NetConfig.ncsnpp(), seed=0)


def spec(B_, F, T, seed, scale=0.3):
    g = torch.Generator().manual_seed(seed)
    return torch.complex(torch.randn(B_, 2, F, T, generator=g), torch.randn(B_, 2, F, T, generator=g)) * scale


def forward_poisoned_and_not(eng, x, t):
    eng.set_option("workspace_poison", 0)
    a = eng.dnn_forward(x, t).clone()
    eng.set_option("workspace_poison", 1)
    b = eng.dnn_forward(x, t).clone()
    eng.set_option("workspace_poison", 0)
    assert torch.equal(torch.view_as_real(a), torch.view_as_real(b)), "workspace_poison changed the result"
    return a


# tf32_tc at T = 512 measures 1.70e-3 against the oracle (tests/test_gpu_tf32.py); the bounds allow about 2x that
def test_full_size_forward_past_the_full_row_attention(full_sd):
    """T = 4800 (38.4 s): S = 4800 tokens at the attention level, past what the full-row fp32 kernel holds."""
    x, t = spec(1, 256, 4800, 21), torch.tensor([0.4])
    with torch.no_grad():
        ref = o_net.forward(full_sd, NetConfig.ncsnpp(), x, t)
    report = []
    for mode, tol in (("tf32_tc", 4.0e-3), ("fp32", 1.0e-3)):
        eng = Engine(EngineConfig(mode=mode, max_batch=1))
        eng.load_state_dict(full_sd)
        out = forward_poisoned_and_not(eng, x.cuda(), t.cuda())
        err = rel_l2(out, ref)
        report.append(f"{mode} rel-L2 {err:.3e} (workspace {eng.counter('workspace_bytes') / 1e9:.2f} GB)")
        eng.close()
        assert err < tol, report
    print("full-size ncsnpp forward T=4800: " + "; ".join(report))


def test_48k_tf32_forward_at_5120_frames():
    """41 s at 48 kHz in tf32_tc against fp32 mode on the GPU (without buffer reuse this needs over 80 GB)."""
    ncfg = NetConfig.ncsnpp_48k()
    sd = o_w.make_state_dict(ncfg, seed=2)
    x, t = spec(1, 768, 5120, 5), torch.tensor([0.6])
    outs = {}
    for mode in ("fp32", "tf32_tc"):
        eng = Engine(EngineConfig.ncsnpp_48k(mode=mode, max_batch=1))
        eng.load_state_dict(sd)
        outs[mode] = forward_poisoned_and_not(eng, x.cuda(), t.cuda()).cpu()
        eng.close()
    err = rel_l2(outs["tf32_tc"], outs["fp32"])
    print(f"ncsnpp_48k T=5120: tf32_tc vs fp32 rel-L2 {err:.3e}")
    assert torch.isfinite(torch.view_as_real(outs["tf32_tc"])).all() and err < 4.0e-3


def test_16k_fp16_clip_of_240_s(full_sd):
    """240 s at 16 kHz (T = 30016): one fp16_tc forward against fp32 mode, then an N = 30 enhancement."""
    L = 240 * 16000
    probe = Engine(EngineConfig(mode="fp16_tc", max_batch=1))
    T = probe.padded_frames(L)
    assert T == 30016
    probe.close()
    x, t = spec(1, 256, T, 8), torch.tensor([0.3])
    outs = {}
    for mode in ("fp32", "fp16_tc"):
        eng = Engine(EngineConfig(mode=mode, max_batch=1))
        eng.load_state_dict(full_sd)
        outs[mode] = forward_poisoned_and_not(eng, x.cuda(), t.cuda()).cpu()
        if mode == "fp16_tc":
            g = torch.Generator().manual_seed(4)
            wav = (0.1 * torch.randn(1, L, generator=g)).cuda()
            enh = eng.enhance(wav, N=30, seed=1)
            torch.cuda.synchronize()
            assert enh.shape == wav.shape and torch.isfinite(enh).all() and enh.abs().max() > 0
        eng.close()
    err = rel_l2(outs["fp16_tc"], outs["fp32"])
    print(f"ncsnpp 240 s: fp16_tc vs fp32 rel-L2 {err:.3e}")
    assert err < 6.0e-3


@pytest.mark.parametrize("mode", ["fp16_tc", "tf32_tc", "fp32"])
def test_poison_leaves_every_path_bit_identical(full_sd, mode):
    """T = 512: eager forward, PC sampler (capture, then replay), two lanes, and the ODE sampler, each with every buffer
    poisoned after its last reader, against the same runs without poisoning."""
    eng = Engine(EngineConfig(mode=mode, max_batch=4))
    eng.load_state_dict(full_sd)
    x, t = spec(2, 256, 512, 31).cuda(), torch.tensor([0.7, 0.2]).cuda()
    y = spec(2, 256, 512, 32)[:, :1].contiguous().cuda()

    def runs():
        r = {"forward": eng.dnn_forward(x, t).clone()}
        eng.set_option("lanes", 1)
        r["pc"] = eng.pc_sample(y, N=3, seed=5)[0].clone()
        r["pc replay"] = eng.pc_sample(y, N=3, seed=5)[0].clone()
        eng.set_option("lanes", 2)
        r["pc lanes=2"] = eng.pc_sample(y, N=3, seed=5)[0].clone()
        r["pc lanes=2 replay"] = eng.pc_sample(y, N=3, seed=5)[0].clone()
        eng.set_option("lanes", 1)
        r["ode"] = eng.ode_sample(y[:1], rtol=1e-2, atol=1e-2, denoise=False)[0].clone()
        torch.cuda.synchronize()
        return r

    plain = runs()
    eng.set_option("workspace_poison", 1)
    poisoned = runs()
    eng.set_option("workspace_poison", 0)
    eng.close()
    for k in plain:
        assert torch.isfinite(torch.view_as_real(plain[k])).all(), k
        assert torch.equal(torch.view_as_real(plain[k]), torch.view_as_real(poisoned[k])), f"{mode} {k}: poisoning changed it"
    assert torch.equal(torch.view_as_real(plain["pc"]), torch.view_as_real(plain["pc replay"]))
    print(f"workspace_poison {mode}: {', '.join(plain)} bit-identical")
