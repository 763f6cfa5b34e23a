"""Where the time of one score-network evaluation goes: per-kernel totals under torch.profiler (needs a GPU).

    python tools/kernel_breakdown.py --out DIR [--batch 16] [--T 512] [--opt key=value]

Builds the engine at the benchmark shape (B = 16, T = 512 by default), runs one eager forward to warm every shape,
then profiles one more eager forward with CUDA activities.  Writes DIR/kernel_breakdown.json and a text table
DIR/kernel_breakdown.txt: for each kernel name (template arguments stripped, so that all instantiations of a kernel
add up) the launch count, the total device time and its share of the summed kernel time, plus the GPU name.
"""
import argparse
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile

from sgmse_b200 import Engine, EngineConfig
from sgmse_b200.synth import synthetic_blob


def base_name(name: str) -> str:
    """conv_tc_kernel<128, 4, false>(...) / void sgmse::(anonymous namespace)::conv_tc_kernel<...>(...) -> conv_tc_kernel"""
    name = re.sub(r"\(.*$", "", name.replace("(anonymous namespace)", ""))
    depth, out = 0, []
    for ch in name:                                 # drop template argument lists, nested ones included
        depth += ch == "<"
        if depth == 0:
            out.append(ch)
        depth -= ch == ">"
    return "".join(out).split("::")[-1].replace("void ", "").strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--T", type=int, default=512)
    ap.add_argument("--mode", default="fp16_tc")
    ap.add_argument("--opt", action="append", default=[], metavar="KEY=VALUE", help="Engine.set_option before the forwards")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("kernel_breakdown.py needs a CUDA device")

    cfg = EngineConfig(mode=a.mode, max_batch=a.batch, use_graphs=False)
    eng = Engine(cfg)
    eng.load_blob(synthetic_blob(eng, 0))
    for kv in a.opt:
        k, v = kv.split("=")
        eng.set_option(k, int(v))
    F = cfg.n_fft // 2 + 1
    g = torch.Generator().manual_seed(0)
    x = (torch.complex(torch.randn(a.batch, 2, F, a.T, generator=g), torch.randn(a.batch, 2, F, a.T, generator=g)) * 0.3).cuda()
    t = torch.full((a.batch,), 0.5).cuda()
    eng.dnn_forward(x, t)                           # warm-up: module load, workspaces, every shape once
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.dnn_forward(x, t)
        torch.cuda.synchronize()

    rows = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA or ev.device_time_total <= 0:
            continue
        if ev.name.startswith(("Memcpy", "Memset", "cudaMemcpy", "cudaMemset")):
            continue
        r = rows.setdefault(base_name(ev.name), {"launches": 0, "us": 0.0})
        r["launches"] += 1
        r["us"] += ev.device_time_total
    total = sum(r["us"] for r in rows.values())
    table = sorted(({"kernel": k, **r, "share": r["us"] / total} for k, r in rows.items()), key=lambda r: -r["us"])
    for r in table:
        r["us"] = round(r["us"], 1)
        r["share"] = round(r["share"], 4)
    res = {"gpu": torch.cuda.get_device_name(0), "batch": a.batch, "T": a.T, "mode": a.mode, "opts": a.opt,
           "total_kernel_us": round(total, 1), "kernels": table}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "kernel_breakdown.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    lines = [f"{res['gpu']}  B={a.batch} T={a.T} {a.mode}  summed kernel time {total / 1e3:.2f} ms", "",
             f"{'kernel':<40} {'launches':>8} {'ms':>9} {'share':>7}"]
    lines += [f"{r['kernel']:<40} {r['launches']:>8} {r['us'] / 1e3:>9.3f} {100 * r['share']:>6.1f}%" for r in table]
    with open(os.path.join(a.out, "kernel_breakdown.txt"), "w") as fh:
        fh.write("\n".join(lines) + "\n")
    print("\n".join(lines))
    eng.close()


if __name__ == "__main__":
    main()
