"""profiles/r02_conv_traffic.json (read by bench.py) from an ncu metrics pass of the CURRENT build:

    ncu --clock-control none -k regex:conv_tc_kernel -s 54 -c 1 --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum \\
        --csv --log-file /tmp/conv_traffic.csv python tools/profile_forward.py --batch 16 --evals 2
    python tools/make_conv_traffic.py /tmp/conv_traffic.csv > profiles/r02_conv_traffic.json

-s N skips the first forward's N conv_tc launches (cold, N = tc_convs_last_forward of the profiled forward), so the captured
launch is the first conv_tc launch of the second forward.  The file records a digest of the kernel's sources; bench.py reports
`roofline.traffic` only while that digest matches the sources it is run with (a stale capture is reported as null)."""
import csv
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL_SOURCES = ["sgmse_b200/csrc/conv_tc.cu", "sgmse_b200/csrc/common.cuh"]    # the kernel and its device helpers (kernels.h holds declarations only)


def source_digest():
    h = hashlib.sha256()
    for f in KERNEL_SOURCES:
        h.update(open(os.path.join(ROOT, f), "rb").read())
    return h.hexdigest()[:16]


def main(path):
    rows = [r for r in csv.reader(l for l in open(path) if l.startswith('"'))]
    hdr, rows = rows[0], rows[1:]
    first = rows[0][hdr.index("ID")]
    m = {r[hdr.index("Metric Name")]: float(r[hdr.index("Metric Value")].replace(",", "")) for r in rows if r[hdr.index("ID")] == first}
    name = rows[0][hdr.index("Kernel Name")]
    rd, wr = m["dram__bytes_read.sum"], m["dram__bytes_write.sum"]
    B, H, W, C = 16, 256, 512, 128
    alg = B * H * W * C * 2 * 2                                   # fp16 input once + fp16 output once
    print(json.dumps({
        "kernel": name[:80], "shape": "3x3 conv 128->128 at [16,256,512] (ResBlock m4 Conv_0), one launch",
        "dram_bytes_read": int(rd), "dram_bytes_write": int(wr), "traffic_bytes_per_launch": int(rd + wr),
        "algorithmic_bytes_per_launch": alg, "ratio": round((rd + wr) / alg, 4),
        "launch_us_under_ncu": round(m.get("gpu__time_duration.sum", 0) / 1e3, 1),
        "source": "ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum (tools/make_conv_traffic.py), same build as the bench",
        "source_digest": source_digest(), "digest_of": KERNEL_SOURCES}, indent=1))


if __name__ == "__main__":
    main(sys.argv[1])
