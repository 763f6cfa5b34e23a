"""Per-kernel SASS comparison of two builds of sgmse_b200/csrc (no GPU needed: nvcc + cuobjdump).

    python tools/sass_diff.py <git-rev>            # <git-rev> (e.g. the last GPU-verified commit) against the working tree

Builds the .cu files of <git-rev> into a scratch directory with the flags of sgmse_b200/build.py, dumps the SASS of
every kernel of both builds, demangles and normalises the names (anonymous-namespace hashes; template parameters that
were renamed are listed as missing/new) and reports which kernels have an identical instruction stream: a refactor that leaves the default kernels
instruction-for-instruction unchanged needs no new GPU verification.
"""
import difflib
import glob
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sgmse_b200 import build as B  # noqa: E402


def kernels(obj):
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
    res, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            res[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;\s*/\*", line)
        if m and cur:
            res[cur].append(m.group(1))
    return res


def norm(name):
    d = subprocess.run(["cu++filt", name], capture_output=True, text=True).stdout.strip()
    return re.sub(r"_GLOBAL__N__[0-9a-f_a-z]+", "ANON", d)


def build_rev(rev, tmp):
    subprocess.run(f"git -C {ROOT} archive {rev} sgmse_b200/csrc include | tar -x -C {tmp}", shell=True, check=True)
    src = os.path.join(tmp, "sgmse_b200", "csrc")
    procs = [subprocess.Popen([B.NVCC, *B.ARCH, *B.CFLAGS, "-c", f, "-o", f + ".o"], cwd=src) for f in sorted(glob.glob(os.path.join(src, "*.cu")))]
    assert all(p.wait() == 0 for p in procs), "nvcc failed on the old revision"
    return glob.glob(os.path.join(src, "*.o"))


def main():
    rev = sys.argv[1]
    B.build()
    with tempfile.TemporaryDirectory() as tmp:
        old, new = {}, {}
        for o in build_rev(rev, tmp):
            old.update({norm(k): v for k, v in kernels(o).items()})
        for o in glob.glob(os.path.join(B.LIBDIR, "obj", "*.o")):
            new.update({norm(k): v for k, v in kernels(o).items()})
    same = [k for k in old if new.get(k) == old[k]]
    changed = [k for k in old if k in new and new[k] != old[k]]
    print(f"{len(same)} kernels identical, {len(changed)} changed, {len(set(old) - set(new))} only in {rev}, {len(set(new) - set(old))} only in the working tree")
    for k in changed:
        d = [l for l in difflib.unified_diff(old[k], new[k], lineterm="", n=0) if not l.startswith(("---", "+++", "@@"))]
        ops = lambda ls: sorted(l.split()[0 if not l.startswith("@") else 1] for l in ls)   # noqa: E731
        kind = "register allocation / scheduling only" if ops(old[k]) == ops(new[k]) else "DIFFERENT INSTRUCTION MIX"
        print(f"  changed ({kind}, {len(d)} lines): {k[:140]}")
    new_only = sorted(set(new) - set(old))
    for k in sorted(set(old) - set(new)):
        base = lambda x: x.split("(")[0].split("<")[0].split()[-1]   # noqa: E731  (drop return type, template and argument lists)
        twins = [n for n in new_only if new[n] == old[k] and base(n) == base(k)]
        if twins:
            print(f"  renamed, identical instruction stream: {k[:110]}  ->  {twins[0][:110]}")
            new_only = [n for n in new_only if n != twins[0]]
        else:
            print(f"  ONLY IN {rev} (no identical twin): {k[:160]}")
    for k in new_only:
        print(f"  new kernel: {k[:160]}")


if __name__ == "__main__":
    main()
