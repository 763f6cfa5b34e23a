"""CPU checks of the wgmma convolution's two operand rings and dy-halo strips (sgmse_b200/csrc/conv_tc.cu, conv_tc_sched.h).

tests/c/conv_tc_strips.cu includes conv_tc.cu and replays the kernel's producer and consumer loops: the A fills (slot,
box coordinates, rows), the B fills (slot, packed weight column) and, per k-block a consumer reads, both slots, the A
fill and the strip row offset.  Here that replay is checked for coverage of the packed K columns and for tap-shifted A
rows, drives a numpy emulation of the kernel's GEMM in its own K order against F.conv2d, and drives a model of both
rings' mbarriers under several interleavings.  The strip rule is compared with the Python rule the GPU tests use, and
ptxas must report no spills for any conv_tc_kernel instantiation."""
import collections
import os
import random
import re
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from sgmse_b200 import build as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMEM_LIMIT = 227 * 1024
STRIP_MAX_ROWS = 160


def strip_rows(bw, bh, bn, taps):
    """tc_strip_rows: rows of segment 0's bw x (bh + 2) strips, 0 where the segment takes one box per k-block."""
    rows = (bh + 2) * bw
    return rows if taps == 9 and bn == 1 and bw % 8 == 0 and rows <= STRIP_MAX_ROWS else 0


Fill = collections.namedtuple("Fill", "stage phase seg chunk dx y rows")
Use = collections.namedtuple("Use", "j kb bstage bphase astage aphase fill dy1 last")


@pytest.fixture(scope="module")
def replay(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("conv_tc_strips") / "replay")
    r = subprocess.run([B.NVCC, *B.ARCH, "-std=c++17", "--expt-relaxed-constexpr", "-diag-suppress", "177", "-I", B.CSRC,
                        os.path.join(ROOT, "tests", "c", "conv_tc_strips.cu"), "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

    def run(lines):
        return subprocess.run([exe], input="".join(l + "\n" for l in lines), capture_output=True, text=True,
                              check=True).stdout.splitlines()
    return run


def run_cases(replay, cases, depths=(0, 0)):
    """cases: (num_tiles, grid, (bw, bh, bn), fused, block_n, esize, segs [(chunks, taps)]) -> per case, per CTA:
    {"P": producer events in order, "A": {(j, f): Fill}, "B": {(j, kb): (stage, phase, col)}, "C": {wg: [Use]}}"""
    lines = []
    for t, g, (bw, bh, bn), fused, block_n, esize, segs in cases:
        s = list(segs) + [(0, 0)] * (3 - len(segs))
        lines.append(f"P {t} {g} {bw} {bh} {bn} {int(fused)} {block_n} {esize} {len(segs)} "
                     + " ".join(f"{taps} {ch}" for ch, taps in s) + f" {depths[0]} {depths[1]}")
    results, ctas = [], []
    for line in replay(lines):
        f = line.split()
        if f[0] == "L":
            continue
        if f[0] == "E":
            results.append(ctas)
            ctas = []
        elif f[0] == "B":
            ctas.append({"P": [], "A": {}, "B": {}, "C": {0: [], 1: []}})
        elif f[0] == "PA":
            j, fi, st, ph, seg, ch, dx, y, rows = map(int, f[1:])
            ctas[-1]["A"][(j, fi)] = Fill(st, ph, seg, ch, dx, y, rows)
            ctas[-1]["P"].append(("A", j, fi, st, ph))
        elif f[0] == "PB":
            j, kb, st, ph, col = map(int, f[1:])
            ctas[-1]["B"][(j, kb)] = (st, ph, col)
            ctas[-1]["P"].append(("B", j, kb, st, ph))
        elif f[0] == "C":
            ctas[-1]["C"][int(f[1])].append(Use(*map(int, f[2:])))
    assert len(results) == len(cases)
    return results


def decode(col, segs):
    """packed k-block col -> (segment, tap, chunk); K is ordered (segment, tap, chunk)"""
    for s, (ch, taps) in enumerate(segs):
        if col < ch * taps:
            return s, col // ch, col % ch
        col -= ch * taps
    raise AssertionError("column past K")


# (num_tiles, grid, box, fused, block_n, esize, segs)
BOX_8x16, BOX_16x8, BOX_4x16x2, BOX_8x4x4 = (8, 16, 1), (16, 8, 1), (4, 16, 2), (8, 4, 4)
CASES = [
    (7, 3, BOX_8x16, False, 128, 2, [(2, 9)]),
    (5, 2, BOX_16x8, False, 64, 2, [(4, 9)]),
    (9, 4, BOX_8x16, False, 64, 2, [(1, 9), (2, 1), (1, 1)]),
    (4, 1, BOX_8x16, False, 128, 2, [(6, 9), (4, 1)]),
    (6, 6, BOX_8x16, False, 64, 4, [(4, 9)]),                 # TF32: 32-channel chunks
    (3, 2, BOX_16x8, False, 64, 4, [(3, 9), (2, 1)]),
    (5, 2, BOX_4x16x2, False, 64, 2, [(4, 9), (4, 1)]),       # per-tap boxes
    (3, 1, BOX_8x4x4, False, 128, 2, [(4, 9)]),
    (6, 2, BOX_8x16, True, 128, 2, [(4, 9)]),                 # the fused producer keeps per-tap tiles
    (8, 3, BOX_8x16, False, 128, 2, [(1, 1)]),                # k_blocks = 1
]


def test_layouts_fit_shared_memory(replay):
    layouts = [tuple(map(int, l.split()[1:])) for l in replay([]) if l.startswith("L")]
    assert [(bn, st, es) for bn, st, es, _, _ in layouts] == [(128, 4, 2), (64, 7, 2), (64, 6, 4)]
    for bn, st, es, a_stages, dyn in layouts:
        print(f"conv_tc<{bn}, {st}, esize {es}>: A ring {a_stages} x 20 KB, {dyn} B dynamic shared memory")
        assert a_stages >= 2 and dyn <= SMEM_LIMIT


def test_strip_rule_matches_python_for_product_levels(replay):
    from test_gpu_kernel_ops import KernelOps, build_shim
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        ops = KernelOps(build_shim(d))
        shapes = set()
        for h0 in (256, 768):                                  # config 2 (16 kHz) and config 3 (48 kHz) frequency rows
            for T in (64, 128, 192, 512):
                for lvl in range(7):
                    if h0 >> lvl and T >> lvl and (T >> lvl) << lvl == T:
                        shapes.add((h0 >> lvl, T >> lvl))
        boxes = []
        for H, W in sorted(shapes):
            p = ops.plan(2, H, W, 128)
            if p.bw:
                boxes.append((H, W, p.bw, p.bh, p.bn))
    lines = [f"S {bw} {bh} {bn} {taps}" for _, _, bw, bh, bn in boxes for taps in (9, 1)]
    got = [int(l.split()[1]) for l in replay(lines) if l.startswith("R")]
    want = [strip_rows(bw, bh, bn, taps) for _, _, bw, bh, bn in boxes for taps in (9, 1)]
    assert got == want
    strips = {(H, W): r for (H, W, *_), r in zip(boxes, got[::2])}
    assert strips[(256, 512)] == 144 and strips[(8, 16)] == 160 and strips[(4, 8)] == 0


def test_replay_reads_each_column_once_from_tap_shifted_rows(replay):
    for case, ctas in zip(CASES, run_cases(replay, CASES)):
        _, _, (bw, bh, bn), fused, _, _, segs = case
        k_blocks = sum(ch * taps for ch, taps in segs)
        sc = 0 if fused else (segs[0][0] if strip_rows(bw, bh, bn, segs[0][1]) else 0)
        for cta in ctas:
            for wg in (0, 1):
                by_tile = collections.defaultdict(list)
                for u in cta["C"][wg]:
                    by_tile[u.j].append(u)
                for j, uses in by_tile.items():
                    assert j % 2 == wg and [u.kb for u in uses] == list(range(k_blocks))
                    cols = []
                    for u in uses:
                        bst, bph, col = cta["B"][(j, u.kb)]
                        a = cta["A"][(j, u.fill)]
                        assert (u.bstage, u.bphase, u.astage, u.aphase) == (bst, bph, a.stage, a.phase), (case, u)
                        seg, tap, chunk = decode(col, segs)
                        dy, dx = (tap // 3 - 1, tap % 3 - 1) if segs[seg][1] == 9 else (0, 0)
                        assert (a.seg, a.chunk, a.dx, a.y + u.dy1) == (seg, chunk, dx, dy), (case, u, a, col)
                        assert u.dy1 * bw + 128 <= a.rows
                        assert a.rows == (strip_rows(bw, bh, bn, 9) if u.kb < 9 * sc else 128)
                        cols.append(col)
                    assert sorted(cols) == list(range(k_blocks)), case
                    # after the strip segment (and everywhere without one) the k-blocks follow the packed order
                    assert cols[9 * sc:] == list(range(9 * sc, k_blocks)), case
                    # the fills of a strip serve exactly three consecutive k-blocks, the last one releases it
                    lasts = [u.kb for u in uses if u.last]
                    assert lasts == [3 * f + 2 for f in range(3 * sc)] + list(range(9 * sc, k_blocks)), case
        if sc:
            assert any(a.rows > 128 for cta in ctas for a in cta["A"].values())


def emulate(x, segs_x, packed, uses, fills, cols, bw, bh, dy1_of=lambda u: u.dy1):
    """The kernel's GEMM in float64, k-block by k-block in the consumer's order: each k-block reads 128 rows of its A
    fill starting dy1 * bw rows in, against the B tile of its packed column."""
    N, H, W, _ = x[0].shape
    cout = packed.shape[0]
    out = np.zeros((N, H, W, cout))
    for n in range(N):
        for y0 in range(0, H, bh):
            for x0 in range(0, W, bw):
                acc = np.zeros((128, cout))
                for u, col in zip(uses, cols):
                    a = fills[u.fill]
                    src = segs_x[a.seg]
                    r = np.arange(a.rows)
                    px, py = x0 + a.dx + r % bw, y0 + a.y + r // bw
                    inside = (px >= 0) & (px < W) & (py >= 0) & (py < H)
                    tile = np.zeros((a.rows, 64))
                    tile[inside] = src[n, py[inside], px[inside], a.chunk * 64:(a.chunk + 1) * 64]
                    rows = tile[dy1_of(u) * bw:dy1_of(u) * bw + 128]
                    acc += rows @ packed[:, col * 64:(col + 1) * 64].T
                r = np.arange(128)
                out[n, y0 + r // bw, x0 + r % bw] = acc
    return out


def test_strip_order_emulation_matches_conv2d(replay):
    """bw x bh = 8 x 16 strips over a 32 x 16 image, 2 chunks of 3x3 plus a 1x1 segment: the replayed K order and A rows
    give F.conv2d; the same emulation with the strip's dy offsets reversed does not."""
    segs = [(2, 9), (1, 1)]
    (ctas,) = run_cases(replay, [(1, 1, BOX_8x16, False, 128, 2, segs)])
    cta = ctas[0]
    uses = cta["C"][0]
    fills = {f: a for (j, f), a in cta["A"].items()}
    cols = [cta["B"][(0, u.kb)][2] for u in uses]
    g = torch.Generator().manual_seed(5)
    N, H, W, cout = 1, 32, 16, 16
    xs = [torch.randn(N, H, W, ch * 64, generator=g, dtype=torch.float64) for ch, _ in segs]
    ws = [torch.randn(cout, ch * 64, 3 if t == 9 else 1, 3 if t == 9 else 1, generator=g, dtype=torch.float64)
          for ch, t in segs]
    packed = torch.cat([w.permute(0, 2, 3, 1).reshape(cout, -1) for w in ws], 1).numpy()
    ref = sum(F.conv2d(x.permute(0, 3, 1, 2), w, padding=w.shape[-1] // 2) for x, w in zip(xs, ws)).permute(0, 2, 3, 1)
    xn = [x.numpy() for x in xs]
    got = emulate(xn, xn, packed, uses, fills, cols, 8, 16)
    np.testing.assert_allclose(got, ref.numpy(), rtol=1e-10, atol=1e-9)
    bad = emulate(xn, xn, packed, uses, fills, cols, 8, 16, dy1_of=lambda u: 2 - u.dy1 if u.kb < 18 else 0)
    assert not np.allclose(bad, ref.numpy(), rtol=1e-6)


def consumer_ops(uses, n_local, wg, early=False):
    """The consumer protocol of conv_tc_kernel: per k-block wait A full, wait B full, issue (the slots gain a reader),
    then retire the previous k-block (its readers leave; its B stage and, if it was the fill's last reader, its A slot are
    released); at the tile's end pass the MMA turn and retire the last k-block.  early: a strip slot is released one
    k-block before its last reader retires."""
    ops, prev = [], None
    strip_fills = sum(1 for u in uses if u.j == uses[0].j and u.dy1 == 2) if uses else 0

    def retire(p):
        out = [("unread", "A", p.astage), ("unread", "B", p.bstage), ("release", "B", p.bstage)]
        if (p.dy1 == 1) if early and p.fill < strip_fills else p.last:
            out.append(("release", "A", p.astage))
        return out

    for i, u in enumerate(uses):
        if u.kb == 0 and u.j > 0:
            ops.append(("turn_wait", wg))
        ops += [("full_wait", "A", u.astage, u.aphase, (u.j, u.fill)), ("full_wait", "B", u.bstage, u.bphase, (u.j, u.kb)),
                ("read", "A", u.astage), ("read", "B", u.bstage)]
        if prev is not None and prev.j == u.j:
            ops += retire(prev)
        prev = u
        if i + 1 == len(uses) or uses[i + 1].j != u.j:
            if u.j + 1 < n_local:
                ops.append(("turn_arrive", 1 - wg))
            ops += retire(u)
            prev = None
    return ops


def simulate(cta, stages, rng, early=False):
    n_local = max(j for _, j, *_ in cta["P"]) + 1 if cta["P"] else 0
    full = {r: [0] * stages[r] for r in "AB"}
    empty = {r: [0] * stages[r] for r in "AB"}
    content = {r: [None] * stages[r] for r in "AB"}
    readers = {r: [0] * stages[r] for r in "AB"}
    turn, taken = [0, 0], {"A": [], "B": []}
    roles = {"P": [("fill",) + p for p in cta["P"]]}
    for wg in (0, 1):
        roles[wg] = consumer_ops(cta["C"][wg], n_local, wg, early)
    pos = {r: 0 for r in roles}

    def runnable(r):
        op = roles[r][pos[r]]
        if op[0] == "fill":
            _, ring, _, _, st, ph = op
            return (empty[ring][st] & 1) != (ph ^ 1)
        if op[0] == "full_wait":
            return (full[op[1]][op[2]] & 1) != op[3]
        if op[0] == "turn_wait":
            return turn[op[1]] > 0
        return True

    while True:
        live = [r for r in roles if pos[r] < len(roles[r])]
        if not live:
            break
        ready = [r for r in live if runnable(r)]
        assert ready, f"deadlock: {[(r, roles[r][pos[r]]) for r in live]}"
        r = ready[0] if rng is None else rng.choice(ready)
        op = roles[r][pos[r]]
        pos[r] += 1
        if op[0] == "fill":
            _, ring, j, idx, st, _ = op
            assert content[ring][st] is None and readers[ring][st] == 0, \
                f"{ring} slot {st} refilled with {(j, idx)} while holding {content[ring][st]} ({readers[ring][st]} readers)"
            content[ring][st] = (j, idx)
            full[ring][st] += 1
        elif op[0] == "full_wait":
            _, ring, st, _, want = op
            assert content[ring][st] == want, f"warpgroup {r} expected {want} in {ring} slot {st}, found {content[ring][st]}"
            assert want[0] % 2 == r
            if not taken[ring] or taken[ring][-1] != want:
                taken[ring].append(want)
        elif op[0] == "read":
            readers[op[1]][op[2]] += 1
        elif op[0] == "unread":
            readers[op[1]][op[2]] -= 1
        elif op[0] == "release":                       # a reader may remain: the fill above asserts there is none
            content[op[1]][op[2]] = None
            empty[op[1]][op[2]] += 1
        elif op[0] == "turn_wait":
            turn[op[1]] -= 1
        elif op[0] == "turn_arrive":
            turn[op[1]] += 1
    return taken


RING_DEPTHS = {(128, 2): {"B": 4, "A": 4}, (64, 2): {"B": 7, "A": 6}, (64, 4): {"B": 6, "A": 5}}


@pytest.mark.parametrize("seed", [None, 0, 1, 2, 3])
def test_two_rings_take_fills_in_producer_order(replay, seed):
    rng = None if seed is None else random.Random(seed)
    for case, ctas in zip(CASES, run_cases(replay, CASES)):
        stages = RING_DEPTHS[(case[4], case[5])]
        for cta in ctas:
            taken = simulate(cta, stages, rng)
            for ring in "AB":
                assert taken[ring] == [p[1:3] for p in cta["P"] if p[0] == ring], (case, ring)


def test_model_catches_a_strip_slot_released_one_k_block_early(replay):
    """At the kernel's depths the B ring keeps the producer too close behind the consumers to refill an A slot early;
    with a B ring deeper than the A ring the model must see the slot refilled under its last reader."""
    case = (6, 1, BOX_8x16, False, 128, 2, [(2, 9)])
    (ctas,) = run_cases(replay, [case], depths=(8, 2))
    simulate(ctas[0], {"B": 8, "A": 2}, random.Random(0))
    with pytest.raises(AssertionError, match="refilled"):
        for seed in range(50):
            simulate(ctas[0], {"B": 8, "A": 2}, random.Random(seed), early=True)


def test_conv_tc_instantiations_do_not_spill_and_keep_their_mma_instructions():
    r = subprocess.run([B.NVCC, *B.ARCH, *B.CFLAGS, *B.PRODUCT_DEFS, "-Xptxas", "-v", "-c", os.path.join(B.CSRC, "conv_tc.cu"),
                        "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    blocks = [b for b in re.split(r"Compiling entry function ", r.stderr) if re.match(r"'\S*conv_tc_kernel", b)]
    assert len(blocks) == 5
    for b in blocks:
        assert re.search(r"0 bytes spill stores, 0 bytes spill loads", b), b
    lib = B.build()
    assert os.path.exists(lib)
    sass = subprocess.run(["cuobjdump", "-sass", os.path.join(B.LIBDIR, "obj", "conv_tc.o")], capture_output=True,
                          text=True, check=True).stdout
    for instr in ("HGMMA.64x128x16.F32", "HGMMA.64x64x16.F32", "HGMMA.64x64x8.F32.TF32"):
        assert instr in sass, instr
