"""CPU check of the wgmma convolution's ring schedule (sgmse_b200/csrc/conv_tc_sched.h).

conv_tc_kernel has one producer and two "ping-pong" consumer warpgroups around an mbarrier-guarded ring of shared-memory
stages.  tests/c/conv_tc_schedule.cu replays the kernel's loops on the host with the same helpers and prints every
(tile, k-block) -> (stage, phase) of each role.  Here those sequences drive a model of the mbarriers (a parity wait
passes once the phase of that parity has completed) and of the named-barrier hand-off of the MMA turn, under several
interleavings.  It asserts that the consumers take the fills in exactly the producer's order, alternating warpgroups
per tile, that no stage is refilled before its consumer released it, and that nothing deadlocks."""
import os
import random
import subprocess

import pytest

from sgmse_b200.build import CSRC, NVCC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = [(t, g, k, s) for t in (1, 2, 3, 8, 33) for g in (1, 2, 5) for k in (1, 2, 3, 5, 18) for s in (2, 4, 7)]


@pytest.fixture(scope="module")
def replay(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("conv_tc_schedule") / "replay")
    subprocess.run([NVCC, "-x", "cu", "-std=c++17", "-I", CSRC, os.path.join(ROOT, "tests", "c", "conv_tc_schedule.cu"),
                    "-o", exe], check=True, capture_output=True)

    def run(cases):
        out = subprocess.run([exe], input="".join(f"{t} {g} {k} {s}\n" for t, g, k, s in cases),
                             capture_output=True, text=True, check=True).stdout
        results, ctas = [], None
        for line in out.splitlines():
            f = line.split()
            if f[0] == "B":
                ctas = [] if ctas is None else ctas
                ctas.append({"P": [], "C": {0: [], 1: []}})
            elif f[0] == "P":
                ctas[-1]["P"].append(tuple(map(int, f[1:])))
            elif f[0] == "C":
                ctas[-1]["C"][int(f[1])].append(tuple(map(int, f[2:])))
            else:
                results.append(ctas or [])
                ctas = None
        assert len(results) == len(cases)
        return results

    return run


def consumer_ops(seq, n_local, wg, handoff=True):
    """The consumer warpgroup's protocol as in the kernel: wait for the turn, wait full / release the previous stage per
    k-block, pass the turn, release the last stage."""
    ops, prev, cur = [], None, None
    for j, kb, stage, phase in seq:
        if j != cur:
            cur = j
            if j > 0 and handoff:
                ops.append(("turn_wait", wg))
        ops.append(("full_wait", stage, phase, (j, kb)))
        if kb > 0:
            ops.append(("release", prev))
        prev = stage
        if kb == max(k for jj, k, _, _ in seq if jj == j):
            if j + 1 < n_local and handoff:
                ops.append(("turn_arrive", 1 - wg))
            ops.append(("release", stage))
    return ops


def simulate(cta, stages, rng, handoff=True):
    """Run the producer and both consumers of one CTA to completion under the scheduling choices of rng (None: always the
    first runnable role).  Returns the fills in the order the consumers took them."""
    fills = cta["P"]
    n_local = fills[-1][0] + 1 if fills else 0
    full, empty = [0] * stages, [0] * stages        # completed phases of each mbarrier
    content = [None] * stages
    turn = [0, 0]
    taken = []
    roles = {"P": [("fill",) + f for f in fills]}
    for wg in (0, 1):
        roles[wg] = consumer_ops(cta["C"][wg], n_local, wg, handoff)
    pos = {r: 0 for r in roles}

    def runnable(r):
        op = roles[r][pos[r]]
        if op[0] == "fill":
            return (empty[op[3]] & 1) != (op[4] ^ 1)
        if op[0] == "full_wait":
            return (full[op[1]] & 1) != op[2]
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
            _, j, kb, stage, _ = op
            assert content[stage] is None, f"stage {stage} refilled with {(j, kb)} before {content[stage]} was released"
            content[stage] = (j, kb)
            full[stage] += 1
        elif op[0] == "full_wait":
            _, stage, _, want = op
            assert content[stage] == want, f"warpgroup {r} expected {want} in stage {stage}, found {content[stage]}"
            assert want[0] % 2 == r
            taken.append(want)
        elif op[0] == "release":
            content[op[1]] = None
            empty[op[1]] += 1
        elif op[0] == "turn_wait":
            turn[op[1]] -= 1
        elif op[0] == "turn_arrive":
            turn[op[1]] += 1
    return taken


def test_replay_covers_every_local_tile(replay):
    for (t, g, k, s), ctas in zip(CASES, replay(CASES)):
        tiles = sorted(c + j * g for c, cta in enumerate(ctas) for j in {f[0] for f in cta["P"]})
        assert tiles == list(range(t)), (t, g, k, s)
        for cta in ctas:
            n_local = len(cta["P"]) // k
            assert [f[:2] for f in cta["P"]] == [(j, kb) for j in range(n_local) for kb in range(k)]
            for wg in (0, 1):
                assert [c[:2] for c in cta["C"][wg]] == [(j, kb) for j in range(wg, n_local, 2) for kb in range(k)]


@pytest.mark.parametrize("seed", [None, 0, 1, 2])
def test_consumers_take_fills_in_producer_order(replay, seed):
    rng = None if seed is None else random.Random(seed)
    for (t, g, k, s), ctas in zip(CASES, replay(CASES)):
        for cta in ctas:
            taken = simulate(cta, s, rng)
            assert taken == [f[:2] for f in cta["P"]], (t, g, k, s)


def test_model_catches_a_missing_turn_handoff(replay):
    """Without the hand-off the second warpgroup can wait on a stage whose parity still shows an older round: the model
    has to report that, or the checks above prove nothing."""
    case = (8, 1, 3, 2)
    (ctas,) = replay([case])
    with pytest.raises(AssertionError):
        for seed in range(20):
            simulate(ctas[0], case[3], random.Random(seed), handoff=False)
