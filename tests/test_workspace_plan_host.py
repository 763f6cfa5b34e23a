"""Host tests (no GPU) of the liveness-planned activation workspace (sgmse_b200_workspace_plan).

Every buffer of one forward lives from the launch step after its allocation to the launch of its last reader, and the
plan packs buffers whose lifetimes do not intersect into shared address ranges.  The GPU side (the same results with
freed ranges poisoned) is tests/test_gpu_long_clips.py."""
import numpy as np
import pytest

from sgmse_b200 import Engine, EngineConfig

CONFIGS = {"ncsnpp": (EngineConfig.ncsnpp_16k, 256), "ncsnpp_48k": (EngineConfig.ncsnpp_48k, 768),
           "ncsnpp_v2": (EngineConfig.ncsnpp_v2, 256)}
MODES = ("fp16_tc", "tf32_tc", "fp32")


def live_peak(plan):
    """max over steps of the bytes of the buffers live at that step"""
    b = plan["buffers"]
    delta = np.zeros(plan["steps"] + 2, dtype=np.int64)
    np.add.at(delta, b[:, 2], b[:, 1])
    np.add.at(delta, b[:, 3] + 1, -b[:, 1])
    return int(np.cumsum(delta).max())


def assert_no_live_overlap(plan):
    b = plan["buffers"]
    for i in range(len(b)):
        off, n, first, last, _ = b[i]
        clash = (b[:, 2] <= last) & (first <= b[:, 3]) & (b[:, 0] < off + n) & (off < b[:, 0] + b[:, 1])
        clash[i] = False
        assert not clash.any(), f"buffer {i} {tuple(b[i])} overlaps {b[clash][:3].tolist()} while both are live"


@pytest.mark.parametrize("backbone", list(CONFIGS))
@pytest.mark.parametrize("mode", MODES)
def test_plan_is_sound_and_tight(backbone, mode):
    make, F = CONFIGS[backbone]
    eng, twin = Engine(make(mode=mode)), Engine(make(mode=mode))
    for B, T in ((1, 64), (1, 512), (3, 256), (1, 4800)):
        plan = eng.workspace_plan(B, F, T)
        b = plan["buffers"]
        assert len(b) > 100 and plan["steps"] > 100
        assert (b[:, 0] % 256 == 0).all()
        assert (b[:, 2] <= b[:, 3]).all() and (b[:, 3] <= plan["steps"]).all()
        assert_no_live_overlap(plan)
        assert (b[:, 0] + b[:, 1] <= plan["bytes"]).all()
        peak = live_peak(plan)
        assert plan["bytes"] <= 1.25 * peak, (B, T, plan["bytes"], peak)
        # the network output is read after the forward; without taps nothing else is
        assert (b[:, 3] == plan["steps"]).sum() == 1 and not b[:, 4].any()
        other = twin.workspace_plan(B, F, T)
        assert other["bytes"] == plan["bytes"] and np.array_equal(other["buffers"], b)
        # the layout without reuse: every buffer in its own range
        assert eng.workspace_bytes(B, F, T) >= int(b[:, 1].sum())


@pytest.mark.parametrize("backbone", ["ncsnpp", "ncsnpp_48k"])
def test_fp16_plan_is_a_third_of_the_bump_layout(backbone):
    make, F = CONFIGS[backbone]
    eng = Engine(make(mode="fp16_tc"))
    bump = eng.workspace_bytes(1, F, 512)
    planned = eng.workspace_plan(1, F, 512)["bytes"]
    print(f"{backbone} fp16_tc (1, {F}, 512): {planned / 1e9:.3f} GB planned, {bump / 1e9:.2f} GB without reuse")
    assert planned <= bump / 3


@pytest.mark.parametrize("mode", MODES)
def test_taps_live_to_the_end(mode):
    eng = Engine(EngineConfig.ncsnpp_16k(mode=mode))
    plain = eng.workspace_plan(1, 256, 256)
    eng.set_option("record_taps", 1)
    tapped = eng.workspace_plan(1, 256, 256)
    b0, b1, steps = plain["buffers"], tapped["buffers"], tapped["steps"]
    assert steps == plain["steps"] and np.array_equal(b0[:, [1, 2]], b1[:, [1, 2]])
    t = b1[:, 4] == 1
    # one tap per block-level module plus the input conv (data and GroupNorm statistics) and one per output pyramid level
    assert t.sum() > 100
    assert (b1[t, 3] == steps).all()
    assert (b1[~t, 3] == b0[~t, 3]).all()
    assert_no_live_overlap(tapped)
    assert tapped["bytes"] > plain["bytes"]
    eng.set_option("record_taps", 0)
    assert np.array_equal(eng.workspace_plan(1, 256, 256)["buffers"], b0)


def test_plan_follows_kernel_options():
    """gn_self folds GroupNorm finalize into the apply at small levels: one launch fewer per folded GroupNorm."""
    eng = Engine(EngineConfig.ncsnpp_16k())
    on = eng.workspace_plan(1, 256, 512)
    eng.set_option("gn_self", 2)
    off = eng.workspace_plan(1, 256, 512)
    assert off["steps"] > on["steps"] and len(off["buffers"]) == len(on["buffers"])
    assert_no_live_overlap(off)


def test_tensors_past_2_to_the_31_elements_are_refused():
    eng = Engine(EngineConfig.ncsnpp_16k())
    assert eng.workspace_plan(1, 256, 32704)["bytes"] > 0              # 261.6 s: 256 x 256 x 32704 < 2^31
    with pytest.raises(RuntimeError, match="2\\^31 elements"):
        eng.workspace_plan(1, 256, 32768)
    eng48 = Engine(EngineConfig.ncsnpp_48k())
    assert eng48.workspace_plan(1, 768, 10880)["bytes"] > 0             # 87.0 s
    with pytest.raises(RuntimeError, match="2\\^31 elements"):
        eng48.workspace_plan(1, 768, 10944)
