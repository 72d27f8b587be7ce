"""The input-stationary planner's choices (make_plan_is in tandem_b200/csrc/conv_tc_is.cuh) for the six launches of the
benchmark window (640x480, 48 / 32 / 8 depth planes) and of the config-1 window (320x256, 32 / 32 / 8), queried through
tdm_debug_conv_plan_n mode 200.  Each stage runs conv0 (its cost volume, 32 >> (stage - 1) channels -> 8) and prob (8 -> 1)
at 1/4, 1/2 and full resolution.  The kernel's batched MMA chains (is_batch) were measured at these plans, so a planner
change that moves them shows up here."""
import ctypes
import math

import pytest

from tandem_b200._lib import CONV_PLAN_KEYS, lib

IS_MODE = 200
MAX_CH = 8          # kIsMaxCh
SMS = 132           # SMs of an H100 SXM: one CTA per SM


def _plan(cin, cpk, D, H, W):
    out = (ctypes.c_longlong * 13)()
    rc = lib().tdm_debug_conv_plan_n(cin, cpk, 3, D, H, W, 1, IS_MODE, 225, out, 13)
    assert rc == 0, lib().tdm_last_error()
    return dict(zip(CONV_PLAN_KEYS, (int(x) for x in out)))


def _launches(H, W, Ds):
    for s, D in enumerate(Ds):
        sc = 4 >> s
        yield f"s{s + 1}.conv0", (32 >> s, 16, D, H // sc, W // sc)
        yield f"s{s + 1}.prob", (8, 8, D, H // sc, W // sc)


# (window, layer) -> (R, TW, DR, nch, grid); conv0 and prob of a stage share the tiling
PLANS = {
    ("bench", "s1"): (15, 32, 16, 4, 120),
    ("bench", "s2"): (24, 30, 32, 6, 110),
    ("bench", "s3"): (30, 32, 8, 8, 320),
    ("config1", "s1"): (6, 40, 6, 2, 132),
    ("config1", "s2"): (12, 40, 11, 4, 132),
    ("config1", "s3"): (24, 30, 8, 6, 121),
}
WINDOWS = {"bench": (480, 640, (48, 32, 8)), "config1": (256, 320, (32, 32, 8))}


@pytest.mark.parametrize("window", sorted(WINDOWS))
def test_input_stationary_plans_of_the_benchmark_windows(window):
    for name, (cin, cpk, D, H, W) in _launches(*WINDOWS[window]):
        p = _plan(cin, cpk, D, H, W)
        key = (window, name)
        # ring depth: three planes in flight (each plane is consumed once, by one chain per sub-chunk)
        assert p["S"] == 3, (key, p)
        assert p["smem"] <= 225 * 1024, (key, p)
        assert p["nch"] <= MAX_CH, (key, p)
        # four consumer warpgroups, every one of them busy in every round of a plane's 2 * nch sub-chunks
        assert p["nwg"] == 4 and (2 * p["nch"]) % p["nwg"] == 0, (key, p)
        assert (p["R"], p["TW"], p["DR"], p["nch"], p["grid"]) == PLANS[(window, name.split(".")[0])], (key, p)


def test_stage3_wave_count():
    """Stage 3 of the benchmark window cannot fit two waves: at most kIsMaxCh chunks of 128 positions per tile, i.e. 1024
    positions with their halo, against 480 x 640 / 264 = 1164 per tile for two waves of 132.  It runs three; the config-1
    window's stage 3 runs one."""
    for window, waves in (("bench", 3), ("config1", 1)):
        H, W, _ = WINDOWS[window]
        for cin, cpk in ((8, 16), (8, 8)):
            p = _plan(cin, cpk, 8, H, W)
            assert math.ceil(p["grid"] / SMS) == waves, (window, cin, cpk, p)
    assert 128 * MAX_CH < 480 * 640 / (2 * SMS)
