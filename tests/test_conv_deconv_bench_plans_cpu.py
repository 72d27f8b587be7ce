"""The tile planner's choices for the transposed convolutions (make_plan mode 1 in tandem_b200/csrc/conv_tc.cuh) of the
benchmark window (640x480, 48 / 32 / 8 depth planes), queried through tdm_debug_conv_plan_n.  Each stage runs conv11
(16 -> 8 channels, N = 64), conv9 (32 -> 16, N = 128) and conv7 (64 -> 32, four N = 64 slices of one output channel group
each) on its input grid, conv9 on four consumer warpgroups and the N = 64 layers on two.  A tile's shared memory
holds, besides the B image and the input ring, two output boxes of 128 bytes per input position and output channel group
of the slice; the plans below were measured with that epilogue."""
import ctypes

import pytest

from tandem_b200._lib import CONV_PLAN_KEYS, lib

MAX_CH = 8          # kDeconvMaxCh


def _plan(cin, npad, D, H, W):
    out = (ctypes.c_longlong * 13)()
    rc = lib().tdm_debug_conv_plan_n(cin, npad, 2, D, H, W, 1, 1, 225, out, 13)
    assert rc == 0, lib().tdm_last_error()
    return dict(zip(CONV_PLAN_KEYS, (int(x) for x in out)))


def _launches(H, W, Ds):
    for s, D in enumerate(Ds):
        sc = 4 >> s
        h, w = H // sc, W // sc
        for lvl, (name, cin, npad) in enumerate([("conv11", 16, 64), ("conv9", 32, 128), ("conv7", 64, 64)]):
            yield f"s{s + 1}.{name}", (cin, npad, max(D >> (lvl + 1), 1), h >> (lvl + 1), w >> (lvl + 1))


def _b_bytes(cin, npad):
    nblk = 4 * (cin // 16)                        # ksteps(cin, 4 taps)
    return (2 * nblk * npad * 32 + 127) // 128 * 128


# layer -> (S, R, TW, DR, nch, grid, smem)
PLANS = {
    "s1.conv11": (3, 6, 40, 4, 2, 120, 111872),
    "s1.conv9": (3, 4, 40, 2, 2, 48, 215296),
    "s1.conv7": (3, 5, 20, 2, 1, 9, 162048),
    "s2.conv11": (3, 15, 32, 6, 4, 120, 196352),
    "s2.conv9": (3, 4, 40, 2, 2, 120, 215296),
    "s2.conv7": (3, 3, 40, 2, 1, 20, 182528),
    "s3.conv11": (3, 12, 30, 4, 3, 220, 153344),
    "s3.conv9": (3, 6, 32, 2, 2, 100, 228608),
    "s3.conv7": (3, 3, 40, 1, 1, 40, 182528),
}


@pytest.mark.parametrize("name", sorted(PLANS))
def test_transposed_conv_plans_of_the_benchmark_window(name):
    (cin, npad, D, H, W), = [a for n, a in _launches(480, 640, (48, 32, 8)) if n == name]
    p = _plan(cin, npad, D, H, W)
    S, R, TW, DR, nch, grid, smem = PLANS[name]
    assert (p["S"], p["R"], p["TW"], p["DR"], p["nch"], p["grid"], p["smem"]) == PLANS[name], (name, p)
    # four consumer warpgroups for the N = 128 conv9, two for the N = 64 layers; with four, a plane's 2 * nch sub-chunks
    # fill whole rounds (or the plan has one chunk); the box offsets of at most kDeconvMaxCh chunks stay in registers
    assert p["nwg"] == (4 if npad == 128 else 2) and nch <= MAX_CH, (name, p)
    assert p["nwg"] == 2 or nch == 1 or (2 * nch) % 4 == 0, (name, p)
    # shared memory: B image + ring + 256 bytes of barriers + two output boxes of npad / 64 channel groups
    slots = S * (cin // 8) * p["slot_pos"] * 16
    boxes = 2 * (npad // 64) * 128 * R * TW
    assert smem == _b_bytes(cin, npad) + slots + 256 + boxes and smem <= 225 * 1024, (name, p)
    # an output box spans 2 TW columns and 2 R rows: TMA box dimensions are at most 256
    assert 2 * TW <= 256 and 2 * R <= 256, (name, p)
    assert grid == p["tiles_w"] * p["tiles_h"] * p["tiles_d"], (name, p)
