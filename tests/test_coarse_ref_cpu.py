"""n7 pin (no GPU): the restatement oracle/coarse_ref_oracle.c, chained with the n1 dense block of oracle/front_oracle.c, equals
the reference's own CoarseTracker::makeCoarseDepthL0 body (CoarseTracker.cpp:148-374) chained with its own dense block
(:655-725) bit for bit: every level's pc_n and its four arrays including slot pc_n, over one or two consecutive keyframes.  The
reference's results are stored in tests/golden/reference_pins_coarse_ref.npz (oracle/gen_reference_pins_coarse_ref.py)."""
import os

import numpy as np
import pytest

from oracle import pins_coarse_ref as P
from oracle.coarse_ref import CoarseRefOracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pins_coarse_ref.npz")


@pytest.mark.parametrize("name", list(P.CASES))
def test_coarse_ref_oracle_pinned_to_reference_makeCoarseDepthL0(name):
    g = np.load(GOLDEN)
    out = P.run_oracle(name, g[f"{name}_T"])
    (_, _), levels, kfs = P.CASES[name]
    assert len(out) == len(kfs)
    for j, (pc_n, arrs) in enumerate(out):
        assert pc_n == g[f"{name}_{j}_pc_n"].tolist(), (j, pc_n)
        for l in range(levels):
            assert P.digest(*arrs[l]) == str(g[f"{name}_{j}_l{l}"]), (j, l)


def test_coarse_ref_oracle_rounds_like_the_reference():
    # (int)(u + 0.5f) in float (monocular) and (int)(u + 0.5) in double (RGB-D) land on different pixels for 0.49999997f
    w, h = 16, 12
    gray = [np.full((h, w), 100.0, np.float32)]
    pts = (np.array([0.49999997], np.float32), np.array([6.0], np.float32), np.array([0.5], np.float32), np.array([1.0], np.float32))
    mono, rgbd = CoarseRefOracle(w, h, 1), CoarseRefOracle(w, h, 1)
    mono.set_coarse_tracking_ref(pts, gray, rgbd=False)
    rgbd.set_coarse_tracking_ref(pts, gray, rgbd=True)
    # pixel (1, 6) monocular: dilated onto (2, 5) / (2, 7); pixel (0, 6) RGB-D: its diagonal neighbours wrap to column w-1
    assert mono.set_coarse_tracking_ref(pts, gray, rgbd=False) == [2]
    assert rgbd.set_coarse_tracking_ref(pts, gray, rgbd=True) == [0]


def test_coarse_ref_oracle_rejects_points_outside_the_image():
    o = CoarseRefOracle(16, 12, 1)
    gray = [np.zeros((12, 16), np.float32)]
    for u in (-1.5, 15.5, np.nan):
        with pytest.raises(ValueError):
            o.set_coarse_tracking_ref(([u], [3.0], [1.0], [1.0]), gray)
    # -0.6 + 0.5f truncates to pixel 0: inside, as in the reference
    assert o.set_coarse_tracking_ref(([-0.6], [3.0], [1.0], [1.0]), gray) == [0]


def test_coarse_ref_pins_exercise_the_stale_slot():
    g = np.load(GOLDEN)
    out = P.run_oracle("mono_130x96_l3_two_keyframes", g["mono_130x96_l3_two_keyframes_T"])
    # keyframe 0 leaves its rejected idepth <= 0 candidate (or a dense point) behind the count; the slot is part of the data
    for pc_n, arrs in out:
        assert len(arrs[0][0]) == pc_n[0] + 1
    assert any(not np.array_equal(out[0][1][l][0][:5], out[1][1][l][0][:5]) for l in range(3))
