"""The undilated level-0 cloud of makeCoarseDepthL0 and the MVSNet depth range's quantile over it (no GPU): the restatements
coarse_nodia_oracle / idepth_quantile_oracle (oracle/coarse_nodia_oracle.c) equal the reference's own makeCoarseDepthL0 body
(CoarseTracker.cpp:148-374, pc_*_nodia kept across keyframes) and its own get_idepth_quantile (tandem_backend.cpp:354-361) bit
for bit: pc_n_nodia, the four arrays including slot pc_n_nodia, and the quantile's idepth and depth at fractions 0, 0.2, the
one selecting index n-1, and 1 (NaN).  The reference's results are stored in tests/golden/reference_pins_coarse_nodia.npz
(oracle/gen_reference_pins_coarse_nodia.py)."""
import os

import numpy as np
import pytest

from oracle import pins_coarse_ref as P
from oracle.coarse_nodia import CoarseNodiaOracle, fractions, run_oracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pins_coarse_nodia.npz")


def same_bits(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)].view(np.uint32), b[~np.isnan(b)].view(np.uint32))


@pytest.mark.parametrize("name", list(P.CASES))
def test_coarse_nodia_oracle_pinned_to_reference(name):
    g = np.load(GOLDEN)
    out = run_oracle(name)
    assert len(out) == len(P.CASES[name][2])
    for j, (m, arrs, fr, q) in enumerate(out):
        assert m == int(g[f"{name}_{j}_n"]), (j, m)
        assert P.digest(*arrs) == str(g[f"{name}_{j}_arrays"]), j
        assert np.array_equal(fr, g[f"{name}_{j}_fractions"]), j
        assert same_bits(q, g[f"{name}_{j}_quantile"]), (j, q, g[f"{name}_{j}_quantile"])


def test_pins_cover_the_stale_slot_the_quantile_range_and_nan():
    g = np.load(GOLDEN)
    stale = nan_rgbd = 0
    for name in P.CASES:
        for j, (m, arrs, fr, q) in enumerate(run_oracle(name)):
            assert np.isnan(q[-1]).all()                                   # fraction 1: index n
            if m:
                assert not np.isnan(q[:3]).any()
                assert q[0, 0] == arrs[2][:m].min() and q[2, 0] == arrs[2][:m].max()
                stale += arrs[2][m] <= 0 and arrs[0][m] > 0                # a rejected candidate in slot n
            elif P.CASES[name][2][j]["rgbd"] and P.CASES[name][2][j]["n"]:
                nan_rgbd += 1
                assert np.isnan(q).all() and arrs[0][0] > 0                # RGB-D: every candidate rejected, the last in slot 0
    assert stale >= 2 and nan_rgbd >= 2, (stale, nan_rgbd)
    assert int(g["mono_130x96_l3_two_keyframes_1_n"]) < int(g["mono_130x96_l3_two_keyframes_0_n"])


def test_quantile_index_rounds_like_the_reference():
    o = CoarseNodiaOracle(8, 8)
    vals = np.arange(1, 11, dtype=np.float32)[::-1].copy()
    o.nodia[2 * 64:2 * 64 + 10] = vals
    # (int)(0.2f * 10.f) = 2; 1.0 * 10 = 10: outside
    assert o.quantile(10, 0.2).tolist() == [3.0, np.float32(1.0) / np.float32(3.0)]
    # float(5/6) * 6 is 4.99999988 exactly, but the float product rounds to 5.0f: index 5, not 4
    assert o.quantile(6, np.float32(5 / 6))[0] == 10.0           # of 10, 9, .., 5: the largest
    assert np.isnan(o.quantile(10, 1.0)).all() and np.isnan(o.quantile(0, 0.0)).all()
    assert fractions(10)[2] * np.float32(10) < 10 and int(fractions(10)[2] * np.float32(10)) == 9
