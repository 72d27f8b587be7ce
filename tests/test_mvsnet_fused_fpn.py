"""The fused FPN tail: feat3 = conv3x3(W3)(up2(f.i2b)) + conv3x3(W3 . Ws3)(f.c3) in one tensor-core launch on the coarse
grid (k_conv_tc MODE 3, CIN 64: four channel groups of f.i2b and the four parity sub-tiles of f.c3, hi/lo weights, one
rounding).  The CPU test pins its tile plan at the benchmark window; the GPU tests check feat3 against the fp64
reference on windows whose last tiles are partial in W and H, and on a cached window that runs FeatureNet on one view."""
import ctypes

import numpy as np
import pytest

from oracle import mvsnet_layers as ML
from tandem_b200._lib import lib

PLAN_KEYS = "S R TW P DR nch slot_pos tiles_w tiles_h tiles_d grid smem nwg".split()


def fused_plan(V, H, W, smem_kb=225):
    out = (ctypes.c_longlong * 13)()
    assert lib().tdm_debug_conv_plan_n(64, 64, 1, V, H // 2, W // 2, 0, 3, smem_kb, out, 13) == 0, lib().tdm_last_error()
    return dict(zip(PLAN_KEYS, (int(v) for v in out)))


@pytest.mark.parametrize("V", [7, 1])
def test_fused_plan_at_the_benchmark_window(V):
    """640x480, all 7 views or the one view a sliding window adds: 8-row x 30-column coarse tiles (two 128-position chunks,
    one 64-position sub-chunk per warpgroup), a 3-deep ring of 8 channel-group boxes next to the 72 KB hi/lo B image."""
    p = fused_plan(V, 480, 640)
    b_image = 9 * 4 * 64 * 32                       # 9 taps x 4 K=16 steps x 64 hi/lo columns x 32 bytes
    assert b_image == 72 * 1024
    assert (p["S"], p["R"], p["TW"], p["P"], p["nch"], p["nwg"]) == (3, 8, 30, 32, 2, 4), p
    assert (p["DR"], p["tiles_d"]) == (V, 1), p
    assert (p["tiles_w"], p["tiles_h"], p["grid"]) == (11, 30, 330), p
    assert p["smem"] == b_image + p["S"] * 8 * p["slot_pos"] * 16 + 256 and p["smem"] <= 225 * 1024, p
    assert 2 * p["P"] <= 256 and 2 * (p["R"] + 2) <= 256, p   # the f.c3 sub-tile boxes span 2P columns, 2(R+2) rows


@pytest.mark.parametrize("V,H,W", [(2, 64, 224), (13, 96, 448), (1, 64, 224)])
def test_fused_plan_edge_tiles(V, H, W):
    """The GPU test windows' plans: 64x224 ends in a partial tile along W and along H, 96x448 along H and D."""
    p = fused_plan(V, H, W)
    h, w = H // 2, W // 2
    assert p["tiles_w"] * p["TW"] >= w and p["tiles_h"] * p["R"] >= h and p["tiles_d"] * p["DR"] >= V, p
    if H == 64:
        assert w % p["TW"] and h % p["R"], p
    else:
        assert h % p["R"] and V % p["DR"], p


def _check_feat3(m, precision, label):
    from tandem_b200 import default_weights
    from tandem_b200.weights_io import load_tdmw
    w, _, _ = load_tdmw(default_weights("abl03_view_aggregation"))
    T = {n: m.debug_tensor(n) for n in ("f.i2b", "f.c3", "feat3")}
    assert np.isfinite(T["feat3"]).all(), label
    y_ref, bound, ar = ML.fused_feat3_reference(w, T, precision)
    r = ML.check("feat3", T["feat3"], y_ref, bound, ar)
    idx, worst = r.worst
    print(f"{label} {precision}: feat3 worst error / bound {worst:.4f} at (c, d, h, w) {tuple(int(i) for i in idx)}")
    assert worst <= 1.0, f"{label}: {int((r.ratio > 1).sum())} of {r.ratio.size} feat3 elements out of bound"
    return T["feat3"]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["mixed16", "bf16"])
@pytest.mark.parametrize("V,H,W", [(2, 64, 224), (13, 96, 448)])
def test_fused_feat3_partial_tiles(V, H, W, precision):
    from tandem_b200 import DrMvsnet, default_weights
    from tandem_b200.synthetic import mvs_plane_window
    win = mvs_plane_window(V=V, H=H, W=W, seed=0)
    m = DrMvsnet(default_weights("abl03_view_aggregation"), precision=precision)
    m.set_option("debug_poison", 1)                 # activation interiors start as NaN: a skipped store cannot pass
    m.CallAsync(H, W, V, win["ref_index"], win["bgrs"], win["K"], win["c2ws"], win["depth_min"], win["depth_max"], 10.0)
    m.GetResult()
    assert any(r[0] == "f.fpn3[tc-up2]" for r in m.profile())
    _check_feat3(m, precision, f"{W}x{H}v{V}")


@pytest.mark.gpu
def test_fused_feat3_one_new_view():
    """A cached window that adds one keyframe runs FeatureNet, and the fused launch, over k = 1 plane: its feat3 equals an
    uncached handle's bit for bit, and that one is within the reference bound."""
    from tandem_b200 import DrMvsnet, default_weights
    from tandem_b200.synthetic import mvs_plane_window
    V, H, W = 2, 64, 224
    wins = [mvs_plane_window(V=V, H=H, W=W, seed=s) for s in (0, 1)]
    bgrs = [wins[0]["bgrs"][0], wins[0]["bgrs"][1], wins[1]["bgrs"][1]]
    c2ws = [wins[0]["c2ws"][0], wins[0]["c2ws"][1], wins[1]["c2ws"][1]]
    K, dmin, dmax = wins[0]["K"], wins[0]["depth_min"], wins[0]["depth_max"]
    cached = DrMvsnet(default_weights("abl03_view_aggregation"), precision="mixed16")
    cached.CallAsyncIds(H, W, V, 0, [0, 1], [bgrs[0], bgrs[1]], K, [c2ws[0], c2ws[1]], dmin, dmax, 10.0)
    cached.GetResult()
    cached.CallAsyncIds(H, W, V, 0, [0, 2], [None, bgrs[2]], K, [c2ws[0], c2ws[2]], dmin, dmax, 10.0)
    cached.GetResult()
    assert cached.debug_tensor("f.c3").shape[1] == 1   # FeatureNet ran over the new view only
    plain = DrMvsnet(default_weights("abl03_view_aggregation"), precision="mixed16")
    plain.CallAsync(H, W, V, 0, [bgrs[0], bgrs[2]], K, [c2ws[0], c2ws[2]], dmin, dmax, 10.0)
    plain.GetResult()
    ref = _check_feat3(plain, "mixed16", f"{W}x{H}v{V} uncached")
    got = cached.debug_tensor("feat3")
    assert np.array_equal(got, ref, equal_nan=True), f"k = 1: feat3 differs on {int((got != ref).sum())} values"
