"""Host logic of the feature cache (no GPU): a cached MVSNet call runs FeatureNet over the k views it adds, so the
tensor-core tile planners are asked for FeatureNet tiles over 1..V planes, one plane included.  Each plan must cover the
grid, fit 225 KB of shared memory, the wgmma N limit and the TMA box limit, as at V planes."""
import ctypes

import pytest

from tandem_b200._lib import lib


def featurenet_shapes(H, W, D):
    """(cin, npad, kd, D, H, W, pd, mode) of every tensor-core FeatureNet launch over D planes (kd = 1, pd = 0)."""
    shapes = [(cin, npad, 1, D, H // sc, W // sc, 0, 0) for cin, npad, sc in [(8, 32, 1), (16, 32, 2), (32, 64, 4), (32, 32, 2), (32, 32, 1)]]
    shapes.append((32, 64, 1, D, H // 2, W // 2, 0, 3))                       # f.out3a: up-2 conv on the coarse grid
    shapes += [(cin, npad, 1, D, H // sc, W // sc, 5, 400) for cin, npad, sc in [(8, 16, 2), (16, 32, 4)]]   # conv1.0 / conv2.0
    return shapes


@pytest.mark.parametrize("H,W", [(480, 640), (256, 320), (96, 128)])
@pytest.mark.parametrize("D", [1, 2, 3, 4, 5, 6, 7])
def test_featurenet_plans_for_every_plane_count(H, W, D):
    l = lib()
    out = (ctypes.c_longlong * 13)()
    for (cin, npad, kd, d, h, w, pd, mode) in featurenet_shapes(H, W, D):
        key = (cin, npad, d, h, w, mode)
        assert l.tdm_debug_conv_plan_n(cin, npad, kd, d, h, w, pd, mode, 225, out, 13) == 0, (key, l.tdm_last_error())
        S, R, TW, P, DR, nch, slot_pos, tw, th, td, grid, smem, nwg = [int(x) for x in out]
        assert nwg in (2, 4), key
        assert tw * TW >= w and (tw - 1) * TW < w and th * R >= h and (th - 1) * R < h and td * DR >= d and (td - 1) * DR < d, key
        assert grid == tw * th * td and grid >= 1 and R >= 1 and DR >= 1 and smem <= 225 * 1024, key
        if mode == 400:
            ks = pd
            assert P == TW + ks // 2 and 2 * P <= 256 and 2 <= S <= 5 and nch == (R * P + 127) // 128, key
            assert slot_pos % 8 == 0 and slot_pos >= (R + ks // 2) * P and slot_pos >= nch * 128 + (ks // 2) * (P + 1), key
        else:
            assert P == TW + 2 and P <= 256 and 2 <= S <= 4 and nch == (R * P + 127) // 128 and npad <= 256, key
            assert slot_pos % 8 == 0 and slot_pos >= (R + 2) * P, key
