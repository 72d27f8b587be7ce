"""The output-stationary (k_conv_tc MODE 0), up-2 (MODE 3) and stride-2 (k_conv_tc_s2) epilogues carry each fragment row's
tile position from sub-chunk to sub-chunk (conv_tc.cuh FragRows): STEP = 64 * NWG positions on, STEP / P rows and STEP % P
columns, with one wrap.  These windows put that carry at its edges (a row pitch P of at most 8, where a row half wraps more
than one row; a pitch that divides STEP, where the column step is zero; the widest pitch the planners pick here; partial
tiles in W, H and D, where the grid limits cut rows and columns) and check every layer of each forward against its
reference, in both 16-bit precisions, on activation interiors poisoned with NaN."""
import pytest

from oracle import mvsnet_layers as ML

WINDOWS = [  # (V, H, W, depth numbers)
    (3, 64, 96, (8, 16, 8)),
    (2, 64, 992, (8, 8, 8)),
    (2, 96, 128, (16, 24, 8)),
    (2, 96, 736, (8, 8, 8)),
]
FAMILIES = {0: "mode 0", 3: "mode 3", 400: "stride 2"}
STEP = 64 * 4   # every in-scope instantiation runs four consumer warpgroups


def _situations():
    """family -> set of carry situations the windows reach, and family -> widest pitch."""
    seen, widest = {}, {}
    for V, H, W, dn in WINDOWS:
        for _, args in ML.window_launches(V, H, W, dn):
            if args[-1] not in FAMILIES:
                continue
            pl = ML.query_plan(args)
            fam = FAMILIES[args[-1]]
            assert pl["nwg"] == 4, (fam, args, pl)
            D, Hh, Ww = args[3:6]
            s = seen.setdefault(fam, set())
            if pl["P"] <= 8:
                s.add("pitch <= 8")
            if STEP % pl["P"] == 0:
                s.add("pitch divides the step")
            if Ww % pl["TW"]:
                s.add("partial W tile")
            if Hh % pl["R"]:
                s.add("partial H tile")
            if D % pl["DR"]:
                s.add("partial D tile")
            widest[fam] = max(widest.get(fam, 0), pl["P"])
    return seen, widest


def test_windows_reach_the_carry_edges():
    seen, widest = _situations()
    want = {
        "mode 0": {"pitch <= 8", "pitch divides the step", "partial W tile", "partial H tile", "partial D tile"},
        # stride 2: no window of this size splits D; MODE 3: its coarse grid is at least 16 wide and its tiles at least 30
        "stride 2": {"pitch <= 8", "pitch divides the step", "partial W tile", "partial H tile"},
        "mode 3": {"pitch divides the step", "partial W tile", "partial H tile"},
    }
    for fam, w in want.items():
        assert w <= seen.get(fam, set()), (fam, sorted(w - seen.get(fam, set())))
        assert widest[fam] >= 64, (fam, widest[fam])


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["mixed16", "bf16"])
@pytest.mark.parametrize("window", WINDOWS, ids=[f"{w[2]}x{w[1]}v{w[0]}-" + "-".join(map(str, w[3])) for w in WINDOWS])
def test_carry_windows_match_layer_reference(window, precision):
    from test_mvsnet_layers_gpu import _engine, _submit, _synthetic, check_forward

    V, H, W, dn = window
    win = _synthetic(V, H, W)
    m = _engine("abl03_view_aggregation", precision, dn, debug_poison=1)
    _submit(m, win)
    report = []
    check_forward(m, win, "abl03_view_aggregation", precision, dn, {}, f"{W}x{H}v{V}", report)
    assert report
