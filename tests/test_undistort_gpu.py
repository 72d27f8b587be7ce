"""GPU tests of n11 (tdm_undistort_*): DSO's per-frame input on the device - processFrame, the remap, the BGR remap and
makeImages with its gamma weights - against the reference's own statements (tests/golden/reference_pins_undistort.npz) and
the C oracle (oracle/undistort_oracle.c), bit for bit."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import pins_pyramid as PP
from oracle import pixsel as P
from oracle import trace as T
from oracle import undistort as U
from tandem_b200 import CudaCoarseTracker, ImagePyramid, ImmaturePoints, PixelSelector, TandemError, Undistorter, track_pyramid
from tandem_b200._lib import check, lib, pinned_empty

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_pins_undistort.npz")


def undistorter(name, **over):
    c = U.CASES[name]
    kw = dict(U.camera(name), photometric_calibration=c["mode"], use_exposure=c["use_exposure"],
              gamma_weights=c["gamma_weights"])
    kw.update(over)
    return Undistorter(c["w_org"], c["h_org"], c["w"], c["h"], **kw)


def levels_of(p):
    return [p.level(l) for l in range(p.levels)]


def run_case(name, g, pinned=False):
    """Every frame of a case through the device: [(exposure_time, levels, bgr_out)]."""
    c = U.CASES[name]
    u = undistorter(name)
    for k in range(len(c["gammas"])):
        u.set_gamma(g[f"{name}_binv{k}"])
    p = ImagePyramid(c["w"], c["h"], c["levels"])
    out = []
    for k, (exposure, factor, _) in enumerate(c["frames"]):
        gray, bgr = U.frame_inputs(name, k)
        bo = None
        if pinned:
            pg, pb = pinned_empty(gray.shape, np.uint8), pinned_empty(bgr.shape, np.uint8)
            pg[...], pb[...] = gray, bgr
            gray, bgr = pg, pb
            bo = pinned_empty((c["h"], c["w"], 3), np.uint8)
        t, bgr_out = u.frame(gray, exposure, p, factor, bgr=bgr, bgr_out=bo)
        out.append((t, levels_of(p), bgr_out))
    return u, out


@pytest.mark.parametrize("name", list(U.CASES))
def test_frames_equal_reference_pins(name):
    g = np.load(GOLDEN)
    u, out = run_case(name, g)
    G = u.get_gamma()
    assert (G is not None) == bool(g[f"{name}_valid"])
    if G is not None:
        assert np.array_equal(G, g[f"{name}_G"])
    for k, (t, lv, bgr_out) in enumerate(out):
        assert U.frame_mismatches(g, name, k, t, lv[0][0][..., 0], bgr_out, lv) == [], k


@pytest.mark.parametrize("name", ["tum_640x480_mode2", "down_97x75to91x67_mode0", "vignette_zero_passthrough"])
def test_page_locked_buffers_give_the_same_result(name):
    g = np.load(GOLDEN)
    _, a = run_case(name, g)
    _, b = run_case(name, g, pinned=True)
    for (ta, la, ba), (tb, lb, bb) in zip(a, b):
        assert ta == tb and np.array_equal(ba, bb)
        for (da, aa), (db, ab) in zip(la, lb):
            assert np.array_equal(da, db, equal_nan=True) and np.array_equal(aa, ab, equal_nan=True)


def test_out_of_frame_entries_are_zero_and_the_rest_unchanged():
    """Entries whose footprint leaves the raw frame - rows at or below h_org - 1 (what the reference's table builder lets
    through on landscape frames), columns at or beyond w_org - 1, small negative y, NaN - give 0 in grey and BGR; every other
    pixel equals the result of the unmodified table."""
    name = "down_97x75to91x67_mode0"
    c = U.CASES[name]
    cam = U.camera(name)
    rx, ry = cam["remap_x"].copy(), cam["remap_y"].copy()
    inside = np.flatnonzero(rx >= 0)
    bad = inside[::37][:6]
    rx[bad[0]], ry[bad[0]] = 10.5, c["h_org"] - 1          # yyi + 1 == h_org
    rx[bad[1]], ry[bad[1]] = 20.25, c["h_org"] - 0.5
    rx[bad[2]], ry[bad[2]] = c["w_org"] - 1, 30.5          # xxi + 1 == w_org
    rx[bad[3]], ry[bad[3]] = 12.5, -0.5                     # (int)-0.5 == 0, but yy < 0
    rx[bad[4]], ry[bad[4]] = np.nan, 20.0
    rx[bad[5]], ry[bad[5]] = 15.0, np.float32(c["h_org"] - 1) - np.float32(0.001)   # just inside
    gray, bgr = U.frame_inputs(name, 0)
    exposure, factor, _ = c["frames"][0]
    res = []
    for tx, ty in ((cam["remap_x"], cam["remap_y"]), (rx, ry)):
        u = Undistorter(c["w_org"], c["h_org"], c["w"], c["h"], tx, ty, cam["response"], cam["vignette"], c["mode"])
        p = ImagePyramid(c["w"], c["h"], 1)
        _, bo = u.frame(gray, exposure, p, factor, bgr=bgr)
        res.append((p.level(0)[0][..., 0].ravel().copy(), bo.reshape(-1, 3).copy()))
    (g0, b0), (g1, b1) = res
    assert np.all(g1[bad[:5]] == 0) and np.all(b1[bad[:5]] == 0)
    assert g1[bad[5]] != 0
    keep = np.setdiff1d(np.arange(g0.size), bad)
    assert np.array_equal(g0[keep], g1[keep]) and np.array_equal(b0[keep], b1[keep])
    # the oracle states the same rule
    valid, G, vinv = U.create(name)
    img = np.zeros(c["w"] * c["h"], np.float32)
    U._lib().undistort_oracle_frame(U._p(gray, U._up), c["w_org"], c["h_org"], c["w"], c["h"], U._p(rx), U._p(ry), int(valid),
                                    c["mode"], 1, U._p(G), U._p(vinv), U.ctypes.c_float(exposure), U.ctypes.c_float(factor),
                                    U._p(np.zeros(c["w_org"] * c["h_org"], np.float32)), U._p(img))
    assert np.array_equal(img, g1)


@pytest.mark.parametrize("gamma_weights", [0, 1])
def test_passthrough_mode0_equals_pyramid_build(gamma_weights):
    h, w = 480, 640
    gray, _ = U.render(w, h, 2)
    u = Undistorter(w, h, w, h, photometric_calibration=0, gamma_weights=gamma_weights)
    a = ImagePyramid(w, h, 5)
    t, _ = u.frame(gray, 7.0, a)
    b = ImagePyramid(w, h, 5)
    b.build(gray.astype(np.float32))
    assert t == 7.0
    for (da, aa), (db, ab) in zip(levels_of(a), levels_of(b)):
        assert np.array_equal(da, db) and np.array_equal(aa, ab)


@pytest.mark.parametrize("name", [n for n, c in U.CASES.items() if c["select"]])
def test_selection_on_gamma_weighted_pyramid_equals_pins(name):
    g = np.load(GOLDEN)
    c = U.CASES[name]
    w, h = c["w"], c["h"]
    u = undistorter(name)
    for k in range(len(c["gammas"])):
        u.set_gamma(g[f"{name}_binv{k}"])
    p = ImagePyramid(w, h, c["levels"])
    gray, _ = U.frame_inputs(name, 0)
    exposure, factor, _ = c["frames"][0]
    u.frame(gray, exposure, p, factor)
    want = U.pinned_selection_map(g, name, w, h)
    m, r = PixelSelector(w, h).make_maps(p, 1500.0, 1, 1.0)        # no host wait between the two calls
    assert r["num_selected"] == int(g[f"{name}_f0_select_ret"]) and np.array_equal(m, want)
    s = ImmaturePoints(w, h, 8000)
    got = s.make_new_traces(0, PixelSelector(w, h), p, 1500.0)
    uu, vv, tt = P.new_traces(want, w, h)
    keep = np.isin(uu + vv * w, got["u"] + got["v"] * w)
    assert got["result"]["num_selected"] == int(g[f"{name}_f0_select_ret"])
    assert np.array_equal(got["u"], uu[keep]) and np.array_equal(got["v"], vv[keep]) and np.array_equal(got["type"], tt[keep])
    assert keep.sum() > 0.9 * len(uu)


def _quantised_frame(h, w):
    gray_n = PP.scene(h, w)[0]
    return np.clip(np.round(gray_n), 0, 255).astype(np.uint8)


def test_tracker_reads_the_pyramid_without_a_host_wait():
    h, w, levels = PP.H, PP.W, PP.LEVELS
    gray_n, gray_r, depth_r, _ = PP.scene(h, w)
    raw = _quantised_frame(h, w)
    K = PP.intrinsics(w)
    pyr_ref = ImagePyramid(w, h, levels)
    pyr_ref.build(gray_r)
    results = []
    for mode in ("undistort", "undistort_sync", "build"):
        trackers = []
        for l in range(levels):
            t = CudaCoarseTracker(w >> l, h >> l)
            t.init()
            t.setK(w >> l, h >> l, *PP.level_K(l, K))
            t.setReferenceDense(np.eye(4), 1.0, PP.REF_AFF, depth=np.ascontiguousarray(depth_r[::2 ** l, ::2 ** l]), dense_only=True,
                                ref_gray=np.ascontiguousarray(pyr_ref.level(l)[0][..., 0]))
            trackers.append(t)
        pyr = ImagePyramid(w, h, levels)
        pyr.build(np.zeros((h, w), np.float32))
        if mode == "build":
            pyr.build(raw.astype(np.float32))
        else:
            u = Undistorter(w, h, w, h, photometric_calibration=0)
            u.frame(raw, 1.0, pyr)
            if mode == "undistort_sync":
                pyr.level(0)
        for l, t in enumerate(trackers):
            t.setNewFromPyramid(pyr, l)
        r = track_pyramid(trackers, np.eye(4), PP.REF_AFF, 1.05, affine_opt_mode_a=1e12, affine_opt_mode_b=1e8)
        results.append(r)
    for r in results[1:]:
        assert np.array_equal(r["refToNew"], results[0]["refToNew"]) and np.array_equal(r["aff"], results[0]["aff"])
        assert np.array_equal(r["last_residuals"], results[0]["last_residuals"], equal_nan=True)
        assert np.array_equal(r["iterations"], results[0]["iterations"])


def test_trace_reads_the_pyramid_without_a_host_wait():
    c = T.case_inputs("room_320x240_3hosts")
    h, w = c["h"], c["w"]
    frame = c["frames"][0]
    raw = np.clip(np.round(frame["gray"]), 0, 255).astype(np.uint8)
    slots = [hh["slot"] for hh in c["hosts"]]
    results = []
    for mode in ("undistort", "undistort_sync", "build"):
        d = ImmaturePoints(w, h, 4000)
        hp = []
        for hh in c["hosts"]:
            p = ImagePyramid(w, h, 1)
            p.build(hh["gray"])
            hp.append(p)
            d.add(hh["slot"], p, hh["u"], hh["v"], hh["type"])
        fp = ImagePyramid(w, h, 1)
        if mode == "build":
            fp.build(raw.astype(np.float32))
        else:
            u = Undistorter(w, h, w, h, photometric_calibration=0)
            u.frame(raw, 1.0, fp)
            if mode == "undistort_sync":
                fp.level(0)
        d.trace(fp, slots, [frame["params"][s][0] for s in slots], [frame["params"][s][1] for s in slots],
                [frame["params"][s][2] for s in slots], host_pyramids=hp)
        results.append({s: d.get(s) for s in slots})
    for r in results[1:]:
        for s in slots:
            for k, v in results[0][s].items():
                assert np.array_equal(np.asarray(r[s][k]), np.asarray(v), equal_nan=True), (s, k)


def test_two_undistorters_on_one_device():
    g = np.load(GOLDEN)
    names = ("down_97x75to91x67_mode0", "up_91x67to103x79_noexp")
    us = {}
    for n in names:
        us[n] = undistorter(n)
        for k in range(len(U.CASES[n]["gammas"])):
            us[n].set_gamma(g[f"{n}_binv{k}"])
    pyrs = {n: ImagePyramid(U.CASES[n]["w"], U.CASES[n]["h"], U.CASES[n]["levels"]) for n in names}
    for k in range(2):   # interleaved, no waits between the calls
        outs = {}
        for n in names:
            exposure, factor, _ = U.CASES[n]["frames"][k]
            gray, bgr = U.frame_inputs(n, k)
            outs[n] = us[n].frame(gray, exposure, pyrs[n], factor)
        for n in names:
            lv = levels_of(pyrs[n])
            assert U.frame_mismatches(g, n, k, outs[n][0], lv[0][0][..., 0], None, lv) == [], (n, k)


def test_one_undistorter_feeds_two_pyramids():
    g = np.load(GOLDEN)
    name = "up_91x67to103x79_noexp"
    c = U.CASES[name]
    u = undistorter(name)
    for k in range(len(c["gammas"])):
        u.set_gamma(g[f"{name}_binv{k}"])
    ps = [ImagePyramid(c["w"], c["h"], c["levels"]) for _ in range(2)]
    ts = []
    for k, p in enumerate(ps):
        exposure, factor, _ = c["frames"][k]
        ts.append(u.frame(U.frame_inputs(name, k)[0], exposure, p, factor)[0])
    for k, p in enumerate(ps):
        lv = levels_of(p)
        assert U.frame_mismatches(g, name, k, ts[k], lv[0][0][..., 0], None, lv) == [], k


def test_invalid_input_is_an_error():
    with pytest.raises(TandemError, match="passthrough"):
        Undistorter(64, 48, 60, 48)
    rx = np.zeros(60 * 48, np.float32)
    with pytest.raises(TandemError, match="both remap tables"):
        Undistorter(64, 48, 60, 48, remap_x=rx, remap_y=None)
    with pytest.raises(TandemError, match="n_response"):
        Undistorter(64, 48, 64, 48, response=np.arange(255, dtype=np.float32))
    with pytest.raises(TandemError, match="photometric_calibration"):
        Undistorter(64, 48, 64, 48, photometric_calibration=3)
    with pytest.raises(TandemError, match="positive"):
        Undistorter(0, 48, 0, 48)
    u = Undistorter(64, 48, 64, 48, photometric_calibration=0)
    assert u.get_gamma() is None
    u.set_gamma(None)   # no-op, as setGammaFunction(0)
    gray = np.zeros((48, 64), np.uint8)
    with pytest.raises(TandemError, match="size"):
        u.frame(gray, 1.0, ImagePyramid(32, 48, 1))
    p = ImagePyramid(64, 48, 2)
    with pytest.raises(TandemError, match="null"):
        check(lib().tdm_undistort_frame(u._h, None, 1.0, 1.0, p._h, None, None, None))
    with pytest.raises(TandemError, match="bgr"):
        check(lib().tdm_undistort_frame(u._h, gray.ctypes.data, 1.0, 1.0, p._h, None, gray.ctypes.data, None))
    with pytest.raises(TandemError, match="null"):
        check(lib().tdm_undistort_frame(u._h, gray.ctypes.data, 1.0, 1.0, None, None, None, None))
    with pytest.raises(TandemError, match="null"):
        check(lib().tdm_undistort_create(None, 0, ctypes.byref(ctypes.c_void_p())))
    # the handle still works after the errors
    t, _ = u.frame(gray, 2.0, p)
    assert t == 2.0 and np.array_equal(p.level(0)[0][..., 0], np.zeros((48, 64), np.float32))


def test_shim_matches_the_python_call():
    exe = os.path.join(ROOT, "tests", "cpp", "shim_undistort")
    name = "down_97x75to91x67_mode0"
    g = np.load(GOLDEN)
    c = U.CASES[name]
    cam = U.camera(name)
    gray, bgr = U.frame_inputs(name, 0)
    exposure, factor, _ = c["frames"][0]
    tmp = tempfile.mkdtemp()
    files = dict(remap_x=cam["remap_x"], remap_y=cam["remap_y"], response=cam["response"], vignette=cam["vignette"],
                 binv0=g[f"{name}_binv0"], binv1=g[f"{name}_binv1"], gray=gray, bgr=bgr)
    for k, a in files.items():
        np.ascontiguousarray(a).tofile(os.path.join(tmp, k + ".bin"))
    r = subprocess.run([exe, tmp, str(c["w_org"]), str(c["h_org"]), str(c["w"]), str(c["h"]), str(c["mode"]), str(exposure),
                        str(factor), str(c["levels"])], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    lv = []
    for l in range(c["levels"]):
        wl, hl = c["w"] >> l, c["h"] >> l
        lv.append((np.fromfile(os.path.join(tmp, f"dI{l}.bin"), np.float32).reshape(hl, wl, 3),
                   np.fromfile(os.path.join(tmp, f"ag{l}.bin"), np.float32).reshape(hl, wl)))
    bo = np.fromfile(os.path.join(tmp, "bgr_out.bin"), np.uint8).reshape(c["h"], c["w"], 3)
    t = float(r.stdout.split("exposure_time")[1].split()[0])
    assert U.frame_mismatches(g, name, 0, t, lv[0][0][..., 0], bo, lv) == []
