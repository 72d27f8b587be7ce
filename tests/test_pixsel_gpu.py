"""n10 on the device: PixelSelector.make_maps (tdm_selector_make_maps) equals the C oracle of DSO's makeMaps
(oracle/pixsel_oracle.c, itself pinned to the reference by tests/test_pixsel_cpu.py) bit for bit - the whole map, the
return value, n2 / n3 / n4, the potentials and the re-selection flag - on every call of every pin case (and the pins
themselves) and on seeded RoomScene keyframe sequences at 640x480 and 752x480.  ImmaturePoints.make_new_traces
(tdm_immature_make_new_traces) leaves a slot exactly as `add` with the oracle's kept pixels does, behind the slot's points.
Identical calls give identical results; the call is ordered behind an asynchronous trace and before a pyramid rebuild;
invalid input is an error that launches nothing, and a capacity overflow leaves the set and the potential unchanged; the C++
shim runs the same calls."""
import os
import subprocess

import numpy as np
import pytest

from oracle import pixsel as P
from oracle import trace as T
from oracle.cpu import FrontOracle
from tandem_b200 import ImagePyramid, ImmaturePoints, PixelSelector, TandemError
from tandem_b200._lib import check, lib

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_pins_pixsel.npz")
POINT_FIELDS = ("u", "v", "type", "energy_th", "color", "weights", "grad_h", "idepth_min", "idepth_max", "quality", "status",
                "uv", "interval")


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return False
    if a.dtype.kind == "f":
        na, nb = np.isnan(a), np.isnan(b)
        return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))
    return np.array_equal(a, b)


def pyramid(gray, levels=3):
    h, w = gray.shape
    p = ImagePyramid(w, h, levels)
    p.build(np.ascontiguousarray(gray, np.float32))
    return p


def assert_equal_to_oracle(m, r, o):
    assert same_bits(m, o["map"])
    assert r["num_selected"] == o["ret"]
    assert [r["n2"], r["n3"], r["n4"]] == o["n"].tolist()
    assert r["potential_used"] == o["pot_used"] and r["potential_after"] == o["pot_after"]
    assert r["reselected"] == o["reselected"]
    assert r["nonuniform_cells"] == o["nonuniform"]


class DeviceSelectors:
    """One device selector per settings of a case, the potential carried from call to call as the oracle's is."""

    def __init__(self, w, h):
        self.w, self.h, self.sel, self.potential = w, h, {}, 3

    def make_maps(self, pyr, c):
        key = tuple(sorted(c["settings"].items()))
        if key not in self.sel:
            self.sel[key] = PixelSelector(self.w, self.h, **c["settings"])
        s = self.sel[key]
        s.potential = c["pot"] if c["pot"] is not None else self.potential
        m, r = s.make_maps(pyr, c["density"], c["rec"], c["th"])
        assert s.potential == r["potential_after"]
        self.potential = s.potential
        return m, r


@pytest.mark.parametrize("name", list(P.CASES))
def test_make_maps_equals_oracle_and_pins(name):
    (h, w), calls = P.CASES[name]
    g = np.load(GOLDEN)
    dev = DeviceSelectors(w, h)
    for i, (c, img, o) in enumerate(zip(calls, P.case_images(name), P.run_oracle(name))):
        m, r = dev.make_maps(pyramid(img), c)
        assert_equal_to_oracle(m, r, o)
        pre = f"{name}_{i}_"
        idx, typ = P.selected(m)
        assert np.array_equal(idx, g[pre + "index"]) and np.array_equal(typ, g[pre + "type"]), i
        assert r["num_selected"] == int(g[pre + "ret"]) and [r["n2"], r["n3"], r["n4"]] == g[pre + "n"].tolist(), i
        assert r["potential_after"] == int(g[pre + "pot_after"]) and r["potential_used"] == int(g[pre + "pot_used"]), i


def keyframes(seed, n, h, w):
    rng = np.random.default_rng(seed)
    ks = np.sort(rng.uniform(0, 12, n))
    return [T.gray(T.pose(k, jitter=rng.uniform(-0.02, 0.02)), h, w).astype(np.float32) for k in ks]


@pytest.mark.parametrize("seed,hw", [(0, (480, 640)), (1, (480, 640)), (2, (480, 752))])
def test_make_maps_on_keyframe_sequences(seed, hw):
    h, w = hw
    o = P.PixelSelectorOracle(w, h)
    sel = PixelSelector(w, h)
    for img in keyframes(seed, 6, h, w):
        ro = o.make_maps(img, 1500.0)
        m, r = sel.make_maps(pyramid(img), 1500.0)
        assert_equal_to_oracle(m, r, ro)
        assert sel.potential == o.potential


def oracle_new_traces(o, img, density=1500.0):
    ro = o.make_maps(img, density)
    return ro, P.new_traces(ro["map"], o.w, o.h)


@pytest.mark.parametrize("seed,hw", [(3, (480, 640)), (4, (247, 331))])
def test_make_new_traces_equals_add_of_the_oracle_pixels(seed, hw):
    h, w = hw
    o = P.PixelSelectorOracle(w, h)
    sel = PixelSelector(w, h)
    d = ImmaturePoints(w, h, 6000)
    ref = ImmaturePoints(w, h, 6000)
    imgs = keyframes(seed, 5, h, w)
    # pre-existing points in the slot: the new ones go behind them
    p0 = pyramid(imgs[0])
    u0, v0 = T.select(T.level0(imgs[0], FrontOracle()), 300, np.random.default_rng(seed))
    assert d.add(5, p0, u0, v0) == ref.add(5, p0, u0, v0)
    for img in imgs[1:]:
        ro, (u, v, t) = oracle_new_traces(o, img)
        p = pyramid(img)
        before = d.count(5)
        got = d.make_new_traces(5, sel, p, 1500.0)
        n_ref = ref.add(5, p, u, v, t)
        r = got["result"]
        assert r["num_selected"] == ro["ret"] and [r["n2"], r["n3"], r["n4"]] == ro["n"].tolist()
        assert r["potential_after"] == ro["pot_after"] == sel.potential
        assert got["n_added"] == n_ref == d.count(5) - before
        a, b = d.get(5), ref.get(5)
        for k in POINT_FIELDS:
            assert same_bits(a[k], b[k]), k
        assert np.array_equal(got["u"], a["u"][before:].astype(np.int32))
        assert np.array_equal(got["v"], a["v"][before:].astype(np.int32))
        assert same_bits(got["type"], a["type"][before:])
        assert set(np.unique(got["type"]).tolist()) <= {1.0, 2.0, 4.0}


def test_two_identical_calls_give_identical_results():
    h, w = 480, 752
    img = keyframes(7, 1, h, w)[0]
    p = pyramid(img)
    outs = []
    for _ in range(2):
        sel = PixelSelector(w, h)
        d = ImmaturePoints(w, h, 4000)
        m, r = sel.make_maps(p, 1500.0)
        sel.potential = 3
        t = d.make_new_traces(1, sel, p, 1500.0)
        outs.append((m, r, t, d.get(1)))
    (m0, r0, t0, g0), (m1, r1, t1, g1) = outs
    assert same_bits(m0, m1) and r0 == r1 and t0["result"] == t1["result"]
    for k in ("u", "v", "type"):
        assert same_bits(t0[k], t1[k])
    for k in POINT_FIELDS:
        assert same_bits(g0[k], g1[k]), k


def test_ordered_behind_a_trace_and_before_a_rebuild():
    c = T.case_inputs("room_320x240_3hosts")
    h, w = c["h"], c["w"]
    hosts = c["hosts"]
    frame = c["frames"][0]
    img = keyframes(9, 1, h, w)[0]
    o = P.PixelSelectorOracle(w, h)
    ro, (u, v, t) = oracle_new_traces(o, img)
    results = []
    for sync_first in (True, False):
        d = ImmaturePoints(w, h, 4000)
        hp = [pyramid(hh["gray"], 1) for hh in hosts]
        for hh, p in zip(hosts, hp):
            d.add(hh["slot"], p, hh["u"], hh["v"], hh["type"])
        fp = pyramid(frame["gray"], 1)
        slots = [hh["slot"] for hh in hosts]
        d.trace(fp, slots, [frame["params"][s][0] for s in slots], [frame["params"][s][1] for s in slots],
                [frame["params"][s][2] for s in slots], host_pyramids=hp)
        if sync_first:
            d.count(0)
            d.get(slots[0])
        p = pyramid(img)
        sel = PixelSelector(w, h)
        got = d.make_new_traces(1, sel, p, 1500.0)
        # rebuild the pyramid at once: the selection already made is the one of `img`
        p.build(np.zeros((h, w), np.float32))
        results.append((got, {s: d.get(s) for s in slots + [1]}))
        assert got["result"]["num_selected"] == ro["ret"]
    ref = ImmaturePoints(w, h, 4000)
    assert ref.add(1, pyramid(img), u, v, t) == results[0][0]["n_added"]
    want = ref.get(1)
    for k in POINT_FIELDS:
        assert same_bits(results[0][1][1][k], want[k]), k
    (g0, s0), (g1, s1) = results
    assert g0["result"] == g1["result"] and same_bits(g0["u"], g1["u"]) and same_bits(g0["v"], g1["v"])
    for s in s0:
        for k in POINT_FIELDS:
            assert same_bits(s0[s][k], s1[s][k]), (s, k)
    # after the rebuild the same pyramid selects from the flat image: nothing
    sel = PixelSelector(w, h)
    m, r = sel.make_maps(p, 1500.0)
    assert r["num_selected"] == 0 and not m.any()


def test_invalid_input_is_an_error_and_launches_nothing():
    h, w = 247, 331
    img = keyframes(11, 1, h, w)[0]
    p = pyramid(img)
    sel = PixelSelector(w, h)
    sel.potential = 5
    d = ImmaturePoints(w, h, 4000)
    d.add(0, p, [50, 60], [50, 60])
    two = pyramid(img, 2)
    other = pyramid(np.zeros((h, w + 2), np.float32))
    wrong_set = ImmaturePoints(w + 2, h, 100)
    bad = [
        lambda: sel.make_maps(two),
        lambda: sel.make_maps(other),
        lambda: sel.make_maps(p, -1.0),
        lambda: sel.make_maps(p, float("nan")),
        lambda: sel.make_maps(p, float("inf")),
        lambda: sel.make_maps(p, 1500.0, -1),
        lambda: sel.make_maps(p, 1500.0, 17),
        lambda: sel.make_maps(p, 1500.0, 1, 0.0),
        lambda: sel.make_maps(p, 1500.0, 1, -1.0),
        lambda: sel.make_maps(p, 1500.0, 1, float("nan")),
        lambda: setattr(sel, "potential", 0),
        lambda: d.make_new_traces(8, sel, p),
        lambda: d.make_new_traces(-1, sel, p),
        lambda: d.make_new_traces(0, sel, two),
        lambda: d.make_new_traces(0, sel, other),
        lambda: d.make_new_traces(0, sel, p, -5.0),
        lambda: wrong_set.make_new_traces(0, sel, other),
        lambda: check(lib().tdm_selector_make_maps(None, p._h, 1500.0, 1, 1.0, None, None)),
        lambda: check(lib().tdm_selector_make_maps(sel._h, None, 1500.0, 1, 1.0, None, None)),
        lambda: check(lib().tdm_immature_make_new_traces(d._h, 0, None, p._h, 1500.0, None, None, None, None, None)),
        lambda: PixelSelector(31, 100),
        lambda: PixelSelector(100, 31),
        lambda: PixelSelector(w, h, min_grad_hist_cut=1.0),
        lambda: PixelSelector(w, h, select_direction_distribution=2),
    ]
    for f in bad:
        with pytest.raises(TandemError):
            f()
    assert sel.potential == 5 and d.count(0) == 2
    o = P.PixelSelectorOracle(w, h)
    o.potential = 5
    assert_equal_to_oracle(*sel.make_maps(p, 1500.0), o.make_maps(img, 1500.0))


def test_capacity_overflow_leaves_the_set_and_the_potential_unchanged():
    h, w = 480, 640
    img = keyframes(13, 1, h, w)[0]
    p = pyramid(img)
    sel = PixelSelector(w, h)
    d = ImmaturePoints(w, h, 1000)
    d.add(2, p, [100, 120, 140], [100, 100, 100])
    before = d.get(2)
    with pytest.raises(TandemError):
        d.make_new_traces(2, sel, p, 1500.0)
    assert sel.potential == 3 and d.count(2) == 3
    after = d.get(2)
    for k in POINT_FIELDS:
        assert same_bits(before[k], after[k]), k
    # the same call with room for the points succeeds and matches the oracle
    o = P.PixelSelectorOracle(w, h)
    ro, (u, v, t) = oracle_new_traces(o, img)
    big = ImmaturePoints(w, h, 4000)
    got = big.make_new_traces(2, sel, p, 1500.0)
    assert got["result"]["num_selected"] == ro["ret"] and sel.potential == ro["pot_after"]


def test_shim_matches_the_python_call(tmp_path):
    exe = os.path.join(ROOT, "tests", "cpp", "shim_pixsel")
    out = str(tmp_path / "shim_pixsel.bin")
    r = subprocess.run([exe, out], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "shim_pixsel:" in r.stdout
    b = open(out, "rb").read()
    pos = 0

    def take(dtype, n):
        nonlocal pos
        a = np.frombuffer(b, dtype, n, pos)
        pos += a.nbytes
        return a

    w, h = (int(x) for x in take(np.int32, 2))
    gray = take(np.float32, w * h).reshape(h, w)
    p = pyramid(gray)
    sel = PixelSelector(w, h)
    o = P.PixelSelectorOracle(w, h)
    for density in (300.0, 600.0):
        n, pot = take(np.int32, 2)
        m = take(np.float32, w * h).reshape(h, w)
        mp, rp = sel.make_maps(p, density)
        ro = o.make_maps(gray, density)
        assert same_bits(m, mp) and n == rp["num_selected"] == ro["ret"] and pot == sel.potential == ro["pot_after"]
        assert same_bits(m, ro["map"])
    n, pot = (int(x) for x in take(np.int32, 2))
    u, v, t = take(np.int32, n), take(np.int32, n), take(np.float32, n)
    assert pos == len(b)
    sel2 = PixelSelector(w, h)
    sel2.potential = 2
    d = ImmaturePoints(w, h, 4000)
    got = d.make_new_traces(2, sel2, p, 500.0)
    assert got["n_added"] == n and pot == sel2.potential
    assert np.array_equal(got["u"], u) and np.array_equal(got["v"], v) and same_bits(got["type"], t)
