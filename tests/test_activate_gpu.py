"""n9 on the device: ImmaturePoints.activate (tdm_immature_activate) equals the C oracle of DSO's optimizeImmaturePoint
(oracle/activate_oracle.c, itself pinned to the reference by tests/test_activate_cpu.py) bit for bit - all four outputs on
every variant of every pin case (and the pins themselves), and on seeded windows of 7 hosts x ~1500 points plus the newest
keyframe at 640x480 - and leaves the set's rows untouched, is ordered behind an asynchronous trace and before a pyramid
rebuild, rejects invalid input without launching, and runs through the C++ shim."""
import os
import subprocess

import numpy as np
import pytest

from oracle import activate as A
from oracle import trace as T
from oracle.pins_coarse_ref import K4
from tandem_b200 import ImagePyramid, ImmaturePoints, TandemError

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_pins_activate.npz")
FIELDS = ("u", "v", "energy_th", "idepth_min", "idepth_max", "color", "weights", "status", "interval", "quality")


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return False
    if a.dtype.kind == "f":
        na, nb = np.isnan(a), np.isnan(b)
        return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))
    return np.array_equal(a, b)


def pyramid(gray):
    h, w = gray.shape
    p = ImagePyramid(w, h, 1)
    p.build(gray)
    return p


def build_device(c, capacity=4096):
    """The case's points on the device, made and traced as build_points makes them on the oracle."""
    d = ImmaturePoints(c["w"], c["h"], capacity)
    fp = [pyramid(f["gray"]) for f in c["frames"]]
    hosts = [(f, p) for f, p in zip(c["frames"], fp) if f["slot"] >= 0]
    for f, p in hosts:
        d.add(f["slot"], p, f["u"], f["v"], f["type"])
    for t in c["traces"]:
        tp = pyramid(t["gray"])
        slots = [f["slot"] for f, _ in hosts]
        d.trace(tp, slots, [t["params"][s][0] for s in slots], [t["params"][s][1] for s in slots],
                [t["params"][s][2] for s in slots], host_pyramids=[p for _, p in hosts])
    for f, p in hosts:
        d.add(f["slot"], p, f["u2"], f["v2"])
    return d, fp


def device_activate(d, c, fp, cf, ci, s):
    return d.activate([f["slot"] for f in c["frames"]], fp, c["precalc"], c["calib4"], cf, ci, **s)


def assert_equal_to_oracle(got, r):
    assert np.array_equal(got["result"], r["result"])
    assert same_bits(got["idepth"], r["idepth"])
    assert np.array_equal(got["res_state"].astype(np.int32), r["state"])
    assert same_bits(got["res_energy"], r["energy"])


def slots_of(c):
    return [f["slot"] for f in c["frames"] if f["slot"] >= 0]


@pytest.mark.parametrize("name", list(A.CASES))
def test_activate_equals_oracle_and_pins(name):
    c = A.case_inputs(name)
    g = np.load(GOLDEN)
    o = A.build_points(c)
    d, fp = build_device(c)
    for s in slots_of(c):
        got = d.get(s)
        for k in FIELDS:
            assert same_bits(got[k], o.pts[s][k]), (s, k)
    for v, (s, cf, ci, r) in enumerate(A.run_oracle(c, o)):
        pre = f"{name}_v{v}_"
        got = device_activate(d, c, fp, cf, ci, s)
        assert_equal_to_oracle(got, r)
        assert np.array_equal(got["result"], g[pre + "result"])
        assert same_bits(np.where(got["result"] == 1, got["idepth"], np.nan), g[pre + "idepth"])
        assert np.array_equal(got["res_state"], g[pre + "state"])
        assert same_bits(got["res_energy"], g[pre + "energy"])


def random_window(seed, n_hosts=7, npts=1500, h=480, w=640):
    """7 hosts at random poses and the newest keyframe; every host's points traced three times."""
    from oracle.cpu import FrontOracle
    rng = np.random.default_rng(seed)
    front = FrontOracle()
    frames = []
    for j in range(n_hosts + 1):
        p = T.pose(rng.uniform(-2, 6), jitter=rng.uniform(-0.05, 0.05))
        g = T.gray(p, h, w).astype(np.float32)
        dI = T.level0(g, front)
        f = dict(slot=j if j < n_hosts else -1, pose=p, gray=g, dI=dI)
        if j < n_hosts:
            u, v = T.select(dI, npts, rng)
            f.update(u=u, v=v, type=np.ones(len(u), np.float32), u2=u[:0], v2=v[:0])
        frames.append(f)
    traces = []
    for _ in range(3):
        c2w = T.pose(rng.uniform(-2, 8), jitter=rng.uniform(-0.05, 0.05))
        g = T.gray(c2w, h, w).astype(np.float32)
        traces.append(dict(gray=g, dI=T.level0(g, front),
                           params={f["slot"]: T.frame_params("real", c2w, f["pose"], K4(h, w)) for f in frames[:n_hosts]}))
    n = n_hosts + 1
    pc = np.full((n, n, 14), np.nan, np.float32)
    for a in range(n):
        for b in range(n):
            if a != b:
                Tm = np.linalg.inv(frames[b]["pose"]) @ frames[a]["pose"]
                pc[a, b, :9] = Tm[:3, :3].astype(np.float32).ravel()
                pc[a, b, 9:12] = Tm[:3, 3].astype(np.float32)
                pc[a, b, 12:] = (rng.uniform(0.9, 1.1), rng.uniform(-5, 5))
    return dict(w=w, h=h, calib4=np.array(K4(h, w), np.float32), frames=frames, traces=traces, precalc=pc,
                variants=[({}, "act")])


@pytest.mark.parametrize("seed", [21, 22])
def test_activate_random_windows_of_seven_hosts(seed):
    c = random_window(seed)
    o = A.build_points(c)
    d, fp = build_device(c)
    (s, cf, ci, r), = A.run_oracle(c, o)
    assert len(cf) > 2000, len(cf)
    got = device_activate(d, c, fp, cf, ci, s)
    assert_equal_to_oracle(got, r)
    assert (r["result"] == 1).sum() > len(cf) // 2
    # a 500-candidate subset in another order of hosts is the same per candidate
    sub = np.sort(np.random.default_rng(seed).choice(len(cf), 500, replace=False))[::-1]
    got = device_activate(d, c, fp, cf[sub], ci[sub], s)
    assert np.array_equal(got["result"], r["result"][sub]) and same_bits(got["res_energy"], r["energy"][sub])


def test_the_set_is_not_changed_and_pyramid_rebuilds_wait():
    c = A.case_inputs("room_331x247_5f")
    d, fp = build_device(c, capacity=700)
    (s, cf, ci, r) = A.run_oracle(c)[0]
    raw = {sl: d.get(sl) for sl in slots_of(c)}
    got = device_activate(d, c, fp, cf, ci, s)
    for sl in raw:
        after = d.get(sl)
        for k in raw[sl]:
            assert raw[sl][k].tobytes() == after[k].tobytes(), (sl, k)
    # rebuild every pyramid with another image right after the call: its result is unchanged, and a call on the
    # restored images gives it again
    for p in fp:
        p.build(c["traces"][0]["gray"])
    assert_equal_to_oracle(got, r)
    for p, f in zip(fp, c["frames"]):
        p.build(f["gray"])
    assert_equal_to_oracle(device_activate(d, c, fp, cf, ci, s), r)


def test_activate_right_behind_an_asynchronous_trace_sees_the_traced_state():
    c = A.case_inputs("room_640x480_8f")
    last = c["traces"][-1]
    c_pre = dict(c, traces=c["traces"][:-1])
    d, fp = build_device(c_pre)
    # the device traced all but the last frame before the fresh points were added; trace the last one now (asynchronous)
    # and activate at once, on the candidates the fully traced oracle state gives
    tp = pyramid(last["gray"])
    slots = slots_of(c)
    o2 = A.build_points(c_pre)
    o2.trace(last["dI"], last["params"])
    (s, cf, ci, r) = A.run_oracle(c, o2)[0]
    d.count(0)   # the set's stream is idle: the trace below is the only work in flight
    d.trace(tp, slots, [last["params"][s][0] for s in slots], [last["params"][s][1] for s in slots],
            [last["params"][s][2] for s in slots])
    got = device_activate(d, c, fp, cf, ci, s)
    assert_equal_to_oracle(got, r)


def test_invalid_input_is_an_error_and_launches_nothing():
    c = A.case_inputs("room_331x247_5f")
    d, fp = build_device(c, capacity=700)
    (s, cf, ci, r) = A.run_oracle(c)[0]
    slots = [f["slot"] for f in c["frames"]]
    other = ImagePyramid(c["w"] + 2, c["h"], 1)
    other.build(np.zeros((c["h"], c["w"] + 2), np.float32))
    pc, cal = c["precalc"], c["calib4"]
    n_slot0 = d.count(slots[0])
    newest = len(slots) - 1

    def act(slots=slots, fp=fp, pc=pc, cf=cf, ci=ci, **kw):
        return d.activate(slots, fp, pc, cal, cf, ci, **kw)

    bad = [
        lambda: act(slots=[], fp=[], pc=np.zeros(0, np.float32), cf=[], ci=[]),       # n_frames 0
        lambda: act(slots=list(range(9)), fp=[fp[0]] * 9, pc=np.zeros((9, 9, 14), np.float32), cf=[], ci=[]),
        lambda: act(slots=[8] + slots[1:]),
        lambda: act(slots=[-2] + slots[1:]),
        lambda: act(slots=[slots[1]] + slots[1:]),                                     # a slot twice
        lambda: act(fp=[other] + fp[1:]),
        lambda: act(fp=[None] + fp[1:]),
        lambda: act(cf=[len(slots)], ci=[0]),
        lambda: act(cf=[-1], ci=[0]),
        lambda: act(cf=[newest], ci=[0]),                                              # the frame without a slot
        lambda: act(cf=[0], ci=[n_slot0]),
        lambda: act(cf=[0], ci=[-1]),
        lambda: act(cf=[0, 0], ci=[3, 3]),                                             # a candidate twice
        lambda: act(gn_iterations=-1),
        lambda: act(gn_iterations=101),
        lambda: act(min_obs=-1),
    ]
    for f in bad:
        with pytest.raises(TandemError):
            f()
    empty = act(cf=[], ci=[])
    assert len(empty["result"]) == 0
    assert_equal_to_oracle(device_activate(d, c, fp, cf, ci, s), r)
    fresh, ffp = build_device(c, capacity=700)
    assert_equal_to_oracle(device_activate(fresh, c, ffp, cf, ci, s), r)


def test_shim_matches_the_python_call(tmp_path):
    exe = os.path.join(ROOT, "tests", "cpp", "shim_activate")
    out = str(tmp_path / "shim_activate.bin")
    r = subprocess.run([exe, out], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "shim_activate: OK" in r.stdout
    b = open(out, "rb").read()
    pos = 0

    def take(dtype, n):
        nonlocal pos
        a = np.frombuffer(b, dtype, n, pos)
        pos += a.nbytes
        return a

    w, h, nf, nh, n, k = take(np.int32, 6)
    grays = take(np.float32, nf * h * w).reshape(nf, h, w)
    slots = take(np.int32, nf)
    uv = take(np.int32, 2 * nh * n).reshape(nh, 2, n)
    K = take(np.float32, 9 * nh).reshape(nh, 9)
    Kt = take(np.float32, 3 * nh).reshape(nh, 3)
    pc = take(np.float32, nf * nf * 14)
    cal = take(np.float32, 4)
    cf, ci = take(np.int32, k), take(np.int32, k)
    res, idepth = take(np.int32, k), take(np.float32, k)
    state, energy = take(np.int8, k * nf).reshape(k, nf), take(np.float32, k * nf).reshape(k, nf)
    assert pos == len(b)
    d = ImmaturePoints(int(w), int(h), 1000)
    fp = [pyramid(np.ascontiguousarray(g)) for g in grays]
    for j in range(nh):
        assert d.add(int(slots[j]), fp[j], uv[j, 0], uv[j, 1]) == n
        d.trace(fp[nf - 1], [int(slots[j])], [K[j]], [Kt[j]], [np.array([1, 0], np.float32)], host_pyramids=[fp[j]])
    got = d.activate(slots, fp, pc, cal, cf, ci)
    assert np.array_equal(got["result"], res) and same_bits(got["idepth"], idepth)
    assert np.array_equal(got["res_state"], state) and same_bits(got["res_energy"], energy)
