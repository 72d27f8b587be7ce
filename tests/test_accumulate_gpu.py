"""n13 on the device: ActivePoints.accumulate / resubstitute (tdm_active_accumulate, tdm_active_resubstitute) against the C
oracle of solveSystemF's accumulators (oracle/accumulate_oracle.c) on every case of oracle/accumulate.py: the per-point
outputs and the steps bit for bit, the raw double sums within the worst-case bound of any summation order, the stitch bit
for bit against the oracle's stitch of the device's own raw sums, repeated calls bit for bit, and a closed optimize()-shaped
loop with an accepted and a rejected step whose re-linearisation moves the newest frame's threshold."""
import numpy as np
import pytest

from oracle import accumulate as A
from oracle import linearize as L
from tandem_b200 import ActivePoints, ImagePyramid, TandemError
from tandem_b200._lib import lib

pytestmark = pytest.mark.gpu
PER_POINT = ("hdi", "idepth_hessian")
WORST = {}


def pyramids(win):
    out = []
    for g in win["gray"]:
        p = ImagePyramid(win["w"], win["h"], 1)
        p.build(np.ascontiguousarray(g, np.float32))
        out.append(p)
    return out


class AccDevice:
    """ActivePoints over one window with the oracle's call signature."""

    def __init__(self, win, fp=None):
        self.win = win
        self.fp = fp or pyramids(win)
        self.d = ActivePoints(win["w"], win["h"], max(len(win["host"]), 1), **win["settings"])
        self.load()

    def load(self):
        W = self.win
        self.d.load(W["n_frames"], W["host"], W["u"], W["v"], W["color"], W["weights"], W["res_point"], W["res_target"],
                    W["max_rel_baseline"], W["num_good"])

    def linearize(self, ids, idz, precalc, frame_th, fix):
        return self.d.linearize(self.fp, precalc, frame_th, self.win["calib4"], ids, idz, fix=fix)

    def apply_res(self):
        self.d.apply_res()

    def accumulate(self, inp):
        return self.d.accumulate(**inp)


def check_accumulate(d, o, inp, tag=""):
    """Compares one device accumulate with the oracle's (DOUBLE mode) and returns the device's outputs."""
    b = d.accumulate(inp)
    a = o.accumulate(inp, A.DOUBLE)
    ab = o.accumulate(inp, A.ABS)
    o.accumulate(inp, A.DOUBLE)   # the oracle's state for resubstitute
    for k in PER_POINT:
        assert L.same_bits(b[k], a[k]), (tag, k)
    assert b["n_active"] == a["n_active"], tag
    raw = d.d.get_accumulators()
    for k in ("top_num", "d_num"):
        assert np.array_equal(raw[k], a["raw"][k]), (tag, k)
    bars = A.summation_bars(ab["raw"])
    for k, bar in bars.items():
        err = np.abs(raw[k] - a["raw"][k])
        assert (err <= bar).all(), (tag, k, float(np.max(err - bar)))
        nz = bar > 0
        if nz.any():
            WORST[k] = max(WORST.get(k, 0.0), float(np.max(err[nz] / bar[nz])))
    s = A.stitch(raw, inp, d.win["n_frames"])
    for k in ("H_top", "b_top", "H_sc", "b_sc"):
        assert L.same_bits(b[k], s[k]), (tag, k)
    return b


def run_loop(name, iterations=3):
    """load, linearize, apply, then per iteration: accumulate, solve, resubstitute, step the depths; the second iteration's
    trial is rejected (restore, re-linearize with a moved newest-frame threshold, no apply)."""
    win = A.case(name)
    inp = A.inputs(win)
    o, d = A.AccumulateOracle(win), AccDevice(win)
    st = L.steps(win)
    idz = win["idepth"].copy()
    ids = idz.copy()
    th = win["frame_th"].copy()
    pc = A.precalc(win)
    for be in (o, d):
        be.linearize(ids, idz, pc, th, 0)
        be.apply_res()
    for it in range(iterations):
        b = check_accumulate(d, o, inp, f"{name} it{it}")
        x = A.solve(b)
        sd, so = d.d.resubstitute(x), o.resubstitute(x)
        assert L.same_bits(sd, so), (name, it)
        trial = (ids + sd).astype(np.float32)
        pc_t = A.precalc(win, [[L._small_motion(np.random.default_rng(it * 64 + a * 8 + c), 0.001, 0.001) for c in range(win["n_frames"])]
                               for a in range(win["n_frames"])])
        ra = o.linearize(trial, idz, pc_t, th, 0)
        rb = d.linearize(trial, idz, pc_t, th, 0)
        assert L.compare(rb, ra, exact_energy=False) == [], (name, it)
        if it == 1:   # rejected: restore and re-linearize with another threshold for the newest frame, no apply
            th2 = th.copy()
            th2[-1] = ra["new_frame_energy_th"] * 0.25
            ra = o.linearize(ids, idz, pc, th2, 0)
            rb = d.linearize(ids, idz, pc, th2, 0)
            assert L.compare(rb, ra, exact_energy=False) == []
        else:         # accepted
            for be in (o, d):
                be.apply_res()
            ids, pc = trial, pc_t
            th[-1] = ra["new_frame_energy_th"]
    # linearize(fix) takes the data as apply does
    for be in (o, d):
        be.linearize(ids, idz, pc, th, 1)
    check_accumulate(d, o, inp, f"{name} fix")
    return o, d, inp


@pytest.mark.parametrize("name", list(A.CASES))
def test_closed_loop_equals_oracle(name):
    run_loop(name)
    print("largest error / summation bound:", {k: f"{v:.3g}" for k, v in WORST.items()})


def test_rejected_step_reads_the_taken_data():
    """After a rejected trial the next accumulate reads what the last apply took, not the trial's Jacobians: the trial's
    re-linearisation with a strict newest-frame threshold changes new states, and the accumulate still equals the oracle's
    and the one before the trial."""
    win = A.case("seeded")
    inp = A.inputs(win)
    o, d = A.AccumulateOracle(win), AccDevice(win)
    st = L.steps(win)
    for be in (o, d):
        be.linearize(st[0]["idepth_scaled"], st[0]["idepth_zero_scaled"], A.precalc(win), win["frame_th"], 0)
        be.apply_res()
    before = check_accumulate(d, o, inp)
    th = win["frame_th"].copy()
    th[-1] = 5.0
    r = d.linearize(st[2]["idepth_scaled"], st[2]["idepth_zero_scaled"], st[2]["precalc"], th, 0)
    o.linearize(st[2]["idepth_scaled"], st[2]["idepth_zero_scaled"], st[2]["precalc"], th, 0)
    assert (r["new_state"] != d.d.get_state()["state"]).sum() > 100
    after = check_accumulate(d, o, inp)
    for k in ("H_top", "b_top", "H_sc", "b_sc") + PER_POINT:
        assert L.same_bits(after[k], before[k]), k


def test_repeated_calls_and_no_jacobian_download():
    win = A.case("seeded")
    inp = A.inputs(win)
    d = AccDevice(win)
    st = L.steps(win)
    d.d.linearize(d.fp, A.precalc(win), win["frame_th"], win["calib4"], st[0]["idepth_scaled"], st[0]["idepth_zero_scaled"],
                  jacobians=False)
    d.apply_res()
    r = [d.accumulate(inp) for _ in range(3)]
    x = A.solve(r[0])
    s = [d.d.resubstitute(x) for _ in range(2)]
    for k in ("H_top", "b_top", "H_sc", "b_sc") + PER_POINT:
        assert all(L.same_bits(q[k], r[0][k]) for q in r[1:]), k
    assert L.same_bits(s[0], s[1])
    o = A.AccumulateOracle(win)
    o.linearize(st[0]["idepth_scaled"], st[0]["idepth_zero_scaled"], A.precalc(win), win["frame_th"], 0)
    o.apply_res()
    check_accumulate(d, o, inp)


def test_max_rel_baseline_of_points_without_active_residuals_is_zeroed():
    win = A.case("room")
    win["max_rel_baseline"] = np.full(len(win["host"]), 0.5, np.float32)
    inp = A.inputs(win)
    d = AccDevice(win)
    st = L.steps(win)
    d.linearize(st[0]["idepth_scaled"], st[0]["idepth_zero_scaled"], A.precalc(win), win["frame_th"], 0)
    d.apply_res()
    b = d.accumulate(inp)
    dead = b["hdi"] == 0
    assert dead.sum() > 5
    r = d.linearize(st[0]["idepth_scaled"], st[0]["idepth_zero_scaled"], A.precalc(win), win["frame_th"], 1)
    assert (r["max_rel_baseline"][dead] == 0).all()
    assert (r["max_rel_baseline"][~dead] >= 0.5).all()


def test_zero_residuals_and_reload():
    win = A.case("room")
    fp = pyramids(win)
    n = win["n_frames"]
    d = ActivePoints(win["w"], win["h"], len(win["host"]))
    inp = A.inputs(win)
    pc = A.precalc(win)
    d.load(n, win["host"][:3], win["u"][:3], win["v"][:3], win["color"][:3], win["weights"][:3], [], [])
    d.apply_res()
    i3 = dict(inp, point_prior=inp["point_prior"][:3], point_delta=inp["point_delta"][:3])
    b = d.accumulate(**i3)
    assert b["n_active"] == 0 and (b["hdi"] == 0).all() and (b["idepth_hessian"] == 0).all()
    assert (b["H_sc"] == 0).all() and (b["b_sc"] == 0).all()
    assert np.array_equal(np.diag(b["H_top"])[4:], inp["frame_prior"].ravel())
    assert (d.resubstitute(np.ones(8 * n + 4)) == 0).all()
    # a reload clears the taken data: accumulate needs an apply first
    dev = AccDevice(win, fp=fp)
    with pytest.raises(TandemError):
        dev.d.accumulate(**inp)
    o = A.AccumulateOracle(win)
    for be in (o, dev):
        be.linearize(win["idepth"], win["idepth"], pc, win["frame_th"], 0)
        be.apply_res()
    dev.load()
    with pytest.raises(TandemError):
        dev.d.accumulate(**inp)
    o.load()
    for be in (o, dev):
        be.linearize(win["idepth"], win["idepth"], pc, win["frame_th"], 0)
        be.apply_res()
    check_accumulate(dev, o, inp)


def test_invalid_order_and_input_is_an_error():
    win = A.case("room")
    inp = A.inputs(win)
    d = AccDevice(win)
    n = win["n_frames"]
    with pytest.raises(TandemError):   # no apply since load
        d.accumulate(inp)
    with pytest.raises(TandemError):   # no accumulate
        d.d.resubstitute(np.zeros(8 * n + 4))
    st = L.steps(win)
    d.linearize(st[0]["idepth_scaled"], st[0]["idepth_zero_scaled"], A.precalc(win), win["frame_th"], 0)
    d.apply_res()
    assert lib().tdm_active_accumulate(None, *([None] * 15)) < 0
    assert lib().tdm_active_accumulate(d.d._h, *([None] * 15)) < 0
    assert lib().tdm_active_resubstitute(None, None, None) < 0
    assert lib().tdm_active_resubstitute(d.d._h, None, None) < 0
    assert lib().tdm_active_get_accumulators(None, *([None] * 8)) < 0
    with pytest.raises(ValueError):
        d.d.accumulate(**dict(inp, point_prior=inp["point_prior"][:-1]))
    b = d.accumulate(inp)
    raw0 = d.d.get_accumulators()
    x = A.solve(b)
    s0 = d.d.resubstitute(x)
    # the rejected calls above and below launch nothing: the accumulators, the step and the next accumulate are as before
    for f in (lambda: lib().tdm_active_accumulate(d.d._h, *([None] * 15)), lambda: lib().tdm_active_resubstitute(d.d._h, None, None)):
        assert f() < 0
    raw1 = d.d.get_accumulators()
    assert all(L.same_bits(raw1[k], raw0[k]) for k in raw0)
    assert L.same_bits(d.d.resubstitute(x), s0)
    c = d.accumulate(inp)
    assert all(L.same_bits(c[k], b[k]) for k in ("H_top", "b_top", "H_sc", "b_sc", "hdi", "idepth_hessian"))
    d.apply_res()
    with pytest.raises(TandemError):   # an apply since the accumulate
        d.d.resubstitute(np.zeros(8 * n + 4))
    # caller arrays: page-locked accepted, wrong shape / dtype / read-only rejected
    from tandem_b200._lib import pinned_empty
    dim = 8 * n + 4
    out = dict(H_top=pinned_empty((dim, dim), np.float64), hdi=pinned_empty((len(win["host"]),), np.float32))
    c = d.d.accumulate(**inp, out=out)
    assert c["H_top"] is out["H_top"] and L.same_bits(c["H_top"], b["H_top"]) and L.same_bits(c["hdi"], b["hdi"])
    for bad in (dict(H_top=np.empty((dim, dim - 1))), dict(hdi=np.empty(len(win["host"]))), dict(b_sc=np.empty(dim)[::-1]),
                dict(H_top=np.broadcast_to(0.0, (dim, dim))), dict(energy=np.empty(1))):
        with pytest.raises((ValueError, TypeError)):
            d.d.accumulate(**inp, out=bad)
    # duplicate (point, target) residuals are rejected by accumulate (load still accepts them)
    rp = np.concatenate([win["res_point"], win["res_point"][:1]])
    rt = np.concatenate([win["res_target"], win["res_target"][:1]])
    d.d.load(n, win["host"], win["u"], win["v"], win["color"], win["weights"], rp, rt)
    d.d.apply_res()
    with pytest.raises(TandemError):
        d.accumulate(inp)


def test_shim_runs_accumulate_and_resubstitute(tmp_path):
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "tests", "cpp", "shim_accumulate")
    if not os.path.exists(exe):
        pytest.fail("tests/cpp/shim_accumulate was not built")
    win = A.case("room")
    inp = A.inputs(win)
    n, npt, m = win["n_frames"], len(win["host"]), len(win["res_point"])
    o = A.AccumulateOracle(win)
    pc = A.precalc(win)
    o.linearize(win["idepth"], win["idepth"], pc, win["frame_th"], 0)
    o.apply_res()
    a = o.accumulate(inp, A.DOUBLE)
    x = A.solve(a)
    path = str(tmp_path / "window.bin")
    with open(path, "wb") as f:
        f.write(np.array([win["w"], win["h"], n, npt, m, 1], np.int32).tobytes())
        for g in win["gray"]:
            f.write(np.ascontiguousarray(g, np.float32).tobytes())
        f.write(win["calib4"].tobytes())
        f.write(win["frame_th"].tobytes())
        f.write(win["host"].astype(np.int32).tobytes())
        for k in ("u", "v", "color", "weights", "max_rel_baseline"):
            f.write(win[k].astype(np.float32).tobytes())
        f.write(win["num_good"].astype(np.int32).tobytes())
        f.write(win["res_point"].tobytes())
        f.write(win["res_target"].tobytes())
        f.write(win["idepth"].astype(np.float32).tobytes())
        f.write(win["idepth"].astype(np.float32).tobytes())
        f.write(np.ascontiguousarray(pc, np.float32).tobytes())
        f.write(A._c_layout(inp["ad_host"], n).tobytes())
        f.write(A._c_layout(inp["ad_target"], n).tobytes())
        for k in ("frame_prior", "frame_delta_prior", "c_prior"):
            f.write(np.ascontiguousarray(inp[k], np.float64).tobytes())
        for k in ("c_delta", "point_prior", "point_delta"):
            f.write(np.ascontiguousarray(inp[k], np.float32).tobytes())
        f.write(np.ascontiguousarray(x, np.float64).tobytes())
    out = str(tmp_path / "out.bin")
    r = subprocess.run([exe, path, out], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "shim_accumulate: OK" in r.stdout
    b = open(out, "rb").read()
    dim = 8 * n + 4
    pos = 0

    def take(dtype, k):
        nonlocal pos
        v = np.frombuffer(b, dtype, k, pos)
        pos += v.nbytes
        return v

    got = dict(H_top=take(np.float64, dim * dim).reshape(dim, dim), b_top=take(np.float64, dim),
               H_sc=take(np.float64, dim * dim).reshape(dim, dim), b_sc=take(np.float64, dim), n_active=int(take(np.int32, 1)[0]),
               hdi=take(np.float32, npt), idepth_hessian=take(np.float32, npt), step=take(np.float32, npt))
    assert pos == len(b)
    assert got["n_active"] == a["n_active"]
    for k in ("hdi", "idepth_hessian"):
        assert L.same_bits(got[k], a[k]), k
    assert L.same_bits(got["step"], o.resubstitute(x))
    # the system: within the summation bound of the oracle's double sums, through the stitch (checked bit for bit above)
    for k in ("H_top", "b_top", "H_sc", "b_sc"):
        assert np.allclose(got[k], a[k], rtol=1e-9, atol=1e-6 * np.abs(a[k]).max()), k
