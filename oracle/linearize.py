"""n12 test infrastructure: ctypes binding of oracle/linearize_oracle.c (DSO's linearizeAll, PointFrameResidual::linearize,
applyRes and setNewFrameEnergyTH restated in C), the windows its pins and the GPU tests run, and the optimize()-shaped call
sequence.  CPU only; no reference code.

A window is the active residuals of one FullSystem::optimize:
- "room": the points n9's C oracle activates on oracle/activate.py's room_640x480_8f case (points the reference's own
  statements made, traced and activated, as tests/test_activate_cpu.py pins them) with their IN residuals, in
  activeResiduals order (frames, then each host's points, then each point's residuals in frame order);
- "seeded": random points of the same 8 frames at the scene's inverse depth off by a few percent, each with a random subset
  of the other frames as targets.
A sequence is linearize(false) -> apply, a perturbed step that is applied, a perturbed step that is rejected (no apply), and
linearize(true); the newest frame's frameEnergyTH is the previous call's new threshold, as setNewFrameEnergyTH leaves it."""
import ctypes
import functools
import os
import subprocess

import numpy as np

from oracle import activate as A
from oracle import trace as T

_HERE = os.path.dirname(os.path.abspath(__file__))
_fp = ctypes.POINTER(ctypes.c_float)
_dp = ctypes.POINTER(ctypes.c_double)
_ip = ctypes.POINTER(ctypes.c_int)

#: util/settings.cpp defaults (tdm_linearize_settings order)
DEFAULTS = dict(huber_th=9.0, outlier_th_sum_component=2500.0, affine_opt_mode_a=1e12, affine_opt_mode_b=1e8,
                frame_energy_th_n=0.7, frame_energy_th_const_weight=0.5, frame_energy_th_fac_median=1.5,
                overall_energy_th_weight=1.0)
IN, OOB, OUTLIER = 0, 1, 2
JACOBIAN_FLOATS = 74
PRECALC = 27


def settings_array(s):
    s = dict(DEFAULTS, **s)
    return np.array([s[k] for k in DEFAULTS], np.float32)


def _lib():
    path = os.path.join(_HERE, "_build", "liblinearize_oracle.so")
    if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(os.path.join(_HERE, "linearize_oracle.c")):
        subprocess.run(["make", "-s", "-C", _HERE, "-f", "linearize_oracle.mk"], check=True)
    return ctypes.CDLL(path)


def _p(a, t=_fp):
    return a.ctypes.data_as(t)


def precalc(poses, calib4, aff, b0, delta=None):
    """n x n x 27 records: PRE_KRKiTll, PRE_KtTll at the current poses (poses, or poses with delta[a][b] applied to the
    host -> target transform), PRE_RTll_0, PRE_tTll_0 at the linearisation point, PRE_aff_mode, PRE_b0_mode."""
    n = len(poses)
    fx, fy, cx, cy = (float(x) for x in calib4)
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])
    Ki = np.linalg.inv(K)
    pc = np.full((n, n, PRECALC), np.nan, np.float32)
    for a in range(n):
        for b in range(n):
            if a == b:
                continue
            T0 = np.linalg.inv(poses[b]) @ poses[a]   # host -> target, FrameFramePrecalc::set's leftToLeft_0
            Tc = T0 if delta is None else delta[a][b] @ T0
            pc[a, b, 0:9] = (K @ Tc[:3, :3] @ Ki).astype(np.float32).ravel()
            pc[a, b, 9:12] = (K @ Tc[:3, 3]).astype(np.float32)
            pc[a, b, 12:21] = T0[:3, :3].astype(np.float32).ravel()
            pc[a, b, 21:24] = T0[:3, 3].astype(np.float32)
            pc[a, b, 24:26] = aff[a][b]
            pc[a, b, 26] = b0[a][b]
    return pc


def _small_motion(rng, rot, trans):
    w = rng.normal(0, rot, 3)
    th = np.linalg.norm(w)
    k = w / th if th > 0 else np.zeros(3)
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    M = np.eye(4)
    M[:3, :3] = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
    M[:3, 3] = rng.normal(0, trans, 3)
    return M


# name -> (source, settings overrides, options)
#   drop_newest: no residual targets the newest frame; oob_points: fraction of points whose idepth is thrown far off in the
#   applied perturbed step (their residuals go OOB there and stay OOB); nan_frame: a frame with NaN patches
VARIANTS = {
    "base": ({}, {}),
    "affine_off": (dict(affine_opt_mode_a=-1.0, affine_opt_mode_b=-1.0), {}),
    "no_newest": ({}, dict(drop_newest=True)),
    "sticky_oob": ({}, dict(oob_points=0.08)),
    "nan_pixels": ({}, dict(nan_frame=3)),
}


@functools.lru_cache(maxsize=None)
def _room_case():
    c = A.case_inputs("room_640x480_8f")
    o = A.build_points(c)
    cf, ci = A.candidates(c, o.pts, "act")
    rec = np.concatenate([A.point_records(o.pts[c["frames"][j]["slot"]], ci[cf == j]) for j in np.unique(cf)])
    r = A.activate(c["w"], c["h"], [f["dI"] for f in c["frames"]], c["precalc"], c["calib4"], cf, rec)
    return c, cf, rec, r


def window(source="room", variant="base", seed=0, n_points=2000):
    """dict(w, h, n_frames, gray [n], dI [n] (level 0 of gray), poses [n], calib4, aff, b0, frame_th, settings, host, u, v, color, weights, idepth,
    max_rel_baseline, num_good, res_point, res_target, options)."""
    c, cf, rec, r = _room_case()
    w, h, n = c["w"], c["h"], len(c["frames"])
    sover, opts = VARIANTS[variant]
    rng = np.random.default_rng(1000 * seed + 7)
    if source == "room":
        made = np.flatnonzero(r["result"] == 1)
        host = cf[made].astype(np.int32)
        u, v = rec[made, 0], rec[made, 1]
        color, weights = rec[made, 5:13], rec[made, 13:21]
        idepth = r["idepth"][made].astype(np.float32)
        res = [(k, f) for k, i in enumerate(made) for f in range(n) if r["state"][i, f] == IN]
    else:
        from oracle.pins_coarse_ref import K4
        from tandem_b200.synthetic import RoomScene
        host = np.sort(rng.integers(0, n - 1, n_points)).astype(np.int32)
        u, v = np.zeros(n_points, np.float32), np.zeros(n_points, np.float32)
        idepth = np.zeros(n_points, np.float32)
        color, weights = np.zeros((n_points, 8), np.float32), np.zeros((n_points, 8), np.float32)
        pat = np.array([[0, -2], [-1, -1], [1, -1], [-2, 0], [0, 0], [2, 0], [-1, 1], [0, 2]])
        for f in range(n - 1):
            sel = np.flatnonzero(host == f)
            dIf = c["frames"][f]["dI"]
            _, z = RoomScene().render(c["frames"][f]["pose"], h, w, *K4(h, w))
            xs, ys = T.select(dIf, len(sel), rng, border=4)
            u[sel], v[sel] = xs, ys
            # the scene's inverse depth, off by a few percent as a solve leaves it
            idepth[sel] = (1.0 / z[ys, xs]) * (1 + rng.normal(0, 0.02, len(sel)))
            px, py = xs[:, None] + pat[:, 0], ys[:, None] + pat[:, 1]
            color[sel] = dIf[py, px, 0]
            g2 = dIf[py, px, 1] ** 2 + dIf[py, px, 2] ** 2
            weights[sel] = np.sqrt(2500.0 / (2500.0 + g2))
        res = []
        for k in range(n_points):
            others = [f for f in range(n) if f != host[k]]
            m = int(rng.integers(1, n))
            res += [(k, f) for f in sorted(rng.choice(others, m, replace=False).tolist())]
    res_point = np.array([a for a, _ in res], np.int32)
    res_target = np.array([b for _, b in res], np.int32)
    if opts.get("drop_newest"):
        keep = res_target != n - 1
        res_point, res_target = res_point[keep], res_target[keep]
    gray = [f["gray"] for f in c["frames"]]
    dI = [np.ascontiguousarray(f["dI"], np.float32) for f in c["frames"]]
    if "nan_frame" in opts:   # NaN grey pixels: their samples (and their neighbours' gradients) are not finite
        from oracle.cpu import FrontOracle
        k = opts["nan_frame"]
        g = gray[k].copy()
        g[rng.integers(3, h - 4, 300), rng.integers(3, w - 4, 300)] = np.nan
        gray[k] = g
        dI[k] = np.ascontiguousarray(T.level0(g, FrontOracle()), np.float32)
    aff = [[(1.0 + 0.01 * (a - b), 0.5 * (b - a)) for b in range(n)] for a in range(n)]
    b0 = [[0.25 * (a - b) for b in range(n)] for a in range(n)]
    frame_th = np.full(n, 12 * 12 * 8, np.float32)
    frame_th[2] = 60.0   # a strict host / target: outliers
    return dict(w=w, h=h, n_frames=n, gray=gray, dI=dI, poses=[f["pose"] for f in c["frames"]], calib4=np.asarray(c["calib4"], np.float32),
                aff=aff, b0=b0, frame_th=frame_th, settings=sover, host=host, u=np.asarray(u, np.float32),
                v=np.asarray(v, np.float32), color=np.ascontiguousarray(color, np.float32),
                weights=np.ascontiguousarray(weights, np.float32), idepth=idepth,
                max_rel_baseline=np.zeros(len(host), np.float32), num_good=np.zeros(len(host), np.int32),
                res_point=res_point, res_target=res_target, options=opts, seed=seed)


def steps(win):
    """The optimize()-shaped sequence: [dict(fix, apply, idepth_scaled, idepth_zero_scaled, precalc)]; frame_th is the
    caller's (the newest frame's entry follows each call's new threshold)."""
    rng = np.random.default_rng(win["seed"] + 11)
    n, idz = win["n_frames"], win["idepth"]
    pc0 = precalc(win["poses"], win["calib4"], win["aff"], win["b0"])
    out = [dict(fix=0, apply=1, idepth_scaled=idz.copy(), idepth_zero_scaled=idz.copy(), precalc=pc0)]
    for k, apply in ((1, 1), (2, 0)):
        ids = (idz * (1 + rng.normal(0, 0.03, len(idz)))).astype(np.float32)
        if k == 1 and win["options"].get("oob_points"):
            bad = rng.random(len(idz)) < win["options"]["oob_points"]
            ids[bad] = -50.0 * np.abs(ids[bad]) - 5.0   # behind the camera: the pattern projections fail
        delta = [[_small_motion(rng, 0.002, 0.003) for _ in range(n)] for _ in range(n)]
        out.append(dict(fix=0, apply=apply, idepth_scaled=ids, idepth_zero_scaled=idz.copy(),
                        precalc=precalc(win["poses"], win["calib4"], win["aff"], win["b0"], delta)))
    out.append(dict(fix=1, apply=0, idepth_scaled=out[1]["idepth_scaled"].copy(), idepth_zero_scaled=idz.copy(),
                    precalc=out[1]["precalc"]))
    return out


class LinearizeOracle:
    """The C oracle over one window: load(), linearize(...) -> dict, apply_res()."""

    def __init__(self, win):
        self.win = win
        self.lib = _lib()
        self.s = settings_array(win["settings"])
        self.load()

    def load(self):
        m, np_ = len(self.win["res_point"]), len(self.win["host"])
        self.state = np.zeros(m, np.int32)
        self.energy = np.zeros(m)
        self.new_state = np.full(m, OUTLIER, np.int32)
        self.new_energy = np.zeros(m)
        self.active = np.zeros(m, np.int32)
        self.max_rel_baseline = self.win["max_rel_baseline"].copy()
        self.num_good = self.win["num_good"].copy()
        assert np_ == len(self.max_rel_baseline)

    def linearize(self, idepth_scaled, idepth_zero_scaled, precalc, frame_th, fix):
        W = self.win
        m, n = len(W["res_point"]), W["n_frames"]
        dI = [np.ascontiguousarray(d, np.float32) for d in W["dI"]]
        arr = (_fp * n)(*[_p(d) for d in dI])
        pc = np.ascontiguousarray(precalc, np.float32)
        th = np.ascontiguousarray(frame_th, np.float32)
        ids = np.ascontiguousarray(idepth_scaled, np.float32)
        idz = np.ascontiguousarray(idepth_zero_scaled, np.float32)
        wo = np.zeros(m)
        center = np.full((m, 3), np.nan, np.float32)
        J = np.zeros((m, JACOBIAN_FLOATS), np.float32)
        removed = np.zeros(m, np.int32)
        new_th = np.zeros(1, np.float32)
        self.lib.linearize_all_oracle.restype = ctypes.c_double
        e = self.lib.linearize_all_oracle(
            W["w"], W["h"], n, arr, _p(pc), _p(th), _p(W["calib4"]), _p(self.s), len(W["host"]), _p(W["host"], _ip),
            _p(W["u"]), _p(W["v"]), _p(W["color"]), _p(W["weights"]), _p(ids), _p(idz), _p(self.max_rel_baseline),
            _p(self.num_good, _ip), m, _p(W["res_point"], _ip), _p(W["res_target"], _ip), int(fix), _p(self.state, _ip),
            _p(self.energy, _dp), _p(self.new_state, _ip), _p(self.new_energy, _dp), _p(wo, _dp), _p(self.active, _ip),
            _p(center), _p(J), _p(removed, _ip), _p(new_th))
        for k, a in (("new_energy", self.new_energy), ("new_energy_with_outlier", wo), ("energy", self.energy)):
            assert (np.isnan(a) | (a.astype(np.float32).astype(np.float64) == a)).all(), k   # every energy is a float value
        out = dict(energy=float(e), new_frame_energy_th=float(new_th[0]), new_state=self.new_state.astype(np.int8),
                   new_energy=self.new_energy.astype(np.float32), new_energy_with_outlier=wo.astype(np.float32),
                   center_projected_to=center, jacobians=J)
        if fix:
            out.update(state=self.state.astype(np.int8), removed=removed.astype(np.uint8),
                       max_rel_baseline=self.max_rel_baseline.copy(), num_good_residuals=self.num_good.copy())
        return out

    def apply_res(self):
        self.lib.apply_res_oracle(len(self.state), _p(self.state, _ip), _p(self.energy, _dp), _p(self.new_state, _ip),
                                  _p(self.new_energy, _dp), _p(self.active, _ip))


def run_sequence(backend, win):
    """Runs steps(win) on a backend with linearize(ids, idz, precalc, frame_th, fix) -> dict and apply_res(); returns
    [(step, outputs, state after the step as dict(state, energy) or None)]."""
    th = win["frame_th"].copy()
    out = []
    for st in steps(win):
        r = backend.linearize(st["idepth_scaled"], st["idepth_zero_scaled"], st["precalc"], th.copy(), st["fix"])
        if st["apply"]:
            backend.apply_res()
        out.append((st, r, th.copy()))
        th[-1] = r["new_frame_energy_th"]
    return out


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return False
    if a.dtype.kind == "f":
        na, nb = np.isnan(a), np.isnan(b)
        return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32 if a.dtype == np.float32 else np.uint64),
                                                          b[~nb].view(np.uint32 if b.dtype == np.float32 else np.uint64))
    return np.array_equal(a, b)


def compare(got, ref, exact_energy=True):
    """[mismatching keys]: every per-residual output bit for bit, the Jacobians where new_state is not OOB, the threshold,
    the fix outputs, and the energy to the last bit (exact_energy) or within 1e-12 relative."""
    bad = []
    for k in ("new_state", "new_energy", "new_energy_with_outlier", "center_projected_to", "state", "removed", "max_rel_baseline",
              "num_good_residuals"):
        if k in ref and not same_bits(np.asarray(got[k]).astype(np.asarray(ref[k]).dtype), ref[k]):
            bad.append(k)
    live = np.asarray(ref["new_state"]) != OOB
    if not same_bits(np.asarray(got["jacobians"])[live], np.asarray(ref["jacobians"])[live]):
        bad.append("jacobians")
    if not same_bits(np.float32(got["new_frame_energy_th"]), np.float32(ref["new_frame_energy_th"])):
        bad.append("new_frame_energy_th")
    e, r = got["energy"], ref["energy"]
    if exact_energy:
        if not same_bits(np.float64(e), np.float64(r)):
            bad.append("energy")
    elif not (e == r or abs(e - r) <= 1e-12 * abs(r)):
        bad.append("energy")
    return bad


DIGESTED = ("new_energy", "new_energy_with_outlier", "center_projected_to", "max_rel_baseline")


def _digest(a):
    import hashlib
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def pin_record(r):
    """The form the pins store one call's outputs in: the energy and threshold, the integer arrays as they are, and SHA-256
    digests of the float arrays' bytes (the Jacobians only of the residuals whose new state is not OOB)."""
    out = dict(energy=np.float64(r["energy"]), new_frame_energy_th=np.float32(r["new_frame_energy_th"]))
    for k in ("new_state", "state", "removed", "num_good_residuals"):
        if k in r:
            out[k] = np.asarray(r[k])
    for k in DIGESTED:
        if k in r:
            out[k + "_digest"] = _digest(np.asarray(r[k], np.float32))
    live = np.asarray(r["new_state"]) != OOB
    out["jacobians_digest"] = _digest(np.asarray(r["jacobians"], np.float32)[live])
    return out


def compare_pins(r, pins, exact_energy=True):
    """[mismatching keys] of pin_record(r) against a stored record."""
    got = pin_record(r)
    bad = [k for k in pins if k != "energy" and k in got and not np.array_equal(got[k], pins[k])]
    bad += [k for k in pins if k not in got]
    e, ref = float(got["energy"]), float(pins["energy"])
    if exact_energy and np.float64(e).tobytes() != np.float64(ref).tobytes():
        bad.append("energy")
    elif not exact_energy and not (e == ref or abs(e - ref) <= 1e-12 * abs(ref)):
        bad.append("energy")
    return bad
