"""n9 test infrastructure: ctypes binding of oracle/activate_oracle.c (DSO's optimizeImmaturePoint and linearizeResidual
restated in C) and the cases its pins and the GPU tests run.  CPU only; no reference code.

A case is a window of keyframes in frameHessians order: RoomScene renders at the poses of oracle/trace.py, every frame but
the newest a host whose immature points live in a set slot.  The points are made on the host's level 0, traced into a few
frames (so they carry real depth intervals, as activatePointsMT sees them), and a few fresh points are added behind them
(idepth_max still NaN).  Each case runs under several settings; a run's candidates are every activatable point of every
host (activatePointsMT's canActivate, FullSystem.cpp:757-775, without the distance map) or every point."""
import ctypes
import os
import subprocess

import numpy as np

from oracle import trace as T
from oracle.pins_coarse_ref import K4

_HERE = os.path.dirname(os.path.abspath(__file__))
_fp = ctypes.POINTER(ctypes.c_float)
_ip = ctypes.POINTER(ctypes.c_int)

#: util/settings.cpp:62, 142 and activatePointsMT_Reductor's minObs (FullSystem.cpp:699)
DEFAULTS = dict(min_idepth_h_act=100.0, gn_iterations=3, min_obs=1)
MIN_TRACE_QUALITY = 3.0   # setting_minTraceQuality
#: the return paths of optimizeImmaturePoint, numbered as activate_oracle.c's optimize returns them
PATHS = {1: "0: initial energy not finite", 2: "0: initial Hdd below the threshold", 3: "0: Hdd below the threshold in an iteration",
         4: "0: lastEnergy not finite in an iteration", 5: "-1: idepth not finite", 6: "-1: fewer than minObs IN residuals",
         7: "-1: energyTH not finite", 8: "1: PointHessian"}
#: what a candidate's solve went through (activate_oracle.c F_*)
FLAGS = {1: "accept", 2: "reject", 4: "small-step break", 8: "iterations run out", 16: "OOB on the first linearisation",
         32: "sticky OOB", 64: "leaves the image at pattern index > 0", 128: "outlier clamp, slack 1000",
         256: "outlier clamp, slack 1", 512: "NaN target pixel", 1024: "projection fails"}
IN, OOB, OUTLIER = 0, 1, 2
POINT_RECORD = 21   # u, v, energyTH, idepth_min, idepth_max, color 8, weights 8


def _lib():
    path = os.path.join(_HERE, "_build", "libactivate_oracle.so")
    if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(os.path.join(_HERE, "activate_oracle.c")):
        subprocess.run(["make", "-s", "-C", _HERE, "-f", "activate_oracle.mk"], check=True)
    return ctypes.CDLL(path)


def _p(a, t=_fp):
    return a.ctypes.data_as(t)


def point_records(pts, index):
    """The oracle's point records of points `index` of one slot's fields (TraceOracle.pts[slot] or ImmaturePoints.get)."""
    i = np.asarray(index, np.int64)
    return np.concatenate([np.stack([pts["u"][i], pts["v"][i], pts["energy_th"][i], pts["idepth_min"][i], pts["idepth_max"][i]], 1),
                           pts["color"][i], pts["weights"][i]], 1).astype(np.float32)


def activate(w, h, dIs, precalc, calib4, cand_frame, records, huber=9.0, **settings):
    """activate_oracle over the candidates: dict(result, idepth, state, energy, new_state, new_energy, path, flags)."""
    s = dict(DEFAULTS, **settings)
    n_frames, n = len(dIs), len(cand_frame)
    dIs = [np.ascontiguousarray(d, np.float32) for d in dIs]
    arr = (_fp * n_frames)(*[_p(d) for d in dIs])
    pc = np.ascontiguousarray(precalc, np.float32)
    cal = np.ascontiguousarray(calib4, np.float32)
    cf = np.ascontiguousarray(cand_frame, np.int32)
    rec = np.ascontiguousarray(records, np.float32).reshape(n, POINT_RECORD)
    o = dict(result=np.zeros(n, np.int32), idepth=np.zeros(n, np.float32), state=np.zeros((n, n_frames), np.int32),
             energy=np.zeros((n, n_frames), np.float32), new_state=np.zeros((n, n_frames), np.int32),
             new_energy=np.zeros((n, n_frames), np.float32), path=np.zeros(n, np.int32), flags=np.zeros(n, np.int32))
    _lib().activate_oracle(w, h, n_frames, arr, _p(pc), _p(cal), ctypes.c_float(huber), ctypes.c_float(s["min_idepth_h_act"]),
                           int(s["gn_iterations"]), int(s["min_obs"]), n, _p(cf, _ip), _p(rec), _p(o["result"], _ip),
                           _p(o["idepth"]), _p(o["state"], _ip), _p(o["energy"]), _p(o["new_state"], _ip), _p(o["new_energy"]),
                           _p(o["path"], _ip), _p(o["flags"], _ip))
    return o


def activatable(pts):
    """canActivate of activatePointsMT (FullSystem.cpp:760-775) on a slot's trace state."""
    st = pts["status"]
    return (np.isfinite(pts["idepth_max"]) & np.isin(st, [0, 1, 3, 4]) & (pts["interval"] < 8)
            & (pts["quality"] > MIN_TRACE_QUALITY) & ((pts["idepth_max"] + pts["idepth_min"]) > 0))


# ---- cases ----
def rot_y(deg):
    c, s = np.cos(np.radians(deg)), np.sin(np.radians(deg))
    return np.array([[c, 0, s, 0], [0, 1, 0, 0], [-s, 0, c, 0], [0, 0, 0, 1]])


# name -> (h, w), frames [(pose index, yaw in degrees, slot)] in frameHessians order (the newest last, slot -1), points per
#   host, fresh points per host, trace frames [pose index], PRE_aff_mode overrides {(host frame, target frame): (a, b)},
#   frames with NaN pixels, variants [(settings overrides, "act" | "all")]
#   (1, nan): a non-finite PRE_aff_mode; (1, 20000): every residual above 1000 energyTH; host 6 at (1, 60): outliers
CASES = {
    "room_640x480_8f": ((480, 640), [(0, 0, 0), (1, 0, 1), (2, 0, 2), (3, 0, 3), (4, 0, 4), (5, 0, 5), (6, 0, 6), (7, 0, -1)],
                        250, 20, [7.5, 3.5, -1.0], {(2, 5): (1.0, np.nan), (4, 1): (1.0, 20000.0), **{(6, t): (1.0, 60.0) for t in range(6)}},
                        [], [({}, "act"), (dict(min_obs=2), "act"), (dict(gn_iterations=0), "act"),
                             (dict(min_idepth_h_act=np.nan), "all")]),
    "room_331x247_5f": ((247, 331), [(0, 0, 3), (1.5, 0, 0), (2.5, 12, 7), (-1, 0, 5), (3, 0, -1)], 300, 30, [4.0, 0.5, 2.0], {},
                        [3, 4], [({}, "act"), (dict(min_idepth_h_act=2000.0), "act"), (dict(min_obs=2, gn_iterations=6), "act"),
                                 (dict(min_idepth_h_act=np.nan, gn_iterations=1), "all")]),
}


def case_inputs(name):
    """dict(w, h, calib4, frames=[dict(slot, pose, gray, dI, u, v, type, u2, v2)], traces=[dict(gray, dI, params={slot: (K, Kt,
    aff)})], precalc (n, n, 14), variants)."""
    from oracle.cpu import FrontOracle
    (h, w), fr, npts, nfresh, traces, aff_over, nan_frames, variants = CASES[name]
    front = FrontOracle()
    k4 = K4(h, w)
    frames = []
    for j, (k, yaw, slot) in enumerate(fr):
        p = T.pose(k) @ rot_y(yaw)
        g = T.gray(p, h, w).astype(np.float32)
        rng = np.random.default_rng(100 * j + w)
        if j in nan_frames:   # non-finite target pixels; the host's own points there are rejected by the constructor
            g[rng.integers(3, h - 4, 300), rng.integers(3, w - 4, 300)] = np.nan
        dI = T.level0(g, front)
        f = dict(slot=slot, pose=p, gray=g, dI=dI)
        if slot >= 0:
            u, v = T.select(dI, npts + nfresh, rng)
            f.update(u=u[:npts], v=v[:npts], type=np.ones(npts, np.float32), u2=u[npts:], v2=v[npts:])
        frames.append(f)
    tr = []
    for k in traces:
        c2w = T.pose(k)
        g = T.gray(c2w, h, w).astype(np.float32)
        tr.append(dict(gray=g, dI=T.level0(g, front),
                       params={f["slot"]: T.frame_params("real", c2w, f["pose"], k4) for f in frames if f["slot"] >= 0}))
    n = len(frames)
    pc = np.full((n, n, 14), np.nan, np.float32)   # the diagonal is never read
    for a in range(n):
        for b in range(n):
            if a == b:
                continue
            Tm = np.linalg.inv(frames[b]["pose"]) @ frames[a]["pose"]   # host -> target, FrameFramePrecalc::set's leftToLeft
            pc[a, b, :9] = Tm[:3, :3].astype(np.float32).ravel()
            pc[a, b, 9:12] = Tm[:3, 3].astype(np.float32)
            pc[a, b, 12:] = aff_over.get((a, b), (1.0 + 0.01 * (a - b), 0.5 * (b - a)))
    return dict(w=w, h=h, calib4=np.array(k4, np.float32), frames=frames, traces=tr, precalc=pc, variants=variants)


def build_points(c):
    """Adds and traces every host's points on the C oracle (n8), then adds the fresh ones: the TraceOracle."""
    o = T.TraceOracle(c["w"], c["h"])
    hosts = [f for f in c["frames"] if f["slot"] >= 0]
    for f in hosts:
        o.add(f["slot"], f["dI"], f["u"], f["v"], f["type"])
    for t in c["traces"]:
        o.trace(t["dI"], t["params"])
    for f in hosts:
        o.add(f["slot"], f["dI"], f["u2"], f["v2"])
    return o


def candidates(c, pts, which):
    """(cand_frame, cand_index): the hosts in frame order, each host's points in index order."""
    cf, ci = [], []
    for j, f in enumerate(c["frames"]):
        if f["slot"] < 0:
            continue
        p = pts[f["slot"]]
        idx = np.flatnonzero(activatable(p)) if which == "act" else np.arange(len(p["u"]))
        cf.append(np.full(len(idx), j, np.int32))
        ci.append(idx.astype(np.int32))
    return np.concatenate(cf), np.concatenate(ci)


def run_oracle(c, o=None):
    """Every variant of a case on the C oracle: [(settings, cand_frame, cand_index, outputs)]."""
    o = o or build_points(c)
    out = []
    for sover, which in c["variants"]:
        cf, ci = candidates(c, o.pts, which)
        rec = np.concatenate([point_records(o.pts[c["frames"][j]["slot"]], ci[cf == j]) for j in np.unique(cf)])
        order = np.argsort(cf, kind="stable")
        assert (order == np.arange(len(cf))).all()
        r = activate(c["w"], c["h"], [f["dI"] for f in c["frames"]], c["precalc"], c["calib4"], cf, rec, **sover)
        out.append((dict(DEFAULTS, **sover), cf, ci, r))
    return out
