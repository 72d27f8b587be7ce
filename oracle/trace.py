"""n8 test infrastructure: ctypes binding of oracle/trace_oracle.c (DSO's ImmaturePoint constructor and traceOn restated in
C) and the cases its pins and the GPU tests run.  CPU only; no reference code.

A case is a set of host keyframes (each a level-0 pyramid image and the pixels whose immature points it adds) and a sequence
of frames; every frame is traced from every host in turn, so the point state carries over between traces as in DSO's
traceNewCoarse.  The images are RoomScene renders and their level-0 (I, dx, dy) comes from the pinned pyramid definition
(oracle/front_oracle.c, n2)."""
import ctypes
import hashlib
import os
import subprocess

import numpy as np

from oracle.pins_coarse_ref import GRAY_W, K4
from tandem_b200.synthetic import RoomScene, look_at_pose

_HERE = os.path.dirname(os.path.abspath(__file__))
_fp = ctypes.POINTER(ctypes.c_float)
_ip = ctypes.POINTER(ctypes.c_int)

# util/settings.cpp:84-148, in the order of trace_oracle.c's settings array / tdm_trace_settings
DEFAULT_SETTINGS = dict(max_pix_search=0.027, trace_stepsize=1.0, trace_gn_threshold=0.1, trace_extra_slack_on_th=1.2,
                        trace_slack_interval=1.5, trace_min_improvement_factor=2.0, huber_th=9.0, outlier_th=144.0,
                        outlier_th_sum_component=2500.0, overall_energy_th_weight=1.0, min_trace_test_radius=2,
                        trace_gn_iterations=3)
# the twelve return statements of traceOn (ImmaturePoint.cpp:75-414), numbered as trace_oracle.c's trace_one returns them
PATHS = {1: "sticky OOB", 2: "OOB uMin", 3: "OOB uMax", 4: "SKIPPED dist", 5: "OOB uMax coarse", 6: "OOB scale",
         7: "BADCONDITION", 8: "OOB dx/dy not finite", 9: "OUTLIER twice -> OOB", 10: "OUTLIER energy",
         11: "OUTLIER idepth", 12: "GOOD"}
IPS_OOB, IPS_UNINITIALIZED = 1, 5
STATE = ("idepth_min", "idepth_max", "quality", "status", "uv", "interval")
POINT = ("u", "v", "type", "energy_th", "color", "weights", "grad_h")


def digest(a):
    """sha256 of an array's bytes, every NaN written as the same quiet NaN (the pins compare NaN equal to NaN)."""
    a = np.array(a)
    if a.dtype == np.float32:
        a = np.where(np.isnan(a), np.float32(np.nan), a).astype(np.float32)
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:20]


def settings_array(s):
    return np.array([s[k] for k in DEFAULT_SETTINGS], np.float32)


def _lib():
    path = os.path.join(_HERE, "_build", "libtrace_oracle.so")
    if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(os.path.join(_HERE, "trace_oracle.c")):
        subprocess.run(["make", "-s", "-C", _HERE, "-f", "trace_oracle.mk"], check=True)
    lib = ctypes.CDLL(path)
    lib.trace_oracle_add.restype = ctypes.c_int
    return lib


def _p(a, t=_fp):
    return a.ctypes.data_as(t)


class TraceOracle:
    """The point sets of up to 8 hosts, traced on the CPU."""

    def __init__(self, w, h, settings=None):
        self.w, self.h = w, h
        self.s = settings_array(settings or DEFAULT_SETTINGS)
        self._l = _lib()
        self.pts = {}

    def add(self, slot, dI, u, v, typ=None):
        n = len(u)
        u, v = np.ascontiguousarray(u, np.int32), np.ascontiguousarray(v, np.int32)
        typ = np.ones(n, np.float32) if typ is None else np.ascontiguousarray(typ, np.float32)
        dI = np.ascontiguousarray(dI, np.float32)
        o = dict(u=np.zeros(n, np.float32), v=np.zeros(n, np.float32), type=np.zeros(n, np.float32),
                 energy_th=np.zeros(n, np.float32), color=np.zeros((n, 8), np.float32), weights=np.zeros((n, 8), np.float32),
                 grad_h=np.zeros((n, 4), np.float32))
        m = self._l.trace_oracle_add(self.w, self.h, _p(dI), _p(self.s), n, _p(u, _ip), _p(v, _ip), _p(typ), _p(o["u"]),
                                     _p(o["v"]), _p(o["type"]), _p(o["energy_th"]), _p(o["color"]), _p(o["weights"]),
                                     _p(o["grad_h"]))
        o = {k: a[:m] for k, a in o.items()}
        o.update(idepth_min=np.zeros(m, np.float32), idepth_max=np.full(m, np.nan, np.float32),
                 quality=np.full(m, 10000, np.float32), status=np.full(m, IPS_UNINITIALIZED, np.int32),
                 uv=np.zeros((m, 2), np.float32), interval=np.zeros(m, np.float32))
        if slot in self.pts:
            self.pts[slot] = {k: np.concatenate([self.pts[slot][k], o[k]]) for k in o}
        else:
            self.pts[slot] = o
        return m

    def trace(self, dI, per_host):
        """per_host: {slot: (KRKi 9, Kt 3, aff 2)}.  Returns {slot: (path, steps, oob_read)}."""
        dI = np.ascontiguousarray(dI, np.float32)
        diag = {}
        for slot, (K, Kt, aff) in per_host.items():
            p = self.pts[slot]
            n = len(p["u"])
            K, Kt, aff = (np.ascontiguousarray(a, np.float32) for a in (K, Kt, aff))
            path, steps, oob = (np.zeros(n, np.int32) for _ in range(3))
            self._l.trace_oracle_trace(self.w, self.h, _p(dI), _p(self.s), _p(K), _p(Kt), _p(aff), n, _p(p["u"]), _p(p["v"]),
                                       _p(p["color"]), _p(p["weights"]), _p(p["grad_h"]), _p(p["energy_th"]),
                                       _p(p["idepth_min"]), _p(p["idepth_max"]), _p(p["quality"]), _p(p["status"], _ip),
                                       _p(p["uv"]), _p(p["interval"]), _p(path, _ip), _p(steps, _ip), _p(oob, _ip))
            diag[slot] = (path, steps, oob)
        return diag

    def state(self, slot):
        return {k: self.pts[slot][k].copy() for k in STATE}


# ---- cases ----
BASE_EYE, BASE_TARGET = np.array([0.3, 0.0, -0.2]), np.array([2.5, 0.2, 0.5])


def pose(k, jitter=0.0):
    """cam->world of a camera moved sideways by k * 4 cm (and a little forward / up) from the base pose."""
    off = np.array([0.04 * k, 0.012 * k + jitter, 0.015 * k])
    return look_at_pose(BASE_EYE + off, BASE_TARGET + off * 0.5).astype(np.float64)


def level0(bgr_or_gray, front):
    g = bgr_or_gray if bgr_or_gray.ndim == 2 else bgr_or_gray.astype(np.float32) @ GRAY_W
    return front.make_images(g.astype(np.float32), 1)[0][0]


def gray(p, h, w):
    bgr, _ = RoomScene().render(p, h, w, *K4(h, w))
    return bgr.astype(np.float32) @ GRAY_W


def select(dI, n, rng, border=3):
    """n pixels of [border, w-border-1) x [border, h-border-1): most of them where the gradient is strong, some anywhere."""
    h, w = dI.shape[:2]
    g = dI[..., 1] ** 2 + dI[..., 2] ** 2
    ys, xs = np.mgrid[border:h - border - 1, border:w - border - 1]
    ys, xs = ys.ravel(), xs.ravel()
    gg = np.nan_to_num(g[ys, xs], nan=0.0, posinf=0.0)
    strong = np.flatnonzero(gg > np.quantile(gg, 0.8))
    k = min(len(strong), n - n // 5)
    pick = np.concatenate([rng.choice(strong, k, replace=False), rng.choice(len(xs), n - k, replace=False)])
    rng.shuffle(pick)
    return xs[pick].astype(np.int32), ys[pick].astype(np.int32)


def hostToNew(c2w_frame, c2w_host):
    return np.linalg.inv(c2w_frame) @ c2w_host


# name -> (h, w), settings overrides, host pose indices, points per host, frames
#   frame: (pose index, kind) with kind "real" (KRKi/Kt of the poses), "aff" (a brightness offset of 60 on the host side:
#   every residual is large, energy outliers), "scale2" (KRKi and Kt doubled: the same lines, ptpMin[2] out of range) or
#   "rot" (a 15 degree turn: points leave the image)
CASES = {
    "room_320x240_3hosts": ((240, 320), {}, [0, 1, 2], 500,
                            [(3, "real"), (4, "real"), (5, "real"), (6, "real"), (8, "real"), (7, "aff"), (7, "aff"),
                             (9, "real"), (4, "scale2"), (10, "rot")]),
    "room_160x120_nan_hosts": ((120, 160), {}, [0, 2], 400,
                               [(1, "real"), (3, "real"), (-2, "real"), (5, "aff"), (6, "real")]),
    "room_160x120_no_search": ((120, 160), dict(max_pix_search=0.0), [0], 200, [(2, "real"), (3, "real")]),
    "room_2560x1440_cap": ((1440, 2560), {}, [0], 300, [(2, "real"), (3, "real")]),
}


def frame_params(kind, c2w_frame, c2w_host, K4_):
    from oracle.cpu import FrontOracle
    T = hostToNew(c2w_frame, c2w_host)
    if kind == "rot":
        c, s = np.cos(np.radians(15)), np.sin(np.radians(15))
        T = np.array([[c, 0, s, 0], [0, 1, 0, 0], [-s, 0, c, 0], [0, 0, 0, 1]]) @ T
    K, Kt = FrontOracle().krki(T, *K4_)
    aff = np.array([1.0, 60.0 if kind == "aff" else 0.0], np.float32)
    if kind == "scale2":
        K, Kt = K * 2, Kt * 2
    return K, Kt, aff


def case_inputs(name):
    """Returns dict(w, h, settings, hosts=[dict(slot, pose, gray, dI, u, v, type)],
    frames=[dict(gray, dI, params={slot: (K, Kt, aff)})])."""
    from oracle.cpu import FrontOracle
    (h, w), sover, host_poses, npts, frames = CASES[name]
    front = FrontOracle()
    st = dict(DEFAULT_SETTINGS, **sover)
    hosts = []
    for j, k in enumerate(host_poses):
        g = gray(pose(k), h, w)
        rng = np.random.default_rng(1000 * j + h)
        if "nan" in name:   # a few non-finite pixels among the selected ones: the constructor rejects those points
            g[rng.integers(3, h - 4, 40), rng.integers(3, w - 4, 40)] = np.nan
        dI = level0(g, front)
        u, v = select(dI, npts, rng)
        if "nan" in name:
            ys, xs = np.nonzero(~np.isfinite(g[3:h - 4, 3:w - 4]))
            u, v = np.concatenate([u, xs[:20] + 3 + 1]), np.concatenate([v, ys[:20] + 3])
        hosts.append(dict(slot=[0, 3, 7][j], pose=pose(k), gray=g.astype(np.float32), dI=dI, u=u.astype(np.int32), v=v.astype(np.int32),
                          type=rng.choice([1.0, 2.0, 4.0], len(u)).astype(np.float32)))
    out_frames = []
    for k, kind in frames:
        c2w = pose(k)
        g = gray(c2w, h, w).astype(np.float32)
        out_frames.append(dict(gray=g, dI=level0(g, front), params={hh["slot"]: frame_params(kind, c2w, hh["pose"], K4(h, w)) for hh in hosts}))
    return dict(w=w, h=h, settings=st, hosts=hosts, frames=out_frames)


def run_oracle(c):
    """Runs a case on the C oracle: (adds {slot: (count, point fields)}, traces [{slot: (state, path, steps, oob_read)}])."""
    o = TraceOracle(c["w"], c["h"], c["settings"])
    adds = {}
    for hh in c["hosts"]:
        m = o.add(hh["slot"], hh["dI"], hh["u"], hh["v"], hh["type"])
        adds[hh["slot"]] = (m, {k: o.pts[hh["slot"]][k].copy() for k in POINT})
    traces = []
    for f in c["frames"]:
        d = o.trace(f["dI"], f["params"])
        traces.append({s: (o.state(s),) + d[s] for s in d})
    return adds, traces
