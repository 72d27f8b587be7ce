"""n13 test infrastructure: ctypes binding of oracle/accumulate_oracle.c (DSO's takeDataF, the top and Schur-complement
accumulators, their stitch and resubstituteF_MT restated in C), the solveSystemF inputs of a window (the adjoints with
setAdjointsF's formula, frame and calibration priors, the points' priorF and deltaF), and the optimize()-shaped sequence the
GPU tests and the benchmark run.  CPU only; no reference code.

A case is one of oracle/linearize.py's windows, optionally cut to a subset of its frames, or with the linearisation-point
translation of one host / target pair set to zero (its residuals' Jpdd are 0, so a point whose only active residuals go
there hits the 1e-10 clamp of its depth Hessian)."""
import ctypes
import functools
import os
import subprocess

import numpy as np

from oracle import linearize as L

_HERE = os.path.dirname(os.path.abspath(__file__))
_fp = ctypes.POINTER(ctypes.c_float)
_dp = ctypes.POINTER(ctypes.c_double)
_ip = ctypes.POINTER(ctypes.c_int)
TIERS, DOUBLE, ABS = 0, 1, 2
RAW_KEYS = ("top", "top_num", "acc_e", "acc_eb", "acc_d", "d_num", "hcc", "bc")


@functools.lru_cache(maxsize=None)
def _lib():
    path = os.path.join(_HERE, "_build", "libaccumulate_oracle.so")
    if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(os.path.join(_HERE, "accumulate_oracle.c")):
        subprocess.run(["make", "-s", "-C", _HERE, "-f", "accumulate_oracle.mk"], check=True)
    return ctypes.CDLL(path)


def _p(a, t=_fp):
    return a.ctypes.data_as(t)


def subset(win, frames):
    """The window cut to the given frames: their points and the residuals between them, re-indexed."""
    frames = list(frames)
    fmap = -np.ones(win["n_frames"], np.int32)
    fmap[frames] = np.arange(len(frames))
    keep_p = np.flatnonzero(fmap[win["host"]] >= 0)
    pmap = -np.ones(len(win["host"]), np.int32)
    pmap[keep_p] = np.arange(len(keep_p))
    keep_r = (pmap[win["res_point"]] >= 0) & (fmap[win["res_target"]] >= 0)
    w = dict(win)
    w.update(n_frames=len(frames), gray=[win["gray"][f] for f in frames], dI=[win["dI"][f] for f in frames],
             poses=[win["poses"][f] for f in frames], aff=[[win["aff"][a][b] for b in frames] for a in frames],
             b0=[[win["b0"][a][b] for b in frames] for a in frames], frame_th=win["frame_th"][frames].copy(),
             host=fmap[win["host"][keep_p]].astype(np.int32))
    for k in ("u", "v", "color", "weights", "idepth", "max_rel_baseline", "num_good"):
        w[k] = np.ascontiguousarray(win[k][keep_p])
    w["res_point"] = pmap[win["res_point"][keep_r]].astype(np.int32)
    w["res_target"] = fmap[win["res_target"][keep_r]].astype(np.int32)
    return w


#: name -> (oracle/linearize.py source, variant, options); frames: a subset of the window's frames; clamp: the target frame
#: whose linearisation-point translation from every host is zero
CASES = {
    "room": ("room", "base", {}),
    "room_affine_off": ("room", "affine_off", {}),
    "room_no_newest": ("room", "no_newest", {}),
    "room_sticky_oob": ("room", "sticky_oob", {}),
    "seeded": ("seeded", "base", {}),
    "seeded_clamp": ("seeded", "base", dict(clamp=6)),
    "seeded_n2": ("seeded", "base", dict(frames=(2, 3))),
}


def case(name):
    source, variant, opts = CASES[name]
    win = L.window(source, variant)
    if "frames" in opts:
        win = subset(win, opts["frames"])
    win["clamp"] = opts.get("clamp")
    return win


def precalc(win, delta=None):
    pc = L.precalc(win["poses"], win["calib4"], win["aff"], win["b0"], delta)
    if win.get("clamp") is not None:
        pc[:, win["clamp"], 21:24] = 0.0
    return pc


def _adj(T):
    """Sophus SE3::Adj(): [[R, hat(t) R], [0, R]] (translation first)."""
    R, t = T[:3, :3], T[:3, 3]
    hat = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    A = np.zeros((6, 6))
    A[:3, :3] = R
    A[3:, 3:] = R
    A[:3, 3:] = hat @ R
    return A


def inputs(win, seed=0):
    """solveSystemF's inputs for a window: dict(ad_host, ad_target (n, n, 8, 8) [host][target] as setAdjointsF forms them,
    frame_prior, frame_delta_prior (n, 8), c_prior (4,), c_delta (4,) float32, point_prior, point_delta float32).  Every
    third point has a depth prior; a few points have deltaF = 0."""
    rng = np.random.default_rng(seed + 101)
    n, npt = win["n_frames"], len(win["host"])
    aH, aT = np.zeros((n, n, 8, 8)), np.zeros((n, n, 8, 8))
    scale = np.array([0.5, 0.5, 0.5, 1.0, 1.0, 1.0, 10.0, 1000.0])   # SCALE_XI_TRANS, SCALE_XI_ROT, SCALE_A, SCALE_B
    for h in range(n):
        for t in range(n):
            T = np.linalg.inv(win["poses"][t]) @ win["poses"][h]
            AH, AT = np.eye(8), np.eye(8)
            AH[:6, :6] = -_adj(T).T
            a = float(np.float32(win["aff"][h][t][0]))
            AT[6, 6], AH[6, 6], AT[7, 7], AH[7, 7] = -a, a, -1.0, a
            aH[h, t] = AH * scale[:, None]
            aT[h, t] = AT * scale[:, None]
    fp = np.zeros((n, 8))
    fp[0, :6] = 1e10   # the first frame's pose prior, the affine priors of every frame
    fp[:, 6], fp[:, 7] = 1e4, 1e3
    fdp = rng.normal(0, 1e-3, (n, 8))
    pp = np.where(np.arange(npt) % 3 == 0, 2500.0, 0.0).astype(np.float32)
    pd = (rng.normal(0, 0.01, npt) * (np.arange(npt) % 7 != 0)).astype(np.float32)
    return dict(ad_host=aH, ad_target=aT, frame_prior=fp, frame_delta_prior=fdp, c_prior=np.full(4, 5e9),
                c_delta=rng.normal(0, 0.1, 4).astype(np.float32), point_prior=pp, point_delta=pd)


def _c_layout(a, n):
    """[host][target] -> the C record order host + n * target."""
    return np.ascontiguousarray(np.swapaxes(np.asarray(a, np.float64).reshape(n, n, 8, 8), 0, 1))


def stitch(raw, inp, n):
    """stitch_oracle over raw accumulators in get_accumulators' [host][target] form: dict(H_top, b_top, H_sc, b_sc)."""
    dim = 8 * n + 4
    c = {k: np.ascontiguousarray(np.swapaxes(raw[k], 0, 1)) for k in ("top", "acc_e", "acc_eb")}
    c["top_num"] = np.ascontiguousarray(np.swapaxes(raw["top_num"], 0, 1), np.int32)
    c["acc_d"] = np.ascontiguousarray(np.swapaxes(raw["acc_d"], 0, 2))
    c["d_num"] = np.ascontiguousarray(np.swapaxes(raw["d_num"], 0, 2), np.int32)
    out = dict(H_top=np.zeros((dim, dim)), b_top=np.zeros(dim), H_sc=np.zeros((dim, dim)), b_sc=np.zeros(dim))
    aH, aT = _c_layout(inp["ad_host"], n), _c_layout(inp["ad_target"], n)
    f64 = lambda a: np.ascontiguousarray(a, np.float64)
    _lib().stitch_oracle(n, _p(c["top"], _dp), _p(c["top_num"], _ip), _p(c["acc_e"], _dp), _p(c["acc_eb"], _dp), _p(c["acc_d"], _dp),
                         _p(c["d_num"], _ip), _p(f64(raw["hcc"]), _dp), _p(f64(raw["bc"]), _dp), _p(aH, _dp), _p(aT, _dp),
                         _p(f64(inp["frame_prior"]), _dp), _p(f64(inp["frame_delta_prior"]), _dp), _p(f64(inp["c_prior"]), _dp),
                         _p(np.ascontiguousarray(inp["c_delta"], np.float32)), _p(out["H_top"], _dp), _p(out["b_top"], _dp),
                         _p(out["H_sc"], _dp), _p(out["b_sc"], _dp))
    return out


class AccumulateOracle(L.LinearizeOracle):
    """LinearizeOracle plus the data each applyRes(true) takes (takeDataF) and the accumulators over it."""

    def load(self):
        super().load()
        m = len(self.win["res_point"])
        self.Jt = np.zeros((m, L.JACOBIAN_FLOATS), np.float32)
        self.last_J = np.zeros((m, L.JACOBIAN_FLOATS), np.float32)
        self.acc = None

    def linearize(self, idepth_scaled, idepth_zero_scaled, precalc, frame_th, fix):
        before = self.state.copy()
        r = super().linearize(idepth_scaled, idepth_zero_scaled, precalc, frame_th, fix)
        self.last_J = r["jacobians"].copy()
        if fix:
            self._take(before)
        return r

    def apply_res(self):
        before = self.state.copy()
        super().apply_res()
        self._take(before)

    def _take(self, before):
        took = (before != L.OOB) & (self.new_state == L.IN)
        self.Jt[took] = self.last_J[took]
        self.acc = None

    def accumulate(self, inp, mode=DOUBLE):
        """dict(raw accumulators in [host][target] form, per-point hdi, idepth_hessian, bd_sum, hcd, n_active, and the
        stitch H_top, b_top, H_sc, b_sc of those raw sums)."""
        W = self.win
        n, npt, m = W["n_frames"], len(W["host"]), len(W["res_point"])
        jpjd = np.zeros((m, 8), np.float32)
        lib = _lib()
        lib.take_data_oracle(m, _p(self.Jt), _p(jpjd))
        c = dict(top=np.zeros((n * n, 91)), top_num=np.zeros(n * n, np.int32), acc_e=np.zeros((n * n, 8, 4)),
                 acc_eb=np.zeros((n * n, 8)), acc_d=np.zeros((n ** 3, 8, 8)), d_num=np.zeros(n ** 3, np.int32), hcc=np.zeros((4, 4)),
                 bc=np.zeros(4))
        pt = dict(hdi=np.zeros(npt, np.float32), idepth_hessian=np.zeros(npt, np.float32), bd_sum=np.zeros(npt, np.float32),
                  hcd=np.zeros((npt, 4), np.float32))
        active = np.ascontiguousarray(self.active, np.int32)
        pp = np.ascontiguousarray(inp["point_prior"], np.float32)
        pd = np.ascontiguousarray(inp["point_delta"], np.float32)
        na = lib.accumulate_oracle(mode, n, npt, _p(W["host"], _ip), m, _p(W["res_point"], _ip), _p(W["res_target"], _ip), _p(self.Jt),
                                   _p(jpjd), _p(active, _ip), _p(pp), _p(pd), _p(c["top"], _dp), _p(c["top_num"], _ip),
                                   _p(c["acc_e"], _dp), _p(c["acc_eb"], _dp), _p(c["acc_d"], _dp), _p(c["d_num"], _ip),
                                   _p(c["hcc"], _dp), _p(c["bc"], _dp), _p(pt["hdi"]), _p(pt["idepth_hessian"]), _p(pt["bd_sum"]),
                                   _p(pt["hcd"]))
        raw = dict(top=c["top"].reshape(n, n, 91), top_num=c["top_num"].reshape(n, n), acc_e=c["acc_e"].reshape(n, n, 8, 4),
                   acc_eb=c["acc_eb"].reshape(n, n, 8), acc_d=c["acc_d"].reshape(n, n, n, 8, 8), d_num=c["d_num"].reshape(n, n, n),
                   hcc=c["hcc"], bc=c["bc"])
        # C order [target][host] -> [host][target]
        for k in ("top", "top_num", "acc_e", "acc_eb"):
            raw[k] = np.ascontiguousarray(np.swapaxes(raw[k], 0, 1))
        for k in ("acc_d", "d_num"):
            raw[k] = np.ascontiguousarray(np.swapaxes(raw[k], 0, 2))
        raw["n_points_active"] = int((pt["hdi"] != 0).sum())
        out = dict(raw=raw, n_active=int(na), jpjd=jpjd, **pt)
        out.update(stitch(raw, inp, n))
        self.acc = (inp, out)
        return out

    def resubstitute(self, x):
        inp, a = self.acc
        W = self.win
        n, npt, m = W["n_frames"], len(W["host"]), len(W["res_point"])
        step = np.zeros(npt, np.float32)
        x = np.ascontiguousarray(x, np.float64)
        _lib().resubstitute_oracle(n, npt, _p(W["host"], _ip), m, _p(W["res_point"], _ip), _p(W["res_target"], _ip),
                                   _p(np.ascontiguousarray(self.active, np.int32), _ip), _p(a["jpjd"]), _p(a["hdi"]), _p(a["bd_sum"]),
                                   _p(a["hcd"]), _p(_c_layout(inp["ad_host"], n), _dp), _p(_c_layout(inp["ad_target"], n), _dp),
                                   _p(x, _dp), _p(step))
        return step


def solve(a):
    """A step x for the system a (H_top - H_sc, b_top - b_sc), as the host's dense solve would give one: a regularised
    solve, scaled to a small norm so that the stepped depths stay in front of the cameras."""
    H = a["H_top"] - a["H_sc"]
    b = a["b_top"] - a["b_sc"]
    d = np.sqrt(np.abs(np.diag(H))) + 1.0
    Hs = H / d[:, None] / d[None, :] + 1e-3 * np.eye(len(b))
    x = -np.linalg.solve(Hs, b / d) / d
    nx = np.linalg.norm(x)
    return x * (1e-3 / nx) if nx > 1e-3 else x


def summation_bars(abs_raw):
    """Per raw entry the worst-case bound of any summation order of its terms in double, N 2^-53 sum |terms|, from the ABS
    mode's raw sums (N: the entry's update count)."""
    n_pts = abs_raw["n_points_active"]
    N = dict(top=abs_raw["top_num"][..., None], acc_e=abs_raw["top_num"][..., None, None], acc_eb=abs_raw["top_num"][..., None],
             acc_d=abs_raw["d_num"][..., None, None], hcc=n_pts, bc=n_pts)
    return {k: N[k] * 2.0 ** -53 * abs_raw[k] for k in N}


PIN_KEYS = ("H_top", "b_top", "H_sc", "b_sc", "hdi", "idepth_hessian", "step")


def pin_sequence(o, inp, accumulate, resubstitute):
    """The optimize()-shaped sequence of the reference pins over an AccumulateOracle `o` (its linearize and apply), with
    accumulate() -> dict and resubstitute(x) -> step from the backend under test: linearize, apply, accumulate, a solved x,
    resubstitute; a stepped linearize and apply, accumulate, resubstitute; a rejected trial (linearize with another
    newest-frame threshold, no apply), accumulate; linearize(fix), accumulate.  Returns one dict per accumulate."""
    W = o.win
    st = L.steps(W)
    idz = W["idepth"].copy()
    th = W["frame_th"].copy()
    out = []
    o.linearize(idz, idz, precalc(W), th, 0)
    o.apply_res()
    r = dict(accumulate())
    r["step"] = resubstitute(solve(r))
    out.append(r)
    ids = (idz + r["step"]).astype(np.float32)
    pc1 = st[1]["precalc"] if W.get("clamp") is None else precalc(W, None)
    o.linearize(ids, idz, pc1, th, 0)
    o.apply_res()
    r = dict(accumulate())
    r["step"] = resubstitute(solve(r))
    out.append(r)
    th2 = th.copy()
    th2[-1] = 5.0
    o.linearize(st[2]["idepth_scaled"], idz, st[2]["precalc"], th2, 0)
    out.append(dict(accumulate()))
    o.linearize(ids, idz, pc1, th, 1)
    out.append(dict(accumulate()))
    return out


def pin_record(r):
    """The form the pins store one accumulate in: n_active, and SHA-256 digests of the arrays' bytes."""
    import hashlib
    out = dict(n_active=np.int32(r["n_active"]))
    for k in PIN_KEYS:
        if k in r:
            a = np.ascontiguousarray(r[k], np.float64 if k[0] in "Hb" else np.float32)
            out[k + "_digest"] = np.frombuffer(hashlib.sha256(a.tobytes()).digest(), np.uint8)
    return out
