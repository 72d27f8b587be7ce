"""n12 / n13: the active residuals of DSO's window for one FullSystem::optimize, kept in device memory, and their linearisation
(FullSystem::linearizeAll, FullSystemOptimize.cpp:142-210: PointFrameResidual::linearize for every residual,
setNewFrameEnergyTH, and with fixLinearization applyRes and the maxRelBaseline / numGoodResiduals update) over the C ABI
(include/tandem_b200.h, block n12)."""
import ctypes

import numpy as np

from ._lib import LinearizeSettings, check, lib

_dp = ctypes.POINTER(ctypes.c_double)
_fp = ctypes.POINTER(ctypes.c_float)
_ip = ctypes.POINTER(ctypes.c_int)
_bp = ctypes.POINTER(ctypes.c_byte)
_ubp = ctypes.POINTER(ctypes.c_ubyte)

#: util/settings.cpp defaults
LINEARIZE_DEFAULTS = dict(huber_th=9.0, outlier_th_sum_component=2500.0, affine_opt_mode_a=1e12, affine_opt_mode_b=1e8,
                          frame_energy_th_n=0.7, frame_energy_th_const_weight=0.5, frame_energy_th_fac_median=1.5,
                          overall_energy_th_weight=1.0)
JACOBIAN_FLOATS = 74
#: the array outputs of ActivePoints.linearize
OUTPUTS = ("new_state", "new_energy", "new_energy_with_outlier", "center_projected_to", "jacobians", "state", "removed",
           "max_rel_baseline", "num_good_residuals")
#: the array outputs of ActivePoints.accumulate
ACC_OUTPUTS = ("H_top", "b_top", "H_sc", "b_sc", "hdi", "idepth_hessian")
#: ResState
IN, OOB, OUTLIER = 0, 1, 2


def _p(a, t=_fp):
    return None if a is None else a.ctypes.data_as(t)


class ActivePoints:
    """The active residuals of one w x h camera's window: up to capacity_points points, 8 residuals per point."""

    def __init__(self, w, h, capacity_points, device=0, **settings):
        unknown = set(settings) - set(LINEARIZE_DEFAULTS)
        if unknown:
            raise TypeError(f"unknown linearize settings {sorted(unknown)}")
        self.w, self.h = w, h
        self.settings = dict(LINEARIZE_DEFAULTS, **settings)
        st = LinearizeSettings(**self.settings)
        self._h = ctypes.c_void_p()
        self.n_frames = self.n_points = self.n_residuals = 0
        check(lib().tdm_active_create(w, h, capacity_points, ctypes.byref(st), device, ctypes.byref(self._h)))

    def close(self):
        if self._h is not None:
            lib().tdm_active_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def load(self, n_frames, host, u, v, color, weights, res_point, res_target, max_rel_baseline=None, num_good_residuals=None):
        """Loads the window (blocking): per point its host frame, u, v, color (n, 8), weights (n, 8), maxRelBaseline and
        numGoodResiduals (0 by default); per residual, in activeResiduals order, its point and target frame.  Every residual
        is reset as resetOOB does."""
        host = np.ascontiguousarray(host, np.int32).ravel()
        n = len(host)
        u, v = np.ascontiguousarray(u, np.float32).ravel(), np.ascontiguousarray(v, np.float32).ravel()
        color = np.ascontiguousarray(color, np.float32).reshape(n, 8)
        weights = np.ascontiguousarray(weights, np.float32).reshape(n, 8)
        mrb = np.zeros(n, np.float32) if max_rel_baseline is None else np.ascontiguousarray(max_rel_baseline, np.float32).ravel()
        ng = np.zeros(n, np.int32) if num_good_residuals is None else np.ascontiguousarray(num_good_residuals, np.int32).ravel()
        rp = np.ascontiguousarray(res_point, np.int32).ravel()
        rt = np.ascontiguousarray(res_target, np.int32).ravel()
        if not (len(u) == len(v) == len(mrb) == len(ng) == n) or len(rp) != len(rt):
            raise ValueError("per-point or per-residual arrays differ in length")
        check(lib().tdm_active_load(self._h, n_frames, n, _p(host, _ip), _p(u), _p(v), _p(color), _p(weights), _p(mrb), _p(ng, _ip),
                                    len(rp), _p(rp, _ip), _p(rt, _ip)))
        self.n_frames, self.n_points, self.n_residuals = n_frames, n, len(rp)

    def linearize(self, frame_pyramids, precalc, frame_energy_th, calib, idepth_scaled, idepth_zero_scaled, fix=False,
                  jacobians=True, out=None):
        """linearizeAll(fix) (blocking).  precalc (n, n, 27): [host][target] PRE_KRKiTll, PRE_KtTll, PRE_RTll_0, PRE_tTll_0,
        PRE_aff_mode, PRE_b0_mode; calib (fxl, fyl, cxl, cyl).  Returns dict(energy, new_frame_energy_th, new_state,
        new_energy, new_energy_with_outlier, center_projected_to (m, 3), jacobians (m, 74) unless jacobians=False, and with
        fix also state, removed, max_rel_baseline, num_good_residuals).  `out` may hold preallocated arrays (such as
        page-locked ones) for any of these array keys, each of the exact shape and dtype the call returns; an entry for a key
        the call does not return is not written."""
        n, m, npt = self.n_frames, self.n_residuals, self.n_points
        if len(frame_pyramids) != n:
            raise ValueError("one pyramid per frame")
        pc = np.ascontiguousarray(precalc, np.float32)
        if pc.size != n * n * 27:
            raise ValueError("precalc must hold n_frames x n_frames x 27 floats")
        th = np.ascontiguousarray(frame_energy_th, np.float32).ravel()
        cal = np.ascontiguousarray(calib, np.float32).ravel()
        if th.size != n or cal.size != 4:
            raise ValueError("frame_energy_th needs n_frames entries, calib fxl, fyl, cxl, cyl")
        ids = np.ascontiguousarray(idepth_scaled, np.float32).ravel()
        idz = np.ascontiguousarray(idepth_zero_scaled, np.float32).ravel()
        if ids.size != npt or idz.size != npt:
            raise ValueError("one idepth per point")
        shapes = dict(new_state=((m,), np.int8), new_energy=((m,), np.float32), new_energy_with_outlier=((m,), np.float32),
                      center_projected_to=((m, 3), np.float32))
        if jacobians:
            shapes["jacobians"] = ((m, JACOBIAN_FLOATS), np.float32)
        if fix:
            shapes.update(state=((m,), np.int8), removed=((m,), np.uint8), max_rel_baseline=((npt,), np.float32),
                          num_good_residuals=((npt,), np.int32))
        out = out or {}
        unknown = set(out) - set(OUTPUTS)
        if unknown:
            raise TypeError(f"unknown outputs {sorted(unknown)}")
        o = {}
        for k, (s, t) in shapes.items():   # keys not requested by this call (jacobians=False, no fix) are not written
            a = out.get(k)
            if a is None:
                a = np.empty(s, t)
            elif not (isinstance(a, np.ndarray) and a.shape == s and a.dtype == t and a.flags.c_contiguous and a.flags.writeable):
                raise ValueError(f"out[{k!r}] must be a writeable C-contiguous {np.dtype(t).name} array of shape {s}")
            o[k] = a
        e, nth = ctypes.c_double(), ctypes.c_float()
        fp = (ctypes.c_void_p * n)(*[p._h.value for p in frame_pyramids])
        check(lib().tdm_active_linearize(self._h, fp, _p(pc), _p(th), _p(cal), _p(ids), _p(idz), int(bool(fix)), ctypes.byref(e),
                                         ctypes.byref(nth), _p(o.get("new_state"), _bp), _p(o.get("new_energy")),
                                         _p(o.get("new_energy_with_outlier")), _p(o.get("center_projected_to")),
                                         _p(o.get("jacobians")), _p(o.get("state"), _bp), _p(o.get("removed"), _ubp),
                                         _p(o.get("max_rel_baseline")), _p(o.get("num_good_residuals"), _ip)))
        r = {k: o[k] for k in shapes}
        r.update(energy=e.value, new_frame_energy_th=nth.value)
        return r

    def apply_res(self):
        """applyRes_Reductor on the device (asynchronous)."""
        check(lib().tdm_active_apply_res(self._h))

    def get_state(self):
        """dict(state, energy): every residual's state_state and state_energy (synchronises)."""
        s, e = np.empty(self.n_residuals, np.int8), np.empty(self.n_residuals, np.float32)
        check(lib().tdm_active_get_state(self._h, _p(s, _bp), _p(e)))
        return dict(state=s, energy=e)

    def accumulate(self, ad_host, ad_target, frame_prior, frame_delta_prior, c_prior, c_delta, point_prior, point_delta, out=None):
        """accumulateAF_MT + accumulateLF_MT + accumulateSCF_MT over the data the last apply took (blocking).  ad_host,
        ad_target (n, n, 8, 8) [host][target]; frame_prior, frame_delta_prior (n, 8); c_prior (4,) doubles; c_delta (4,)
        floats; point_prior, point_delta one float per point.  Returns dict(H_top, b_top, H_sc, b_sc, n_active, hdi,
        idepth_hessian) with H (8n+4, 8n+4) and b (8n+4,) doubles.  `out` may hold preallocated arrays (such as page-locked
        ones) for the array keys, each of the exact shape and dtype the call returns."""
        n, npt = self.n_frames, self.n_points
        dim = 8 * n + 4
        f64 = lambda a: np.ascontiguousarray(a, np.float64)
        f32 = lambda a: np.ascontiguousarray(a, np.float32).ravel()
        # [host][target] -> the C layout's record index host + n * target
        aH, aT = (f64(np.swapaxes(np.asarray(a, np.float64).reshape(n, n, 8, 8), 0, 1)) for a in (ad_host, ad_target))
        fpr, fdp, cp, cd = f64(frame_prior), f64(frame_delta_prior), f64(c_prior).ravel(), f32(c_delta)
        pp, pd = f32(point_prior), f32(point_delta)
        if aH.size != n * n * 64 or aT.size != n * n * 64:
            raise ValueError("ad_host and ad_target need n_frames x n_frames 8x8 records")
        if fpr.size != 8 * n or fdp.size != 8 * n or cp.size != 4 or cd.size != 4:
            raise ValueError("frame_prior / frame_delta_prior need n_frames x 8 entries, c_prior and c_delta 4")
        if pp.size != npt or pd.size != npt:
            raise ValueError("one point_prior and point_delta per point")
        shapes = dict(H_top=((dim, dim), np.float64), b_top=((dim,), np.float64), H_sc=((dim, dim), np.float64),
                      b_sc=((dim,), np.float64), hdi=((npt,), np.float32), idepth_hessian=((npt,), np.float32))
        o = self._outputs(shapes, out, ACC_OUTPUTS)
        na = ctypes.c_int()
        check(lib().tdm_active_accumulate(self._h, _p(aH, _dp), _p(aT, _dp), _p(fpr, _dp), _p(fdp, _dp), _p(cp, _dp), _p(cd), _p(pp),
                                          _p(pd), _p(o["H_top"], _dp), _p(o["b_top"], _dp), _p(o["H_sc"], _dp), _p(o["b_sc"], _dp),
                                          ctypes.byref(na), _p(o["hdi"]), _p(o["idepth_hessian"])))
        return dict(o, n_active=na.value)

    def resubstitute(self, x, out=None):
        """resubstituteF_MT's per-point step for the solved x (8n+4 doubles) with the last accumulate's adjoints (blocking).
        Returns one float per point; `out` may be a preallocated float32 array of that shape."""
        x = np.ascontiguousarray(x, np.float64).ravel()
        if x.size != 8 * self.n_frames + 4:
            raise ValueError("x needs 8 n_frames + 4 entries")
        o = self._outputs(dict(step=((self.n_points,), np.float32)), None if out is None else dict(step=out), ("step",))
        check(lib().tdm_active_resubstitute(self._h, _p(x, _dp), _p(o["step"])))
        return o["step"]

    def get_accumulators(self):
        """The last accumulate's raw sums before the stitch (synchronises): dict(top (n, n, 91) [host][target], top_num
        (n, n), acc_e (n, n, 8, 4), acc_eb (n, n, 8), acc_d (n, n, n, 8, 8) [host][t1][t2], d_num (n, n, n), hcc (4, 4),
        bc (4,))."""
        n = self.n_frames
        # the C layout is [target][host] (index host + n * target); returned transposed to [host][target]
        r = dict(top=np.empty((n, n, 91)), top_num=np.empty((n, n), np.int32), acc_e=np.empty((n, n, 8, 4)),
                 acc_eb=np.empty((n, n, 8)), acc_d=np.empty((n, n, n, 8, 8)), d_num=np.empty((n, n, n), np.int32),
                 hcc=np.empty((4, 4)), bc=np.empty(4))
        check(lib().tdm_active_get_accumulators(self._h, _p(r["top"], _dp), _p(r["top_num"], _ip), _p(r["acc_e"], _dp),
                                                _p(r["acc_eb"], _dp), _p(r["acc_d"], _dp), _p(r["d_num"], _ip), _p(r["hcc"], _dp),
                                                _p(r["bc"], _dp)))
        for k in ("top", "top_num", "acc_e", "acc_eb"):
            r[k] = np.ascontiguousarray(np.swapaxes(r[k], 0, 1))
        for k in ("acc_d", "d_num"):
            r[k] = np.ascontiguousarray(np.swapaxes(r[k], 0, 2))
        return r

    @staticmethod
    def _outputs(shapes, out, allowed):
        out = out or {}
        unknown = set(out) - set(allowed)
        if unknown:
            raise TypeError(f"unknown outputs {sorted(unknown)}")
        o = {}
        for k, (s, t) in shapes.items():
            a = out.get(k)
            if a is None:
                a = np.empty(s, t)
            elif not (isinstance(a, np.ndarray) and a.shape == s and a.dtype == t and a.flags.c_contiguous and a.flags.writeable):
                raise ValueError(f"out[{k!r}] must be a writeable C-contiguous {np.dtype(t).name} array of shape {s}")
            o[k] = a
        return o
