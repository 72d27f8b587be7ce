"""Host-side mirror of `class CudaCoarseTracker`
(tandem/libdr/cuda_coarse_tracker/include/public/cuda_coarse_tracker.h:9-82) over the C ABI.
Eigen types of the reference signature become numpy arrays (Vec6 -> (6,), Mat88 -> (8,8), Vec8 -> (8,))."""
import ctypes

import numpy as np

from ._lib import CoarseNodiaResult, TrackNewCoarseResult, TrackPyramidResult, TrackResult, TrackTry, check, lib

_fp = ctypes.POINTER(ctypes.c_float)
_dp = ctypes.POINTER(ctypes.c_double)


def _f(a):
    return np.ascontiguousarray(a, np.float32)


class ImagePyramid:
    """FrameHessian::makeImages on the device (HessianBlocks.cpp:128-191; SURVEY 8f row n2)."""

    def __init__(self, w, h, levels, device=0):
        self.w, self.h, self.levels = w, h, levels
        self._h = ctypes.c_void_p()
        check(lib().tdm_pyramid_create(w, h, levels, device, ctypes.byref(self._h)))

    def close(self):
        if self._h is not None:
            lib().tdm_pyramid_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def build(self, gray):
        g = _f(gray)
        assert g.size == self.w * self.h
        check(lib().tdm_pyramid_build(self._h, g.ctypes.data_as(_fp)))

    def level(self, lvl):
        """(dI (h_l, w_l, 3), absSquaredGrad (h_l, w_l)) of one level, copied to the host."""
        wl, hl = self.w >> lvl, self.h >> lvl
        dI = np.empty((hl, wl, 3), np.float32)
        ag = np.empty((hl, wl), np.float32)
        check(lib().tdm_pyramid_get_level(self._h, lvl, dI.ctypes.data_as(_fp), ag.ctypes.data_as(_fp)))
        return dI, ag


class CudaCoarseTracker:
    def __init__(self, w, h, setting_huberTH=9.0, setting_coarseCutoffTH=20.0, device=0):
        self.w, self.h = w, h
        self._args = (w, h, float(setting_huberTH), float(setting_coarseCutoffTH), device)
        self._h = None

    def init(self, n_max=0):
        if self._h is not None:
            raise RuntimeError("Cannot call CudaCoarseTracker::init more than once.")
        w, h, hub, cut, dev = self._args
        self._h = ctypes.c_void_p()
        check(lib().tdm_tracker_create(w, h, hub, cut, n_max, dev, ctypes.byref(self._h)))

    def free(self):
        if self._h is not None:
            lib().tdm_tracker_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def setK(self, w, h, fx, fy, cx, cy):
        check(lib().tdm_tracker_set_k(self._h, w, h, fx, fy, cx, cy))

    def setReference(self, n, pc_u, pc_v, pc_idepth, pc_color, ref_exposure, ref_aff_g2l):
        u, v, i, c = _f(pc_u), _f(pc_v), _f(pc_idepth), _f(pc_color)
        aff = np.ascontiguousarray(ref_aff_g2l, np.float64)
        check(lib().tdm_tracker_set_reference(self._h, n, u.ctypes.data_as(_fp), v.ctypes.data_as(_fp),
                                              i.ctypes.data_as(_fp), c.ctypes.data_as(_fp), float(ref_exposure),
                                              aff.ctypes.data_as(_dp)))

    def setNew(self, dInew):
        d = _f(dInew)
        assert d.size == self.w * self.h * 3
        check(lib().tdm_tracker_set_new(self._h, d.ctypes.data_as(_fp)))

    def calcRes(self, refToNew, new_exposure, aff_g2l, cutoffTH):
        T = np.ascontiguousarray(refToNew, np.float64)
        aff = np.ascontiguousarray(aff_g2l, np.float64)
        res = np.zeros(6, np.float64)
        check(lib().tdm_tracker_calc_res(self._h, T.ctypes.data_as(_dp), float(new_exposure), aff.ctypes.data_as(_dp),
                                         float(cutoffTH), res.ctypes.data_as(_dp)))
        return res

    def calcG(self, new_exposure, aff_g2l):
        aff = np.ascontiguousarray(aff_g2l, np.float64)
        H = np.zeros((8, 8), np.float64)
        b = np.zeros(8, np.float64)
        check(lib().tdm_tracker_calc_g(self._h, float(new_exposure), aff.ctypes.data_as(_dp), H.ctypes.data_as(_dp),
                                       b.ctypes.data_as(_dp)))
        return H, b

    def calcResBatch(self, refToNews, new_exposure, aff_g2ls, cutoffTH):
        """calcRes of several motion hypotheses in one launch (extension): refToNews (n,4,4), aff_g2ls (n,2) -> res (n,6)."""
        T = np.ascontiguousarray(refToNews, np.float64).reshape(-1, 16)
        n = T.shape[0]
        aff = np.ascontiguousarray(aff_g2ls, np.float64).reshape(n, 2)
        res = np.zeros((n, 6), np.float64)
        check(lib().tdm_tracker_calc_res_batch(self._h, n, T.ctypes.data_as(_dp), float(new_exposure), aff.ctypes.data_as(_dp),
                                               float(cutoffTH), res.ctypes.data_as(_dp)))
        return res

    def calcResAndG(self, refToNew, new_exposure, aff_g2l, cutoffTH):
        T = np.ascontiguousarray(refToNew, np.float64)
        aff = np.ascontiguousarray(aff_g2l, np.float64)
        res = np.zeros(6, np.float64)
        H = np.zeros((8, 8), np.float64)
        b = np.zeros(8, np.float64)
        check(lib().tdm_tracker_calc_res_g(self._h, T.ctypes.data_as(_dp), float(new_exposure), aff.ctypes.data_as(_dp),
                                           float(cutoffTH), res.ctypes.data_as(_dp), H.ctypes.data_as(_dp),
                                           b.ctypes.data_as(_dp)))
        return res, H, b

    # ---- SURVEY 8(f) n1-n3: device-side neighbours of the evaluation ----
    def setNewFromPyramid(self, pyramid, level=0):
        check(lib().tdm_tracker_set_new_from_pyramid(self._h, pyramid._h, level))

    def setReferenceDense(self, T_depth_to_ref, ref_exposure, ref_aff_g2l, depth=None, fusion=None, render_index=0,
                          tracking_step=1, dense_only=True, sparse=None, idepth0=None, ref_gray=None, pyramid=None):
        """Dense part of CoarseTracker::setCoarseTrackingRef + setReference (CoarseTracker.cpp:655-732).
        sparse = (pc_u, pc_v, pc_idepth, pc_color), each n_sparse + 1 long (the last entry is the slot `++pc_n` skips)."""
        T = np.ascontiguousarray(T_depth_to_ref, np.float64)
        aff = np.ascontiguousarray(ref_aff_g2l, np.float64)
        keep = []

        def ptr(a):
            if a is None:
                return None
            a = _f(a)
            keep.append(a)
            return a.ctypes.data_as(_fp)

        ns = 0 if sparse is None else len(sparse[0]) - 1
        sp = [None] * 4 if sparse is None else [ptr(a) for a in sparse]
        n = ctypes.c_int()
        check(lib().tdm_tracker_set_reference_dense(
            self._h, ptr(depth), None if fusion is None else fusion._h, render_index, T.ctypes.data_as(_dp), int(tracking_step),
            int(bool(dense_only)), ns, sp[0], sp[1], sp[2], sp[3], ptr(idepth0), ptr(ref_gray),
            None if pyramid is None else pyramid._h, float(ref_exposure), aff.ctypes.data_as(_dp), ctypes.byref(n)))
        return n.value

    def getReference(self, n):
        out = [np.empty(n, np.float32) for _ in range(4)]
        check(lib().tdm_tracker_get_reference(self._h, n, *[a.ctypes.data_as(_fp) for a in out]))
        return out

    def getCoarseNodia(self, n):
        """The first n entries of (pc_u, pc_v, pc_idepth, pc_color)_nodia, the undilated level-0 cloud this tracker holds as
        levels[0] of set_coarse_tracking_ref_nodia (n = pc_n_nodia + 1 includes the slot behind the count)."""
        out = [np.empty(n, np.float32) for _ in range(4)]
        check(lib().tdm_tracker_get_coarse_nodia(self._h, n, *[a.ctypes.data_as(_fp) for a in out]))
        return out

    def track(self, refToNew, aff_g2l, new_exposure, coarse_cutoff=20.0, max_iterations=10,
              lambda_extrapolation_limit=0.001, fix_a=False, fix_b=False):
        """One pyramid level of CoarseTracker::trackNewestCoarse (CoarseTracker.cpp:761-916) on the device."""
        T = np.ascontiguousarray(refToNew, np.float64)
        aff = np.ascontiguousarray(aff_g2l, np.float64)
        r = TrackResult()
        check(lib().tdm_tracker_track(self._h, T.ctypes.data_as(_dp), aff.ctypes.data_as(_dp), float(new_exposure),
                                      float(coarse_cutoff), int(max_iterations), float(lambda_extrapolation_limit),
                                      int(bool(fix_a)), int(bool(fix_b)), ctypes.byref(r)))
        return dict(refToNew=np.array(r.ref_to_new, np.float64).reshape(4, 4), aff=np.array(r.aff_g2l, np.float64),
                    res=np.array(r.res, np.float64), iterations=r.iterations, evaluations=r.evaluations,
                    cutoff_repeat=r.cutoff_repeat, device_ms=r.device_ms)

    def getWarped(self, n):
        """Test accessor: (7, n) float32 - u, v, dx, dy, idepth, residual, weight of the first n points as the last calcRes
        wrote them (zeros at points it did not accept)."""
        out = np.empty((7, n), np.float32)
        check(lib().tdm_tracker_get_warped(self._h, n, out.ctypes.data_as(_fp)))
        return out

    def synchronize(self):
        check(lib().tdm_tracker_synchronize(self._h))

    def run_resident(self, iters):
        ms = ctypes.c_float()
        check(lib().tdm_tracker_run_resident(self._h, iters, ctypes.byref(ms)))
        return ms.value


def track_pyramid(trackers, refToNew, aff_g2l, new_exposure, coarse_cutoff=20.0, max_iterations=(10, 20, 50, 50, 50),
                  lambda_extrapolation_limit=0.001, affine_opt_mode_a=0.0, affine_opt_mode_b=0.0, min_res_for_abort=None):
    """CoarseTracker::trackNewestCoarse (CoarseTracker.cpp:750-936) for one motion hypothesis, every level on the device with
    one host wait.  trackers[l] is the CudaCoarseTracker of pyramid level l ((w >> l) x (h >> l)), each with setK, a reference and
    a new image; len(trackers) - 1 is the coarsest level.  affine_opt_mode_a/b are setting_affineOptModeA/B (< 0: fixed).
    min_res_for_abort: 5 values, NaN (the default) never aborts.  Returns a dict like CudaCoarseTracker.track plus the
    coarse-to-fine outcome (ok, aborted_level, repeated_level, per-level last_residuals / iterations / evaluations /
    cutoff_repeat, last_flow_indicators)."""
    n = len(trackers)
    hs = (ctypes.c_void_p * max(n, 1))(*[t._h for t in trackers])
    T = np.ascontiguousarray(refToNew, np.float64)
    aff = np.ascontiguousarray(aff_g2l, np.float64)
    its = np.zeros(5, np.int32)
    its[:min(len(max_iterations), 5)] = np.asarray(max_iterations, np.int32)[:5]
    mr = np.full(5, np.nan) if min_res_for_abort is None else np.ascontiguousarray(min_res_for_abort, np.float64)
    assert T.size == 16 and aff.size == 2 and mr.size == 5
    r = TrackPyramidResult()
    check(lib().tdm_tracker_track_pyramid(hs, n - 1, T.ctypes.data_as(_dp), aff.ctypes.data_as(_dp), float(new_exposure),
                                          float(coarse_cutoff), its.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                                          float(lambda_extrapolation_limit), float(affine_opt_mode_a), float(affine_opt_mode_b),
                                          mr.ctypes.data_as(_dp), ctypes.byref(r)))
    return dict(refToNew=np.array(r.ref_to_new, np.float64).reshape(4, 4), aff=np.array(r.aff_g2l, np.float64), ok=bool(r.ok),
                aborted_level=r.aborted_level, repeated_level=r.repeated_level,
                last_residuals=np.array(r.last_residuals, np.float64), last_flow_indicators=np.array(r.last_flow_indicators, np.float64),
                iterations=np.array(r.iterations[:], np.int32), evaluations=np.array(r.evaluations[:], np.int32),
                cutoff_repeat=np.array(r.cutoff_repeat[:], np.float32), device_ms=r.device_ms)


def track_new_coarse(trackers, tries, aff_last_2_l, new_exposure, last_coarse_rmse, retrack_threshold=1.5, coarse_cutoff=20.0,
                     max_iterations=(10, 20, 50, 50, 50), lambda_extrapolation_limit=0.001, affine_opt_mode_a=0.0,
                     affine_opt_mode_b=0.0):
    """FullSystem::trackNewCoarse's loop over the motion hypotheses (FullSystem.cpp:538-617, monocular): every try is a
    track_pyramid run from tries[i] (n x 4 x 4, 1 <= n <= 64) and aff_last_2_l with min_res_for_abort = achievedRes, the winner /
    takeover / break rules run after each try, all on the device with one host wait.  trackers as for track_pyramid;
    retrack_threshold is setting_reTrackThreshold.  Returns dict(refToNew (lastF_2_fh), aff (aff_g2l), flow_vecs,
    achieved_res (the new lastCoarseRMSE), have_one_good, tries (tryIterations), winner (last winning try, -1: none), device_ms,
    per_try: a list of dict(ok, aborted_level, repeated_level, last_residuals, evaluations) for the tries run)."""
    n = len(trackers)
    hs = (ctypes.c_void_p * max(n, 1))(*[t._h for t in trackers])
    T = np.ascontiguousarray(tries, np.float64).reshape(-1, 16)
    aff = np.ascontiguousarray(aff_last_2_l, np.float64)
    its = np.zeros(5, np.int32)
    its[:min(len(max_iterations), 5)] = np.asarray(max_iterations, np.int32)[:5]
    rmse = np.ascontiguousarray(last_coarse_rmse, np.float64)
    assert aff.size == 2 and rmse.size == 5
    r = TrackNewCoarseResult()
    recs = (TrackTry * max(T.shape[0], 1))()
    check(lib().tdm_tracker_track_new_coarse(hs, n - 1, T.ctypes.data_as(_dp), T.shape[0], aff.ctypes.data_as(_dp), float(new_exposure),
                                             float(coarse_cutoff), its.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                                             float(lambda_extrapolation_limit), float(affine_opt_mode_a), float(affine_opt_mode_b),
                                             rmse.ctypes.data_as(_dp), float(retrack_threshold), ctypes.byref(r), recs))
    per_try = [dict(ok=bool(t.ok), aborted_level=t.aborted_level, repeated_level=t.repeated_level,
                    last_residuals=np.array(t.last_residuals, np.float64), evaluations=np.array(t.evaluations[:], np.int32))
               for t in recs[:r.tries]]
    return dict(refToNew=np.array(r.ref_to_new, np.float64).reshape(4, 4), aff=np.array(r.aff_g2l, np.float64),
                flow_vecs=np.array(r.flow_vecs, np.float64), achieved_res=np.array(r.achieved_res, np.float64),
                have_one_good=bool(r.have_one_good), tries=r.tries, winner=r.winner, device_ms=r.device_ms, per_try=per_try)


def _coarse_ref_call(levels, points, ref_pyramid, depth, fusion, render_index, T_depth_to_ref, tracking_step, dense_only, rgbd_init,
                     ref_exposure, ref_aff_g2l, nodia=None):
    """n7 (nodia None) or its nodia entry (nodia = (quantile_fraction, CoarseNodiaResult)); returns pc_n."""
    n_levels = len(levels)
    hs = (ctypes.c_void_p * max(n_levels, 1))(*[t._h for t in levels])
    keep = []

    def ptr(a):
        if a is None:
            return None
        a = _f(a)
        keep.append(a)
        return a.ctypes.data_as(_fp)

    n = 0 if points is None else len(points[0])
    pts = [None] * 4 if points is None else [ptr(a) for a in points]
    assert points is None or all(len(a) == n for a in points)
    T = None if T_depth_to_ref is None else np.ascontiguousarray(T_depth_to_ref, np.float64)
    aff = np.ascontiguousarray(ref_aff_g2l, np.float64)
    pc_n = np.zeros(5, np.int32)
    args = [hs, n_levels, int(bool(rgbd_init)), n, pts[0], pts[1], pts[2], pts[3], ref_pyramid._h, ptr(depth),
            None if fusion is None else fusion._h, int(render_index), None if T is None else T.ctypes.data_as(_dp),
            int(tracking_step), int(bool(dense_only)), float(ref_exposure), aff.ctypes.data_as(_dp)]
    pc_n_p = pc_n.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
    if nodia is None:
        check(lib().tdm_tracker_set_coarse_tracking_ref(*args, pc_n_p))
    else:
        check(lib().tdm_tracker_set_coarse_tracking_ref_nodia(*args, float(nodia[0]), pc_n_p, ctypes.byref(nodia[1])))
    return [int(x) for x in pc_n[:n_levels]]


def set_coarse_tracking_ref(levels, points, ref_pyramid, depth=None, fusion=None, render_index=0, T_depth_to_ref=None,
                            tracking_step=1, dense_only=False, rgbd_init=False, ref_exposure=1.0, ref_aff_g2l=(0.0, 0.0)):
    """CoarseTracker::setCoarseTrackingRef with makeCoarseDepthL0 (CoarseTracker.cpp:148-374, :633-733) for every level in one
    call on the device.  levels[l] is the CudaCoarseTracker of pyramid level l ((w >> l) x (h >> l)), levels[0] with setK.
    points = (u, v, idepth, hessian) in the reference's order - monocular: centerProjectedTo[0..2] and efPoint->HdiF of the
    points passing the lastResiduals[0] test; rgbd_init: ph->u, ph->v, ph->idepth, ph->idepth_hessian - or None for no points.
    Colours come from ref_pyramid (an ImagePyramid of the reference keyframe).  The optional dense map is a host depth image or
    the render_index-th render of a DrFusion, warped with T_depth_to_ref (4x4) and appended behind level 0's points.
    Returns pc_n, one count per level; each level then holds its reference as after setReference."""
    return _coarse_ref_call(levels, points, ref_pyramid, depth, fusion, render_index, T_depth_to_ref, tracking_step, dense_only,
                            rgbd_init, ref_exposure, ref_aff_g2l)


def set_coarse_tracking_ref_nodia(levels, points, ref_pyramid, quantile_fraction=0.2, depth=None, fusion=None, render_index=0,
                                  T_depth_to_ref=None, tracking_step=1, dense_only=False, rgbd_init=False, ref_exposure=1.0,
                                  ref_aff_g2l=(0.0, 0.0)):
    """set_coarse_tracking_ref, plus in the same call the undilated level-0 cloud pc_*_nodia (CoarseTracker.cpp:150-218, held
    by levels[0], see CudaCoarseTracker.getCoarseNodia) and get_idepth_quantile over it (tandem_backend.cpp:354-361), from
    which FullSystem::deliverDrFrame takes MVSNet's depth range (depth_max = 3 * depth_quantile).
    Returns (pc_n, pc_n_nodia, depth_quantile); depth_quantile is NaN when the cloud has no entry at the quantile's index."""
    r = CoarseNodiaResult()
    pc_n = _coarse_ref_call(levels, points, ref_pyramid, depth, fusion, render_index, T_depth_to_ref, tracking_step, dense_only,
                            rgbd_init, ref_exposure, ref_aff_g2l, nodia=(quantile_fraction, r))
    return pc_n, r.pc_n_nodia, r.depth_quantile
