"""Frame loop over the three libdr components in the order TANDEM drives them (SURVEY.md 8(d) config 4).

This is host orchestration only - the harness that stands in for `tandem_dataset` here, where DSO itself cannot be
built (no Eigen / Sophus in the image).  Per frame (FullSystem::addActiveFrame -> trackNewCoarse,
CoarseTracker::trackNewestCoarse, CoarseTracker.cpp:761-916): grey image -> device pyramid (n2) -> coarse-to-fine over
the pyramid levels, one tracker instance per level fed device-to-device (setNewFromPyramid) and one device LM loop per
level (n3, maxIterations = 10/20/50/50 as in settings.cpp) against the current reference.  Per keyframe, in the order of TandemBackendImpl::CallAsync / CallSequential
(tandem/src/tandem/tandem_backend.cpp:137-283): (1) GetResult of the PREVIOUS window, (3.5) CallAsync of the current
window, (3) IntegrateScanAsync of the previous result, (4) RenderAsync at the new keyframe's pose, (5) GetRenderResult,
(5.5) dense tracking reference from the rendered depth, kept on the device for level 0 (n1); the coarser levels - which in
TANDEM use DSO's sparse points, not available here - get the same construction from the sub-sampled host copy.  Until the first MVSNet result exists
(7 keyframes + 1, as in TANDEM's initialisation by the sparse front end) the sensor depth handed in by the caller is
integrated instead.
"""
import time

import numpy as np

from .fusion import DrFusion, DrFusionOptions
from .mvsnet import DrMvsnet
from .tracker import CudaCoarseTracker, ImagePyramid

GRAY_W = np.array([0.114, 0.587, 0.299], np.float32)


class TandemLoop:
    def __init__(self, H, W, K4, weights, window=7, keyframe_every=5, depth_min=0.1, depth_max=8.0, discard=2.5,
                 precision="mixed16", device=0, integrate="mvsnet", max_iterations=(10, 20, 50, 50, 50), tracking_step=1,
                 fusion_options=None, levels=None, feature_cache=False):
        """feature_cache=True submits each window through DrMvsnet.CallAsyncIds with the keyframe index as the view id,
        so that FeatureNet runs only for the keyframe each window adds."""
        self.H, self.W, self.K4 = H, W, tuple(float(k) for k in K4)
        self.feature_cache = feature_cache
        self.n_keyframes = 0
        fx, fy, cx, cy = self.K4
        self.K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
        self.window, self.kf_every = window, keyframe_every
        self.dmin, self.dmax, self.discard = depth_min, depth_max, discard
        self.integrate = integrate
        self.max_iterations, self.tracking_step = max_iterations, tracking_step
        self.mvsnet = DrMvsnet(weights, precision=precision, device=device)
        fo = dict(height=H, width=W, fx=fx, fy=fy, cx=cx, cy=cy, num_render_streams=1)
        fo.update(fusion_options or {})
        self.fusion = DrFusion(DrFusionOptions(**fo), device=device)
        if levels is None:                                    # setGlobalCalib, globalCalib.cpp:43-53
            levels, wl, hl = 1, W, H
            while wl % 2 == 0 and hl % 2 == 0 and wl * hl > 5000 and levels < 5:
                wl, hl, levels = wl // 2, hl // 2, levels + 1
        self.levels = levels
        self.Kl = [(fx / 2 ** l, fy / 2 ** l, (cx + 0.5) / 2 ** l - 0.5, (cy + 0.5) / 2 ** l - 0.5) for l in range(levels)]   # :84-90
        self.trackers = []
        for l in range(levels):
            t = CudaCoarseTracker(W >> l, H >> l, device=device)
            t.init()
            t.setK(W >> l, H >> l, *self.Kl[l])
            self.trackers.append(t)
        self.tracker = self.trackers[0]
        self.pyr = ImagePyramid(W, H, levels, device=device)       # new frame
        self.pyr_ref = ImagePyramid(W, H, levels, device=device)   # reference keyframe (grey values of the dense points)
        self.kfs = []                 # (bgr, c2w, true_depth, keyframe index) of the keyframes in the window
        self.pending = None           # window submitted to MVSNet whose result has not been fetched
        self.ref_c2w = None
        self.have_ref = False
        self.frame_id = 0
        self.last_c2w = None
        self.aff = np.zeros(2)
        self.stats = dict(track_ms=[], track_dev_ms=[], iterations=[], kf_ms=[], mvs_absrel=[], n_ref=[])
        self.trace = []               # per tracked frame: dict(refToNew0, aff0, result) for the oracle comparison

    # ------------------------------------------------------------------------------------------
    def _keyframe(self, bgr, gray, c2w, sensor_depth, true_depth):
        t0 = time.perf_counter()
        self.kfs.append((bgr, np.asarray(c2w, np.float32), true_depth, self.n_keyframes))
        self.n_keyframes += 1
        if len(self.kfs) > self.window:
            self.kfs.pop(0)
        out_prev = None
        if self.pending is not None:                                   # (1) previous window's result
            out_prev = self.mvsnet.GetResult()
        prev = self.pending
        self.pending = None
        if len(self.kfs) == self.window:                               # (3.5) current window, asynchronous
            ref_index = self.window - 2                                 # FullSystem.cpp:1127
            bgrs = [k[0] for k in self.kfs]
            c2ws = [k[1] for k in self.kfs]
            if self.feature_cache:
                self.mvsnet.CallAsyncIds(self.H, self.W, self.window, ref_index, [k[3] for k in self.kfs], bgrs, self.K, c2ws,
                                         self.dmin, self.dmax, self.discard)
            else:
                self.mvsnet.CallAsync(self.H, self.W, self.window, ref_index, bgrs, self.K, c2ws, self.dmin, self.dmax, self.discard)
            self.pending = dict(bgr=bgrs[ref_index], c2w=c2ws[ref_index], true_depth=self.kfs[ref_index][2])
        if out_prev is not None and prev.get("true_depth") is not None:
            td = prev["true_depth"]
            m = (td > 0) & (out_prev.depth_dense > 0)
            self.stats["mvs_absrel"].append(float(np.mean(np.abs(out_prev.depth_dense[m] - td[m]) / td[m])))
        if out_prev is not None and self.integrate == "mvsnet":        # (3) integrate the previous result, read on the device
            self.fusion.IntegrateScanFromMvsnet(self.mvsnet)            # (= its depth, prev["bgr"] and prev["c2w"])
        else:
            self.fusion.IntegrateScanAsync(bgr, sensor_depth, c2w)
        self.fusion.RenderAsync([np.asarray(c2w, np.float32)])          # (4) at the new keyframe's pose
        _, depth_r = self.fusion.GetRenderResult()                      # (5)
        self.pyr_ref.build(gray)                                        # (5.5) dense reference, device resident
        n = self.tracker.setReferenceDense(np.eye(4), 1.0, np.zeros(2), fusion=self.fusion, render_index=0,
                                           tracking_step=self.tracking_step, dense_only=True, pyramid=self.pyr_ref)
        self.n_ref = [n]
        for l in range(1, self.levels):                                 # coarser levels: sub-sampled host copy
            g = np.ascontiguousarray(self.pyr_ref.level(l)[0][..., 0])
            self.n_ref.append(self.trackers[l].setReferenceDense(np.eye(4), 1.0, np.zeros(2),
                                                                 depth=np.ascontiguousarray(depth_r[0][::2 ** l, ::2 ** l]),
                                                                 dense_only=True, ref_gray=g))
        self.stats["n_ref"].append(n)
        self.ref_c2w = np.asarray(c2w, np.float64)
        self.have_ref = n > 100
        self.aff = np.zeros(2)
        self.stats["kf_ms"].append((time.perf_counter() - t0) * 1e3)

    def step(self, bgr, sensor_depth=None, c2w_init=None, true_depth=None):
        """One frame. Returns the estimated cam->world pose (4x4 float64)."""
        bgr = np.ascontiguousarray(bgr, np.uint8)
        gray = bgr.astype(np.float32) @ GRAY_W
        if not self.have_ref:
            assert c2w_init is not None and sensor_depth is not None, "the first frame needs a pose and a depth map"
            c2w = np.asarray(c2w_init, np.float64)
            self._keyframe(bgr, gray, c2w, sensor_depth, true_depth)
        else:
            t0 = time.perf_counter()
            self.pyr.build(gray)
            T = np.linalg.inv(self.last_c2w) @ self.ref_c2w             # refToNew under a constant-position model
            aff, dev_ms, its = self.aff, 0.0, 0
            for l in range(self.levels - 1, -1, -1):                     # CoarseTracker.cpp:761
                self.trackers[l].setNewFromPyramid(self.pyr, l)
                T0, aff0 = T, aff
                r = self.trackers[l].track(T0, aff0, 1.0, max_iterations=self.max_iterations[l])
                T, aff = r["refToNew"], r["aff"]
                dev_ms += r["device_ms"]
                its += r["iterations"]
            self.stats["track_ms"].append((time.perf_counter() - t0) * 1e3)
            self.stats["track_dev_ms"].append(dev_ms)
            self.stats["iterations"].append(its)
            self.trace.append(dict(frame=self.frame_id, refToNew0=T0, aff0=np.array(aff0), result=r))   # level 0
            self.aff = r["aff"]
            c2w = self.ref_c2w @ np.linalg.inv(r["refToNew"])
            if self.frame_id % self.kf_every == 0:
                assert sensor_depth is not None
                self._keyframe(bgr, gray, c2w, sensor_depth, true_depth)
        self.last_c2w = c2w
        self.frame_id += 1
        return c2w

    def finish(self):
        if self.pending is not None:
            self.mvsnet.GetResult()
            self.pending = None
        self.fusion.Synchronize()
