"""The MVSNet -> TSDF keyframe handoff (tdm_fusion_integrate_mvsnet, DrFusion.IntegrateScanFromMvsnet): integrating the
result the last GetResult returned, read on the device, must build the volume the host path builds from the same bytes
(GetResult's depth, the window's reference BGR image and pose) - block map, voxels, counters and renders bit for bit - in
TANDEM's call order GetResult(k) -> CallAsync(k+1) -> integrate(k) -> render, whatever the next window has overwritten."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tandem_b200 import DrMvsnet, DrMvsnetOutput, TandemError, default_weights
from tandem_b200._lib import lib
from tandem_b200.fusion import DrFusion, DrFusionOptions
from tandem_b200.synthetic import mvs_plane_window
from tandem_b200.tracker import CudaCoarseTracker

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WEIGHTS = default_weights("abl03_view_aggregation")
H, W, V = 128, 160, 4
# the options tests/cpp/shim_keyframe.cpp uses as well
SMALL = dict(num_buckets=100003, num_blocks=200000)


class Seq:
    """A camera moving along a textured plane: window k = frames k .. k+V-1, reference at V-2, so consecutive windows have
    different reference images and poses."""

    def __init__(self, n_frames, seed, H=H, W=W, V=V):
        win = mvs_plane_window(V=n_frames, H=H, W=W, seed=seed)
        self.H, self.W, self.V = H, W, V
        self.bgrs, self.c2ws, self.K = win["bgrs"], win["c2ws"], win["K"]
        self.ref = V - 2
        self.n = n_frames - V + 1

    def call(self, m, k):
        m.CallAsync(self.H, self.W, self.V, self.ref, self.bgrs[k:k + self.V], self.K, self.c2ws[k:k + self.V], 0.5, 5.0, 2.5)

    def ref_bgr(self, k):
        return self.bgrs[k + self.ref]

    def ref_c2w(self, k):
        return self.c2ws[k + self.ref]

    def fusion(self):
        K = self.K
        return DrFusion(DrFusionOptions(height=self.H, width=self.W, fx=float(K[0, 0]), fy=float(K[1, 1]), cx=float(K[0, 2]),
                                        cy=float(K[1, 2]), **SMALL))


def _same_volume(a, b):
    ca, va = a.dump_blocks()
    cb, vb = b.dump_blocks()
    assert len(ca) > 0
    assert np.array_equal(ca, cb)
    assert va.tobytes() == vb.tobytes()
    assert a.stats() == b.stats()


def _render(f, pose):
    f.RenderAsync([np.asarray(pose, np.float32)])
    bgrs, depths = f.GetRenderResult()
    return bgrs[0].copy(), depths[0].copy()


def _same_render(fs, pose):
    rs = [_render(f, pose) for f in fs]
    assert (rs[0][1] > 0).mean() > 0.3, "the render should see the integrated plane"
    for b, d in rs[1:]:
        assert b.tobytes() == rs[0][0].tobytes() and d.tobytes() == rs[0][1].tobytes()
    return rs[0]


@pytest.mark.parametrize("outputs", ["pageable", "pinned"])
@pytest.mark.parametrize("precision", ["mixed16", "fp32"])
def test_same_volume_in_tandem_order(precision, outputs):
    """Per keyframe: host path, new call with pose=NULL and new call with the explicit reference pose, all bit-identical."""
    s = Seq(8, seed=11)
    m = DrMvsnet(WEIGHTS, precision=precision)
    out = DrMvsnetOutput(H, W, pinned=outputs == "pinned")
    if outputs == "pinned":
        m.set_option("eager_d2h", 0)
    host, dev_null, dev_pose = s.fusion(), s.fusion(), s.fusion()
    s.call(m, 0)
    for k in range(s.n):
        r = m.GetResult(out=out)                                       # GetResult(k)
        if k + 1 < s.n:
            s.call(m, k + 1)                                           # CallAsync(k+1)
        host.IntegrateScanAsync(s.ref_bgr(k), r.depth, s.ref_c2w(k))   # integrate(k)
        dev_null.IntegrateScanFromMvsnet(m)
        dev_pose.IntegrateScanFromMvsnet(m, s.ref_c2w(k))
        _same_volume(host, dev_null)
        _same_volume(host, dev_pose)
        _same_render([host, dev_null, dev_pose], s.ref_c2w(k))


def test_same_volume_golden_sample():
    """The shipped 512x320 window, with the reference view moving through the views from keyframe to keyframe."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "sample_512x320.npz"))
    nv, gh, gw = g["bgr"].shape[:3]
    bgrs = [np.ascontiguousarray(g["bgr"][v]) for v in range(nv)]
    c2ws = [np.ascontiguousarray(g["c2w"][v]) for v in range(nv)]
    Ks = np.stack([g["K1"], g["K2"], g["K3"]]).astype(np.float32)
    K = g["K3"]
    opts = DrFusionOptions(height=gh, width=gw, fx=float(K[0, 0]), fy=float(K[1, 1]), cx=float(K[0, 2]), cy=float(K[1, 2]), **SMALL)
    host, dev = DrFusion(opts), DrFusion(opts)
    m = DrMvsnet(default_weights("abl04_fewer_depth_planes"), precision="mixed16")
    refs = [int(g["ref_index"]), 1, 4]
    call = lambda ref: m.CallAsyncStageK(gh, gw, nv, ref, bgrs, Ks, c2ws, float(g["depth_min"]), float(g["depth_max"]),
                                         float(g["discard"]))
    call(refs[0])
    for k, ref in enumerate(refs):
        r = m.GetResult()
        if k + 1 < len(refs):
            call(refs[k + 1])
        host.IntegrateScanAsync(bgrs[ref], r.depth, c2ws[ref])
        dev.IntegrateScanFromMvsnet(m)
        _same_volume(host, dev)
        _same_render([host, dev], c2ws[ref])


def test_engine_destroyed_right_after_the_call():
    s = Seq(6, seed=12)
    host, dev = s.fusion(), s.fusion()
    m = DrMvsnet(WEIGHTS)
    s.call(m, 0)
    r = m.GetResult()
    s.call(m, 1)                                   # the next window in flight
    host.IntegrateScanAsync(s.ref_bgr(0), r.depth, s.ref_c2w(0))
    dev.IntegrateScanFromMvsnet(m)
    m.close()                                      # before any synchronisation
    _same_volume(host, dev)
    _same_render([host, dev], s.ref_c2w(0))


def test_next_forward_finished_before_the_integration():
    """Wait() on window k+1's forward: its upload and forward have overwritten the engine's images and stage-3 depth, the
    handoff still holds window k."""
    s = Seq(7, seed=13)
    host, dev = s.fusion(), s.fusion()
    m = DrMvsnet(WEIGHTS)
    s.call(m, 0)
    for k in range(s.n - 1):
        r = m.GetResult()
        s.call(m, k + 1)
        m.Wait()
        host.IntegrateScanAsync(s.ref_bgr(k), r.depth, s.ref_c2w(k))
        dev.IntegrateScanFromMvsnet(m)
        _same_volume(host, dev)
        _same_render([host, dev], s.ref_c2w(k))
    m.GetResult()


def test_get_result_before_the_integration_hands_over_the_new_window():
    s = Seq(6, seed=14)
    host, dev = s.fusion(), s.fusion()
    m = DrMvsnet(WEIGHTS)
    s.call(m, 0)
    m.GetResult()
    s.call(m, 1)
    r1 = m.GetResult()                             # GetResult(k+1) before integrate(k): window k+1 is integrated
    host.IntegrateScanAsync(s.ref_bgr(1), r1.depth, s.ref_c2w(1))
    dev.IntegrateScanFromMvsnet(m)
    _same_volume(host, dev)
    _same_render([host, dev], s.ref_c2w(1))
    dev.IntegrateScanFromMvsnet(m)                 # the same result again, until the next GetResult
    host.IntegrateScanAsync(s.ref_bgr(1), r1.depth, s.ref_c2w(1))
    _same_volume(host, dev)
    _same_render([host, dev], s.ref_c2w(1))


def test_two_engines_feed_one_fusion_and_one_engine_two_fusions():
    a, b = Seq(7, seed=15), Seq(7, seed=16)
    ma, mb = DrMvsnet(WEIGHTS), DrMvsnet(WEIGHTS, precision="fp32")
    host_in, dev_in = a.fusion(), a.fusion()        # fan-in: a's and b's results alternately
    host_out, dev_out1, dev_out2 = a.fusion(), a.fusion(), a.fusion()   # fan-out: a's results into two fusions
    a.call(ma, 0)
    b.call(mb, 0)
    for k in range(a.n):
        ra, rb = ma.GetResult(), mb.GetResult()
        if k + 1 < a.n:
            a.call(ma, k + 1)
            b.call(mb, k + 1)
        s, m, r = (a, ma, ra) if k % 2 == 0 else (b, mb, rb)
        host_in.IntegrateScanAsync(s.ref_bgr(k), r.depth, s.ref_c2w(k))
        dev_in.IntegrateScanFromMvsnet(m)
        host_out.IntegrateScanAsync(a.ref_bgr(k), ra.depth, a.ref_c2w(k))
        dev_out1.IntegrateScanFromMvsnet(ma)
        dev_out2.IntegrateScanFromMvsnet(ma)
        _same_volume(host_in, dev_in)
        _same_volume(host_out, dev_out1)
        _same_volume(host_out, dev_out2)
        _same_render([host_in, dev_in], s.ref_c2w(k))
        _same_render([host_out, dev_out1, dev_out2], a.ref_c2w(k))


def test_tracking_reference_down_the_chain():
    """New call -> render -> tdm_tracker_set_reference_dense(fusion=...) gives the host chain's points and pc_n."""
    s = Seq(6, seed=17)
    host, dev = s.fusion(), s.fusion()
    m = DrMvsnet(WEIGHTS)
    K = s.K
    trk = []
    for _ in range(2):
        t = CudaCoarseTracker(W, H)
        t.init()
        t.setK(W, H, float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]))
        trk.append(t)
    gray = (s.ref_bgr(0).astype(np.float32) @ np.array([0.114, 0.587, 0.299], np.float32)).astype(np.float32)
    s.call(m, 0)
    r = m.GetResult()
    s.call(m, 1)
    host.IntegrateScanAsync(s.ref_bgr(0), r.depth, s.ref_c2w(0))
    dev.IntegrateScanFromMvsnet(m)
    pose = np.asarray(s.ref_c2w(0), np.float32)
    ns = []
    for t, f in zip(trk, (host, dev)):
        f.RenderAsync([pose])
        f.GetRenderResult()
        ns.append(t.setReferenceDense(np.eye(4), 1.0, np.zeros(2), fusion=f, render_index=0, dense_only=True, ref_gray=gray))
    assert ns[0] == ns[1] and ns[0] > 1000
    for x, y in zip(trk[0].getReference(ns[0]), trk[1].getReference(ns[1])):
        assert x.tobytes() == y.tobytes()
    m.GetResult()


def _c_call(f, m, pose=None):
    fp = ctypes.POINTER(ctypes.c_float)
    p = None if pose is None else np.ascontiguousarray(pose, np.float32).ctypes.data_as(fp)
    return lib().tdm_fusion_integrate_mvsnet(None if f is None else f._h, None if m is None else m._h, p)


def test_errors_launch_nothing():
    s = Seq(5, seed=18)
    f = s.fusion()
    f.IntegrateScanAsync(s.ref_bgr(0), np.full((H, W), 2.0, np.float32), s.ref_c2w(0))   # a volume to leave untouched
    f.RenderAsync([s.ref_c2w(0)])
    f.GetRenderResult()
    before = (f.stats(), f.dump_blocks())
    m = DrMvsnet(WEIGHTS)

    def unchanged():
        st, (c, v) = f.stats(), f.dump_blocks()
        assert st == before[0] and np.array_equal(c, before[1][0]) and v.tobytes() == before[1][1].tobytes()

    assert _c_call(None, m) < 0 and "null" in lib().tdm_last_error().decode()
    assert _c_call(f, None) < 0 and "null" in lib().tdm_last_error().decode()
    assert _c_call(f, m) < 0 and "GetResult" in lib().tdm_last_error().decode()        # nothing submitted
    s.call(m, 0)
    assert _c_call(f, m) < 0 and "GetResult" in lib().tdm_last_error().decode()        # submitted, not fetched
    unchanged()
    m.GetResult()
    other = DrFusion(DrFusionOptions(height=H + 32, width=W, fx=float(s.K[0, 0]), fy=float(s.K[1, 1]), cx=float(s.K[0, 2]),
                                     cy=float(s.K[1, 2]), **SMALL))
    assert _c_call(other, m) < 0 and "height / width" in lib().tdm_last_error().decode()
    assert other.stats()["allocated_blocks"] == 0
    assert _c_call(f, m, np.zeros((4, 4))) < 0 and "singular" in lib().tdm_last_error().decode()
    unchanged()
    f.IntegrateScanFromMvsnet(m)                                   # a legal call, then one out of order
    after = (f.stats(), f.dump_blocks())
    assert _c_call(f, m) < 0 and "call order" in lib().tdm_last_error().decode()
    st, (c, v) = f.stats(), f.dump_blocks()
    assert st == after[0] and np.array_equal(c, after[1][0]) and v.tobytes() == after[1][1].tobytes()
    with pytest.raises(TandemError, match="call order"):
        f.IntegrateScanFromMvsnet(m)
    f.RenderAsync([s.ref_c2w(0)])
    f.GetRenderResult()


def test_errors_different_devices():
    if lib().tdm_device_count() < 2:
        pytest.skip("needs two GPUs")
    s = Seq(5, seed=19)
    f = s.fusion()
    m = DrMvsnet(WEIGHTS, device=1)
    s.call(m, 0)
    m.GetResult()
    assert _c_call(f, m) < 0 and "different devices" in lib().tdm_last_error().decode()
    assert f.stats()["allocated_blocks"] == 0
    f.IntegrateScanAsync(s.ref_bgr(0), np.full((H, W), 2.0, np.float32), s.ref_c2w(0))   # the call order is untouched
    f.RenderAsync([s.ref_c2w(0)])
    f.GetRenderResult()


def test_cpp_shim_keyframe_chain(tmp_path):
    """tests/cpp/shim_keyframe.cpp drives DrMvsnet and DrFusion::IntegrateScanAsync(DrMvsnet const&) in CallSequential's
    order; its renders equal the host path's."""
    exe = os.path.join(ROOT, "tests", "cpp", "shim_keyframe")
    if not os.path.exists(exe):
        pytest.skip("tests/cpp/shim_keyframe not built (run __graft_entry__.build())")
    s = Seq(7, seed=20)
    nf = len(s.bgrs)
    inp, outp = tmp_path / "frames.bin", tmp_path / "renders.bin"
    with open(inp, "wb") as fh:
        fh.write(b"TDMK0001")
        fh.write(np.array([nf, V, H, W], np.int32).tobytes())
        fh.write(np.ascontiguousarray(s.K, np.float32).tobytes())
        fh.write(np.array([0.5, 5.0, 2.5], np.float32).tobytes())
        for i in range(nf):
            fh.write(np.ascontiguousarray(s.c2ws[i], np.float32).tobytes())
            fh.write(np.ascontiguousarray(s.bgrs[i], np.uint8).tobytes())
    env = dict(os.environ, TDM_PRECISION="mixed16", TDM_DEVICE="0")
    r = subprocess.run([exe, WEIGHTS, str(inp), str(outp)], capture_output=True, text=True, timeout=300, env=env)
    print(r.stdout[-1000:], r.stderr[-1000:])
    assert r.returncode == 0
    data = outp.read_bytes()
    per = H * W * 4 + H * W * 3
    assert len(data) == s.n * per
    host = s.fusion()
    m = DrMvsnet(WEIGHTS, precision="mixed16")
    s.call(m, 0)
    for k in range(s.n):
        res = m.GetResult()
        if k + 1 < s.n:
            s.call(m, k + 1)
        host.IntegrateScanAsync(s.ref_bgr(k), res.depth, s.ref_c2w(k))
        b, d = _render(host, s.ref_c2w(k))
        assert (d > 0).mean() > 0.3
        assert data[k * per:k * per + H * W * 4] == d.tobytes()
        assert data[k * per + H * W * 4:(k + 1) * per] == b.tobytes()
