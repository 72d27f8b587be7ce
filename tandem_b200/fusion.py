"""Host-side mirror of `class DrFusion` (tandem/libdr/dr_fusion/src/dr_fusion/dr_fusion.h:44-73) over the C ABI.

    f = DrFusion(DrFusionOptions(...))           # defaults = FullSystem::initDr (FullSystem.cpp:259-276)
    f.IntegrateScanAsync(bgr, depth, pose)       # bgr (H,W,3) u8, depth (H,W) f32, pose 4x4 cam->world
    f.RenderAsync([pose])                        # len == num_render_streams
    bgrs, depths = f.GetRenderResult()           # views into the pinned double buffer, valid until the next call
"""
import ctypes

import numpy as np

from ._lib import FusionOptions, FusionStats, TandemError, check, lib


def DrFusionOptions(height=480, width=640, fx=320.0, fy=320.0, cx=319.5, cy=239.5, **kw):
    """DrFusionOptions with the values hard-coded in FullSystem::initDr (FullSystem.cpp:259-276)."""
    o = FusionOptions()
    o.voxel_size = 0.01
    o.num_buckets = 1000000
    o.bucket_size = 10
    o.num_blocks = 1000000
    o.block_size = 8
    o.max_sdf_weight = 64
    o.truncation_distance = 0.04
    o.max_sensor_depth = 10.0
    o.min_sensor_depth = 0.1
    o.num_render_streams = 1
    o.fx, o.fy, o.cx, o.cy = fx, fy, cx, cy
    o.height, o.width = height, width
    for k, v in kw.items():
        if not hasattr(o, k):
            raise TandemError(f"unknown DrFusionOptions field {k}")
        setattr(o, k, v)
    return o


VOXEL_DTYPE = np.dtype([("sdf", "<f4"), ("color", "u1", (3,)), ("weight", "u1")])  # voxel.h:13-21, 8 bytes


class DrFusion:
    def __init__(self, options, device=0):
        self.options = options
        self._h = ctypes.c_void_p()
        check(lib().tdm_fusion_create(ctypes.byref(options), device, ctypes.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None):
            lib().tdm_fusion_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def IntegrateScanAsync(self, bgr, depth, pose):
        o = self.options
        bgr = np.ascontiguousarray(bgr, np.uint8)
        depth = np.ascontiguousarray(depth, np.float32)
        pose = np.ascontiguousarray(pose, np.float32)
        if bgr.size != o.height * o.width * 3 or depth.size != o.height * o.width or pose.size != 16:
            raise TandemError("IntegrateScanAsync: wrong input size")
        fp = ctypes.POINTER(ctypes.c_float)
        check(lib().tdm_fusion_integrate_async(self._h, bgr.ctypes.data, depth.ctypes.data_as(fp), pose.ctypes.data_as(fp)))

    def IntegrateScanFromMvsnet(self, mvsnet, pose=None):
        """IntegrateScanAsync of the result mvsnet.GetResult() last returned, read where it sits on the device: its filtered
        depth, the window's reference BGR image and, with pose=None, the window's reference cam->world pose (what
        tandem_backend.cpp:166 passes).  Non-blocking; legal until the next GetResult replaces the result, also after the
        next CallAsync (include/tandem_b200.h: tdm_fusion_integrate_mvsnet)."""
        fp = ctypes.POINTER(ctypes.c_float)
        if pose is None:
            check(lib().tdm_fusion_integrate_mvsnet(self._h, mvsnet._h, None))
            return
        pose = np.ascontiguousarray(pose, np.float32)
        if pose.size != 16:
            raise TandemError("IntegrateScanFromMvsnet: pose must be 4x4")
        check(lib().tdm_fusion_integrate_mvsnet(self._h, mvsnet._h, pose.ctypes.data_as(fp)))

    def RenderAsync(self, camera_poses):
        poses = [np.ascontiguousarray(p, np.float32) for p in camera_poses]
        fp = ctypes.POINTER(ctypes.c_float)
        arr = (fp * max(len(poses), 1))(*[p.ctypes.data_as(fp) for p in poses])
        check(lib().tdm_fusion_render_async(self._h, arr, len(poses)))
        self._n = len(poses)

    def GetRenderResult(self):
        n = self._n
        o = self.options
        bp = (ctypes.c_void_p * max(n, 1))()
        dp = (ctypes.POINTER(ctypes.c_float) * max(n, 1))()
        check(lib().tdm_fusion_get_render_result(self._h, bp, dp, n))
        bgrs, depths = [], []
        for i in range(n):
            b = np.ctypeslib.as_array(ctypes.cast(bp[i], ctypes.POINTER(ctypes.c_ubyte)), (o.height, o.width, 3))
            d = np.ctypeslib.as_array(dp[i], (o.height, o.width))
            bgrs.append(b)
            depths.append(d)
        return bgrs, depths

    # ---- mesh (dr_fusion.h:56-68) ---------------------------------------------------------------
    def ExtractMeshAsync(self, lower_corner, upper_corner):
        fp = ctypes.POINTER(ctypes.c_float)
        lo = np.ascontiguousarray(lower_corner, np.float32)
        up = np.ascontiguousarray(upper_corner, np.float32)
        check(lib().tdm_fusion_extract_mesh_async(self._h, lo.ctypes.data_as(fp), up.ctypes.data_as(fp)))

    def GetMeshSync(self, max_vertices=60000000):
        """-> (vert (n,3) f32, cols (n,3) f32 rgb in [0,1]); n = 3 * triangles (dr_mesh_num / dr_mesh_vert / dr_mesh_cols)."""
        fp = ctypes.POINTER(ctypes.c_float)
        # the reference copies into 60 M-vertex host arrays; size ours from a first count-only query
        n = check(lib().tdm_fusion_get_mesh(self._h, None, None, 0))
        if n > max_vertices:
            raise TandemError("Did not provide enough storage for mesh.")
        vert = np.empty((n, 3), np.float32)
        cols = np.empty((n, 3), np.float32)
        n2 = check(lib().tdm_fusion_get_mesh(self._h, vert.ctypes.data_as(fp), cols.ctypes.data_as(fp), max(n, 1)))
        assert n2 == n
        self.dr_mesh_num, self.dr_mesh_vert, self.dr_mesh_cols = n, vert, cols
        return vert, cols

    def GetMesh(self, lower_corner, upper_corner):
        """Blocking TsdfVolume::ExtractMesh (no call-order requirement) -> (vert, cols)."""
        fp = ctypes.POINTER(ctypes.c_float)
        lo = np.ascontiguousarray(lower_corner, np.float32)
        up = np.ascontiguousarray(upper_corner, np.float32)
        n = check(lib().tdm_fusion_extract_mesh(self._h, lo.ctypes.data_as(fp), up.ctypes.data_as(fp), None, None, 0))
        vert = np.empty((n, 3), np.float32)
        cols = np.empty((n, 3), np.float32)
        check(lib().tdm_fusion_extract_mesh(self._h, lo.ctypes.data_as(fp), up.ctypes.data_as(fp), vert.ctypes.data_as(fp),
                                            cols.ctypes.data_as(fp), max(n, 1)))
        return vert, cols

    def SaveMeshToFile(self, filename, lower_corner, upper_corner):
        vert, cols = self.GetMesh(lower_corner, upper_corner)
        with open(filename, "w") as f:
            for v, c in zip(vert, cols):
                f.write(f"v {v[0]:g} {v[1]:g} {v[2]:g} {c[0]:g} {c[1]:g} {c[2]:g}\n")
            for i in range(0, len(vert) - 2, 3):
                f.write(f"f {i + 1} {i + 2} {i + 3}\n")

    def last_mesh_ms(self):
        ms = ctypes.c_float()
        check(lib().tdm_fusion_last_mesh_ms(self._h, ctypes.byref(ms)))
        return ms.value

    def set_slab(self, z_block_lo, z_block_hi):
        """Multi-GPU extension: keep only voxel blocks with z_block_lo <= z < z_block_hi (see include/tandem_b200.h)."""
        check(lib().tdm_fusion_set_slab(self._h, int(z_block_lo), int(z_block_hi)))

    def set_interleave(self, rank, world, k_blocks=4, z0_block=0):
        """Interleaved Z-slab partition (include/tandem_b200.h): block row z -> rank ((z - z0) div k) mod world, + halo rows."""
        check(lib().tdm_fusion_set_interleave(self._h, int(rank), int(world), int(k_blocks), int(z0_block)))

    def peer_export(self):
        """bytes of this instance's tdm_fusion_peer_handle (picklable: gather it over the ranks, then peer_attach)."""
        from ._lib import FusionPeerHandle
        h = FusionPeerHandle()
        check(lib().tdm_fusion_peer_export(self._h, ctypes.byref(h)))
        return bytes(h)

    def peer_attach(self, handles, rank):
        """handles: list of world peer_export() blobs in rank order.  Enables the pixel-partitioned ray-cast (tandem_b200.h)."""
        from ._lib import FusionPeerHandle
        arr = (FusionPeerHandle * len(handles))(*[FusionPeerHandle.from_buffer_copy(b) for b in handles])
        check(lib().tdm_fusion_peer_attach(self._h, arr, len(handles), int(rank)))

    def render_keys_device(self, render_index=0):
        """Device pointer (int) of the packed nearest-hit keys of a render + element count (see include/tandem_b200.h)."""
        ptr = ctypes.c_void_p()
        check(lib().tdm_fusion_render_keys_device(self._h, int(render_index), ctypes.byref(ptr)))
        return ptr.value, self.options.height * self.options.width

    def stream(self):
        """cudaStream_t (int) all of this handle's work is ordered on - for collectives enqueued behind the ray-cast."""
        p = ctypes.c_void_p()
        check(lib().tdm_fusion_stream(self._h, ctypes.byref(p)))
        return p.value or 0

    def unpack_keys(self, keys_dev_ptr, out=None):
        o = self.options
        depth, bgr = out if out is not None else (np.empty((o.height, o.width), np.float32), np.empty((o.height, o.width, 3), np.uint8))
        check(lib().tdm_fusion_unpack_keys(self._h, ctypes.c_void_p(keys_dev_ptr), depth.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                                           bgr.ctypes.data))
        return depth, bgr

    def Synchronize(self):
        check(lib().tdm_fusion_synchronize(self._h))

    # ---- introspection used by tests / bench -------------------------------------------------
    def stats(self):
        s = FusionStats()
        check(lib().tdm_fusion_get_stats(self._h, ctypes.byref(s)))
        return dict(allocated_blocks=s.allocated_blocks, visible_blocks=s.visible_blocks,
                    dropped_blocks=s.dropped_blocks, candidate_blocks=s.candidate_blocks)

    def dump_blocks(self, with_voxels=True):
        n = check(lib().tdm_fusion_dump_blocks(self._h, None, None, 0))
        coords = np.empty((n, 3), np.int32)
        vox = np.empty((n, 512), VOXEL_DTYPE) if with_voxels else None
        check(lib().tdm_fusion_dump_blocks(self._h, coords.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                                           vox.ctypes.data if with_voxels else None, n))
        return coords, vox

    def set_option(self, name, value):
        check(lib().tdm_fusion_set_option(self._h, name.encode(), int(value)))

    def last_alloc_ms(self):
        ms = ctypes.c_float()
        check(lib().tdm_fusion_last_alloc_ms(self._h, ctypes.byref(ms)))
        return ms.value

    def run_resident(self, iters):
        a, b = ctypes.c_float(), ctypes.c_float()
        check(lib().tdm_fusion_run_resident(self._h, iters, ctypes.byref(a), ctypes.byref(b)))
        return a.value, b.value
