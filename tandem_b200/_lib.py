"""ctypes loader for libtandem_b200.so (the C ABI declared in include/tandem_b200.h).

There is deliberately no fallback: if the shared library is missing this raises, and every compute
entry point fails loudly on a box without a CUDA device.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtandem_b200.so")
_lib = None


class TandemError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise TandemError(
                f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                f"or `make -C tandem_b200/csrc` (no CPU fallback exists)")
        _lib = ctypes.CDLL(LIB_PATH)
        _declare(_lib)
    return _lib


def check(rc):
    if rc < 0:
        raise TandemError(lib().tdm_last_error().decode())
    return rc


#: the values tdm_debug_conv_plan_n writes, in order (include/tandem_b200.h; tdm_debug_conv_plan writes the first 12); nwg
#: is the consumer-warpgroup count of the kernel the plan is made for
CONV_PLAN_KEYS = ("S", "R", "TW", "P", "DR", "nch", "slot_pos", "tiles_w", "tiles_h", "tiles_d", "grid", "smem", "nwg")


class FusionOptions(ctypes.Structure):
    """Field-for-field DrFusionOptions (dr_fusion.h:18-36)."""
    _fields_ = [("voxel_size", ctypes.c_float), ("num_buckets", ctypes.c_int), ("bucket_size", ctypes.c_int),
                ("num_blocks", ctypes.c_int), ("block_size", ctypes.c_int), ("max_sdf_weight", ctypes.c_int),
                ("truncation_distance", ctypes.c_float), ("max_sensor_depth", ctypes.c_float),
                ("min_sensor_depth", ctypes.c_float), ("num_render_streams", ctypes.c_int),
                ("fx", ctypes.c_float), ("fy", ctypes.c_float), ("cx", ctypes.c_float), ("cy", ctypes.c_float),
                ("height", ctypes.c_int), ("width", ctypes.c_int)]


class FusionStats(ctypes.Structure):
    _fields_ = [("allocated_blocks", ctypes.c_longlong), ("visible_blocks", ctypes.c_longlong),
                ("dropped_blocks", ctypes.c_longlong), ("candidate_blocks", ctypes.c_longlong)]


class FusionPeerHandle(ctypes.Structure):
    """tdm_fusion_peer_handle (include/tandem_b200.h): one rank's exported hash table + voxel pool."""
    _fields_ = [("keys_ptr", ctypes.c_ulonglong), ("ptrs_ptr", ctypes.c_ulonglong), ("voxels_ptr", ctypes.c_ulonglong),
                ("pid", ctypes.c_longlong), ("device", ctypes.c_int), ("num_buckets", ctypes.c_int), ("bucket_size", ctypes.c_int),
                ("slab_lo", ctypes.c_int), ("slab_hi", ctypes.c_int), ("reserved", ctypes.c_int),
                ("ipc_keys", ctypes.c_ubyte * 64), ("ipc_ptrs", ctypes.c_ubyte * 64), ("ipc_voxels", ctypes.c_ubyte * 64)]


class TrackResult(ctypes.Structure):
    _fields_ = [("ref_to_new", ctypes.c_double * 16), ("aff_g2l", ctypes.c_double * 2), ("res", ctypes.c_double * 6),
                ("iterations", ctypes.c_int), ("evaluations", ctypes.c_int), ("cutoff_repeat", ctypes.c_float), ("device_ms", ctypes.c_float)]


class TrackPyramidResult(ctypes.Structure):
    """tdm_track_pyramid_result (include/tandem_b200.h)."""
    _fields_ = [("ref_to_new", ctypes.c_double * 16), ("aff_g2l", ctypes.c_double * 2), ("last_residuals", ctypes.c_double * 5),
                ("last_flow_indicators", ctypes.c_double * 3), ("ok", ctypes.c_int), ("aborted_level", ctypes.c_int),
                ("repeated_level", ctypes.c_int), ("iterations", ctypes.c_int * 5), ("evaluations", ctypes.c_int * 5),
                ("cutoff_repeat", ctypes.c_float * 5), ("device_ms", ctypes.c_float)]


class TrackTry(ctypes.Structure):
    """tdm_track_try (include/tandem_b200.h)."""
    _fields_ = [("last_residuals", ctypes.c_double * 5), ("ok", ctypes.c_int), ("aborted_level", ctypes.c_int),
                ("repeated_level", ctypes.c_int), ("evaluations", ctypes.c_int * 5)]


class TrackNewCoarseResult(ctypes.Structure):
    """tdm_track_new_coarse_result (include/tandem_b200.h)."""
    _fields_ = [("ref_to_new", ctypes.c_double * 16), ("aff_g2l", ctypes.c_double * 2), ("achieved_res", ctypes.c_double * 5),
                ("flow_vecs", ctypes.c_double * 3), ("have_one_good", ctypes.c_int), ("tries", ctypes.c_int), ("winner", ctypes.c_int),
                ("device_ms", ctypes.c_float)]


def _declare(l):
    c = ctypes
    P = c.POINTER
    vp, f, i, cp = c.c_void_p, c.c_float, c.c_int, c.c_char_p
    fp, dp, ip = P(c.c_float), P(c.c_double), P(c.c_int)
    sigs = {
        "tdm_last_error": (cp, []),
        "tdm_version": (cp, []),
        "tdm_device_count": (i, []),
        "tdm_host_alloc_pinned": (i, [c.c_size_t, P(vp)]),
        "tdm_host_free_pinned": (i, [vp]),
        "tdm_mvsnet_create": (i, [cp, i, i, P(vp)]),
        "tdm_mvsnet_destroy": (None, [vp]),
        "tdm_mvsnet_call_async": (i, [vp, i, i, i, i, P(vp), fp, P(vp), f, f, f]),
        "tdm_mvsnet_call_async_k": (i, [vp, i, i, i, i, P(vp), fp, P(vp), f, f, f]),
        "tdm_mvsnet_call_async_ids": (i, [vp, i, i, i, i, P(c.c_longlong), P(vp), fp, i, P(vp), f, f, f]),
        "tdm_mvsnet_feature_cache": (i, [vp, P(c.c_longlong), i, ip, ip]),
        "tdm_mvsnet_run_resident_new": (i, [vp, i, i, fp, ip]),
        "tdm_mvsnet_get_result": (i, [vp, fp, fp, fp, fp]),
        "tdm_mvsnet_ready": (i, [vp]),
        "tdm_mvsnet_wait": (i, [vp]),
        "tdm_mvsnet_set_option": (i, [vp, cp, i]),
        "tdm_mvsnet_stage_output": (i, [vp, i, cp, fp, c.c_size_t]),
        "tdm_mvsnet_debug_tensor": (c.c_longlong, [vp, cp, fp, c.c_size_t, ip]),
        "tdm_mvsnet_run_resident": (i, [vp, i, fp, ip]),
        "tdm_mvsnet_run_resident_multi": (i, [P(vp), i, i, fp, ip]),
        "tdm_debug_homography": (i, [fp, fp, fp, fp, fp]),
        "tdm_debug_conv_plan": (i, [i, i, i, i, i, i, i, i, i, P(c.c_longlong)]),
        "tdm_debug_conv_plan_n": (i, [i, i, i, i, i, i, i, i, i, P(c.c_longlong), i]),
        "tdm_mvsnet_profile": (c.c_longlong, [vp, cp, c.c_size_t]),
        "tdm_fusion_create": (i, [P(FusionOptions), i, P(vp)]),
        "tdm_fusion_destroy": (None, [vp]),
        "tdm_fusion_integrate_async": (i, [vp, vp, fp, fp]),
        "tdm_fusion_integrate_mvsnet": (i, [vp, vp, fp]),
        "tdm_fusion_render_async": (i, [vp, P(fp), i]),
        "tdm_fusion_get_render_result": (i, [vp, P(vp), P(fp), i]),
        "tdm_fusion_synchronize": (i, [vp]),
        "tdm_fusion_set_slab": (i, [vp, i, i]),
        "tdm_fusion_set_interleave": (i, [vp, i, i, i, i]),
        "tdm_fusion_peer_export": (i, [vp, P(FusionPeerHandle)]),
        "tdm_fusion_peer_attach": (i, [vp, P(FusionPeerHandle), i, i]),
        "tdm_fusion_extract_mesh": (c.c_longlong, [vp, fp, fp, fp, fp, c.c_size_t]),
        "tdm_fusion_extract_mesh_async": (i, [vp, fp, fp]),
        "tdm_fusion_get_mesh": (c.c_longlong, [vp, fp, fp, c.c_size_t]),
        "tdm_fusion_last_mesh_ms": (i, [vp, fp]),
        "tdm_fusion_render_keys_device": (i, [vp, i, P(vp)]),
        "tdm_fusion_unpack_keys": (i, [vp, vp, fp, vp]),
        "tdm_fusion_stream": (i, [vp, P(vp)]),
        "tdm_debug_mesh_axis_table": (i, [f, f, f, ip, fp, ip, ip, i]),
        "tdm_debug_hash_slot": (i, [i, i, i, i, ip]),
        "tdm_fusion_set_option": (i, [vp, cp, i]),
        "tdm_fusion_last_alloc_ms": (i, [vp, fp]),
        "tdm_fusion_get_stats": (i, [vp, P(FusionStats)]),
        "tdm_fusion_dump_blocks": (c.c_longlong, [vp, ip, vp, c.c_size_t]),
        "tdm_fusion_run_resident": (i, [vp, i, fp, fp]),
        "tdm_tracker_create": (i, [i, i, f, f, i, i, P(vp)]),
        "tdm_tracker_destroy": (None, [vp]),
        "tdm_tracker_set_k": (i, [vp, i, i, f, f, f, f]),
        "tdm_tracker_set_reference": (i, [vp, i, fp, fp, fp, fp, f, dp]),
        "tdm_tracker_set_new": (i, [vp, fp]),
        "tdm_tracker_calc_res": (i, [vp, dp, f, dp, f, dp]),
        "tdm_tracker_calc_g": (i, [vp, f, dp, dp, dp]),
        "tdm_tracker_calc_res_g": (i, [vp, dp, f, dp, f, dp, dp, dp]),
        "tdm_tracker_calc_res_batch": (i, [vp, i, dp, f, dp, f, dp]),
        "tdm_tracker_synchronize": (i, [vp]),
        "tdm_tracker_run_resident": (i, [vp, i, fp]),
        "tdm_tracker_get_warped": (i, [vp, i, fp]),
        "tdm_pyramid_create": (i, [i, i, i, i, P(vp)]),
        "tdm_pyramid_destroy": (None, [vp]),
        "tdm_pyramid_build": (i, [vp, fp]),
        "tdm_pyramid_get_level": (i, [vp, i, fp, fp]),
        "tdm_tracker_set_new_from_pyramid": (i, [vp, vp, i]),
        "tdm_tracker_set_reference_dense": (i, [vp, fp, vp, i, dp, i, i, i, fp, fp, fp, fp, fp, fp, vp, f, dp, ip]),
        "tdm_tracker_get_reference": (i, [vp, i, fp, fp, fp, fp]),
        "tdm_tracker_track": (i, [vp, dp, dp, f, f, i, f, i, i, P(TrackResult)]),
        "tdm_tracker_track_pyramid": (i, [P(vp), i, dp, dp, f, f, ip, f, f, f, dp, P(TrackPyramidResult)]),
        "tdm_tracker_track_new_coarse": (i, [P(vp), i, dp, i, dp, f, f, ip, f, f, f, dp, f, P(TrackNewCoarseResult), P(TrackTry)]),
    }
    missing = []
    for name, (res, args) in sigs.items():
        fn = getattr(l, name, None)
        if fn is None:  # reported by tests/test_abi.py; calling a missing entry raises AttributeError
            missing.append(name)
            continue
        fn.restype = res
        fn.argtypes = args
    l._tdm_missing = missing


def pinned_empty(shape, dtype):
    """numpy array over page-locked host memory (tdm_host_alloc_pinned); freed when the array is collected.  DrMvsnet DMA's
    straight from / into such arrays (no staging copy)."""
    import numpy as np
    import weakref
    dt = np.dtype(dtype)
    n = int(np.prod(shape)) * dt.itemsize
    p = ctypes.c_void_p()
    check(lib().tdm_host_alloc_pinned(max(n, 1), ctypes.byref(p)))
    buf = (ctypes.c_char * max(n, 1)).from_address(p.value)
    a = np.frombuffer(buf, dtype=dt, count=int(np.prod(shape))).reshape(shape)
    weakref.finalize(buf, lambda addr=p.value: lib().tdm_host_free_pinned(ctypes.c_void_p(addr)))
    return a


API_SYMBOLS = None


def declared_symbols():
    """All function names declared in include/tandem_b200.h (parsed from the header)."""
    import re
    hdr = os.path.join(os.path.dirname(_HERE), "include", "tandem_b200.h")
    txt = open(hdr).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(tdm_[a-z0-9_]+)\s*\(", txt)))
