"""Runs the reference's own code on the inputs of oracle/pins.py and stores what it computed under tests/golden/, so that
the tests pinned against it run on any checkout.  Needs what oracle/ref_build.mk builds into oracle/_ref/ (and, for the
model, the reference's Python sources); the GPU part needs a CUDA device (the stored file was made on an H100).

    make -C oracle -f ref_build.mk REFERENCE=REFERENCE_DIR
    python oracle/gen_reference_pins.py cpu REFERENCE_DIR   # -> tests/golden/reference_pins_cpu.npz
    python oracle/gen_reference_pins.py gpu                 # -> tests/golden/reference_pins_gpu.npz
"""
import ctypes
import os
import sys
import types

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from oracle import pins  # noqa: E402

GOLDEN = os.path.join(REPO, "tests", "golden")
REF_DIR = os.path.join(REPO, "oracle", "_ref")
_fp = ctypes.POINTER(ctypes.c_float)


def cpu(reference_dir):
    import torch
    from oracle.cpu import FrontRef, TrackerOracle
    out = {}
    ref = FrontRef()
    for (size, levels) in pins.MAKE_IMAGES_CASES:
        b = ref.make_images(pins.make_images_input(size), levels)
        for lvl in range(levels):
            out[f"make_images_{size[0]}x{size[1]}_l{lvl}_dI"] = np.array(pins.digest(b[lvl][0]))
            out[f"make_images_{size[0]}x{size[1]}_l{lvl}_ag"] = np.array(pins.digest(b[lvl][1]))
    for (step, with_sparse, size) in pins.DENSE_REF_CASES:
        x = pins.dense_reference_input(step, with_sparse, size)
        n_ref, arrs_ref, T = ref.dense_reference(x["depth"], x["pose_d"], x["pose_r"].astype(np.float64), x["K4"], step,
                                                 x["dense_only"], x["sparse"], x["idepth0"], x["gray_r"])
        k = f"dense_ref_{step}_{int(with_sparse)}_{size[0]}x{size[1]}"
        out[k + "_n"] = np.array(n_ref)
        out[k + "_T"] = np.asarray(T, np.float64)
        for a, name in zip(arrs_ref, ("u", "v", "idepth", "color")):
            out[f"{k}_{name}"] = np.array(pins.digest(a))
    # the reference's LM level loop, driving the CPU tracker oracle through callbacks
    l = ctypes.CDLL(os.path.join(REF_DIR, "liblm_ref.so"))
    l.ref_lm_track_level0.restype = ctypes.c_int
    dp = ctypes.POINTER(ctypes.c_double)
    RES = ctypes.CFUNCTYPE(None, ctypes.c_void_p, dp, ctypes.c_float, dp, ctypes.c_float, dp)
    G = ctypes.CFUNCTYPE(None, ctypes.c_void_p, ctypes.c_float, dp, dp, dp)
    for (start, fix_a, fix_b, cutoff) in pins.LM_CASES:
        c = pins.lm_case()
        t = TrackerOracle(c["w"], c["h"])
        t.setK(c["w"], c["h"], c["fx"], c["fy"], c["cx"], c["cy"])
        t.setReference(c["n"], c["pc_u"], c["pc_v"], c["pc_idepth"], c["pc_color"], c["ref_exposure"], c["ref_aff"])
        t.setNew(c["dInew"])

        def res_cb(_, T16, expo, aff2, cut, out6):
            r = t.calcRes(np.array([T16[i] for i in range(16)]).reshape(4, 4), expo, np.array([aff2[0], aff2[1]]), cut)
            for i in range(6):
                out6[i] = r[i]

        def g_cb(_, expo, aff2, H64, b8):
            H, b = t.calcG(expo, np.array([aff2[0], aff2[1]]))
            for i in range(8):
                b8[i] = b[i]
                for j in range(8):
                    H64[8 * i + j] = H[i, j]
        T = np.ascontiguousarray(pins.lm_start(c, start), np.float64).copy()
        aff = np.array(c["ref_aff"], np.float64).copy()
        out5 = np.zeros(5)
        counts = (ctypes.c_int * 2)()
        ok = l.ref_lm_track_level0(None, RES(res_cb), G(g_cb), T.ctypes.data_as(dp), aff.ctypes.data_as(dp),
                                   ctypes.c_float(c["new_exposure"]), ctypes.c_float(c["ref_exposure"]),
                                   np.array(c["ref_aff"], np.float64).ctypes.data_as(dp), ctypes.c_float(cutoff), int(fix_a),
                                   int(fix_b), out5.ctypes.data_as(dp), counts)
        assert ok == 1
        k = f"lm_{start}_{int(fix_a)}_{int(fix_b)}_{cutoff}"
        out[k + "_counts"] = np.array([counts[0], counts[1]])
        out[k + "_T"], out[k + "_aff"], out[k + "_out5"] = T, aff, out5
    # the reference model itself on a seeded synthetic window (abl03 checkpoint)
    sys.path.insert(0, os.path.join(reference_dir, "cva_mvsnet"))
    pkg = types.ModuleType("models")
    pkg.__path__ = [os.path.join(reference_dir, "cva_mvsnet", "models")]
    sys.modules["models"] = pkg
    from models.cva_mvsnet import CvaMVSNet, StageTensor
    ck = torch.load(os.path.join(reference_dir, "cva_mvsnet", "pretrained", "ablation", "abl03_view_aggregation.ckpt"),
                    map_location="cpu", weights_only=False)
    net = CvaMVSNet(depth_num=ck["hparams"]["MODEL.DEPTH_NUM"], view_aggregation=True).eval()
    net.load_state_dict({k[len("cva_mvsnet."):]: v for k, v in ck["state_dict"].items()})
    img, Ks, c2w = pins.fresh_model_input()
    with torch.no_grad():
        r = net(img[None], StageTensor(*[k[None] for k in Ks]), c2w[None], torch.tensor([0.5]), torch.tensor([5.0]),
                torch.tensor([10.0]))
    for s in range(3):
        for name in ("depth_dense", "depth", "confidence"):
            out[f"model_s{s}_{name}"] = getattr(r[s], name)[0].numpy().astype(np.float32)
    np.savez_compressed(os.path.join(GOLDEN, "reference_pins_cpu.npz"), **out)


def gpu():
    from oracle.cpu import TrackerOracle
    out = {}
    l = ctypes.CDLL(os.path.join(REF_DIR, "libdr_fusion_ref.so"))
    l.ref_fusion_create.restype = ctypes.c_void_p
    # fusion pin: the reference's ray-cast after each of four integrations
    opt, poses, frames, _ = pins.fusion_setup(2, True)
    H, W = opt.height, opt.width
    ref = ctypes.c_void_p(l.ref_fusion_create(ctypes.byref(opt)))
    for k, (pose, (bgr, depth)) in enumerate(zip(poses, frames)):
        b, d = np.ascontiguousarray(bgr), np.ascontiguousarray(depth)
        l.ref_fusion_integrate(ref, ctypes.c_void_p(b.ctypes.data), d.ctypes.data_as(_fp), pose.ctypes.data_as(_fp))
        rp = poses[max(k - 1, 0)] if k % 2 else pose
        rb = np.zeros((H, W, 3), np.uint8)
        rd = np.zeros((H, W), np.float32)
        l.ref_fusion_render(ref, rp.ctypes.data_as(_fp), ctypes.c_void_p(rb.ctypes.data), rd.ctypes.data_as(_fp), H * W)
        out[f"fusion_{k}_depth"], out[f"fusion_{k}_bgr"] = rd, rb
    l.ref_fusion_destroy(ref)
    # tracker pin: the reference's two kernels, one evaluation
    lt = ctypes.CDLL(os.path.join(REF_DIR, "libtracker_ref.so"))
    for size, step in pins.TRACKER_CASES:
        h, w = size
        c = pins.tracker_pin_case(size, step)
        nn = c["n"]
        orc = TrackerOracle(w, h)
        orc.setK(w, h, c["fx"], c["fy"], c["cx"], c["cy"])
        orc.setReference(nn, c["pc_u"], c["pc_v"], c["pc_idepth"], c["pc_color"], c["ref_exposure"], c["ref_aff"])
        aff = orc._aff(c["new_exposure"], c["new_aff"])
        T = np.ascontiguousarray(c["refToNew"], np.float32)
        Ki = np.array([1.0 / c["fx"], 0, -c["cx"] / c["fx"], 0, 1.0 / c["fy"], -c["cy"] / c["fy"], 0, 0, 1], np.float32)
        o7, o45 = np.zeros(7, np.float32), np.zeros(45, np.float32)
        warped = np.zeros((7, nn), np.float32)
        f = ctypes.c_float
        rc_ = lt.ref_tracker_eval(w, h, f(c["fx"]), f(c["fy"]), f(c["cx"]), f(c["cy"]), T.ctypes.data_as(_fp), Ki.ctypes.data_as(_fp),
                                  f(aff[0]), f(aff[1]), f(c["ref_aff"][1]), f(9.0), f(c["cutoffTH"]), nn,
                                  c["pc_u"].ctypes.data_as(_fp), c["pc_v"].ctypes.data_as(_fp), c["pc_idepth"].ctypes.data_as(_fp),
                                  c["pc_color"].ctypes.data_as(_fp), np.ascontiguousarray(c["dInew"]).ctypes.data_as(_fp),
                                  o7.ctypes.data_as(_fp), o45.ctypes.data_as(_fp), warped.ctypes.data_as(_fp))
        assert rc_ == 0
        k = f"tracker_{h}x{w}_{step}"
        idx = pins.warped_sample(nn)
        out[k + "_o7"], out[k + "_o45"] = o7, o45
        out[k + "_warped5"], out[k + "_warped6"] = warped[5][idx], warped[6][idx]
    np.savez_compressed(os.path.join(GOLDEN, "reference_pins_gpu.npz"), **out)


if __name__ == "__main__":
    if sys.argv[1] == "cpu":
        cpu(sys.argv[2])
    elif sys.argv[1] == "gpu":
        gpu()
    else:
        sys.exit("usage: gen_reference_pins.py cpu REFERENCE_DIR | gpu")
