"""Every layer of the 16-bit and fp32 MVSNet forwards against an fp64 reference computed on the engine's own stored input
(oracle/mvsnet_layers.py), with an a-priori per-element error bound; the soft-argmin against fp64, the edge filter bit for
bit.  test_layers_launch_classes runs the windows of oracle/mvsnet_layers.py WINDOWS in fp16 and bf16, which together run
every launch class the tile planners can reach (tests/test_mvsnet_layers_cpu.py checks that they do)."""
import time

import numpy as np
import pytest

from oracle import mvsnet_layers as ML
from oracle.mvsnet_oracle import stage_intrinsics_cpp
from tandem_b200 import DrMvsnet, default_weights
from tandem_b200.synthetic import mvs_plane_window
from tandem_b200.weights_io import load_tdmw

pytestmark = pytest.mark.gpu

_W = {}


def _weights(name):
    if name not in _W:
        _W[name] = load_tdmw(default_weights(name))
    return _W[name]


def _golden(g):
    V = g["bgr"].shape[0]
    return dict(bgrs=[np.ascontiguousarray(g["bgr"][v]) for v in range(V)], c2ws=[np.ascontiguousarray(g["c2w"][v]) for v in range(V)],
                Ks=np.stack([g["K1"], g["K2"], g["K3"]]).astype(np.float32), ref_index=int(g["ref_index"]),
                depth_min=float(g["depth_min"]), depth_max=float(g["depth_max"]), discard=float(g["discard"]))


def _synthetic(V, H, W, seed=0):
    win = mvs_plane_window(V=V, H=H, W=W, seed=seed)
    win["discard"] = 10.0
    return win


def _checkerboard(V, H, W):
    win = _synthetic(V, H, W)
    y, x = np.mgrid[0:H, 0:W]
    for v in range(V):
        b = (((x + v) // 4 + y // 4) % 2 * 255).astype(np.uint8)
        win["bgrs"][v] = np.ascontiguousarray(np.repeat(b[..., None], 3, axis=2))
    return win


def _submit(m, win):
    H, W = win["bgrs"][0].shape[:2]
    V = len(win["bgrs"])
    if "Ks" in win:
        m.CallAsyncStageK(H, W, V, win["ref_index"], win["bgrs"], win["Ks"], win["c2ws"], win["depth_min"], win["depth_max"], win["discard"])
    else:
        m.CallAsync(H, W, V, win["ref_index"], win["bgrs"], win["K"], win["c2ws"], win["depth_min"], win["depth_max"], win["discard"])
    return m.GetResult()


def _engine(weights, precision, dn=None, **opts):
    m = DrMvsnet(default_weights(weights), precision=precision)
    if dn:
        for s, D in enumerate(dn):
            m.set_option(f"depth_num_stage{s + 1}", D)
    for k, v in opts.items():
        m.set_option(k, v)
    return m


def _tensors(m, layers):
    names = set()
    for L in layers:
        names.update(n for n in (L.inp, L.out, L.res, L.res_up2) if n)
    names.update(("f.img", "f.i2b", "f.c3", "f.c0_0", "feat1", "feat2", "feat3"))
    return {n: m.debug_tensor(n) for n in names}


def _paths(m):
    """weight key -> launch path, from the engine's own per-kernel profile ('' = direct FMA kernel)."""
    out = {}
    for name, *_ in m.profile():
        if "[" in name:
            k, p = name[:-1].split("[")
            out[k] = p
        else:
            out[name] = ""
    return out


def check_forward(m, win, weights, precision, dn, opts, label, report, volume=False):
    """All layer checks of the forward m last ran on win (volume: the cost volume too, whose fp64 restatement is the slowest
    reference).  Returns the number of layers checked."""
    w, dn0, _ = _weights(weights)
    dn = tuple(dn or dn0)
    fp32 = precision == "fp32"              # no fused FPN tail, no k_conv00_u8: f.conv0.0 is a direct conv of f.img
    fused_fpn = not fp32 and opts.get("use_tc", 1) == 1
    direct00 = not fp32 and opts.get("direct_conv00", 1) == 1
    layers = ML.layer_table(dn, fused_fpn, direct00)
    T = _tensors(m, layers)
    outs = {(s, k): m.stage_output(s, k) for s in (1, 2, 3) for k in ("depth", "confidence", "depth_dense", "confidence_dense")}
    outs["thr"] = m.debug_tensor("thr")
    outs["edge"] = m.debug_tensor("s3.edge")
    paths = _paths(m)                       # runs two more forwards of the same window: read everything before
    so = lambda s, k: outs[(s, k)]          # noqa: E731
    shapes = {k: v.shape for k, v in T.items()}
    tail = opts.get("fused_regress", 0) == 1
    failures = []

    def record(name, path, ar, y, y_ref, bound, L=None):
        assert np.isfinite(y).all(), f"{label} {name}: non-finite output"
        r = ML.check(name, y, y_ref, bound, ar)
        idx, worst = r.worst
        report.append((label, precision, name, path or "direct", ar.desc, worst))
        if worst > 1.0:
            where = ""
            if L is not None:
                args = ML.plan_args(L, path, shapes, tail and L.plain)
                if args is not None:
                    pl = ML.query_plan(args, opts.get("tc_smem_kb", 225))
                    c, d, h, ww = idx
                    where = f" tile (td, th, tw) {ML.tile_of(args, pl, c, d, h, ww)} of plan {pl}"
            failures.append(f"{label} {name} [{path or 'direct'}]: worst (c, d, h, w) {tuple(int(i) for i in idx)}{where}: "
                            f"err {r.err[idx]:.3e} bound {r.bound[idx]:.3e} ratio {worst:.3f}; "
                            f"{int((r.ratio > 1).sum())} of {r.ratio.size} elements out of bound")

    V = len(win["bgrs"])
    order = [win["ref_index"]] + [v for v in range(V) if v != win["ref_index"]]
    if direct00:
        y_ref, bound, ar = ML.conv00_u8_reference(w, np.stack([win["bgrs"][v] for v in order]), precision)
        record("f.c0_0", paths.get("f.conv0.0", ""), ar, T["f.c0_0"], y_ref, bound)
    else:
        # k_preprocess_bgr: RGB of the reference-first window as exact u8 / 256 (16-bit engines) or as fl32(u8 / 255) (fp32
        # engine, IEEE division as numpy's), channels 3..7 zero
        u8 = np.stack([win["bgrs"][v] for v in order])[..., ::-1].transpose(3, 0, 1, 2).astype(np.float32)
        img = u8 / np.float32(255) if fp32 else u8 / 256
        got = T["f.img"][:3]
        report.append((label, precision, "f.img", "preprocess", "u8 / 255" if fp32 else "u8 / 256", float(np.any(got != img))))
        assert np.array_equal(got.view(np.uint32), img.view(np.uint32)) and not T["f.img"][3:].any(), \
            f"{label}: f.img is not {'u8/255' if fp32 else 'u8/256'} of the window on {int((got != img).sum())} values"
    checked = 0
    for L in layers:
        path = paths.get(L.wkey, "")
        Wt, _ = ML.fold(w, L.conv_w, L.bn, L.bias, L.transposed)
        cin, cout = (Wt.shape[0], Wt.shape[1]) if L.transposed else (Wt.shape[1], Wt.shape[0])
        ar = ML.arith_for(path, precision, cin, cout, 1 if L.dim == 2 else 3, L.plain, L.transposed,
                          residual=bool(L.res or L.res_up2), family=ML.direct_family(L, shapes[L.out]) if fp32 else "")
        # f.img is stored as exact u8/256 on the 16-bit engines: the remaining 256/255 lives in the weights
        scale = 256.0 / 255.0 if L.out == "f.c0_0" and not fp32 else 1.0
        y_ref, bound = ML.reference(L, w, T, ar, scale)
        record(L.out, path, ar, T[L.out], y_ref, bound, L)
        checked += 1
    assert checked == len(layers)
    if fused_fpn:
        y_ref, bound, ar = ML.fused_feat3_reference(w, T, precision)
        record("feat3", paths.get("f.out3b", ""), ar, T["feat3"], y_ref, bound)
    # cost volume and soft-argmin on the engine's own features and logits
    K_st = win["Ks"] if "Ks" in win else np.stack([k.numpy() for k in stage_intrinsics_cpp(win["K"])])
    c2w_ord = [win["c2ws"][v] for v in order]
    prev = None
    for s in (1, 2, 3):
        lg = T[f"s{s}.logits"][0]
        D, H, W = lg.shape
        hy = ML.hypotheses(s, D, win["depth_min"], win["depth_max"], dn[0], prev, H, W)
        d_ref, c_ref, isum, conf_at = ML.regress_reference(lg, hy)
        dtol, itol, ctol = ML.regress_tolerances(D, hy, isum)
        d = so(s, "depth_dense")
        c = so(s, "confidence_dense")
        rd = np.abs(d - d_ref) / dtol
        # where the fp64 isum lies within the fp32 error of an integer, trunc(isum) may go either way: there the engine's
        # confidence must match one of the two windows, and only pixels that took the other window count as flipped
        near = np.abs(isum - np.round(isum)) <= itol
        c_alt = conf_at(np.where(isum >= np.round(isum), isum - 0.5, isum + 0.5))
        e0, e1 = np.abs(c - c_ref), np.abs(c - c_alt)
        flip = near & (e0 > ctol) & (e1 <= ctol)
        rc = np.where(near, np.minimum(e0, e1), e0) / ctol
        report.append((label, precision, f"s{s}.depth_dense", "regress", f"D {D}", float(rd.max())))
        report.append((label, precision, f"s{s}.confidence_dense", "regress", f"D {D}", float(rc.max())))
        print(f"{label} s{s}: {int(near.sum())} pixels with isum within the fp32 error of an integer, {int(flip.sum())} took the other window")
        if rd.max() > 1:
            failures.append(f"{label} s{s}.depth_dense: worst {np.unravel_index(rd.argmax(), rd.shape)} ratio {rd.max():.3f}")
        if rc.max() > 1:
            failures.append(f"{label} s{s}.confidence_dense: worst {np.unravel_index(rc.argmax(), rc.shape)} ratio {rc.max():.3f}")
        if flip.sum() >= 1e-3 * flip.size:
            failures.append(f"{label} s{s}: {int(flip.sum())} of {flip.size} pixels took the other confidence window")
        if volume:
            vol, feats = T[f"s{s}.volume"], T[f"feat{s}"]
            car = ML.cv_arith(precision, opts.get("cv_variant", 3), feats.shape[0], D)
            v_ref, vb, excl = ML.cost_volume_reference(w, s, feats, hy, K_st[s - 1], c2w_ord, car,
                                                       ML.stage_interval(win["depth_min"], win["depth_max"], dn[0], s))
            assert np.isfinite(vol).all() and (np.abs(vol) < 65504 * 32).all(), f"{label} s{s}.volume: not finite or saturated"
            rv = np.where(excl[None], 0.0, np.abs(vol - v_ref) / vb)
            report.append((label, precision, f"s{s}.volume", "cost volume", car.desc, float(rv.max())))
            print(f"{label} s{s}.volume: {int(excl.sum())} of {excl.size} entries excluded (q.z within its error of the 0.001 cut)")
            if rv.max() > 1:
                i = np.unravel_index(rv.argmax(), rv.shape)
                failures.append(f"{label} s{s}.volume [{car.desc}]: worst (c, d, h, w) {tuple(int(k) for k in i)} err "
                                f"{abs(vol[i] - v_ref[i]):.3e} bound {vb[i]:.3e}; {int((rv > 1).sum())} entries out of bound")
            # a pixel whose adaptive range is clamped at 0.001 has its first hypothesis exactly on the cut
            clamped = int((hy[0] <= 0.001).sum()) if s > 1 else 0
            if excl.sum() > clamped + 1e-3 * excl.size:
                failures.append(f"{label} s{s}.volume: {int(excl.sum())} of {excl.size} entries excluded, {clamped} clamped pixels")
        prev = d
    assert not failures, "\n".join(failures)
    check_filter(outs, win["discard"], (3,), label, {3: outs["edge"]})
    return checked


def _outputs(m, stages):
    outs = {(s, k): m.stage_output(s, k) for s in (1, 2, 3) for k in ("depth", "confidence", "depth_dense", "confidence_dense")}
    outs["thr"] = m.debug_tensor("thr")
    return outs, {s: m.debug_tensor(f"s{s}.edge") for s in stages}


def check_filter(outs, discard, stages, label, edges):
    thr = outs["thr"].reshape(-1)
    for s in stages:
        dd, cd = outs[(s, "depth_dense")], outs[(s, "confidence_dense")]
        d_ref, c_ref, e_ref, t_ref = ML.filter_reference(dd, cd, discard)
        e = edges[s][0, 0]
        assert np.array_equal(e.view(np.uint32), e_ref.view(np.uint32)), f"{label} s{s}: edge metric differs on {int((e != e_ref).sum())} pixels"
        assert thr[s - 1].view(np.uint32) == t_ref.view(np.uint32), f"{label} s{s} discard {discard}: threshold {thr[s - 1]!r} != {t_ref!r}"
        assert np.array_equal(outs[(s, "depth")].view(np.uint32), d_ref.view(np.uint32)), f"{label} s{s}: filtered depth"
        assert np.array_equal(outs[(s, "confidence")].view(np.uint32), c_ref.view(np.uint32)), f"{label} s{s}: filtered confidence"


REPORT = []


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    t0 = time.time()
    yield
    worst = {}
    for label, prec, name, path, desc, ratio in REPORT:
        key = (prec, path, desc if path != "regress" else "")
        if ratio >= worst.get(key, (-1,))[0]:
            worst[key] = (ratio, f"{label} {name}")
    print(f"\nworst error / bound per kernel family and precision ({len(REPORT)} checks, {time.time() - t0:.0f} s):")
    for (prec, path, desc), (ratio, where) in sorted(worst.items()):
        print(f"  {prec:8s} {path:10s} {desc:45s} {ratio:8.4f}  ({where})")


SYNTH = [  # (V, H, W, depth numbers): every MAXD instantiation of the regression with D < MAXD and D = MAXD
    (2, 96, 128, (16, 24, 40)),
    (16, 224, 288, (56, 64, 8)),
    (4, 352, 480, (24, 40, 56)),
    (2, 32, 64, (8, 8, 8)),           # single-tile stride-2 layers
]
# fp32: the direct kernels split the output channels of a layer with >= 16 of them over blockIdx.y below 128 * 592 output
# positions (mvsnet.cu conv_inst); 128x96v2 runs every such layer split, 288x224v16 and 480x352v4 run the full-resolution
# FeatureNet layers unsplit and the coarse CostRegNet layers split
SYNTH_PRECISIONS = [(c, "mixed16") for c in SYNTH] + [(c, "fp32") for c in SYNTH if c[0] * c[1] * c[2] <= 4 * 352 * 480]


@pytest.mark.parametrize("V,H,W,dn,precision", [c + (p,) for c, p in SYNTH_PRECISIONS],
                         ids=[f"{c[2]}x{c[1]}v{c[0]}" + ("-fp32" if p == "fp32" else "") for c, p in SYNTH_PRECISIONS])
def test_layers_synthetic_windows(V, H, W, dn, precision):
    win = _synthetic(V, H, W)
    m = _engine("abl03_view_aggregation", precision, dn)
    _submit(m, win)
    if precision == "fp32":
        split = [L.out for L in ML.layer_table(dn, False, False)
                 if not L.plain and "split" in ML.direct_family(L, ML.shapes(V, H, W, dn)[L.out])]
        print(f"{W}x{H}v{V} fp32: {len(split)} layers with the 8-channel split: {split}")
    check_forward(m, win, "abl03_view_aggregation", precision, dn, {}, f"{W}x{H}v{V}", REPORT, volume=H <= 96)


def test_fp32_windows_straddle_the_channel_split():
    """The fp32 windows of test_layers_synthetic_windows run k_conv_direct both with and without the 8-channel split."""
    fams = {ML.direct_family(L, ML.shapes(V, H, W, dn)[L.out])
            for (V, H, W, dn), p in SYNTH_PRECISIONS if p == "fp32" for L in ML.layer_table(dn, False, False)}
    assert any("8-channel split" in f for f in fams) and any("all channels" in f for f in fams), fams


def test_layers_benchmark_window(golden_full):
    win = _golden(golden_full)
    m = _engine("abl03_view_aggregation", "mixed16")
    _submit(m, win)
    check_forward(m, win, "abl03_view_aggregation", "mixed16", None, {}, "640x480", REPORT)


@pytest.mark.parametrize("precision", ["mixed16", "bf16", "fp32"])
def test_layers_four_depth_planes(golden_small, precision):
    """abl04: D = 4 at stages 2 and 3, where conv5 / conv7 run with stride (1, 2, 2) on the direct kernels."""
    win = _golden(golden_small)
    m = _engine("abl04_fewer_depth_planes", precision)
    _submit(m, win)
    check_forward(m, win, "abl04_fewer_depth_planes", precision, None, {}, "512x320", REPORT, volume=True)


OPTIONS = [dict(use_is=0), dict(use_tc=0), dict(prob_direct=1, fused_regress=1, direct_conv00=0), dict(fused_regress=1),
           dict(tc_smem_kb=113), dict(fork_fpn=0, use_pdl=2), dict(cv_variant=4)]


def _run_options(opts, precision, **extra):
    V, H, W, dn = 2, 96, 128, (16, 24, 8)
    win = _synthetic(V, H, W)
    m = _engine("abl03_view_aggregation", precision, dn, **opts, **extra)
    _submit(m, win)
    check_forward(m, win, "abl03_view_aggregation", precision, dn, opts, "128x96v2 " + ",".join(f"{k}={v}" for k, v in opts.items()), REPORT,
                  volume="cv_variant" in opts)


@pytest.mark.parametrize("opts", OPTIONS, ids=["-".join(f"{k}{v}" for k, v in o.items()) for o in OPTIONS])
def test_layers_options(opts):
    _run_options(opts, "mixed16")


@pytest.mark.parametrize("opts", OPTIONS, ids=["-".join(f"{k}{v}" for k, v in o.items()) for o in OPTIONS])
def test_layers_options_bf16(opts):
    """The bf16 engine's own instantiation of every kernel an option selects, with NaN-poisoned activation interiors."""
    _run_options(opts, "bf16", debug_poison=1)


def _run_prob_tail(use_is, precision, **extra):
    V, H, W, dn = 4, 352, 480, (24, 40, 56)
    win = _synthetic(V, H, W)
    opts = dict(fused_regress=1, use_is=use_is)
    m = _engine("abl03_view_aggregation", precision, dn, **opts, **extra)
    _submit(m, win)
    assert sum(r[0].startswith("s") and r[0].endswith("regress") for r in m.profile()) == 0
    check_forward(m, win, "abl03_view_aggregation", precision, dn, opts, f"480x352v4 fused_regress use_is={use_is}", REPORT)


@pytest.mark.parametrize("use_is", [1, 0])
def test_layers_prob_tail_partial_tiles(use_is):
    """fused_regress at 480x352 (D 24 / 40 / 56: RegressTail<32>, <48>, <64>): the soft-argmin tail of the input-stationary
    (use_is=1) and the output-stationary (use_is=0) prob kernel, with partial last tiles along H (and W for the latter)."""
    _run_prob_tail(use_is, "mixed16")


@pytest.mark.parametrize("use_is", [1, 0])
def test_layers_prob_tail_partial_tiles_bf16(use_is):
    _run_prob_tail(use_is, "bf16", debug_poison=1)


def _window_id(w):
    V, H, W, dn, opts, _ = w
    return f"{W}x{H}v{V}-" + "-".join(map(str, dn)) + "".join(f"-{k}{v}" for k, v in opts.items())


@pytest.mark.parametrize("precision", ["mixed16", "bf16"])
@pytest.mark.parametrize("window", ML.WINDOWS, ids=[_window_id(w) for w in ML.WINDOWS])
def test_layers_launch_classes(window, precision):
    """Every launch class the tile planners can reach (tile edges, idle / ragged warpgroups, full register partials, ring
    depth, narrow pitch, N slicing: oracle/mvsnet_layers.py launch_classes), on a fresh engine whose activation interiors
    start as NaN, so that a store a kernel skipped cannot pass as a zero or as a previous forward's value."""
    V, H, W, dn, opts, listed = window
    smem = opts.get("tc_smem_kb", 225)
    hit = set()
    for _, args in ML.window_launches(V, H, W, dn, opts):
        key, cls = ML.launch_classes(args, ML.query_plan(args, smem))
        hit |= {key + (c,) for c in cls}
    assert set(listed) <= hit, f"the window no longer reaches {sorted(set(listed) - hit)}"
    weights = "abl04_fewer_depth_planes" if 4 in dn else "abl03_view_aggregation"
    win = _synthetic(V, H, W)
    m = _engine(weights, precision, dn, debug_poison=1, **opts)
    _submit(m, win)
    check_forward(m, win, weights, precision, dn, opts, _window_id(window), REPORT)


def test_layers_smem_113_at_view_maximum():
    """tc_smem_kb = 113 gives other tilings (e.g. conv0 with partial depth tiles at stage 2 of 288x224)."""
    V, H, W, dn = 16, 224, 288, (56, 64, 8)
    win = _synthetic(V, H, W)
    m = _engine("abl03_view_aggregation", "mixed16", dn, tc_smem_kb=113)
    _submit(m, win)
    check_forward(m, win, "abl03_view_aggregation", "mixed16", dn, dict(tc_smem_kb=113), "288x224v16 smem113", REPORT)


def test_edge_filter_bit_exact():
    """filter_all_stages: the same select state serves three stages per forward and every discard percentage,
    including 0 % (nothing masked) and 100 % (everything above the minimum masked)."""
    win = _synthetic(3, 96, 128, seed=1)
    m = _engine("abl03_view_aggregation", "mixed16", None, filter_all_stages=1)
    for discard in (0.0, 2.5, 10.0, 37.3, 100.0, 10.0):
        win["discard"] = discard
        _submit(m, win)
        outs, edges = _outputs(m, (1, 2, 3))
        check_filter(outs, discard, (1, 2, 3), f"discard={discard}", edges)


def test_replays_are_bit_identical():
    """Eager forward, graph capture, graph replay, a re-plan to another size and back, then run_resident: every debug
    tensor and threshold is bit-identical."""
    win = _synthetic(2, 96, 128)
    other = _synthetic(3, 128, 160, seed=2)
    m = _engine("abl03_view_aggregation", "mixed16", None, filter_all_stages=1)
    layers = ML.layer_table((48, 32, 8), True, True)
    snaps = []

    def snap():
        T = _tensors(m, layers)
        T["thr"] = m.debug_tensor("thr")
        for s in (1, 2, 3):
            for k in ("depth", "confidence", "depth_dense", "confidence_dense"):
                T[f"s{s}.{k}"] = m.stage_output(s, k)
        return T

    for _ in range(3):
        _submit(m, win)
        snaps.append(snap())
    _submit(m, other)
    _submit(m, win)
    snaps.append(snap())
    m.run_resident(2)
    snaps.append(snap())
    for i, S in enumerate(snaps[1:], 1):
        for k, v in snaps[0].items():
            assert np.array_equal(v.view(np.uint32), S[k].view(np.uint32)), f"forward {i}: {k} differs"


def test_saturated_checkerboard_sixteen_views():
    """A 0/255 checkerboard seen by 16 views: every layer stays finite and within its bound.  Reports the largest stored
    fp16 cost-volume value (the volume is stored x 2^-5) against the fp16 maximum 65504."""
    V, H, W, dn = 16, 96, 128, (16, 24, 8)
    win = _checkerboard(V, H, W)
    m = _engine("abl03_view_aggregation", "mixed16", dn)
    _submit(m, win)
    for s in (1, 2, 3):
        vmax = float(np.abs(m.debug_tensor(f"s{s}.volume")).max()) / 32.0
        print(f"checkerboard V=16 s{s}: largest stored volume value {vmax:.1f} of 65504")
        assert vmax < 65504
    check_forward(m, win, "abl03_view_aggregation", "mixed16", dn, {}, "checkerboard 128x96v16", REPORT, volume=True)
