"""CPU-side checks of the drop-in boundary: the shared library loads without a GPU, exports every symbol that
include/tandem_b200.h declares, and refuses to compute without a CUDA device (no CPU fallback)."""
import ctypes
import os
import re

import numpy as np
import pytest

from tandem_b200._lib import LIB_PATH, declared_symbols, lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_loads_and_exports_every_declared_symbol():
    l = lib()
    assert l._tdm_missing == []
    raw = ctypes.CDLL(LIB_PATH)
    names = declared_symbols()
    assert len(names) >= 35
    for n in names:
        assert hasattr(raw, n), f"{n} declared in include/tandem_b200.h but not exported"
    assert b"sm_90a" in l.tdm_version()


def test_header_cites_reference_interfaces():
    txt = open(os.path.join(ROOT, "include", "tandem_b200.h")).read()
    for cite in ("dr_mvsnet.h:36-66", "dr_fusion.h:44-73", "cuda_coarse_tracker.h:9-82"):
        assert cite in txt


def test_no_cpu_fallback():
    from tandem_b200 import CudaCoarseTracker, DrFusion, DrFusionOptions, DrMvsnet, TandemError, default_weights
    if lib().tdm_device_count() > 0:
        pytest.skip("GPU present")
    with pytest.raises(TandemError, match="no CPU fallback"):
        DrMvsnet(default_weights())
    with pytest.raises(TandemError, match="no CPU fallback"):
        DrFusion(DrFusionOptions())
    t = CudaCoarseTracker(640, 480)
    with pytest.raises(TandemError, match="no CPU fallback"):
        t.init()


def test_product_does_not_import_oracle():
    """Only tests/, __graft_entry__.smoke() and bench.py may touch oracle/."""
    pat = re.compile(r"^\s*(from|import)\s+oracle|oracle/|oracle\.", re.M)
    for dp, _, fs in os.walk(os.path.join(ROOT, "tandem_b200")):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                src = open(os.path.join(dp, f)).read()
                code = "\n".join(l for l in src.splitlines() if not l.strip().startswith(("//", "#", "*", '"""')))
                assert not re.search(r"^\s*(from|import)\s+oracle", code, re.M), f"{f} imports the oracle"
                assert "oracle/_build" not in code and "libtsdf_oracle" not in code, f


def test_mesh_axis_tables_match_a_float32_restatement():
    """Host logic of the mesh extractor (no GPU): the per-axis cell table equals an independent float32 restatement of
    mesh_extractor.cu:248-261 + TrilinearInterpolation's index arithmetic (:28-34) + WorldToGlobalVoxel (tsdf_volume.cu:109-113),
    and every cell is owned by exactly one voxel block whose 12-voxel tile contains all its reads."""
    f32 = np.float32
    l = lib()
    for lower, upper, s in [(-1.28, 1.28, 0.01), (-1.2345, 1.3, 0.01), (0.105, 0.9, 0.01), (-5.0, 5.0, 0.01), (3.3, -0.7, 0.02)]:
        cap = 4096
        ints = np.zeros((cap, 5), np.int32); flts = np.zeros((cap, 4), np.float32); rng = np.zeros((cap, 2), np.int32)
        bm = np.zeros(2, np.int32)
        ip, fp = ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_float)
        n = l.tdm_debug_mesh_axis_table(lower, upper, s, ints.ctypes.data_as(ip), flts.ctypes.data_as(fp), rng.ctypes.data_as(ip),
                                        bm.ctypes.data_as(ip), cap)
        lo, up, vs = f32(lower), f32(upper), f32(s)
        assert n == int(f32(abs(lo - up)) / vs) and 0 < n <= cap
        h = vs / f32(2)

        def w2g(x):
            x = f32(x)
            sg = f32(int(x > 0) - int(x < 0))
            return int(f32(f32(x / vs) + f32(sg * f32(0.5))))

        for i in list(range(0, n, max(1, n // 97))) + [n - 1]:
            # fp32 fma: product and sum are exact in 80-bit extended precision (12 + 24 bits, then one add), one rounding to fp32
            pos = f32(np.longdouble(i) * np.longdouble(vs) + np.longdouble(lo))
            cM, cP = f32(pos + (-h)), f32(pos + h)
            exp = []
            for c in (cM, cP):
                pd = f32(c - h)
                exp += [w2g(f32(pd + f32(0))), w2g(f32(pd + vs))]
            exp.append(w2g(pos))
            assert list(ints[i]) == exp, (lower, upper, i, list(ints[i]), exp)
            vpM, vpP = f32(cM / vs), f32(cP / vs)
            assert flts[i, 0] == f32(vpM - np.floor(vpM)) and flts[i, 1] == f32(vpP - np.floor(vpP))
            assert flts[i, 2] == cM and flts[i, 3] == cP
        # ownership: contiguous, disjoint cell ranges per block, every read inside the 12-voxel tile of the owner
        first, nb = int(bm[0]), int(bm[1])
        covered = 0
        for b in range(nb):
            a, c = int(rng[b, 0]), int(rng[b, 1])
            if c == 0:
                continue
            assert a == covered
            covered += c
            blk = first + b
            g = ints[a:a + c]
            assert (g[:, 0] >> 3 == blk).all() and g.min() >= 8 * blk and g.max() < 8 * blk + 12
        assert covered == n


def test_wgmma_tile_planner_invariants():
    """Host logic of the wgmma convolutions (no GPU): for every layer shape of the benchmark config (640x480, 7 views,
    (48,32,8)) and of the small config-1 windows the planner returns a tiling that covers the grid, fits 225 KB of shared
    memory, the wgmma N limit and the TMA box limit.  Stride-2 plans (mode 400) read sub-tiles of pitch P = TW + KS/2,
    whose TMA boxes span 2 * P columns."""
    l = lib()
    out = (ctypes.c_longlong * 13)()
    shapes = []
    for (H, W, V, Ds) in [(480, 640, 7, (48, 32, 8)), (256, 320, 4, (32, 32, 8)), (96, 128, 2, (32, 8, 8))]:
        # FeatureNet: 2-D convs over V planes (kd = 1, pd = 0)
        for cin, npad, sc in [(8, 32, 1), (16, 32, 2), (32, 64, 4), (32, 32, 2), (32, 32, 1)]:
            shapes.append((cin, npad, 1, V, H // sc, W // sc, 0, 0))
        shapes.append((32, 64, 1, V, H // 2, W // 2, 0, 3))                 # f.out3a: up-2 conv on the coarse grid
        # conv1.0 / conv2.0: 5x5 stride 2 (pd carries the kernel size, D H W are the output dims)
        for cin, npad, sc in [(8, 16, 2), (16, 32, 4)]:
            shapes.append((cin, npad, 1, V, H // sc, W // sc, 5, 400))
        for s, D in enumerate(Ds):
            sc = 4 >> s
            h, w = H // sc, W // sc
            c0 = (32, 16, 8)[s]
            shapes.append((c0, 32, 3, D, h, w, 1, 0))                       # conv0, hi/lo (N = 2 x 16), 3 kd
            shapes.append((8, 32, 3, D, h, w, 1, 0))                        # prob
            shapes.append((8, 32, 3, D, h, w, 1, 100))                      # prob with the soft-argmin tail: tiles span all D planes
            for lvl, (cin, npad) in enumerate([(16, 32), (32, 32), (64, 32)]):
                d2, h2, w2 = max(D >> (lvl + 1), 1), h >> (lvl + 1), w >> (lvl + 1)
                shapes.append((cin, npad, 3, d2, h2, w2, 1, 0))             # conv2 / conv4 / conv6
            for lvl, (cin, npad) in enumerate([(16, 64), (32, 128), (64, 64)]):
                d2, h2, w2 = max(D >> (lvl + 1), 1), h >> (lvl + 1), w >> (lvl + 1)
                shapes.append((cin, npad, 2, d2, h2, w2, 1, 1))             # conv11 / conv9 / conv7 (transposed as GEMM)
            for lvl, (cin, npad) in enumerate([(8, 16), (16, 32), (32, 32)]):
                d2, h2, w2 = max(D >> (lvl + 1), 1), h >> (lvl + 1), w >> (lvl + 1)
                shapes.append((cin, npad, 3, d2, h2, w2, 3, 400))           # conv1 / conv3 / conv5: 3x3x3 stride 2
    assert len(shapes) > 40
    for (cin, npad, kd, D, H, W, pd, mode) in shapes:
        rc = l.tdm_debug_conv_plan_n(cin, npad, kd, D, H, W, pd, mode, 225, out, 13)
        assert rc == 0, (cin, npad, kd, D, H, W, mode, l.tdm_last_error())
        S, R, TW, P, DR, nch, slot_pos, tw, th, td, grid, smem, nwg = [int(x) for x in out]
        assert nwg in (2, 4), (cin, npad, kd, D, H, W, mode, nwg)       # consumer warpgroups of 128 threads + 1 producer warp
        if mode >= 100 and mode != 400:
            assert td == 1 and DR == D, (D, H, W, DR, td)
            mode -= 100
        key = (cin, npad, kd, D, H, W, mode)
        if mode == 400:
            ks = pd
            # 4 parity sub-tiles per channel group, each (R + KS/2) rows of P positions, and the A reads of the last chunk
            assert P == TW + ks // 2 and 2 * P <= 256 and R >= 1 and DR >= 1 and 2 <= S <= 5, key
            assert tw * TW >= W and (tw - 1) * TW < W and th * R >= H and (th - 1) * R < H and td * DR >= D and (td - 1) * DR < D, key
            assert grid == tw * th * td and grid >= 1 and nch == (R * P + 127) // 128, key
            assert slot_pos % 8 == 0 and slot_pos >= (R + ks // 2) * P and slot_pos >= nch * 128 + (ks // 2) * (P + 1), key
            assert smem <= 225 * 1024 and 4 * slot_pos <= 32767, key
            continue
        assert P == TW + 2 and P <= 256 and R >= 1 and DR >= 1 and 2 <= S <= 4, key
        assert tw * TW >= W and (tw - 1) * TW < W and th * R >= H and (th - 1) * R < H and td * DR >= D and (td - 1) * DR < D, key
        assert grid == tw * th * td and grid >= 1, key
        assert nch == (R * P + 127) // 128 and npad % 8 == 0 and npad <= 256, key      # wgmma m64nNk16: N <= 256
        assert smem <= 225 * 1024 and slot_pos % 8 == 0 and slot_pos >= (R + 2) * P, key


def test_conv_plan_twelve_value_entry_point_writes_twelve():
    """tdm_debug_conv_plan keeps its 12-entry output for existing callers; tdm_debug_conv_plan_n adds the warpgroup count."""
    l = lib()
    for args in [(8, 32, 1, 7, 480, 640, 0, 0), (8, 8, 3, 48, 120, 160, 1, 300), (32, 32, 3, 8, 30, 40, 3, 400)]:
        a = (ctypes.c_longlong * 13)(*([-7] * 13))
        b = (ctypes.c_longlong * 13)()
        assert l.tdm_debug_conv_plan(*args, 225, a) == 0 and l.tdm_debug_conv_plan_n(*args, 225, b, 13) == 0, l.tdm_last_error()
        assert list(a[:12]) == list(b[:12]) and a[12] == -7 and b[12] in (2, 4), (args, list(a), list(b))
    c = (ctypes.c_longlong * 14)()
    assert l.tdm_debug_conv_plan_n(8, 32, 1, 7, 480, 640, 0, 0, 225, c, 14) != 0


def test_constant_division_is_correctly_rounded(tmp_path):
    """The TSDF ray-cast replaces div.rn.f32 by a 3-instruction FMA sequence for its constant divisors (cdiv_ in
    tandem_b200/csrc/fusion.cu: voxel_size, fx, fy).  Parity with the oracle's `/` rests on that sequence being CORRECTLY ROUNDED:
    checked exhaustively for the deployment's voxel size 0.01f over every float the ray-cast can produce (|x| in [1e-6, 4096]),
    for the config intrinsics over the pixel-ray range, and on 2e8 random (x, d) pairs."""
    import ctypes
    import subprocess
    src = os.path.join(ROOT, "tests", "cpp", "cdiv_check.c")
    so = str(tmp_path / "libcdiv_check.so")
    subprocess.run(["gcc", "-O2", "-mfma", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-o", so, src, "-lm"], check=True)
    l = ctypes.CDLL(so)
    l.cdiv_check_exhaustive.restype = ctypes.c_long
    l.cdiv_check_exhaustive.argtypes = [ctypes.c_float, ctypes.c_float, ctypes.c_float]
    l.cdiv_check_random.restype = ctypes.c_long
    l.cdiv_check_random.argtypes = [ctypes.c_uint64, ctypes.c_long]
    assert l.cdiv_check_exhaustive(0.01, 1e-6, 4096.0) == 0
    for fx in (320.0, 80.0, 300.0, 525.0, 481.2):
        assert l.cdiv_check_exhaustive(fx, 1e-3, 16384.0) == 0
    assert l.cdiv_check_random(1, 200_000_000) == 0


def test_division_free_hash_equals_the_reference_expression():
    """Host logic (no GPU): the bucket the voxel-hashing kernels compute with a precomputed reciprocal (fast_umod, fusion.cu)
    equals ((x * 73856093) ^ (y * 19349669) ^ (z * 83492791)) % num_buckets on 32-bit ints with the +num_buckets fix-up
    (hash_table.cu:157-168) - against the C expression compiled beside it and against Python's integers."""
    import random
    l = lib()
    ref = ctypes.c_int(0)
    rnd = random.Random(7)
    edge = [0, 1, -1, 2, -2, (1 << 20) - 1, -(1 << 20) + 1, 12345, -54321]
    for n in (1, 2, 3, 7, 10, 1000, 200003, 999983, 1000000, 1000003, 1 << 20, (1 << 31) - 1):
        pts = [(x, y, z) for x in edge for y in edge[:4] for z in edge[:4]]
        pts += [tuple(rnd.randint(-(1 << 20), 1 << 20) for _ in range(3)) for _ in range(4000)]
        for x, y, z in pts:
            got = l.tdm_debug_hash_slot(x, y, z, n, ctypes.byref(ref))
            h = ((x * 73856093) & 0xFFFFFFFF) ^ ((y * 19349669) & 0xFFFFFFFF) ^ ((z * 83492791) & 0xFFFFFFFF)
            h -= (h >> 31) << 32
            assert got == ref.value == h % n, (n, x, y, z, got, ref.value, h % n)
    assert l.tdm_debug_hash_slot(1, 2, 3, 0, None) < 0          # rejected, not a division by zero

