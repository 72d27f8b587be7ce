"""CPU-side invariants of the input-stationary tile planner (make_plan_is in tandem_b200/csrc/conv_tc_is.cuh), queried
through tdm_debug_conv_plan_n mode 200 (300: tiles span all D planes) for every stride-1 3x3x3 layer it serves: each stage's conv0 and prob."""
import ctypes

from tandem_b200._lib import lib

IS_MODE = 200
MAX_CH = 8          # kIsMaxCh: 128-position chunks per plane = sub-chunks per consumer warpgroup (register-resident partials)


def _shapes():
    shapes = []
    # 640x480 benchmark window (48/32/8 planes), 320x256 (config-1 window), 512x320 and the abl04 checkpoint's D = 4
    for (H, W, Ds) in [(480, 640, (48, 32, 8)), (256, 320, (32, 32, 8)), (320, 512, (32, 8, 4)), (96, 128, (4, 8, 48))]:
        for s, D in enumerate(Ds):
            sc = 4 >> s
            for cin in (32, 16, 8):
                shapes.append((cin, 16, D, H // sc, W // sc))       # conv0: 8 channels, [hi 8 | lo 8] per kd
            shapes.append((8, 8, D, H // sc, W // sc))              # prob: 1 channel, hi / lo in columns 0 / 1
            shapes.append((8, 8, D, H // sc, W // sc, 300))         # prob with the soft-argmin tail: tiles span all D planes
    return shapes


def test_input_stationary_plans_cover_the_layer_and_fit_the_sm():
    l = lib()
    out = (ctypes.c_longlong * 13)()
    for (cin, cpk, D, H, W, *mode) in _shapes():
        mode = mode[0] if mode else IS_MODE
        rc = l.tdm_debug_conv_plan_n(cin, cpk, 3, D, H, W, 1, mode, 225, out, 13)
        key = (cin, cpk, D, H, W, mode)
        assert rc == 0, (key, l.tdm_last_error())
        S, R, TW, P, DR, nch, slot_pos, tw, th, td, grid, smem, nwg = [int(x) for x in out]
        # the kernel's partial arrays hold 2 * MAX_CH / nwg sub-chunks per warpgroup, exactly its share
        assert nwg in (2, 4) and (2 * MAX_CH) % nwg == 0, (key, nwg)
        # coverage: the tiles partition the output exactly
        assert P == TW + 2 and P <= 256 and R >= 1 and DR >= 1, key
        assert tw * TW >= W and (tw - 1) * TW < W and th * R >= H and (th - 1) * R < H, key
        assert td * DR >= D and (td - 1) * DR < D and grid == tw * th * td, key
        if mode == 300:
            assert td == 1 and DR == D, key
        # ring: every input plane is consumed once, so 2 or 3 slots
        assert 2 <= S <= 3, key
        # registers: two rolling partials per sub-chunk, at most MAX_CH sub-chunks per warpgroup
        assert nch == (R * P + 127) // 128 and 1 <= nch <= MAX_CH, key
        # wgmma m64nNk16 with N = 3 kd blocks: a multiple of 8, at most 256
        n = 3 * cpk
        assert n % 8 == 0 and n <= 256, key
        # shared memory: B image + S slots (each with the A reads' overrun of the last sub-chunk) + barriers
        nblk = 9 * (cin // 16) if cin >= 16 else 5
        assert slot_pos % 8 == 0 and slot_pos >= (R + 2) * P and slot_pos >= nch * 128 + 2 * P + 2, key
        assert smem == (nblk * n * 32 + 127) // 128 * 128 + S * (cin // 8) * slot_pos * 16 + 256, key
        assert smem <= 225 * 1024, key
