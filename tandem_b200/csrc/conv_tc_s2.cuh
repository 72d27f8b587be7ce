// Stride-2 convolutions (3x3x3 s2 p1 of CostRegNet conv1/conv3/conv5, module.py:544-552; 5x5 s2 p2 of FeatureNet
// conv1.0/conv2.0, module.py:466-474) on wgmma, fed by TILED TMA with element strides.
//
// A stride-2 conv reads input position 2*o + k + c0 (c0 = 1 - pad in padded coordinates) for output o and tap k.  Along
// the flattened (contiguous) W axis that is a stride of two positions = 32 B between MMA rows, which no canonical wgmma
// layout can express.  The TMA engine de-interleaves instead: a tensor map over the P8 tensor with elementStrides
// {1,2,2,1} loads every second column / row, so a tile's input plane lands in shared memory as 4 parity sub-tiles
// (row parity x column parity), each a dense [R + KS/2][TW + KS/2][8] array.  Inside a sub-tile, tap (kh,kw) of output
// (hh,ww) sits at (hh + kh/2)*P + (ww + kw/2): once more a CONSTANT shift of the flattened index, so everything
// downstream (descriptors with SBO = 128 B, register accumulators, epilogue) is the stride-1 machinery of conv_tc.cuh.
// Out-of-bounds rows / columns (the 5x5 kernels reach one position beyond the stored halo) are zero-filled by TMA.
#pragma once
#include "conv_tc.cuh"

namespace tdm {
namespace tc {

constexpr int kMaxTaps = 25;

struct GeomS2 : Tile {     // Tile: OUTPUT grid; P = TW + KS/2, slot_pos = one parity sub-tile
  int oHp, oWp, opd;       // output padded dims / D halo
  long long out_gs;
  int iDp;                 // input padded plane count (D_in + 2*pd_in): tensor-map dim 3 = cg * iDp + plane
  int c0;                  // 1 - pad (0 for 3x3 p1, -1 for 5x5 p2): padded input coordinate = 2*o + k + c0
  int RR;                  // sub-tile rows, R + KS/2
  int relu, cout;
  short tap_off[kMaxTaps + 1];   // position offset of tap t inside a channel group's 4 sub-tiles (table order)
};

template <typename TIn, typename TOut, int CIN, int NPAD, int KD, int KS, int NWG>
__global__ void __launch_bounds__(conv_threads(NWG), 1)
k_conv_tc_s2(const __grid_constant__ CUtensorMap tmap, const TIn* __restrict__ bimg, const float* __restrict__ bias,
             TOut* __restrict__ out, const __grid_constant__ GeomS2 g) {
  constexpr int CG = CIN / 8;
  constexpr int NTAPS = KS * KS;
  constexpr int NBLK = ksteps(CIN, NTAPS);
  constexpr int B_BYTES = KD * NBLK * NPAD * 32;

  extern __shared__ __align__(128) uint8_t smem[];
  const int ns = blockIdx.y;
  const uint32_t sub_bytes = (uint32_t)g.slot_pos * 16u;
  const uint32_t cg_bytes = sub_bytes * 4u;
  Ring<NWG> ring = Ring<NWG>::start(smem, B_BYTES, bimg + (size_t)ns * (B_BYTES / sizeof(TIn)), cg_bytes * CG, g.S);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const TileOrigin o = tile_origin(g);
  const int nin = KD == 3 ? 2 * o.ndo + 1 : o.ndo;

  if (warp == 4 * NWG) {
    // ===================== TMA producer: 4 parity sub-tiles per channel group per input plane =====================
    if (lane == 0) {
      const uint32_t box_bytes = (uint32_t)g.P * (uint32_t)g.RR * 16u;
      const int col0 = 2 * o.w0 + g.c0, row0 = 2 * o.h0 + g.c0;
      ring.produce(nin, box_bytes * 4u * CG, [&](uint8_t* dst, int rp, uint64_t* bar) {
        // padded input plane: 3-D: 2*(d0+od) + kd + c0 (+1 halo, -pad) -> 2*d0 + rp ; 2-D: the view index itself
        const int pp = KD == 3 ? 2 * o.d0 + rp + g.c0 : o.d0 + rp;
#pragma unroll 1
        for (int cg = 0; cg < CG; ++cg) {
#pragma unroll
          for (int sub = 0; sub < 4; ++sub)
            tma_load_4d(dst + (size_t)cg * cg_bytes + (size_t)sub * sub_bytes, &tmap, 0, col0 + (sub & 1), row0 + (sub >> 1),
                        cg * g.iDp + pp, bar);
        }
      });
    }
    return;
  }
  // ===================== consumers: MMA + epilogue =====================
  const int wg = warp >> 2, wq = warp & 3;
  const uint32_t cgb16 = cg_bytes >> 4;
  auto tap_off = [&](int t) -> int { return g.tap_off[t]; };
  auto aoff = [&](int b) -> uint32_t { return kstep_aoff<CIN, NTAPS>(b, cgb16, tap_off); };
  auto alo = [&](int b) -> uint32_t { return kstep_alo<CIN, NTAPS>(b, cgb16, tap_off); };
  const uint32_t sB16 = smem_u32(smem) >> 4;
  const uint32_t b_lbo16 = (uint32_t)(NPAD * 16 >> 4);
  const int nsub = 2 * g.nch;
  ring.wait_weights();
  float bv[NPAD / 8][2];
  load_bias<false>(bv, bias, ns * NPAD, g.cout, lane);
  const FragRows<NWG> fr0(g, o, wg, wq, lane);
  for (int od = 0; od < o.ndo; ++od) {
    const int first = KD == 3 ? 2 * od : od;
    ring.wait(first + KD - 1);
    uint32_t slot16[KD];
#pragma unroll
    for (int kd = 0; kd < KD; ++kd) slot16[kd] = ring.slot16(first + kd);
    const int d = o.d0 + od;
    // this lane's first element of output pixel (h0, w0), column block 0 of the N slice, in plane d; fragment row half i
    // adds its P8 offset (hh * oWp + ww) * 8
    TOut* const ob = out + (((long long)(d + g.opd) * g.oHp + o.h0 + 1) * g.oWp + o.w0 + 1) * 8 + (ns * NPAD / 8) * g.out_gs + 2 * (lane & 3);
    FragRows<NWG> fr = fr0;
    for (int sc = wg; sc < nsub; sc += NWG) {
      float acc[NPAD / 2];
      mma_subchunk<NPAD, TIn, KD, NBLK>(acc, slot16, (uint32_t)sc * 64u, sB16, b_lbo16, aoff, alo);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        if (!fr.in(i)) continue;
        TOut* const op = ob + (fr.hh[i] * g.oWp + fr.ww[i]) * 8;
#pragma unroll
        for (int j = 0; j < NPAD / 8; ++j) {
          if (ns * NPAD + 8 * j >= g.cout) continue;
          float x[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            x[e] = acc[4 * j + 2 * i + e] + bv[j][e];
            if (g.relu) x[e] = fmaxf(x[e], 0.f);
          }
          store2<TOut>(op + j * g.out_gs, x[0], x[1]);
        }
      }
      fr.next(g.P);
    }
    ring.release(first);                   // KD = 3: input planes 2*od and 2*od+1 are dead after output plane od
    if (KD == 3) ring.release(first + 1);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
// tap table order: sub-tile (row parity, col parity) major, then (kh/2, kw/2).  Returns (kh,kw) per table slot.
inline void s2_tap_table(int KS, int P, int sub_pos, std::vector<std::pair<int, int>>& taps, short* off) {
  taps.clear();
  for (int sub = 0; sub < 4; ++sub)
    for (int a = 0; a <= KS / 2; ++a)
      for (int b = 0; b <= KS / 2; ++b) {
        const int kh = 2 * a + (sub >> 1), kw = 2 * b + (sub & 1);
        if (kh >= KS || kw >= KS) continue;
        off[taps.size()] = (short)(sub * sub_pos + a * P + b);
        taps.push_back({kh, kw});
      }
}

struct PlanS2 {
  GeomS2 g;
  int grid;
  size_t smem;
  int nwg;                 // as Plan::nwg
};

// D,H,W: OUTPUT dims.  kd in {1,3}.
inline PlanS2 make_plan_s2(int cin, int npad, int kd, int ks, int D, int H, int W, size_t smem_limit = 225 * 1024) {
  PlanS2 p{};
  const int nblk = ksteps(cin, ks * ks);
  const int hk = ks / 2;
  // a TMA box reads 2 * P columns (every second one): P <= 128
  const TileLimits lim{kd == 3 ? 5 : 3, kd == 3 ? 4 : 2, hk, 4, 128, 16, INT_MAX, 1, false};
  auto amp = [&](int R, int TW, int, int DR) {
    return (double)(2 * R + ks - 2) / (2 * R) * (double)(2 * TW + ks - 2) / (2 * TW) * (kd == 3 ? (double)(2 * DR + 1) / (2 * DR) : 1.0);
  };
  const int nwg = conv_nwg(0, npad, 0);
  auto tile_clk = [&](int DR, int nch) { return (8500.0 + (double)DR * nch * nblk * kd * (45.0 + 0.35 * npad)) * wg_balance(nch, nwg); };
  static_cast<Tile&>(p.g) = plan_tiles(D, H, W, cin / 8, b_image_bytes(kd, nblk, npad), smem_limit, lim, amp, tile_clk, p.smem);
  TDM_CHECK(4 * p.g.slot_pos <= SHRT_MAX, "conv_tc_s2: tap offsets overflow");
  p.g.RR = p.g.R + hk;
  p.grid = p.g.tiles_w * p.g.tiles_h * p.g.tiles_d;
  p.nwg = nwg;
  return p;
}

// B image for the stride-2 kernel: w folded fp32 [tap][cin][cout] with tap = (kd*KS + kh)*KS + kw.
template <typename T>
inline void build_b_image_s2(const float* w, int cin, int cout, int npad, int kd_n, int ks,
                             const std::vector<std::pair<int, int>>& taps, std::vector<T>& img, T (*cvt)(float), int nsplit = 1) {
  const int ntaps = (int)taps.size();
  const int nblk = ksteps(cin, ntaps);
  const size_t slice = (size_t)kd_n * nblk * npad * 16;
  img.assign(slice * nsplit, cvt(0.f));
  for (int kd = 0; kd < kd_n; ++kd)
    for (int b = 0; b < nblk; ++b)
      for (int half = 0; half < 2; ++half)
        for (int nn = 0; nn < cout; ++nn)
          for (int e = 0; e < 8; ++e) {
            const int t = kstep_tap(cin, ntaps, b, half), ci = kstep_ch(cin, b, half) + e;
            if (!kstep_live(cin, ntaps, b, half) || ci >= cin) continue;
            const int tap = (kd * ks + taps[t].first) * ks + taps[t].second;
            const int n = nn % npad;
            T* simg = img.data() + slice * (nn / npad);
            simg[b_index(kd * nblk + b, half, n, e, npad)] = cvt(w[((size_t)tap * cin + ci) * cout + nn]);
          }
}

}  // namespace tc
}  // namespace tdm
