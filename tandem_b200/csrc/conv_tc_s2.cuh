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

struct GeomS2 {
  int D, H, W;             // OUTPUT dims
  int oHp, oWp, opd;       // output padded dims / D halo
  long long out_gs;
  int iDp;                 // input padded plane count (D_in + 2*pd_in): tensor-map dim 3 = cg * iDp + plane
  int ipd;                 // input D halo (1: 3-D, 0: 2-D over views)
  int c0;                  // 1 - pad (0 for 3x3 p1, -1 for 5x5 p2): padded input coordinate = 2*o + k + c0
  int R, TW, DR, P, RR;    // tile rows / cols / planes (output coords); sub-tile pitch P = TW + KS/2, rows RR = R + KS/2
  int nch, sub_pos, S;
  int tiles_w, tiles_h, tiles_d;
  int relu, cout;
  int ntaps;               // KS*KS
  short tap_off[kMaxTaps + 1];   // position offset of tap t inside a channel group's 4 sub-tiles (table order)
};

template <int CIN, int KS> constexpr int s2_blocks() { return CIN >= 16 ? KS * KS * (CIN / 16) : (KS * KS + 1) / 2; }

template <typename TIn, typename TOut, int CIN, int NPAD, int KD, int KS>
__global__ void __launch_bounds__(kThreads, 1)
k_conv_tc_s2(const __grid_constant__ CUtensorMap tmap, const TIn* __restrict__ bimg, const float* __restrict__ bias,
             TOut* __restrict__ out, const __grid_constant__ GeomS2 g) {
  constexpr int CG = CIN / 8;
  constexpr int NBLK = s2_blocks<CIN, KS>();
  constexpr int B_BYTES = KD * NBLK * NPAD * 32;

  extern __shared__ __align__(128) uint8_t smem[];
  const int ns = blockIdx.y;
  bimg += (size_t)ns * (B_BYTES / sizeof(TIn));
  uint8_t* sB = smem;
  uint8_t* sA = smem + ((B_BYTES + 127) / 128) * 128;
  const uint32_t sub_bytes = (uint32_t)g.sub_pos * 16u;
  const uint32_t cg_bytes = sub_bytes * 4u;
  const uint32_t slot_bytes = cg_bytes * CG;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sA + (size_t)slot_bytes * g.S);
  uint64_t* full = bars;
  uint64_t* empty = bars + 8;
  uint64_t* b_full = bars + 16;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  int tile = blockIdx.x;
  const int tw = tile % g.tiles_w; tile /= g.tiles_w;
  const int th = tile % g.tiles_h; tile /= g.tiles_h;
  const int td = tile;
  const int w0 = tw * g.TW, h0 = th * g.R, d0 = td * g.DR;
  const int ndo = min(g.DR, g.D - d0);
  const int nin = KD == 3 ? 2 * ndo + 1 : ndo;

  if (threadIdx.x == 0) {
    for (int s = 0; s < g.S; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4 * kConsumerWG); }
    mbar_init(b_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(b_full, B_BYTES);          // weights do not depend on the previous kernel: fetch them before pdl_wait
    bulk_g2s(sB, bimg, B_BYTES, b_full);
  }
  __syncthreads();
  pdl_wait();   // from here on activations written by the previous kernel are read and our outputs are written
  // trigger the dependents only now: a trigger BEFORE the wait lets the whole chain of later kernels become resident early (each
  // one's prologue would trigger the next), and their idle CTAs then hold the shared memory the running kernel's tiles need
  if (threadIdx.x == 0) pdl_launch_dependents();

  if (warp == kProducerWarp) {
    // ===================== TMA producer: 4 parity sub-tiles per channel group per input plane =====================
    if (lane == 0) {
      const uint32_t box_bytes = (uint32_t)g.P * (uint32_t)g.RR * 16u;
      const int col0 = 2 * w0 + g.c0, row0 = 2 * h0 + g.c0;
      for (int rp = 0; rp < nin; ++rp) {
        const int slot = rp % g.S;
        if (rp >= g.S) mbar_wait(&empty[slot], ((rp / g.S) - 1) & 1);
        mbar_expect_tx(&full[slot], box_bytes * 4u * CG);
        // padded input plane: 3-D: 2*(d0+od) + kd + c0 (+1 halo, -pad) -> 2*d0 + rp ; 2-D: the view index itself
        const int pp = KD == 3 ? 2 * d0 + rp + g.c0 : d0 + rp;
#pragma unroll 1
        for (int cg = 0; cg < CG; ++cg) {
          uint8_t* dst = sA + (size_t)slot * slot_bytes + (size_t)cg * cg_bytes;
#pragma unroll
          for (int sub = 0; sub < 4; ++sub)
            tma_load_4d(dst + (size_t)sub * sub_bytes, &tmap, 0, col0 + (sub & 1), row0 + (sub >> 1), cg * g.iDp + pp, &full[slot]);
        }
      }
    }
    return;
  }
  // ===================== consumers: MMA + epilogue =====================
  const int wg = warp >> 2, wq = warp & 3;
  const uint32_t cgb16 = cg_bytes >> 4;
  auto aoff = [&](int b) -> uint32_t {
    if constexpr (CIN >= 16) {
      return (uint32_t)(2 * (b % (CIN / 16))) * cgb16 + (uint32_t)g.tap_off[b / (CIN / 16)];
    } else {
      // taps paired in table (= address) order; an odd last tap is paired with its predecessor against zero weights
      const int t1 = min(2 * b + 1, g.ntaps - 1);
      return (uint32_t)g.tap_off[t1 - 1];
    }
  };
  auto alo = [&](int b) -> uint32_t {
    if constexpr (CIN >= 16) {
      return cgb16;
    } else {
      const int t1 = min(2 * b + 1, g.ntaps - 1);
      return (uint32_t)(g.tap_off[t1] - g.tap_off[t1 - 1]);
    }
  };
  const uint32_t sB16 = smem_u32(sB) >> 4, sA16 = smem_u32(sA) >> 4;
  const uint32_t b_lbo16 = (uint32_t)(NPAD * 16 >> 4);
  const int nsub = 2 * g.nch;
  mbar_wait(b_full, 0);
  int next_wait = 0;
  for (int od = 0; od < ndo; ++od) {
    const int first = KD == 3 ? 2 * od : od;
    while (next_wait <= first + KD - 1) {
      mbar_wait(&full[next_wait % g.S], (next_wait / g.S) & 1);
      ++next_wait;
    }
    uint32_t slot16[KD];
#pragma unroll
    for (int kd = 0; kd < KD; ++kd) slot16[kd] = sA16 + (uint32_t)((first + kd) % g.S) * (slot_bytes >> 4);
    const int d = d0 + od;
    for (int sc = wg; sc < nsub; sc += kConsumerWG) {
      float acc[NPAD / 2];
      mma_subchunk<NPAD, TIn, KD, NBLK>(acc, slot16, (uint32_t)sc * 64u, sB16, b_lbo16, aoff, alo);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int l = sc * 64 + wq * 16 + (lane >> 2) + 8 * i;
        const int hh = l / g.P, ww = l - hh * g.P;
        const int h = h0 + hh, w = w0 + ww;
        if (!(hh < g.R && ww < g.TW && h < g.H && w < g.W)) continue;
        const long long pos = ((((long long)(d + g.opd)) * g.oHp + (h + 1)) * g.oWp + (w + 1)) * 8;
#pragma unroll
        for (int j = 0; j < NPAD / 8; ++j) {
          const int co = ns * NPAD + 8 * j;
          if (co >= g.cout) continue;
          const int c = co + 2 * (lane & 3);
          float x[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            x[e] = acc[4 * j + 2 * i + e] + (bias ? bias[c + e] : 0.f);
            if (g.relu) x[e] = fmaxf(x[e], 0.f);
          }
          store2<TOut>(out + pos + (co >> 3) * g.out_gs + (c & 7), x[0], x[1]);
        }
      }
    }
    __syncwarp();
    if (lane == 0) {               // input planes no longer read by this warp -> producer may refill
      if (KD == 3) {               // input planes 2*od and 2*od+1 are dead after output plane od
        mbar_arrive(&empty[(2 * od) % g.S]);
        mbar_arrive(&empty[(2 * od + 1) % g.S]);
      } else {
        mbar_arrive(&empty[od % g.S]);
      }
    }
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
};

// D,H,W: OUTPUT dims.  kd in {1,3}.
inline PlanS2 make_plan_s2(int cin, int npad, int kd, int ks, int D, int H, int W, size_t smem_limit = 225 * 1024) {
  PlanS2 p{};
  GeomS2& g = p.g;
  g.D = D; g.H = H; g.W = W;
  const int cg = cin / 8;
  const int nblk = cin >= 16 ? ks * ks * (cin / 16) : (ks * ks + 1) / 2;
  const size_t bbytes = (((size_t)kd * nblk * npad * 32) + 127) / 128 * 128;
  const int hk = ks / 2;
  double best_cost = 1e30;
  int bR = 0, bTW = 0, bS = 0, bDR = 0;
  const int s_hi = kd == 3 ? 5 : 3, s_lo = kd == 3 ? 4 : 2;
  for (int S = s_hi; S >= s_lo; --S) {
    for (int tiles_w = 1; tiles_w <= 20; ++tiles_w) {
      const int TW = (W + tiles_w - 1) / tiles_w;
      if (TW + hk > 128) continue;             // TMA box dim 2*P <= 256
      if (tiles_w > 1 && TW < 16) break;
      const int tw_n = (W + TW - 1) / TW;
      const int P = TW + hk;
      for (int R = 1; R <= 32 && R <= H; ++R) {
        const int RR = R + hk;
        if (2 * RR > 256) break;
        const int nch = (R * P + 127) / 128;
        int sub_pos = std::max(RR * P, nch * 128 + hk * (P + 1)) + 8;
        sub_pos = (sub_pos + 7) / 8 * 8;       // 128-byte aligned TMA destinations
        const size_t smem = bbytes + (size_t)S * cg * 4 * sub_pos * 16 + 256;
        if (smem > smem_limit || sub_pos * 4 > 32000) break;
        const int th_n = (H + R - 1) / R;
        for (int dsplit = 1; dsplit <= D; ++dsplit) {
          const int DR = (D + dsplit - 1) / dsplit;
          const int td_n = (D + DR - 1) / DR;
          const double T = (double)tw_n * th_n * td_n;
          const double amp = (double)(2 * R + ks - 2) / (2 * R) * (double)(2 * TW + ks - 2) / (2 * TW) *
                             (kd == 3 ? (double)(2 * DR + 1) / (2 * DR) : 1.0);
          // same time model as conv_tc.cuh::make_plan
          const double tile_clk = 8500.0 + (double)DR * nch * nblk * kd * (45.0 + 0.35 * npad);
          const double cost = std::ceil(T / 132.0) * tile_clk * (1.0 + 0.25 * (amp - 1.0)) * (S == s_hi ? 1.0 : 1.05);
          if (cost < best_cost - 1e-9) { best_cost = cost; bR = R; bTW = TW; bS = S; bDR = DR; }
          if (T > 4000) break;
        }
      }
    }
    if (bR > 0 && S == s_hi) break;
  }
  if (bR == 0 && smem_limit < 225 * 1024) return make_plan_s2(cin, npad, kd, ks, D, H, W, 225 * 1024);   // soft limit
  TDM_CHECK(bR > 0, "conv_tc_s2: no tile fits shared memory");
  g.S = bS; g.R = bR; g.TW = bTW; g.DR = bDR;
  g.P = bTW + hk; g.RR = bR + hk;
  g.nch = (g.R * g.P + 127) / 128;
  g.sub_pos = (std::max(g.RR * g.P, g.nch * 128 + hk * (g.P + 1)) + 8 + 7) / 8 * 8;
  g.tiles_w = (W + g.TW - 1) / g.TW;
  g.tiles_h = (H + g.R - 1) / g.R;
  g.tiles_d = (D + g.DR - 1) / g.DR;
  g.ntaps = ks * ks;
  p.grid = g.tiles_w * g.tiles_h * g.tiles_d;
  p.smem = bbytes + (size_t)g.S * cg * 4 * g.sub_pos * 16 + 256;
  return p;
}

// B image for the stride-2 kernel: w folded fp32 [tap][cin][cout] with tap = (kd*KS + kh)*KS + kw.
template <typename T>
inline void build_b_image_s2(const float* w, int cin, int cout, int npad, int kd_n, int ks,
                             const std::vector<std::pair<int, int>>& taps, std::vector<T>& img, T (*cvt)(float), int nsplit = 1) {
  const int ntaps = (int)taps.size();
  const int nblk = cin >= 16 ? ntaps * (cin / 16) : (ntaps + 1) / 2;
  const size_t slice = (size_t)kd_n * nblk * npad * 16;
  img.assign(slice * nsplit, cvt(0.f));
  for (int kd = 0; kd < kd_n; ++kd)
    for (int b = 0; b < nblk; ++b)
      for (int half = 0; half < 2; ++half)
        for (int nn = 0; nn < cout; ++nn)
          for (int e = 0; e < 8; ++e) {
            int t, ci;
            if (cin >= 16) { t = b / (cin / 16); ci = (b % (cin / 16)) * 16 + half * 8 + e; }
            else {
              const int t1 = std::min(2 * b + 1, ntaps - 1), t0 = t1 - 1;
              t = half == 0 ? t0 : t1;
              if (half == 0 && 2 * b + 1 > ntaps - 1) t = -1;   // odd last block: first half re-reads the previous tap x 0
              ci = e;
            }
            if (t < 0 || ci >= cin) continue;
            const int tap = (kd * ks + taps[t].first) * ks + taps[t].second;
            const int n = nn % npad;
            T* simg = img.data() + slice * (nn / npad);
            simg[(((size_t)(kd * nblk + b) * 2 + half) * (npad / 8) + n / 8) * 64 + (n % 8) * 8 + e] =
                cvt(w[((size_t)tap * cin + ci) * cout + nn]);
          }
}

}  // namespace tc
}  // namespace tdm
