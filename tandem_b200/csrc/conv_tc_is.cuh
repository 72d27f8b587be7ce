// Input-stationary 3x3x3 stride-1 tensor-core convolution for the narrow-output 3-D layers of CostRegNet: each stage's
// conv0 (cost volume -> 8 channels) and prob (8 -> 1 channel), module.py:577-600.
//
// The output-stationary k_conv_tc (conv_tc.cuh) computes one output plane per K chain over its three input planes, so
// every input plane is streamed out of shared memory as the A operand three times.  These layers have few output
// columns, and their wgmma is bound by that operand stream, not by the tensor pipe.  Here each input plane p is read
// once: per 64-position sub-chunk, one chain of NBLK wgmma with
//   N = 3 * CPK,   B = [ W(kd=2) | W(kd=1) | W(kd=0) ],
// writes a fresh fragment whose column block kd holds plane p's contribution to output plane p+1-kd.  The weights are
// carried as hi + lo 16-bit halves (see HILO in conv_tc.cuh), packed tightly: CPK = 16 columns per kd for 8 output
// channels ([hi 0..7 | lo 0..7]), CPK = 8 for the single prob channel (hi in column 0, lo in column 1).
// The blocks are folded into two rolling fp32 partials per sub-chunk, held in registers:
//   output p-1 = partial(p-1) + block kd=2   -> complete: bias / ReLU / store
//   partial(p) += block kd=1,   partial(p+1) = block kd=0
// so a consumer warpgroup owns the same sub-chunks on every plane of the tile, and the planner bounds the sub-chunks per
// warpgroup by kIsMaxCh (registers).  As in k_conv_tc, a warpgroup waits for its chain before it folds and stores, and the
// other consumer warpgroup's MMAs overlap that epilogue (keeping the next chain in flight with wgmma.wait_group 1 made
// ptxas serialise every wgmma, C7514).  Ring, producer warp, roles and tile geometry are those of k_conv_tc.
#pragma once
#include "conv_tc.cuh"

namespace tdm {
namespace tc {

// 128-position chunks per plane, i.e. 64-position sub-chunks per consumer warpgroup: two rolling partials of 4 floats each
// per sub-chunk stay in registers
constexpr int kIsMaxCh = 8;

// Tail: the prob layer's softmax / soft-argmin / confidence, as in k_conv_tc (tiles that span all D planes, make_plan_is(full_depth)).
template <typename TIn, typename TOut, int CIN, int CPK, bool OUT_PLAIN, typename Tail = NoTail>
__global__ void __launch_bounds__(kThreads, 1)
k_conv_tc_is(const __grid_constant__ CUtensorMap tmap /*P8 input, as k_conv_tc*/, const TIn* __restrict__ bimg /*build_b_image_is*/,
             const float* __restrict__ bias, TOut* __restrict__ out, float* __restrict__ plain_out, const __grid_constant__ Geom g,
             const __grid_constant__ Tail tail) {
  static_assert(CPK == 16 || (CPK == 8 && OUT_PLAIN), "16 columns per kd for 8 channels, 8 for the single prob channel");
  static_assert(!Tail::enabled || OUT_PLAIN, "a per-pixel tail only exists for the single-channel fp32 output");
  constexpr int CG = CIN / 8;
  constexpr int NBLK = blocks_per_kd<CIN>();
  constexpr int N = 3 * CPK;                    // instruction N
  constexpr int B_BYTES = NBLK * N * 32;
  constexpr int PN = CPK == 16 ? 4 : 2;         // folded values per thread and sub-chunk: (row half i, column e) or row half i

  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* sB = smem;
  uint8_t* sA = smem + ((B_BYTES + 127) / 128) * 128;
  const uint32_t cg_bytes = (uint32_t)g.slot_pos * 16u;
  const uint32_t slot_bytes = cg_bytes * CG;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sA + (size_t)slot_bytes * g.S);
  uint64_t* full = bars;                 // [S]
  uint64_t* empty = bars + 8;            // [S]
  uint64_t* b_full = bars + 16;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  int tile = blockIdx.x;
  const int tw = tile % g.tiles_w; tile /= g.tiles_w;
  const int th = tile % g.tiles_h; tile /= g.tiles_h;
  const int w0 = tw * g.TW, h0 = th * g.R, d0 = tile * g.DR;
  const int ndo = min(g.DR, g.D - d0);
  const int nin = ndo + 2;               // padded input planes d0 .. d0+ndo+1 (the zero D halos cover the borders)

  if (threadIdx.x == 0) {
    for (int s = 0; s < g.S; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4 * kConsumerWG); }
    mbar_init(b_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(b_full, B_BYTES);
    bulk_g2s(sB, bimg, B_BYTES, b_full);
  }
  __syncthreads();
  pdl_wait();
  if (threadIdx.x == 0) pdl_launch_dependents();

  if (warp == kProducerWarp) {
    if (lane == 0) {
      const uint32_t box_bytes = (uint32_t)g.P * (uint32_t)(g.R + 2) * 16u;
      for (int rp = 0; rp < nin; ++rp) {
        const int slot = rp % g.S;
        if (rp >= g.S) mbar_wait(&empty[slot], ((rp / g.S) - 1) & 1);
        mbar_expect_tx(&full[slot], box_bytes * CG);
#pragma unroll 1
        for (int cg = 0; cg < CG; ++cg)
          tma_load_4d(sA + (size_t)slot * slot_bytes + (size_t)cg * cg_bytes, &tmap, 0, w0, h0, cg * g.iDp + d0 + rp, &full[slot]);
      }
    }
    return;
  }
  const int wg = warp >> 2, wq = warp & 3;
  const int P = g.P;
  const uint32_t cgb16 = cg_bytes >> 4;
  const uint32_t sB16 = smem_u32(sB) >> 4, sA16 = smem_u32(sA) >> 4;
  const uint32_t b_lbo16 = (uint32_t)(N * 16 >> 4);
  const int nch = g.nch;                         // sub-chunks sc = 2k + wg, k < nch, of every plane belong to this warpgroup
  float pa[kIsMaxCh][PN], pb[kIsMaxCh][PN];      // partials of output planes rp-1 and rp (after input plane rp)
#pragma unroll
  for (int k = 0; k < kIsMaxCh; ++k)
#pragma unroll
    for (int q = 0; q < PN; ++q) pa[k][q] = pb[k][q] = 0.f;
  float fr[N / 2];
  // this thread's bias values, loaded once per CTA (channels 2 * (lane % 4) + e, or the single prob channel)
  float bv[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) bv[e] = bias ? bias[OUT_PLAIN ? 0 : 2 * (lane & 3) + e] : 0.f;

  // value q of column block s (0: kd=2, 1: kd=1, 2: kd=0) of fragment f, hi + lo
  auto blk = [&](const float (&f)[N / 2], int s, int q) -> float {
    if constexpr (CPK == 16) return f[8 * s + q] + f[8 * s + 4 + q];      // d[4j + 2i + e], j = 2s (hi) / 2s+1 (lo), q = 2i+e
    else return f[4 * s + 2 * q] + f[4 * s + 2 * q + 1];                   // columns 0 (hi) and 1 (lo) of block j = s, q = i
  };
  auto fold = [&](int k, const float (&f)[N / 2], int rp) {
    float o[PN];
#pragma unroll
    for (int q = 0; q < PN; ++q) {
      o[q] = pa[k][q] + blk(f, 0, q);
      pa[k][q] = pb[k][q] + blk(f, 1, q);
      pb[k][q] = blk(f, 2, q);
    }
    if (rp < 2) return;
    const int d = d0 + rp - 2;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int l = (2 * k + wg) * 64 + wq * 16 + (lane >> 2);
      int hh = l / P, ww = l - hh * P;   // row half 1 is 8 positions on: one division serves both halves
      if (i) {
        ww += 8;
        while (ww >= P) { ww -= P; ++hh; }
      }
      const int h = h0 + hh, w = w0 + ww;
      if (!(hh < g.R && ww < g.TW && h < g.H && w < g.W)) continue;
      if constexpr (OUT_PLAIN) {
        if ((lane & 3) == 0) plain_out[((long long)d * g.H + h) * g.W + w] = o[i] + bv[0];
      } else {
        const int co = 2 * (lane & 3);
        float x[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          x[e] = o[2 * i + e] + bv[e];
          if (g.relu) x[e] = fmaxf(x[e], 0.f);
        }
        const long long pos = ((((long long)(d + 1)) * g.Hp + (h + 1)) * g.Wp + (w + 1)) * 8;
        store2<TOut>(out + pos + co, x[0], x[1]);
      }
    }
  };

  mbar_wait(b_full, 0);
  for (int rp = 0; rp < nin; ++rp) {
    mbar_wait(&full[rp % g.S], (rp / g.S) & 1);
    const uint32_t slot16 = sA16 + (uint32_t)(rp % g.S) * (slot_bytes >> 4);
#pragma unroll
    for (int k = 0; k < kIsMaxCh; ++k) {
      if (k < nch) {
        const uint32_t a0 = slot16 + (uint32_t)(2 * k + wg) * 64u;
        fence_frag(fr);
        wgmma_fence();
#pragma unroll
        for (int b = 0; b < NBLK; ++b)
          wgmma<N, TIn>(fr, desc(a0 + stencil_aoff<CIN>(b, P, cgb16), stencil_alo<CIN>(b, P, cgb16)),
                        desc(sB16 + (uint32_t)(b * N * 2), b_lbo16), b != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait_all();
        fence_frag(fr);
        fold(k, fr, rp);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[rp % g.S]);   // this warp no longer reads input plane rp
  }
  if constexpr (Tail::enabled) {
    // ndo == D (host-checked): this thread wrote all D logits of its pixels itself (program order makes them visible to it)
    if ((lane & 3) == 0) {
      for (int sc = wg; sc < 2 * nch; sc += kConsumerWG)
        for (int i = 0; i < 2; ++i) {
          const int l = sc * 64 + wq * 16 + (lane >> 2) + 8 * i;
          const int hh = l / P, ww = l - hh * P;
          const int h = h0 + hh, w = w0 + ww;
          if (hh < g.R && ww < g.TW && h < g.H && w < g.W) tail(plain_out, h * g.W + w, w, h, g.H * g.W);
        }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
// Columns per kd block: 16 for 8 output channels, 8 for 1 (hi, lo in columns 0, 1).
inline int is_cols_per_kd(int cout) { return cout == 1 ? 8 : 16; }

// B image of k_conv_tc_is: per K=16 step b the 3*CPK columns are [kd=2 | kd=1 | kd=0], each [hi | lo] as above, in the
// canonical K-major no-swizzle order of build_b_image.  w: folded fp32 [tap27][cin][cout], tap27 = (kd*3+kh)*3+kw.
template <typename T, int CIN>
inline void build_b_image_is(const float* w, int cin, int cout, std::vector<T>& img, T (*cvt)(float), float (*back)(T)) {
  constexpr int NBLK = blocks_per_kd<CIN>();
  const int cpk = is_cols_per_kd(cout), n3 = 3 * cpk;
  img.assign((size_t)NBLK * n3 * 16, cvt(0.f));
  for (int s = 0; s < 3; ++s) {
    const int kd = 2 - s;
    for (int b = 0; b < NBLK; ++b)
      for (int half = 0; half < 2; ++half)
        for (int n = 0; n < cout; ++n)
          for (int e = 0; e < 8; ++e) {
            int tap9, ci;
            if (CIN >= 16) { tap9 = b / (CIN / 16); ci = (b % (CIN / 16)) * 16 + half * 8 + e; }
            else { tap9 = b < 4 ? 2 * b + half : (half == 0 ? -1 : 8); ci = e; }  // block 4 = (zero, tap 8)
            if (tap9 < 0 || ci >= cin) continue;
            const float val = w[((size_t)(kd * 9 + tap9) * cin + ci) * cout + n];
            T* blkp = img.data() + ((size_t)b * 2 + half) * (n3 / 8) * 64;
            const int c_hi = s * cpk + (cout == 1 ? 0 : n), c_lo = s * cpk + (cout == 1 ? 1 : 8 + n);
            const T hi = cvt(val);
            blkp[(c_hi / 8) * 64 + (c_hi % 8) * 8 + e] = hi;
            blkp[(c_lo / 8) * 64 + (c_lo % 8) * 8 + e] = cvt(val - back(hi));
          }
  }
}

// Tile planner of k_conv_tc_is.  Same tile geometry and ring layout as make_plan (3-D, pd = 1), with its own limits: at
// most kIsMaxCh 128-position chunks per plane (the register-resident partials), a ring of 3 or 2 planes (each input plane
// is consumed once), and a cost that counts one N = 3*cpk chain per input plane instead of three per output plane.
inline Plan make_plan_is(int cin, int cpk, int D, int H, int W, size_t smem_limit = 225 * 1024,
                         bool full_depth = false /* tiles span all D planes (the prob layer's tail) */) {
  Plan p{};
  Geom& g = p.g;
  g.D = D; g.H = H; g.W = W; g.Hp = H + 2; g.Wp = W + 2; g.pd = 1;
  const int cg = cin / 8;
  const int nblk = cin >= 16 ? 9 * (cin / 16) : 5;
  const int n3 = 3 * cpk;
  const size_t bbytes = (((size_t)nblk * n3 * 32) + 127) / 128 * 128;
  double best_cost = 1e30;
  int bestR = 0, bestTW = 0, bestS = 0, bestDR = 0;
  for (int S = 3; S >= 2; --S) {
    for (int tiles_w = 1; tiles_w <= 20; ++tiles_w) {
      const int TW = (W + tiles_w - 1) / tiles_w;
      if (TW + 2 > 256) continue;
      if (tiles_w > 1 && TW < 30) break;
      const int tw_n = (W + TW - 1) / TW;
      const int P = TW + 2;
      for (int R = 1; R <= 32 && R <= H; ++R) {
        const int nch = (R * P + 127) / 128;
        if (nch > kIsMaxCh) break;
        const int slot_pos = (std::max((R + 2) * P, nch * 128 + 2 * P + 2) + 8 + 7) / 8 * 8;
        const size_t smem = bbytes + (size_t)S * cg * slot_pos * 16 + 256;
        if (smem > smem_limit) break;
        const int th_n = (H + R - 1) / R;
        for (int dsplit = 1; dsplit <= (full_depth ? 1 : D); ++dsplit) {
          const int DR = (D + dsplit - 1) / dsplit;
          const int td_n = (D + DR - 1) / DR;
          const double T = (double)tw_n * th_n * td_n;
          const double amp = (double)(R + 2) / R * (double)P / TW * (double)(DR + 2) / DR;
          // a model for ranking tilings (as in make_plan), not a measurement
          const double tile_clk = 8500.0 + (double)(DR + 2) * nch * nblk * (45.0 + 0.35 * n3);
          const double cost = std::ceil(T / 132.0) * tile_clk * (1.0 + 0.25 * (amp - 1.0)) * (S == 3 ? 1.0 : 1.05);
          if (cost < best_cost - 1e-9) { best_cost = cost; bestR = R; bestTW = TW; bestS = S; bestDR = DR; }
          if (T > 4000) break;
        }
      }
    }
    if (bestR > 0 && S == 3) break;
  }
  TDM_CHECK(bestR > 0, "conv_tc_is: no tile fits shared memory");
  g.S = bestS; g.R = bestR; g.TW = bestTW; g.P = bestTW + 2; g.DR = bestDR;
  g.nch = (g.R * g.P + 127) / 128;
  g.slot_pos = (std::max((g.R + 2) * g.P, g.nch * 128 + 2 * g.P + 2) + 8 + 7) / 8 * 8;
  g.tiles_w = (W + g.TW - 1) / g.TW;
  g.tiles_h = (H + g.R - 1) / g.R;
  g.tiles_d = (D + g.DR - 1) / g.DR;
  p.grid = g.tiles_w * g.tiles_h * g.tiles_d;
  p.smem = bbytes + (size_t)g.S * cg * g.slot_pos * 16 + 256;
  return p;
}

}  // namespace tc
}  // namespace tdm
