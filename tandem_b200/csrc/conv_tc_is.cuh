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
// so consumer warpgroup wg owns sub-chunks NWG * k + wg on every plane of the tile, and the planner bounds the chunks per
// plane by kIsMaxCh (registers: 2 * kIsMaxCh / NWG sub-chunks per warpgroup).  The chains are short (5 to 18 wgmma), so a
// warpgroup issues the chains of KB = is_batch(...) of its sub-chunks of a plane back to back, each into its own fragment,
// then commits once, waits once (wait_group 0) and folds them in sub-chunk order; nothing stays in flight across the wait
// (keeping a chain in flight with wgmma.wait_group 1 made ptxas serialise every wgmma, C7514).  The other consumer
// warpgroups' MMAs overlap the folds and stores.  Every output comes from the same chain and the same fold order as with
// one chain per wait.  Ring, producer warp, roles and tile geometry are those of k_conv_tc.
#pragma once
#include "conv_tc.cuh"

namespace tdm {
namespace tc {

// Most 128-position chunks per plane, i.e. 2 * kIsMaxCh / NWG 64-position sub-chunks per consumer warpgroup: two rolling
// partials of 4 floats each per sub-chunk stay in registers
constexpr int kIsMaxCh = 8;

// Chains a consumer warpgroup issues back to back before one wait (a divisor of its 2 * kIsMaxCh / NWG sub-chunks), the
// most that build without spills (-Xptxas -v, DESIGN.md section 5): the prob layer's 12-float fragments four at a time
// with four warpgroups.  conv0's 24-float fragments spill with two next to the partials and the output offsets, and
// keep one chain per wait, as do the prob tail's two-warpgroup instantiations, already at 168 registers.
__host__ __device__ constexpr int is_batch(int cpk, int nwg) { return cpk == 8 && nwg == 4 ? 4 : 1; }

// Tail: the prob layer's softmax / soft-argmin / confidence, as in k_conv_tc (tiles that span all D planes, make_plan_is(full_depth)).
template <typename TIn, typename TOut, int CIN, int CPK, bool OUT_PLAIN, typename Tail, int NWG>
__global__ void __launch_bounds__(conv_threads(NWG), 1)
k_conv_tc_is(const __grid_constant__ CUtensorMap tmap /*P8 input, as k_conv_tc*/, const TIn* __restrict__ bimg /*build_b_image_is*/,
             const float* __restrict__ bias, TOut* __restrict__ out, float* __restrict__ plain_out, const __grid_constant__ Geom g,
             const __grid_constant__ Tail tail) {
  static_assert(CPK == 16 || (CPK == 8 && OUT_PLAIN), "16 columns per kd for 8 channels, 8 for the single prob channel");
  static_assert(!Tail::enabled || OUT_PLAIN, "a per-pixel tail only exists for the single-channel fp32 output");
  constexpr int CG = CIN / 8;
  constexpr int NBLK = ksteps(CIN, 9);
  constexpr int N = 3 * CPK;                    // instruction N
  constexpr int B_BYTES = NBLK * N * 32;
  constexpr int PN = CPK == 16 ? 4 : 2;         // folded values per thread and sub-chunk: (row half i, column e) or row half i
  constexpr int KSUB = 2 * kIsMaxCh / NWG;      // most sub-chunks per plane that one warpgroup owns
  static_assert((2 * kIsMaxCh) % NWG == 0, "the partial arrays hold exactly this warpgroup's share of 2 * kIsMaxCh sub-chunks");
  constexpr int KB = is_batch(CPK, NWG);        // chains in flight per warpgroup between two waits
  static_assert(KSUB % KB == 0, "a warpgroup's sub-chunks split into whole batches");

  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t cg_bytes = (uint32_t)g.slot_pos * 16u;
  Ring<NWG> ring = Ring<NWG>::start(smem, B_BYTES, bimg, cg_bytes * CG, g.S);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const TileOrigin o = tile_origin(g);
  const int nin = o.ndo + 2;             // padded input planes d0 .. d0+ndo+1 (the zero D halos cover the borders)

  if (warp == 4 * NWG) {
    if (lane == 0) {
      const uint32_t box_bytes = (uint32_t)g.P * (uint32_t)(g.R + 2) * 16u;
      ring.produce(nin, box_bytes * CG, [&](uint8_t* dst, int rp, uint64_t* bar) {
#pragma unroll 1
        for (int cg = 0; cg < CG; ++cg) tma_load_4d(dst + (size_t)cg * cg_bytes, &tmap, 0, o.w0, o.h0, cg * g.iDp + o.d0 + rp, bar);
      });
    }
    return;
  }
  const int wg = warp >> 2, wq = warp & 3;
  const int P = g.P;
  const uint32_t cgb16 = cg_bytes >> 4;
  const uint32_t sB16 = smem_u32(smem) >> 4;
  const uint32_t b_lbo16 = (uint32_t)(N * 16 >> 4);
  auto tap_off = [&](int t) -> int { return stencil_off(t, P); };
  const int nsub = 2 * g.nch;                    // sub-chunks sc = NWG * k + wg < nsub of every plane belong to this warpgroup
  float pa[KSUB][PN], pb[KSUB][PN];              // partials of output planes rp-1 and rp (after input plane rp)
#pragma unroll
  for (int k = 0; k < KSUB; ++k)
#pragma unroll
    for (int q = 0; q < PN; ++q) pa[k][q] = pb[k][q] = 0.f;
  // channels 2 * (lane % 4) + e, or the single prob channel
  float bv[1][2];
  if constexpr (OUT_PLAIN) bv[0][0] = bias ? bias[0] : 0.f;
  else load_bias<false>(bv, bias, 0, 8, lane);

  // A sub-chunk covers the same pixels on every plane: the in-plane element offset of each fragment row half this thread
  // stores (h * W + w, or the P8 position ((h + 1) * Wp + w + 1) * 8), -1 for pad columns and positions beyond the grid.
  // Four warpgroups keep them in registers, decoded once per CTA; the two-warpgroup tail instantiations, which own twice
  // the sub-chunks and sit at 168 registers, would spill and decode them in every fold.
  constexpr bool POFF_REG = NWG == 4;
  const long long pstride = OUT_PLAIN ? (long long)g.H * g.W : (long long)g.Hp * g.Wp * 8;
  auto pix_off = [&](int k, int i) -> int {
    int h, w;
    const bool in = frag_pixel(g, o, (NWG * k + wg) * 64 + wq * 16 + (lane >> 2), i, h, w);
    return !in ? -1 : OUT_PLAIN ? h * g.W + w : ((h + 1) * g.Wp + (w + 1)) * 8;
  };
  int poff[POFF_REG ? KSUB : 1][2];
  if constexpr (POFF_REG) {
#pragma unroll
    for (int k = 0; k < KSUB; ++k)
#pragma unroll
      for (int i = 0; i < 2; ++i) poff[k][i] = pix_off(k, i);
  }

  // value q of column block s (0: kd=2, 1: kd=1, 2: kd=0) of fragment f, hi + lo
  auto blk = [&](const float (&f)[N / 2], int s, int q) -> float {
    if constexpr (CPK == 16) return f[8 * s + q] + f[8 * s + 4 + q];      // d[4j + 2i + e], j = 2s (hi) / 2s+1 (lo), q = 2i+e
    else return f[4 * s + 2 * q] + f[4 * s + 2 * q + 1];                   // columns 0 (hi) and 1 (lo) of block j = s, q = i
  };
  auto fold = [&](int k, const float (&f)[N / 2], int rp) {
    float x[PN];
#pragma unroll
    for (int q = 0; q < PN; ++q) {
      x[q] = pa[k][q] + blk(f, 0, q);
      pa[k][q] = pb[k][q] + blk(f, 1, q);
      pb[k][q] = blk(f, 2, q);
    }
    if (rp < 2) return;
    const long long plane = (long long)(o.d0 + rp - 2 + (OUT_PLAIN ? 0 : 1)) * pstride;   // output plane d (padded: d + 1)
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int off = POFF_REG ? poff[POFF_REG ? k : 0][i] : pix_off(k, i);
      if (off < 0) continue;
      if constexpr (OUT_PLAIN) {
        if ((lane & 3) == 0) plain_out[plane + off] = x[i] + bv[0][0];
      } else {
        const int co = 2 * (lane & 3);
        float y[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          y[e] = x[2 * i + e] + bv[0][e];
          if (g.relu) y[e] = fmaxf(y[e], 0.f);
        }
        store2<TOut>(out + plane + off + co, y[0], y[1]);
      }
    }
  };

  ring.wait_weights();
  for (int rp = 0; rp < nin; ++rp) {
    ring.wait(rp);
    const uint32_t slot16 = ring.slot16(rp);
#pragma unroll
    for (int k0 = 0; k0 < KSUB; k0 += KB) {
      // sub-chunks NWG * k + wg grow with k: if the batch's first one is beyond the plane, all of them are
      if (NWG * k0 + wg < nsub) {
        // the batch's chains are issued back to back into their own fragments and retired by one wait
        float fr[KB][N / 2];
#pragma unroll
        for (int j = 0; j < KB; ++j) fence_frag(fr[j]);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < KB; ++j) {
          if (NWG * (k0 + j) + wg < nsub) {
            const uint32_t a0 = slot16 + (uint32_t)(NWG * (k0 + j) + wg) * 64u;
#pragma unroll
            for (int b = 0; b < NBLK; ++b)
              wgmma<N, TIn>(fr[j], desc(a0 + kstep_aoff<CIN, 9>(b, cgb16, tap_off), kstep_alo<CIN, 9>(b, cgb16, tap_off)),
                            desc(sB16 + (uint32_t)(b * N * 2), b_lbo16), b != 0 ? 1u : 0u);
          }
        }
        wgmma_commit();
        wgmma_wait_all();
#pragma unroll
        for (int j = 0; j < KB; ++j) {
          if (NWG * (k0 + j) + wg < nsub) {
            fence_frag(fr[j]);
            fold(k0 + j, fr[j], rp);
          }
        }
      }
    }
    ring.release(rp);   // this warp no longer reads input plane rp
  }
  if constexpr (Tail::enabled) run_tail<NWG>(tail, plain_out, g, o, wg, wq, lane);
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
// Columns per kd block: 16 for 8 output channels, 8 for 1 (hi, lo in columns 0, 1).
inline int is_cols_per_kd(int cout) { return cout == 1 ? 8 : 16; }

// B image of k_conv_tc_is: per K=16 step b the 3*CPK columns are [kd=2 | kd=1 | kd=0], each [hi | lo] as above, in the
// canonical K-major no-swizzle order of build_b_image.  w: folded fp32 [tap27][cin][cout], tap27 = (kd*3+kh)*3+kw.
template <typename T>
inline void build_b_image_is(const float* w, int cin, int cout, std::vector<T>& img, T (*cvt)(float), float (*back)(T)) {
  const int nblk = ksteps(cin, 9);
  const int cpk = is_cols_per_kd(cout), n3 = 3 * cpk;
  img.assign((size_t)nblk * n3 * 16, cvt(0.f));
  for (int s = 0; s < 3; ++s) {
    const int kd = 2 - s;
    for (int b = 0; b < nblk; ++b)
      for (int half = 0; half < 2; ++half)
        for (int n = 0; n < cout; ++n)
          for (int e = 0; e < 8; ++e) {
            const int tap9 = kstep_tap(cin, 9, b, half), ci = kstep_ch(cin, b, half) + e;
            if (!kstep_live(cin, 9, b, half) || ci >= cin) continue;
            const float val = w[((size_t)(kd * 9 + tap9) * cin + ci) * cout + n];
            const int c_hi = s * cpk + (cout == 1 ? 0 : n), c_lo = s * cpk + (cout == 1 ? 1 : 8 + n);
            const T hi = cvt(val);
            img[b_index(b, half, c_hi, e, n3)] = hi;
            img[b_index(b, half, c_lo, e, n3)] = cvt(val - back(hi));
          }
  }
}

// Tile planner of k_conv_tc_is.  Same tile geometry and ring layout as make_plan (3-D, pd = 1), with its own limits: at
// most kIsMaxCh 128-position chunks per plane (the register-resident partials), a ring of 3 or 2 planes (each input plane
// is consumed once), and a cost that counts one N = 3*cpk chain per input plane instead of three per output plane.
inline Plan make_plan_is(int cin, int cpk, int D, int H, int W, size_t smem_limit = 225 * 1024,
                         bool full_depth = false /* tiles span all D planes (the prob layer's tail) */) {
  Plan p{};
  const int nblk = ksteps(cin, 9);
  const int n3 = 3 * cpk;
  const TileLimits lim{3, 2, 2, 1, 256, 30, kIsMaxCh, 1, full_depth};
  auto amp = [&](int R, int TW, int P, int DR) { return (double)(R + 2) / R * (double)P / TW * (double)(DR + 2) / DR; };
  const int nwg = conv_nwg(0, n3, full_depth ? D : 0);
  auto tile_clk = [&](int DR, int nch) { return (8500.0 + (double)(DR + 2) * nch * nblk * (45.0 + 0.35 * n3)) * wg_balance(nch, nwg); };
  static_cast<Tile&>(p.g) = plan_tiles(D, H, W, cin / 8, b_image_bytes(1, nblk, n3), smem_limit, lim, amp, tile_clk, p.smem);
  p.g.Hp = H + 2; p.g.Wp = W + 2; p.g.pd = 1;
  p.grid = p.g.tiles_w * p.g.tiles_h * p.g.tiles_d;
  p.nwg = nwg;
  return p;
}

}  // namespace tc
}  // namespace tdm
