// n8: the immature points of the active keyframes, kept in device memory, and their epipolar trace into each new frame
// (FullSystem::traceNewCoarse, tandem/src/FullSystem/FullSystem.cpp:650-691, calling ImmaturePoint::traceOn,
// ImmaturePoint.cpp:75-414, per point), plus the constructor (ImmaturePoint.cpp:32-61) and activatePointsMT's compaction
// (FullSystem.cpp:849-856).  Every float operation is the reference's own, correctly rounded and in its order (__f*_rn, no
// contraction); oracle/trace_oracle.c restates the same statements on the CPU.
//
// Shape (DESIGN.md, n8): one warp per point.  Every lane evaluates the point's prologue (projections, interval, error bound)
// - the same values, so every branch is warp-uniform - the lanes share the discrete search (lane l takes steps l, l+32, ...,
// rebuilding ptx / pty by the reference's chain of additions), a shuffle reduction picks the best step (first index on ties,
// as the strict < does) and the second best outside its radius, and every lane runs the Gauss-Newton steps; lane 0 stores.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include <cub/block/block_scan.cuh>

#include "dso_sample.cuh"
#include "tracker.h"

namespace tdm {

namespace {

enum { IPS_GOOD = 0, IPS_OOB, IPS_OUTLIER, IPS_SKIPPED, IPS_BADCONDITION, IPS_UNINITIALIZED };
// one row of 8 * cap 32-bit words per field (ImmatureRow, tracker.h); point i of slot s is word s * cap + i of every row
constexpr int kRows = IM_ROWS, kSlots = 8;
constexpr int kMaxSteps = 99;   // `if(numSteps >= 100) numSteps = 99;`

struct Settings {   // tdm_trace_settings
  float max_pix_search, stepsize, gn_threshold, extra_slack_on_th, slack_interval, min_improvement_factor, huber, outlier_th,
      outlier_th_sum_component, overall_energy_th_weight;
  int min_trace_test_radius, gn_iterations;
};

struct TraceHost {
  float K[9], Kt[3], aff[2];
  int slot, n, first_warp;
};
struct TraceLaunch {
  TraceHost host[kSlots];
  int n_hosts, w, h, cap;
  Settings s;
};

__device__ __forceinline__ float huber_weight(float residual, float huber) {
  return fabsf(residual) < huber ? 1.f : fd(huber, fabsf(residual));
}

__global__ void __launch_bounds__(128) k_trace(TraceLaunch L, uint32_t* __restrict__ st, const float* __restrict__ dI) {
  const int warp = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  int hi = 0;
  while (hi + 1 < L.n_hosts && warp >= L.host[hi + 1].first_warp) ++hi;
  const TraceHost& H = L.host[hi];
  const int i = warp - H.first_warp;
  if (i < 0 || i >= H.n) return;   // warp-uniform
  const size_t stride = (size_t)kSlots * L.cap, p = (size_t)H.slot * L.cap + i;
  float* f = reinterpret_cast<float*>(st);
  auto F = [&](int r) -> float& { return f[r * stride + p]; };
  const int w = L.w, h = L.h;
  const Settings& S = L.s;
  const float* K = H.K;
  const float* Kt = H.Kt;

  int status = (int)st[IM_STATUS * stride + p];
  if (status == IPS_OOB) return;                                              // :77
  float idepth_min = F(IM_IDMIN), idepth_max = F(IM_IDMAX);
  const float u = F(IM_U), v = F(IM_V);
  float uvx = -1.f, uvy = -1.f, interval = 0.f, quality = F(IM_QUALITY);
  bool done = true;
  const float maxPixSearch = fm((float)(w + h), S.max_pix_search);
  const float pr0 = fa(fa(fm(K[0], u), fm(K[1], v)), fm(K[2], 1.f));
  const float pr1 = fa(fa(fm(K[3], u), fm(K[4], v)), fm(K[5], 1.f));
  const float pr2 = fa(fa(fm(K[6], u), fm(K[7], v)), fm(K[8], 1.f));
  const float pm2 = fa(pr2, fm(Kt[2], idepth_min));
  const float uMin = fd(fa(pr0, fm(Kt[0], idepth_min)), pm2), vMin = fd(fa(pr1, fm(Kt[1], idepth_min)), pm2);
  float dist = 0.f, uMax = 0.f, vMax = 0.f, dx = 0.f, dy = 0.f, errorInPixel = 0.f;
  float bestU = 0.f, bestV = 0.f;
  if (!(uMin > 4 && vMin > 4 && uMin < w - 5 && vMin < h - 5)) {               // :102
    status = IPS_OOB;
  } else {
    bool oob = false;
    if (isfinite(idepth_max)) {
      const float q2 = fa(pr2, fm(Kt[2], idepth_max));
      uMax = fd(fa(pr0, fm(Kt[0], idepth_max)), q2);
      vMax = fd(fa(pr1, fm(Kt[1], idepth_max)), q2);
      if (!(uMax > 4 && vMax > 4 && uMax < w - 5 && vMax < h - 5)) {           // :122
        status = IPS_OOB; oob = true;
      } else {
        dist = __fsqrt_rn(fa(fm(fs(uMin, uMax), fs(uMin, uMax)), fm(fs(vMin, vMax), fs(vMin, vMax))));
        if (dist < S.slack_interval) {                                         // :135
          uvx = fm(fa(uMax, uMin), 0.5f); uvy = fm(fa(vMax, vMin), 0.5f); interval = dist; status = IPS_SKIPPED; oob = true;
        }
      }
    } else {
      dist = maxPixSearch;
      const float q2 = fa(pr2, fm(Kt[2], 0.01f));
      uMax = fd(fa(pr0, fm(Kt[0], 0.01f)), q2);
      vMax = fd(fa(pr1, fm(Kt[1], 0.01f)), q2);
      const float ddx = fs(uMax, uMin), ddy = fs(vMax, vMin);
      const float d = fd(1.0f, __fsqrt_rn(fa(fm(ddx, ddx), fm(ddy, ddy))));
      uMax = fa(uMin, fm(fm(dist, ddx), d));
      vMax = fa(vMin, fm(fm(dist, ddy), d));
      if (!(uMax > 4 && vMax > 4 && uMax < w - 5 && vMax < h - 5)) { status = IPS_OOB; oob = true; }   // :165
    }
    if (!oob) {
      if (!(idepth_min < 0 || (pm2 > 0.75f && pm2 < 1.5f))) {                  // :177
        status = IPS_OOB;
      } else {
        dx = fm(S.stepsize, fs(uMax, uMin));
        dy = fm(S.stepsize, fs(vMax, vMin));
        const float* g = &F(IM_GRADH);
        const float g00 = g[0], g01 = g[stride], g10 = g[2 * stride], g11 = g[3 * stride];
        const float a = fa(fm(fa(fm(dx, g00), fm(dy, g10)), dx), fm(fa(fm(dx, g01), fm(dy, g11)), dy));
        const float b = fa(fm(fa(fm(dy, g00), fm(-dx, g10)), dy), fm(fa(fm(dy, g01), fm(-dx, g11)), -dx));
        errorInPixel = fa(0.2f, fd(fm(0.2f, fa(a, b)), a));
        if (fm(errorInPixel, S.min_improvement_factor) > dist && isfinite(idepth_max)) {   // :194
          uvx = fm(fa(uMax, uMin), 0.5f); uvy = fm(fa(vMax, vMin), 0.5f); interval = dist; status = IPS_BADCONDITION;
        } else {
          done = false;
        }
      }
    }
  }
  if (!done) {
    if (errorInPixel > 10) errorInPixel = 10;
    dx = fd(dx, dist);
    dy = fd(dy, dist);
    if (dist > maxPixSearch) {
      uMax = fa(uMin, fm(maxPixSearch, dx));
      vMax = fa(vMin, fm(maxPixSearch, dy));
      dist = maxPixSearch;
    }
    int numSteps = (int)fa(1.9999f, fd(dist, S.stepsize));
    const float randShift = fs(fm(uMin, 1000.f), floorf(fm(uMin, 1000.f)));
    const float ptx0 = fs(uMin, fm(randShift, dx)), pty0 = fs(vMin, fm(randShift, dy));
    float rpx[8], rpy[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float px = (float)c_pattern[k][0], py = (float)c_pattern[k][1];
      rpx[k] = fa(fm(K[0], px), fm(K[1], py));
      rpy[k] = fa(fm(K[3], px), fm(K[4], py));
    }
    if (!isfinite(dx) || !isfinite(dy)) {                                       // :243
      status = IPS_OOB;
    } else {
      if (numSteps >= 100) numSteps = kMaxSteps;
      const float affa = H.aff[0], affb = H.aff[1];
      float col[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) col[k] = F(IM_COLOR + k);
      // discrete search: lane l evaluates steps l, l + 32, l + 64, l + 96
      float px = ptx0, py = pty0;
      for (int k = 0; k < lane; ++k) { px = fa(px, dx); py = fa(py, dy); }
      float err[4], lbE = 1e10f, lbU = 0.f, lbV = 0.f;
      int lbI = -1;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int step = lane + 32 * r;
        float energy = 0.f;
        if (step < numSteps) {
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const float x = fa(px, rpx[k]), y = fa(py, rpy[k]);
            float hit;
            if (!inside(x, y, w, h)) { energy = fa(energy, 1e5f); continue; }
            interp<1>(dI, x, y, w, &hit);
            if (!isfinite(hit)) { energy = fa(energy, 1e5f); continue; }
            const float residual = fs(hit, fa(fm(affa, col[k]), affb));
            const float hw = huber_weight(residual, S.huber);
            energy = fa(energy, fm(fm(fm(hw, residual), residual), fs(2.f, hw)));
          }
          if (energy < lbE) { lbE = energy; lbI = step; lbU = px; lbV = py; }
        }
        err[r] = energy;
        if (r < 3)
          for (int k = 0; k < 32; ++k) { px = fa(px, dx); py = fa(py, dy); }
      }
      // best step: smallest energy below 1e10, first index on ties
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        const float oE = __shfl_xor_sync(0xffffffffu, lbE, o), oU = __shfl_xor_sync(0xffffffffu, lbU, o),
                    oV = __shfl_xor_sync(0xffffffffu, lbV, o);
        const int oI = __shfl_xor_sync(0xffffffffu, lbI, o);
        if (oI >= 0 && (lbI < 0 || oE < lbE || (oE == lbE && oI < lbI))) { lbE = oE; lbI = oI; lbU = oU; lbV = oV; }
      }
      float bestEnergy = lbE;
      const int bestIdx = lbI;
      bestU = lbU; bestV = lbV;
      const int R = S.min_trace_test_radius;
      float sb = 1e10f;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int step = lane + 32 * r;
        if (step < numSteps && (step < bestIdx - R || step > bestIdx + R) && err[r] < sb) sb = err[r];
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) sb = fminf(sb, __shfl_xor_sync(0xffffffffu, sb, o));
      const float newQuality = fd(sb, bestEnergy);
      if (newQuality < quality || numSteps > 10) quality = newQuality;            // :299

      // Gauss-Newton (:303-364), the same on every lane
      float uBak = bestU, vBak = bestV, stepBack = 0.f;
      const float gnstepsize = 1.f;
      if (S.gn_iterations > 0) bestEnergy = 1e5f;
      for (int it = 0; it < S.gn_iterations; it++) {
        float Hh = 1.f, bb = 0.f, energy = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float x = fa(bestU, rpx[k]), y = fa(bestV, rpy[k]);
          float hit[3];
          if (!inside(x, y, w, h)) { energy = fa(energy, 1e5f); continue; }
          interp<3>(dI, x, y, w, hit);
          if (!isfinite(hit[0])) { energy = fa(energy, 1e5f); continue; }
          const float residual = fs(hit[0], fa(fm(affa, col[k]), affb));
          const float dResdDist = fa(fm(dx, hit[1]), fm(dy, hit[2]));
          const float hw = huber_weight(residual, S.huber);
          const float wk = F(IM_WEIGHTS + k);
          Hh = fa(Hh, fm(fm(hw, dResdDist), dResdDist));
          bb = fa(bb, fm(fm(hw, residual), dResdDist));
          energy = fa(energy, fm(fm(fm(fm(fm(wk, wk), hw), residual), residual), fs(2.f, hw)));
        }
        if (energy > bestEnergy) {
          stepBack = fm(stepBack, 0.5f);
          bestU = fa(uBak, fm(stepBack, dx));
          bestV = fa(vBak, fm(stepBack, dy));
        } else {
          float step = fd(fm(-gnstepsize, bb), Hh);
          if (step < -0.5f) step = -0.5f;
          else if (step > 0.5f) step = 0.5f;
          if (!isfinite(step)) step = 0.f;
          uBak = bestU;
          vBak = bestV;
          stepBack = step;
          bestU = fa(bestU, fm(step, dx));
          bestV = fa(bestV, fm(step, dy));
          bestEnergy = energy;
        }
        if (fabsf(stepBack) < S.gn_threshold) break;
      }
      if (!(bestEnergy < fm(F(IM_ETH), S.extra_slack_on_th))) {                    // :371
        status = status == IPS_OUTLIER ? IPS_OOB : IPS_OUTLIER;
      } else {
        float lo, hi2;
        if (fm(dx, dx) > fm(dy, dy)) {
          const float e0 = fs(bestU, fm(errorInPixel, dx)), e1 = fa(bestU, fm(errorInPixel, dx));
          lo = fd(fs(fm(pr2, e0), pr0), fs(Kt[0], fm(Kt[2], e0)));
          hi2 = fd(fs(fm(pr2, e1), pr0), fs(Kt[0], fm(Kt[2], e1)));
        } else {
          const float e0 = fs(bestV, fm(errorInPixel, dy)), e1 = fa(bestV, fm(errorInPixel, dy));
          lo = fd(fs(fm(pr2, e0), pr1), fs(Kt[1], fm(Kt[2], e0)));
          hi2 = fd(fs(fm(pr2, e1), pr1), fs(Kt[1], fm(Kt[2], e1)));
        }
        if (lo > hi2) { const float t = lo; lo = hi2; hi2 = t; }
        idepth_min = lo;
        idepth_max = hi2;
        if (!isfinite(lo) || !isfinite(hi2) || hi2 < 0) {                         // :402
          status = IPS_OUTLIER;
        } else {
          interval = fm(2.f, errorInPixel); uvx = bestU; uvy = bestV; status = IPS_GOOD;
        }
      }
    }
  }
  if (lane == 0) {
    F(IM_IDMIN) = idepth_min; F(IM_IDMAX) = idepth_max; F(IM_QUALITY) = quality;
    st[IM_STATUS * stride + p] = (uint32_t)status;
    F(IM_UVX) = uvx; F(IM_UVY) = uvy; F(IM_INTERVAL) = interval;
  }
}

// The constructor for n candidate pixels of one slot (u at cand[c], v at cand[cs + c], the type's bits at cand[2 cs + c];
// n read from n_dev when it is given); the points with a finite energyTH are appended in input order behind the slot's
// `count` points, up to the slot's capacity, and *added receives the number kept, those beyond the capacity included.
// One block.
constexpr int kAddThreads = 256;
__global__ void __launch_bounds__(kAddThreads) k_add(Settings S, uint32_t* __restrict__ st, int cap, int slot, int count,
                                                     const float* __restrict__ dI, int w, int n, const int* __restrict__ n_dev,
                                                     int cs, const int* __restrict__ cand, int* __restrict__ added) {
  using Scan = cub::BlockScan<int, kAddThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const size_t stride = (size_t)kSlots * cap;
  float* f = reinterpret_cast<float*>(st);
  if (n_dev) n = *n_dev;
  int base = count;
  for (int c0 = 0; c0 < n; c0 += kAddThreads) {
    const int c = c0 + threadIdx.x;
    float col[8], wt[8], g00 = 0.f, g01 = 0.f, g10 = 0.f, g11 = 0.f;
    int ok = 0, u = 0, v = 0;
    float type = 0.f;
    if (c < n) {
      u = cand[c]; v = cand[cs + c]; type = __int_as_float(cand[2 * cs + c]);
      ok = 1;
      for (int k = 0; k < 8; ++k) {
        // getInterpolatedElement33BiLin (globalFuncs.h:166-188) at integer coordinates
        const float x = (float)(u + c_pattern[k][0]), y = (float)(v + c_pattern[k][1]);
        const int ix = (int)x, iy = (int)y;
        const float* bp = dI + 3 * ((long long)ix + (long long)iy * w);
        const float tl = __ldg(bp), tr = __ldg(bp + 3), bl = __ldg(bp + 3 * w), br = __ldg(bp + 3 * w + 3);
        const float dx = fs(x, (float)ix), dy = fs(y, (float)iy);
        const float topInt = fa(fm(dx, tr), fm(fs(1.f, dx), tl));
        const float botInt = fa(fm(dx, br), fm(fs(1.f, dx), bl));
        const float leftInt = fa(fm(dy, bl), fm(fs(1.f, dy), tl));
        const float rightInt = fa(fm(dy, br), fm(fs(1.f, dy), tr));
        const float p0 = fa(fm(dx, rightInt), fm(fs(1.f, dx), leftInt)), p1 = fs(rightInt, leftInt), p2 = fs(botInt, topInt);
        col[k] = p0;
        if (!isfinite(p0)) { ok = 0; break; }
        g00 = fa(g00, fm(p1, p1)); g01 = fa(g01, fm(p1, p2)); g10 = fa(g10, fm(p2, p1)); g11 = fa(g11, fm(p2, p2));
        wt[k] = __fsqrt_rn(fd(S.outlier_th_sum_component, fa(S.outlier_th_sum_component, fa(fm(p1, p1), fm(p2, p2)))));
      }
    }
    int pos, tot;
    Scan(tmp).ExclusiveSum(ok, pos, tot);
    if (ok && base + pos < cap) {
      const size_t p = (size_t)slot * cap + base + pos;
      float eth = fm(8.f, S.outlier_th);
      eth = fm(eth, fm(S.overall_energy_th_weight, S.overall_energy_th_weight));
      f[IM_U * stride + p] = (float)u; f[IM_V * stride + p] = (float)v; f[IM_TYPE * stride + p] = type; f[IM_ETH * stride + p] = eth;
      f[IM_IDMIN * stride + p] = 0.f; f[IM_IDMAX * stride + p] = __int_as_float(0x7fc00000); f[IM_QUALITY * stride + p] = 10000.f;
      st[IM_STATUS * stride + p] = IPS_UNINITIALIZED;
      f[IM_UVX * stride + p] = 0.f; f[IM_UVY * stride + p] = 0.f; f[IM_INTERVAL * stride + p] = 0.f;
      for (int k = 0; k < 8; ++k) { f[(IM_COLOR + k) * stride + p] = col[k]; f[(IM_WEIGHTS + k) * stride + p] = wt[k]; }
      f[IM_GRADH * stride + p] = g00; f[(IM_GRADH + 1) * stride + p] = g01; f[(IM_GRADH + 2) * stride + p] = g10;
      f[(IM_GRADH + 3) * stride + p] = g11;
    }
    base += tot;
    __syncthreads();   // tmp is reused by the next chunk
  }
  if (threadIdx.x == 0) *added = base - count;
}

// activatePointsMT's compaction as a gather: new point i of the slot is old point src[i]
__global__ void k_gather(const uint32_t* __restrict__ st, uint32_t* __restrict__ scratch, int cap, int slot, int n,
                         const int* __restrict__ src) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * kRows) return;
  const int r = i / n, j = i % n;
  scratch[(size_t)r * cap + j] = st[(size_t)r * kSlots * cap + (size_t)slot * cap + src[j]];
}
__global__ void k_scatter_back(uint32_t* __restrict__ st, const uint32_t* __restrict__ scratch, int cap, int slot, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * kRows) return;
  const int r = i / n, j = i % n;
  st[(size_t)r * kSlots * cap + (size_t)slot * cap + j] = scratch[(size_t)r * cap + j];
}

// ---- n9: activation (FullSystem::optimizeImmaturePoint, FullSystemOptPoint.cpp:51-205, with
// ImmaturePoint::linearizeResidual, ImmaturePoint.cpp:476-543, and the 5-argument projectPoint / derive_idepth,
// ResidualProjections.h:36-87) for every candidate of activatePointsMT in one launch.
//
// Shape (DESIGN.md, n9): one warp per candidate.  Residual r (to frame r, or r + 1 past the host) and pattern index i form
// pair q = 8 r + i; lane l evaluates pairs l and l + 32 (so its pattern index is l & 7) at the current inverse depth and
// leaves (in image, energy term, Hdd term, bd term) in shared memory.  Every lane then runs the reference's three serial
// chains - the residual's energy, Hdd / bd across (residual, pattern index), lastEnergy across residuals - over the 56 slots
// in the reference's order, so every lane holds the same state and every branch is warp-uniform; lane 0 stores.
constexpr int kActThreads = 128, kActWarps = kActThreads / 32, kActPairs = 64;
enum { RS_IN = 0, RS_OOB = 1, RS_OUTLIER = 2 };   // ResState
struct ActivateLaunch {
  const float* dI[kSlots];          // level 0 of frame f
  float pc[kSlots][kSlots][14];     // [host][target]: PRE_RTll row-major, PRE_tTll, PRE_aff_mode
  int slot[kSlots];
  int n_frames, n_cand, w, h, cap, gn_its, min_obs;
  float fxl, fyl, cxl, cyl, fxli, fyli, huber, min_h;
};

struct ActPair {
  float e, hdd, bd;
  int ok;
};

// linearizeResidual of every residual at `idepth` with `slack`, in the reference's order: *energy (lastEnergy / newEnergy)
// is a float increased by each residual's double return; ns / nE receive state_NewState / state_NewEnergy
__device__ __forceinline__ void act_linearize(const ActivateLaunch& L, ActPair* sm, int lane, int hf, float u, float v, float eth,
                                              float col, float wt, float idepth, float slack, const int (&ss)[kSlots - 1],
                                              const float (&se)[kSlots - 1], int (&ns)[kSlots - 1], float (&nE)[kSlots - 1],
                                              float* energy, float* Hdd, float* bd) {
  const int nres = L.n_frames - 1, i = lane & 7;
  const float wM3G = (float)(L.w - 3), hM3G = (float)(L.h - 3);
  __syncwarp();   // the previous evaluation's slots have been read
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int q = lane + 32 * half, r = q >> 3;
    if (r >= nres) continue;
    const int t = r < hf ? r : r + 1;
    const float* P = L.pc[hf][t];
    ActPair a{0.f, 0.f, 0.f, 0};
    // projectPoint, 5-argument form
    const float K0 = fm(fs(fa(u, (float)c_pattern[i][0]), L.cxl), L.fxli), K1 = fm(fs(fa(v, (float)c_pattern[i][1]), L.cyl), L.fyli);
    const float p0 = fa(fa(fa(fm(P[0], K0), fm(P[1], K1)), fm(P[2], 1.f)), fm(P[9], idepth));
    const float p1 = fa(fa(fa(fm(P[3], K0), fm(P[4], K1)), fm(P[5], 1.f)), fm(P[10], idepth));
    const float p2 = fa(fa(fa(fm(P[6], K0), fm(P[7], K1)), fm(P[8], 1.f)), fm(P[11], idepth));
    const float drescale = fd(1.0f, p2);
    if (drescale > 0) {
      const float pu = fm(p0, drescale), pv = fm(p1, drescale);
      const float Ku = fa(fm(pu, L.fxl), L.cxl), Kv = fa(fm(pv, L.fyl), L.cyl);
      if (Ku > 1.1f && Kv > 1.1f && Ku < wM3G && Kv < hM3G) {
        float hit[3];
        interp<3>(L.dI[t], Ku, Kv, L.w, hit);
        if (isfinite(hit[0])) {
          const float residual = fs(hit[0], fa(fm(P[12], col), P[13]));
          float hw = fabsf(residual) < L.huber ? 1.f : fd(L.huber, fabsf(residual));
          a.e = fm(fm(fm(fm(fm(wt, wt), hw), residual), residual), fs(2.f, hw));
          const float dxInterp = fm(hit[1], L.fxl), dyInterp = fm(hit[2], L.fyl);
          // derive_idepth; SCALE_IDEPTH is 1
          const float d_idepth = fa(fm(fm(dxInterp, drescale), fs(P[9], fm(P[11], pu))),
                                    fm(fm(dyInterp, drescale), fs(P[10], fm(P[11], pv))));
          hw = fm(hw, fm(wt, wt));
          a.hdd = fm(fm(hw, d_idepth), d_idepth);
          a.bd = fm(fm(hw, residual), d_idepth);
          a.ok = 1;
        }
      }
    }
    sm[q] = a;
  }
  __syncwarp();
  const float th = fm(eth, slack);
#pragma unroll
  for (int r = 0; r < kSlots - 1; ++r) {
    if (r >= nres) break;
    double ret;
    if (ss[r] == RS_OOB) {   // sticky
      ns[r] = RS_OOB;
      ret = (double)se[r];
    } else {
      float el = 0.f;
      bool oob = false;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const ActPair a = sm[8 * r + k];
        if (!a.ok) { oob = true; break; }   // the Hdd / bd of pattern indices 0..k-1 stay added
        el = fa(el, a.e);
        *Hdd = fa(*Hdd, a.hdd);
        *bd = fa(*bd, a.bd);
      }
      if (oob) {
        ns[r] = RS_OOB;
        ret = (double)se[r];
      } else {
        if (el > th) { el = th; ns[r] = RS_OUTLIER; } else { ns[r] = RS_IN; }
        nE[r] = el;
        ret = (double)el;
      }
    }
    *energy = __double2float_rn(__dadd_rn((double)*energy, ret));
  }
}

__global__ void __launch_bounds__(kActThreads) k_activate(ActivateLaunch L, const uint32_t* __restrict__ st,
                                                          const int* __restrict__ cand, int* __restrict__ result,
                                                          float* __restrict__ out_idepth, float* __restrict__ out_energy,
                                                          signed char* __restrict__ out_state) {
  __shared__ ActPair smem[kActWarps][kActPairs];
  const int k = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (k >= L.n_cand) return;   // warp-uniform
  ActPair* sm = smem[threadIdx.x >> 5];
  const int hf = cand[k];
  const size_t stride = (size_t)kSlots * L.cap, p = (size_t)L.slot[hf] * L.cap + cand[L.n_cand + k];
  const float* f = reinterpret_cast<const float*>(st);
  const float u = f[IM_U * stride + p], v = f[IM_V * stride + p], eth = f[IM_ETH * stride + p];
  const float idmin = f[IM_IDMIN * stride + p], idmax = f[IM_IDMAX * stride + p];
  const float col = f[(IM_COLOR + (lane & 7)) * stride + p], wt = f[(IM_WEIGHTS + (lane & 7)) * stride + p];
  const int nres = L.n_frames - 1;

  int ss[kSlots - 1], ns[kSlots - 1];
  float se[kSlots - 1], nE[kSlots - 1];
#pragma unroll
  for (int r = 0; r < kSlots - 1; ++r) { ss[r] = RS_IN; ns[r] = RS_OUTLIER; se[r] = 0.f; nE[r] = 0.f; }
  float lastEnergy = 0.f, lastHdd = 0.f, lastbd = 0.f;
  float currentIdepth = fm(fa(idmax, idmin), 0.5f);
  act_linearize(L, sm, lane, hf, u, v, eth, col, wt, currentIdepth, 1000.f, ss, se, ns, nE, &lastEnergy, &lastHdd, &lastbd);
#pragma unroll
  for (int r = 0; r < kSlots - 1; ++r) { ss[r] = ns[r]; se[r] = nE[r]; }
  int res;
  if (!isfinite(lastEnergy) || lastHdd < L.min_h) {
    res = 0;
  } else {
    res = 1;
    float lambda = 0.1f;
    for (int it = 0; it < L.gn_its; it++) {
      const float H = fm(lastHdd, fa(1.f, lambda));
      const float step = __double2float_rn(__dmul_rn(__ddiv_rn(1.0, (double)H), (double)lastbd));
      const float newIdepth = fs(currentIdepth, step);
      float newHdd = 0.f, newbd = 0.f, newEnergy = 0.f;
      act_linearize(L, sm, lane, hf, u, v, eth, col, wt, newIdepth, 1.f, ss, se, ns, nE, &newEnergy, &newHdd, &newbd);
      if (!isfinite(lastEnergy) || newHdd < L.min_h) { res = 0; break; }
      if (newEnergy < lastEnergy) {
        currentIdepth = newIdepth;
        lastHdd = newHdd;
        lastbd = newbd;
        lastEnergy = newEnergy;
#pragma unroll
        for (int r = 0; r < kSlots - 1; ++r) { ss[r] = ns[r]; se[r] = nE[r]; }
        lambda = __double2float_rn(__dmul_rn((double)lambda, 0.5));
      } else {
        lambda = __double2float_rn(__dmul_rn((double)lambda, 5.0));
      }
      if ((double)fabsf(step) < __dmul_rn(0.0001, (double)currentIdepth)) break;
    }
    if (res) {
      int good = 0;
#pragma unroll
      for (int r = 0; r < kSlots - 1; ++r) good += r < nres && ss[r] == RS_IN;
      if (!isfinite(currentIdepth) || good < L.min_obs || !isfinite(eth)) res = -1;
    }
  }
  if (lane == 0) {
    result[k] = res;
    out_idepth[k] = currentIdepth;
    const size_t o = (size_t)k * L.n_frames;
    out_state[o + hf] = -1;
    out_energy[o + hf] = __int_as_float(0x7fc00000);
#pragma unroll
    for (int r = 0; r < kSlots - 1; ++r) {
      if (r >= nres) break;
      const int t = r < hf ? r : r + 1;
      out_state[o + t] = (signed char)ss[r];
      out_energy[o + t] = se[r];
    }
  }
}

class ImmatureImpl final : public ImmatureIface {
 public:
  ImmatureImpl(int w, int h, int cap, const float* settings, int device) : w_(w), h_(h), cap_(cap), device_(device) {
    int nd = 0;
    if (cudaGetDeviceCount(&nd) != cudaSuccess || nd == 0)
      throw Error("tandem_b200: no CUDA device visible - this library has no CPU fallback");
    TDM_CHECK(w >= 10 && h >= 10 && cap >= 1 && (long long)cap * kSlots <= (1 << 24), "bad immature-point set shape");
    TDM_CHECK(settings, "null argument");
    std::memcpy(&s_, settings, sizeof s_);
    TDM_CHECK(s_.gn_iterations >= 0 && s_.gn_iterations <= 1000 && s_.min_trace_test_radius >= 0, "bad trace settings");
    TDM_CUDA(cudaSetDevice(device_));
    stream_ = make_stream(0);
    done_ = make_event(cudaEventDisableTiming);
    st_ = make_dev<uint32_t>(4ull * kRows * kSlots * cap);
    scratch_ = make_dev<uint32_t>(4ull * kRows * cap);
    d_cand_ = make_dev<int>(4ull * 3 * cap);
    h_cand_ = make_host<int>(4ull * 3 * cap);
    d_added_ = make_dev<int>(4);
    h_added_ = make_host<int>(4);
    h_rows_ = make_host<float>(4ull * kRows * cap);
  }
  ~ImmatureImpl() override {
    cudaSetDevice(device_);
    cudaStreamSynchronize(stream_.get());
  }

  int add(int slot, const PyramidIface& host, int n, const int* u, const int* v, const float* type) override {
    check_slot(slot);
    check_pyramid(host);
    TDM_CHECK(n >= 0 && (n == 0 || (u && v && type)), "null argument");
    TDM_CHECK((long long)count_[slot] + n <= cap_, "immature-point set: the slot's capacity cannot hold the candidates");
    for (int i = 0; i < n; ++i)
      TDM_CHECK(u[i] >= 2 && u[i] <= w_ - 4 && v[i] >= 2 && v[i] <= h_ - 4,
                "immature-point candidate: the pattern around the pixel leaves the image");
    if (n == 0) return 0;
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));   // h_cand_ is free
    std::memcpy(h_cand_.get(), u, 4ull * n);
    std::memcpy(h_cand_.get() + n, v, 4ull * n);
    std::memcpy(h_cand_.get() + 2 * n, type, 4ull * n);
    TDM_CUDA(cudaMemcpyAsync(d_cand_.get(), h_cand_.get(), 12ull * n, cudaMemcpyHostToDevice, stream_.get()));
    TDM_CUDA(cudaStreamWaitEvent(stream_.get(), (cudaEvent_t)host.ready_event(), 0));
    k_add<<<1, kAddThreads, 0, stream_.get()>>>(s_, st_.get(), cap_, slot, count_[slot], host.level_dI(0), w_, n, nullptr, n,
                                                d_cand_.get(), d_added_.get());
    TDM_CUDA(cudaGetLastError());
    TDM_CUDA(cudaMemcpyAsync(h_added_.get(), d_added_.get(), 4, cudaMemcpyDeviceToHost, stream_.get()));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    count_[slot] += *h_added_;
    return *h_added_;
  }

  void trace(const PyramidIface& frame, int n_hosts, const int* slots, const PyramidIface* const* host_pyramids,
             const float* KRKi, const float* Kt, const float* aff) override {
    TDM_CHECK(n_hosts >= 0 && n_hosts <= kSlots, "n_hosts outside 0..8");
    TDM_CHECK(n_hosts == 0 || (slots && KRKi && Kt && aff), "null argument");
    check_pyramid(frame);
    TraceLaunch L{};
    L.n_hosts = n_hosts; L.w = w_; L.h = h_; L.cap = cap_; L.s = s_;
    int warps = 0;
    for (int j = 0; j < n_hosts; ++j) {
      check_slot(slots[j]);
      for (int q = 0; q < j; ++q) TDM_CHECK(slots[q] != slots[j], "a host slot appears twice");
      if (host_pyramids && host_pyramids[j]) check_pyramid(*host_pyramids[j]);
      TraceHost& H = L.host[j];
      std::memcpy(H.K, KRKi + 9 * j, sizeof H.K);
      std::memcpy(H.Kt, Kt + 3 * j, sizeof H.Kt);
      std::memcpy(H.aff, aff + 2 * j, sizeof H.aff);
      H.slot = slots[j]; H.n = count_[slots[j]]; H.first_warp = warps;
      warps += H.n;
    }
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaStreamWaitEvent(stream_.get(), (cudaEvent_t)frame.ready_event(), 0));
    for (int j = 0; j < n_hosts; ++j)
      if (host_pyramids && host_pyramids[j]) TDM_CUDA(cudaStreamWaitEvent(stream_.get(), (cudaEvent_t)host_pyramids[j]->ready_event(), 0));
    if (warps > 0) {
      k_trace<<<cdiv(warps, 4), 128, 0, stream_.get()>>>(L, st_.get(), frame.level_dI(0));
      TDM_CUDA(cudaGetLastError());
    }
    // a later build or destroy of a pyramid read here waits for the trace
    TDM_CUDA(cudaEventRecord(done_.get(), stream_.get()));
    frame.wait_for(done_.get());
    for (int j = 0; j < n_hosts; ++j)
      if (host_pyramids && host_pyramids[j]) host_pyramids[j]->wait_for(done_.get());
  }

  void activate(int n_frames, const int* frame_slots, const PyramidIface* const* frame_pyramids, const float* precalc,
                const float* calib4, float min_idepth_h_act, int gn_iterations, int min_obs, int n_cand, const int* cand_frame,
                const int* cand_index, int* result, float* idepth, signed char* res_state, float* res_energy) override {
    TDM_CHECK(n_frames >= 1 && n_frames <= kSlots, "n_frames outside 1..8");
    TDM_CHECK(frame_slots && frame_pyramids && precalc && calib4, "null argument");
    TDM_CHECK(gn_iterations >= 0 && gn_iterations <= 100 && min_obs >= 0, "bad activation settings");
    TDM_CHECK(n_cand >= 0 && (n_cand == 0 || (cand_frame && cand_index)), "null argument");
    ActivateLaunch L{};
    L.n_frames = n_frames; L.n_cand = n_cand; L.w = w_; L.h = h_; L.cap = cap_; L.gn_its = gn_iterations; L.min_obs = min_obs;
    for (int f = 0; f < n_frames; ++f) {
      TDM_CHECK(frame_slots[f] >= -1 && frame_slots[f] < kSlots, "frame slot outside -1..7");
      for (int q = 0; q < f; ++q) TDM_CHECK(frame_slots[f] < 0 || frame_slots[q] != frame_slots[f], "a frame slot appears twice");
      TDM_CHECK(frame_pyramids[f], "null argument");
      check_pyramid(*frame_pyramids[f]);
      L.dI[f] = frame_pyramids[f]->level_dI(0);
      L.slot[f] = frame_slots[f];
      for (int t = 0; t < n_frames; ++t) std::memcpy(L.pc[f][t], precalc + 14 * ((size_t)f * n_frames + t), sizeof L.pc[f][t]);
    }
    std::vector<std::vector<char>> seen(n_frames);
    for (int k = 0; k < n_cand; ++k) {
      const int f = cand_frame[k];
      TDM_CHECK(f >= 0 && f < n_frames && frame_slots[f] >= 0, "candidate frame outside the frames with a slot");
      const int n = count_[frame_slots[f]];
      TDM_CHECK(cand_index[k] >= 0 && cand_index[k] < n, "candidate index outside its slot's points");
      seen[f].resize(n, 0);
      TDM_CHECK(!seen[f][cand_index[k]], "a candidate appears twice");
      seen[f][cand_index[k]] = 1;
    }
    if (n_cand == 0) return;
    L.fxl = calib4[0]; L.fyl = calib4[1]; L.cxl = calib4[2]; L.cyl = calib4[3];
    L.fxli = 1.0f / L.fxl; L.fyli = 1.0f / L.fyl;   // CalibHessian::setValueScaled (HessianBlocks.h:435-436)
    L.huber = s_.huber; L.min_h = min_idepth_h_act;
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));   // the staging buffers are free
    reserve_activate(n_cand);
    int* hc = h_act_cand_.get();
    std::memcpy(hc, cand_frame, 4ull * n_cand);
    std::memcpy(hc + n_cand, cand_index, 4ull * n_cand);
    TDM_CUDA(cudaMemcpyAsync(d_act_cand_.get(), hc, 8ull * n_cand, cudaMemcpyHostToDevice, stream_.get()));
    for (int f = 0; f < n_frames; ++f)
      TDM_CUDA(cudaStreamWaitEvent(stream_.get(), (cudaEvent_t)frame_pyramids[f]->ready_event(), 0));
    // output layout: result int[n], idepth float[n], energy float[n * n_frames], state int8[n * n_frames]
    char* d = d_act_out_.get();
    const size_t nn = (size_t)n_cand * n_frames, bytes = 8ull * n_cand + 5ull * nn;
    k_activate<<<cdiv(n_cand, kActWarps), kActThreads, 0, stream_.get()>>>(
        L, st_.get(), d_act_cand_.get(), reinterpret_cast<int*>(d), reinterpret_cast<float*>(d + 4ull * n_cand),
        reinterpret_cast<float*>(d + 8ull * n_cand), reinterpret_cast<signed char*>(d + 8ull * n_cand + 4 * nn));
    TDM_CUDA(cudaGetLastError());
    TDM_CUDA(cudaMemcpyAsync(h_act_out_.get(), d, bytes, cudaMemcpyDeviceToHost, stream_.get()));
    // a later build or destroy of a pyramid read here waits for the activation
    TDM_CUDA(cudaEventRecord(done_.get(), stream_.get()));
    for (int f = 0; f < n_frames; ++f) frame_pyramids[f]->wait_for(done_.get());
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    const char* h = h_act_out_.get();
    if (result) std::memcpy(result, h, 4ull * n_cand);
    if (idepth) std::memcpy(idepth, h + 4ull * n_cand, 4ull * n_cand);
    if (res_energy) std::memcpy(res_energy, h + 8ull * n_cand, 4 * nn);
    if (res_state) std::memcpy(res_state, h + 8ull * n_cand + 4 * nn, nn);
  }

  int make_new_traces(int slot, SelectorIface& sel, const PyramidIface& p, float density, SelectResult* r, int* u, int* v,
                      float* type) override {
    check_slot(slot);
    check_pyramid(p);
    TDM_CHECK(sel.width() == w_ && sel.height() == h_, "pixel selector and immature-point set differ in image size");
    TDM_CHECK(sel.device() == device_, "pixel selector and immature-point set live on different devices");
    sel.check(p, density, 1, 1.f);
    TDM_CUDA(cudaSetDevice(device_));
    const int count = count_[slot], free = cap_ - count;
    sel.enqueue(stream_.get(), p, density, 1, 1.f, true);
    const SelectorIface::Candidates c = sel.candidates();
    k_add<<<1, kAddThreads, 0, stream_.get()>>>(s_, st_.get(), cap_, slot, count, p.level_dI(0), w_, 0, c.count, c.stride, c.cand,
                                                d_added_.get());
    TDM_CUDA(cudaGetLastError());
    TDM_CUDA(cudaMemcpyAsync(h_added_.get(), d_added_.get(), 4, cudaMemcpyDeviceToHost, stream_.get()));
    // rows IM_U, IM_V, IM_TYPE of the slot's free part
    if ((u || v || type) && free > 0)
      TDM_CUDA(cudaMemcpy2DAsync(h_rows_.get(), 4ull * free, st_.get() + (size_t)slot * cap_ + count, 4ull * kSlots * cap_, 4ull * free,
                                 3, cudaMemcpyDeviceToHost, stream_.get()));
    // a later build or destroy of the pyramid waits for the call
    TDM_CUDA(cudaEventRecord(done_.get(), stream_.get()));
    p.wait_for(done_.get());
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    const int added = *h_added_;
    TDM_CHECK(added <= free, "make_new_traces: the slot's free capacity cannot hold the kept points");
    SelectResult tmp;
    sel.result(r ? r : &tmp, true);
    count_[slot] += added;
    const float* rows = h_rows_.get();
    for (int i = 0; i < added; ++i) {
      if (u) u[i] = (int)rows[i];
      if (v) v[i] = (int)rows[free + i];
      if (type) type[i] = rows[2 * free + i];
    }
    return added;
  }

  int count(int slot) override { check_slot(slot); return count_[slot]; }

  void get(int slot, int first, int n, float* const* rows) override {
    check_slot(slot);
    TDM_CHECK(first >= 0 && n >= 0 && (long long)first + n <= count_[slot], "get: range outside the slot's points");
    TDM_CUDA(cudaSetDevice(device_));
    if (n > 0) {
      TDM_CUDA(cudaMemcpy2DAsync(h_rows_.get(), 4ull * n, st_.get() + (size_t)slot * cap_ + first, 4ull * kSlots * cap_, 4ull * n,
                                 kRows, cudaMemcpyDeviceToHost, stream_.get()));
    }
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    for (int r = 0; r < kRows; ++r)
      if (rows[r]) std::memcpy(rows[r], h_rows_.get() + (size_t)r * n, 4ull * n);
  }

  void remove(int slot, int n_removed, const int* indices) override {
    check_slot(slot);
    const int n = count_[slot];
    TDM_CHECK(n_removed >= 0 && (n_removed == 0 || indices), "null argument");
    std::vector<int> idx(n);
    std::vector<char> null(n, 0);
    for (int k = 0; k < n_removed; ++k) {
      TDM_CHECK(indices[k] >= 0 && indices[k] < n, "remove: index outside the slot's points");
      TDM_CHECK(!null[indices[k]], "remove: an index appears twice");
      null[indices[k]] = 1;
    }
    if (n_removed == 0) return;
    // FullSystem.cpp:849-856: a null entry takes back(), which is popped, and is looked at again
    for (int i = 0; i < n; ++i) idx[i] = i;
    int m = n;
    for (int i = 0; i < m; i++) {
      if (null[idx[i]]) {
        idx[i] = idx[m - 1];
        --m;
        i--;
      }
    }
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));   // h_cand_ is free
    if (m > 0) {
      std::memcpy(h_cand_.get(), idx.data(), 4ull * m);
      TDM_CUDA(cudaMemcpyAsync(d_cand_.get(), h_cand_.get(), 4ull * m, cudaMemcpyHostToDevice, stream_.get()));
      k_gather<<<cdiv((long long)m * kRows, 256), 256, 0, stream_.get()>>>(st_.get(), scratch_.get(), cap_, slot, m, d_cand_.get());
      k_scatter_back<<<cdiv((long long)m * kRows, 256), 256, 0, stream_.get()>>>(st_.get(), scratch_.get(), cap_, slot, m);
      TDM_CUDA(cudaGetLastError());
    }
    count_[slot] = m;
  }

  void drop_host(int slot) override { check_slot(slot); count_[slot] = 0; }
  void synchronize() override { TDM_CUDA(cudaSetDevice(device_)); TDM_CUDA(cudaStreamSynchronize(stream_.get())); }
  int width() const override { return w_; }
  int height() const override { return h_; }
  int device() const override { return device_; }

 private:
  void check_slot(int slot) const { TDM_CHECK(slot >= 0 && slot < kSlots, "host slot outside 0..7"); }
  void check_pyramid(const PyramidIface& p) const {
    TDM_CHECK(p.width(0) == w_ && p.height(0) == h_, "pyramid level 0 is not the set's image size");
    TDM_CHECK(p.device() == device_, "pyramid and immature-point set live on different devices");
  }
  // the activation's candidate and output buffers, made on first use for at least n candidates (at most every point of
  // every slot); kept only once all of them exist.  The stream is idle when this runs.
  void reserve_activate(int n) {
    if (n <= act_cap_) return;
    const int c = (int)std::min<long long>(std::max<long long>(n, 2ll * act_cap_), (long long)kSlots * cap_);
    const size_t out = 8ull * c + 5ull * c * kSlots;
    DevPtr<int> dc = make_dev<int>(8ull * c);
    HostPtr<int> hc = make_host<int>(8ull * c);
    DevPtr<char> dout = make_dev<char>(out);
    HostPtr<char> hout = make_host<char>(out);
    d_act_cand_ = std::move(dc); h_act_cand_ = std::move(hc); d_act_out_ = std::move(dout); h_act_out_ = std::move(hout);
    act_cap_ = c;
  }
  int w_, h_, cap_, device_;
  Settings s_;
  int count_[kSlots] = {};
  Stream stream_;
  Event done_;
  DevPtr<uint32_t> st_, scratch_;
  DevPtr<int> d_cand_, d_added_;
  HostPtr<int> h_cand_, h_added_;
  HostPtr<float> h_rows_;
  int act_cap_ = 0;
  DevPtr<int> d_act_cand_;
  HostPtr<int> h_act_cand_;
  DevPtr<char> d_act_out_;
  HostPtr<char> h_act_out_;
};

}  // namespace

static_assert(sizeof(Settings) == 12 * 4, "tdm_trace_settings layout");

ImmatureIface* make_immature(int w, int h, int capacity_per_host, const float* settings, int device) {
  return new ImmatureImpl(w, h, capacity_per_host, settings, device);
}

}  // namespace tdm
