// Dense photometric tracker, pyramid level 0, behind the CudaCoarseTracker call surface
// (tandem/libdr/cuda_coarse_tracker/include/public/cuda_coarse_tracker.h:9-82).
//
// Reference being replaced (SURVEY.md §8 a14-a16, Appendix A.3):
//   calcResKernelNew<128>  cuda_coarse_tracker_private.cu:41-214   7 x cub::BlockReduce + 7 float atomics / block
//   calcGKernel<128,float> cuda_coarse_tracker_private.cu:261-394  45 serialized block reductions, <1 wave
//   host wrapper           cuda_coarse_tracker.cpp:195-356          memset + H2D + kernel + sync + D2H per call
// Design: K8 = ONE kernel template for calcRes, calcG and the fused calcRes+calcG.  264 persistent CTAs
// (2 per SM) grid-stride over the points, per-thread fp32 partials are widened to double, reduced with warp
// shuffles and one shared-memory pass, each CTA writes its partial vector, and the last CTA to finish (atomic
// ticket) adds the partials in a fixed order and writes the result straight into mapped pinned host memory:
// deterministic (the reference's float atomics are not), one launch, no memset, no D2H copy.
#include <climits>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include <cub/device/device_radix_sort.cuh>

#include "tracker.h"

namespace tdm {

namespace {

constexpr int kThreads = 256;
constexpr int kBlocks = 264;  // 2 x 132 SMs (H100 SXM)
constexpr int kRes = 7;       // E, numTermsInE, numTermsInWarped, numSaturated, shiftT, shiftRT, shiftNum
constexpr int kG = 45;
constexpr int kOut = kRes + kG;

struct TrkParams {
  int w, h, n;
  float fx, fy, cx, cy;
  float RKi[9], Ki[9], t[3];
  float affa, affb;     // affLL
  float ref_b;          // ref_aff_g2l.b  (calcG's b0)
  float huber, cutoff, maxEnergy;
};

// pose-dependent parameters as the device-side LM loop (tdm_tracker_track) hands them from one evaluation to the next
struct TrkPose {
  float RKi[9], t[3];
  float affa, affb;
  float cutoff, maxEnergy;
};

struct LmCtx;
struct TrkBufs {
  LmCtx* lm;            // device LM loop (tdm_tracker_track / _track_pyramid): level, pose in, LM step out; nullptr for the plain calls
  const float *pc_u, *pc_v, *pc_idepth, *pc_color, *dInew;
  float* warped;        // 7 x n_max: u, v, dx, dy, idepth, residual, weight
  long long n_max;
  double* partials;     // [kBlocks][kOut]
  unsigned* ticket;
  double* out;          // mapped pinned host memory, kOut doubles
  const TrkPose* batch; // MODE 3: one pose per blockIdx.y (motion hypotheses evaluated in ONE launch); partials / ticket / out are
                        // then arrays indexed by blockIdx.y
};

// ---- device LM loop (n3 one level, n5 coarse-to-fine), see the n3 / n5 section below ----
constexpr int kMaxLevels = 5;   // CoarseTracker::trackNewestCoarse: coarsestLvl < 5
struct LmConfig {
  float Ki[9];
  float ref_exposure, new_exposure;
  double ref_aff[2];
  float huber, coarse_cutoff;
  int max_iter;
  float lambda_limit;
  int fix_a, fix_b;
};
struct LmLevel {             // one pyramid level: its tracker's parameters and buffers, as the host hands them over
  TrkParams p;               // pose-dependent fields are taken from LmCtx::pose
  const float *pc_u, *pc_v, *pc_idepth, *pc_color, *dInew;
  LmConfig cfg;
};
struct LmIn {                // uploaded once per call
  LmLevel lv[kMaxLevels];    // lv[l] = pyramid level l
  double T0[16], aff0[2];
  double min_res[kMaxLevels];   // minResForAbort (pyramid mode)
  float mode_a, mode_b;         // setting_affineOptModeA/B (pyramid mode; < 0 = fixed)
  int coarsest;
  int pyramid;               // 0: one level (tdm_tracker_track), 1: the coarse-to-fine rules of trackNewestCoarse,
                             // 2: those rules once per motion hypothesis of trackNewCoarse (LmCtx::rin)
  int max_evals;             // bound on the evaluations of the whole call (the rules never exceed it)
};
struct LmState {
  double T[16], aff[2];      // accepted
  double Tn[16], affn[2];    // candidate under evaluation
  double res_old[6], H[64], b[8];
  float lambda;              // float as in the reference (CoarseTracker.cpp:798), like its extrapolation factor (:842)
  double inc_norm;
  float repeat;
  int phase, iter, evals;    // of the current pass over the current level
};
struct LmResult {            // mapped pinned host memory (device copy in LmCtx::r)
  double T[16], aff[2];
  double res[kMaxLevels][6];       // resOld of each level's last pass
  double last_res[kMaxLevels];     // lastResiduals, NaN for levels not reached (pyramid mode)
  double flow[3];                  // lastFlowIndicators (pyramid mode)
  int iterations[kMaxLevels], evaluations[kMaxLevels];   // summed over the passes of a level
  float repeat[kMaxLevels];        // largest levelCutoffRepeat of each level's passes
  int num_warped;
  int ok, aborted_level, repeated_level;
  int done;                        // written last: 1 = finished, 2 = evaluation bound exceeded (internal error)
};
// ---- n6: the motion-hypothesis loop of FullSystem::trackNewCoarse around n5 (pyramid mode 2), see the n6 section below ----
constexpr int kMaxTries = 64;     // as calc_res_batch; the reference builds at most 31
struct TryRec {              // one try's outcome (tdm_track_try)
  double last_res[kMaxLevels];
  int ok, aborted_level, repeated_level;
  int evaluations[kMaxLevels];
};
struct RetrackOut {          // mapped pinned host memory of tdm_tracker_track_new_coarse, written only in mode 2
  double T[16], aff[2], achieved[kMaxLevels], flow[3];   // lastF_2_fh, aff_g2l, achievedRes, flowVecs
  int have_one_good, tries, winner;
  int done;                  // written after everything else: 1 = finished, 2 = evaluation bound exceeded (internal error)
  TryRec rec[kMaxTries];
};
struct RetrackIn {           // uploaded by tdm_tracker_track_new_coarse only: this header + n_tries poses
  RetrackOut* out;           // device pointer of the mapped result
  double last_rmse0;         // lastCoarseRMSE[0]
  float threshold;           // setting_reTrackThreshold
  int n_tries;
  double tries[kMaxTries][16];   // lastF_2_fh_tries, row-major
};
struct RetrackState {
  double achieved[kMaxLevels], T[16], aff[2], flow[3];   // achievedRes; pose, aff and flow of the last winner
  int have_one_good, cur, winner;                       // cur = the try under way
};
struct LmCtx {               // device memory, one per tracker
  LmIn in;
  LmState s;
  TrkPose pose;
  int lvl;                   // level under evaluation
  int have_repeated, total_evals;
  LmResult r;
  LmResult* out;             // mapped pinned host memory
  cudaGraphConditionalHandle loop;   // the WHILE node around the evaluation kernel
  RetrackIn rin;             // n6 only
  RetrackState rs;
};

__device__ __noinline__ void lm_step(LmCtx* c, const double* o);

__device__ __forceinline__ float3 bilinear33(const float* __restrict__ mat, float x, float y, int width) {  // cu:22-38
  const int ix = (int)x, iy = (int)y;
  const float dx = x - ix, dy = y - iy, dxdy = dx * dy;
  const float* bp = mat + 3 * (ix + iy * width);
  const float w11 = dxdy, w01 = dy - dxdy, w10 = dx - dxdy, w00 = 1.0f - dx - dy + dxdy;
  float3 r;
  r.x = w11 * bp[3 * (1 + width)] + w01 * bp[3 * width] + w10 * bp[3] + w00 * bp[0];
  r.y = w11 * bp[3 * (1 + width) + 1] + w01 * bp[3 * width + 1] + w10 * bp[4] + w00 * bp[1];
  r.z = w11 * bp[3 * (1 + width) + 2] + w01 * bp[3 * width + 2] + w10 * bp[5] + w00 * bp[2];
  return r;
}

__device__ __forceinline__ float mad3(const float* m, float x, float y) {  // row . (x,y,1) without contraction
  return __fadd_rn(__fadd_rn(__fmul_rn(m[0], x), __fmul_rn(m[1], y)), __fmul_rn(m[2], 1.0f));
}

__device__ __forceinline__ void accumulate_g(float* g, float dxI, float dyI, float u, float v, float id, float refc,
                                             float res, float hw, const TrkParams& p) {  // cu:305-346
  const float dx = dxI * p.fx, dy = dyI * p.fy;
  float J[9];
  J[0] = id * dx; J[1] = id * dy; J[2] = -id * (u * dx + v * dy);
  J[3] = -(u * v * dx + dy + dy * v * v); J[4] = u * v * dy + dx + dx * u * u; J[5] = u * dy - v * dx;
  J[6] = p.affa * (p.ref_b - refc); J[7] = -1.f; J[8] = res;
  int k = 0;
#pragma unroll
  for (int j1 = 0; j1 < 9; ++j1) {
    const float jw = J[j1] * hw;
#pragma unroll
    for (int j2 = j1; j2 < 9; ++j2) g[k++] += jw * J[j2];
  }
}

// MODE 0: calcRes (stats + warped buffers)   1: calcG from warped buffers   2: fused (stats + G, no buffers)
// MODE 4: MODE 2 inside the device LM loop: the level's parameters, buffers and pose come from b.lm, the LM step runs in the
//         last CTA.  Same arithmetic as MODE 2; a template of its own so that the plain MODE 2 keeps its registers.
// MODE 3: calcRes statistics of blockIdx.y = 0..n_hyp-1 independent poses in one launch (no buffers): the motion hypotheses
//         DSO tries one after the other (FullSystem.cpp:437-530) evaluated as a batch - SURVEY 8(e)'s only parallel axis of the
//         tracker.  Same per-thread point striding and the same fixed-order reduction as MODE 0 -> identical numbers.
template <int MODE>
__global__ void __launch_bounds__(kThreads)
k_tracker(const __grid_constant__ TrkParams p_in, TrkBufs b) {
  constexpr bool FUSED = MODE == 2 || MODE == 4;
  TrkParams p = p_in;
  const float* Ki = p.Ki;
  if (MODE == 4) {                       // the current level's parameters and buffers, the LM step's candidate pose
    const LmLevel& L = b.lm->in.lv[b.lm->lvl];
    p = L.p;
    Ki = L.p.Ki;                         // read where the flow statistics need it: keeps 9 registers free
    b.pc_u = L.pc_u; b.pc_v = L.pc_v; b.pc_idepth = L.pc_idepth; b.pc_color = L.pc_color; b.dInew = L.dInew;
    const TrkPose* q = &b.lm->pose;
#pragma unroll
    for (int i = 0; i < 9; ++i) p.RKi[i] = q->RKi[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) p.t[i] = q->t[i];
    p.affa = q->affa; p.affb = q->affb; p.cutoff = q->cutoff; p.maxEnergy = q->maxEnergy;
  }
  if (MODE == 3) {
    const TrkPose* q = b.batch + blockIdx.y;
#pragma unroll
    for (int i = 0; i < 9; ++i) p.RKi[i] = q->RKi[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) p.t[i] = q->t[i];
    p.affa = q->affa; p.affb = q->affb; p.cutoff = q->cutoff; p.maxEnergy = q->maxEnergy;
    b.partials += (size_t)blockIdx.y * kBlocks * kOut;
    b.ticket += blockIdx.y;
    b.out += (size_t)blockIdx.y * kOut;
  }
  constexpr int NV = (MODE == 0 || MODE == 3) ? kRes : (MODE == 1 ? kG : kOut);
  constexpr int OFF = MODE == 1 ? kRes : 0;
  float acc[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) acc[k] = 0.f;
  float* st = acc;                               // stats (MODE 0, 2, 4)
  float* g = acc + (FUSED ? kRes : 0);           // 45 products (MODE 1, 2, 4)
  const long long nm = b.n_max;

  for (int i = blockIdx.x * kThreads + threadIdx.x; i < p.n; i += kBlocks * kThreads) {
    if (MODE == 1) {
      const float hw = b.warped[6 * nm + i];
      if (hw != 0.f)
        accumulate_g(g, b.warped[2 * nm + i], b.warped[3 * nm + i], b.warped[i], b.warped[nm + i], b.warped[4 * nm + i],
                     b.pc_color[i], b.warped[5 * nm + i], hw, p);
      continue;
    }
    const float id = b.pc_idepth[i], x = b.pc_u[i], y = b.pc_v[i];
    float pt[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) pt[r] = mad3(p.RKi + 3 * r, x, y);
    float p1[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) p1[r] = __fadd_rn(pt[r], __fmul_rn(p.t[r], id));
    const float u = __fdiv_rn(p1[0], p1[2]), v = __fdiv_rn(p1[1], p1[2]);
    const float Ku = __fadd_rn(__fmul_rn(p.fx, u), p.cx), Kv = __fadd_rn(__fmul_rn(p.fy, v), p.cy);
    const float nid = __fdiv_rn(id, p1[2]);
    if (i % 32 == 0) {  // flow statistics on every 32nd point (cu:119-166)
      float ptK[3], a[3], c[3], d[3];
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        ptK[r] = mad3(Ki + 3 * r, x, y);
        const float tid = __fmul_rn(p.t[r], id);
        a[r] = __fadd_rn(ptK[r], tid); c[r] = __fsub_rn(ptK[r], tid); d[r] = __fsub_rn(pt[r], tid);
      }
      const float KuT = p.fx * (a[0] / a[2]) + p.cx, KvT = p.fy * (a[1] / a[2]) + p.cy;
      const float KuT2 = p.fx * (c[0] / c[2]) + p.cx, KvT2 = p.fy * (c[1] / c[2]) + p.cy;
      const float Ku3 = p.fx * (d[0] / d[2]) + p.cx, Kv3 = p.fy * (d[1] / d[2]) + p.cy;
      st[4] += (KuT - x) * (KuT - x) + (KvT - y) * (KvT - y) + (KuT2 - x) * (KuT2 - x) + (KvT2 - y) * (KvT2 - y);
      st[5] += (Ku - x) * (Ku - x) + (Kv - y) * (Kv - y) + (Ku3 - x) * (Ku3 - x) + (Kv3 - y) * (Kv3 - y);
      st[6] += 2.f;
    }
    float wu = 0, wv = 0, wdx = 0, wdy = 0, wid = 0, wres = 0, whw = 0;
    if (Ku > 2 && Kv > 2 && Ku < p.w - 3 && Kv < p.h - 3 && nid > 0) {
      const float refc = b.pc_color[i];
      const float3 hit = bilinear33(b.dInew, Ku, Kv, p.w);
      if (isfinite(hit.x)) {
        const float res = __fsub_rn(hit.x, __fadd_rn(__fmul_rn(p.affa, refc), p.affb));
        const float ar = fabsf(res);
        const float hw = ar < p.huber ? 1.f : p.huber / ar;
        if (ar > p.cutoff) {
          st[0] += p.maxEnergy; st[1] += 1.f; st[3] += 1.f;
        } else {
          st[0] += hw * res * res * (2.f - hw); st[1] += 1.f; st[2] += 1.f;
          wu = u; wv = v; wdx = hit.y; wdy = hit.z; wid = nid; wres = res; whw = hw;
          if (FUSED) accumulate_g(g, hit.y, hit.z, u, v, nid, refc, res, hw, p);
        }
      }
    }
    if (MODE == 0) {  // un-compacted buffers, zeros at rejected points (cu:75-81,191-197)
      b.warped[i] = wu; b.warped[nm + i] = wv; b.warped[2 * nm + i] = wdx; b.warped[3 * nm + i] = wdy;
      b.warped[4 * nm + i] = wid; b.warped[5 * nm + i] = wres; b.warped[6 * nm + i] = whw;
    }
  }

  // ---- reduction: double, warp shuffle -> shared -> per-CTA partial -> last CTA sums in a fixed order ----
  __shared__ double sm[kThreads / 32][NV];
  __shared__ bool is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    double v = (double)acc[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if (lane == 0) sm[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < NV) {
    double s = 0;
#pragma unroll
    for (int wv = 0; wv < kThreads / 32; ++wv) s += sm[wv][threadIdx.x];
    b.partials[(size_t)blockIdx.x * kOut + OFF + threadIdx.x] = s;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(b.ticket, 1u) == kBlocks - 1);
  __syncthreads();
  if (is_last) {
    __threadfence();
    if (threadIdx.x < NV) {
      double s = 0;
      for (int blk = 0; blk < kBlocks; ++blk) s += __ldcg(&b.partials[(size_t)blk * kOut + OFF + threadIdx.x]);
      b.out[OFF + threadIdx.x] = s;
    }
    if (threadIdx.x == 0) *b.ticket = 0;
    if (MODE == 4) {                             // n3 / n5: the LM step rides on the evaluation's last CTA - no extra launch
      __threadfence();
      __syncthreads();
      if (threadIdx.x == 0) lm_step(b.lm, b.out);
    }
  }
}


// ================================================================================================
// n2 (SURVEY 8f): FrameHessian::makeImages on the device (HessianBlocks.cpp:128-191).  Level 0 takes the grey image,
// level l > 0 the 2x2 mean of level l-1; gradients are central differences over the FLAT index range [w, w*(h-1)) as in
// the reference (so x = 0 / w-1 wrap to the neighbouring rows), non-finite -> 0; rows 0 and h-1 are zero.
// ================================================================================================
__global__ void k_pyr_level(const float* __restrict__ src /*grey w*h (lvl 0) or previous level's float3*/, int src_is_dI,
                            int wprev, float* __restrict__ gray /*scratch wl*hl*/, int wl, int hl) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= wl * hl) return;
  if (!src_is_dI) { gray[i] = src[i]; return; }
  const int y = i / wl, x = i - y * wl;
  const float* q = src + 3 * (size_t)(2 * x + 2 * y * wprev);
  gray[i] = __fmul_rn(0.25f, __fadd_rn(__fadd_rn(__fadd_rn(q[0], q[3]), q[3 * wprev]), q[3 * wprev + 3]));
}
// kGamma (n11): absSquaredGrad of [w, w*(h-1)) times gw * gw, gw = CalibHessian::getBGradOnly(I) (HessianBlocks.h:446-452)
// on the camera's B (256 floats) - makeImages' setting_gammaWeightsPixelSelect branch (HessianBlocks.cpp:184-188).
// (int)(I + 0.5f) is undefined in C for NaN, +-inf and values beyond int; the reference's x86 build converts with cvttss2si,
// which gives INT_MIN there (clamped to 5).  That is reproduced; CUDA's own conversion would give 0 or INT_MAX.
template <bool kGamma>
__global__ void k_pyr_grad(const float* __restrict__ gray, float* __restrict__ dI, float* __restrict__ absgrad, int wl, int hl,
                           const float* __restrict__ B) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= wl * hl) return;
  float dx = 0.f, dy = 0.f;
  const bool inner = i >= wl && i < wl * (hl - 1);
  if (inner) {
    dx = __fmul_rn(0.5f, __fsub_rn(gray[i + 1], gray[i - 1]));
    dy = __fmul_rn(0.5f, __fsub_rn(gray[i + wl], gray[i - wl]));
    if (!isfinite(dx)) dx = 0.f;
    if (!isfinite(dy)) dy = 0.f;
  }
  const float g = gray[i];
  dI[3 * (size_t)i] = g;
  dI[3 * (size_t)i + 1] = dx;
  dI[3 * (size_t)i + 2] = dy;
  float a = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
  if constexpr (kGamma) {
    if (inner) {
      const float v = __fadd_rn(g, 0.5f);
      int c = (v >= -2147483648.f && v < 2147483648.f) ? __float2int_rz(v) : INT_MIN;
      c = c < 5 ? 5 : (c > 250 ? 250 : c);
      const float gw = __fsub_rn(__ldg(B + c + 1), __ldg(B + c));
      a = __fmul_rn(a, __fmul_rn(gw, gw));
    }
  }
  absgrad[i] = a;
}

// ================================================================================================
// n1 (SURVEY 8f): CoarseTracker::setCoarseTrackingRef's dense part on the device (CoarseTracker.cpp:655-732):
// forward-warp the rendered depth into the reference keyframe (nearest depth wins: atomicMin on the bit pattern of
// the positive float), then append the hit pixels behind the sparse points in RASTER order (row counts -> row offsets
// -> ordered intra-row compaction), so the point order - and with it our deterministic reduction - is reproducible.
// ================================================================================================
struct DenseWarp {
  float KRKi[9], Kt[3];
};
__global__ void k_dense_warp(const float* __restrict__ depth, int w, int h, int step, DenseWarp m, unsigned* __restrict__ proj) {
  const int nx = (w + step - 1) / step, ny = (h + step - 1) / step;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nx * ny) return;
  const int y = (i / nx) * step, x = (i - (i / nx) * nx) * step;
  const float z = depth[x + (size_t)y * w];
  if (!(z > 0.f)) return;
  const float ox = __fmul_rn((float)x, z), oy = __fmul_rn((float)y, z);
  float p[3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
    p[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m.KRKi[3 * r], ox), __fmul_rn(m.KRKi[3 * r + 1], oy)), __fmul_rn(m.KRKi[3 * r + 2], z)), m.Kt[r]);
  if (!(p[2] > 0.f)) return;
  const int pu = (int)__fadd_rn(__fdiv_rn(p[0], p[2]), 0.5f), pv = (int)__fadd_rn(__fdiv_rn(p[1], p[2]), 0.5f);
  if (pu > w - 4 || pv > h - 4 || pu < 3 || pv < 3) return;
  atomicMin(proj + pu + (size_t)pv * w, __float_as_uint(p[2]));
}
// The raster-order compaction (row counts -> row offsets -> ordered intra-row emit) is shared with n7's normalise-and-compact
// pass: a selector classifies each pixel of [2, w-2) x [2, h-2) as 0 (skip), 1 (append) or 2 (a candidate the reference writes
// to slot pc_n and then rejects, n7 only) and writes the point of an appended pixel.
struct DenseSel {             // n1: the hit pixels of the warp that the sparse image leaves free
  static constexpr bool kStale = false;
  const unsigned* proj;
  const float* idepth0;
  int dense_only;
  const float* gray;
  int gstride;
  __device__ __forceinline__ int cls(int i) const {
    return proj[i] != 0xFFFFFFFFu && (dense_only || !idepth0 || idepth0[i] <= 0.f) ? 1 : 0;
  }
  __device__ __forceinline__ void emit(int o, int x, int y, int i, float* pc_u, float* pc_v, float* pc_idepth, float* pc_color) const {
    pc_u[o] = (float)x;
    pc_v[o] = (float)y;
    pc_idepth[o] = __fdiv_rn(1.f, __uint_as_float(proj[i]));
    pc_color[o] = gray[(size_t)i * gstride];
  }
  __device__ __forceinline__ void finish(int, int) const {}
};
struct NormSel {              // n7: CoarseTracker.cpp:346-370 on one level (idepth normalised in place, rejected -> -1)
  static constexpr bool kStale = true;
  float* idepth;
  const float* wsum;
  const float* gray;          // the level's (I, dx, dy) image
  __device__ __forceinline__ int cls(int i) const {
    if (!(wsum[i] > 0.f)) return 0;
    const float d = __fdiv_rn(idepth[i], wsum[i]);
    return isfinite(gray[3 * (size_t)i]) && d > 0.f ? 1 : 2;
  }
  __device__ __forceinline__ void emit(int o, int x, int y, int i, float* pc_u, float* pc_v, float* pc_idepth, float* pc_color) const {
    pc_u[o] = (float)x;
    pc_v[o] = (float)y;
    pc_idepth[o] = __fdiv_rn(idepth[i], wsum[i]);
    pc_color[o] = gray[3 * (size_t)i];
  }
  __device__ __forceinline__ void finish(int i, int c) const {   // after every read of pixel i (only its own thread reads it)
    idepth[i] = c == 1 ? __fdiv_rn(idepth[i], wsum[i]) : -1.f;
  }
};
struct NodiaSel {             // the undilated level-0 cloud, CoarseTracker.cpp:186-218 (pc_*_nodia)
  static constexpr bool kStale = true;
  const float* idepth_nodia;  // unweighted idepth sums
  const float* wsum;          // level 0's weights before the dilation
  const float* gray;          // level 0's (I, dx, dy) image
  __device__ __forceinline__ int cls(int i) const {
    if (!(wsum[i] > 0.f)) return 0;
    return isfinite(gray[3 * (size_t)i]) && idepth_nodia[i] > 0.f ? 1 : 2;
  }
  __device__ __forceinline__ void emit(int o, int x, int y, int i, float* pc_u, float* pc_v, float* pc_idepth, float* pc_color) const {
    pc_u[o] = (float)x;
    pc_v[o] = (float)y;
    pc_idepth[o] = idepth_nodia[i];
    pc_color[o] = gray[3 * (size_t)i];
  }
  __device__ __forceinline__ void finish(int, int) const {}   // the -1 the reference writes back only marks the nodia image
};
// rowlast[y] = (last x of class 1, last x of class 2) in row y, -1 for none; only for selectors with kStale
template <class Sel>
__global__ void __launch_bounds__(256) k_compact_rowcount(Sel s, int w, int h, int* __restrict__ rowcnt, int2* __restrict__ rowlast) {
  const int y = blockIdx.x;
  int c = 0, la = 0, lr = 0;   // last x + 1
  if (y >= 2 && y < h - 2)
    for (int x = 2 + threadIdx.x; x < w - 2; x += 256) {
      const int k = s.cls(x + y * w);
      c += k == 1 ? 1 : 0;
      if (Sel::kStale) {
        if (k == 1) la = x + 1;
        if (k == 2) lr = x + 1;
      }
    }
  __shared__ int sm[3][8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
  if (Sel::kStale) {
    la = __reduce_max_sync(0xffffffffu, (unsigned)la);
    lr = __reduce_max_sync(0xffffffffu, (unsigned)lr);
  }
  if ((threadIdx.x & 31) == 0) { sm[0][threadIdx.x >> 5] = c; sm[1][threadIdx.x >> 5] = la; sm[2][threadIdx.x >> 5] = lr; }
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0, a = 0, r = 0;
    for (int k = 0; k < 8; ++k) { t += sm[0][k]; a = max(a, sm[1][k]); r = max(r, sm[2][k]); }
    rowcnt[y] = t;
    if (Sel::kStale) rowlast[y] = make_int2(a - 1, r - 1);
  }
}
// rowoff[y] = (*start, or 0) + the counts of the rows above; *total_out = the count of all rows.  With rowlast: *stale_out = the
// raster index of the last class-2 pixel behind the last class-1 pixel (the candidate left in slot pc_n), -1 for none.
__global__ void k_compact_rowscan(const int* __restrict__ rowcnt, const int2* __restrict__ rowlast, int w, int h,
                                  const int* __restrict__ start, int* __restrict__ rowoff, int* __restrict__ total_out,
                                  int* __restrict__ stale_out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const int s0 = start ? *start : 0;
  int s = s0, la = -1, lr = -1;
  for (int y = 0; y < h; ++y) {
    rowoff[y] = s;
    s += rowcnt[y];
    if (rowlast && y >= 2 && y < h - 2) {
      if (rowlast[y].x >= 0) la = rowlast[y].x + y * w;
      if (rowlast[y].y >= 0) lr = rowlast[y].y + y * w;
    }
  }
  *total_out = s - s0;
  if (stale_out) *stale_out = lr > la ? lr : -1;
}
// Points go to slots first + rowoff[y] + (rank in the row), those at or beyond cap are dropped (the caller checks the count
// against its capacity afterwards).  With kStale the class-2 pixel *stale goes to slot *total.
template <class Sel>
__global__ void __launch_bounds__(256) k_compact_emit(Sel s, int w, int h, const int* __restrict__ rowoff, int first, int cap,
                                                       const int* __restrict__ stale, const int* __restrict__ total,
                                                       float* __restrict__ pc_u, float* __restrict__ pc_v,
                                                       float* __restrict__ pc_idepth, float* __restrict__ pc_color) {
  const int y = blockIdx.x;
  if (y < 2 || y >= h - 2) return;
  __shared__ int wsum[8];
  __shared__ int base;
  if (threadIdx.x == 0) base = first + rowoff[y];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int x0 = 2; x0 < w - 2; x0 += 256) {
    const int x = x0 + threadIdx.x;
    const int i = x + y * w;
    const int c = x < w - 2 ? s.cls(i) : 0;
    const bool take = c == 1;
    const unsigned bal = __ballot_sync(0xffffffffu, take);
    if (lane == 0) wsum[warp] = __popc(bal);
    __syncthreads();
    int before = 0, all = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) { before += k < warp ? wsum[k] : 0; all += wsum[k]; }
    if (take) {
      const int o = base + before + __popc(bal & ((1u << lane) - 1u));
      if (o < cap) s.emit(o, x, y, i, pc_u, pc_v, pc_idepth, pc_color);
    }
    if (Sel::kStale && c == 2 && i == *stale && *total < cap) s.emit(*total, x, y, i, pc_u, pc_v, pc_idepth, pc_color);
    if (Sel::kStale && x < w - 2) s.finish(i, c);
    __syncthreads();
    if (threadIdx.x == 0) base += all;
    __syncthreads();
  }
}

// ================================================================================================
// n7 (SURVEY 8f): CoarseTracker::makeCoarseDepthL0 (CoarseTracker.cpp:148-374) on the device, every level, then n1's dense
// append on level 0 (setCoarseTrackingRef, :633-733).  Every float operation is the reference's, correctly rounded.
// ================================================================================================
// Scatter (:155-182): the points arrive sorted by (pixel, input index) - a stable radix sort of the pixel keys - and each
// pixel's run is summed sequentially in input order, so the sums do not depend on scheduling.  a = centerProjectedTo[2] or
// ph->idepth, b = HdiF (monocular) or idepth_hessian (RGB-D).  kNodia also sums a unweighted into idepth_nodia (:167,
// monocular only; in RGB-D mode it keeps the zeros it was cleared to).
template <bool kNodia>
__global__ void k_coarse_scatter(const int* __restrict__ pix, const int* __restrict__ order, const float* __restrict__ a,
                                 const float* __restrict__ b, int n, int rgbd, float* __restrict__ idepth, float* __restrict__ wsum,
                                 float* __restrict__ idepth_nodia) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n || (k > 0 && pix[k - 1] == pix[k])) return;
  const int p = pix[k];
  float s = 0.f, ws = 0.f, sn = 0.f;
  for (int j = k; j < n && pix[j] == p; ++j) {
    const int q = order[j];
    // sqrtf(1e-3 / (HdiF + 1e-12)): double literals, so the quotient is a double narrowed to float for sqrtf
    const float wt = rgbd ? b[q] : __fsqrt_rn(__double2float_rn(__ddiv_rn(1e-3, __dadd_rn((double)b[q], 1e-12))));
    s = __fadd_rn(s, __fmul_rn(a[q], wt));
    ws = __fadd_rn(ws, wt);
    if (kNodia) sn = __fadd_rn(sn, a[q]);
  }
  idepth[p] = s;
  wsum[p] = ws;
  if (kNodia && !rgbd) idepth_nodia[p] = sn;
}
// get_idepth_quantile (tandem_backend.cpp:354-361) on the first *count keys: keys[k] = pc_idepth_nodia[k] below the count, +inf
// from there to n (the slot at *count, a rejected candidate, is not a key).  Accepted values are > 0, so +inf sorts behind them.
__global__ void k_nodia_keys(const float* __restrict__ pc_idepth, const int* __restrict__ count, int n, float* __restrict__ keys) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) keys[k] = k < *count ? pc_idepth[k] : __int_as_float(0x7f800000);
}
// out[0] = the idepth at index (int)(fraction * (float)count) of the sorted keys, out[1] = 1.0f / it, both as float bits; NaN
// when the index is not below the count (no keys at all, or fraction 1), where the reference reads outside its vector.
__global__ void k_nodia_quantile(const float* __restrict__ sorted, const int* __restrict__ count, float fraction, int* __restrict__ out) {
  const int m = *count;
  const int k = __float2int_rz(__fmul_rn(fraction, __int2float_rn(m)));
  float v = __int_as_float(0x7fc00000), d = v;
  if (m > 0 && k < m) {
    v = sorted[k];
    d = __fdiv_rn(1.f, v);
  }
  out[0] = __float_as_int(v);
  out[1] = __float_as_int(d);
}
// Sum pyramid (:222-243): level l from the un-dilated level l-1, a + b + c + d left to right.
__global__ void k_coarse_sum(const float* __restrict__ id_lm, const float* __restrict__ ws_lm, int wlm1, float* __restrict__ id_l,
                             float* __restrict__ ws_l, int wl, int hl) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= wl * hl) return;
  const int y = i / wl, x = i - y * wl, b = 2 * x + 2 * y * wlm1;
  id_l[i] = __fadd_rn(__fadd_rn(__fadd_rn(id_lm[b], id_lm[b + 1]), id_lm[b + wlm1]), id_lm[b + wlm1 + 1]);
  ws_l[i] = __fadd_rn(__fadd_rn(__fadd_rn(ws_lm[b], ws_lm[b + 1]), ws_lm[b + wlm1]), ws_lm[b + wlm1 + 1]);
}
// Dilation (:246-322) over the flat range [w, w*h - w): a pixel without weight takes the mean of its weighted neighbours - the
// 4 diagonal ones on levels 0 and 1, the 4 axis ones above - read from the pre-dilation weights wbak (so column 0 and w-1 see
// the neighbouring rows).  idepth is updated in place (only pixels with wbak <= 0 are written, only pixels with wbak > 0 are
// read), the weights go to wout.  On levels 0 / 1 the first and the last pixel of the range have one diagonal neighbour outside
// the image (index -1 and w*h, the padding of the reference's allocation): it counts as unweighted.
template <bool kDiag>
__global__ void k_coarse_dilate(float* __restrict__ idepth, const float* __restrict__ wbak, float* __restrict__ wout, int w, int h) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = w * h;
  if (i >= n) return;
  float wi = wbak[i];
  if (i >= w && i < n - w && wi <= 0.f) {
    const int nb[4] = {kDiag ? i + 1 + w : i + 1, kDiag ? i - 1 - w : i - 1, kDiag ? i + w - 1 : i + w, kDiag ? i - w + 1 : i - w};
    float sum = 0.f, num = 0.f, numn = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int j = nb[k];
      if (j < 0 || j >= n) continue;
      const float wj = wbak[j];
      if (wj > 0.f) {
        sum = __fadd_rn(sum, idepth[j]);
        num = __fadd_rn(num, wj);
        numn = __fadd_rn(numn, 1.f);
      }
    }
    if (numn > 0.f) {
      idepth[i] = __fdiv_rn(sum, numn);
      wi = __fdiv_rn(num, numn);
    }
  }
  wout[i] = wi;
}

// ================================================================================================
// n3 (SURVEY 8f): the level's Levenberg-Marquardt loop of CoarseTracker::trackNewestCoarse (CoarseTracker.cpp:761-916)
// and n5: the coarse-to-fine loop around it (CoarseTracker.cpp:750-936), with ONE host wait per call.  A CUDA graph
// runs k_lm_init and then a conditional WHILE node around k_tracker<4>; the evaluation's last CTA runs lm_step (one
// thread, double), which turns the 52 sums into the accept/reject decision, the damped 8x8 solve, the SE3 update and the
// next candidate's TrkPose, moves on to the next level (or repeats one) and ends the WHILE loop when the call is done.
// Every level runs through the same kernel: it reads its parameters and buffers from LmCtx::in.lv[lvl].
// ================================================================================================
__device__ void lm_pose_from(const LmConfig& c, const double* T, const double* aff, float cutoff, TrkPose* o) {
  float R[9];
  for (int r = 0; r < 3; ++r) {
    for (int k = 0; k < 3; ++k) R[3 * r + k] = (float)T[4 * r + k];
    o->t[r] = (float)T[4 * r + 3];
  }
  for (int r = 0; r < 3; ++r)
    for (int q = 0; q < 3; ++q) {
      float s = 0.f;
      for (int k = 0; k < 3; ++k) s = __fadd_rn(s, __fmul_rn(R[3 * r + k], c.Ki[3 * k + q]));
      o->RKi[3 * r + q] = s;
    }
  float eF = c.ref_exposure, eT = c.new_exposure;       // AffLight::fromToVecExposure, cuda_coarse_tracker.cpp:42-52
  if (eF == 0 || eT == 0) eT = eF = 1;
  // rounded operations, no FMA contraction: the same bits as the host's prepare() computes for calcRes / calcResAndG
  const double a = exp(aff[0] - c.ref_aff[0]) * eT / eF;
  const double bb = __dsub_rn(aff[1], __dmul_rn(a, c.ref_aff[1]));
  o->affa = (float)a; o->affb = (float)bb;
  o->cutoff = cutoff;
  o->maxEnergy = __fsub_rn(__fmul_rn(__fmul_rn(2.f, c.huber), cutoff), __fmul_rn(c.huber, c.huber));
}

__device__ void lm_se3_exp(const double* xi, double* T) {   // Sophus convention (upsilon, omega)
  const double wx = xi[3], wy = xi[4], wz = xi[5];
  const double th2 = wx * wx + wy * wy + wz * wz, th = sqrt(th2);
  double A, B, C;
  if (th < 1e-8) { A = 1.0 - th2 / 6; B = 0.5 - th2 / 24; C = 1.0 / 6 - th2 / 120; }
  else { A = sin(th) / th; B = (1 - cos(th)) / th2; C = (th - sin(th)) / (th2 * th); }
  const double O[9] = {0, -wz, wy, wz, 0, -wx, -wy, wx, 0};
  double O2[9];
  for (int r = 0; r < 3; ++r)
    for (int q = 0; q < 3; ++q) { double s = 0; for (int k = 0; k < 3; ++k) s += O[3 * r + k] * O[3 * k + q]; O2[3 * r + q] = s; }
  for (int i = 0; i < 16; ++i) T[i] = (i % 5 == 0) ? 1.0 : 0.0;
  for (int r = 0; r < 3; ++r) {
    double tv = 0;
    for (int q = 0; q < 3; ++q) {
      const double id = r == q ? 1.0 : 0.0;
      T[4 * r + q] = id + A * O[3 * r + q] + B * O2[3 * r + q];
      tv += (id + B * O[3 * r + q] + C * O2[3 * r + q]) * xi[q];
    }
    T[4 * r + 3] = tv;
  }
}

__device__ void lm_next_candidate(const LmConfig& c, LmState* s, TrkPose* pose) {
  int idx[8], nf = 0;
  for (int i = 0; i < 8; ++i)
    if (!((i == 6 && c.fix_a) || (i == 7 && c.fix_b))) idx[nf++] = i;
  double M[8][9];
  for (int r = 0; r < nf; ++r) {
    for (int q = 0; q < nf; ++q) M[r][q] = s->H[8 * idx[r] + idx[q]] * (r == q ? (double)(1.f + s->lambda) : 1.0);
    M[r][nf] = -s->b[idx[r]];
  }
  // Gaussian elimination, partial pivoting.  A column without a non-zero pivot (a parameter no point constrains: its row
  // and column of the damped H are 0) gets increment 0, as Eigen's LDLT (CoarseTracker.cpp:815) treats a zero pivot.
  for (int k = 0; k < nf; ++k) {
    int piv = k;
    for (int r = k + 1; r < nf; ++r) if (fabs(M[r][k]) > fabs(M[piv][k])) piv = r;
    if (piv != k) for (int q = 0; q <= nf; ++q) { const double t = M[k][q]; M[k][q] = M[piv][q]; M[piv][q] = t; }
    const double d = M[k][k];
    if (d == 0) continue;
    for (int r = k + 1; r < nf; ++r) {
      const double f = M[r][k] / d;
      for (int q = k; q <= nf; ++q) M[r][q] -= f * M[k][q];
    }
  }
  double inc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int k = nf - 1; k >= 0; --k) {
    double v = M[k][nf];
    for (int q = k + 1; q < nf; ++q) v -= M[k][q] * inc[idx[q]];
    inc[idx[k]] = M[k][k] == 0 ? 0.0 : v / M[k][k];
  }
  float extrap = 1.f;
  if (s->lambda < c.lambda_limit) extrap = sqrtf(sqrtf(c.lambda_limit / s->lambda));
  double n2 = 0, sum = 0;
  const double scale[8] = {1.0, 1.0, 1.0, 0.5, 0.5, 0.5, 10.0, 1000.0};
  double sc[8];
  for (int i = 0; i < 8; ++i) { inc[i] *= extrap; n2 += inc[i] * inc[i]; sc[i] = inc[i] * scale[i]; sum += sc[i]; }
  s->inc_norm = sqrt(n2);
  if (!isfinite(sum)) for (int i = 0; i < 8; ++i) sc[i] = 0;
  double E[16];
  lm_se3_exp(sc, E);
  for (int r = 0; r < 4; ++r)
    for (int q = 0; q < 4; ++q) { double v = 0; for (int k = 0; k < 4; ++k) v += E[4 * r + k] * s->T[4 * k + q]; s->Tn[4 * r + q] = v; }
  s->affn[0] = s->aff[0] + sc[6];
  s->affn[1] = s->aff[1] + sc[7];
  lm_pose_from(c, s->Tn, s->affn, c.coarse_cutoff * s->repeat, pose);
}

__device__ void lm_take_g(const double* o, int num_warped, LmState* s) {   // finish_g, cuda_coarse_tracker.cpp:335-355
  const double factor = 1.0 / num_warped;
  const double scale[8] = {1.0, 1.0, 1.0, 0.5, 0.5, 0.5, 10.0, 1000.0};
  for (int r = 0; r < 8; ++r) {
    for (int q = 0; q < 8; ++q) {
      const int lo = r < q ? r : q, hi = r < q ? q : r;
      s->H[8 * r + q] = o[kRes + lo * 9 + hi - lo * (lo + 1) / 2] * factor * scale[r] * scale[q];
    }
    s->b[r] = o[kRes + r * 9 + 8 - r * (r + 1) / 2] * factor * scale[r];
  }
}

__device__ void lm_begin_level(LmCtx* c, int lvl) {   // CoarseTracker.cpp:764,798: levelCutoffRepeat = 1, lambda = 0.01
  LmState* s = &c->s;
  const LmConfig& cfg = c->in.lv[lvl].cfg;
  c->lvl = lvl;
  for (int i = 0; i < 16; ++i) s->Tn[i] = s->T[i];
  s->affn[0] = s->aff[0]; s->affn[1] = s->aff[1];
  s->lambda = 0.01f; s->inc_norm = 0; s->repeat = 1.f; s->phase = 0; s->iter = 0; s->evals = 0;
  lm_pose_from(cfg, s->T, s->aff, cfg.coarse_cutoff, &c->pose);
}

// the per-call state of trackNewestCoarse (:746-747), starting from T0 and in.aff0 on the coarsest level
__device__ void lm_start(LmCtx* c, const double* T0) {
  LmState* s = &c->s;
  for (int i = 0; i < 16; ++i) s->T[i] = T0[i];
  s->aff[0] = c->in.aff0[0]; s->aff[1] = c->in.aff0[1];
  LmResult* r = &c->r;
  for (int l = 0; l < kMaxLevels; ++l) {
    for (int i = 0; i < 6; ++i) r->res[l][i] = 0;
    r->last_res[l] = __longlong_as_double(0x7ff8000000000000ll);   // lastResiduals.setConstant(NAN)  (:746)
    r->iterations[l] = 0; r->evaluations[l] = 0; r->repeat[l] = 1.f;
  }
  for (int i = 0; i < 3; ++i) r->flow[i] = 1000;                    // lastFlowIndicators.setConstant(1000)  (:747)
  r->num_warped = 0; r->ok = 0; r->aborted_level = -1; r->repeated_level = -1; r->done = 0;
  c->have_repeated = 0;
  lm_begin_level(c, c->in.coarsest);
}

__global__ void k_lm_init(LmCtx* c, LmResult* out, cudaGraphConditionalHandle loop) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  c->out = out;
  c->loop = loop;
  c->total_evals = 0;
  if (c->in.pyramid == 2) {                           // FullSystem.cpp:549-551: achievedRes = NaN, no winner yet
    RetrackState* q = &c->rs;
    for (int l = 0; l < kMaxLevels; ++l) q->achieved[l] = __longlong_as_double(0x7ff8000000000000ll);
    q->have_one_good = 0; q->cur = 0; q->winner = -1;
  }
  lm_start(c, c->in.T0);
}

__device__ void rt_publish(LmCtx* ctx, int done);
__device__ void rt_end_try(LmCtx* ctx, int ok);

// Publishes the result and ends the WHILE loop.  `pose_out` = the loop reached the end (lastToNew_out / aff_g2l_out are
// written, :919-920); otherwise the input pose is returned.
__device__ void lm_finish(LmCtx* ctx, int ok, bool pose_out, int done) {
  if (ctx->in.pyramid == 2) { rt_publish(ctx, done); return; }   // n6 reaches this only past the evaluation bound
  LmResult* r = &ctx->r;
  const LmState* s = &ctx->s;
  for (int i = 0; i < 16; ++i) r->T[i] = pose_out ? s->T[i] : ctx->in.T0[i];
  r->aff[0] = pose_out ? s->aff[0] : ctx->in.aff0[0];
  r->aff[1] = pose_out ? s->aff[1] : ctx->in.aff0[1];
  r->ok = ok;
  LmResult* out = ctx->out;
  const int* src = reinterpret_cast<const int*>(r);
  int* dst = reinterpret_cast<int*>(out);
  for (int i = 0; i < (int)(offsetof(LmResult, done) / sizeof(int)); ++i) dst[i] = src[i];
  __threadfence_system();
  out->done = done;                                  // written last: the host checks it after its one wait
  __threadfence_system();
  cudaGraphSetConditional(ctx->loop, 0);
}

// :918-935, after the level loop: the affine sanity checks with the float modes, then fixed parameters reported as 0
__device__ void lm_finish_pyramid(LmCtx* ctx) {
  LmState* s = &ctx->s;
  const float ma = ctx->in.mode_a, mb = ctx->in.mode_b;
  const double a = s->aff[0], b = s->aff[1];
  bool ok = !((ma != 0 && fabsf((float)a) > 1.2) || (mb != 0 && fabsf((float)b) > 200));
  if (ok) {
    const LmConfig& c0 = ctx->in.lv[0].cfg;        // AffLight::fromToVecExposure(lastRef, newFrame, ...).cast<float>()
    float eF = c0.ref_exposure, eT = c0.new_exposure;
    if (eF == 0 || eT == 0) eT = eF = 1;
    const double ra = exp(a - c0.ref_aff[0]) * eT / eF;
    const double rb = __dsub_rn(b, __dmul_rn(ra, c0.ref_aff[1]));   // no FMA contraction, as on the host
    const float rel0 = (float)ra, rel1 = (float)rb;
    ok = !((ma == 0 && fabsf(logf(rel0)) > 1.5) || (mb == 0 && fabsf(rel1) > 200));
  }
  if (ok) {
    if (ma < 0) s->aff[0] = 0;
    if (mb < 0) s->aff[1] = 0;
  }
  if (ctx->in.pyramid == 2) { rt_end_try(ctx, ok ? 1 : 0); return; }
  lm_finish(ctx, ok ? 1 : 0, true, 1);
}

// ================================================================================================
// n6: FullSystem::trackNewCoarse's loop over the motion hypotheses (FullSystem.cpp:538-617, rgbd_flag == false) on the same
// graph.  In mode 2 the points where n5 ends the call end a try instead: the try's outcome is recorded, the winner test, the
// achievedRes takeover and the break test run statement for statement, and either the next try starts on the coarsest level
// (without a launch: the WHILE loop simply goes on) or the result is published and the loop ends.
// ================================================================================================
__device__ void rt_publish(LmCtx* ctx, int done) {
  const RetrackState* q = &ctx->rs;
  RetrackOut* o = ctx->rin.out;
  const bool good = q->have_one_good != 0;            // :610-615: no winner -> tries[0], aff_last_2_l, flow 0
  for (int i = 0; i < 16; ++i) o->T[i] = good ? q->T[i] : ctx->rin.tries[0][i];
  for (int i = 0; i < 2; ++i) o->aff[i] = good ? q->aff[i] : ctx->in.aff0[i];
  for (int i = 0; i < 3; ++i) o->flow[i] = good ? q->flow[i] : 0.0;
  for (int l = 0; l < kMaxLevels; ++l) o->achieved[l] = q->achieved[l];
  o->have_one_good = q->have_one_good; o->tries = q->cur; o->winner = q->winner;
  __threadfence_system();
  o->done = done;                                     // written last: the host checks it after its one wait
  __threadfence_system();
  cudaGraphSetConditional(ctx->loop, 0);
}

__device__ void rt_end_try(LmCtx* ctx, int ok) {
  RetrackState* q = &ctx->rs;
  const LmResult* r = &ctx->r;
  const double* lr = r->last_res;
  const int i = q->cur;
  TryRec* rec = &ctx->rin.out->rec[i];
  for (int l = 0; l < kMaxLevels; ++l) { rec->last_res[l] = lr[l]; rec->evaluations[l] = r->evaluations[l]; }
  rec->ok = ok; rec->aborted_level = r->aborted_level; rec->repeated_level = r->repeated_level;
  if (ok && isfinite((float)lr[0]) && !(lr[0] >= q->achieved[0])) {   // :586-592 a new winner (ok: the pose was written)
    for (int k = 0; k < 16; ++k) q->T[k] = ctx->s.T[k];
    q->aff[0] = ctx->s.aff[0]; q->aff[1] = ctx->s.aff[1];
    for (int k = 0; k < 3; ++k) q->flow[k] = r->flow[k];
    q->have_one_good = 1;
    q->winner = i;
  }
  if (q->have_one_good)                               // :595-602 take over achievedRes (always; NaN where never reached)
    for (int l = 0; l < kMaxLevels; ++l)
      if (!isfinite((float)q->achieved[l]) || q->achieved[l] > lr[l]) q->achieved[l] = lr[l];
  q->cur = i + 1;
  if ((q->have_one_good && q->achieved[0] < ctx->rin.last_rmse0 * (double)ctx->rin.threshold) || q->cur == ctx->rin.n_tries) {
    rt_publish(ctx, 1);                               // :605 break, or the last try
    return;
  }
  for (int l = 0; l < kMaxLevels; ++l) ctx->in.min_res[l] = q->achieved[l];   // :553-559 the next try
  lm_start(ctx, ctx->rin.tries[q->cur]);
}

__device__ __noinline__ void lm_step(LmCtx* ctx, const double* o /*kOut sums of the evaluation just finished*/) {
  const int lvl = ctx->lvl;
  const LmConfig& c = ctx->in.lv[lvl].cfg;
  LmState* s = &ctx->s;
  TrkPose* pose = &ctx->pose;
  double res[6] = {o[0], o[1], o[4] / o[6], 0.0, o[5] / o[6], o[3] / o[1]};   // finish_res, cuda_coarse_tracker.cpp:264-272
  const int num_warped = (int)o[2];
  s->evals++;
  if (++ctx->total_evals > ctx->in.max_evals) { lm_finish(ctx, 0, false, 2); return; }
  bool finished = false;
  if (s->phase == 0) {
    if (res[5] > 0.6 && s->repeat < 50.f) {              // CoarseTracker.cpp:779-790: too many saturated residuals
      s->repeat *= 2.f;
      lm_pose_from(c, s->T, s->aff, c.coarse_cutoff * s->repeat, pose);
      return;
    }
    for (int i = 0; i < 6; ++i) s->res_old[i] = res[i];
    lm_take_g(o, num_warped, s);
    s->phase = 1;
    if (c.max_iter <= 0) finished = true;
  } else {
    const bool accept = (res[0] / res[1]) < (s->res_old[0] / s->res_old[1]);
    if (accept) {
      lm_take_g(o, num_warped, s);
      for (int i = 0; i < 6; ++i) s->res_old[i] = res[i];
      for (int i = 0; i < 16; ++i) s->T[i] = s->Tn[i];
      s->aff[0] = s->affn[0]; s->aff[1] = s->affn[1];
      s->lambda *= 0.5f;
    } else {
      s->lambda *= 4.f;
      if (s->lambda < c.lambda_limit) s->lambda = c.lambda_limit;
    }
    s->iter++;
    if (!(s->inc_norm > 1e-3) || s->iter >= c.max_iter) finished = true;
  }
  if (!finished) {
    lm_next_candidate(c, s, pose);
    return;
  }
  LmResult* r = &ctx->r;
  for (int i = 0; i < 6; ++i) r->res[lvl][i] = s->res_old[i];
  r->iterations[lvl] += s->iter; r->evaluations[lvl] += s->evals; r->num_warped = num_warped;
  r->repeat[lvl] = fmaxf(r->repeat[lvl], s->repeat);
  if (!ctx->in.pyramid) { lm_finish(ctx, 1, true, 1); return; }
  // :906-915 - lastResiduals / lastFlowIndicators, the abort test, the one-time repeat of a level whose cutoff was raised
  const float last_res = sqrtf((float)(s->res_old[0] / s->res_old[1]));
  r->last_res[lvl] = last_res;
  for (int i = 0; i < 3; ++i) r->flow[i] = s->res_old[2 + i];
  if (last_res > 1.5 * ctx->in.min_res[lvl]) {      // NaN never aborts
    r->aborted_level = lvl;
    if (ctx->in.pyramid == 2) { rt_end_try(ctx, 0); return; }
    lm_finish(ctx, 0, false, 1);
    return;
  }
  if (s->repeat > 1 && !ctx->have_repeated) {
    ctx->have_repeated = 1;
    r->repeated_level = lvl;
    lm_begin_level(ctx, lvl);
    return;
  }
  if (lvl > 0) { lm_begin_level(ctx, lvl - 1); return; }
  lm_finish_pyramid(ctx);
}

}  // namespace

// ================================================================================================
class TrackerImpl final : public TrackerIface {
 public:
  TrackerImpl(int w, int h, float huber, float cutoff, int n_max, int device)
      : w_(w), h_(h), huber_(huber), coarse_cutoff_(cutoff), device_(device) {
    int nd = 0;
    if (cudaGetDeviceCount(&nd) != cudaSuccess || nd == 0)
      throw Error("tandem_b200: no CUDA device visible - this library has no CPU fallback");
    if (w * h == 0) throw Error("CudaCoarseTracker::init has w*h==0 (cuda_coarse_tracker.cpp:105)");
    n_max_ = n_max > 0 ? n_max : w * h;
    TDM_CUDA(cudaSetDevice(device_));
    int lo, hi;
    TDM_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    stream_ = make_stream(hi);  // highest priority (cpp:72-74)
    d_pc_ = make_dev<float>((size_t)4 * n_max_ * 4);
    TDM_CUDA(cudaMemset(d_pc_.get(), 0, (size_t)4 * n_max_ * 4));   // like the reference's arrays, they persist across references
    d_warped_ = make_dev<float>((size_t)7 * n_max_ * 4);
    TDM_CUDA(cudaMemset(d_warped_.get(), 0, (size_t)7 * n_max_ * 4));
    d_dI_ = make_dev<float>((size_t)3 * w * h * 4);
    d_partials_ = make_dev<double>((size_t)kBlocks * kOut * 8);
    d_ticket_ = make_dev<unsigned>(4);
    TDM_CUDA(cudaMemset(d_ticket_.get(), 0, 4));
    h_pc_ = make_host<float>((size_t)4 * n_max_ * 4);
    h_dI_ = make_host<float>((size_t)3 * w * h * 4);
    h_out_ = make_host<double>(kOut * 8, cudaHostAllocMapped);
    TDM_CUDA(cudaHostGetDevicePointer(&d_out_, h_out_.get(), 0));
  }
  ~TrackerImpl() override {
    cudaSetDevice(device_);
    cudaStreamSynchronize(stream_.get());
  }

  void set_k(int w, int h, float fx, float fy, float cx, float cy) override {
    if (w != w_ || h != h_) throw Error("CudaCoarseTracker::setK wrong h,w. (cuda_coarse_tracker.cpp:359)");
    fx_ = fx; fy_ = fy; cx_ = cx; cy_ = cy;
    // Ki = K^-1 in double, used as float (cpp:365-371, :201-204)
    const double Ki[9] = {1.0 / fx, 0, -(double)cx / fx, 0, 1.0 / fy, -(double)cy / fy, 0, 0, 1};
    for (int i = 0; i < 9; ++i) Ki_[i] = (float)Ki[i];
    have_k_ = true;
  }

  void set_reference(int n, const float* u, const float* v, const float* idepth, const float* color, float ref_exposure,
                     const double ref_aff[2]) override {
    if (n > n_max_) throw Error("Called CudaCoarseTracker::setReference with n > n_max points. (cuda_coarse_tracker.cpp:82)");
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));  // pinned staging may still be in flight
    n_ = n;
    const size_t nm = (size_t)n_max_;
    std::memcpy(h_pc_.get(), u, 4 * (size_t)n);
    std::memcpy(h_pc_.get() + nm, v, 4 * (size_t)n);
    std::memcpy(h_pc_.get() + 2 * nm, idepth, 4 * (size_t)n);
    std::memcpy(h_pc_.get() + 3 * nm, color, 4 * (size_t)n);
    for (int a = 0; a < 4; ++a)
      TDM_CUDA(cudaMemcpyAsync(d_pc_.get() + a * nm, h_pc_.get() + a * nm, 4 * (size_t)n, cudaMemcpyHostToDevice, stream_.get()));
    ref_exposure_ = ref_exposure;
    ref_aff_[0] = ref_aff[0]; ref_aff_[1] = ref_aff[1];
    have_ref_ = true;
    have_params_ = false;   // a calcG now needs a calcRes against the new reference first
  }

  void set_new(const float* dI) override {
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    std::memcpy(h_dI_.get(), dI, (size_t)3 * w_ * h_ * 4);
    TDM_CUDA(cudaMemcpyAsync(d_dI_.get(), h_dI_.get(), (size_t)3 * w_ * h_ * 4, cudaMemcpyHostToDevice, stream_.get()));
    have_new_ = true;
    have_params_ = false;   // calcG is only defined on the buffers of a calcRes against THIS image (cuda_coarse_tracker.cpp:277-281)
  }

  void calc_res(const double* refToNew, float new_exposure, const double aff[2], float cutoffTH, double res6[6]) override {
    prepare(refToNew, new_exposure, aff, cutoffTH);
    launch(0);
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    finish_res(res6);
  }
  void calc_g(float new_exposure, const double aff[2], double H[64], double b[8]) override {
    TDM_CHECK(have_params_, "calcG before calcRes (or the reference / new image changed since the last calcRes)");
    set_aff(new_exposure, aff);
    launch(1);
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    finish_g(H, b);
  }
  // The fused path writes no warped buffers, so what a later calc_g refers to - the parameters and count of the last
  // calc_res - is put back afterwards (as calc_res_batch does); on error too.
  void calc_res_g(const double* refToNew, float new_exposure, const double aff[2], float cutoffTH, double res6[6],
                  double H[64], double b[8]) override {
    const TrkParams saved = p_;
    const bool saved_have = have_params_;
    const int saved_warped = num_warped_;
    try {
      prepare(refToNew, new_exposure, aff, cutoffTH);
      launch(2);
      TDM_CUDA(cudaStreamSynchronize(stream_.get()));
      finish_res(res6);
      finish_g(H, b);
    } catch (...) {
      p_ = saved; have_params_ = saved_have; num_warped_ = saved_warped;
      throw;
    }
    p_ = saved; have_params_ = saved_have; num_warped_ = saved_warped;
  }

  // ---------------------------------------------------------------------------------------------- n1
  int set_reference_dense(const DenseRefArgs& a) override {
    TDM_CHECK(have_k_, "setReferenceDense before setK");
    TDM_CHECK(a.depth && a.T_depth_to_ref && a.ref_gray && a.ref_aff, "null argument");
    TDM_CHECK(a.step >= 1 && a.n_sparse >= 0, "bad tracking step / sparse count");
    TDM_CHECK(a.n_sparse == 0 || (a.pc_u && a.pc_v && a.pc_idepth && a.pc_color), "sparse arrays missing");
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    const size_t npx = (size_t)w_ * h_, nm = (size_t)n_max_;
    ensure_front_buffers();
    const int ns1 = a.n_sparse + 1;
    if ((long long)ns1 > n_max_) throw Error("setReferenceDense: more sparse points than n_max");
    const float* d_depth = a.depth;
    if (!a.depth_on_device) {
      std::memcpy(h_front_.get(), a.depth, 4 * npx);
      TDM_CUDA(cudaMemcpyAsync(d_depth_.get(), h_front_.get(), 4 * npx, cudaMemcpyHostToDevice, stream_.get()));
      d_depth = d_depth_.get();
    } else if (a.depth_ready) {
      TDM_CUDA(cudaStreamWaitEvent(stream_.get(), (cudaEvent_t)a.depth_ready, 0));
    }
    const float* d_id0 = nullptr;
    if (a.idepth0) {
      std::memcpy(h_front_.get() + npx, a.idepth0, 4 * npx);
      TDM_CUDA(cudaMemcpyAsync(d_idepth0_.get(), h_front_.get() + npx, 4 * npx, cudaMemcpyHostToDevice, stream_.get()));
      d_id0 = d_idepth0_.get();
    }
    const float* d_gray = a.ref_gray;
    int gstride = a.gray_stride;
    if (!a.gray_on_device) {
      std::memcpy(h_front_.get() + 2 * npx, a.ref_gray, 4 * npx);
      TDM_CUDA(cudaMemcpyAsync(d_gray_.get(), h_front_.get() + 2 * npx, 4 * npx, cudaMemcpyHostToDevice, stream_.get()));
      d_gray = d_gray_.get();
      gstride = 1;
    } else if (a.gray_ready) {
      TDM_CUDA(cudaStreamWaitEvent(stream_.get(), (cudaEvent_t)a.gray_ready, 0));
    }
    const DenseWarp m = dense_warp(a.T_depth_to_ref);
    TDM_CUDA(cudaMemsetAsync(d_proj_.get(), 0xFF, 4 * npx, stream_.get()));
    const int nx = (w_ + a.step - 1) / a.step, ny = (h_ + a.step - 1) / a.step;
    k_dense_warp<<<(nx * ny + 255) / 256, 256, 0, stream_.get()>>>(d_depth, w_, h_, a.step, m, d_proj_.get());
    const DenseSel sel{d_proj_.get(), d_id0, a.dense_only, d_gray, gstride};
    k_compact_rowcount<<<h_, 256, 0, stream_.get()>>>(sel, w_, h_, d_rowcnt_.get(), nullptr);
    k_compact_rowscan<<<1, 32, 0, stream_.get()>>>(d_rowcnt_.get(), nullptr, w_, h_, nullptr, d_rowoff_.get(), d_total_.get(), nullptr);
    TDM_CUDA(cudaMemcpyAsync(h_total_.get(), d_total_.get(), 4, cudaMemcpyDeviceToHost, stream_.get()));
    TDM_CUDA(cudaGetLastError());
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    const int total = *h_total_;
    if ((long long)a.n_sparse + 1 + total > n_max_) throw Error("setReferenceDense: n_max too small for the dense points");
    // Only now is the current reference overwritten, so that a call refused above leaves it as it was.
    // Sparse points [0, n_sparse] (the last one is the reference's stale slot, CoarseTracker.cpp:717-722).
    const float* src[4] = {a.pc_u, a.pc_v, a.pc_idepth, a.pc_color};
    for (int k = 0; k < 4; ++k) {
      if (src[k]) {
        std::memcpy(h_pc_.get() + k * nm, src[k], 4 * (size_t)ns1);
        TDM_CUDA(cudaMemcpyAsync(d_pc_.get() + k * nm, h_pc_.get() + k * nm, 4 * (size_t)ns1, cudaMemcpyHostToDevice, stream_.get()));
      } else {
        TDM_CUDA(cudaMemsetAsync(d_pc_.get() + k * nm, 0, 4, stream_.get()));
      }
    }
    k_compact_emit<<<h_, 256, 0, stream_.get()>>>(sel, w_, h_, d_rowoff_.get(), a.n_sparse + 1, n_max_, nullptr, nullptr,
                                            d_pc_.get(), d_pc_.get() + nm, d_pc_.get() + 2 * nm, d_pc_.get() + 3 * nm);
    TDM_CUDA(cudaGetLastError());
    n_ = a.n_sparse + total;      // the pre-increment quirk: the last appended point is not counted
    ref_exposure_ = a.ref_exposure;
    ref_aff_[0] = a.ref_aff[0]; ref_aff_[1] = a.ref_aff[1];
    have_ref_ = true;
    have_params_ = false;
    return n_;
  }
  int width() const override { return w_; }
  int height() const override { return h_; }
  int device() const override { return device_; }
  void get_reference(int n, float* u, float* v, float* idepth, float* color) override {
    TDM_CHECK(n >= 0 && n <= n_max_, "get_reference: bad n");
    TDM_CUDA(cudaSetDevice(device_));
    const size_t nm = (size_t)n_max_;
    float* dst[4] = {u, v, idepth, color};
    for (int k = 0; k < 4; ++k)
      if (dst[k]) TDM_CUDA(cudaMemcpyAsync(dst[k], d_pc_.get() + k * nm, 4 * (size_t)n, cudaMemcpyDeviceToHost, stream_.get()));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
  }
  void get_warped(int n, float* out) override {
    TDM_CHECK(n >= 0 && n <= n_max_, "get_warped: bad n");
    TDM_CUDA(cudaSetDevice(device_));
    for (int k = 0; k < 7; ++k)
      TDM_CUDA(cudaMemcpyAsync(out + (size_t)k * n, d_warped_.get() + (size_t)k * n_max_, 4 * (size_t)n, cudaMemcpyDeviceToHost, stream_.get()));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
  }
  // ---------------------------------------------------------------------------------------------- n2
  void set_new_device(const float* d_dI, void* ready_event) override {
    TDM_CUDA(cudaSetDevice(device_));
    if (ready_event) TDM_CUDA(cudaStreamWaitEvent(stream_.get(), (cudaEvent_t)ready_event, 0));
    TDM_CUDA(cudaMemcpyAsync(d_dI_.get(), d_dI, (size_t)3 * w_ * h_ * 4, cudaMemcpyDeviceToDevice, stream_.get()));
    have_new_ = true;
    have_params_ = false;   // calcG is only defined on the buffers of a calcRes against THIS image (cuda_coarse_tracker.cpp:277-281)
  }
  // ---------------------------------------------------------------------------------------------- n3
  void track(const TrackArgs& a, TrackResult* r) override {
    TDM_CHECK(have_k_, "track before setK");
    TDM_CHECK(have_new_, "track before setNew");
    TDM_CHECK(a.refToNew && a.aff && r, "null argument");
    TDM_CHECK(a.max_iterations >= 0 && a.max_iterations <= kMaxIterations, "max_iterations out of range");
    TDM_CUDA(cudaSetDevice(device_));
    LmIn& in = lm_in();
    fill_level(&in.lv[0], a.new_exposure, a.coarse_cutoff, a.max_iterations, a.lambda_extrapolation_limit, a.fix_a, a.fix_b);
    in.coarsest = 0;
    in.pyramid = 0;
    in.max_evals = 1 + 6 + a.max_iterations;   // initial + 6 cutoff doublings (2^6 > 50) + one per iteration
    const LmResult* o = run_lm(a.refToNew, a.aff, &r->device_ms);
    for (int i = 0; i < 16; ++i) r->refToNew[i] = o->T[i];
    r->aff[0] = o->aff[0]; r->aff[1] = o->aff[1];
    for (int i = 0; i < 6; ++i) r->res[i] = o->res[0][i];
    r->iterations = o->iterations[0]; r->evaluations = o->evaluations[0]; r->cutoff_repeat = o->repeat[0];
    // num_warped_ stays that of the last calc_res: the loop writes no warped buffers, calc_g still refers to them
  }
  // ---------------------------------------------------------------------------------------------- n5
  void track_pyramid(TrackerIface* const* levels, int coarsest, const PyramidArgs& a, PyramidResult* r) override {
    TDM_CHECK(levels && a.refToNew && a.aff && a.max_iterations && a.min_res_for_abort && r, "null argument");
    LmIn& in = pyramid_in(levels, coarsest, a.new_exposure, a.coarse_cutoff, a.max_iterations, a.lambda_extrapolation_limit,
                          a.affine_mode_a, a.affine_mode_b);
    for (int l = 0; l <= coarsest; ++l) in.min_res[l] = a.min_res_for_abort[l];
    in.pyramid = 1;
    const LmResult* o = run_lm(a.refToNew, a.aff, &r->device_ms);
    for (int i = 0; i < 16; ++i) r->refToNew[i] = o->T[i];
    r->aff[0] = o->aff[0]; r->aff[1] = o->aff[1];
    for (int l = 0; l < kMaxLevels; ++l) {
      r->last_residuals[l] = o->last_res[l];
      r->iterations[l] = o->iterations[l]; r->evaluations[l] = o->evaluations[l]; r->cutoff_repeat[l] = o->repeat[l];
    }
    for (int i = 0; i < 3; ++i) r->last_flow_indicators[i] = o->flow[i];
    r->ok = o->ok; r->aborted_level = o->aborted_level; r->repeated_level = o->repeated_level;
  }
  // ---------------------------------------------------------------------------------------------- n6
  void track_new_coarse(TrackerIface* const* levels, int coarsest, const NewCoarseArgs& a, NewCoarseResult* r, TryResult* tries) override {
    TDM_CHECK(levels && a.tries && a.aff_last_2_l && a.max_iterations && a.last_coarse_rmse && r, "null argument");
    TDM_CHECK(a.n_tries >= 1 && a.n_tries <= kMaxTries, "n_tries must be in 1..64");
    LmIn& in = pyramid_in(levels, coarsest, a.new_exposure, a.coarse_cutoff, a.max_iterations, a.lambda_extrapolation_limit,
                          a.affine_mode_a, a.affine_mode_b);
    in.max_evals *= a.n_tries;                       // the n5 bound of every try
    for (int l = 0; l < kMaxLevels; ++l) in.min_res[l] = std::nan("");   // achievedRes of the first try (FullSystem.cpp:549)
    in.pyramid = 2;
    ensure_rt_buffers();
    RetrackIn& q = *h_rt_in_;                        // free: lm_in() waited for the previous upload
    q.out = d_rt_out_;
    q.last_rmse0 = a.last_coarse_rmse[0];
    q.threshold = a.retrack_threshold;
    q.n_tries = a.n_tries;
    std::memcpy(q.tries, a.tries, (size_t)a.n_tries * 16 * sizeof(double));
    run_lm(a.tries, a.aff_last_2_l, &r->device_ms, &h_rt_out_->done, offsetof(RetrackIn, tries) + (size_t)a.n_tries * 16 * sizeof(double));
    const volatile RetrackOut* o = h_rt_out_.get();
    for (int i = 0; i < 16; ++i) r->refToNew[i] = o->T[i];
    for (int i = 0; i < 2; ++i) r->aff[i] = o->aff[i];
    for (int l = 0; l < kMaxLevels; ++l) r->achieved_res[l] = o->achieved[l];
    for (int i = 0; i < 3; ++i) r->flow_vecs[i] = o->flow[i];
    r->have_one_good = o->have_one_good; r->tries = o->tries; r->winner = o->winner;
    if (tries)
      for (int k = 0; k < o->tries; ++k) {
        const volatile TryRec& t = o->rec[k];
        for (int l = 0; l < kMaxLevels; ++l) { tries[k].last_residuals[l] = t.last_res[l]; tries[k].evaluations[l] = t.evaluations[l]; }
        tries[k].ok = t.ok; tries[k].aborted_level = t.aborted_level; tries[k].repeated_level = t.repeated_level;
      }
  }
  // ---------------------------------------------------------------------------------------------- n7
  void set_coarse_tracking_ref(TrackerIface* const* levels, const CoarseRefArgs& a, int pc_n[kMaxLevels],
                               CoarseNodiaResult* nodia) override {
    TDM_CHECK(levels && a.ref_pyramid && a.ref_aff && pc_n, "null argument");
    TDM_CHECK(!nodia || (std::isfinite(a.quantile_fraction) && a.quantile_fraction >= 0.f && a.quantile_fraction <= 1.f),
              "quantile_fraction must be finite and in [0, 1]");
    TDM_CHECK(a.n_levels >= 1 && a.n_levels <= kMaxLevels, "n_levels must be in 1..5");
    TDM_CHECK(a.n_points >= 0, "negative point count");
    TDM_CHECK(a.n_points == 0 || (a.pt_u && a.pt_v && a.pt_idepth && a.pt_hessian), "point arrays missing");
    TDM_CHECK(!a.depth || (a.T_depth_to_ref && a.step >= 1), "dense map without T_depth_to_ref, or bad tracking step");
    const int L = a.n_levels;
    TrackerImpl* lv[kMaxLevels] = {};
    for (int l = 0; l < L; ++l) {
      const std::string at = "set_coarse_tracking_ref level " + std::to_string(l) + ": ";
      TDM_CHECK(levels[l], at + "null tracker");
      lv[l] = dynamic_cast<TrackerImpl*>(levels[l]);
      TDM_CHECK(lv[l], at + "not a tracker of this library");
      TDM_CHECK(lv[l]->w_ == (w_ >> l) && lv[l]->h_ == (h_ >> l), at + "size must be level 0's size >> level");
      TDM_CHECK(lv[l]->device_ == device_, at + "trackers live on different devices");
    }
    TDM_CHECK(have_k_, "set_coarse_tracking_ref level 0: setK missing (the dense part needs K[0])");
    const PyramidIface& P = *a.ref_pyramid;
    TDM_CHECK(P.levels() >= L && P.width(0) == w_ && P.height(0) == h_, "reference pyramid: too few levels or another level-0 size");
    TDM_CHECK(P.device() == device_, "pyramid and tracker live on different devices");
    TDM_CUDA(cudaSetDevice(device_));
    ensure_front_buffers();
    ensure_coarse_buffers(a.n_points);
    if (nodia) ensure_nodia_buffers();
    // Pack (pixel, input index, value, weight input) and check the pixels: the reference would write outside idepth[0] there.
    const int n = a.n_points;
    const size_t cap = (size_t)coarse_cap_;
    int* pk = reinterpret_cast<int*>(h_pts_.get());
    for (int k = 0; k < n; ++k) {
      int u, v;
      if (a.rgbd_init) {   // int u = ph->u + 0.5 (double)
        const double fu = (double)a.pt_u[k] + 0.5, fv = (double)a.pt_v[k] + 0.5;
        TDM_CHECK(fu > -1.0 && fu < w_ && fv > -1.0 && fv < h_, "point " + std::to_string(k) + " rounds to a pixel outside the image");
        u = (int)fu; v = (int)fv;
      } else {             // int u = centerProjectedTo[0] + 0.5f (float)
        const float fu = a.pt_u[k] + 0.5f, fv = a.pt_v[k] + 0.5f;
        TDM_CHECK(fu > -1.f && fu < (float)w_ && fv > -1.f && fv < (float)h_, "point " + std::to_string(k) + " rounds to a pixel outside the image");
        u = (int)fu; v = (int)fv;
      }
      pk[k] = u + w_ * v;
      pk[cap + k] = k;
    }
    if (n) {
      std::memcpy(h_pts_.get() + 2 * cap, a.pt_idepth, 4 * (size_t)n);
      std::memcpy(h_pts_.get() + 3 * cap, a.pt_hessian, 4 * (size_t)n);
    }
    // Ordered after the pending work of every level (their references are overwritten), the pyramid and the dense map.
    for (int l = 1; l < L; ++l) lv[l]->order_before(stream_.get());
    TDM_CUDA(cudaStreamWaitEvent(stream_.get(), (cudaEvent_t)P.ready_event(), 0));
    if (a.depth && a.depth_on_device && a.depth_ready) TDM_CUDA(cudaStreamWaitEvent(stream_.get(), (cudaEvent_t)a.depth_ready, 0));
    size_t off[kMaxLevels + 1] = {0};
    for (int l = 0; l < kMaxLevels; ++l) off[l + 1] = off[l] + (size_t)(w_ >> l) * (h_ >> l);
    float *id = d_coarse_.get(), *ws = d_coarse_.get() + off[kMaxLevels], *ws2 = d_coarse_.get() + 2 * off[kMaxLevels];
    // 1. scatter (:150-182)
    TDM_CUDA(cudaMemsetAsync(id, 0, 4 * off[1], stream_.get()));
    TDM_CUDA(cudaMemsetAsync(ws, 0, 4 * off[1], stream_.get()));
    if (nodia) TDM_CUDA(cudaMemsetAsync(d_nodia_.get(), 0, 4 * off[1], stream_.get()));
    if (n) {
      int* d_pk = reinterpret_cast<int*>(d_pts_.get());
      TDM_CUDA(cudaMemcpyAsync(d_pts_.get(), h_pts_.get(), 16 * cap, cudaMemcpyHostToDevice, stream_.get()));
      int bits = 1;
      while ((1ll << bits) < (long long)w_ * h_) ++bits;
      size_t tb = 0;
      TDM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, d_pk, d_pk + 4 * cap, d_pk + cap, d_pk + 5 * cap, n, 0, bits, stream_.get()));
      grow_coarse_tmp(tb);
      TDM_CUDA(cub::DeviceRadixSort::SortPairs(d_coarse_tmp_.get(), tb, d_pk, d_pk + 4 * cap, d_pk + cap, d_pk + 5 * cap, n, 0, bits, stream_.get()));
      if (nodia)
        k_coarse_scatter<true><<<(n + 255) / 256, 256, 0, stream_.get()>>>(d_pk + 4 * cap, d_pk + 5 * cap, d_pts_.get() + 2 * cap, d_pts_.get() + 3 * cap,
                                                                     n, a.rgbd_init, id, ws, d_nodia_.get());
      else
        k_coarse_scatter<false><<<(n + 255) / 256, 256, 0, stream_.get()>>>(d_pk + 4 * cap, d_pk + 5 * cap, d_pts_.get() + 2 * cap, d_pts_.get() + 3 * cap,
                                                                      n, a.rgbd_init, id, ws, nullptr);
    }
    // 2. sum pyramid from the un-dilated level below (:222-243)
    for (int l = 1; l < L; ++l) {
      const int wl = w_ >> l, hl = h_ >> l;
      k_coarse_sum<<<(wl * hl + 255) / 256, 256, 0, stream_.get()>>>(id + off[l - 1], ws + off[l - 1], w_ >> (l - 1), id + off[l], ws + off[l], wl, hl);
    }
    // 3. dilation (:246-322): diagonal neighbours on levels 0 / 1, axis neighbours above; weights ws -> ws2
    for (int l = 0; l < L; ++l) {
      const int wl = w_ >> l, hl = h_ >> l, g = (wl * hl + 255) / 256;
      if (l < 2) k_coarse_dilate<true><<<g, 256, 0, stream_.get()>>>(id + off[l], ws + off[l], ws2 + off[l], wl, hl);
      else k_coarse_dilate<false><<<g, 256, 0, stream_.get()>>>(id + off[l], ws + off[l], ws2 + off[l], wl, hl);
    }
    // 4. normalise and compact each level into its tracker's arrays (:325-370); counts in d_coarse_cnt_[l]
    for (int l = 0; l < L; ++l) {
      const int wl = w_ >> l, hl = h_ >> l;
      const NormSel sel{id + off[l], ws2 + off[l], P.level_dI(l)};
      const size_t nm = (size_t)lv[l]->n_max_;
      float* pc = lv[l]->d_pc_.get();
      k_compact_rowcount<<<hl, 256, 0, stream_.get()>>>(sel, wl, hl, d_rowcnt_.get(), d_rowlast_.get());
      k_compact_rowscan<<<1, 32, 0, stream_.get()>>>(d_rowcnt_.get(), d_rowlast_.get(), wl, hl, nullptr, d_rowoff_.get(), d_coarse_cnt_.get() + l, d_coarse_stale_.get() + l);
      k_compact_emit<<<hl, 256, 0, stream_.get()>>>(sel, wl, hl, d_rowoff_.get(), 0, lv[l]->n_max_, d_coarse_stale_.get() + l, d_coarse_cnt_.get() + l,
                                              pc, pc + nm, pc + 2 * nm, pc + 3 * nm);
    }
    // 5. n1's dense append behind level 0's points, against the normalised idepth[0] (:655-732)
    if (a.depth) {
      const size_t npx = (size_t)w_ * h_, nm = (size_t)n_max_;
      const float* d_depth = a.depth;
      if (!a.depth_on_device) {
        std::memcpy(h_front_.get(), a.depth, 4 * npx);
        TDM_CUDA(cudaMemcpyAsync(d_depth_.get(), h_front_.get(), 4 * npx, cudaMemcpyHostToDevice, stream_.get()));
        d_depth = d_depth_.get();
      }
      TDM_CUDA(cudaMemsetAsync(d_proj_.get(), 0xFF, 4 * npx, stream_.get()));
      const int nx = (w_ + a.step - 1) / a.step, ny = (h_ + a.step - 1) / a.step;
      k_dense_warp<<<(nx * ny + 255) / 256, 256, 0, stream_.get()>>>(d_depth, w_, h_, a.step, dense_warp(a.T_depth_to_ref), d_proj_.get());
      const DenseSel sel{d_proj_.get(), id, a.dense_only, P.level_dI(0), 3};
      k_compact_rowcount<<<h_, 256, 0, stream_.get()>>>(sel, w_, h_, d_rowcnt_.get(), nullptr);
      k_compact_rowscan<<<1, 32, 0, stream_.get()>>>(d_rowcnt_.get(), nullptr, w_, h_, d_coarse_cnt_.get(), d_rowoff_.get(), d_coarse_cnt_.get() + kMaxLevels, nullptr);
      k_compact_emit<<<h_, 256, 0, stream_.get()>>>(sel, w_, h_, d_rowoff_.get(), 1, n_max_, nullptr, nullptr,
                                              d_pc_.get(), d_pc_.get() + nm, d_pc_.get() + 2 * nm, d_pc_.get() + 3 * nm);
    } else {
      TDM_CUDA(cudaMemsetAsync(d_coarse_cnt_.get() + kMaxLevels, 0, 4, stream_.get()));
    }
    if (nodia) {
      // 6. the undilated level-0 cloud (:186-218) from ws[0], which the dilation left as it was, into the persistent nodia
      //    arrays; count in d_coarse_cnt_[kMaxLevels + 1].  Slot pc_n_nodia < (w-4)(h-4) + 1 <= w*h always fits.
      const size_t npx = (size_t)w_ * h_;
      float* pc = d_nodia_.get() + npx;
      int* cnt = d_coarse_cnt_.get() + kMaxLevels + 1;
      const NodiaSel sel{d_nodia_.get(), ws, P.level_dI(0)};
      k_compact_rowcount<<<h_, 256, 0, stream_.get()>>>(sel, w_, h_, d_rowcnt_.get(), d_rowlast_.get());
      k_compact_rowscan<<<1, 32, 0, stream_.get()>>>(d_rowcnt_.get(), d_rowlast_.get(), w_, h_, nullptr, d_rowoff_.get(), cnt, d_coarse_stale_.get() + kMaxLevels);
      k_compact_emit<<<h_, 256, 0, stream_.get()>>>(sel, w_, h_, d_rowoff_.get(), 0, (int)npx, d_coarse_stale_.get() + kMaxLevels, cnt,
                                              pc, pc + npx, pc + 2 * npx, pc + 3 * npx);
      // 7. the quantile (tandem_backend.cpp:354-361) into d_coarse_cnt_[kMaxLevels + 2, + 3].  Every accepted pixel holds at
      //    least one point, so pc_n_nodia <= n: n keys padded with +inf hold every value.  The packed points are dead by now,
      //    their buffer holds the keys and their sorted copy.
      float *keys = d_pts_.get(), *sorted = d_pts_.get() + cap;
      if (n) {
        k_nodia_keys<<<(n + 255) / 256, 256, 0, stream_.get()>>>(pc + 2 * npx, cnt, n, keys);
        size_t tb = 0;
        TDM_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, keys, sorted, n, 0, 32, stream_.get()));
        grow_coarse_tmp(tb);
        TDM_CUDA(cub::DeviceRadixSort::SortKeys(d_coarse_tmp_.get(), tb, keys, sorted, n, 0, 32, stream_.get()));
      }
      k_nodia_quantile<<<1, 1, 0, stream_.get()>>>(sorted, cnt, a.quantile_fraction, d_coarse_cnt_.get() + kMaxLevels + 2);
    }
    TDM_CUDA(cudaGetLastError());
    TDM_CUDA(cudaMemcpyAsync(h_coarse_cnt_.get(), d_coarse_cnt_.get(), 4 * (kMaxLevels + (nodia ? 4 : 1)), cudaMemcpyDeviceToHost, stream_.get()));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    if (nodia) {   // written whether or not the levels fit below
      nodia->pc_n_nodia = h_coarse_cnt_.get()[kMaxLevels + 1];
      std::memcpy(&nodia->idepth_quantile, h_coarse_cnt_.get() + kMaxLevels + 2, 4);
      std::memcpy(&nodia->depth_quantile, h_coarse_cnt_.get() + kMaxLevels + 3, 4);
      have_nodia_ = true;
    }
    // Capacity: each level needs room for its count and the slot behind it; level 0 also for the dense points.
    int cnt[kMaxLevels];
    bool fits = true;
    for (int l = 0; l < L; ++l) {
      cnt[l] = h_coarse_cnt_.get()[l] + (l == 0 ? h_coarse_cnt_.get()[kMaxLevels] : 0);   // the `++pc_n` quirk: the last dense point is not counted
      fits = fits && (long long)h_coarse_cnt_.get()[l] + 1 + (l == 0 ? h_coarse_cnt_.get()[kMaxLevels] : 0) <= lv[l]->n_max_;
    }
    for (int l = 0; l < L; ++l) {
      TrackerImpl& t = *lv[l];
      t.n_ = fits ? cnt[l] : 0;
      t.have_ref_ = fits;
      t.have_params_ = false;
      t.ref_exposure_ = a.ref_exposure;
      t.ref_aff_[0] = a.ref_aff[0]; t.ref_aff_[1] = a.ref_aff[1];
    }
    if (!fits) throw Error("set_coarse_tracking_ref: a level's n_max is too small for its points; every level's reference is now empty");
    for (int l = 0; l < kMaxLevels; ++l) pc_n[l] = l < L ? cnt[l] : 0;
  }
  void get_coarse_nodia(int n, float* u, float* v, float* idepth, float* color) override {
    TDM_CHECK(have_nodia_, "get_coarse_nodia before any set_coarse_tracking_ref call with the nodia outputs on this tracker");
    const size_t npx = (size_t)w_ * h_;
    TDM_CHECK(n >= 0 && (size_t)n <= npx, "get_coarse_nodia: bad n");
    TDM_CUDA(cudaSetDevice(device_));
    float* dst[4] = {u, v, idepth, color};
    for (int k = 0; k < 4; ++k)
      if (dst[k]) TDM_CUDA(cudaMemcpyAsync(dst[k], d_nodia_.get() + (k + 1) * npx, 4 * (size_t)n, cudaMemcpyDeviceToHost, stream_.get()));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
  }
  void synchronize() override {
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
  }
  void run_resident(int iters, float* ms) override {
    TDM_CHECK(have_params_, "run_resident before calcRes");
    TDM_CUDA(cudaSetDevice(device_));
    const Event e0 = make_event(), e1 = make_event();
    TDM_CUDA(cudaEventRecord(e0.get(), stream_.get()));
    for (int i = 0; i < iters; ++i) launch(2);
    TDM_CUDA(cudaEventRecord(e1.get(), stream_.get()));
    TDM_CUDA(cudaEventSynchronize(e1.get()));
    TDM_CUDA(cudaEventElapsedTime(ms, e0.get(), e1.get()));
  }

 private:
  // Each lazy group below is made in locals and kept only once all of it exists, so its guard means "complete".
  void ensure_front_buffers() {
    if (d_proj_) return;
    const size_t npx = (size_t)w_ * h_;
    DevPtr<unsigned> proj = make_dev<unsigned>(4 * npx);
    DevPtr<float> depth = make_dev<float>(4 * npx), idepth0 = make_dev<float>(4 * npx), gray = make_dev<float>(4 * npx);
    DevPtr<int> rowcnt = make_dev<int>(4 * (size_t)h_), rowoff = make_dev<int>(4 * (size_t)h_), total = make_dev<int>(4);
    HostPtr<float> front = make_host<float>(3 * 4 * npx);
    HostPtr<int> htotal = make_host<int>(4);
    d_depth_ = std::move(depth); d_idepth0_ = std::move(idepth0); d_gray_ = std::move(gray);
    d_rowcnt_ = std::move(rowcnt); d_rowoff_ = std::move(rowoff); d_total_ = std::move(total);
    h_front_ = std::move(front); h_total_ = std::move(htotal);
    d_proj_ = std::move(proj);
  }
  // n7 scratch: idepth, weights and dilated weights of every level (levels concatenated), the packed points (pixel, index,
  // value, weight input), their sorted copies (pixel, index) and the sort's temporary storage; grown to the largest point count
  void ensure_coarse_buffers(int n) {
    if (!d_coarse_) {
      size_t tot = 0;
      for (int l = 0; l < kMaxLevels; ++l) tot += (size_t)(w_ >> l) * (h_ >> l);
      DevPtr<float> coarse = make_dev<float>(3 * 4 * tot);
      DevPtr<int2> rowlast = make_dev<int2>(8 * (size_t)h_);
      // counts per level, the dense count, then (nodia) pc_n_nodia and the quantile's idepth and depth bits
      DevPtr<int> cnt = make_dev<int>(4 * (kMaxLevels + 4)), stale = make_dev<int>(4 * (kMaxLevels + 1));
      HostPtr<int> hcnt = make_host<int>(4 * (kMaxLevels + 4));
      d_rowlast_ = std::move(rowlast); d_coarse_cnt_ = std::move(cnt); d_coarse_stale_ = std::move(stale);
      h_coarse_cnt_ = std::move(hcnt);
      d_coarse_ = std::move(coarse);
    }
    if (n > coarse_cap_) {   // the old set is freed first; coarse_cap_ is 0 until the new one is complete
      const int cap = n > 1024 ? n : 1024;
      d_pts_.reset(); h_pts_.reset(); d_coarse_tmp_.reset(); coarse_tmp_bytes_ = 0; coarse_cap_ = 0;
      d_pts_ = make_dev<float>(6 * 4 * (size_t)cap);
      h_pts_ = make_host<float>(4 * 4 * (size_t)cap);
      size_t tb = 0;
      TDM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, (const int*)nullptr, (int*)nullptr, (const int*)nullptr, (int*)nullptr, cap));
      d_coarse_tmp_ = make_dev(tb);
      coarse_tmp_bytes_ = tb;
      coarse_cap_ = cap;
    }
  }
  void grow_coarse_tmp(size_t tb) {
    if (tb <= coarse_tmp_bytes_) return;
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    d_coarse_tmp_.reset(); coarse_tmp_bytes_ = 0;
    d_coarse_tmp_ = make_dev(tb);
    coarse_tmp_bytes_ = tb;
  }
  // the nodia image (unweighted idepth sums of level 0) and the persistent pc_u/v/idepth/color_nodia, w*h floats each; the
  // arrays start zeroed, so a slot nothing has written reads as 0
  void ensure_nodia_buffers() {
    if (d_nodia_) return;
    const size_t npx = (size_t)w_ * h_;
    DevPtr<float> nodia = make_dev<float>(5 * 4 * npx);
    TDM_CUDA(cudaMemsetAsync(nodia.get() + npx, 0, 4 * 4 * npx, stream_.get()));
    d_nodia_ = std::move(nodia);
  }
  // KRKi = (K R) Ki, Kt = K t in float, k = 0,1,2 (CoarseTracker.cpp:676-677)
  DenseWarp dense_warp(const double* T) const {
    DenseWarp m;
    const float K[9] = {fx_, 0, cx_, 0, fy_, cy_, 0, 0, 1};
    const float Ki[9] = {1.0f / fx_, 0, -cx_ / fx_, 0, 1.0f / fy_, -cy_ / fy_, 0, 0, 1};
    float R[9], t[3], KR[9];
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) R[3 * r + c] = (float)T[4 * r + c];
      t[r] = (float)T[4 * r + 3];
    }
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        volatile float s = 0;
        for (int k = 0; k < 3; ++k) { volatile float q = K[3 * r + k] * R[3 * k + c]; s = s + q; }
        KR[3 * r + c] = s;
      }
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) {
        volatile float s = 0;
        for (int k = 0; k < 3; ++k) { volatile float q = KR[3 * r + k] * Ki[3 * k + c]; s = s + q; }
        m.KRKi[3 * r + c] = s;
      }
      volatile float s = 0;
      for (int k = 0; k < 3; ++k) { volatile float q = K[3 * r + k] * t[k]; s = s + q; }
      m.Kt[r] = s;
    }
    return m;
  }
  // The device LM loop as a graph, built once per tracker: k_lm_init, then WHILE (handle, default 1) { k_tracker<4> }.
  // Every parameter that changes between calls (levels, sizes, buffers, pose) travels in LmCtx::in, so the graph never
  // needs an update.
  void ensure_lm_buffers() {
    if (lm_exec_) return;
    DevPtr<LmCtx> ctx = make_dev<LmCtx>(sizeof(LmCtx));
    DevPtr<double> out = make_dev<double>(kOut * 8);
    HostPtr<LmIn> in = make_host<LmIn>(sizeof(LmIn));
    HostPtr<LmResult> res = make_host<LmResult>(sizeof(LmResult), cudaHostAllocMapped);
    LmResult* d_res = nullptr;
    TDM_CUDA(cudaHostGetDevicePointer(&d_res, res.get(), 0));
    Event in_free = make_event(cudaEventDisableTiming), e0 = make_event(), e1 = make_event();
    const Graph g = make_graph();
    cudaGraphConditionalHandle loop;
    TDM_CUDA(cudaGraphConditionalHandleCreate(&loop, g.get(), 1, cudaGraphCondAssignDefault));
    cudaKernelNodeParams kp = {};
    LmCtx* d_ctx = ctx.get();
    void* init_args[] = {&d_ctx, &d_res, &loop};
    kp.func = (void*)k_lm_init;
    kp.gridDim = dim3(1); kp.blockDim = dim3(32);
    kp.kernelParams = init_args;
    cudaGraphNode_t init;
    TDM_CUDA(cudaGraphAddKernelNode(&init, g.get(), nullptr, 0, &kp));
    cudaGraphNodeParams cp = {};
    cp.type = cudaGraphNodeTypeConditional;
    cp.conditional.handle = loop;
    cp.conditional.type = cudaGraphCondTypeWhile;
    cp.conditional.size = 1;
    cudaGraphNode_t while_node;
    TDM_CUDA(cudaGraphAddNode(&while_node, g.get(), &init, 1, &cp));
    TrkParams p{};                                 // unused: the kernel reads the level's parameters from LmCtx
    TrkBufs b{};
    b.lm = d_ctx; b.partials = d_partials_.get(); b.ticket = d_ticket_.get(); b.out = out.get();
    void* eval_args[] = {&p, &b};
    kp.func = (void*)k_tracker<4>;
    kp.gridDim = dim3(kBlocks); kp.blockDim = dim3(kThreads);
    kp.kernelParams = eval_args;
    cudaGraphNode_t eval;
    TDM_CUDA(cudaGraphAddKernelNode(&eval, cp.conditional.phGraph_out[0], nullptr, 0, &kp));
    GraphExec exec = make_graph_exec(g.get());
    d_lm_ctx_ = std::move(ctx); d_lm_out_ = std::move(out); h_lm_in_ = std::move(in); h_lm_res_ = std::move(res);
    d_lm_res_ = d_res;
    lm_in_free_ = std::move(in_free); lm_e0_ = std::move(e0); lm_e1_ = std::move(e1);
    lm_exec_ = std::move(exec);
  }
  // the staging of LmCtx::in; free once the previous call's upload has completed (normally long since)
  LmIn& lm_in() {
    ensure_lm_buffers();
    TDM_CUDA(cudaEventSynchronize(lm_in_free_.get()));
    return *h_lm_in_;
  }
  // Checks the levels of an n5 / n6 call and fills LmCtx::in's staging with them (everything but min_res and the mode); an
  // invalid call throws before anything is touched.
  LmIn& pyramid_in(TrackerIface* const* levels, int coarsest, float new_exposure, float coarse_cutoff, const int* max_iterations,
                   float lambda_limit, float mode_a, float mode_b) {
    TDM_CHECK(coarsest >= 0 && coarsest < kMaxLevels, "coarsest_level must be in 0..4");
    TrackerImpl* lv[kMaxLevels] = {};
    for (int l = 0; l <= coarsest; ++l) {
      const std::string at = "track_pyramid level " + std::to_string(l) + ": ";
      TDM_CHECK(levels[l], at + "null tracker");
      lv[l] = dynamic_cast<TrackerImpl*>(levels[l]);
      TDM_CHECK(lv[l], at + "not a tracker of this library");
      TDM_CHECK(lv[l]->w_ == (w_ >> l) && lv[l]->h_ == (h_ >> l), at + "size must be level 0's size >> level");
      TDM_CHECK(lv[l]->device_ == device_, at + "trackers live on different devices");
      TDM_CHECK(lv[l]->have_k_, at + "setK missing");
      TDM_CHECK(lv[l]->have_ref_, at + "no reference set");
      TDM_CHECK(lv[l]->have_new_, at + "no new image set");
      TDM_CHECK(max_iterations[l] >= 0 && max_iterations[l] <= kMaxIterations, at + "max_iterations out of range");
    }
    TDM_CUDA(cudaSetDevice(device_));
    LmIn& in = lm_in();
    in.max_evals = 0;
    for (int l = 0; l <= coarsest; ++l) {
      lv[l]->fill_level(&in.lv[l], new_exposure, coarse_cutoff, max_iterations[l], lambda_limit, mode_a < 0, mode_b < 0);
      in.max_evals += 2 * (1 + 6 + max_iterations[l]);   // a level may run twice (the repeat rule)
      if (l > 0) lv[l]->order_before(stream_.get());           // reference upload, setNewFromPyramid copy of that tracker
    }
    in.mode_a = mode_a; in.mode_b = mode_b;
    in.coarsest = coarsest;
    return in;
  }
  // this tracker's parameters and buffers as one level of the device LM loop
  void fill_level(LmLevel* L, float new_exposure, float coarse_cutoff, int max_iter, float lambda_limit, int fix_a, int fix_b) const {
    L->p = TrkParams{};
    L->p.w = w_; L->p.h = h_; L->p.n = n_;
    L->p.fx = fx_; L->p.fy = fy_; L->p.cx = cx_; L->p.cy = cy_;
    for (int i = 0; i < 9; ++i) L->p.Ki[i] = Ki_[i];
    L->p.huber = huber_; L->p.ref_b = (float)ref_aff_[1];
    const size_t nm = (size_t)n_max_;
    L->pc_u = d_pc_.get(); L->pc_v = d_pc_.get() + nm; L->pc_idepth = d_pc_.get() + 2 * nm; L->pc_color = d_pc_.get() + 3 * nm; L->dInew = d_dI_.get();
    LmConfig& c = L->cfg;
    for (int i = 0; i < 9; ++i) c.Ki[i] = Ki_[i];
    c.ref_exposure = ref_exposure_; c.new_exposure = new_exposure;
    c.ref_aff[0] = ref_aff_[0]; c.ref_aff[1] = ref_aff_[1];
    c.huber = huber_; c.coarse_cutoff = coarse_cutoff; c.max_iter = max_iter;
    c.lambda_limit = lambda_limit; c.fix_a = fix_a; c.fix_b = fix_b;
  }
  // orders this tracker's pending stream work before work enqueued later on `other`
  void order_before(cudaStream_t other) {
    if (!ready_) ready_ = make_event(cudaEventDisableTiming);
    TDM_CUDA(cudaEventRecord(ready_.get(), stream_.get()));
    TDM_CUDA(cudaStreamWaitEvent(other, ready_.get(), 0));
  }
  // Runs the graph on h_lm_in_ (filled by the caller) with one host wait; returns the mapped result.  n6 passes its own mapped
  // completion flag and the first rt_bytes of h_rt_in_ to upload next to LmIn.
  const LmResult* run_lm(const double* T0, const double* aff0, float* device_ms, volatile int* done = nullptr, size_t rt_bytes = 0) {
    LmIn& in = *h_lm_in_;
    for (int i = 0; i < 16; ++i) in.T0[i] = T0[i];
    in.aff0[0] = aff0[0]; in.aff0[1] = aff0[1];
    if (!done) done = &h_lm_res_->done;
    *done = 0;
    TDM_CUDA(cudaEventRecord(lm_e0_.get(), stream_.get()));
    TDM_CUDA(cudaMemcpyAsync(&d_lm_ctx_->in, h_lm_in_.get(), sizeof(LmIn), cudaMemcpyHostToDevice, stream_.get()));
    if (rt_bytes) TDM_CUDA(cudaMemcpyAsync(&d_lm_ctx_->rin, h_rt_in_.get(), rt_bytes, cudaMemcpyHostToDevice, stream_.get()));
    TDM_CUDA(cudaEventRecord(lm_in_free_.get(), stream_.get()));
    TDM_CUDA(cudaGraphLaunch(lm_exec_.get(), stream_.get()));
    TDM_CUDA(cudaEventRecord(lm_e1_.get(), stream_.get()));
    TDM_CUDA(cudaEventSynchronize(lm_e1_.get()));
    TDM_CUDA(cudaEventElapsedTime(device_ms, lm_e0_.get(), lm_e1_.get()));
    if (*done != 1) throw Error("track: the device loop did not finish (internal error)");
    return h_lm_res_.get();
  }
  // n6: the try list's pinned staging (guarded like LmCtx::in's, by lm_in_free_) and the mapped result with the per-try records
  void ensure_rt_buffers() {
    if (h_rt_in_) return;
    HostPtr<RetrackIn> in = make_host<RetrackIn>(sizeof(RetrackIn));
    HostPtr<RetrackOut> out = make_host<RetrackOut>(sizeof(RetrackOut), cudaHostAllocMapped);
    TDM_CUDA(cudaHostGetDevicePointer(&d_rt_out_, out.get(), 0));
    h_rt_out_ = std::move(out);
    h_rt_in_ = std::move(in);
  }
  void set_aff(float new_exposure, const double aff[2]) {  // AffLight::fromToVecExposure, cpp:42-52
    float eF = ref_exposure_, eT = new_exposure;
    if (eF == 0 || eT == 0) eT = eF = 1;
    const double a = std::exp(aff[0] - ref_aff_[0]) * eT / eF;
    const double b = aff[1] - a * ref_aff_[1];
    p_.affa = (float)a; p_.affb = (float)b; p_.ref_b = (float)ref_aff_[1];
  }
  void prepare(const double* refToNew, float new_exposure, const double aff[2], float cutoffTH) {
    TDM_CHECK(have_k_, "calcRes before setK");
    TDM_CHECK(have_new_, "calcRes before setNew");
    TDM_CUDA(cudaSetDevice(device_));
    p_.w = w_; p_.h = h_; p_.n = n_;
    p_.fx = fx_; p_.fy = fy_; p_.cx = cx_; p_.cy = cy_;
    float R[9];
    for (int r = 0; r < 3; ++r) {
      for (int k = 0; k < 3; ++k) R[3 * r + k] = (float)refToNew[4 * r + k];
      p_.t[r] = (float)refToNew[4 * r + 3];
    }
    for (int i = 0; i < 9; ++i) p_.Ki[i] = Ki_[i];
    for (int r = 0; r < 3; ++r)
      for (int q = 0; q < 3; ++q) {
        volatile float s = 0;
        for (int k = 0; k < 3; ++k) { volatile float m = R[3 * r + k] * Ki_[3 * k + q]; s = s + m; }
        p_.RKi[3 * r + q] = s;
      }
    set_aff(new_exposure, aff);
    p_.huber = huber_; p_.cutoff = cutoffTH;
    p_.maxEnergy = 2 * huber_ * cutoffTH - huber_ * huber_;
    have_params_ = true;
  }
  void launch(int mode) {
    TDM_CUDA(cudaSetDevice(device_));   // another handle of this thread may have switched the current device
    TrkBufs b;
    const size_t nm = (size_t)n_max_;
    b.lm = nullptr;
    b.pc_u = d_pc_.get(); b.pc_v = d_pc_.get() + nm; b.pc_idepth = d_pc_.get() + 2 * nm; b.pc_color = d_pc_.get() + 3 * nm;
    b.dInew = d_dI_.get(); b.warped = d_warped_.get(); b.n_max = n_max_;
    b.partials = d_partials_.get(); b.ticket = d_ticket_.get(); b.out = d_out_; b.batch = nullptr;
    if (mode == 0) k_tracker<0><<<kBlocks, kThreads, 0, stream_.get()>>>(p_, b);
    else if (mode == 1) k_tracker<1><<<kBlocks, kThreads, 0, stream_.get()>>>(p_, b);
    else k_tracker<2><<<kBlocks, kThreads, 0, stream_.get()>>>(p_, b);
    TDM_CUDA(cudaGetLastError());
  }
  // Batched calcRes over n_hyp poses (motion hypotheses of FullSystem::trackNewCoarse, FullSystem.cpp:437-530) in ONE launch and
  // one synchronisation: res6 of hypothesis k equals calc_res(refToNew + 16 k, ..., aff + 2 k, ...) bit for bit.  Leaves the
  // buffers of the last calcRes untouched (calcG still refers to them).
  void calc_res_batch(int n_hyp, const double* refToNew, float new_exposure, const double* aff, float cutoffTH, double* res6) override {
    TDM_CHECK(n_hyp >= 1 && n_hyp <= kMaxHyp, "calcResBatch: 1..64 hypotheses");
    TDM_CHECK(have_k_ && have_new_, "calcResBatch before setK / setNew");
    TDM_CUDA(cudaSetDevice(device_));
    if (!d_batch_) {
      DevPtr<TrkPose> batch = make_dev<TrkPose>(kMaxHyp * sizeof(TrkPose));
      HostPtr<TrkPose> hbatch = make_host<TrkPose>(kMaxHyp * sizeof(TrkPose));
      DevPtr<double> partials = make_dev<double>((size_t)kMaxHyp * kBlocks * kOut * 8);
      DevPtr<unsigned> ticket = make_dev<unsigned>(kMaxHyp * 4);
      TDM_CUDA(cudaMemset(ticket.get(), 0, kMaxHyp * 4));
      HostPtr<double> out = make_host<double>((size_t)kMaxHyp * kOut * 8, cudaHostAllocMapped);
      TDM_CUDA(cudaHostGetDevicePointer(&d_batch_out_, out.get(), 0));
      h_batch_ = std::move(hbatch); d_batch_partials_ = std::move(partials); d_batch_ticket_ = std::move(ticket);
      h_batch_out_ = std::move(out);
      d_batch_ = std::move(batch);
    }
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));   // the pinned pose staging may still be in flight from the previous batch
    const TrkParams saved = p_;
    const bool saved_have = have_params_;
    for (int k = 0; k < n_hyp; ++k) {
      prepare(refToNew + 16 * k, new_exposure, aff + 2 * k, cutoffTH);   // the exact host arithmetic of calcRes, per pose
      TrkPose& q = h_batch_.get()[k];
      for (int i = 0; i < 9; ++i) q.RKi[i] = p_.RKi[i];
      for (int i = 0; i < 3; ++i) q.t[i] = p_.t[i];
      q.affa = p_.affa; q.affb = p_.affb; q.cutoff = p_.cutoff; q.maxEnergy = p_.maxEnergy;
    }
    TrkParams pb = p_;
    p_ = saved;                                   // calcG keeps referring to the last plain calcRes
    have_params_ = saved_have;
    TDM_CUDA(cudaMemcpyAsync(d_batch_.get(), h_batch_.get(), n_hyp * sizeof(TrkPose), cudaMemcpyHostToDevice, stream_.get()));
    TrkBufs b;
    const size_t nm = (size_t)n_max_;
    b.lm = nullptr;
    b.pc_u = d_pc_.get(); b.pc_v = d_pc_.get() + nm; b.pc_idepth = d_pc_.get() + 2 * nm; b.pc_color = d_pc_.get() + 3 * nm;
    b.dInew = d_dI_.get(); b.warped = nullptr; b.n_max = n_max_;
    b.partials = d_batch_partials_.get(); b.ticket = d_batch_ticket_.get(); b.out = d_batch_out_; b.batch = d_batch_.get();
    k_tracker<3><<<dim3(kBlocks, n_hyp), kThreads, 0, stream_.get()>>>(pb, b);
    TDM_CUDA(cudaGetLastError());
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    for (int k = 0; k < n_hyp; ++k) {
      const volatile double* o = h_batch_out_.get() + (size_t)k * kOut;
      double* r = res6 + 6 * k;
      r[0] = o[0]; r[1] = o[1]; r[2] = o[4] / o[6]; r[3] = 0; r[4] = o[5] / o[6]; r[5] = o[3] / o[1];
    }
  }
  void finish_res(double res6[6]) {  // cpp:264-272
    const volatile double* o = h_out_.get();
    res6[0] = o[0]; res6[1] = o[1];
    res6[2] = o[4] / o[6]; res6[3] = 0; res6[4] = o[5] / o[6];
    res6[5] = o[3] / o[1];
    num_warped_ = (int)o[2];
  }
  void finish_g(double H[64], double b[8]) {  // cpp:335-355
    const volatile double* o = h_out_.get() + kRes;
    const double factor = 1.0 / num_warped_;
    static const double scale[8] = {1.0, 1.0, 1.0, 0.5, 0.5, 0.5, 10.0, 1000.0};
    for (int r = 0; r < 8; ++r) {
      for (int q = 0; q < 8; ++q) {
        const int lo = r < q ? r : q, hi = r < q ? q : r;
        H[8 * r + q] = o[lo * 9 + hi - lo * (lo + 1) / 2] * factor * scale[r] * scale[q];
      }
      b[r] = o[r * 9 + 8 - r * (r + 1) / 2] * factor * scale[r];
    }
  }

  int w_, h_;
  float huber_, coarse_cutoff_;
  int device_;
  int n_max_ = 0, n_ = 0;
  float fx_ = 0, fy_ = 0, cx_ = 0, cy_ = 0, Ki_[9];
  bool have_k_ = false, have_ref_ = false, have_new_ = false, have_params_ = false;
  static constexpr int kMaxIterations = 200;
  float ref_exposure_ = 1.f;
  double ref_aff_[2] = {0, 0};
  Stream stream_;
  DevPtr<float> d_pc_, d_warped_, d_dI_;
  HostPtr<float> h_pc_, h_dI_;
  static constexpr int kMaxHyp = 64;
  DevPtr<TrkPose> d_batch_;
  HostPtr<TrkPose> h_batch_;
  DevPtr<double> d_batch_partials_;
  HostPtr<double> h_batch_out_;
  double* d_batch_out_ = nullptr;
  DevPtr<unsigned> d_batch_ticket_;
  DevPtr<double> d_partials_;
  HostPtr<double> h_out_;
  double* d_out_ = nullptr;
  DevPtr<unsigned> d_ticket_;
  TrkParams p_{};
  int num_warped_ = 0;
  // n1 buffers
  DevPtr<unsigned> d_proj_;
  DevPtr<float> d_depth_, d_idepth0_, d_gray_;
  HostPtr<float> h_front_;
  DevPtr<int> d_rowcnt_, d_rowoff_, d_total_;
  HostPtr<int> h_total_;
  // n3 buffers
  DevPtr<LmCtx> d_lm_ctx_;
  DevPtr<double> d_lm_out_;
  HostPtr<LmIn> h_lm_in_;
  HostPtr<LmResult> h_lm_res_;
  LmResult* d_lm_res_ = nullptr;
  GraphExec lm_exec_;
  Event lm_in_free_, lm_e0_, lm_e1_;
  Event ready_;   // order_before
  // n6 buffers
  HostPtr<RetrackIn> h_rt_in_;
  HostPtr<RetrackOut> h_rt_out_;
  RetrackOut* d_rt_out_ = nullptr;
  // n7 buffers (ensure_coarse_buffers)
  DevPtr<float> d_coarse_, d_pts_;
  HostPtr<float> h_pts_;
  DevPtr<int2> d_rowlast_;
  DevPtr<int> d_coarse_cnt_, d_coarse_stale_;
  HostPtr<int> h_coarse_cnt_;
  DevPtr<void> d_coarse_tmp_;
  size_t coarse_tmp_bytes_ = 0;
  int coarse_cap_ = 0;
  DevPtr<float> d_nodia_;   // ensure_nodia_buffers
  bool have_nodia_ = false;
};


// ================================================================================================
class PyramidImpl final : public PyramidIface {
 public:
  PyramidImpl(int w, int h, int levels, int device) : w_(w), h_(h), levels_(levels), device_(device) {
    int nd = 0;
    if (cudaGetDeviceCount(&nd) != cudaSuccess || nd == 0)
      throw Error("tandem_b200: no CUDA device visible - this library has no CPU fallback");
    TDM_CHECK(w > 0 && h > 0 && levels >= 1 && levels <= 8 && (w >> (levels - 1)) >= 3 && (h >> (levels - 1)) >= 3, "bad pyramid shape");
    TDM_CUDA(cudaSetDevice(device_));
    stream_ = make_stream(0);
    ready_ = make_event(cudaEventDisableTiming);
    size_t tot = 0;
    for (int l = 0; l < levels; ++l) { off_.push_back(tot); tot += (size_t)(w >> l) * (h >> l); }
    d_dI_ = make_dev<float>(3 * 4 * tot);
    d_abs_ = make_dev<float>(4 * tot);
    d_gray_ = make_dev<float>(4 * (size_t)w * h);
    d_in_ = make_dev<float>(4 * (size_t)w * h);
    h_in_ = make_host<float>(4 * (size_t)w * h);
  }
  ~PyramidImpl() override {
    cudaSetDevice(device_);
    cudaStreamSynchronize(stream_.get());
  }
  void build(const float* gray_host) override {
    TDM_CHECK(gray_host, "null argument");
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    std::memcpy(h_in_.get(), gray_host, 4 * (size_t)w_ * h_);
    TDM_CUDA(cudaMemcpyAsync(d_in_.get(), h_in_.get(), 4 * (size_t)w_ * h_, cudaMemcpyHostToDevice, stream_.get()));
    for (int l = 0; l < levels_; ++l) {
      const int wl = w_ >> l, hl = h_ >> l, n = wl * hl;
      const float* src = l == 0 ? d_in_.get() : d_dI_.get() + 3 * off_[l - 1];
      k_pyr_level<<<(n + 255) / 256, 256, 0, stream_.get()>>>(src, l > 0, l > 0 ? (w_ >> (l - 1)) : 0, d_gray_.get(), wl, hl);
      k_pyr_grad<false><<<(n + 255) / 256, 256, 0, stream_.get()>>>(d_gray_.get(), d_dI_.get() + 3 * off_[l], d_abs_.get() + off_[l],
                                                                    wl, hl, nullptr);
    }
    TDM_CUDA(cudaGetLastError());
    TDM_CUDA(cudaEventRecord(ready_.get(), stream_.get()));
  }
  float* device_input() override { return d_gray_.get(); }
  void* stream() const override { return (void*)stream_.get(); }
  void build_device(const float* d_B) override {
    TDM_CUDA(cudaSetDevice(device_));
    for (int l = 0; l < levels_; ++l) {
      const int wl = w_ >> l, hl = h_ >> l, n = wl * hl;
      if (l > 0)
        k_pyr_level<<<(n + 255) / 256, 256, 0, stream_.get()>>>(d_dI_.get() + 3 * off_[l - 1], 1, w_ >> (l - 1), d_gray_.get(), wl, hl);
      float* dI = d_dI_.get() + 3 * off_[l];
      float* ag = d_abs_.get() + off_[l];
      if (d_B)
        k_pyr_grad<true><<<(n + 255) / 256, 256, 0, stream_.get()>>>(d_gray_.get(), dI, ag, wl, hl, d_B);
      else
        k_pyr_grad<false><<<(n + 255) / 256, 256, 0, stream_.get()>>>(d_gray_.get(), dI, ag, wl, hl, nullptr);
    }
    TDM_CUDA(cudaGetLastError());
    TDM_CUDA(cudaEventRecord(ready_.get(), stream_.get()));
  }
  void get_level(int lvl, float* dI_host, float* absgrad_host) override {
    TDM_CHECK(lvl >= 0 && lvl < levels_, "bad level");
    TDM_CUDA(cudaSetDevice(device_));
    const size_t n = (size_t)(w_ >> lvl) * (h_ >> lvl);
    if (dI_host) TDM_CUDA(cudaMemcpyAsync(dI_host, d_dI_.get() + 3 * off_[lvl], 12 * n, cudaMemcpyDeviceToHost, stream_.get()));
    if (absgrad_host) TDM_CUDA(cudaMemcpyAsync(absgrad_host, d_abs_.get() + off_[lvl], 4 * n, cudaMemcpyDeviceToHost, stream_.get()));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
  }
  const float* level_dI(int lvl) const override { return d_dI_.get() + 3 * off_.at(lvl); }
  const float* level_abs(int lvl) const override { return d_abs_.get() + off_.at(lvl); }
  void* ready_event() const override { return (void*)ready_.get(); }
  void wait_for(void* event) const override {
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaStreamWaitEvent(stream_.get(), (cudaEvent_t)event, 0));
  }
  int width(int lvl) const override { return w_ >> lvl; }
  int height(int lvl) const override { return h_ >> lvl; }
  int levels() const override { return levels_; }
  int device() const override { return device_; }

 private:
  int w_, h_, levels_, device_;
  Stream stream_;
  Event ready_;
  std::vector<size_t> off_;
  DevPtr<float> d_dI_, d_abs_, d_gray_, d_in_;
  HostPtr<float> h_in_;
};

PyramidIface* make_pyramid(int w, int h, int levels, int device) { return new PyramidImpl(w, h, levels, device); }

TrackerIface* make_tracker(int w, int h, float huber, float cutoff, int n_max, int device) {
  return new TrackerImpl(w, h, huber, cutoff, n_max, device);
}

}  // namespace tdm
