// n12: the active residuals of DSO's window, kept in device memory for one FullSystem::optimize, and their linearisation
// (FullSystem::linearizeAll, tandem/src/FullSystem/FullSystemOptimize.cpp:142-210, calling PointFrameResidual::linearize,
// Residuals.cpp:78-274, per residual), the newest frame's outlier threshold (setNewFrameEnergyTH, :93-141), applyRes
// (Residuals.cpp:306-328) and the reductor's fixLinearization branch (:52-85).  Every float operation is the reference's own,
// correctly rounded and in its order (__f*_rn, no contraction); oracle/linearize_oracle.c restates the same statements.
//
// Shape (DESIGN.md, n12): a group of 8 lanes per residual, lane i on pattern index i, 4 residuals per warp.  Every lane of the
// group evaluates the centre projection (the same values, so every OOB return is uniform in the group; lane 0 stores the
// d_xi / d_C / d_d rows), samples its own pattern pixel, and the twelve serial sums run in pattern order 0..7 through
// shuffles.  The energy
// is each residual's double return summed by a fixed tree (deterministic, independent of the launch); the threshold's k-th
// smallest value comes from a radix sort of the candidates' float bits.
#include <cmath>
#include <cstring>
#include <vector>

#include <cub/device/device_radix_sort.cuh>

#include "dso_sample.cuh"
#include "tracker.h"

namespace tdm {

namespace {

constexpr int kFrames = 8, kPre = 27, kJ = 74;
constexpr int kLinThreads = 128, kFinishThreads = 512;
enum { RS_IN = 0, RS_OOB = 1, RS_OUTLIER = 2 };   // ResState
// precalc record [host * n + target] (tdm_active_linearize)
enum { PC_KRKI = 0, PC_KT = 9, PC_R0 = 12, PC_T0 = 21, PC_AFF = 24, PC_B0 = 26 };
// Jacobian record: RawResidualJacobian's members in declaration order, the 2x2 matrices column-major
enum { J_RESF = 0, J_PDXI = 8, J_PDC = 20, J_PDD = 28, J_IDX = 30, J_ABF = 46, J_IDX2 = 62, J_ABJIDX = 66, J_AB2 = 70 };
constexpr float kScaleF = 50.f, kScaleC = 50.f, kScaleIdepth = 1.f;   // HessianBlocks.h:59-63

struct Settings {   // tdm_linearize_settings
  float huber, outlier_th_sum_component, affine_opt_mode_a, affine_opt_mode_b, frame_energy_th_n, const_weight, fac_median,
      overall_energy_th_weight;
};

struct Points {   // one row per field, capacity entries each
  const int* host;
  const float *u, *v, *color, *weights;   // color / weights: row k at k * cap
};
struct Residuals {
  const int *point, *target;
  signed char *state, *new_state;
  float *energy, *new_energy, *new_energy_wo, *center, *J, *relbs;
  double* ret;
  unsigned* key;
  unsigned char *removed, *active, *took;   // active, took: the taken data's flags (accumulate.cu)
};
struct LinLaunch {
  const float* dI[kFrames];
  const float* pre;      // n * n * kPre
  const float* th;       // frameEnergyTH per frame
  const float *ids, *idz;   // idepth_scaled, idepth_zero_scaled per point
  int n_frames, n_res, w, h, cap, fix;
  float fxl, fyl, cxl, cyl, fxli, fyli;
  Settings s;
};

__device__ __forceinline__ float fmaxf_ref(float a, float b) { return a < b ? b : a; }   // std::max<float>

// PointFrameResidual::linearize of residual r (group of 8 lanes, lane i = pattern index i) and, with fix, applyRes and the
// reductor's relBS.  ret[r] is linearize's double return; key[r] the threshold candidate (setNewFrameEnergyTH), ~0u if none.
__global__ void __launch_bounds__(kLinThreads) k_linearize(LinLaunch L, Points P, Residuals R, unsigned* __restrict__ n_key) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x, r = t >> 3, i = threadIdx.x & 7;
  if (r >= L.n_res) return;   // group-uniform
  const unsigned gmask = 0xFFu << (threadIdx.x & 24);
  const int gbase = threadIdx.x & 24;
  const int p = R.point[r], tg = R.target[r], hf = P.host[p];
  const int cap = L.cap;
  const int state = R.state[r];
  const float* pc = L.pre + (size_t)(hf * L.n_frames + tg) * kPre;
  float* J = R.J + (size_t)r * kJ;
  int ns = RS_OOB;
  float nE = R.new_energy[r], nEwo = -1.f, cx = __int_as_float(0x7fc00000), cy = cx, cz = cx;
  double ret = (double)R.energy[r];
  if (state != RS_OOB) {
    const float u0 = P.u[p], v0 = P.v[p];
    const float idz = L.idz[p], ids = L.ids[p];
    const float wM3G = (float)(L.w - 3), hM3G = (float)(L.h - 3);
    // projectPoint, 13-argument form (ResidualProjections.h:62-87), dx = dy = 0
    const float* R0 = pc + PC_R0;
    const float* t0 = pc + PC_T0;
    const float K0 = fm(fs(fa(u0, 0.f), L.cxl), L.fxli), K1 = fm(fs(fa(v0, 0.f), L.cyl), L.fyli);
    const float p0 = fa(fa(fa(fm(R0[0], K0), fm(R0[1], K1)), fm(R0[2], 1.f)), fm(t0[0], idz));
    const float p1 = fa(fa(fa(fm(R0[3], K0), fm(R0[4], K1)), fm(R0[5], 1.f)), fm(t0[1], idz));
    const float p2 = fa(fa(fa(fm(R0[6], K0), fm(R0[7], K1)), fm(R0[8], 1.f)), fm(t0[2], idz));
    const float drescale = fd(1.0f, p2);
    const float new_idepth = fm(idz, drescale);
    bool ok = drescale > 0;
    float u = 0.f, v = 0.f;
    if (ok) {
      u = fm(p0, drescale);
      v = fm(p1, drescale);
      const float Ku = fa(fm(u, L.fxl), L.cxl), Kv = fa(fm(v, L.fyl), L.cyl);
      ok = Ku > 1.1f && Kv > 1.1f && Ku < wM3G && Kv < hM3G;
      if (ok) { cx = Ku; cy = Kv; cz = new_idepth; }
    }
    if (ok) {
      if (i == 0) {   // the rows of d[x,y] / d[xi, C, idepth]; the same on every lane of the group, stored by lane 0
        const float fxl = L.fxl, fyl = L.fyl;
        J[J_PDD] = fm(fm(fm(drescale, fs(t0[0], fm(t0[2], u))), kScaleIdepth), fxl);
        J[J_PDD + 1] = fm(fm(fm(drescale, fs(t0[1], fm(t0[2], v))), kScaleIdepth), fyl);
        float cx2 = fm(drescale, fs(fm(R0[6], u), R0[0]));
        float cx3 = fm(fm(fm(fxl, drescale), fs(fm(R0[7], u), R0[1])), L.fyli);
        float cx0 = fm(K0, cx2), cx1 = fm(K1, cx3);
        float cy2 = fm(fm(fm(fyl, drescale), fs(fm(R0[6], v), R0[3])), L.fxli);
        float cy3 = fm(drescale, fs(fm(R0[7], v), R0[4]));
        float cy0 = fm(K0, cy2), cy1 = fm(K1, cy3);
        cx0 = fm(fa(cx0, u), kScaleF); cx1 = fm(cx1, kScaleF); cx2 = fm(fa(cx2, 1.f), kScaleC); cx3 = fm(cx3, kScaleC);
        cy0 = fm(cy0, kScaleF); cy1 = fm(fa(cy1, v), kScaleF); cy2 = fm(cy2, kScaleC); cy3 = fm(fa(cy3, 1.f), kScaleC);
        float* C = J + J_PDC;
        C[0] = cx0; C[1] = cx1; C[2] = cx2; C[3] = cx3; C[4] = cy0; C[5] = cy1; C[6] = cy2; C[7] = cy3;
        float* X = J + J_PDXI;
        X[0] = fm(new_idepth, fxl);
        X[1] = 0.f;
        X[2] = fm(fm(-new_idepth, u), fxl);
        X[3] = fm(fm(-u, v), fxl);
        X[4] = fm(fa(1.f, fm(u, u)), fxl);
        X[5] = fm(-v, fxl);
        X[6] = 0.f;
        X[7] = fm(new_idepth, fyl);
        X[8] = fm(fm(-new_idepth, v), fyl);
        X[9] = fm(-fa(1.f, fm(v, v)), fyl);
        X[10] = fm(fm(u, v), fyl);
        X[11] = fm(u, fyl);
      }
      // pattern index i: projectPoint, 6-argument form (:50-60), and its sample
      const float* K = pc + PC_KRKI;
      const float* Kt = pc + PC_KT;
      const float x = fa(u0, (float)c_pattern[i][0]), y = fa(v0, (float)c_pattern[i][1]);
      const float q0 = fa(fa(fa(fm(K[0], x), fm(K[1], y)), fm(K[2], 1.f)), fm(Kt[0], ids));
      const float q1 = fa(fa(fa(fm(K[3], x), fm(K[4], y)), fm(K[5], 1.f)), fm(Kt[1], ids));
      const float q2 = fa(fa(fa(fm(K[6], x), fm(K[7], y)), fm(K[8], 1.f)), fm(Kt[2], ids));
      const float Ku = fd(q0, q2), Kv = fd(q1, q2);
      float hit[3] = {0.f, 0.f, 0.f};
      bool good = Ku > 1.1f && Kv > 1.1f && Ku < wM3G && Kv < hM3G;
      if (good) {
        interp<3>(L.dI[tg], Ku, Kv, L.w, hit);
        good = isfinite(hit[0]);
      }
      if (__all_sync(gmask, good)) {
        const float col = P.color[(size_t)i * cap + p], wt = P.weights[(size_t)i * cap + p];
        const float residual = fs(hit[0], fa(fm(pc[PC_AFF], col), pc[PC_AFF + 1]));
        const float drdA = fs(col, pc[PC_B0]);
        const Settings& S = L.s;
        float w = __fsqrt_rn(fd(S.outlier_th_sum_component, fa(S.outlier_th_sum_component, fa(fm(hit[1], hit[1]), fm(hit[2], hit[2])))));
        w = fm(0.5f, fa(w, wt));
        float hw = fabsf(residual) < S.huber ? 1.f : fd(S.huber, fabsf(residual));
        const float e = fm(fm(fm(fm(fm(w, w), hw), residual), residual), fs(2.f, hw));
        if (hw < 1) hw = __fsqrt_rn(hw);
        hw = fm(hw, w);
        const float h1 = fm(hit[1], hw), h2 = fm(hit[2], hw);
        const float dh = fm(drdA, hw);
        J[J_RESF + i] = fm(residual, hw);
        J[J_IDX + i] = h1;
        J[J_IDX + 8 + i] = h2;
        J[J_ABF + i] = S.affine_opt_mode_a < 0 ? 0.f : dh;
        J[J_ABF + 8 + i] = S.affine_opt_mode_b < 0 ? 0.f : hw;
        // the twelve serial sums, pattern index 0..7
        float term[12] = {e, fm(h1, h1), fm(h2, h2), fm(h1, h2), fm(dh, h1), fm(dh, h2), fm(hw, h1), fm(hw, h2),
                          fm(fm(fm(drdA, drdA), hw), hw), fm(dh, hw), fm(hw, hw), fm(fm(hw, hw), fa(fm(h1, h1), fm(h2, h2)))};
        float sum[12];
#pragma unroll
        for (int k = 0; k < 12; ++k) sum[k] = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int k = 0; k < 12; ++k) sum[k] = fa(sum[k], __shfl_sync(gmask, term[k], gbase + j));
        if (i == 0) {
          // JIdx2 (00, 10, 10, 11), JabJIdx (00, 10, 01, 11), Jab2 (00, 01, 01, 11), column-major
          J[J_IDX2] = sum[1]; J[J_IDX2 + 1] = sum[3]; J[J_IDX2 + 2] = sum[3]; J[J_IDX2 + 3] = sum[2];
          J[J_ABJIDX] = sum[4]; J[J_ABJIDX + 1] = sum[6]; J[J_ABJIDX + 2] = sum[5]; J[J_ABJIDX + 3] = sum[7];
          J[J_AB2] = sum[8]; J[J_AB2 + 1] = sum[9]; J[J_AB2 + 2] = sum[9]; J[J_AB2 + 3] = sum[10];
        }
        float energyLeft = sum[0];
        nEwo = energyLeft;
        const float th = fmaxf_ref(L.th[hf], L.th[tg]);
        if (energyLeft > th || sum[11] < 2) {
          energyLeft = th;
          ns = RS_OUTLIER;
        } else {
          ns = RS_IN;
        }
        nE = energyLeft;
        ret = (double)energyLeft;
      }
    }
  }
  if (i != 0) return;
  R.new_state[r] = (signed char)ns;
  R.new_energy[r] = nE;
  R.new_energy_wo[r] = nEwo;
  R.center[3 * (size_t)r] = cx; R.center[3 * (size_t)r + 1] = cy; R.center[3 * (size_t)r + 2] = cz;
  R.ret[r] = ret;
  unsigned key = ~0u;
  if (nEwo >= 0 && tg == L.n_frames - 1) {
    key = nEwo == 0.f ? 0u : __float_as_uint(nEwo);
    atomicAdd(n_key, 1u);
  }
  R.key[r] = key;
  if (L.fix) {
    // applyRes(true): a residual OOB on entry stays OOB with its energy
    int st = state;
    if (state != RS_OOB) {
      st = ns;
      R.state[r] = (signed char)ns;
      R.energy[r] = nE;
      R.active[r] = ns == RS_IN;
    }
    R.took[r] = st == RS_IN;
    float relBS = __int_as_float(0x7fc00000);
    if (st == RS_IN) {   // efResidual->isActive(); isNew is always true
      const float* K = pc + PC_KRKI;
      const float* Kt = pc + PC_KT;
      const float u0 = P.u[p], v0 = P.v[p], ids = L.ids[p];
      const float i0 = fa(fa(fm(K[0], u0), fm(K[1], v0)), fm(K[2], 1.f));
      const float i1 = fa(fa(fm(K[3], u0), fm(K[4], v0)), fm(K[5], 1.f));
      const float i2 = fa(fa(fm(K[6], u0), fm(K[7], v0)), fm(K[8], 1.f));
      const float q0 = fa(i0, fm(Kt[0], ids)), q1 = fa(i1, fm(Kt[1], ids)), q2 = fa(i2, fm(Kt[2], ids));
      const float a = fs(fd(i0, i2), fd(q0, q2)), b = fs(fd(i1, i2), fd(q1, q2));
      const float norm = __fsqrt_rn(fa(fm(a, a), fm(b, b)));
      relBS = __double2float_rn(__dmul_rn(0.01, (double)norm));
    }
    R.relbs[r] = relBS;
    R.removed[r] = st != RS_IN;
  }
}

// applyRes_Reductor (FullSystemOptimize.cpp:87-92); active / took: isActiveAndIsGoodNEW and whether takeDataF runs
__global__ void k_apply(int n, signed char* __restrict__ state, float* __restrict__ energy, const signed char* __restrict__ new_state,
                        const float* __restrict__ new_energy, unsigned char* __restrict__ active, unsigned char* __restrict__ took) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  if (state[r] == RS_OOB) { took[r] = 0; return; }
  state[r] = new_state[r];
  energy[r] = new_energy[r];
  active[r] = took[r] = new_state[r] == RS_IN;
}

// the fix branch's per-point part: numGoodResiduals++ and the maxRelBaseline update for every residual whose final state is
// IN, in activeResiduals order (res_of[off[p]..off[p+1]))
__global__ void k_points(int n, const int* __restrict__ off, const int* __restrict__ res_of, const signed char* __restrict__ state,
                         const float* __restrict__ relbs, float* __restrict__ max_rel_baseline, int* __restrict__ num_good) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  float m = max_rel_baseline[p];
  int g = num_good[p];
  for (int k = off[p]; k < off[p + 1]; ++k) {
    const int r = res_of[k];
    if (state[r] != RS_IN) continue;
    if (relbs[r] > m) m = relbs[r];
    g++;
  }
  max_rel_baseline[p] = m;
  num_good[p] = g;
}

// lastEnergyP (a fixed tree over the double returns) and setNewFrameEnergyTH from the sorted candidate keys
__global__ void __launch_bounds__(kFinishThreads) k_finish(int n, const double* __restrict__ ret, const unsigned* __restrict__ sorted,
                                                           const unsigned* __restrict__ n_key, Settings S, double* __restrict__ out_energy,
                                                           float* __restrict__ out_th) {
  __shared__ double sh[kFinishThreads];
  double s = 0.0;
  for (int r = threadIdx.x; r < n; r += kFinishThreads) s = __dadd_rn(s, ret[r]);
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int o = kFinishThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] = __dadd_rn(sh[threadIdx.x], sh[threadIdx.x + o]);
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  *out_energy = sh[0];
  const unsigned cnt = *n_key;
  if (cnt == 0) { *out_th = 12 * 12 * 8; return; }   // 12*12*patternNum
  const int nthIdx = (int)fm(S.frame_energy_th_n, (float)cnt);
  const float nth = __fsqrt_rn(__uint_as_float(sorted[nthIdx]));
  float th = fm(nth, S.fac_median);
  th = fa(fm(26.0f, S.const_weight), fm(th, fs(1.f, S.const_weight)));
  th = fm(th, th);
  th = fm(th, fm(S.overall_energy_th_weight, S.overall_energy_th_weight));
  *out_th = th;
}

class ActiveImpl final : public ActiveIface {
 public:
  ActiveImpl(int w, int h, int cap, const float* settings, int device) : w_(w), h_(h), cap_(cap), device_(device) {
    int nd = 0;
    if (cudaGetDeviceCount(&nd) != cudaSuccess || nd == 0)
      throw Error("tandem_b200: no CUDA device visible - this library has no CPU fallback");
    TDM_CHECK(w >= 10 && h >= 10 && cap >= 1 && cap <= (1 << 21), "bad active-residual set shape");
    TDM_CHECK(settings, "null argument");
    std::memcpy(&s_, settings, sizeof s_);
    TDM_CHECK(s_.frame_energy_th_n >= 0.f && s_.frame_energy_th_n < 1.f, "frame_energy_th_n outside [0, 1)");
    TDM_CUDA(cudaSetDevice(device_));
    const size_t rc = 8ull * cap;
    stream_ = make_stream(0);
    done_ = make_event(cudaEventDisableTiming);
    d_pint_ = make_dev<int>(4ull * (3 * cap + 1));                 // host, num_good, CSR offsets (cap + 1)
    d_pf_ = make_dev<float>(4ull * (2 + 16 + 1) * cap);           // u, v, color 8, weights 8, maxRelBaseline
    d_rint_ = make_dev<int>(4ull * 3 * rc);                        // point, target, CSR list
    d_rs_ = make_dev<signed char>(3 * rc);                          // state, new_state, removed
    d_rf_ = make_dev<float>(4ull * (5 + 3 + kJ) * rc);              // energy, new_energy, new_energy_wo, relbs, spare, centre, J
    d_ret_ = make_dev<double>(8ull * rc);
    d_key_ = make_dev<unsigned>(4ull * 2 * rc + 4);                 // keys, sorted keys, count
    d_in_ = make_dev<float>(4ull * (kFrames * kFrames * kPre + kFrames + 2 * cap));
    h_in_ = make_host<float>(4ull * (kFrames * kFrames * kPre + kFrames + 2 * cap));
    h_load_ = make_host<int>(4ull * (22 * cap + 1 + 3 * rc));   // load()'s staging: 22 words per point, 3 per residual
    d_small_ = make_dev<double>(16);
    h_small_ = make_host<double>(16);
    size_t tb = 0;
    TDM_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, (const unsigned*)nullptr, (unsigned*)nullptr, (int)rc, 0, 32, stream_.get()));
    sort_bytes_ = tb;
    d_sort_ = make_dev<char>(tb + 16);
    acc_.reset(make_acc(cap));
  }
  ~ActiveImpl() override {
    cudaSetDevice(device_);
    cudaStreamSynchronize(stream_.get());
  }

  void load(int n_frames, int n_points, const int* host, const float* u, const float* v, const float* color, const float* weights,
            const float* max_rel_baseline, const int* num_good, int n_res, const int* res_point, const int* res_target) override {
    TDM_CHECK(n_frames >= 2 && n_frames <= kFrames, "n_frames outside 2..8");
    TDM_CHECK(n_points >= 0 && n_points <= cap_, "active-residual set: more points than its capacity");
    TDM_CHECK(n_res >= 0 && (long long)n_res <= 8ll * cap_, "active-residual set: more residuals than its capacity (8 per point)");
    TDM_CHECK(n_points == 0 || (host && u && v && color && weights && max_rel_baseline && num_good), "null argument");
    TDM_CHECK(n_res == 0 || (res_point && res_target), "null argument");
    for (int p = 0; p < n_points; ++p) TDM_CHECK(host[p] >= 0 && host[p] < n_frames, "point host frame outside 0..n_frames-1");
    std::vector<int> off(n_points + 1, 0), list(n_res);
    for (int r = 0; r < n_res; ++r) {
      TDM_CHECK(res_point[r] >= 0 && res_point[r] < n_points, "residual point index outside the loaded points");
      TDM_CHECK(res_target[r] >= 0 && res_target[r] < n_frames, "residual target frame outside 0..n_frames-1");
      TDM_CHECK(res_target[r] != host[res_point[r]], "residual target frame is its point's host");
      off[res_point[r] + 1]++;
    }
    for (int p = 0; p < n_points; ++p) off[p + 1] += off[p];
    {
      std::vector<int> fill(off.begin(), off.end() - 1);
      for (int r = 0; r < n_res; ++r) list[fill[res_point[r]]++] = r;
    }
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));   // h_load_ is free and no earlier call still reads the set
    const size_t cap = cap_, rc = 8ull * cap_, np = n_points, nr = n_res;
    int* pi = d_pint_.get();
    float* pf = d_pf_.get();
    int* ri = d_rint_.get();
    cudaStream_t st = stream_.get();
    // staging (page-locked, 32-bit words): host, num_good, CSR offsets, res_point, res_target, CSR list, u, v, color / weights
    // rows (one per pattern index), maxRelBaseline
    int* hi = h_load_.get();
    int* h_host = hi;
    int* h_good = h_host + np;
    int* h_off = h_good + np;
    int* h_rp = h_off + np + 1;
    int* h_rt = h_rp + nr;
    int* h_list = h_rt + nr;
    float* h_u = reinterpret_cast<float*>(h_list + nr);
    float* h_v = h_u + np;
    float* h_rows = h_v + np;
    float* h_mrb = h_rows + 16 * np;
    if (np > 0) {
      std::memcpy(h_host, host, 4 * np);
      std::memcpy(h_good, num_good, 4 * np);
      std::memcpy(h_u, u, 4 * np);
      std::memcpy(h_v, v, 4 * np);
      std::memcpy(h_mrb, max_rel_baseline, 4 * np);
      // color / weights arrive n x 8; the set keeps one row per pattern index
      for (size_t p = 0; p < np; ++p)
        for (int k = 0; k < 8; ++k) {
          h_rows[k * np + p] = color[8 * p + k];
          h_rows[(8 + k) * np + p] = weights[8 * p + k];
        }
    }
    std::memcpy(h_off, off.data(), 4 * (np + 1));
    if (nr > 0) {
      std::memcpy(h_rp, res_point, 4 * nr);
      std::memcpy(h_rt, res_target, 4 * nr);
      std::memcpy(h_list, list.data(), 4 * nr);
    }
    if (np > 0) {
      TDM_CUDA(cudaMemcpyAsync(pi, h_host, 4 * np, cudaMemcpyHostToDevice, st));
      TDM_CUDA(cudaMemcpyAsync(pi + cap, h_good, 4 * np, cudaMemcpyHostToDevice, st));
      TDM_CUDA(cudaMemcpyAsync(pf, h_u, 4 * np, cudaMemcpyHostToDevice, st));
      TDM_CUDA(cudaMemcpyAsync(pf + cap, h_v, 4 * np, cudaMemcpyHostToDevice, st));
      TDM_CUDA(cudaMemcpy2DAsync(pf + 2 * cap, 4 * cap, h_rows, 4 * np, 4 * np, 16, cudaMemcpyHostToDevice, st));
      TDM_CUDA(cudaMemcpyAsync(pf + 18 * cap, h_mrb, 4 * np, cudaMemcpyHostToDevice, st));
    }
    TDM_CUDA(cudaMemcpyAsync(pi + 2 * cap, h_off, 4 * (np + 1), cudaMemcpyHostToDevice, st));
    if (nr > 0) {
      TDM_CUDA(cudaMemcpyAsync(ri, h_rp, 4 * nr, cudaMemcpyHostToDevice, st));
      TDM_CUDA(cudaMemcpyAsync(ri + rc, h_rt, 4 * nr, cudaMemcpyHostToDevice, st));
      TDM_CUDA(cudaMemcpyAsync(ri + 2 * rc, h_list, 4 * nr, cudaMemcpyHostToDevice, st));
      // resetOOB: state IN, energies 0, new state OUTLIER
      TDM_CUDA(cudaMemsetAsync(d_rs_.get(), RS_IN, nr, st));
      TDM_CUDA(cudaMemsetAsync(d_rs_.get() + rc, RS_OUTLIER, nr, st));
      TDM_CUDA(cudaMemsetAsync(d_rf_.get(), 0, 4 * nr, st));
      TDM_CUDA(cudaMemsetAsync(d_rf_.get() + rc, 0, 4 * nr, st));
    }
    n_frames_ = n_frames; n_points_ = n_points; n_res_ = n_res;
    unique_targets_ = true;
    for (int p = 0; p < n_points && unique_targets_; ++p) {
      unsigned seen = 0;
      for (int k = off[p]; k < off[p + 1]; ++k) {
        const unsigned bit = 1u << res_target[list[k]];
        if (seen & bit) unique_targets_ = false;
        seen |= bit;
      }
    }
    acc_->load(view(), host, st);
    // every later reader runs on the set's stream; the upload has landed when load returns
    TDM_CUDA(cudaStreamSynchronize(st));
  }

  void linearize(const PyramidIface* const* frames, const float* precalc, const float* frame_energy_th, const float* calib4,
                 const float* idepth_scaled, const float* idepth_zero_scaled, int fix, Outputs& o) override {
    const int n = n_frames_;
    TDM_CHECK(n >= 2, "linearize before load");
    TDM_CHECK(frames && precalc && frame_energy_th && calib4, "null argument");
    TDM_CHECK(n_points_ == 0 || (idepth_scaled && idepth_zero_scaled), "null argument");
    for (int f = 0; f < n; ++f) {
      TDM_CHECK(frames[f], "null argument");
      TDM_CHECK(frames[f]->width(0) == w_ && frames[f]->height(0) == h_, "pyramid level 0 is not the set's image size");
      TDM_CHECK(frames[f]->device() == device_, "pyramid and active-residual set live on different devices");
    }
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));   // h_in_ is free
    const size_t cap = cap_, rc = 8ull * cap_;
    const size_t npc = (size_t)n * n * kPre, nin = npc + n + 2ull * n_points_;
    float* hin = h_in_.get();
    std::memcpy(hin, precalc, 4 * npc);
    std::memcpy(hin + npc, frame_energy_th, 4ull * n);
    if (n_points_ > 0) {
      std::memcpy(hin + npc + n, idepth_scaled, 4ull * n_points_);
      std::memcpy(hin + npc + n + n_points_, idepth_zero_scaled, 4ull * n_points_);
    }
    float* din = d_in_.get();
    TDM_CUDA(cudaMemcpyAsync(din, hin, 4 * nin, cudaMemcpyHostToDevice, stream_.get()));
    for (int f = 0; f < n; ++f) TDM_CUDA(cudaStreamWaitEvent(stream_.get(), (cudaEvent_t)frames[f]->ready_event(), 0));

    LinLaunch L{};
    for (int f = 0; f < n; ++f) L.dI[f] = frames[f]->level_dI(0);
    L.pre = din; L.th = din + npc; L.ids = din + npc + n; L.idz = din + npc + n + n_points_;
    L.n_frames = n; L.n_res = n_res_; L.w = w_; L.h = h_; L.cap = cap_; L.fix = fix ? 1 : 0;
    L.fxl = calib4[0]; L.fyl = calib4[1]; L.cxl = calib4[2]; L.cyl = calib4[3];
    L.fxli = 1.0f / L.fxl; L.fyli = 1.0f / L.fyl;   // CalibHessian::setValueScaled (HessianBlocks.h:435-436)
    L.s = s_;
    const int* pi = d_pint_.get();
    float* pf = d_pf_.get();
    Points P{pi, pf, pf + cap, pf + 2 * cap, pf + 10 * cap};
    Residuals R = res_view();
    unsigned* keys = d_key_.get();
    unsigned* sorted = keys + rc;
    unsigned* n_key = keys + 2 * rc;
    TDM_CUDA(cudaMemsetAsync(n_key, 0, 4, stream_.get()));
    if (n_res_ > 0) {
      k_linearize<<<cdiv(8ll * n_res_, kLinThreads), kLinThreads, 0, stream_.get()>>>(L, P, R, n_key);
      TDM_CUDA(cudaGetLastError());
      size_t tb = sort_bytes_;
      TDM_CUDA(cub::DeviceRadixSort::SortKeys(d_sort_.get(), tb, keys, sorted, n_res_, 0, 32, stream_.get()));
      if (fix && n_points_ > 0) {
        k_points<<<cdiv(n_points_, 128), 128, 0, stream_.get()>>>(n_points_, pi + 2 * cap, d_rint_.get() + 2 * rc, R.state, R.relbs,
                                                                  pf + 18 * cap, const_cast<int*>(pi) + cap);
        TDM_CUDA(cudaGetLastError());
      }
    }
    if (fix) acc_->take(view(), stream_.get());   // applyRes(true) took the data of every residual now IN
    double* ds = d_small_.get();
    k_finish<<<1, kFinishThreads, 0, stream_.get()>>>(n_res_, R.ret, sorted, n_key, s_, ds, reinterpret_cast<float*>(ds + 1));
    TDM_CUDA(cudaGetLastError());
    TDM_CUDA(cudaMemcpyAsync(h_small_.get(), ds, 16, cudaMemcpyDeviceToHost, stream_.get()));
    const size_t nr = n_res_;
    auto down = [&](void* dst, const void* src, size_t bytes) {
      if (dst && bytes) TDM_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, stream_.get()));
    };
    down(o.new_state, R.new_state, nr);
    down(o.new_energy, R.new_energy, 4 * nr);
    down(o.new_energy_with_outlier, R.new_energy_wo, 4 * nr);
    down(o.center_projected_to, R.center, 12 * nr);
    down(o.jacobians, R.J, 4ull * kJ * nr);
    if (fix) {
      down(o.state, R.state, nr);
      down(o.removed, R.removed, nr);
      down(o.max_rel_baseline, pf + 18 * cap, 4ull * n_points_);
      down(o.num_good_residuals, pi + cap, 4ull * n_points_);
    }
    // a later build or destroy of a pyramid read here waits for the call
    TDM_CUDA(cudaEventRecord(done_.get(), stream_.get()));
    for (int f = 0; f < n; ++f) frames[f]->wait_for(done_.get());
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    if (o.energy) *o.energy = h_small_.get()[0];
    if (o.new_frame_energy_th) std::memcpy(o.new_frame_energy_th, h_small_.get() + 1, 4);
  }

  void apply_res() override {
    TDM_CUDA(cudaSetDevice(device_));
    if (n_res_ > 0) {
      Residuals R = res_view();
      k_apply<<<cdiv(n_res_, 256), 256, 0, stream_.get()>>>(n_res_, R.state, R.energy, R.new_state, R.new_energy, R.active, R.took);
      TDM_CUDA(cudaGetLastError());
    }
    if (n_frames_ >= 2) acc_->take(view(), stream_.get());
  }

  void accumulate(const AccInputs& in, AccOutputs& o) override {
    TDM_CUDA(cudaSetDevice(device_));
    acc_->accumulate(view(), stream_.get(), in, o);
  }
  void resubstitute(const double* x, float* step) override {
    TDM_CUDA(cudaSetDevice(device_));
    acc_->resubstitute(view(), stream_.get(), x, step);
  }
  void get_accumulators(double* top, int* top_num, double* acc_e, double* acc_eb, double* acc_d, int* d_num, double* hcc,
                        double* bc) override {
    TDM_CUDA(cudaSetDevice(device_));
    acc_->get_accumulators(view(), stream_.get(), top, top_num, acc_e, acc_eb, acc_d, d_num, hcc, bc);
  }

  void get_state(signed char* state, float* energy) override {
    TDM_CUDA(cudaSetDevice(device_));
    Residuals R = res_view();
    if (state && n_res_) TDM_CUDA(cudaMemcpyAsync(state, R.state, n_res_, cudaMemcpyDeviceToHost, stream_.get()));
    if (energy && n_res_) TDM_CUDA(cudaMemcpyAsync(energy, R.energy, 4ull * n_res_, cudaMemcpyDeviceToHost, stream_.get()));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
  }
  const float* device_jacobians() const override { return d_rf_.get() + 8ull * 8 * cap_; }
  int n_frames() const override { return n_frames_; }
  int n_residuals() const override { return n_res_; }
  int device() const override { return device_; }

 private:
  Residuals res_view() const {
    const size_t rc = 8ull * cap_;
    signed char* s = d_rs_.get();
    float* f = d_rf_.get();
    const int* ri = d_rint_.get();
    Residuals R;
    R.point = ri; R.target = ri + rc;
    R.state = s; R.new_state = s + rc; R.removed = reinterpret_cast<unsigned char*>(s + 2 * rc);
    R.energy = f; R.new_energy = f + rc; R.new_energy_wo = f + 2 * rc; R.relbs = f + 3 * rc;
    R.center = f + 5 * rc; R.J = f + 8 * rc;
    R.ret = d_ret_.get();
    R.key = d_key_.get();
    R.active = acc_->active();
    R.took = acc_->took();
    return R;
  }
  ActiveView view() const {
    const size_t cap = cap_, rc = 8ull * cap_;
    ActiveView v;
    v.n_frames = n_frames_; v.n_points = n_points_; v.n_res = n_res_; v.unique_targets = unique_targets_;
    v.host = d_pint_.get(); v.off = d_pint_.get() + 2 * cap; v.res_of = d_rint_.get() + 2 * rc; v.res_target = d_rint_.get() + rc;
    v.J = d_rf_.get() + 8 * rc;
    v.max_rel_baseline = d_pf_.get() + 18 * cap;
    return v;
  }
  int w_, h_, cap_, device_;
  Settings s_;
  int n_frames_ = 0, n_points_ = 0, n_res_ = 0;
  bool unique_targets_ = true;
  size_t sort_bytes_ = 0;
  Stream stream_;
  Event done_;
  DevPtr<int> d_pint_, d_rint_;
  DevPtr<float> d_pf_, d_rf_, d_in_;
  DevPtr<signed char> d_rs_;
  DevPtr<double> d_ret_, d_small_;
  DevPtr<unsigned> d_key_;
  DevPtr<char> d_sort_;
  HostPtr<float> h_in_;
  HostPtr<int> h_load_;
  HostPtr<double> h_small_;
  std::unique_ptr<AccIface> acc_;   // after the buffers: destroyed first
};

}  // namespace

static_assert(sizeof(Settings) == 8 * 4, "tdm_linearize_settings layout");

ActiveIface* make_active(int w, int h, int capacity_points, const float* settings, int device) {
  return new ActiveImpl(w, h, capacity_points, settings, device);
}

}  // namespace tdm
