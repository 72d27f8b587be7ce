// n13: the hot part of DSO's EnergyFunctional::solveSystemF (tandem/src/OptimizationBackend/EnergyFunctional.cpp:775-913) over
// the residuals of an ActiveImpl (linearize.cu): takeDataF at every applyRes(true) (EnergyFunctionalStructs.cpp:39-50),
// accumulateAF_MT + accumulateLF_MT + accumulateSCF_MT (AccumulatedTopHessian.cpp:39-238, AccumulatedSCHessian.cpp:34-219) and
// resubstituteF_MT (EnergyFunctional.cpp:263-317).  Every per-residual and per-point float value is the reference's own
// expression, correctly rounded and in its order (__f*_rn, no contraction); oracle/accumulate_oracle.c restates the same
// statements.
//
// Shape (DESIGN.md, n13):
// - k_take: after each apply, the taken Jacobian (a coalesced copy of the 74-float record) and JpJdF of every residual whose
//   new state is IN.
// - k_point: one thread per point walks its residuals in the set's order: the pattern sums JI_r, Jab_r, rr, and the serial
//   float sums bd_accAF, Hdd_accAF, Hcd_accAF; then HdiF, bdSumF, idepth_hessian.
// - k_chunk: the accumulator sums in double.  The points are ordered by host; a CTA takes a fixed range of one host's points,
//   stages 32 of them at a time in shared memory, and each thread owns up to 21 of the host's 5236 accumulator entries (8 x 91
//   top terms, accE, accEB, 64 x 64 accD, accHcc, accbc and the update counts), adding its terms point by point.
// - k_reduce: every entry sums its host's CTA partials in CTA order.  No atomics: the bits depend only on the load.
// - k_stitch: one thread per entry of H_top, b_top, H_sc, b_sc replays the reference's (h, t[, k]) loop and product order.
#include <cstring>
#include <vector>

#include "dso_sample.cuh"
#include "tracker.h"

namespace tdm {

namespace {

constexpr int kF = 8, kJ = 74, kRec = 43, kStage = 32, kAccThreads = 256, kPer = 21;
enum { RS_IN = 0, RS_OOB = 1 };
// Jacobian record (linearize.cu)
enum { J_RESF = 0, J_PDXI = 8, J_PDC = 20, J_PDD = 28, J_IDX = 30, J_ABF = 46, J_IDX2 = 62, J_ABJIDX = 66, J_AB2 = 70 };
// staged (point, target) record: x = [Jpdc[0], Jpdxi[0]], y = [Jpdc[1], Jpdxi[1]], JIdx2 00 01 11, Jab2 00 01 11,
// updateTopRight's TR00 TR10 TR01 TR11 TR02 TR12, Jab_r, rr, JpJdF
enum { R_X = 0, R_Y = 10, R_A = 20, R_B = 21, R_C = 22, R_B00 = 23, R_B01 = 24, R_B11 = 25, R_TR = 26, R_JABR = 32, R_RR = 34,
       R_JPJD = 35 };
// one host's accumulator entries (targets indexed 0..7 whatever n is)
enum { L_TOP = 0, L_NTOP = 728, L_E = 736, L_EB = 992, L_D = 1056, L_ND = 5152, L_HCC = 5216, L_BC = 5232, kLocal = 5236 };
// per-point record of k_point: HdiF, bdSumF, Hcd (accAF + accLF), idepth_hessian
enum { P_HDI = 0, P_BDS = 1, P_HCD = 2, P_IDH = 6, kPt = 8 };
static_assert(kAccThreads * kPer >= kLocal, "entries per thread");

// AccumulatorApprox::update's Data index -> (r, c), c >= r (MatrixAccumulators.h:754-847)
struct TopRC { unsigned char r[55], c[55]; };
__constant__ TopRC c_rc;
// BotRight entries in updateBotRight's order: Jab2(0,0), Jab2(0,1), Jab_r[0], Jab2(1,1), Jab_r[1], rr
__constant__ unsigned char c_br[6] = {R_B00, R_B01, R_JABR, R_B11, R_JABR + 1, R_RR};

// takeDataF for every residual that applyRes(true) just took: the Jacobian record and JpJdF
__global__ void k_take(long long n, const unsigned char* __restrict__ took, const float* __restrict__ J, float* __restrict__ Jt,
                       float* __restrict__ jpjd) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= n * kJ) return;
  const long long r = idx / kJ;
  const int k = (int)(idx - r * kJ);
  if (!took[r]) return;
  Jt[idx] = J[idx];
  if (k >= 8) return;
  const float* R = J + r * kJ;
  const float D0 = R[J_PDD], D1 = R[J_PDD + 1];
  float v;
  if (k < 6) {   // Jpdxi[0][k] * (JIdx2 * Jpdd)[0] + Jpdxi[1][k] * (JIdx2 * Jpdd)[1]
    const float ji0 = fa(fm(R[J_IDX2], D0), fm(R[J_IDX2 + 2], D1)), ji1 = fa(fm(R[J_IDX2 + 1], D0), fm(R[J_IDX2 + 3], D1));
    v = fa(fm(R[J_PDXI + k], ji0), fm(R[J_PDXI + 6 + k], ji1));
  } else {       // (JabJIdx * Jpdd)[k - 6]
    const int i = k - 6;
    v = fa(fm(R[J_ABJIDX + i], D0), fm(R[J_ABJIDX + 2 + i], D1));
  }
  jpjd[r * 8 + k] = v;
}

struct PointLaunch {
  int n_points;
  const int *off, *res_of;
  const signed char* active;
  const float *Jt, *prior, *delta;
  float *rx, *ppt, *mrb;
  int *nact, *n_active;
};

// addPoint<0>'s per-residual pattern sums and per-point sums, addPoint<1>'s zeros, and the per-point head of the SC addPoint
__global__ void k_point(PointLaunch L) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= L.n_points) return;
  float bd = 0.f, hdd = 0.f, hcd[4] = {0.f, 0.f, 0.f, 0.f};
  int na = 0;
  for (int k = L.off[p]; k < L.off[p + 1]; ++k) {
    const int r = L.res_of[k];
    if (!L.active[r]) continue;
    const float* J = L.Jt + (size_t)r * kJ;
    float ji0 = 0.f, ji1 = 0.f, ja0 = 0.f, ja1 = 0.f, rr = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float res = J[J_RESF + i];
      ji0 = fa(ji0, fm(res, J[J_IDX + i]));
      ji1 = fa(ji1, fm(res, J[J_IDX + 8 + i]));
      ja0 = fa(ja0, fm(res, J[J_ABF + i]));
      ja1 = fa(ja1, fm(res, J[J_ABF + 8 + i]));
      rr = fa(rr, fm(res, res));
    }
    float* x = L.rx + (size_t)r * 5;
    x[0] = ji0; x[1] = ji1; x[2] = ja0; x[3] = ja1; x[4] = rr;
    const float D0 = J[J_PDD], D1 = J[J_PDD + 1];
    const float Ji0 = fa(fm(J[J_IDX2], D0), fm(J[J_IDX2 + 2], D1)), Ji1 = fa(fm(J[J_IDX2 + 1], D0), fm(J[J_IDX2 + 3], D1));
    bd = fa(bd, fa(fm(ji0, D0), fm(ji1, D1)));
    hdd = fa(hdd, fa(fm(Ji0, D0), fm(Ji1, D1)));
#pragma unroll
    for (int i = 0; i < 4; ++i) hcd[i] = fa(hcd[i], fa(fm(J[J_PDC + i], Ji0), fm(J[J_PDC + 4 + i], Ji1)));
    na++;
  }
  float* o = L.ppt + (size_t)p * kPt;
  L.nact[p] = na;
  if (na) atomicAdd(L.n_active, na);   // an integer count: the same whatever the order
  if (na == 0) {
    o[P_HDI] = 0.f; o[P_BDS] = 0.f; o[P_IDH] = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) o[P_HCD + i] = 0.f;
    L.mrb[p] = 0.f;
    return;
  }
  const float prior = L.prior[p];
  float H = fa(fa(hdd, 0.f), prior);   // Hdd_accAF + Hdd_accLF + priorF
  if ((double)H < 1e-10) H = (float)1e-10;
  o[P_IDH] = H;
  o[P_HDI] = __double2float_rn(__ddiv_rn(1.0, (double)H));
  o[P_BDS] = fa(fa(bd, 0.f), fm(prior, L.delta[p]));
#pragma unroll
  for (int i = 0; i < 4; ++i) o[P_HCD + i] = fa(hcd[i], 0.f);
}

struct ChunkLaunch {
  const int* chunk;   // per CTA: host, first, end (positions in order)
  const int *order, *off, *res_of, *res_target;
  const signed char* active;
  const float *Jt, *rx, *jpjd, *ppt;
  const int* nact;
  double* partial;    // per CTA kLocal
};

// one accumulator entry's term for one staged point; 0 when the point adds nothing to it
__device__ __forceinline__ double entry_term(int e, const float (*rec)[kRec], unsigned mask, const float* pf) {
  if (e < L_NTOP) {
    const int t = e / 91, k = e - 91 * t;
    if (!(mask >> t & 1)) return 0.0;
    const float* R = rec[t];
    if (k < 55) {   // update: a*x[c]*x[r] + c*y[c]*y[r] + b*(x[c]*y[r] + y[c]*x[r])
      const int r = c_rc.r[k], c = c_rc.c[k];
      const float xc = R[R_X + c], xr = R[R_X + r], yc = R[R_Y + c], yr = R[R_Y + r];
      return (double)fa(fa(fm(fm(R[R_A], xc), xr), fm(fm(R[R_C], yc), yr)), fm(R[R_B], fa(fm(xc, yr), fm(yc, xr))));
    }
    if (k < 85) {   // updateTopRight: x[r]*TR0c + y[r]*TR1c
      const int q = k - 55, r = q / 3, c = q - 3 * r;
      return (double)fa(fm(R[R_X + r], R[R_TR + 2 * c]), fm(R[R_Y + r], R[R_TR + 2 * c + 1]));
    }
    return (double)R[c_br[k - 85]];
  }
  if (e < L_E) return (mask >> (e - L_NTOP) & 1) ? 1.0 : 0.0;
  if (e < L_EB) {   // accE: (HdiF * JpJdF[i]) * Hcd[j]
    const int q = e - L_E, t = q >> 5, i = (q & 31) >> 2, j = q & 3;
    if (!(mask >> t & 1)) return 0.0;
    return (double)fm(fm(pf[P_HDI], rec[t][R_JPJD + i]), pf[P_HCD + j]);
  }
  if (e < L_D) {    // accEB: (HdiF * bdSumF) * JpJdF[i]
    const int q = e - L_EB, t = q >> 3, i = q & 7;
    if (!(mask >> t & 1)) return 0.0;
    return (double)fm(fm(pf[P_HDI], pf[P_BDS]), rec[t][R_JPJD + i]);
  }
  if (e < L_ND) {   // accD[t1][t2]: (HdiF * JpJdF_t1[i]) * JpJdF_t2[j]
    const int q = e - L_D, t1 = q >> 9, t2 = (q >> 6) & 7, i = (q >> 3) & 7, j = q & 7;
    if (!(mask >> t1 & 1) || !(mask >> t2 & 1)) return 0.0;
    return (double)fm(fm(pf[P_HDI], rec[t1][R_JPJD + i]), rec[t2][R_JPJD + j]);
  }
  if (e < L_HCC) {
    const int q = e - L_ND;
    return ((mask >> (q >> 3) & 1) && (mask >> (q & 7) & 1)) ? 1.0 : 0.0;
  }
  if (!mask) return 0.0;
  if (e < L_BC) {   // accHcc: (HdiF * Hcd[i]) * Hcd[j]
    const int q = e - L_HCC;
    return (double)fm(fm(pf[P_HDI], pf[P_HCD + (q >> 2)]), pf[P_HCD + (q & 3)]);
  }
  return (double)fm(fm(pf[P_BDS], pf[P_HDI]), pf[P_HCD + (e - L_BC)]);   // accbc: (bdSumF * HdiF) * Hcd[i]
}

__global__ void __launch_bounds__(kAccThreads) k_chunk(ChunkLaunch L) {
  __shared__ float rec[kStage][kF][kRec];
  __shared__ float pf[kStage][kPt];
  __shared__ unsigned mask[kStage];
  const int* ch = L.chunk + 3 * blockIdx.x;
  const int first = ch[1], end = ch[2];
  double acc[kPer];
#pragma unroll
  for (int j = 0; j < kPer; ++j) acc[j] = 0.0;
  for (int base = first; base < end; base += kStage) {
    const int ns = min(kStage, end - base);
    if (threadIdx.x < ns) {
      const int p = L.order[base + threadIdx.x];
      unsigned m = 0;
      if (L.nact[p])
        for (int k = L.off[p]; k < L.off[p + 1]; ++k)
          if (L.active[L.res_of[k]]) m |= 1u << L.res_target[L.res_of[k]];
      mask[threadIdx.x] = m;
#pragma unroll
      for (int i = 0; i < kPt; ++i) pf[threadIdx.x][i] = L.ppt[(size_t)p * kPt + i];
    }
    for (int idx = threadIdx.x; idx < ns * kF; idx += kAccThreads) {
      const int s = idx / kF, p = L.order[base + s];
      int r = -1;
      for (int k = L.off[p]; k < L.off[p + 1]; ++k) {
        const int q = L.res_of[k];
        if (L.active[q] && L.res_target[q] == idx % kF) r = q;
      }
      if (r < 0) continue;
      float* R = rec[s][idx % kF];
      const float* J = L.Jt + (size_t)r * kJ;
      const float* x = L.rx + (size_t)r * 5;
#pragma unroll
      for (int i = 0; i < 4; ++i) { R[R_X + i] = J[J_PDC + i]; R[R_Y + i] = J[J_PDC + 4 + i]; }
#pragma unroll
      for (int i = 0; i < 6; ++i) { R[R_X + 4 + i] = J[J_PDXI + i]; R[R_Y + 4 + i] = J[J_PDXI + 6 + i]; }
      R[R_A] = J[J_IDX2]; R[R_B] = J[J_IDX2 + 2]; R[R_C] = J[J_IDX2 + 3];
      R[R_B00] = J[J_AB2]; R[R_B01] = J[J_AB2 + 2]; R[R_B11] = J[J_AB2 + 3];
      R[R_TR] = J[J_ABJIDX]; R[R_TR + 1] = J[J_ABJIDX + 2]; R[R_TR + 2] = J[J_ABJIDX + 1]; R[R_TR + 3] = J[J_ABJIDX + 3];
      R[R_TR + 4] = x[0]; R[R_TR + 5] = x[1];
      R[R_JABR] = x[2]; R[R_JABR + 1] = x[3]; R[R_RR] = x[4];
#pragma unroll
      for (int i = 0; i < 8; ++i) R[R_JPJD + i] = L.jpjd[(size_t)r * 8 + i];
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int e = threadIdx.x + j * kAccThreads;
      if (e < kLocal)
        for (int s = 0; s < ns; ++s) acc[j] = __dadd_rn(acc[j], entry_term(e, rec[s], mask[s], pf[s]));
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < kPer; ++j) {
    const int e = threadIdx.x + j * kAccThreads;
    if (e < kLocal) L.partial[(size_t)blockIdx.x * kLocal + e] = acc[j];
  }
}

// global raw layout (doubles): top [h + n t][91], accE [h + n t][32], accEB [h + n t][8], accD [h + n t1 + n^2 t2][64],
// accHcc [16], accbc [4]; counts (ints): top [h + n t], accD [h + n t1 + n^2 t2]
struct RawLayout {
  int n;
  __host__ __device__ long long top() const { return 0; }
  __host__ __device__ long long e() const { return 91ll * n * n; }
  __host__ __device__ long long eb() const { return e() + 32ll * n * n; }
  __host__ __device__ long long d() const { return eb() + 8ll * n * n; }
  __host__ __device__ long long hcc() const { return d() + 64ll * n * n * n; }
  __host__ __device__ long long bc() const { return hcc() + 16; }
  __host__ __device__ long long size() const { return bc() + 4; }
  __host__ __device__ long long nums() const { return (long long)n * n + (long long)n * n * n; }
};

// every raw entry: the sum of its host's CTA partials in CTA order (accHcc / accbc: every CTA's)
__global__ void k_reduce(RawLayout G, int n_chunks, const int* __restrict__ hchunk /* n + 1 */, const double* __restrict__ partial,
                         double* __restrict__ raw, int* __restrict__ num) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const int n = G.n, n2 = n * n;
  int h = -1, le = 0;
  bool is_num = false;
  long long out = idx;
  if (idx < G.e()) { const int a = (int)(idx / 91), k = (int)(idx % 91); h = a % n; le = L_TOP + 91 * (a / n) + k; }
  else if (idx < G.eb()) { const long long q = idx - G.e(); const int a = (int)(q / 32); h = a % n; le = L_E + 32 * (a / n) + (int)(q % 32); }
  else if (idx < G.d()) { const long long q = idx - G.eb(); const int a = (int)(q / 8); h = a % n; le = L_EB + 8 * (a / n) + (int)(q % 8); }
  else if (idx < G.hcc()) {
    const long long q = idx - G.d();
    const int a = (int)(q / 64), t1 = (a / n) % n, t2 = a / n2;
    h = a % n; le = L_D + 64 * (8 * t1 + t2) + (int)(q % 64);
  } else if (idx < G.bc()) { le = L_HCC + (int)(idx - G.hcc()); }
  else if (idx < G.size()) { le = L_BC + (int)(idx - G.bc()); }
  else if (idx < G.size() + n2) { const int a = (int)(idx - G.size()); h = a % n; le = L_NTOP + a / n; is_num = true; out = a; }
  else if (idx < G.size() + G.nums()) {
    const int a = (int)(idx - G.size() - n2), t1 = (a / n) % n, t2 = a / n2;
    h = a % n; le = L_ND + 8 * t1 + t2; is_num = true; out = n2 + a;
  } else return;
  const int c0 = h < 0 ? 0 : hchunk[h], c1 = h < 0 ? n_chunks : hchunk[h + 1];
  double s = 0.0;
  for (int c = c0; c < c1; ++c) s = __dadd_rn(s, partial[(size_t)c * kLocal + le]);
  if (is_num) num[out] = (int)s;
  else raw[out] = s;
}

struct StitchLaunch {
  RawLayout G;
  const double *raw, *adH, *adT, *fprior, *fdelta, *cprior;
  const int* num;
  const float* cdelta;
  double *H_top, *b_top, *H_sc, *b_sc;
};

// accH(r, c) of one pair: 0 + the raw top sums (AccumulatorApprox::finish's layout)
__device__ __forceinline__ double accH(const double* top, int r, int c) {
  if (r > c) { const int t = r; r = c; c = t; }
  double v;
  if (c < 10) v = top[r * 10 - r * (r - 1) / 2 + (c - r)];
  else if (r < 10) v = top[55 + 3 * r + (c - 10)];
  else v = top[85 + (r == 10 ? (c - 10) : r == 11 ? 3 + (c - 11) : 5)];
  return __dadd_rn(0.0, v);
}
// (A * B * C^T)(i, j) for 8x8 row-major A, C and B given by a functor: the inner product first, each sum in k order
template <class B>
__device__ __forceinline__ double triple(const double* A, B b, const double* C, int i, int j) {
  double s = 0.0;
#pragma unroll
  for (int m = 0; m < 8; ++m) {
    double t = __dmul_rn(A[i * 8], b(0, m));
#pragma unroll
    for (int k = 1; k < 8; ++k) t = __dadd_rn(t, __dmul_rn(A[i * 8 + k], b(k, m)));
    s = m == 0 ? __dmul_rn(t, C[j * 8]) : __dadd_rn(s, __dmul_rn(t, C[j * 8 + m]));
  }
  return s;
}
template <class B>
__device__ __forceinline__ double matvec(const double* A, B b, int i) {
  double s = __dmul_rn(A[i * 8], b(0));
#pragma unroll
  for (int k = 1; k < 8; ++k) s = __dadd_rn(s, __dmul_rn(A[i * 8 + k], b(k)));
  return s;
}

// the top stitch before the transposed copies: H(row, col) with row a frame row, or both calib; b(row)
__device__ double top_pre(const StitchLaunch& S, int row, int col) {
  const int n = S.G.n;
  double v = 0.0;
  for (int k = 0; k < n * n; ++k) {
    const int h = k % n, t = k / n;
    if (!S.num[k]) continue;
    const double* top = S.raw + 91ll * k;
    const double *aH = S.adH + 64 * k, *aT = S.adT + 64 * k;
    auto H88 = [&](int r, int c) { return accH(top, 4 + r, 4 + c); };
    if (row < 4) {   // topLeftCorner += accH(0:4, 0:4), b.head += accH(0:4, 12)
      v = __dadd_rn(v, col < 0 ? accH(top, row, 12) : accH(top, row, col));
      continue;
    }
    const int R = (row - 4) >> 3, i = (row - 4) & 7;
    if (col < 0) {   // b.segment(h) += adHost * accH(4:12, 12); b.segment(t) += adTarget * ...
      auto bv = [&](int m) { return accH(top, 4 + m, 12); };
      if (R == h) v = __dadd_rn(v, matvec(aH, bv, i));
      if (R == t) v = __dadd_rn(v, matvec(aT, bv, i));
      continue;
    }
    if (col < 4) {   // block(h, calib) += adHost * accH(4:12, 0:4); block(t, calib) += adTarget * ...
      auto cv = [&](int m) { return accH(top, 4 + m, col); };
      if (R == h) v = __dadd_rn(v, matvec(aH, cv, i));
      if (R == t) v = __dadd_rn(v, matvec(aT, cv, i));
      continue;
    }
    const int C = (col - 4) >> 3, j = (col - 4) & 7;
    if (R == h && C == h) v = __dadd_rn(v, triple(aH, H88, aH, i, j));
    if (R == t && C == t) v = __dadd_rn(v, triple(aT, H88, aT, i, j));
    if (R == h && C == t) v = __dadd_rn(v, triple(aH, H88, aT, i, j));
  }
  return v;
}

// the SC stitch (stitchDoubleInternal, one thread's order) before the transposed calib copy
__device__ double sc_pre(const StitchLaunch& S, int row, int col) {
  const int n = S.G.n, n2 = n * n;
  if (row < 4) return __dadd_rn(0.0, col < 0 ? S.raw[S.G.bc() + row] : S.raw[S.G.hcc() + 4 * row + col]);
  const int R = (row - 4) >> 3, r = (row - 4) & 7;
  double v = 0.0;
  for (int ij = 0; ij < n2; ++ij) {
    const int i = ij % n, j = ij / n;
    const double *aHij = S.adH + 64 * ij, *aTij = S.adT + 64 * ij;
    if (col < 4) {   // Hpc = 0 + accE, bp = 0 + accEB
      if (col < 0) {
        auto bp = [&](int m) { return __dadd_rn(0.0, S.raw[S.G.eb() + 8ll * ij + m]); };
        if (R == i) v = __dadd_rn(v, matvec(aHij, bp, r));
        if (R == j) v = __dadd_rn(v, matvec(aTij, bp, r));
      } else {
        auto hp = [&](int m) { return __dadd_rn(0.0, S.raw[S.G.e() + 32ll * ij + 4 * m + col]); };
        if (R == i) v = __dadd_rn(v, matvec(aHij, hp, r));
        if (R == j) v = __dadd_rn(v, matvec(aTij, hp, r));
      }
      continue;
    }
    const int C = (col - 4) >> 3, c = (col - 4) & 7;
    if (R != i && R != j) continue;
    for (int kk = 0; kk < n; ++kk) {
      const bool s1 = R == i && C == i, s2 = R == j && C == kk, s3 = R == j && C == i, s4 = R == i && C == kk;
      if (!(s1 || s2 || s3 || s4)) continue;
      const long long ijk = ij + (long long)kk * n2;
      const double* D = S.raw + S.G.d() + 64 * ijk;
      const bool has = S.num[n2 + ijk] != 0;
      auto dm = [&](int a, int b) { return has ? __dadd_rn(0.0, D[8 * a + b]) : 0.0; };
      const int ik = i + n * kk;
      const double *aHik = S.adH + 64 * ik, *aTik = S.adT + 64 * ik;
      if (s1) v = __dadd_rn(v, triple(aHij, dm, aHik, r, c));
      if (s2) v = __dadd_rn(v, triple(aTij, dm, aTik, r, c));
      if (s3) v = __dadd_rn(v, triple(aTij, dm, aHik, r, c));
      if (s4) v = __dadd_rn(v, triple(aHij, dm, aTik, r, c));
    }
  }
  return v;
}

// blockIdx.y: 0 H_top, 1 b_top, 2 H_sc, 3 b_sc
__global__ void k_stitch(StitchLaunch S) {
  const int dim = 8 * S.G.n + 4;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x, which = blockIdx.y;
  const bool vec = which & 1;
  if (idx >= (vec ? dim : dim * dim)) return;
  const int row = vec ? idx : idx / dim, col = vec ? -1 : idx % dim;
  if (which == 0) {
    double a;
    if (row >= 4 && col >= 4) {
      const int R = (row - 4) >> 3, C = (col - 4) >> 3;
      a = R == C ? top_pre(S, row, col) : __dadd_rn(top_pre(S, row, col), top_pre(S, col, row));
    } else {
      a = row < 4 && col >= 4 ? top_pre(S, col, row) : top_pre(S, row, col);
    }
    double l = 0.0;   // HL_top: the priors on the diagonal
    if (row == col) l = __dadd_rn(0.0, row < 4 ? S.cprior[row] : S.fprior[row - 4]);
    S.H_top[idx] = __dadd_rn(a, l);
  } else if (which == 1) {
    const double a = top_pre(S, row, -1);
    const double l = __dadd_rn(0.0, row < 4 ? __dmul_rn(S.cprior[row], (double)S.cdelta[row])
                                            : __dmul_rn(S.fprior[row - 4], S.fdelta[row - 4]));
    S.b_top[idx] = __dadd_rn(a, l);
  } else if (which == 2) {
    S.H_sc[idx] = row < 4 && col >= 4 ? sc_pre(S, col, row) : sc_pre(S, row, col);
  } else {
    S.b_sc[idx] = sc_pre(S, row, -1);
  }
}

// resubstituteF_MT: xAd[h n + t] = xF(h)^T adHostF[h + n t] + xF(t)^T adTargetF[h + n t]
__global__ void k_xad(int n, const double* __restrict__ x, const double* __restrict__ adH, const double* __restrict__ adT,
                      float* __restrict__ xad) {
  const int idx = threadIdx.x;
  if (idx >= n * n * 8) return;
  const int j = idx & 7, a = idx >> 3, h = a / n, t = a % n, ht = h + n * t;
  float s1 = 0.f, s2 = 0.f;
  for (int k = 0; k < 8; ++k) {
    const float ph = fm(__double2float_rn(x[4 + 8 * h + k]), __double2float_rn(adH[64 * ht + 8 * k + j]));
    const float pt = fm(__double2float_rn(x[4 + 8 * t + k]), __double2float_rn(adT[64 * ht + 8 * k + j]));
    s1 = k == 0 ? ph : fa(s1, ph);
    s2 = k == 0 ? pt : fa(s2, pt);
  }
  xad[idx] = fa(s1, s2);
}

struct ResubLaunch {
  int n, n_points;
  const int *off, *res_of, *res_target, *host, *nact;
  const signed char* active;
  const float *ppt, *jpjd, *xad;
  const double* x;
  float* step;
};

// resubstituteFPt
__global__ void k_resub(ResubLaunch L) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= L.n_points) return;
  if (!L.nact[p]) { L.step[p] = 0.f; return; }
  const float* o = L.ppt + (size_t)p * kPt;
  float b = o[P_BDS];
  float d = fm(__double2float_rn(L.x[0]), o[P_HCD]);
  for (int i = 1; i < 4; ++i) d = fa(d, fm(__double2float_rn(L.x[i]), o[P_HCD + i]));
  b = fs(b, d);
  const int h = L.host[p];
  for (int k = L.off[p]; k < L.off[p + 1]; ++k) {
    const int r = L.res_of[k];
    if (!L.active[r]) continue;
    const float* xa = L.xad + 8 * (h * L.n + L.res_target[r]);
    const float* jp = L.jpjd + (size_t)r * 8;
    float s = fm(xa[0], jp[0]);
    for (int i = 1; i < 8; ++i) s = fa(s, fm(xa[i], jp[i]));
    b = fs(b, s);
  }
  L.step[p] = fm(-b, o[P_HDI]);
}

class AccImpl final : public AccIface {
 public:
  AccImpl(int cap) : cap_(cap) {
    const size_t rc = 8ull * cap;
    max_chunks_ = kMaxChunkCtas + kF;
    d_flags_ = make_dev<unsigned char>(2 * rc);                   // active, took
    d_rf_ = make_dev<float>(4ull * (kJ + 8 + 5) * rc);           // taken Jacobians, JpJdF, JI_r / Jab_r / rr
    d_pf_ = make_dev<float>(4ull * ((kPt + 3) * cap + 4 + kF * kF * 8));   // per point, cDeltaF, priorF, deltaF, step, xAd
    d_pi_ = make_dev<int>(4ull * (2 * cap + 3 * max_chunks_ + kF + 2));    // order, nact, chunk table, host chunk starts, n_active
    d_part_ = make_dev<double>(8ull * kLocal * max_chunks_);
    const RawLayout G{kF};
    // the raw sums, then adHost, adTarget, frame priors, cPrior, then H_top, b_top, H_sc, b_sc, then x
    d_raw_ = make_dev<double>(8ull * (G.size() + 2 * 64 * kF * kF + 16 * kF + 4 + 3 * (8 * kF + 4) * (8 * kF + 5)));
    d_num_ = make_dev<int>(4ull * G.nums());
    h_d_ = make_host<double>(8ull * (2 * 64 * kF * kF + 16 * kF + 4 + 2 * (8 * kF + 4) * (8 * kF + 5) + 1));
    h_f_ = make_host<float>(4ull * (4 + 2 * cap));
    h_i_ = make_host<int>(4ull * (cap + 3 * max_chunks_ + kF + 1));
    h_step_ = make_host<float>(4ull * cap);
    TopRC rc2{};
    int q = 0;
    for (int r = 0; r < 10; ++r)
      for (int c = r; c < 10; ++c) { rc2.r[q] = (unsigned char)r; rc2.c[q] = (unsigned char)c; ++q; }
    TDM_CUDA(cudaMemcpyToSymbol(c_rc, &rc2, sizeof rc2));
  }

  unsigned char* active() override { return d_flags_.get(); }
  unsigned char* took() override { return d_flags_.get() + 8ull * cap_; }

  void load(const ActiveView& v, const int* host, cudaStream_t st) override {
    // order the points by host (stable) and cut each host's run into CTA ranges; a range is at least kStage points and there
    // are at most kMaxChunkCtas + one per host of them
    const int np = v.n_points, n = v.n_frames;
    const int per = std::max(kStage, (np + kMaxChunkCtas - 1) / kMaxChunkCtas);
    int* order = h_i_.get();
    int* chunk = order + cap_;
    int* hchunk = chunk + 3 * max_chunks_;
    std::vector<int> cnt(n + 1, 0);
    for (int p = 0; p < np; ++p) cnt[host[p] + 1]++;
    for (int f = 0; f < n; ++f) cnt[f + 1] += cnt[f];
    std::vector<int> fill(cnt.begin(), cnt.end() - 1);
    for (int p = 0; p < np; ++p) order[fill[host[p]]++] = p;
    int nc = 0;
    for (int f = 0; f < n; ++f) {
      hchunk[f] = nc;
      for (int b = cnt[f]; b < cnt[f + 1]; b += per) {
        chunk[3 * nc] = f; chunk[3 * nc + 1] = b; chunk[3 * nc + 2] = std::min(b + per, cnt[f + 1]);
        ++nc;
      }
    }
    hchunk[n] = nc;
    n_chunks_ = nc;
    int* di = d_pi_.get();
    if (np) TDM_CUDA(cudaMemcpyAsync(di, order, 4ull * np, cudaMemcpyHostToDevice, st));
    TDM_CUDA(cudaMemcpyAsync(di + 2 * cap_, chunk, 4ull * (3 * max_chunks_ + kF + 1), cudaMemcpyHostToDevice, st));
    if (v.n_res) TDM_CUDA(cudaMemsetAsync(d_flags_.get(), 0, v.n_res, st));   // nothing active before the first apply
    taken_ = false;
    valid_ = false;
  }

  void take(const ActiveView& v, cudaStream_t st) override {
    if (v.n_res) {
      k_take<<<cdiv(1ll * kJ * v.n_res, 256), 256, 0, st>>>(v.n_res, took(), v.J, d_rf_.get(), jpjd());
      TDM_CUDA(cudaGetLastError());
    }
    taken_ = true;
    valid_ = false;
  }

  void accumulate(const ActiveView& v, cudaStream_t st, const ActiveIface::AccInputs& in, ActiveIface::AccOutputs& o) override {
    const int n = v.n_frames, np = v.n_points, dim = 8 * n + 4;
    TDM_CHECK(n >= 2, "accumulate before load");
    TDM_CHECK(taken_, "accumulate before any apply since load: no taken Jacobians");
    TDM_CHECK(v.unique_targets, "accumulate needs at most one residual per point and target frame");
    TDM_CHECK(in.ad_host && in.ad_target && in.frame_prior && in.frame_delta_prior && in.c_prior && in.c_delta, "null argument");
    TDM_CHECK(np == 0 || (in.point_prior && in.point_delta), "null argument");
    TDM_CUDA(cudaStreamSynchronize(st));   // the staging buffers are free
    const RawLayout G{n};
    // staging: adHost, adTarget, frame prior, delta_prior, cPrior | cDeltaF, priorF, deltaF
    double* hd = h_d_.get();
    const size_t nad = 64ull * n * n;
    std::memcpy(hd, in.ad_host, 8 * nad);
    std::memcpy(hd + nad, in.ad_target, 8 * nad);
    std::memcpy(hd + 2 * nad, in.frame_prior, 64ull * n);
    std::memcpy(hd + 2 * nad + 8 * n, in.frame_delta_prior, 64ull * n);
    std::memcpy(hd + 2 * nad + 16 * n, in.c_prior, 32);
    float* hf = h_f_.get();
    std::memcpy(hf, in.c_delta, 16);
    if (np) {
      std::memcpy(hf + 4, in.point_prior, 4ull * np);
      std::memcpy(hf + 4 + np, in.point_delta, 4ull * np);
    }
    double* din = d_raw_.get() + G.size();   // inputs after the raws
    TDM_CUDA(cudaMemcpyAsync(din, hd, 8 * (2 * nad + 16 * n + 4), cudaMemcpyHostToDevice, st));
    float* pin = d_pf_.get() + (size_t)kPt * cap_;   // cDeltaF, priorF, deltaF
    TDM_CUDA(cudaMemcpyAsync(pin, hf, 4ull * (4 + 2 * np), cudaMemcpyHostToDevice, st));
    int* di = d_pi_.get();
    int* n_active = di + 2 * cap_ + 3 * max_chunks_ + kF + 1;
    TDM_CUDA(cudaMemsetAsync(n_active, 0, 4, st));
    if (np) {
      PointLaunch P{np, v.off, v.res_of, reinterpret_cast<const signed char*>(active()), d_rf_.get(), pin + 4, pin + 4 + np,
                    rx(), d_pf_.get(), v.max_rel_baseline, di + cap_, n_active};
      k_point<<<cdiv(np, 128), 128, 0, st>>>(P);
      TDM_CUDA(cudaGetLastError());
    }
    if (n_chunks_) {
      ChunkLaunch C{di + 2 * cap_, di, v.off, v.res_of, v.res_target, reinterpret_cast<const signed char*>(active()),
                    d_rf_.get(), rx(), jpjd(), d_pf_.get(), di + cap_, d_part_.get()};
      k_chunk<<<n_chunks_, kAccThreads, 0, st>>>(C);
      TDM_CUDA(cudaGetLastError());
    }
    const long long nraw = G.size() + G.nums();
    k_reduce<<<cdiv(nraw, 256), 256, 0, st>>>(G, n_chunks_, di + 2 * cap_ + 3 * max_chunks_, d_part_.get(), d_raw_.get(), d_num_.get());
    TDM_CUDA(cudaGetLastError());
    double* dout = din + 2 * nad + 16 * n + 4;   // H_top, b_top, H_sc, b_sc
    StitchLaunch S{G, d_raw_.get(), din, din + nad, din + 2 * nad, din + 2 * nad + 8 * n, din + 2 * nad + 16 * n, d_num_.get(), pin,
                   dout, dout + dim * dim, dout + dim * dim + dim, dout + 2 * dim * dim + dim};
    k_stitch<<<dim3(cdiv(dim * dim, 128), 4), 128, 0, st>>>(S);
    TDM_CUDA(cudaGetLastError());
    // downloads (through the page-locked staging for the system, straight for the per-point arrays)
    double* hs = hd + 2 * nad + 16 * n + 4;
    TDM_CUDA(cudaMemcpyAsync(hs, dout, 8ull * 2 * (dim * dim + dim), cudaMemcpyDeviceToHost, st));
    TDM_CUDA(cudaMemcpyAsync(hs + 2 * (dim * dim + dim), n_active, 4, cudaMemcpyDeviceToHost, st));
    if (np && o.hdi) TDM_CUDA(cudaMemcpy2DAsync(o.hdi, 4, d_pf_.get() + P_HDI, 4 * kPt, 4, np, cudaMemcpyDeviceToHost, st));
    if (np && o.idepth_hessian)
      TDM_CUDA(cudaMemcpy2DAsync(o.idepth_hessian, 4, d_pf_.get() + P_IDH, 4 * kPt, 4, np, cudaMemcpyDeviceToHost, st));
    TDM_CUDA(cudaStreamSynchronize(st));
    if (o.H_top) std::memcpy(o.H_top, hs, 8ull * dim * dim);
    if (o.b_top) std::memcpy(o.b_top, hs + dim * dim, 8ull * dim);
    if (o.H_sc) std::memcpy(o.H_sc, hs + dim * dim + dim, 8ull * dim * dim);
    if (o.b_sc) std::memcpy(o.b_sc, hs + 2 * dim * dim + dim, 8ull * dim);
    if (o.n_active) std::memcpy(o.n_active, hs + 2 * (dim * dim + dim), 4);
    n_acc_ = n;
    valid_ = true;
  }

  void resubstitute(const ActiveView& v, cudaStream_t st, const double* x, float* step) override {
    TDM_CHECK(valid_, "resubstitute without an accumulate since the last apply or load");
    TDM_CHECK(x && (step || v.n_points == 0), "null argument");
    const int n = n_acc_, dim = 8 * n + 4, np = v.n_points;
    TDM_CUDA(cudaStreamSynchronize(st));
    const RawLayout G{n};
    double* din = d_raw_.get() + G.size();
    const size_t nad = 64ull * n * n;
    double* dx = din + 2 * nad + 16 * n + 4 + 2 * (dim * dim + dim);
    std::memcpy(h_d_.get(), x, 8ull * dim);
    TDM_CUDA(cudaMemcpyAsync(dx, h_d_.get(), 8ull * dim, cudaMemcpyHostToDevice, st));
    float* xad = d_pf_.get() + (size_t)(kPt + 3) * cap_ + 4;
    k_xad<<<1, 512, 0, st>>>(n, dx, din, din + nad, xad);
    TDM_CUDA(cudaGetLastError());
    if (np) {
      ResubLaunch R{n, np, v.off, v.res_of, v.res_target, v.host, d_pi_.get() + cap_, reinterpret_cast<const signed char*>(active()),
                    d_pf_.get(), jpjd(), xad, dx, d_pf_.get() + (size_t)(kPt + 2) * cap_ + 4};
      k_resub<<<cdiv(np, 128), 128, 0, st>>>(R);
      TDM_CUDA(cudaGetLastError());
      TDM_CUDA(cudaMemcpyAsync(h_step_.get(), R.step, 4ull * np, cudaMemcpyDeviceToHost, st));
    }
    TDM_CUDA(cudaStreamSynchronize(st));
    if (np) std::memcpy(step, h_step_.get(), 4ull * np);
  }

  void get_accumulators(const ActiveView& v, cudaStream_t st, double* top, int* top_num, double* acc_e, double* acc_eb, double* acc_d,
                        int* d_num, double* hcc, double* bc) override {
    TDM_CHECK(valid_, "no accumulate since the last apply or load");
    const RawLayout G{n_acc_};
    const int n2 = n_acc_ * n_acc_;
    auto down = [&](void* dst, const void* src, size_t bytes) {
      if (dst && bytes) TDM_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st));
    };
    const double* r = d_raw_.get();
    down(top, r + G.top(), 8 * (G.e() - G.top()));
    down(acc_e, r + G.e(), 8 * (G.eb() - G.e()));
    down(acc_eb, r + G.eb(), 8 * (G.d() - G.eb()));
    down(acc_d, r + G.d(), 8 * (G.hcc() - G.d()));
    down(hcc, r + G.hcc(), 8 * 16);
    down(bc, r + G.bc(), 8 * 4);
    down(top_num, d_num_.get(), 4ull * n2);
    down(d_num, d_num_.get() + n2, 4ull * n2 * n_acc_);
    TDM_CUDA(cudaStreamSynchronize(st));
  }

 private:
  static constexpr int kMaxChunkCtas = 128;
  float* jpjd() const { return d_rf_.get() + 8ull * cap_ * kJ; }
  float* rx() const { return d_rf_.get() + 8ull * cap_ * (kJ + 8); }
  int cap_, max_chunks_ = 0, n_chunks_ = 0, n_acc_ = 0;
  bool taken_ = false, valid_ = false;
  DevPtr<unsigned char> d_flags_;
  DevPtr<float> d_rf_, d_pf_;
  DevPtr<int> d_pi_, d_num_;
  DevPtr<double> d_part_, d_raw_;
  HostPtr<double> h_d_;
  HostPtr<float> h_f_, h_step_;
  HostPtr<int> h_i_;
};

}  // namespace

AccIface* make_acc(int capacity_points) { return new AccImpl(capacity_points); }

}  // namespace tdm
