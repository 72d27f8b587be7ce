/* CPU oracle of n13 (TEST INFRASTRUCTURE ONLY): the hot part of DSO's EnergyFunctional::solveSystemF,
 *   EFResidual::takeDataF                     tandem/src/OptimizationBackend/EnergyFunctionalStructs.cpp:39-50
 *   AccumulatedTopHessianSSE::addPoint<0/1>   AccumulatedTopHessian.cpp:39-159, stitchDoubleInternal :240-300, and the
 *                                             transposed copies of stitchDoubleMT (AccumulatedTopHessian.h:88-137)
 *   AccumulatedSCHessianSSE::addPoint         AccumulatedSCHessian.cpp:34-77, stitchDoubleInternal :78-150, stitchDoubleMT's
 *                                             copy (AccumulatedSCHessian.h:93-131)
 *   AccumulatorApprox, AccumulatorXX, AccumulatorX   MatrixAccumulators.h:36-237, 595-972
 *   resubstituteF_MT / resubstituteFPt        EnergyFunctional.cpp:263-317
 * restated in C, single-threaded (the MT = false branches), every float expression in the reference's order and the
 * fixed-size products of Eigen summed in k order.  Built with -ffp-contract=off, so each float operation is one correctly
 * rounded IEEE operation, as in the __f*_rn kernels of tandem_b200/csrc/accumulate.cu it checks.
 *
 * The accumulator sums have two modes: TIERS, the reference's float sums with their shiftUp tiers of 1000 updates, and
 * DOUBLE, the sequential double sum of the same float terms that the device is held to (ABS sums their magnitudes).  Points are walked host by host
 * (EnergyFunctional's frames, then each frame's points) and each point's residuals in the set's order.
 *
 * Layouts (as tdm_active_get_accumulators): records [host + n * target]; top: 91 terms (55 of update, 30 of updateTopRight,
 * 6 of updateBotRight); acc_e 8x4; acc_eb 8; acc_d [host + n t1 + n^2 t2] 8x8; hcc 4x4; bc 4.  Jacobian record (74 floats):
 * RawResidualJacobian's members in declaration order, the 2x2 matrices column-major. */
#include <math.h>
#include <stdlib.h>
#include <string.h>

enum { J_RESF = 0, J_PDXI = 8, J_PDC = 20, J_PDD = 28, J_IDX = 30, J_ABF = 46, J_IDX2 = 62, J_ABJIDX = 66, J_AB2 = 70 };
enum { TIERS = 0, DOUBLE = 1, ABS = 2 };   /* ABS: the double sums of |term|, for the summation bound */

/* takeDataF's JpJdF of one Jacobian record */
static void jp_jd(const float* J, float* o) {
  float D0 = J[J_PDD], D1 = J[J_PDD + 1];
  float ji0 = J[J_IDX2] * D0 + J[J_IDX2 + 2] * D1, ji1 = J[J_IDX2 + 1] * D0 + J[J_IDX2 + 3] * D1;   /* JIdx2 * Jpdd */
  for (int i = 0; i < 6; i++) o[i] = J[J_PDXI + i] * ji0 + J[J_PDXI + 6 + i] * ji1;
  o[6] = J[J_ABJIDX] * D0 + J[J_ABJIDX + 2] * D1;   /* JabJIdx * Jpdd */
  o[7] = J[J_ABJIDX + 1] * D0 + J[J_ABJIDX + 3] * D1;
}

void take_data_oracle(int n_res, const float* J, float* jpjd) {
  for (long r = 0; r < n_res; r++) jp_jd(J + 74 * r, jpjd + 8 * r);
}

/* one accumulator of m float entries: the reference's tiers, or a double sum */
typedef struct {
  int m, mode;
  float a[91], a1k[91], a1m[91];
  float numIn1, numIn1k;
  double d[91];
  long num;
} Acc;

static void acc_init(Acc* A, int m, int mode) {
  memset(A, 0, sizeof *A);
  A->m = m;
  A->mode = mode;
}
/* shiftUp: level 0 into 1k after more than 1000 updates, 1k into 1m after more than 1000 of those, or both when forced */
static void acc_shift(Acc* A, int force) {
  if (A->numIn1 > 1000 || force) {
    for (int i = 0; i < A->m; i++) { A->a1k[i] = A->a[i] + A->a1k[i]; A->a[i] = 0; }
    A->numIn1k += A->numIn1;
    A->numIn1 = 0;
  }
  if (A->numIn1k > 1000 || force) {
    for (int i = 0; i < A->m; i++) { A->a1m[i] = A->a1k[i] + A->a1m[i]; A->a1k[i] = 0; }
    A->numIn1k = 0;
  }
}
static void acc_add(Acc* A, int i, float v) {
  if (A->mode == TIERS) A->a[i] += v;
  else if (A->mode == DOUBLE) A->d[i] += (double)v;
  else A->d[i] += fabs((double)v);
}
/* AccumulatorXX::update / AccumulatorX::update: the terms, numIn1++, shiftUp(false) */
static void acc_update_done(Acc* A) {
  A->num++;
  if (A->mode != TIERS) return;
  A->numIn1++;
  acc_shift(A, 0);
}
static void acc_finish(Acc* A, double* out) {
  if (A->mode == TIERS) {
    acc_shift(A, 1);
    for (int i = 0; i < A->m; i++) out[i] = (double)A->a1m[i];
  } else {
    for (int i = 0; i < A->m; i++) out[i] = A->d[i];
  }
}

/* AccumulatorApprox::update + updateBotRight + updateTopRight of one residual (addPoint<0>'s order: update, which shifts,
 * then updateBotRight, then updateTopRight) */
static void approx_update(Acc* A, const float* J, const float* x5) {
  float x[10], y[10];
  for (int i = 0; i < 4; i++) { x[i] = J[J_PDC + i]; y[i] = J[J_PDC + 4 + i]; }
  for (int i = 0; i < 6; i++) { x[4 + i] = J[J_PDXI + i]; y[4 + i] = J[J_PDXI + 6 + i]; }
  const float a = J[J_IDX2], b = J[J_IDX2 + 2], c = J[J_IDX2 + 3];   /* JIdx2(0,0), (0,1), (1,1) */
  int idx = 0;
  for (int r = 0; r < 10; r++)
    for (int q = r; q < 10; q++) acc_add(A, idx++, a * x[q] * x[r] + c * y[q] * y[r] + b * (x[q] * y[r] + y[q] * x[r]));
  A->num++;
  if (A->mode == TIERS) {
    A->numIn1++;
    acc_shift(A, 0);
  }
  const float br[6] = {J[J_AB2], J[J_AB2 + 2], x5[2], J[J_AB2 + 3], x5[3], x5[4]};
  for (int i = 0; i < 6; i++) acc_add(A, 85 + i, br[i]);
  const float TR0[3] = {J[J_ABJIDX], J[J_ABJIDX + 1], x5[0]}, TR1[3] = {J[J_ABJIDX + 2], J[J_ABJIDX + 3], x5[1]};
  for (int r = 0; r < 10; r++)
    for (int q = 0; q < 3; q++) acc_add(A, 55 + 3 * r + q, x[r] * TR0[q] + y[r] * TR1[q]);
}

/* accumulateAF_MT's and accumulateSCF_MT's point walks (accumulateLF_MT's addPoint<1> has no residual to walk: its Hdd, bd,
 * Hcd are 0).  Per point out: hdi, idepth_hessian, bdSumF, Hcd (4).  Returns resInA. */
int accumulate_oracle(int mode, int n, int n_points, const int* host, int n_res, const int* res_point, const int* res_target,
                      const float* Jt, const float* jpjd, const int* active, const float* prior, const float* delta, double* top,
                      int* top_num, double* acc_e, double* acc_eb, double* acc_d, int* d_num, double* hcc, double* bc, float* hdi,
                      float* idh, float* bds, float* hcd_out) {
  const int n2 = n * n, n3 = n2 * n;
  Acc* T = malloc(sizeof(Acc) * n2);
  Acc* E = malloc(sizeof(Acc) * n2);
  Acc* EB = malloc(sizeof(Acc) * n2);
  Acc* D = malloc(sizeof(Acc) * n3);
  Acc* HCC = malloc(sizeof(Acc));
  Acc* BC = malloc(sizeof(Acc));
  for (int k = 0; k < n2; k++) { acc_init(T + k, 91, mode); acc_init(E + k, 32, mode); acc_init(EB + k, 8, mode); }
  for (int k = 0; k < n3; k++) acc_init(D + k, 64, mode);
  acc_init(HCC, 16, mode);
  acc_init(BC, 4, mode);
  /* each point's residuals in the set's order */
  int* off = calloc(n_points + 1, sizeof(int));
  int* list = malloc(sizeof(int) * (n_res > 0 ? n_res : 1));
  for (int r = 0; r < n_res; r++) off[res_point[r] + 1]++;
  for (int p = 0; p < n_points; p++) off[p + 1] += off[p];
  int* fill = malloc(sizeof(int) * (n_points + 1));
  memcpy(fill, off, sizeof(int) * (n_points + 1));
  for (int r = 0; r < n_res; r++) list[fill[res_point[r]]++] = r;
  float* x5 = malloc(sizeof(float) * 5 * (n_res > 0 ? n_res : 1));
  int nres = 0;
  for (int h = 0; h < n; h++)
    for (int p = 0; p < n_points; p++) {
      if (host[p] != h) continue;
      /* addPoint<0> */
      float bd_acc = 0, Hdd_acc = 0, Hcd_acc[4] = {0, 0, 0, 0};
      int ngood = 0;
      for (int k = off[p]; k < off[p + 1]; k++) {
        const int r = list[k];
        if (!active[r]) continue;
        const float* J = Jt + 74L * r;
        float* xr = x5 + 5L * r;
        float JI_r0 = 0, JI_r1 = 0, Jab_r0 = 0, Jab_r1 = 0, rr = 0;
        for (int i = 0; i < 8; i++) {
          const float res = J[J_RESF + i];
          JI_r0 += res * J[J_IDX + i];
          JI_r1 += res * J[J_IDX + 8 + i];
          Jab_r0 += res * J[J_ABF + i];
          Jab_r1 += res * J[J_ABF + 8 + i];
          rr += res * res;
        }
        xr[0] = JI_r0; xr[1] = JI_r1; xr[2] = Jab_r0; xr[3] = Jab_r1; xr[4] = rr;
        approx_update(T + h + n * res_target[r], J, xr);
        const float D0 = J[J_PDD], D1 = J[J_PDD + 1];
        const float Ji0 = J[J_IDX2] * D0 + J[J_IDX2 + 2] * D1, Ji1 = J[J_IDX2 + 1] * D0 + J[J_IDX2 + 3] * D1;
        bd_acc += JI_r0 * D0 + JI_r1 * D1;
        Hdd_acc += Ji0 * D0 + Ji1 * D1;
        for (int i = 0; i < 4; i++) Hcd_acc[i] += J[J_PDC + i] * Ji0 + J[J_PDC + 4 + i] * Ji1;
        nres++;
        ngood++;
      }
      /* SC addPoint */
      float* hc = hcd_out + 4L * p;
      if (ngood == 0) {
        hdi[p] = 0; bds[p] = 0; idh[p] = 0;
        for (int i = 0; i < 4; i++) hc[i] = 0;
        continue;
      }
      float H = Hdd_acc + 0.f + prior[p];
      if (H < 1e-10) H = 1e-10;
      idh[p] = H;
      const float HdiF = 1.0 / H;
      hdi[p] = HdiF;
      float bdSumF = bd_acc + 0.f;
      bdSumF += prior[p] * delta[p];
      bds[p] = bdSumF;
      float Hcd[4];
      for (int i = 0; i < 4; i++) hc[i] = Hcd[i] = Hcd_acc[i] + 0.f;
      for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) acc_add(HCC, 4 * i + j, HdiF * Hcd[i] * Hcd[j]);
      acc_update_done(HCC);
      const float wbc = bdSumF * HdiF;
      for (int i = 0; i < 4; i++) acc_add(BC, i, wbc * Hcd[i]);
      acc_update_done(BC);
      for (int k1 = off[p]; k1 < off[p + 1]; k1++) {
        const int r1 = list[k1];
        if (!active[r1]) continue;
        const int r1ht = h + n * res_target[r1];
        const float* L = jpjd + 8L * r1;
        for (int k2 = off[p]; k2 < off[p + 1]; k2++) {
          const int r2 = list[k2];
          if (!active[r2]) continue;
          Acc* A = D + r1ht + n2 * res_target[r2];
          const float* R = jpjd + 8L * r2;
          for (int i = 0; i < 8; i++)
            for (int j = 0; j < 8; j++) acc_add(A, 8 * i + j, HdiF * L[i] * R[j]);
          acc_update_done(A);
        }
        for (int i = 0; i < 8; i++)
          for (int j = 0; j < 4; j++) acc_add(E + r1ht, 4 * i + j, HdiF * L[i] * Hcd[j]);
        acc_update_done(E + r1ht);
        const float web = HdiF * bdSumF;
        for (int i = 0; i < 8; i++) acc_add(EB + r1ht, i, web * L[i]);
        acc_update_done(EB + r1ht);
      }
    }
  for (int k = 0; k < n2; k++) {
    acc_finish(T + k, top + 91L * k);
    top_num[k] = (int)T[k].num;
    acc_finish(E + k, acc_e + 32L * k);
    acc_finish(EB + k, acc_eb + 8L * k);
  }
  for (int k = 0; k < n3; k++) {
    acc_finish(D + k, acc_d + 64L * k);
    d_num[k] = (int)D[k].num;
  }
  acc_finish(HCC, hcc);
  acc_finish(BC, bc);
  free(T); free(E); free(EB); free(D); free(HCC); free(BC); free(off); free(list); free(fill); free(x5);
  return nres;
}

/* ---- the stitch: fixed-size products, each entry summed in k order ---- */
typedef struct { double v[8][8]; } M88;

static double prod_entry(const double* a, int as, const double* b, int bs, int k) {   /* sum_m a[m * as] * b[m * bs] */
  double s = a[0] * b[0];
  for (int m = 1; m < k; m++) s += a[m * as] * b[m * bs];
  return s;
}
/* A * B * C^T, A and C 8x8 row-major, B 8x8 (rows of stride 8) */
static M88 triple(const double* A, const double* B, const double* C) {
  M88 t, o;
  for (int i = 0; i < 8; i++)
    for (int j = 0; j < 8; j++) t.v[i][j] = prod_entry(A + 8 * i, 1, B + j, 8, 8);
  for (int i = 0; i < 8; i++)
    for (int j = 0; j < 8; j++) o.v[i][j] = prod_entry(&t.v[i][0], 1, C + 8 * j, 1, 8);
  return o;
}

/* accH of one pair: Zero + AccumulatorApprox::finish's symmetric 13x13 */
static void acc_h(const double* top, double H[13][13]) {
  int idx = 0;
  for (int r = 0; r < 10; r++)
    for (int c = r; c < 10; c++) { H[r][c] = H[c][r] = 0.0 + top[idx]; idx++; }
  idx = 55;
  for (int r = 0; r < 10; r++)
    for (int c = 0; c < 3; c++) { H[r][c + 10] = H[c + 10][r] = 0.0 + top[idx]; idx++; }
  H[10][10] = 0.0 + top[85];
  H[10][11] = H[11][10] = 0.0 + top[86];
  H[10][12] = H[12][10] = 0.0 + top[87];
  H[11][11] = 0.0 + top[88];
  H[11][12] = H[12][11] = 0.0 + top[89];
  H[12][12] = 0.0 + top[90];
}

/* H_top = HA_top + HL_top, b_top = bA_top + bL_top, H_sc, b_sc (dim = 8n + 4, row-major) */
void stitch_oracle(int n, const double* top, const int* top_num, const double* acc_e, const double* acc_eb, const double* acc_d,
                   const int* d_num, const double* hcc, const double* bc, const double* adH, const double* adT, const double* fprior,
                   const double* fdelta, const double* cprior, const float* cdelta, double* H_top, double* b_top, double* H_sc,
                   double* b_sc) {
  const int dim = 8 * n + 4, n2 = n * n;
  double* HA = calloc((size_t)dim * dim, sizeof(double));
  double* bA = calloc(dim, sizeof(double));
  double* HL = calloc((size_t)dim * dim, sizeof(double));
  double* bL = calloc(dim, sizeof(double));
#define AT(M, r, c) (M)[(size_t)(r) * dim + (c)]
  /* AccumulatedTopHessianSSE::stitchDoubleInternal, usePrior false (accumulateAF) */
  for (int k = 0; k < n2; k++) {
    const int h = k % n, t = k / n, hIdx = 4 + 8 * h, tIdx = 4 + 8 * t;
    if (top_num[k] == 0) continue;
    double H[13][13];
    acc_h(top + 91L * k, H);
    double H88[64];
    for (int i = 0; i < 8; i++)
      for (int j = 0; j < 8; j++) H88[8 * i + j] = H[4 + i][4 + j];
    const double *aH = adH + 64L * k, *aT = adT + 64L * k;
    M88 m;
    m = triple(aH, H88, aH);
    for (int i = 0; i < 8; i++) for (int j = 0; j < 8; j++) AT(HA, hIdx + i, hIdx + j) += m.v[i][j];
    m = triple(aT, H88, aT);
    for (int i = 0; i < 8; i++) for (int j = 0; j < 8; j++) AT(HA, tIdx + i, tIdx + j) += m.v[i][j];
    m = triple(aH, H88, aT);
    for (int i = 0; i < 8; i++) for (int j = 0; j < 8; j++) AT(HA, hIdx + i, tIdx + j) += m.v[i][j];
    for (int i = 0; i < 8; i++)
      for (int c = 0; c < 4; c++) AT(HA, hIdx + i, c) += prod_entry(aH + 8 * i, 1, &H[4][c], 13, 8);
    for (int i = 0; i < 8; i++)
      for (int c = 0; c < 4; c++) AT(HA, tIdx + i, c) += prod_entry(aT + 8 * i, 1, &H[4][c], 13, 8);
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++) AT(HA, r, c) += H[r][c];
    for (int i = 0; i < 8; i++) bA[hIdx + i] += prod_entry(aH + 8 * i, 1, &H[4][12], 13, 8);
    for (int i = 0; i < 8; i++) bA[tIdx + i] += prod_entry(aT + 8 * i, 1, &H[4][12], 13, 8);
    for (int r = 0; r < 4; r++) bA[r] += H[r][12];
  }
  /* accumulateLF: no residual, so only usePrior */
  for (int i = 0; i < 4; i++) { AT(HL, i, i) += cprior[i]; bL[i] += cprior[i] * (double)cdelta[i]; }
  for (int h = 0; h < n; h++)
    for (int i = 0; i < 8; i++) {
      AT(HL, 4 + 8 * h + i, 4 + 8 * h + i) += fprior[8 * h + i];
      bL[4 + 8 * h + i] += fprior[8 * h + i] * fdelta[8 * h + i];
    }
  /* stitchDoubleMT's transposed copies (HL's are zeros) */
  for (double* M = HA; M; M = M == HA ? HL : NULL)
    for (int h = 0; h < n; h++) {
      const int hIdx = 4 + 8 * h;
      for (int i = 0; i < 8; i++) for (int c = 0; c < 4; c++) AT(M, c, hIdx + i) = AT(M, hIdx + i, c);
      for (int t = h + 1; t < n; t++) {
        const int tIdx = 4 + 8 * t;
        for (int i = 0; i < 8; i++) for (int j = 0; j < 8; j++) AT(M, hIdx + i, tIdx + j) += AT(M, tIdx + j, hIdx + i);
        for (int i = 0; i < 8; i++) for (int j = 0; j < 8; j++) AT(M, tIdx + j, hIdx + i) = AT(M, hIdx + i, tIdx + j);
      }
    }
  for (size_t i = 0; i < (size_t)dim * dim; i++) H_top[i] = HA[i] + HL[i];
  for (int i = 0; i < dim; i++) b_top[i] = bA[i] + bL[i];
  /* AccumulatedSCHessianSSE::stitchDoubleInternal (tid = -1) */
  memset(H_sc, 0, sizeof(double) * dim * dim);
  memset(b_sc, 0, sizeof(double) * dim);
  for (int k = 0; k < n2; k++) {
    const int i = k % n, j = k / n, iIdx = 4 + 8 * i, jIdx = 4 + 8 * j;
    double Hpc[32], bp[8];
    for (int q = 0; q < 32; q++) Hpc[q] = 0.0 + acc_e[32L * k + q];
    for (int q = 0; q < 8; q++) bp[q] = 0.0 + acc_eb[8L * k + q];
    const double *aH = adH + 64L * k, *aT = adT + 64L * k;
    for (int r = 0; r < 8; r++) for (int c = 0; c < 4; c++) AT(H_sc, iIdx + r, c) += prod_entry(aH + 8 * r, 1, Hpc + c, 4, 8);
    for (int r = 0; r < 8; r++) for (int c = 0; c < 4; c++) AT(H_sc, jIdx + r, c) += prod_entry(aT + 8 * r, 1, Hpc + c, 4, 8);
    for (int r = 0; r < 8; r++) b_sc[iIdx + r] += prod_entry(aH + 8 * r, 1, bp, 1, 8);
    for (int r = 0; r < 8; r++) b_sc[jIdx + r] += prod_entry(aT + 8 * r, 1, bp, 1, 8);
    for (int kk = 0; kk < n; kk++) {
      const int kIdx = 4 + 8 * kk, ijk = k + kk * n2, ik = i + n * kk;
      double accDM[64];
      for (int q = 0; q < 64; q++) accDM[q] = 0.0;
      if (d_num[ijk] != 0)
        for (int q = 0; q < 64; q++) accDM[q] += acc_d[64L * ijk + q];
      const double *aHik = adH + 64L * ik, *aTik = adT + 64L * ik;
      M88 m;
      m = triple(aH, accDM, aHik);
      for (int r = 0; r < 8; r++) for (int c = 0; c < 8; c++) AT(H_sc, iIdx + r, iIdx + c) += m.v[r][c];
      m = triple(aT, accDM, aTik);
      for (int r = 0; r < 8; r++) for (int c = 0; c < 8; c++) AT(H_sc, jIdx + r, kIdx + c) += m.v[r][c];
      m = triple(aT, accDM, aHik);
      for (int r = 0; r < 8; r++) for (int c = 0; c < 8; c++) AT(H_sc, jIdx + r, iIdx + c) += m.v[r][c];
      m = triple(aH, accDM, aTik);
      for (int r = 0; r < 8; r++) for (int c = 0; c < 8; c++) AT(H_sc, iIdx + r, kIdx + c) += m.v[r][c];
    }
  }
  for (int r = 0; r < 4; r++) {
    for (int c = 0; c < 4; c++) AT(H_sc, r, c) += hcc[4 * r + c];
    b_sc[r] += bc[r];
  }
  for (int h = 0; h < n; h++)
    for (int i = 0; i < 8; i++)
      for (int c = 0; c < 4; c++) AT(H_sc, c, 4 + 8 * h + i) = AT(H_sc, 4 + 8 * h + i, c);
#undef AT
  free(HA); free(bA); free(HL); free(bL);
}

/* resubstituteF_MT's per-point step */
void resubstitute_oracle(int n, int n_points, const int* host, int n_res, const int* res_point, const int* res_target, const int* active,
                         const float* jpjd, const float* hdi, const float* bds, const float* hcd, const double* adH, const double* adT,
                         const double* x, float* step) {
  float xF[68];
  for (int i = 0; i < 8 * n + 4; i++) xF[i] = (float)x[i];
  float* xAd = malloc(sizeof(float) * 8 * n * n);
  for (int h = 0; h < n; h++)
    for (int t = 0; t < n; t++) {
      const int ht = h + n * t;
      for (int j = 0; j < 8; j++) {
        float s1 = xF[4 + 8 * h] * (float)adH[64 * ht + j], s2 = xF[4 + 8 * t] * (float)adT[64 * ht + j];
        for (int k = 1; k < 8; k++) {
          s1 += xF[4 + 8 * h + k] * (float)adH[64 * ht + 8 * k + j];
          s2 += xF[4 + 8 * t + k] * (float)adT[64 * ht + 8 * k + j];
        }
        xAd[8 * (n * h + t) + j] = s1 + s2;
      }
    }
  for (int p = 0; p < n_points; p++) {
    int ngood = 0;
    for (int r = 0; r < n_res; r++) ngood += res_point[r] == p && active[r];
    if (ngood == 0) { step[p] = 0; continue; }
    float b = bds[p];
    float d = xF[0] * hcd[4 * p];
    for (int i = 1; i < 4; i++) d += xF[i] * hcd[4 * p + i];
    b -= d;
    for (int r = 0; r < n_res; r++) {
      if (res_point[r] != p || !active[r]) continue;
      const float* xa = xAd + 8 * (n * host[p] + res_target[r]);
      const float* jp = jpjd + 8L * r;
      float s = xa[0] * jp[0];
      for (int i = 1; i < 8; i++) s += xa[i] * jp[i];
      b -= s;
    }
    step[p] = -b * hdi[p];
  }
  free(xAd);
}
