/* CPU oracle of n12 (TEST INFRASTRUCTURE ONLY): the per-residual part of DSO's windowed bundle adjustment,
 *   FullSystem::linearizeAll, linearizeAll_Reductor, applyRes_Reductor, setNewFrameEnergyTH
 *                                        tandem/src/FullSystem/FullSystemOptimize.cpp:52-210
 *   PointFrameResidual::linearize        tandem/src/FullSystem/Residuals.cpp:78-274
 *   PointFrameResidual::applyRes(true)   tandem/src/FullSystem/Residuals.cpp:306-328
 *   projectPoint (both forms)            tandem/src/FullSystem/ResidualProjections.h:36-87
 * restated in C with every float expression in the reference's order (and the k = 0, 1, 2 summation order of the fixed-size
 * products the reference writes with Eigen).  Built with -ffp-contract=off, so each float operation is one correctly rounded
 * IEEE operation, as in the __f*_rn kernel of tandem_b200/csrc/linearize.cu it checks.  lastEnergyP is summed sequentially
 * in double, as the reference's single-thread branch sums it.  Pinned bit for bit to the reference's own statements by
 * tests/test_linearize_cpu.py.
 *
 * precalc: n_frames x n_frames x 27 floats, [host][target] = PRE_KRKiTll (row-major), PRE_KtTll, PRE_RTll_0 (row-major),
 * PRE_tTll_0, PRE_aff_mode, PRE_b0_mode.  calib4: fxl, fyl, cxl, cyl.  settings8: tdm_linearize_settings.
 * Jacobian record (74 floats): RawResidualJacobian's members in declaration order, the 2x2 matrices column-major. */
#include <math.h>
#include <stdlib.h>
#include <string.h>

enum { IN = 0, OOB = 1, OUTLIER = 2 };   /* ResState, Residuals.h:47 */
static const int pattern[8][2] = {{0, -2}, {-1, -1}, {1, -1}, {-2, 0}, {0, 0}, {2, 0}, {-1, 1}, {0, 2}};   /* staticPattern[8] */
#define SCALE_IDEPTH 1.0f   /* HessianBlocks.h:59-63 */
#define SCALE_F 50.0f
#define SCALE_C 50.0f

typedef struct {
  int w, h, n_frames;
  const float* const* dI;
  const float* precalc;
  const float* frame_th;
  float fxl, fyl, cxl, cyl, fxli, fyli;
  const float* s;   /* huber, outlierTHSumComponent, affineOptModeA, affineOptModeB, frameEnergyTHN, ConstWeight, FacMedian,
                       overallEnergyTHWeight */
} Ctx;

/* the per-residual state of PointFrameResidual (Residuals.h:60-84) and its EFResidual's isActiveAndIsGoodNEW */
typedef struct {
  int* state;
  double* energy;
  int* new_state;
  double* new_energy;
  double* new_energy_wo;
  int* active;
  float* center;   /* 3 per residual */
  float* J;        /* 74 per residual */
} Res;

/* getInterpolatedElement33 (globalFuncs.h:75-89) */
static void interp33(const float* dI, float x, float y, int w, float* out) {
  int ix = (int)x, iy = (int)y;
  float dx = x - ix, dy = y - iy, dxdy = dx * dy;
  const float* bp = dI + 3 * ((long)ix + (long)iy * w);
  for (int k = 0; k < 3; ++k)
    out[k] = dxdy * bp[3 * (1 + w) + k] + (dy - dxdy) * bp[3 * w + k] + (dx - dxdy) * bp[3 + k] + (1 - dx - dy + dxdy) * bp[k];
}

static float max_f(float a, float b) { return a < b ? b : a; }   /* std::max<float> */

/* PointFrameResidual::linearize of residual r (point p of frame hf, target tg) */
static double linearize(const Ctx* c, int hf, int tg, float u_pt, float v_pt, const float* color, const float* weights, float ids,
                        float idz, Res* R, long r) {
  R->new_energy_wo[r] = -1;
  if (R->state[r] == OOB) { R->new_state[r] = OOB; return R->energy[r]; }
  const float* P = c->precalc + 27 * ((long)hf * c->n_frames + tg);
  const float *KRKi = P, *Kt = P + 9, *R0 = P + 12, *t0 = P + 21, *aff = P + 24;
  const float b0 = P[26];
  const float* dIl = c->dI[tg];
  const float wM3G = (float)(c->w - 3), hM3G = (float)(c->h - 3);
  float* J = R->J + 74 * r;
  float energyLeft = 0;
  float d_xi_x[6], d_xi_y[6], d_C_x[4], d_C_y[4], d_d_x, d_d_y;
  {
    /* projectPoint, 13-argument form, dx = dy = 0 */
    float K0 = (u_pt + 0 - c->cxl) * c->fxli, K1 = (v_pt + 0 - c->cyl) * c->fyli, K2 = 1;
    float p0 = R0[0] * K0 + R0[1] * K1 + R0[2] * K2 + t0[0] * idz;
    float p1 = R0[3] * K0 + R0[4] * K1 + R0[5] * K2 + t0[1] * idz;
    float p2 = R0[6] * K0 + R0[7] * K1 + R0[8] * K2 + t0[2] * idz;
    float drescale = 1.0f / p2;
    float new_idepth = idz * drescale;
    if (!(drescale > 0)) { R->new_state[r] = OOB; return R->energy[r]; }
    float u = p0 * drescale, v = p1 * drescale;
    float Ku = u * c->fxl + c->cxl, Kv = v * c->fyl + c->cyl;
    if (!(Ku > 1.1f && Kv > 1.1f && Ku < wM3G && Kv < hM3G)) { R->new_state[r] = OOB; return R->energy[r]; }
    R->center[3 * r] = Ku; R->center[3 * r + 1] = Kv; R->center[3 * r + 2] = new_idepth;
    d_d_x = drescale * (t0[0] - t0[2] * u) * SCALE_IDEPTH * c->fxl;
    d_d_y = drescale * (t0[1] - t0[2] * v) * SCALE_IDEPTH * c->fyl;
    d_C_x[2] = drescale * (R0[6] * u - R0[0]);
    d_C_x[3] = c->fxl * drescale * (R0[7] * u - R0[1]) * c->fyli;
    d_C_x[0] = K0 * d_C_x[2];
    d_C_x[1] = K1 * d_C_x[3];
    d_C_y[2] = c->fyl * drescale * (R0[6] * v - R0[3]) * c->fxli;
    d_C_y[3] = drescale * (R0[7] * v - R0[4]);
    d_C_y[0] = K0 * d_C_y[2];
    d_C_y[1] = K1 * d_C_y[3];
    d_C_x[0] = (d_C_x[0] + u) * SCALE_F;
    d_C_x[1] *= SCALE_F;
    d_C_x[2] = (d_C_x[2] + 1) * SCALE_C;
    d_C_x[3] *= SCALE_C;
    d_C_y[0] *= SCALE_F;
    d_C_y[1] = (d_C_y[1] + v) * SCALE_F;
    d_C_y[2] *= SCALE_C;
    d_C_y[3] = (d_C_y[3] + 1) * SCALE_C;
    d_xi_x[0] = new_idepth * c->fxl;
    d_xi_x[1] = 0;
    d_xi_x[2] = -new_idepth * u * c->fxl;
    d_xi_x[3] = -u * v * c->fxl;
    d_xi_x[4] = (1 + u * u) * c->fxl;
    d_xi_x[5] = -v * c->fxl;
    d_xi_y[0] = 0;
    d_xi_y[1] = new_idepth * c->fyl;
    d_xi_y[2] = -new_idepth * v * c->fyl;
    d_xi_y[3] = -(1 + v * v) * c->fyl;
    d_xi_y[4] = u * v * c->fyl;
    d_xi_y[5] = u * c->fyl;
  }
  memcpy(J + 8, d_xi_x, sizeof d_xi_x);
  memcpy(J + 14, d_xi_y, sizeof d_xi_y);
  memcpy(J + 20, d_C_x, sizeof d_C_x);
  memcpy(J + 24, d_C_y, sizeof d_C_y);
  J[28] = d_d_x;
  J[29] = d_d_y;
  float JIdxJIdx_00 = 0, JIdxJIdx_11 = 0, JIdxJIdx_10 = 0;
  float JabJIdx_00 = 0, JabJIdx_01 = 0, JabJIdx_10 = 0, JabJIdx_11 = 0;
  float JabJab_00 = 0, JabJab_01 = 0, JabJab_11 = 0;
  float wJI2_sum = 0;
  const float huber = c->s[0], sum_comp = c->s[1];
  for (int idx = 0; idx < 8; idx++) {
    /* projectPoint, 6-argument form */
    float x = u_pt + pattern[idx][0], y = v_pt + pattern[idx][1];
    float q0 = KRKi[0] * x + KRKi[1] * y + KRKi[2] * 1 + Kt[0] * ids;
    float q1 = KRKi[3] * x + KRKi[4] * y + KRKi[5] * 1 + Kt[1] * ids;
    float q2 = KRKi[6] * x + KRKi[7] * y + KRKi[8] * 1 + Kt[2] * ids;
    float Ku = q0 / q2, Kv = q1 / q2;
    if (!(Ku > 1.1f && Kv > 1.1f && Ku < wM3G && Kv < hM3G)) { R->new_state[r] = OOB; return R->energy[r]; }
    float hit[3];
    interp33(dIl, Ku, Kv, c->w, hit);
    float residual = hit[0] - (float)(aff[0] * color[idx] + aff[1]);
    float drdA = color[idx] - b0;
    if (!isfinite(hit[0])) { R->new_state[r] = OOB; return R->energy[r]; }
    float w = sqrtf(sum_comp / (sum_comp + (hit[1] * hit[1] + hit[2] * hit[2])));
    w = 0.5f * (w + weights[idx]);
    float hw = fabsf(residual) < huber ? 1 : huber / fabsf(residual);
    energyLeft += w * w * hw * residual * residual * (2 - hw);
    if (hw < 1) hw = sqrtf(hw);
    hw = hw * w;
    hit[1] *= hw;
    hit[2] *= hw;
    J[idx] = residual * hw;
    J[30 + idx] = hit[1];
    J[38 + idx] = hit[2];
    J[46 + idx] = drdA * hw;
    J[54 + idx] = hw;
    JIdxJIdx_00 += hit[1] * hit[1];
    JIdxJIdx_11 += hit[2] * hit[2];
    JIdxJIdx_10 += hit[1] * hit[2];
    JabJIdx_00 += drdA * hw * hit[1];
    JabJIdx_01 += drdA * hw * hit[2];
    JabJIdx_10 += hw * hit[1];
    JabJIdx_11 += hw * hit[2];
    JabJab_00 += drdA * drdA * hw * hw;
    JabJab_01 += drdA * hw * hw;
    JabJab_11 += hw * hw;
    wJI2_sum += hw * hw * (hit[1] * hit[1] + hit[2] * hit[2]);
    if (c->s[2] < 0) J[46 + idx] = 0;
    if (c->s[3] < 0) J[54 + idx] = 0;
  }
  J[62] = JIdxJIdx_00; J[63] = JIdxJIdx_10; J[64] = JIdxJIdx_10; J[65] = JIdxJIdx_11;
  J[66] = JabJIdx_00; J[67] = JabJIdx_10; J[68] = JabJIdx_01; J[69] = JabJIdx_11;
  J[70] = JabJab_00; J[71] = JabJab_01; J[72] = JabJab_01; J[73] = JabJab_11;
  R->new_energy_wo[r] = energyLeft;
  float th = max_f(c->frame_th[hf], c->frame_th[tg]);
  if (energyLeft > th || wJI2_sum < 2) {
    energyLeft = th;
    R->new_state[r] = OUTLIER;
  } else {
    R->new_state[r] = IN;
  }
  R->new_energy[r] = energyLeft;
  return energyLeft;
}

/* applyRes(true); takeDataF is the host's */
static void apply_res(Res* R, long r) {
  if (R->state[r] == OOB) return;
  R->active[r] = R->new_state[r] == IN;
  R->state[r] = R->new_state[r];
  R->energy[r] = R->new_energy[r];
}

static int cmp_float(const void* a, const void* b) {
  float x = *(const float*)a, y = *(const float*)b;
  return x < y ? -1 : x > y ? 1 : 0;
}

/* linearizeAll(fix): returns lastEnergyP; *new_th the newest frame's frameEnergyTH after setNewFrameEnergyTH.  With fix,
 * max_rel_baseline / num_good are updated and removed[r] = !isActive() (the residual goes to toRemove). */
double linearize_all_oracle(int w, int h, int n_frames, const float* const* dI, const float* precalc, const float* frame_th,
                            const float* calib4, const float* settings8, int n_points, const int* host, const float* pu,
                            const float* pv, const float* color, const float* weights, const float* ids, const float* idz,
                            float* max_rel_baseline, int* num_good, int n_res, const int* res_point, const int* res_target, int fix,
                            int* state, double* energy, int* new_state, double* new_energy, double* new_energy_wo, int* active,
                            float* center, float* J, int* removed, float* new_th) {
  Ctx c;
  c.w = w; c.h = h; c.n_frames = n_frames; c.dI = dI; c.precalc = precalc; c.frame_th = frame_th;
  c.fxl = calib4[0]; c.fyl = calib4[1]; c.cxl = calib4[2]; c.cyl = calib4[3];
  c.fxli = 1.0f / c.fxl; c.fyli = 1.0f / c.fyl;   /* CalibHessian::setValueScaled, HessianBlocks.h:435-436 */
  c.s = settings8;
  Res R = {state, energy, new_state, new_energy, new_energy_wo, active, center, J};
  (void)n_points;
  double stats0 = 0;
  for (long k = 0; k < n_res; k++) {
    const int p = res_point[k], hf = host[p], tg = res_target[k];
    stats0 += linearize(&c, hf, tg, pu[p], pv[p], color + 8L * p, weights + 8L * p, ids[p], idz[p], &R, k);
    if (fix) {
      apply_res(&R, k);
      if (active[k]) {
        const float* K = precalc + 27 * ((long)hf * n_frames + tg);
        const float* Kt = K + 9;
        float i0 = K[0] * pu[p] + K[1] * pv[p] + K[2] * 1;
        float i1 = K[3] * pu[p] + K[4] * pv[p] + K[5] * 1;
        float i2 = K[6] * pu[p] + K[7] * pv[p] + K[8] * 1;
        float q0 = i0 + Kt[0] * ids[p], q1 = i1 + Kt[1] * ids[p], q2 = i2 + Kt[2] * ids[p];
        float a = i0 / i2 - q0 / q2, b = i1 / i2 - q1 / q2;
        float relBS = 0.01 * sqrtf(a * a + b * b);
        if (relBS > max_rel_baseline[p]) max_rel_baseline[p] = relBS;
        num_good[p]++;
        removed[k] = 0;
      } else {
        removed[k] = 1;
      }
    }
  }
  /* setNewFrameEnergyTH */
  float* all = (float*)malloc(sizeof(float) * (n_res > 0 ? n_res : 1));
  long m = 0;
  for (long k = 0; k < n_res; k++)
    if (new_energy_wo[k] >= 0 && res_target[k] == n_frames - 1) all[m++] = (float)new_energy_wo[k];
  if (m == 0) {
    *new_th = 12 * 12 * 8;
  } else {
    int nthIdx = settings8[4] * (float)m;
    qsort(all, m, sizeof(float), cmp_float);
    float nthElement = sqrtf(all[nthIdx]);
    float th = nthElement * settings8[6];
    th = 26.0f * settings8[5] + th * (1 - settings8[5]);
    th = th * th;
    th *= settings8[7] * settings8[7];
    *new_th = th;
  }
  free(all);
  return stats0;
}

/* applyRes_Reductor */
void apply_res_oracle(int n_res, int* state, double* energy, const int* new_state, const double* new_energy, int* active) {
  Res R = {state, energy, (int*)new_state, (double*)new_energy, 0, active, 0, 0};
  for (long k = 0; k < n_res; k++) apply_res(&R, k);
}
