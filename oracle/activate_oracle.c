/* CPU oracle of n9 (TEST INFRASTRUCTURE ONLY): DSO's activation solve of one immature point,
 *   FullSystem::optimizeImmaturePoint   tandem/src/FullSystem/FullSystemOptPoint.cpp:51-205
 *   ImmaturePoint::linearizeResidual    tandem/src/FullSystem/ImmaturePoint.cpp:476-543
 *   derive_idepth, projectPoint         tandem/src/FullSystem/ResidualProjections.h:36-87
 * restated in C with every float expression in the reference's order (and the k = 0, 1, 2 summation order of the fixed-size
 * products the reference writes with Eigen).  Built with -ffp-contract=off, so each float operation is one correctly rounded
 * IEEE operation, as in the __f*_rn kernel of tandem_b200/csrc/immature.cu it checks.  The double operations of the
 * reference (the step, the stop test, lambda *= 0.5, the double returned into the float lastEnergy) are written as the
 * reference writes them.  Pinned bit for bit to the reference's own statements by tests/test_activate_cpu.py.
 *
 * Point record (float pt[21]): u, v, energyTH, idepth_min, idepth_max, color[8], weights[8].
 * precalc: n_frames x n_frames x 14 floats, [host][target] = PRE_RTll (row-major 3x3), PRE_tTll, PRE_aff_mode.
 * calib4: fxl, fyl, cxl, cyl. */
#include <math.h>
#include <string.h>

enum { IN = 0, OOB = 1, OUTLIER = 2 };   /* ResState, Residuals.h:47 */
static const int pattern[8][2] = {{0, -2}, {-1, -1}, {1, -1}, {-2, 0}, {0, 0}, {2, 0}, {-1, 1}, {0, 2}};   /* staticPattern[8] */

/* return paths of optimizeImmaturePoint (oracle/activate.py PATHS) */
enum { P_INIT_ENERGY = 1, P_INIT_HDD, P_ITER_HDD, P_ITER_ENERGY, P_IDEPTH, P_MIN_OBS, P_ENERGY_TH, P_ACTIVE };
/* what a candidate's solve went through (oracle/activate.py FLAGS) */
enum {
  F_ACCEPT = 1, F_REJECT = 2, F_SMALL_STEP = 4, F_ITERATIONS_OUT = 8, F_OOB_FIRST = 16, F_OOB_STICKY = 32, F_OOB_LATE = 64,
  F_CLAMP_1000 = 128, F_CLAMP_1 = 256, F_NAN_HIT = 512, F_OOB_PROJECT = 1024
};

typedef struct {
  int state_state, state_NewState;
  double state_energy, state_NewEnergy;
  int target;
} TmpRes;   /* ImmaturePointTemporaryResidual, ImmaturePoint.h:35-43 */

typedef struct {
  int w, h, n_frames;
  const float* const* dI;
  const float* precalc;
  float fxl, fyl, cxl, cyl, fxli, fyli;
  float huber;
} Ctx;

/* getInterpolatedElement33 (globalFuncs.h:75-89) */
static void interp33(const float* dI, float x, float y, int w, float* out) {
  int ix = (int)x, iy = (int)y;
  float dx = x - ix, dy = y - iy, dxdy = dx * dy;
  const float* bp = dI + 3 * ((long)ix + (long)iy * w);
  for (int k = 0; k < 3; ++k)
    out[k] = dxdy * bp[3 * (1 + w) + k] + (dy - dxdy) * bp[3 * w + k] + (dx - dxdy) * bp[3 + k] + (1 - dx - dy + dxdy) * bp[k];
}

/* linearizeResidual for the residual of host `host` to tr->target */
static double linearize(const Ctx* c, int host, const float* pt, float outlierTHSlack, TmpRes* tr, float* Hdd, float* bd,
                        float idepth, int* flags) {
  if (tr->state_state == OOB) { tr->state_NewState = OOB; *flags |= F_OOB_STICKY; return tr->state_energy; }
  const float* P = c->precalc + 14 * ((long)host * c->n_frames + tr->target);
  const float *R = P, *t = P + 9, *aff = P + 12;
  const float* dIl = c->dI[tr->target];
  const float u_pt = pt[0], v_pt = pt[1], energyTH = pt[2];
  const float *color = pt + 5, *weights = pt + 13;
  const float wM3G = (float)(c->w - 3), hM3G = (float)(c->h - 3);
  float energyLeft = 0;
  for (int idx = 0; idx < 8; idx++) {
    int dx = pattern[idx][0], dy = pattern[idx][1];
    /* projectPoint, 5-argument form */
    float K0 = (u_pt + dx - c->cxl) * c->fxli, K1 = (v_pt + dy - c->cyl) * c->fyli, K2 = 1;
    float p0 = R[0] * K0 + R[1] * K1 + R[2] * K2 + t[0] * idepth;
    float p1 = R[3] * K0 + R[4] * K1 + R[5] * K2 + t[1] * idepth;
    float p2 = R[6] * K0 + R[7] * K1 + R[8] * K2 + t[2] * idepth;
    float drescale = 1.0f / p2;
    int ok = drescale > 0;
    float u = 0, v = 0, Ku = 0, Kv = 0;
    if (ok) {
      u = p0 * drescale;
      v = p1 * drescale;
      Ku = u * c->fxl + c->cxl;
      Kv = v * c->fyl + c->cyl;
      ok = Ku > 1.1f && Kv > 1.1f && Ku < wM3G && Kv < hM3G;
    }
    if (!ok) {
      tr->state_NewState = OOB;
      *flags |= F_OOB_PROJECT | (idx > 0 ? F_OOB_LATE : 0);
      return tr->state_energy;
    }
    float hit[3];
    interp33(dIl, Ku, Kv, c->w, hit);
    if (!isfinite(hit[0])) {
      tr->state_NewState = OOB;
      *flags |= F_NAN_HIT | (idx > 0 ? F_OOB_LATE : 0);
      return tr->state_energy;
    }
    float residual = hit[0] - (aff[0] * color[idx] + aff[1]);
    float hw = fabsf(residual) < c->huber ? 1 : c->huber / fabsf(residual);
    energyLeft += weights[idx] * weights[idx] * hw * residual * residual * (2 - hw);
    float dxInterp = hit[1] * c->fxl;
    float dyInterp = hit[2] * c->fyl;
    float d_idepth = (dxInterp * drescale * (t[0] - t[2] * u) + dyInterp * drescale * (t[1] - t[2] * v)) * 1.0f;
    hw *= weights[idx] * weights[idx];
    *Hdd += (hw * d_idepth) * d_idepth;
    *bd += (hw * residual) * d_idepth;
  }
  if (energyLeft > energyTH * outlierTHSlack) {
    energyLeft = energyTH * outlierTHSlack;
    tr->state_NewState = OUTLIER;
    *flags |= outlierTHSlack == 1000 ? F_CLAMP_1000 : F_CLAMP_1;
  } else {
    tr->state_NewState = IN;
  }
  tr->state_NewEnergy = energyLeft;
  return energyLeft;
}

/* optimizeImmaturePoint for one candidate of host frame `host`; res holds n_frames - 1 entries, the targets in frame order.
 * Returns the path (P_*); *idepth receives currentIdepth. */
static int optimize(const Ctx* c, int host, const float* pt, float min_h, int gn_its, int min_obs, TmpRes* res, float* idepth,
                    int* flags) {
  int nres = 0;
  for (int f = 0; f < c->n_frames; ++f) {
    if (f == host) continue;
    res[nres].state_NewEnergy = res[nres].state_energy = 0;
    res[nres].state_NewState = OUTLIER;
    res[nres].state_state = IN;
    res[nres].target = f;
    nres++;
  }
  float lastEnergy = 0;
  float lastHdd = 0;
  float lastbd = 0;
  float currentIdepth = (pt[4] + pt[3]) * 0.5f;
  for (int i = 0; i < nres; i++) {
    lastEnergy += linearize(c, host, pt, 1000, res + i, &lastHdd, &lastbd, currentIdepth, flags);
    if (res[i].state_NewState == OOB) *flags |= F_OOB_FIRST;
    res[i].state_state = res[i].state_NewState;
    res[i].state_energy = res[i].state_NewEnergy;
  }
  *idepth = currentIdepth;
  if (!isfinite(lastEnergy)) return P_INIT_ENERGY;
  if (lastHdd < min_h) return P_INIT_HDD;
  float lambda = 0.1;
  int broke = 0;
  for (int iteration = 0; iteration < gn_its; iteration++) {
    float H = lastHdd;
    H *= 1 + lambda;
    float step = (1.0 / H) * lastbd;
    float newIdepth = currentIdepth - step;
    float newHdd = 0, newbd = 0, newEnergy = 0;
    for (int i = 0; i < nres; i++) newEnergy += linearize(c, host, pt, 1, res + i, &newHdd, &newbd, newIdepth, flags);
    if (!isfinite(lastEnergy)) { *idepth = currentIdepth; return P_ITER_ENERGY; }
    if (newHdd < min_h) { *idepth = currentIdepth; return P_ITER_HDD; }
    if (newEnergy < lastEnergy) {
      currentIdepth = newIdepth;
      lastHdd = newHdd;
      lastbd = newbd;
      lastEnergy = newEnergy;
      for (int i = 0; i < nres; i++) {
        res[i].state_state = res[i].state_NewState;
        res[i].state_energy = res[i].state_NewEnergy;
      }
      lambda *= 0.5;
      *flags |= F_ACCEPT;
    } else {
      lambda *= 5;
      *flags |= F_REJECT;
    }
    if (fabsf(step) < 0.0001 * currentIdepth) { broke = 1; *flags |= F_SMALL_STEP; break; }
  }
  if (!broke && gn_its > 0) *flags |= F_ITERATIONS_OUT;
  *idepth = currentIdepth;
  if (!isfinite(currentIdepth)) return P_IDEPTH;
  int numGoodRes = 0;
  for (int i = 0; i < nres; i++)
    if (res[i].state_state == IN) numGoodRes++;
  if (numGoodRes < min_obs) return P_MIN_OBS;
  if (!isfinite(pt[2])) return P_ENERGY_TH;   /* new PointHessian(point, &Hcalib)->energyTH is the point's */
  return P_ACTIVE;
}

/* Every candidate k (host frame cand_frame[k], point record pts + 21 k).  result: 1 / 0 / -1 as the reference returns a
 * PointHessian / 0 / -1; state, energy, new_state, new_energy: n_cand x n_frames, the host's own column -1 / NaN. */
void activate_oracle(int w, int h, int n_frames, const float* const* dI, const float* precalc, const float* calib4, float huber,
                     float min_h, int gn_its, int min_obs, int n_cand, const int* cand_frame, const float* pts, int* result,
                     float* idepth, int* state, float* energy, int* new_state, float* new_energy, int* path, int* flags) {
  Ctx c;
  c.w = w; c.h = h; c.n_frames = n_frames; c.dI = dI; c.precalc = precalc;
  c.fxl = calib4[0]; c.fyl = calib4[1]; c.cxl = calib4[2]; c.cyl = calib4[3];
  c.fxli = 1.0f / c.fxl; c.fyli = 1.0f / c.fyl;   /* CalibHessian::setValueScaled, HessianBlocks.h:435-436 */
  c.huber = huber;
  for (int k = 0; k < n_cand; ++k) {
    TmpRes res[8];
    flags[k] = 0;
    path[k] = optimize(&c, cand_frame[k], pts + 21L * k, min_h, gn_its, min_obs, res, idepth + k, flags + k);
    result[k] = path[k] == P_ACTIVE ? 1 : path[k] <= P_ITER_ENERGY ? 0 : -1;
    for (int f = 0, i = 0; f < n_frames; ++f) {
      long o = (long)k * n_frames + f;
      if (f == cand_frame[k]) { state[o] = new_state[o] = -1; energy[o] = new_energy[o] = NAN; continue; }
      state[o] = res[i].state_state; new_state[o] = res[i].state_NewState;
      energy[o] = (float)res[i].state_energy; new_energy[o] = (float)res[i].state_NewEnergy;
      ++i;
    }
  }
}
