/* CPU oracle of n8 (TEST INFRASTRUCTURE ONLY): DSO's immature-point constructor and epipolar trace,
 *   ImmaturePoint::ImmaturePoint   tandem/src/FullSystem/ImmaturePoint.cpp:32-61
 *   ImmaturePoint::traceOn         tandem/src/FullSystem/ImmaturePoint.cpp:75-414
 * restated in C with every float expression in the reference's order (and the summation order of the fixed-size products
 * the reference writes with Eigen: k = 0, 1, 2 left to right).  Built with -ffp-contract=off, so each operation is one
 * correctly rounded IEEE operation, as in the __f*_rn kernels of tandem_b200/csrc/immature.cu it checks.  Pinned bit for bit
 * to the reference's own statements by tests/test_trace_cpu.py.
 *
 * One definitional difference: where a sample's 2x2 footprint leaves the w x h image (the reference reads outside its
 * array), the sample counts as a non-finite hit (energy += 1e5 in the search and in the Gauss-Newton steps).
 *
 * Settings (float s[12]): maxPixSearch, trace_stepsize, trace_GNThreshold, trace_extraSlackOnTH, trace_slackInterval,
 * trace_minImprovementFactor, huberTH, outlierTH, outlierTHSumComponent, overallEnergyTHWeight, minTraceTestRadius (int
 * value), trace_GNIterations (int value). */
#include <math.h>
#include <string.h>

enum { IPS_GOOD = 0, IPS_OOB, IPS_OUTLIER, IPS_SKIPPED, IPS_BADCONDITION, IPS_UNINITIALIZED };
static const int pattern[8][2] = {{0, -2}, {-1, -1}, {1, -1}, {-2, 0}, {0, 0}, {2, 0}, {-1, 1}, {0, 2}};   /* staticPattern[8] */

static int inside(float x, float y, int w, int h) {   /* (int)x in 0..w-2 and (int)y in 0..h-2 */
  return x > -1.f && y > -1.f && x < (float)(w - 1) && y < (float)(h - 1);
}

/* getInterpolatedElement33 (globalFuncs.h:75-89); c = 1: getInterpolatedElement31 (:127-140) */
static void interp33(const float* dI, float x, float y, int w, int c, float* out) {
  int ix = (int)x, iy = (int)y;
  float dx = x - ix, dy = y - iy, dxdy = dx * dy;
  const float* bp = dI + 3 * ((long)ix + (long)iy * w);
  float w0 = dxdy, w1 = dy - dxdy, w2 = dx - dxdy, w3 = 1 - dx - dy + dxdy;
  for (int k = 0; k < c; ++k)
    out[k] = w0 * bp[3 * (1 + w) + k] + w1 * bp[3 * w + k] + w2 * bp[3 + k] + w3 * bp[k];
}

/* The constructor for n pixels (u, v) of a host image (level 0, (I, dx, dy) per pixel); keeps the points with a finite
 * energyTH in input order (FullSystem.cpp:1639-1644) and returns their number.  Outputs hold n entries (8n, 4n). */
int trace_oracle_add(int w, int h, const float* dI, const float* s, int n, const int* u, const int* v, const float* type,
                     float* out_u, float* out_v, float* out_type, float* energyTH, float* color, float* weights, float* gradH) {
  (void)h;
  int m = 0;
  for (int i = 0; i < n; ++i) {
    float col[8], wt[8], g[4] = {0, 0, 0, 0};
    int ok = 1;
    for (int idx = 0; idx < 8; ++idx) {
      /* getInterpolatedElement33BiLin (globalFuncs.h:166-188) at integer coordinates */
      float x = (float)(u[i] + pattern[idx][0]), y = (float)(v[i] + pattern[idx][1]);
      int ix = (int)x, iy = (int)y;
      const float* bp = dI + 3 * ((long)ix + (long)iy * w);
      float tl = bp[0], tr = bp[3], bl = bp[3 * w], br = bp[3 * w + 3];
      float dx = x - ix, dy = y - iy;
      float topInt = dx * tr + (1 - dx) * tl;
      float botInt = dx * br + (1 - dx) * bl;
      float leftInt = dy * bl + (1 - dy) * tl;
      float rightInt = dy * br + (1 - dy) * tr;
      float p0 = dx * rightInt + (1 - dx) * leftInt, p1 = rightInt - leftInt, p2 = botInt - topInt;
      col[idx] = p0;
      if (!isfinite(col[idx])) { ok = 0; break; }
      g[0] += p1 * p1; g[1] += p1 * p2; g[2] += p2 * p1; g[3] += p2 * p2;
      wt[idx] = sqrtf(s[8] / (s[8] + (p1 * p1 + p2 * p2)));
    }
    if (!ok) continue;
    float eth = 8 * s[7];
    eth *= s[9] * s[9];
    out_u[m] = (float)u[i]; out_v[m] = (float)v[i]; out_type[m] = type[i]; energyTH[m] = eth;
    memcpy(color + 8 * m, col, sizeof col); memcpy(weights + 8 * m, wt, sizeof wt); memcpy(gradH + 4 * m, g, sizeof g);
    ++m;
  }
  return m;
}

/* traceOn for one point.  gradH row-major (g00, g01, g10, g11).  Returns the statement that returned (1..12, see
 * oracle/trace.py PATHS); *steps receives numSteps after the 99 cap (0 before the search), *oob_read whether a sample left
 * the image. */
static int trace_one(int w, int h, const float* dI, const float* s, const float* K, const float* Kt, const float* aff, float u,
                     float v, const float* color, const float* weights, const float* gH, float energyTH, float* idepth_min,
                     float* idepth_max, float* quality, int* status, float* uv, float* interval, int* steps, int* oob_read) {
  *steps = 0;
  if (*status == IPS_OOB) return 1;
  float maxPixSearch = (float)(w + h) * s[0];
  float pr0 = K[0] * u + K[1] * v + K[2] * 1, pr1 = K[3] * u + K[4] * v + K[5] * 1, pr2 = K[6] * u + K[7] * v + K[8] * 1;
  float pm0 = pr0 + Kt[0] * *idepth_min, pm1 = pr1 + Kt[1] * *idepth_min, pm2 = pr2 + Kt[2] * *idepth_min;
  float uMin = pm0 / pm2, vMin = pm1 / pm2;
  if (!(uMin > 4 && vMin > 4 && uMin < w - 5 && vMin < h - 5)) {
    uv[0] = -1; uv[1] = -1; *interval = 0; *status = IPS_OOB; return 2;
  }
  float dist, uMax, vMax;
  if (isfinite(*idepth_max)) {
    float q0 = pr0 + Kt[0] * *idepth_max, q1 = pr1 + Kt[1] * *idepth_max, q2 = pr2 + Kt[2] * *idepth_max;
    uMax = q0 / q2; vMax = q1 / q2;
    if (!(uMax > 4 && vMax > 4 && uMax < w - 5 && vMax < h - 5)) {
      uv[0] = -1; uv[1] = -1; *interval = 0; *status = IPS_OOB; return 3;
    }
    dist = (uMin - uMax) * (uMin - uMax) + (vMin - vMax) * (vMin - vMax);
    dist = sqrtf(dist);
    if (dist < s[4]) {
      uv[0] = (uMax + uMin) * 0.5f; uv[1] = (vMax + vMin) * 0.5f; *interval = dist; *status = IPS_SKIPPED; return 4;
    }
  } else {
    dist = maxPixSearch;
    float q0 = pr0 + Kt[0] * 0.01f, q1 = pr1 + Kt[1] * 0.01f, q2 = pr2 + Kt[2] * 0.01f;
    uMax = q0 / q2; vMax = q1 / q2;
    float dx = uMax - uMin, dy = vMax - vMin;
    float d = 1.0f / sqrtf(dx * dx + dy * dy);
    uMax = uMin + dist * dx * d;
    vMax = vMin + dist * dy * d;
    if (!(uMax > 4 && vMax > 4 && uMax < w - 5 && vMax < h - 5)) {
      uv[0] = -1; uv[1] = -1; *interval = 0; *status = IPS_OOB; return 5;
    }
  }
  if (!(*idepth_min < 0 || (pm2 > 0.75 && pm2 < 1.5))) {
    uv[0] = -1; uv[1] = -1; *interval = 0; *status = IPS_OOB; return 6;
  }
  float dx = s[1] * (uMax - uMin), dy = s[1] * (vMax - vMin);
  float ta0 = dx * gH[0] + dy * gH[2], ta1 = dx * gH[1] + dy * gH[3];
  float a = ta0 * dx + ta1 * dy;
  float tb0 = dy * gH[0] + (-dx) * gH[2], tb1 = dy * gH[1] + (-dx) * gH[3];
  float b = tb0 * dy + tb1 * (-dx);
  float errorInPixel = 0.2f + 0.2f * (a + b) / a;
  if (errorInPixel * s[5] > dist && isfinite(*idepth_max)) {
    uv[0] = (uMax + uMin) * 0.5f; uv[1] = (vMax + vMin) * 0.5f; *interval = dist; *status = IPS_BADCONDITION; return 7;
  }
  if (errorInPixel > 10) errorInPixel = 10;
  dx /= dist;
  dy /= dist;
  if (dist > maxPixSearch) {
    uMax = uMin + maxPixSearch * dx;
    vMax = vMin + maxPixSearch * dy;
    dist = maxPixSearch;
  }
  int numSteps = 1.9999f + dist / s[1];
  float randShift = uMin * 1000 - floorf(uMin * 1000);
  float ptx = uMin - randShift * dx, pty = vMin - randShift * dy;
  float rp[8][2];
  for (int idx = 0; idx < 8; ++idx) {
    float px = (float)pattern[idx][0], py = (float)pattern[idx][1];
    rp[idx][0] = K[0] * px + K[1] * py;
    rp[idx][1] = K[3] * px + K[4] * py;
  }
  if (!isfinite(dx) || !isfinite(dy)) {
    *interval = 0; uv[0] = -1; uv[1] = -1; *status = IPS_OOB; return 8;
  }
  float errors[100];
  float bestU = 0, bestV = 0, bestEnergy = 1e10f;
  int bestIdx = -1;
  if (numSteps >= 100) numSteps = 99;
  *steps = numSteps;
  const float huber = s[6];
  for (int i = 0; i < numSteps; i++) {
    float energy = 0;
    for (int idx = 0; idx < 8; idx++) {
      float x = ptx + rp[idx][0], y = pty + rp[idx][1], hit;
      if (!inside(x, y, w, h)) { *oob_read = 1; energy += 1e5f; continue; }
      interp33(dI, x, y, w, 1, &hit);
      if (!isfinite(hit)) { energy += 1e5f; continue; }
      float residual = hit - (aff[0] * color[idx] + aff[1]);
      float hw = fabsf(residual) < huber ? 1 : huber / fabsf(residual);
      energy += hw * residual * residual * (2 - hw);
    }
    errors[i] = energy;
    if (energy < bestEnergy) { bestU = ptx; bestV = pty; bestEnergy = energy; bestIdx = i; }
    ptx += dx;
    pty += dy;
  }
  const int radius = (int)s[10];
  float secondBest = 1e10f;
  for (int i = 0; i < numSteps; i++)
    if ((i < bestIdx - radius || i > bestIdx + radius) && errors[i] < secondBest) secondBest = errors[i];
  float newQuality = secondBest / bestEnergy;
  if (newQuality < *quality || numSteps > 10) *quality = newQuality;

  float uBak = bestU, vBak = bestV, gnstepsize = 1, stepBack = 0;
  const int gnIts = (int)s[11];
  if (gnIts > 0) bestEnergy = 1e5f;
  for (int it = 0; it < gnIts; it++) {
    float H = 1, bb = 0, energy = 0;
    for (int idx = 0; idx < 8; idx++) {
      float x = bestU + rp[idx][0], y = bestV + rp[idx][1], hit[3];
      if (!inside(x, y, w, h)) { *oob_read = 1; energy += 1e5f; continue; }
      interp33(dI, x, y, w, 3, hit);
      if (!isfinite(hit[0])) { energy += 1e5f; continue; }
      float residual = hit[0] - (aff[0] * color[idx] + aff[1]);
      float dResdDist = dx * hit[1] + dy * hit[2];
      float hw = fabsf(residual) < huber ? 1 : huber / fabsf(residual);
      H += hw * dResdDist * dResdDist;
      bb += hw * residual * dResdDist;
      energy += weights[idx] * weights[idx] * hw * residual * residual * (2 - hw);
    }
    if (energy > bestEnergy) {
      stepBack *= 0.5f;
      bestU = uBak + stepBack * dx;
      bestV = vBak + stepBack * dy;
    } else {
      float step = -gnstepsize * bb / H;
      if (step < -0.5f) step = -0.5f;
      else if (step > 0.5f) step = 0.5f;
      if (!isfinite(step)) step = 0;
      uBak = bestU;
      vBak = bestV;
      stepBack = step;
      bestU += step * dx;
      bestV += step * dy;
      bestEnergy = energy;
    }
    if (fabsf(stepBack) < s[2]) break;
  }
  if (!(bestEnergy < energyTH * s[3])) {
    *interval = 0; uv[0] = -1; uv[1] = -1;
    if (*status == IPS_OUTLIER) { *status = IPS_OOB; return 9; }
    *status = IPS_OUTLIER; return 10;
  }
  float lo, hi;
  if (dx * dx > dy * dy) {
    lo = (pr2 * (bestU - errorInPixel * dx) - pr0) / (Kt[0] - Kt[2] * (bestU - errorInPixel * dx));
    hi = (pr2 * (bestU + errorInPixel * dx) - pr0) / (Kt[0] - Kt[2] * (bestU + errorInPixel * dx));
  } else {
    lo = (pr2 * (bestV - errorInPixel * dy) - pr1) / (Kt[1] - Kt[2] * (bestV - errorInPixel * dy));
    hi = (pr2 * (bestV + errorInPixel * dy) - pr1) / (Kt[1] - Kt[2] * (bestV + errorInPixel * dy));
  }
  if (lo > hi) { float t = lo; lo = hi; hi = t; }
  *idepth_min = lo;
  *idepth_max = hi;
  if (!isfinite(lo) || !isfinite(hi) || hi < 0) {
    *interval = 0; uv[0] = -1; uv[1] = -1; *status = IPS_OUTLIER; return 11;
  }
  *interval = 2 * errorInPixel;
  uv[0] = bestU; uv[1] = bestV;
  *status = IPS_GOOD;
  return 12;
}

/* One trace of n points of one host into the frame dI (level 0, w x h).  K: KRKi row-major 3x3, Kt 3, aff 2.  State arrays
 * are read and written; uv holds 2n.  path / steps / oob_read (n each) receive the diagnostics of trace_one. */
void trace_oracle_trace(int w, int h, const float* dI, const float* s, const float* K, const float* Kt, const float* aff, int n,
                        const float* u, const float* v, const float* color, const float* weights, const float* gradH,
                        const float* energyTH, float* idepth_min, float* idepth_max, float* quality, int* status, float* uv,
                        float* interval, int* path, int* steps, int* oob_read) {
  for (int i = 0; i < n; ++i) {
    oob_read[i] = 0;
    path[i] = trace_one(w, h, dI, s, K, Kt, aff, u[i], v[i], color + 8 * i, weights + 8 * i, gradH + 4 * i, energyTH[i],
                        idepth_min + i, idepth_max + i, quality + i, status + i, uv + 2 * i, interval + i, steps + i,
                        oob_read + i);
  }
}
