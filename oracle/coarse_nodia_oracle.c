/* ORACLE (test infrastructure - never linked into, or called by, the product library).
 *
 * Plain-C restatement of the rest of CoarseTracker::makeCoarseDepthL0's level-0 output (tandem/src/FullSystem/
 * CoarseTracker.cpp:150-218) that oracle/coarse_ref_oracle.c leaves out: the undilated cloud pc_u/v/idepth/color_nodia and
 * pc_n_nodia.  It is not a debug-only output: FullSystem::deliverDrFrame (FullSystem.cpp:1175-1180) takes every MVSNet
 * window's depth range from it through get_idepth_quantile (tandem/src/tandem/tandem_backend.cpp:354-361), restated here as
 * idepth_quantile_oracle.  Still left out: depth_rel_var and the nodia image (only the debug dumps saveKFDepthMap /
 * saveNKFDepthMap read them).
 * PINNED: oracle/ref_build_coarse_nodia.mk cuts the reference's own makeCoarseDepthL0 body and get_idepth_quantile out of the
 * files where they lie and compiles them, unmodified, in the harness oracle/ref_wrap_coarse_nodia.cpp (pc_*_nodia kept across
 * keyframes); tests/test_coarse_nodia_cpu.py compares this restatement with it bit for bit
 * (tests/golden/reference_pins_coarse_nodia.npz).
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

/* The undilated level-0 cloud of makeCoarseDepthL0 (:150-218): the unweighted idepth sums (monocular only, :167) and the
 * weights of the scatter, then the compaction over [2,w-2) x [2,h-2).  Same points and rounding as oracle/coarse_ref_oracle.c.
 * gray0: level 0's dIp[0][i][0]; pc: 4 arrays (u, v, idepth, color) of w0*h0 floats, the reference's persistent
 * pc_*_nodia, read and written (a rejected candidate stays in slot *pc_n_nodia).  Returns 0, or -1 (nothing written) when a
 * point's rounded pixel lies outside the image. */
int coarse_nodia_oracle(int w0, int h0, int rgbd, int n, const float* pu, const float* pv, const float* pid, const float* phs,
                        const float* gray0, float* pc, int* pc_n_nodia) {
  const size_t n0 = (size_t)w0 * h0;
  int* pix = malloc(sizeof(int) * (size_t)(n > 0 ? n : 1));
  for (int k = 0; k < n; ++k) {
    int u, v;
    if (rgbd) {
      const double fu = (double)pu[k] + 0.5, fv = (double)pv[k] + 0.5;
      if (!(fu > -1.0 && fu < w0 && fv > -1.0 && fv < h0)) { free(pix); return -1; }
      u = (int)fu; v = (int)fv;
    } else {
      const float fu = pu[k] + 0.5f, fv = pv[k] + 0.5f;
      if (!(fu > -1.f && fu < (float)w0 && fv > -1.f && fv < (float)h0)) { free(pix); return -1; }
      u = (int)fu; v = (int)fv;
    }
    pix[k] = u + w0 * v;
  }
  float* ws = calloc(n0, sizeof(float));
  float* nodia = calloc(n0, sizeof(float));
  for (int k = 0; k < n; ++k) {
    ws[pix[k]] += rgbd ? phs[k] : sqrtf((float)(1e-3 / ((double)phs[k] + 1e-12)));
    if (!rgbd) nodia[pix[k]] += pid[k];
  }
  float *cu = pc, *cv = pc + n0, *ci = pc + 2 * n0, *cc = pc + 3 * n0;
  int m = 0;
  for (int y = 2; y < h0 - 2; ++y)
    for (int x = 2; x < w0 - 2; ++x) {
      const int i = x + y * w0;
      if (!(ws[i] > 0)) continue;
      cu[m] = (float)x;
      cv[m] = (float)y;
      ci[m] = nodia[i];
      cc[m] = gray0[i];
      if (isfinite(cc[m]) && nodia[i] > 0) m++;
    }
  *pc_n_nodia = m;
  free(pix);
  free(ws);
  free(nodia);
  return 0;
}

static int cmp_float(const void* a, const void* b) {
  const float x = *(const float*)a, y = *(const float*)b;
  return (x > y) - (x < y);
}

/* get_idepth_quantile (tandem_backend.cpp:354-361): out[0] = the idepth at index (int)(fraction * (float)n) of the sorted
 * idepth[0..n), out[1] = 1.0f / it.  Both NaN when that index is not below n (the reference reads outside its vector). */
void idepth_quantile_oracle(int n, const float* idepth, float fraction, float* out) {
  const int k = (int)(fraction * (float)n);
  out[0] = out[1] = NAN;
  if (n <= 0 || k >= n) return;
  float* s = malloc(sizeof(float) * (size_t)n);
  memcpy(s, idepth, sizeof(float) * (size_t)n);
  qsort(s, (size_t)n, sizeof(float), cmp_float);
  out[0] = s[k];
  out[1] = 1.0f / s[k];
  free(s);
}
