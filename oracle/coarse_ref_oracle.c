/* ORACLE (test infrastructure - never linked into, or called by, the product library).
 *
 * Plain-C restatement of CoarseTracker::makeCoarseDepthL0 (tandem/src/FullSystem/CoarseTracker.cpp:148-374), SURVEY.md 8(f)
 * row n7, for every pyramid level; oracle/coarse_ref.py chains it with the dense block of setCoarseTrackingRef
 * (front_oracle_dense_reference, oracle/front_oracle.c).  Left out, as in the product: idepth_nodia, pc_*_nodia and
 * depth_rel_var (only saveKFDepthMap, a debug dump, reads them).
 * PINNED: oracle/ref_build_coarse_ref.mk cuts the reference's own function body out of CoarseTracker.cpp and compiles it,
 * unmodified, in the harness oracle/ref_wrap_coarse_ref.cpp; tests/test_coarse_ref_cpu.py compares this restatement with it
 * bit for bit (tests/golden/reference_pins_coarse_ref.npz).
 * One documented choice: on levels 0 and 1 the diagonal dilation of the first and the last pixel of its flat range reads one
 * element before / behind the weight image (the padding of the reference's allocAligned buffers, uninitialised there).  Here
 * that neighbour counts as unweighted; the pin harness zero-fills the padding, which gives the same.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define MAX_LEVELS 5

static void dilate(float* idepth, float* ws, float* bak, int w, int h, int diag) {
  const int n = w * h, wh = n - w;
  memcpy(bak, ws, sizeof(float) * (size_t)n);
  for (int i = w; i < wh; ++i) {
    if (bak[i] > 0) continue;
    const int nb[4] = {diag ? i + 1 + w : i + 1, diag ? i - 1 - w : i - 1, diag ? i + w - 1 : i + w, diag ? i - w + 1 : i - w};
    float sum = 0, num = 0, numn = 0;
    for (int k = 0; k < 4; ++k) {
      const int j = nb[k];
      if (j < 0 || j >= n || !(bak[j] > 0)) continue;
      sum += idepth[j];
      num += bak[j];
      numn++;
    }
    if (numn > 0) {
      idepth[i] = sum / numn;
      ws[i] = num / numn;
    }
  }
}

/* gray: levels concatenated, level l holds wl*hl floats (dIp[l][i][0]); idepth: levels concatenated (output, idepth[l] after
 * normalisation); pc: per level 4 arrays (u, v, idepth, color) of wl*hl floats each, level l at 4 * (offset of level l) -
 * the reference's persistent pc_* arrays, read and written.  Returns 0, or -1 (nothing written) when a point's rounded pixel
 * lies outside the level-0 image. */
int coarse_ref_oracle(int w0, int h0, int levels, int rgbd, int n, const float* pu, const float* pv, const float* pid,
                      const float* phs, const float* gray, float* idepth, float* pc, int* pc_n) {
  if (levels < 1 || levels > MAX_LEVELS) return -1;
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
  size_t off[MAX_LEVELS + 1] = {0};
  for (int l = 0; l < levels; ++l) off[l + 1] = off[l] + (size_t)(w0 >> l) * (h0 >> l);
  float* ws = calloc(off[levels], sizeof(float));
  float* bak = malloc(sizeof(float) * (size_t)w0 * h0);
  memset(idepth, 0, sizeof(float) * (size_t)w0 * h0);
  /* scatter in input order (:155-182) */
  for (int k = 0; k < n; ++k) {
    const float wt = rgbd ? phs[k] : sqrtf((float)(1e-3 / ((double)phs[k] + 1e-12)));
    idepth[pix[k]] += pid[k] * wt;
    ws[pix[k]] += wt;
  }
  /* sum pyramid from the un-dilated level below (:222-243) */
  for (int l = 1; l < levels; ++l) {
    const int wl = w0 >> l, hl = h0 >> l, wm = w0 >> (l - 1);
    const float *im = idepth + off[l - 1], *wsm = ws + off[l - 1];
    for (int y = 0; y < hl; ++y)
      for (int x = 0; x < wl; ++x) {
        const int b = 2 * x + 2 * y * wm;
        idepth[off[l] + x + y * wl] = im[b] + im[b + 1] + im[b + wm] + im[b + wm + 1];
        ws[off[l] + x + y * wl] = wsm[b] + wsm[b + 1] + wsm[b + wm] + wsm[b + wm + 1];
      }
  }
  /* dilation (:246-322) */
  for (int l = 0; l < levels; ++l) dilate(idepth + off[l], ws + off[l], bak, w0 >> l, h0 >> l, l < 2);
  /* normalise and compact (:325-370), rejected candidates written to slot lpc_n first */
  for (int l = 0; l < levels; ++l) {
    const int wl = w0 >> l, hl = h0 >> l;
    const size_t nl = (size_t)wl * hl;
    float *id = idepth + off[l], *wsl = ws + off[l];
    const float* g = gray + off[l];
    float *cu = pc + 4 * off[l], *cv = cu + nl, *ci = cu + 2 * nl, *cc = cu + 3 * nl;
    int m = 0;
    for (int y = 2; y < hl - 2; ++y)
      for (int x = 2; x < wl - 2; ++x) {
        const int i = x + y * wl;
        if (wsl[i] > 0) {
          id[i] /= wsl[i];
          cu[m] = (float)x;
          cv[m] = (float)y;
          ci[m] = id[i];
          cc[m] = g[i];
          if (!isfinite(cc[m]) || !(id[i] > 0)) {
            id[i] = -1;
            continue;
          }
          m++;
        } else {
          id[i] = -1;
        }
        wsl[i] = 1;
      }
    pc_n[l] = m;
  }
  free(pix);
  free(ws);
  free(bak);
  return 0;
}
