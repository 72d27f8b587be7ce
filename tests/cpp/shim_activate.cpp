// Links CudaImmaturePoints::activate (shims/cuda_immature_points.cpp) against libtandem_b200.so and runs activatePointsMT's
// solve on a textured scene seen from three keyframes moved sideways: frame f is the image I(x - 3 f, y), R the identity and
// t = (0.1 f, 0, 0), so every point lies at inverse depth 0.3.  Frames 0 and 1 are hosts (slots 4 and 1), frame 2 is the
// newest keyframe (no slot).  The hosts' points are traced into frame 2, every activatable one (canActivate of
// FullSystem.cpp:769-774) is a candidate.  Most candidates must activate near inverse depth 0.3.  Every input and output is
// written to the file named by argv[1], so tests/test_activate_gpu.py can replay the same call through Python and compare.
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "cuda_coarse_tracker/cuda_immature_points.h"   // needs <Eigen/Dense>: tests/cpp/eigen_stub here, the real one in tandem
#include "tandem_b200.h"

static float I(float x, float y) { return 100.f + 50.f * std::sin(0.3f * x) + 30.f * std::cos(0.23f * y) + 20.f * std::sin(0.11f * (x + y)); }

template <typename T>
static void put(FILE *f, const T *p, size_t n) { fwrite(p, sizeof(T), n, f); }

int main(int argc, char **argv) {
  if (argc < 2) { printf("usage: shim_activate OUT\n"); return 2; }
  const int w = 160, h = 120, nf = 3;
  const float fx = 100.f, fy = 100.f, cx = 79.5f, cy = 59.5f;
  std::vector<std::vector<float>> gray(nf, std::vector<float>((size_t)w * h));
  std::vector<tdm_pyramid *> pyr(nf, nullptr);
  for (int f = 0; f < nf; ++f) {
    for (int y = 0; y < h; ++y)
      for (int x = 0; x < w; ++x) gray[f][x + (size_t)y * w] = I((float)x - 3.f * f, (float)y);
    if (tdm_pyramid_create(w, h, 1, 0, &pyr[f]) || tdm_pyramid_build(pyr[f], gray[f].data())) {
      printf("pyramid: %s\n", tdm_last_error());
      return 1;
    }
  }
  const std::vector<int> slots = {4, 1, -1};
  int made = 0, near = 0, k = 0;
  try {
    CudaImmaturePoints pts(w, h, 1000);
    std::vector<int> u, v;
    std::vector<float> type;
    for (int y = 20; y < h - 20; y += 7)
      for (int x = 24; x < w - 40; x += 7) { u.push_back(x); v.push_back(y); type.push_back(1.f); }
    const int n = (int)u.size();
    Eigen::Matrix<float, 3, 3> K;
    K.setZero();
    K(0, 0) = K(1, 1) = K(2, 2) = 1.f;
    Eigen::Matrix<float, 2, 1> aff(1.f, 0.f);
    std::vector<float> Ks, Kts;
    for (int f = 0; f < 2; ++f) {
      if (pts.add(slots[f], pyr[f], u, v, type) != n) { printf("add\n"); return 1; }
      Eigen::Matrix<float, 3, 1> Kt(fx * (0.1f * (2 - f)), 0.f, 0.f);   // host f into the newest frame
      pts.trace(pyr[2], {slots[f]}, {pyr[f]}, {K}, {Kt}, {aff});
      for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) Ks.push_back(K(r, c)); Kts.push_back(Kt(r)); }
    }
    std::vector<CudaImmaturePoints::Precalc> pc(nf * nf);
    std::vector<float> pcf;
    for (int a = 0; a < nf; ++a)
      for (int b = 0; b < nf; ++b) {
        CudaImmaturePoints::Precalc &p = pc[a * nf + b];
        p.PRE_RTll.setZero();
        p.PRE_RTll(0, 0) = p.PRE_RTll(1, 1) = p.PRE_RTll(2, 2) = 1.f;
        p.PRE_tTll = Eigen::Matrix<float, 3, 1>(0.1f * (b - a), 0.f, 0.f);
        p.PRE_aff_mode = Eigen::Matrix<float, 2, 1>(1.f, 0.f);
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) pcf.push_back(p.PRE_RTll(r, c));
        for (int r = 0; r < 3; ++r) pcf.push_back(p.PRE_tTll(r));
        pcf.push_back(1.f);
        pcf.push_back(0.f);
      }
    std::vector<int> cf, ci;
    for (int f = 0; f < 2; ++f) {
      CudaImmaturePoints::State s = pts.get(slots[f]);
      for (int i = 0; i < n; ++i) {
        const int st = s.status[i];
        if (std::isfinite(s.idepth_max[i]) &&
            (st == TDM_IPS_GOOD || st == TDM_IPS_SKIPPED || st == TDM_IPS_BADCONDITION || st == TDM_IPS_OOB) &&
            s.interval[i] < 8 && s.quality[i] > 3 && s.idepth_max[i] + s.idepth_min[i] > 0) {
          cf.push_back(f);
          ci.push_back(i);
        }
      }
    }
    CudaImmaturePoints::Activation a = pts.activate(slots, pyr, pc, fx, fy, cx, cy, cf, ci);
    k = (int)cf.size();
    for (int j = 0; j < k; ++j) {
      if (a.result[j] != 1) continue;
      ++made;
      near += std::fabs(a.idepth[j] - 0.3f) < 0.03f;
    }
    if (k < n / 2 || made < k * 3 / 4 || near < made * 9 / 10) { printf("candidates %d made %d near %d\n", k, made, near); return 1; }
    bool threw = false;
    try { pts.activate(slots, pyr, pc, fx, fy, cx, cy, {2}, {0}); } catch (const std::runtime_error &) { threw = true; }
    if (!threw) { printf("a candidate of the newest frame did not throw\n"); return 1; }
    FILE *o = fopen(argv[1], "wb");
    if (!o) { printf("cannot write %s\n", argv[1]); return 1; }
    const int hdr[6] = {w, h, nf, 2, n, k};
    put(o, hdr, 6);
    for (int f = 0; f < nf; ++f) put(o, gray[f].data(), gray[f].size());
    put(o, slots.data(), 3);
    for (int f = 0; f < 2; ++f) { put(o, u.data(), n); put(o, v.data(), n); }
    put(o, Ks.data(), Ks.size());
    put(o, Kts.data(), Kts.size());
    put(o, pcf.data(), pcf.size());
    const float calib[4] = {fx, fy, cx, cy};
    put(o, calib, 4);
    put(o, cf.data(), k);
    put(o, ci.data(), k);
    put(o, a.result.data(), k);
    put(o, a.idepth.data(), k);
    put(o, a.res_state.data(), a.res_state.size());
    put(o, a.res_energy.data(), a.res_energy.size());
    fclose(o);
  } catch (const std::exception &e) {
    printf("exception: %s\n", e.what());
    return 1;
  }
  for (tdm_pyramid *p : pyr) tdm_pyramid_destroy(p);
  printf("shim_activate: OK (%d of %d candidates activated, %d near the true inverse depth)\n", made, k, near);
  return 0;
}
