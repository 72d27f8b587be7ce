// Links the CudaImmaturePoints shim (shims/cuda_immature_points.cpp) against libtandem_b200.so and traces one keyframe's
// points into a frame shifted sideways: a textured image I(x, y) and the same image moved 3 pixels right, K R K^-1 the
// identity and Kt = (fx * 0.1, 0, 0), so a point's match lies at u + 3 and its inverse depth is 3 / (fx * 0.1).  Most points
// must trace GOOD with an interval containing that inverse depth; remove and dropHost must shrink the slot; an invalid slot
// must throw.
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "cuda_coarse_tracker/cuda_immature_points.h"   // needs <Eigen/Dense>: tests/cpp/eigen_stub here, the real one in tandem
#include "tandem_b200.h"

static float I(float x, float y) { return 100.f + 50.f * std::sin(0.3f * x) + 30.f * std::cos(0.23f * y) + 20.f * std::sin(0.11f * (x + y)); }

int main() {
  const int w = 160, h = 120;
  const float fx = 100.f;
  std::vector<float> g0((size_t)w * h), g1((size_t)w * h);
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) { g0[x + (size_t)y * w] = I((float)x, (float)y); g1[x + (size_t)y * w] = I((float)x - 3.f, (float)y); }
  tdm_pyramid *host = nullptr, *frame = nullptr;
  if (tdm_pyramid_create(w, h, 1, 0, &host) || tdm_pyramid_create(w, h, 1, 0, &frame) || tdm_pyramid_build(host, g0.data()) ||
      tdm_pyramid_build(frame, g1.data())) {
    printf("pyramid: %s\n", tdm_last_error());
    return 1;
  }
  int good = 0, within = 0, n = 0;
  try {
    CudaImmaturePoints pts(w, h, 1000);
    std::vector<int> u, v;
    std::vector<float> type;
    for (int y = 20; y < h - 20; y += 7)
      for (int x = 20; x < w - 40; x += 7) { u.push_back(x); v.push_back(y); type.push_back(1.f); }
    n = pts.add(2, host, u, v, type);
    if (n != (int)u.size()) { printf("add kept %d of %zu\n", n, u.size()); return 1; }
    Eigen::Matrix<float, 3, 3> K;
    K.setZero();
    K(0, 0) = K(1, 1) = K(2, 2) = 1.f;
    Eigen::Matrix<float, 3, 1> Kt(fx * 0.1f, 0.f, 0.f);
    Eigen::Matrix<float, 2, 1> aff(1.f, 0.f);
    pts.trace(frame, {2}, {host}, {K}, {Kt}, {aff});
    CudaImmaturePoints::State s = pts.get(2);
    const float truth = 3.f / (fx * 0.1f);
    for (int i = 0; i < n; ++i) {
      if (s.status[i] != TDM_IPS_GOOD) continue;
      ++good;
      within += s.idepth_min[i] <= truth && truth <= s.idepth_max[i];
    }
    if (good < n * 3 / 4 || within < good * 9 / 10) { printf("good %d within %d of %d\n", good, within, n); return 1; }
    pts.remove(2, {0, n - 1});
    if ((int)pts.get(2).u.size() != n - 2) { printf("remove\n"); return 1; }
    pts.dropHost(2);
    if (!pts.get(2).u.empty()) { printf("dropHost\n"); return 1; }
    bool threw = false;
    try { pts.dropHost(8); } catch (const std::runtime_error &) { threw = true; }
    if (!threw) { printf("slot 8 did not throw\n"); return 1; }
  } catch (const std::exception &e) {
    printf("exception: %s\n", e.what());
    return 1;
  }
  tdm_pyramid_destroy(frame);
  tdm_pyramid_destroy(host);
  printf("shim_trace: OK (%d of %d points GOOD, %d with the true inverse depth inside)\n", good, n, within);
  return 0;
}
