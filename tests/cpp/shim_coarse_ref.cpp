// Links the CudaCoarseTracker shim (shims/cuda_coarse_tracker.cpp) against libtandem_b200.so and builds every level's
// reference the way CoarseTracker::setCoarseTrackingRef would through CudaCoarseTracker::setCoarseTrackingRef: three level
// trackers, a textured keyframe pyramid, sparse points on a fronto-parallel plane (inverse depth 0.5), no dense map.  Then
// trackPyramid from a start pose 2 cm off must come back towards the identity, and a point outside the image must throw.
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "cuda_coarse_tracker/cuda_coarse_tracker.h"   // needs <Eigen/Dense>: tests/cpp/eigen_stub here, the real one in tandem
#include "tandem_b200.h"

static float I(float x, float y) { return 100.f + 50.f * std::sin(0.1f * x) + 30.f * std::cos(0.13f * y); }

int main() {
  const int w0 = 160, h0 = 120, levels = 3;
  std::vector<float> gray((size_t)w0 * h0);
  for (int y = 0; y < h0; ++y)
    for (int x = 0; x < w0; ++x) gray[x + (size_t)y * w0] = I((float)x, (float)y);
  tdm_pyramid* pyr = nullptr;
  if (tdm_pyramid_create(w0, h0, levels, 0, &pyr) != 0 || tdm_pyramid_build(pyr, gray.data()) != 0) {
    printf("pyramid: %s\n", tdm_last_error());
    return 1;
  }
  std::vector<CudaCoarseTracker*> trk;
  for (int l = 0; l < levels; ++l) {
    const int w = w0 >> l, h = h0 >> l;
    const float s = (float)(1 << l);
    CudaCoarseTracker* t = new CudaCoarseTracker(w, h, 9.f, 20.f);
    t->init();
    t->setK(w, h, 80.f / s, 80.f / s, (79.5f + 0.5f) / s - 0.5f, (59.5f + 0.5f) / s - 0.5f);
    t->setNewFromPyramid(pyr, l);
    trk.push_back(t);
  }
  // monocular points on every third pixel: centerProjectedTo = (x, y, 0.5), HdiF = 1
  std::vector<float> u, v, id, hess;
  for (int y = 1; y < h0 - 1; y += 3)
    for (int x = 1; x < w0 - 1; x += 3) { u.push_back((float)x); v.push_back((float)y); id.push_back(0.5f); hess.push_back(1.f); }
  const Eigen::Matrix<double, 4, 4> I4 = Eigen::Matrix<double, 4, 4>::Identity();
  const std::vector<int> pc_n = CudaCoarseTracker::setCoarseTrackingRef(trk, false, (int)u.size(), u.data(), v.data(), id.data(),
                                                                        hess.data(), pyr, nullptr, 0, I4, 1, false, 1.f,
                                                                        Eigen::Vector2d(0, 0));
  printf("setCoarseTrackingRef: %zu points -> pc_n %d / %d / %d\n", u.size(), pc_n[0], pc_n[1], pc_n[2]);
  bool ok = pc_n.size() == (size_t)levels;
  // level 0: the points and their diagonal dilation cover the interior; the upper levels are dense
  for (int l = 0; ok && l < levels; ++l) ok = pc_n[l] > ((w0 >> l) - 4) * ((h0 >> l) - 4) / 3;
  Eigen::Matrix<double, 4, 4> T = I4;
  T(0, 3) = 0.02;
  const int its[5] = {10, 20, 50, 50, 50};
  Eigen::Matrix<double, 5, 1> minRes;
  minRes.setConstant(NAN);
  CudaCoarseTracker::PyramidTrackResult r =
      CudaCoarseTracker::trackPyramid(trk, T, Eigen::Vector2d(0, 0), 1.f, 20.f, its, 0.001f, 1e12f, 1e8f, minRes);
  const double t_err = std::sqrt(r.refToNew(0, 3) * r.refToNew(0, 3) + r.refToNew(1, 3) * r.refToNew(1, 3) + r.refToNew(2, 3) * r.refToNew(2, 3));
  printf("trackPyramid: ok=%d |t| 0.0200 -> %.5f\n", (int)r.ok, t_err);
  ok = ok && r.ok && t_err < 0.25 * 0.02;
  bool threw = false;
  try {
    u[5] = (float)w0 - 0.5f;   // (int)(u + 0.5f) == w0
    CudaCoarseTracker::setCoarseTrackingRef(trk, false, (int)u.size(), u.data(), v.data(), id.data(), hess.data(), pyr, nullptr, 0,
                                            I4, 1, false, 1.f, Eigen::Vector2d(0, 0));
  } catch (std::runtime_error const& e) {
    threw = true;
    printf("point outside the image: %s\n", e.what());
  }
  ok = ok && threw;
  for (CudaCoarseTracker* t : trk) delete t;
  tdm_pyramid_destroy(pyr);
  printf("shim_coarse_ref: %s\n", ok ? "OK" : "FAIL");
  return ok ? 0 : 1;
}
