// Links the CudaCoarseTracker shim (shims/cuda_coarse_tracker.cpp) against libtandem_b200.so and runs
// CudaCoarseTracker::trackPyramid the way CoarseTracker::trackNewestCoarse would call it: three level trackers over an analytic
// textured plane (fronto-parallel, inverse depth 0.5), the new image equal to the reference image, a start pose 2 cm off.
// The loop must come back towards the identity, report every level, and throw on levels given in the wrong order.
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "cuda_coarse_tracker/cuda_coarse_tracker.h"   // needs <Eigen/Dense>: tests/cpp/eigen_stub here, the real one in tandem

static float I(float x, float y) { return 100.f + 50.f * std::sin(0.1f * x) + 30.f * std::cos(0.13f * y); }

int main() {
  const int w0 = 160, h0 = 120, levels = 3;
  std::vector<CudaCoarseTracker*> trk;
  for (int l = 0; l < levels; ++l) {
    const int w = w0 >> l, h = h0 >> l;
    const float s = (float)(1 << l);
    auto Il = [&](float x, float y) { return I((x + 0.5f) * s - 0.5f, (y + 0.5f) * s - 0.5f); };   // level l pixel in level-0 units
    std::vector<float> dI((size_t)3 * w * h);
    for (int y = 0; y < h; ++y)
      for (int x = 0; x < w; ++x) {
        float* p = &dI[3 * (size_t)(x + y * w)];
        p[0] = Il((float)x, (float)y);
        p[1] = 0.5f * (Il((float)x + 1, (float)y) - Il((float)x - 1, (float)y));
        p[2] = 0.5f * (Il((float)x, (float)y + 1) - Il((float)x, (float)y - 1));
      }
    std::vector<float> u, v, id, col;
    for (int y = 4; y < h - 4; ++y)
      for (int x = 4; x < w - 4; ++x) { u.push_back((float)x); v.push_back((float)y); id.push_back(0.5f); col.push_back(Il((float)x, (float)y)); }
    CudaCoarseTracker* t = new CudaCoarseTracker(w, h, 9.f, 20.f);
    t->init();
    t->setK(w, h, 80.f / s, 80.f / s, 80.f / s - 0.5f, 60.f / s - 0.5f);
    t->setReference((int)u.size(), u.data(), v.data(), id.data(), col.data(), 1.f, Eigen::Vector2d(0, 0));
    t->setNew(dI.data());
    trk.push_back(t);
  }
  Eigen::Matrix<double, 4, 4> T = Eigen::Matrix<double, 4, 4>::Identity();
  T(0, 3) = 0.02;
  const int its[5] = {10, 20, 50, 50, 50};
  Eigen::Matrix<double, 5, 1> minRes;
  minRes.setConstant(NAN);
  CudaCoarseTracker::PyramidTrackResult r =
      CudaCoarseTracker::trackPyramid(trk, T, Eigen::Vector2d(0, 0), 1.f, 20.f, its, 0.001f, 1e12f, 1e8f, minRes);
  const double t_err = std::sqrt(r.refToNew(0, 3) * r.refToNew(0, 3) + r.refToNew(1, 3) * r.refToNew(1, 3) + r.refToNew(2, 3) * r.refToNew(2, 3));
  printf("trackPyramid: ok=%d |t| 0.0200 -> %.5f, evaluations %d/%d/%d, lastResiduals %.3f %.3f %.3f, aborted %d repeated %d\n", (int)r.ok,
         t_err, r.evaluations[0], r.evaluations[1], r.evaluations[2], r.lastResiduals(0), r.lastResiduals(1), r.lastResiduals(2),
         r.abortedLevel, r.repeatedLevel);
  bool threw = false;
  try {
    std::vector<CudaCoarseTracker*> wrong = {trk[0], trk[2], trk[1]};
    CudaCoarseTracker::trackPyramid(wrong, T, Eigen::Vector2d(0, 0), 1.f, 20.f, its, 0.001f, 1e12f, 1e8f, minRes);
  } catch (std::runtime_error const& e) {
    threw = true;
    printf("levels in the wrong order: %s\n", e.what());
  }
  bool ok = r.ok && t_err < 0.25 * 0.02 && threw && r.abortedLevel == -1;
  for (int l = 0; l < levels; ++l) ok = ok && r.evaluations[l] > 0 && std::isfinite(r.lastResiduals(l));
  ok = ok && std::isnan(r.lastResiduals(3)) && r.evaluations[3] == 0;
  for (CudaCoarseTracker* t : trk) delete t;
  printf("CudaCoarseTracker::trackPyramid shim: %s\n", ok ? "PASS" : "FAIL");
  return ok ? 0 : 1;
}
