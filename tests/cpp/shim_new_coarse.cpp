// Links the CudaCoarseTracker shim (shims/cuda_coarse_tracker.cpp) against libtandem_b200.so and runs
// CudaCoarseTracker::trackNewCoarse the way FullSystem::trackNewCoarse would call it: three level trackers over the analytic
// textured plane of shim_pyramid.cpp (fronto-parallel, inverse depth 0.5, the new image equal to the reference image, so the
// true pose is the identity) and three tries: try 0 puts the plane behind the camera (no point warps in, every residual is
// NaN, so it cannot win), try 1 is half a centimetre off, try 2 the identity.  Try 1 must win and stop the loop (tries == 2);
// an empty try list must throw.
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
  std::vector<Eigen::Matrix<double, 4, 4>> tries(3, Eigen::Matrix<double, 4, 4>::Identity());
  tries[0](2, 3) = -3.0;
  tries[1](0, 3) = 0.005;
  const int its[5] = {10, 20, 50, 50, 50};
  Eigen::Matrix<double, 5, 1> lastCoarseRMSE;
  lastCoarseRMSE.setConstant(1.0);
  CudaCoarseTracker::NewCoarseResult r =
      CudaCoarseTracker::trackNewCoarse(trk, tries, Eigen::Vector2d(0, 0), 1.f, 20.f, its, 0.001f, 1e12f, 1e8f, lastCoarseRMSE, 1.5f);
  const double t_err = std::sqrt(r.lastF_2_fh(0, 3) * r.lastF_2_fh(0, 3) + r.lastF_2_fh(1, 3) * r.lastF_2_fh(1, 3) +
                                 r.lastF_2_fh(2, 3) * r.lastF_2_fh(2, 3));
  printf("trackNewCoarse: haveOneGood=%d tries %d winner %d |t| %.5f, achievedRes %.3f %.3f %.3f\n", (int)r.haveOneGood,
         r.tryIterations, r.winner, t_err, r.achievedRes(0), r.achievedRes(1), r.achievedRes(2));
  bool threw = false;
  try {
    CudaCoarseTracker::trackNewCoarse(trk, std::vector<Eigen::Matrix<double, 4, 4>>(), Eigen::Vector2d(0, 0), 1.f, 20.f, its, 0.001f,
                                      1e12f, 1e8f, lastCoarseRMSE, 1.5f);
  } catch (std::runtime_error const& e) {
    threw = true;
    printf("empty try list: %s\n", e.what());
  }
  bool ok = r.haveOneGood && r.winner == 1 && r.tryIterations == 2 && t_err < 0.25 * 0.005 && threw;
  ok = ok && r.achievedRes(0) < 1.5 && std::isnan(r.achievedRes(3));
  for (CudaCoarseTracker* t : trk) delete t;
  printf("CudaCoarseTracker::trackNewCoarse shim: %s\n", ok ? "PASS" : "FAIL");
  return ok ? 0 : 1;
}
