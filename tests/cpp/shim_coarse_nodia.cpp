// Links the CudaCoarseTracker shim (shims/cuda_coarse_tracker.cpp) against libtandem_b200.so and builds every level's
// reference together with MVSNet's depth range through the overload of CudaCoarseTracker::setCoarseTrackingRef that returns
// pc_n_nodia and the depth quantile: three level trackers, a textured keyframe pyramid, sparse points on a fronto-parallel
// plane at depth 2 (inverse depth 0.5), one of them with inverse depth -0.5.  The counts must equal the plain overload's, the
// undilated cloud must hold every interior point but the negative one, the quantile must be 1 / 0.5 = 2 exactly, fraction 1
// must give NaN, and a fraction outside [0, 1] must throw.
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
    trk.push_back(t);
  }
  // monocular points on every third pixel: centerProjectedTo = (x, y, 0.5), HdiF = 1; the interior ones but (82, 61), whose
  // inverse depth is -0.5, form the nodia cloud
  std::vector<float> u, v, id, hess;
  int interior = 0;
  for (int y = 1; y < h0 - 1; y += 3)
    for (int x = 1; x < w0 - 1; x += 3) {
      u.push_back((float)x); v.push_back((float)y); id.push_back(x == 82 && y == 61 ? -0.5f : 0.5f); hess.push_back(1.f);
      interior += x >= 2 && x < w0 - 2 && y >= 2 && y < h0 - 2;
    }
  const Eigen::Matrix<double, 4, 4> I4 = Eigen::Matrix<double, 4, 4>::Identity();
  const std::vector<int> plain = CudaCoarseTracker::setCoarseTrackingRef(trk, false, (int)u.size(), u.data(), v.data(), id.data(),
                                                                         hess.data(), pyr, nullptr, 0, I4, 1, false, 1.f,
                                                                         Eigen::Vector2d(0, 0));
  int n_nodia = -1;
  float depth = 0.f;
  const std::vector<int> pc_n = CudaCoarseTracker::setCoarseTrackingRef(trk, false, (int)u.size(), u.data(), v.data(), id.data(),
                                                                        hess.data(), pyr, nullptr, 0, I4, 1, false, 1.f,
                                                                        Eigen::Vector2d(0, 0), 0.2f, &n_nodia, &depth);
  printf("setCoarseTrackingRef: pc_n %d / %d / %d (plain %d / %d / %d), pc_n_nodia %d of %d interior points, depth quantile %g\n",
         pc_n[0], pc_n[1], pc_n[2], plain[0], plain[1], plain[2], n_nodia, interior, depth);
  bool ok = pc_n == plain && n_nodia == interior - 1 && depth == 2.f;
  float depth1 = 0.f;
  CudaCoarseTracker::setCoarseTrackingRef(trk, false, (int)u.size(), u.data(), v.data(), id.data(), hess.data(), pyr, nullptr, 0, I4,
                                          1, false, 1.f, Eigen::Vector2d(0, 0), 1.f, &n_nodia, &depth1);
  printf("fraction 1: depth quantile %g\n", depth1);
  ok = ok && std::isnan(depth1);
  bool threw = false;
  try {
    CudaCoarseTracker::setCoarseTrackingRef(trk, false, (int)u.size(), u.data(), v.data(), id.data(), hess.data(), pyr, nullptr, 0,
                                            I4, 1, false, 1.f, Eigen::Vector2d(0, 0), 1.5f, &n_nodia, &depth);
  } catch (std::runtime_error const& e) {
    threw = true;
    printf("fraction 1.5: %s\n", e.what());
  }
  ok = ok && threw;
  for (CudaCoarseTracker* t : trk) delete t;
  tdm_pyramid_destroy(pyr);
  printf("shim_coarse_nodia: %s\n", ok ? "OK" : "FAIL");
  return ok ? 0 : 1;
}
