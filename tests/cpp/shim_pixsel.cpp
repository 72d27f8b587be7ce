// Links CudaPixelSelector and CudaImmaturePoints::makeNewTraces (shims/cuda_pixel_selector.cpp, shims/cuda_immature_points.cpp)
// against libtandem_b200.so and runs a keyframe's selection on a textured 192 x 144 image: makeMaps twice with the reference's
// defaults (the potential carried from the first call into the second), then makeNewTraces into slot 2 of a set with a second
// selector.  Every input and output is written to the file named by argv[1], so tests/test_pixsel_gpu.py can replay the same
// calls through Python and compare.
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "cuda_coarse_tracker/cuda_immature_points.h"   // needs <Eigen/Dense>: tests/cpp/eigen_stub here, the real one in tandem
#include "cuda_coarse_tracker/cuda_pixel_selector.h"
#include "tandem_b200.h"

static float I(float x, float y) {
  return std::floor(100.f + 50.f * std::sin(0.3f * x) + 30.f * std::cos(0.23f * y) + 20.f * std::sin(0.11f * (x + y)));
}

template <typename T>
static void put(FILE *f, const T *p, size_t n) { fwrite(p, sizeof(T), n, f); }

int main(int argc, char **argv) {
  if (argc < 2) { printf("usage: shim_pixsel OUT\n"); return 2; }
  const int w = 192, h = 144;
  std::vector<float> gray((size_t)w * h);
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) gray[x + (size_t)y * w] = I((float)x, (float)y);
  tdm_pyramid *pyr = nullptr;
  if (tdm_pyramid_create(w, h, 3, 0, &pyr) || tdm_pyramid_build(pyr, gray.data())) {
    printf("pyramid: %s\n", tdm_last_error());
    return 1;
  }
  FILE *f = fopen(argv[1], "wb");
  if (!f) return 1;
  int rc = 0;
  try {
    CudaPixelSelector sel(w, h);
    std::vector<float> map((size_t)w * h);
    const int ints[2] = {w, h};
    put(f, ints, 2);
    put(f, gray.data(), gray.size());
    for (float density : {300.f, 600.f}) {
      const int n = sel.makeMaps(pyr, map.data(), density);
      const int p = sel.currentPotential();
      put(f, &n, 1);
      put(f, &p, 1);
      put(f, map.data(), map.size());
    }
    CudaPixelSelector sel2(w, h);
    sel2.setCurrentPotential(2);
    CudaImmaturePoints pts(w, h, 4000);
    std::vector<int> u, v;
    std::vector<float> type;
    const int n = pts.makeNewTraces(2, sel2, pyr, 500.f, &u, &v, &type);
    const int p = sel2.currentPotential();
    put(f, &n, 1);
    put(f, &p, 1);
    put(f, u.data(), n);
    put(f, v.data(), n);
    put(f, type.data(), n);
    printf("shim_pixsel: makeNewTraces kept %d, potential %d\n", n, p);
  } catch (const std::exception &e) {
    printf("%s\n", e.what());
    rc = 1;
  }
  fclose(f);
  tdm_pyramid_destroy(pyr);
  return rc;
}
