// Links CudaUndistort (shims/cuda_undistort.cpp) against libtandem_b200.so and runs one camera the way DatasetReader and
// FullSystem drive it: the constructor from the calibration arrays, setGammaFunction's two calls (setGamma with getG's G is
// what TANDEM does on start; the case then sets a second Binv), and one frame with its BGR image into a pyramid read back per
// level.  Inputs are raw files in the directory argv[1] (remap_x, remap_y, response (256 floats), vignette, binv0, binv1,
// gray, bgr); outputs go there too (dI<l>, ag<l>, bgr_out), so tests/test_undistort_gpu.py compares them with the pins.
#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <vector>

#include "cuda_coarse_tracker/cuda_undistort.h"
#include "tandem_b200.h"

template <typename T>
static std::vector<T> load(const std::string &dir, const char *name, size_t n) {
  std::vector<T> v(n);
  FILE *f = fopen((dir + "/" + name + ".bin").c_str(), "rb");
  if (!f || fread(v.data(), sizeof(T), n, f) != n) throw std::runtime_error(std::string("cannot read ") + name);
  fclose(f);
  return v;
}
template <typename T>
static void save(const std::string &dir, const std::string &name, const T *p, size_t n) {
  FILE *f = fopen((dir + "/" + name + ".bin").c_str(), "wb");
  fwrite(p, sizeof(T), n, f);
  fclose(f);
}

int main(int argc, char **argv) {
  if (argc < 10) { printf("usage: shim_undistort DIR w_org h_org w h mode exposure factor levels\n"); return 2; }
  const std::string dir = argv[1];
  const int w_org = atoi(argv[2]), h_org = atoi(argv[3]), w = atoi(argv[4]), h = atoi(argv[5]), mode = atoi(argv[6]);
  const float exposure = (float)atof(argv[7]), factor = (float)atof(argv[8]);
  const int levels = atoi(argv[9]);
  try {
    const size_t n = (size_t)w * h, n_org = (size_t)w_org * h_org;
    auto rx = load<float>(dir, "remap_x", n), ry = load<float>(dir, "remap_y", n), resp = load<float>(dir, "response", 256);
    auto vig = load<unsigned short>(dir, "vignette", n_org);
    auto b0 = load<float>(dir, "binv0", 256), b1 = load<float>(dir, "binv1", 256);
    auto gray = load<unsigned char>(dir, "gray", n_org), bgr = load<unsigned char>(dir, "bgr", 3 * n_org);
    CudaUndistort u(w_org, h_org, w, h, rx.data(), ry.data(), resp.data(), 256, vig.data(), mode);
    float G[256];
    if (!u.getG(G)) throw std::runtime_error("calibration not valid");
    u.setGamma(b0.data());
    u.setGamma(b1.data());
    u.setGamma(nullptr);
    tdm_pyramid *pyr = nullptr;
    if (tdm_pyramid_create(w, h, levels, 0, &pyr)) throw std::runtime_error(tdm_last_error());
    std::vector<unsigned char> bgr_out(3 * n);
    const float t = u.undistort(gray.data(), exposure, pyr, factor, bgr.data(), bgr_out.data());
    save(dir, "bgr_out", bgr_out.data(), bgr_out.size());
    for (int l = 0; l < levels; ++l) {
      const size_t nl = (size_t)(w >> l) * (h >> l);
      std::vector<float> dI(3 * nl), ag(nl);
      if (tdm_pyramid_get_level(pyr, l, dI.data(), ag.data())) throw std::runtime_error(tdm_last_error());
      save(dir, "dI" + std::to_string(l), dI.data(), dI.size());
      save(dir, "ag" + std::to_string(l), ag.data(), ag.size());
    }
    tdm_pyramid_destroy(pyr);
    bool threw = false;
    try {
      CudaUndistort bad(w_org, h_org, w + 1, h, nullptr, nullptr, nullptr, 0, nullptr);
    } catch (const std::runtime_error &) {
      threw = true;
    }
    if (!threw) throw std::runtime_error("passthrough with w != w_org was accepted");
    printf("exposure_time %.9g\n", t);
  } catch (const std::exception &e) {
    printf("error: %s\n", e.what());
    return 1;
  }
  return 0;
}
