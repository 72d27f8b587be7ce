// Links CudaActivePoints (shims/cuda_active_points.cpp) against libtandem_b200.so and runs an optimize()-shaped sequence of
// linearizeAll calls on a window read from argv[1] (written by tests/test_linearize_gpu.py): the frames' grey images, the
// calibration, the points, activeResiduals, and per step (fix, apply, idepth_scaled, idepth_zero_scaled, precalc).  The
// newest frame's frameEnergyTH follows each call's new threshold, as setNewFrameEnergyTH leaves it.  Every output is written
// to argv[2], so the test can compare it with the C oracle.
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "cuda_coarse_tracker/cuda_active_points.h"   // needs <Eigen/Dense>: tests/cpp/eigen_stub here, the real one in tandem
#include "tandem_b200.h"

template <typename T>
static void get(FILE *f, T *p, size_t n) {
  if (fread(p, sizeof(T), n, f) != n) throw std::runtime_error("short input");
}
template <typename T>
static void put(FILE *f, const T *p, size_t n) { fwrite(p, sizeof(T), n, f); }

int main(int argc, char **argv) {
  if (argc < 3) { printf("usage: shim_linearize IN OUT\n"); return 2; }
  FILE *in = fopen(argv[1], "rb");
  FILE *out = fopen(argv[2], "wb");
  if (!in || !out) { printf("cannot open the files\n"); return 2; }
  std::vector<tdm_pyramid *> pyr;
  int rc = 0;
  try {
    int hdr[6];
    get(in, hdr, 6);
    const int w = hdr[0], h = hdr[1], n = hdr[2], np = hdr[3], m = hdr[4], steps = hdr[5];
    std::vector<float> gray((size_t)w * h);
    for (int f = 0; f < n; ++f) {
      get(in, gray.data(), gray.size());
      tdm_pyramid *p = nullptr;
      if (tdm_pyramid_create(w, h, 1, 0, &p) || tdm_pyramid_build(p, gray.data())) throw std::runtime_error(tdm_last_error());
      pyr.push_back(p);
    }
    float calib[4];
    get(in, calib, 4);
    std::vector<float> th(n);
    get(in, th.data(), n);
    std::vector<CudaActivePoints::Point> pts(np);
    std::vector<int> ibuf(np);
    std::vector<float> fbuf(8 * (size_t)np);
    get(in, ibuf.data(), np);
    for (int i = 0; i < np; ++i) pts[i].host = ibuf[i];
    get(in, fbuf.data(), np);
    for (int i = 0; i < np; ++i) pts[i].u = fbuf[i];
    get(in, fbuf.data(), np);
    for (int i = 0; i < np; ++i) pts[i].v = fbuf[i];
    get(in, fbuf.data(), 8 * (size_t)np);
    for (int i = 0; i < np; ++i) for (int k = 0; k < 8; ++k) pts[i].color[k] = fbuf[8 * i + k];
    get(in, fbuf.data(), 8 * (size_t)np);
    for (int i = 0; i < np; ++i) for (int k = 0; k < 8; ++k) pts[i].weights[k] = fbuf[8 * i + k];
    get(in, fbuf.data(), np);
    for (int i = 0; i < np; ++i) pts[i].maxRelBaseline = fbuf[i];
    get(in, ibuf.data(), np);
    for (int i = 0; i < np; ++i) pts[i].numGoodResiduals = ibuf[i];
    std::vector<int> res_point(m), res_target(m);
    get(in, res_point.data(), m);
    get(in, res_target.data(), m);

    CudaActivePoints act(w, h, np > 0 ? np : 1);
    act.load(n, pts, res_point, res_target);
    std::vector<float> ids(np), idz(np), pcf(27ull * n * n);
    std::vector<CudaActivePoints::Precalc> pc(n * n);
    for (int s = 0; s < steps; ++s) {
      int fa[2];
      get(in, fa, 2);
      get(in, ids.data(), np);
      get(in, idz.data(), np);
      get(in, pcf.data(), pcf.size());
      for (int k = 0; k < n * n; ++k) {
        const float *d = pcf.data() + 27ull * k;
        CudaActivePoints::Precalc &p = pc[k];
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c) { p.PRE_KRKiTll(r, c) = d[3 * r + c]; p.PRE_RTll_0(r, c) = d[12 + 3 * r + c]; }
        for (int r = 0; r < 3; ++r) { p.PRE_KtTll(r) = d[9 + r]; p.PRE_tTll_0(r) = d[21 + r]; }
        p.PRE_aff_mode(0) = d[24]; p.PRE_aff_mode(1) = d[25]; p.PRE_b0_mode = d[26];
      }
      CudaActivePoints::Result r;
      act.linearize(pyr, pc, th, calib[0], calib[1], calib[2], calib[3], ids, idz, fa[0] != 0, &r);
      if (fa[1]) act.applyRes();
      th[n - 1] = r.newFrameEnergyTH;
      put(out, &r.energy, 1);
      put(out, &r.newFrameEnergyTH, 1);
      put(out, r.state_NewState.data(), m);
      put(out, r.state_NewEnergy.data(), m);
      put(out, r.state_NewEnergyWithOutlier.data(), m);
      for (int k = 0; k < m; ++k) put(out, &r.centerProjectedTo[k](0), 3);
      put(out, r.jacobians.data(), r.jacobians.size());
      if (fa[0]) {
        put(out, r.state_state.data(), m);
        put(out, r.removed.data(), m);
        put(out, r.maxRelBaseline.data(), np);
        put(out, r.numGoodResiduals.data(), np);
      }
    }
    printf("shim_linearize: OK (%d points, %d residuals, %d steps)\n", np, m, steps);
  } catch (std::exception const &e) {
    printf("shim_linearize: %s\n", e.what());
    rc = 1;
  }
  for (tdm_pyramid *p : pyr) tdm_pyramid_destroy(p);
  fclose(in);
  fclose(out);
  return rc;
}
