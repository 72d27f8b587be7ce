// Links CudaActivePoints::accumulate / resubstitute (shims/cuda_active_points.cpp) against libtandem_b200.so and runs one
// solveSystemF on a window read from argv[1] (written by tests/test_accumulate_gpu.py): the frames' grey images, the
// calibration, the points, activeResiduals, one linearize (idepth_scaled, idepth_zero_scaled, precalc) without Jacobians and
// its apply, then accumulate with the inputs that follow (adHost, adTarget as row-major records [h + n t], prior,
// delta_prior, cPrior, cDeltaF, priorF, deltaF) and resubstitute with the x that follows.  Every output is written to
// argv[2], so the test can compare it with the C oracle.
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
  if (argc < 3) { printf("usage: shim_accumulate IN OUT\n"); return 2; }
  FILE *in = fopen(argv[1], "rb");
  FILE *out = fopen(argv[2], "wb");
  if (!in || !out) { printf("cannot open the files\n"); return 2; }
  std::vector<tdm_pyramid *> pyr;
  int rc = 0;
  try {
    int hdr[6];
    get(in, hdr, 6);
    const int w = hdr[0], h = hdr[1], n = hdr[2], np = hdr[3], m = hdr[4];
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
    act.linearize(pyr, pc, th, calib[0], calib[1], calib[2], calib[3], ids, idz, false, &r, false);
    act.applyRes();
    CudaActivePoints::SystemInputs si;
    si.adHost.resize(n * n); si.adTarget.resize(n * n); si.prior.resize(n); si.delta_prior.resize(n);
    std::vector<double> dbuf(64);
    for (auto *v : {&si.adHost, &si.adTarget})
      for (int k = 0; k < n * n; ++k) {
        get(in, dbuf.data(), 64);
        for (int a = 0; a < 8; ++a) for (int b = 0; b < 8; ++b) (*v)[k](a, b) = dbuf[8 * a + b];
      }
    for (auto *v : {&si.prior, &si.delta_prior})
      for (int f = 0; f < n; ++f) {
        get(in, dbuf.data(), 8);
        for (int i = 0; i < 8; ++i) (*v)[f](i) = dbuf[i];
      }
    get(in, dbuf.data(), 4);
    for (int i = 0; i < 4; ++i) si.cPrior(i) = dbuf[i];
    float cd[4];
    get(in, cd, 4);
    for (int i = 0; i < 4; ++i) si.cDeltaF(i) = cd[i];
    si.priorF.resize(np); si.deltaF.resize(np);
    get(in, si.priorF.data(), np);
    get(in, si.deltaF.data(), np);
    const int dim = 8 * n + 4;
    std::vector<double> x(dim);
    get(in, x.data(), dim);
    CudaActivePoints::System sys;
    act.accumulate(si, &sys);
    std::vector<float> step;
    act.resubstitute(x, &step);
    put(out, sys.H_top.data(), sys.H_top.size());
    put(out, sys.b_top.data(), sys.b_top.size());
    put(out, sys.H_sc.data(), sys.H_sc.size());
    put(out, sys.b_sc.data(), sys.b_sc.size());
    put(out, &sys.resInA, 1);
    put(out, sys.HdiF.data(), np);
    put(out, sys.idepth_hessian.data(), np);
    put(out, step.data(), np);
    printf("shim_accumulate: OK (%d points, %d residuals, %d active)\n", np, m, sys.resInA);
  } catch (std::exception const &e) {
    printf("shim_accumulate: %s\n", e.what());
    rc = 1;
  }
  for (tdm_pyramid *p : pyr) tdm_pyramid_destroy(p);
  fclose(in);
  fclose(out);
  return rc;
}
