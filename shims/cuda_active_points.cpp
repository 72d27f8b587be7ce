// CudaActivePoints over the tandem_b200 C ABI.  Errors throw std::runtime_error, as the tracker shim's do.
#include "cuda_coarse_tracker/cuda_active_points.h"

#include <stdexcept>
#include <string>

#include "tandem_b200.h"

static void chk(int rc, const char *where) {
  if (rc != TDM_OK) throw std::runtime_error(std::string(where) + ": " + tdm_last_error());
}

CudaActivePoints::CudaActivePoints(int w, int h, int capacity_points, int device) {
  chk(tdm_active_create(w, h, capacity_points, nullptr, device, &handle_), "CudaActivePoints");
}

CudaActivePoints::~CudaActivePoints() { tdm_active_destroy(handle_); }

void CudaActivePoints::load(int n_frames, std::vector<Point> const &points, std::vector<int> const &res_point,
                            std::vector<int> const &res_target) {
  if (res_point.size() != res_target.size()) throw std::runtime_error("CudaActivePoints::load: sizes differ");
  const size_t n = points.size();
  std::vector<int> host(n), good(n);
  std::vector<float> u(n), v(n), color(8 * n), weights(8 * n), mrb(n);
  for (size_t i = 0; i < n; ++i) {
    const Point &p = points[i];
    host[i] = p.host; u[i] = p.u; v[i] = p.v; mrb[i] = p.maxRelBaseline; good[i] = p.numGoodResiduals;
    for (int k = 0; k < 8; ++k) { color[8 * i + k] = p.color[k]; weights[8 * i + k] = p.weights[k]; }
  }
  chk(tdm_active_load(handle_, n_frames, (int)n, host.data(), u.data(), v.data(), color.data(), weights.data(), mrb.data(),
                      good.data(), (int)res_point.size(), res_point.data(), res_target.data()),
      "CudaActivePoints::load");
  n_frames_ = n_frames; n_points_ = (int)n; n_res_ = (int)res_point.size();
}

void CudaActivePoints::linearize(std::vector<tdm_pyramid *> const &frames, std::vector<Precalc> const &precalc,
                                 std::vector<float> const &frameEnergyTH, float fxl, float fyl, float cxl, float cyl,
                                 std::vector<float> const &idepth_scaled, std::vector<float> const &idepth_zero_scaled,
                                 bool fixLinearization, Result *out, bool jacobians) {
  const int n = n_frames_, m = n_res_, np = n_points_;
  if ((int)frames.size() != n || (int)precalc.size() != n * n || (int)frameEnergyTH.size() != n ||
      (int)idepth_scaled.size() != np || (int)idepth_zero_scaled.size() != np)
    throw std::runtime_error("CudaActivePoints::linearize: sizes differ from the loaded window");
  std::vector<float> pc(27ull * n * n);
  for (int k = 0; k < n * n; ++k) {
    const Precalc &p = precalc[k];
    float *d = pc.data() + 27ull * k;
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) { d[3 * r + c] = p.PRE_KRKiTll(r, c); d[12 + 3 * r + c] = p.PRE_RTll_0(r, c); }
    for (int r = 0; r < 3; ++r) { d[9 + r] = p.PRE_KtTll(r); d[21 + r] = p.PRE_tTll_0(r); }
    d[24] = p.PRE_aff_mode(0); d[25] = p.PRE_aff_mode(1); d[26] = p.PRE_b0_mode;
  }
  const float calib[4] = {fxl, fyl, cxl, cyl};
  Result &r = *out;
  r.state_NewState.resize(m); r.state_NewEnergy.resize(m); r.state_NewEnergyWithOutlier.resize(m);
  std::vector<float> center(3ull * m);
  r.jacobians.resize(jacobians ? (size_t)TDM_JACOBIAN_FLOATS * m : 0);
  r.state_state.resize(fixLinearization ? m : 0); r.removed.resize(fixLinearization ? m : 0);
  r.maxRelBaseline.resize(fixLinearization ? np : 0); r.numGoodResiduals.resize(fixLinearization ? np : 0);
  chk(tdm_active_linearize(handle_, const_cast<tdm_pyramid *const *>(frames.data()), pc.data(), frameEnergyTH.data(), calib,
                           idepth_scaled.data(), idepth_zero_scaled.data(), fixLinearization ? 1 : 0, &r.energy, &r.newFrameEnergyTH,
                           r.state_NewState.data(), r.state_NewEnergy.data(), r.state_NewEnergyWithOutlier.data(), center.data(),
                           jacobians ? r.jacobians.data() : nullptr, fixLinearization ? r.state_state.data() : nullptr,
                           fixLinearization ? r.removed.data() : nullptr, fixLinearization ? r.maxRelBaseline.data() : nullptr,
                           fixLinearization ? r.numGoodResiduals.data() : nullptr),
      "CudaActivePoints::linearize");
  r.centerProjectedTo.resize(m);
  for (int k = 0; k < m; ++k)
    for (int c = 0; c < 3; ++c) r.centerProjectedTo[k](c) = center[3ull * k + c];
}

void CudaActivePoints::applyRes() { chk(tdm_active_apply_res(handle_), "CudaActivePoints::applyRes"); }

void CudaActivePoints::accumulate(SystemInputs const &in, System *out) {
  const int n = n_frames_, dim = 8 * n + 4;
  if ((int)in.adHost.size() != n * n || (int)in.adTarget.size() != n * n || (int)in.prior.size() != n ||
      (int)in.delta_prior.size() != n || (int)in.priorF.size() != n_points_ || (int)in.deltaF.size() != n_points_)
    throw std::runtime_error("CudaActivePoints::accumulate: sizes differ from the loaded window");
  // the C ABI's 8x8 records are row-major; Eigen's fixed matrices are column-major
  std::vector<double> aH(64 * n * n), aT(64 * n * n), pr(8 * n), dp(8 * n);
  for (int k = 0; k < n * n; ++k)
    for (int r = 0; r < 8; ++r)
      for (int c = 0; c < 8; ++c) {
        aH[64 * k + 8 * r + c] = in.adHost[k](r, c);
        aT[64 * k + 8 * r + c] = in.adTarget[k](r, c);
      }
  for (int f = 0; f < n; ++f)
    for (int i = 0; i < 8; ++i) { pr[8 * f + i] = in.prior[f][i]; dp[8 * f + i] = in.delta_prior[f][i]; }
  out->dim = dim;
  out->H_top.resize((size_t)dim * dim); out->H_sc.resize((size_t)dim * dim);
  out->b_top.resize(dim); out->b_sc.resize(dim);
  out->HdiF.resize(n_points_); out->idepth_hessian.resize(n_points_);
  chk(tdm_active_accumulate(handle_, aH.data(), aT.data(), pr.data(), dp.data(), in.cPrior.data(), in.cDeltaF.data(), in.priorF.data(),
                            in.deltaF.data(), out->H_top.data(), out->b_top.data(), out->H_sc.data(), out->b_sc.data(), &out->resInA,
                            out->HdiF.data(), out->idepth_hessian.data()),
      "CudaActivePoints::accumulate");
}

void CudaActivePoints::resubstitute(std::vector<double> const &x, std::vector<float> *step) {
  if ((int)x.size() != 8 * n_frames_ + 4) throw std::runtime_error("CudaActivePoints::resubstitute: x needs 8 n_frames + 4 entries");
  step->resize(n_points_);
  chk(tdm_active_resubstitute(handle_, x.data(), step->data()), "CudaActivePoints::resubstitute");
}
