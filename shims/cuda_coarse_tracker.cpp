// class CudaCoarseTracker over the tandem_b200 C ABI (replaces tandem/libdr/cuda_coarse_tracker/src/cuda_coarse_tracker.cpp).
// Error convention of the reference: throw std::runtime_error (cuda_coarse_tracker.cpp:82,105-106,359).
#include "cuda_coarse_tracker/cuda_coarse_tracker.h"

#include <chrono>
#include <stdexcept>
#include <string>
#include <vector>

#include "tandem_b200.h"

static void chk(int rc, const char* where) {
  if (rc != TDM_OK) throw std::runtime_error(std::string(where) + ": " + tdm_last_error());
}

CudaCoarseTracker::CudaCoarseTracker(int w, int h, float huber, float cutoff)
    : w(w), h(h), setting_huberTH(huber), setting_coarseCutoffTH(cutoff) {}

CudaCoarseTracker::~CudaCoarseTracker() { free(); }

void CudaCoarseTracker::init(int n_max_in) {
  if (w * h == 0) throw std::runtime_error("\"CudaCoarseTracker::init has w*h==0.");
  if (handle_) throw std::runtime_error("\"Cannot call CudaCoarseTracker::init more than once.");
  chk(tdm_tracker_create(w, h, setting_huberTH, setting_coarseCutoffTH, n_max_in, 0, &handle_), "CudaCoarseTracker::init");
}

void CudaCoarseTracker::free() {
  if (handle_) tdm_tracker_destroy(handle_);
  handle_ = nullptr;
}

void CudaCoarseTracker::setK(int w_in, int h_in, float fx, float fy, float cx, float cy) {
  chk(tdm_tracker_set_k(handle_, w_in, h_in, fx, fy, cx, cy), "CudaCoarseTracker::setK");
}

void CudaCoarseTracker::setReference(int n, float const* u, float const* v, float const* idepth, float const* color,
                                     float ref_exposure, Eigen::Vector2d const& ref_aff) {
  const double a[2] = {ref_aff(0), ref_aff(1)};
  chk(tdm_tracker_set_reference(handle_, n, u, v, idepth, color, ref_exposure, a), "CudaCoarseTracker::setReference");
}

void CudaCoarseTracker::setNew(float const* dInew) { chk(tdm_tracker_set_new(handle_, dInew), "CudaCoarseTracker::setNew"); }

static void to_row_major(Eigen::Matrix<double, 4, 4> const& T, double out[16]) {
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) out[4 * r + c] = T(r, c);
}

Eigen::Matrix<double, 6, 1> CudaCoarseTracker::calcRes(Eigen::Matrix<double, 4, 4> const& refToNew, float new_exposure,
                                                        Eigen::Vector2d const& aff, float cutoffTH) {
  double T[16], res[6];
  to_row_major(refToNew, T);
  const double a[2] = {aff(0), aff(1)};
  chk(tdm_tracker_calc_res(handle_, T, new_exposure, a, cutoffTH, res), "CudaCoarseTracker::calcRes");
  Eigen::Matrix<double, 6, 1> r;
  for (int i = 0; i < 6; ++i) r(i) = res[i];
  return r;
}

void CudaCoarseTracker::calcG(Eigen::Matrix<double, 8, 8>& H_out, Eigen::Matrix<double, 8, 1>& b_out, const float new_exposure,
                              const Eigen::Vector2d& aff) {
  double H[64], b[8];
  const double a[2] = {aff(0), aff(1)};
  chk(tdm_tracker_calc_g(handle_, new_exposure, a, H, b), "CudaCoarseTracker::calcG");
  for (int r = 0; r < 8; ++r) {
    for (int c = 0; c < 8; ++c) H_out(r, c) = H[8 * r + c];
    b_out(r) = b[r];
  }
}

Eigen::Matrix<double, 6, 1> CudaCoarseTracker::calcResAndG(Eigen::Matrix<double, 4, 4> const& refToNew, float new_exposure,
                                                            Eigen::Vector2d const& aff, float cutoffTH,
                                                            Eigen::Matrix<double, 8, 8>& H_out,
                                                            Eigen::Matrix<double, 8, 1>& b_out) {
  double T[16], res[6], H[64], b[8];
  to_row_major(refToNew, T);
  const double a[2] = {aff(0), aff(1)};
  chk(tdm_tracker_calc_res_g(handle_, T, new_exposure, a, cutoffTH, res, H, b), "CudaCoarseTracker::calcResAndG");
  Eigen::Matrix<double, 6, 1> r;
  for (int i = 0; i < 6; ++i) r(i) = res[i];
  for (int rr = 0; rr < 8; ++rr) {
    for (int c = 0; c < 8; ++c) H_out(rr, c) = H[8 * rr + c];
    b_out(rr) = b[rr];
  }
  return r;
}

std::vector<Eigen::Matrix<double, 6, 1>> CudaCoarseTracker::calcResBatch(std::vector<Eigen::Matrix<double, 4, 4>> const& refToNew,
                                                                         float new_exposure, std::vector<Eigen::Vector2d> const& aff,
                                                                         float cutoffTH) {
  if (refToNew.size() != aff.size() || refToNew.empty()) throw std::runtime_error("CudaCoarseTracker::calcResBatch: size mismatch");
  const int n = (int)refToNew.size();
  std::vector<double> T(16 * (size_t)n), a(2 * (size_t)n), res(6 * (size_t)n);
  for (int k = 0; k < n; ++k) {
    to_row_major(refToNew[k], &T[16 * (size_t)k]);
    a[2 * (size_t)k] = aff[k](0); a[2 * (size_t)k + 1] = aff[k](1);
  }
  chk(tdm_tracker_calc_res_batch(handle_, n, T.data(), new_exposure, a.data(), cutoffTH, res.data()), "CudaCoarseTracker::calcResBatch");
  std::vector<Eigen::Matrix<double, 6, 1>> out((size_t)n);
  for (int k = 0; k < n; ++k)
    for (int i = 0; i < 6; ++i) out[(size_t)k](i) = res[6 * (size_t)k + i];
  return out;
}

void CudaCoarseTracker::setNewFromPyramid(tdm_pyramid* pyramid, int level) {
  chk(tdm_tracker_set_new_from_pyramid(handle_, pyramid, level), "CudaCoarseTracker::setNewFromPyramid");
}

int CudaCoarseTracker::setReferenceDense(tdm_fusion* fusion, int render_index, Eigen::Matrix<double, 4, 4> const& T_depth_to_ref,
                                         int tracking_step, bool dense_only, int n_sparse, float const* pc_u, float const* pc_v,
                                         float const* pc_idepth, float const* pc_color, float const* idepth0,
                                         tdm_pyramid* ref_pyramid, float ref_exposure, Eigen::Vector2d const& ref_aff) {
  double T[16];
  to_row_major(T_depth_to_ref, T);
  const double a[2] = {ref_aff(0), ref_aff(1)};
  int pc_n = 0;
  chk(tdm_tracker_set_reference_dense(handle_, nullptr, fusion, render_index, T, tracking_step, dense_only ? 1 : 0, n_sparse,
                                      pc_u, pc_v, pc_idepth, pc_color, idepth0, nullptr, ref_pyramid, ref_exposure, a, &pc_n),
      "CudaCoarseTracker::setReferenceDense");
  return pc_n;
}

CudaCoarseTracker::TrackResult CudaCoarseTracker::track(Eigen::Matrix<double, 4, 4> const& refToNew, Eigen::Vector2d const& aff,
                                                        float new_exposure, float coarseCutoffTH, int maxIterations,
                                                        float lambdaExtrapolationLimit, bool fix_a, bool fix_b) {
  double T[16];
  to_row_major(refToNew, T);
  const double a[2] = {aff(0), aff(1)};
  tdm_track_result r;
  chk(tdm_tracker_track(handle_, T, a, new_exposure, coarseCutoffTH, maxIterations, lambdaExtrapolationLimit, fix_a ? 1 : 0,
                        fix_b ? 1 : 0, &r),
      "CudaCoarseTracker::track");
  TrackResult out;
  for (int rr = 0; rr < 4; ++rr)
    for (int c = 0; c < 4; ++c) out.refToNew(rr, c) = r.ref_to_new[4 * rr + c];
  out.aff_g2l = Eigen::Vector2d(r.aff_g2l[0], r.aff_g2l[1]);
  for (int i = 0; i < 6; ++i) out.res(i) = r.res[i];
  out.iterations = r.iterations;
  out.levelCutoffRepeat = r.cutoff_repeat;
  return out;
}

CudaCoarseTracker::PyramidTrackResult CudaCoarseTracker::trackPyramid(
    std::vector<CudaCoarseTracker*> const& levels, Eigen::Matrix<double, 4, 4> const& refToNew, Eigen::Vector2d const& aff,
    float new_exposure, float coarseCutoffTH, const int maxIterations[5], float lambdaExtrapolationLimit, float affineOptModeA,
    float affineOptModeB, Eigen::Matrix<double, 5, 1> const& minResForAbort) {
  std::vector<tdm_tracker*> h;
  for (CudaCoarseTracker* t : levels) h.push_back(t ? t->handle_ : nullptr);
  double T[16], minRes[5];
  to_row_major(refToNew, T);
  const double a[2] = {aff(0), aff(1)};
  for (int i = 0; i < 5; ++i) minRes[i] = minResForAbort(i);
  tdm_track_pyramid_result r;
  chk(tdm_tracker_track_pyramid(h.data(), (int)h.size() - 1, T, a, new_exposure, coarseCutoffTH, maxIterations, lambdaExtrapolationLimit,
                                affineOptModeA, affineOptModeB, minRes, &r),
      "CudaCoarseTracker::trackPyramid");
  PyramidTrackResult out;
  out.ok = r.ok != 0;
  for (int rr = 0; rr < 4; ++rr)
    for (int c = 0; c < 4; ++c) out.refToNew(rr, c) = r.ref_to_new[4 * rr + c];
  out.aff_g2l = Eigen::Vector2d(r.aff_g2l[0], r.aff_g2l[1]);
  for (int i = 0; i < 5; ++i) {
    out.lastResiduals(i) = r.last_residuals[i];
    out.iterations[i] = r.iterations[i]; out.evaluations[i] = r.evaluations[i]; out.levelCutoffRepeat[i] = r.cutoff_repeat[i];
  }
  for (int i = 0; i < 3; ++i) out.lastFlowIndicators(i) = r.last_flow_indicators[i];
  out.abortedLevel = r.aborted_level; out.repeatedLevel = r.repeated_level;
  return out;
}

std::vector<int> CudaCoarseTracker::setCoarseTrackingRef(
    std::vector<CudaCoarseTracker*> const& levels, bool rgbd_init, int n_points, float const* pt_u, float const* pt_v,
    float const* pt_idepth, float const* pt_hessian, tdm_pyramid* ref_pyramid, tdm_fusion* fusion, int render_index,
    Eigen::Matrix<double, 4, 4> const& T_depth_to_ref, int tracking_step, bool dense_only, float ref_exposure,
    Eigen::Vector2d const& ref_aff) {
  std::vector<tdm_tracker*> h;
  for (CudaCoarseTracker* t : levels) h.push_back(t ? t->handle_ : nullptr);
  double T[16];
  to_row_major(T_depth_to_ref, T);
  const double a[2] = {ref_aff(0), ref_aff(1)};
  int pc_n[5] = {0, 0, 0, 0, 0};
  chk(tdm_tracker_set_coarse_tracking_ref(h.data(), (int)h.size(), rgbd_init ? 1 : 0, n_points, pt_u, pt_v, pt_idepth, pt_hessian,
                                          ref_pyramid, nullptr, fusion, render_index, T, tracking_step, dense_only ? 1 : 0,
                                          ref_exposure, a, pc_n),
      "CudaCoarseTracker::setCoarseTrackingRef");
  return std::vector<int>(pc_n, pc_n + (h.size() < 5 ? h.size() : 5));
}

std::vector<int> CudaCoarseTracker::setCoarseTrackingRef(
    std::vector<CudaCoarseTracker*> const& levels, bool rgbd_init, int n_points, float const* pt_u, float const* pt_v,
    float const* pt_idepth, float const* pt_hessian, tdm_pyramid* ref_pyramid, tdm_fusion* fusion, int render_index,
    Eigen::Matrix<double, 4, 4> const& T_depth_to_ref, int tracking_step, bool dense_only, float ref_exposure,
    Eigen::Vector2d const& ref_aff, float quantile_fraction, int* pc_n_nodia, float* depth_quantile) {
  std::vector<tdm_tracker*> h;
  for (CudaCoarseTracker* t : levels) h.push_back(t ? t->handle_ : nullptr);
  double T[16];
  to_row_major(T_depth_to_ref, T);
  const double a[2] = {ref_aff(0), ref_aff(1)};
  int pc_n[5] = {0, 0, 0, 0, 0};
  tdm_coarse_nodia_result r;
  chk(tdm_tracker_set_coarse_tracking_ref_nodia(h.data(), (int)h.size(), rgbd_init ? 1 : 0, n_points, pt_u, pt_v, pt_idepth,
                                                pt_hessian, ref_pyramid, nullptr, fusion, render_index, T, tracking_step,
                                                dense_only ? 1 : 0, ref_exposure, a, quantile_fraction, pc_n, &r),
      "CudaCoarseTracker::setCoarseTrackingRef");
  if (pc_n_nodia) *pc_n_nodia = r.pc_n_nodia;
  if (depth_quantile) *depth_quantile = r.depth_quantile;
  return std::vector<int>(pc_n, pc_n + (h.size() < 5 ? h.size() : 5));
}

CudaCoarseTracker::NewCoarseResult CudaCoarseTracker::trackNewCoarse(
    std::vector<CudaCoarseTracker*> const& levels, std::vector<Eigen::Matrix<double, 4, 4>> const& tries,
    Eigen::Vector2d const& aff_last_2_l, float new_exposure, float coarseCutoffTH, const int maxIterations[5],
    float lambdaExtrapolationLimit, float affineOptModeA, float affineOptModeB, Eigen::Matrix<double, 5, 1> const& lastCoarseRMSE,
    float reTrackThreshold) {
  std::vector<tdm_tracker*> h;
  for (CudaCoarseTracker* t : levels) h.push_back(t ? t->handle_ : nullptr);
  std::vector<double> T(16 * tries.size() + 1);
  for (size_t k = 0; k < tries.size(); ++k) to_row_major(tries[k], &T[16 * k]);
  const double a[2] = {aff_last_2_l(0), aff_last_2_l(1)};
  double rmse[5];
  for (int i = 0; i < 5; ++i) rmse[i] = lastCoarseRMSE(i);
  tdm_track_new_coarse_result r;
  chk(tdm_tracker_track_new_coarse(h.data(), (int)h.size() - 1, T.data(), (int)tries.size(), a, new_exposure, coarseCutoffTH, maxIterations,
                                   lambdaExtrapolationLimit, affineOptModeA, affineOptModeB, rmse, reTrackThreshold, &r, nullptr),
      "CudaCoarseTracker::trackNewCoarse");
  NewCoarseResult out;
  for (int rr = 0; rr < 4; ++rr)
    for (int c = 0; c < 4; ++c) out.lastF_2_fh(rr, c) = r.ref_to_new[4 * rr + c];
  out.aff_g2l = Eigen::Vector2d(r.aff_g2l[0], r.aff_g2l[1]);
  for (int i = 0; i < 3; ++i) out.flowVecs(i) = r.flow_vecs[i];
  for (int i = 0; i < 5; ++i) out.achievedRes(i) = r.achieved_res[i];
  out.haveOneGood = r.have_one_good != 0;
  out.tryIterations = r.tries;
  out.winner = r.winner;
  return out;
}

void CudaCoarseTracker::synchronize() { chk(tdm_tracker_synchronize(handle_), "CudaCoarseTracker::synchronize"); }

void CudaCoarseTracker::startTiming() {
  if (timing_) throw std::runtime_error("CudaCoarseTracker::startTiming. Did not destroy events before correctly.");
  synchronize();
  timing_ = true;
  t_start_ = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

float CudaCoarseTracker::endTimingMilliseconds() {
  if (!timing_) throw std::runtime_error("CudaCoarseTracker::endTimingMilliseconds. Did not start before.");
  synchronize();
  timing_ = false;
  return (float)(std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count() - t_start_);
}
