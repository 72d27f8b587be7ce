// Test infrastructure (never linked into the product): harness around the motion-hypothesis loop of the REFERENCE's
//   FullSystem::trackNewCoarse      tandem/src/FullSystem/FullSystem.cpp:538-617
// cut out of the file where it lies by oracle/ref_build_retrack.mk (-> oracle/_ref/gen/retrack.inc, git-ignored build output)
// and compiled here, unmodified, with rgbd_flag = false and setting_debugout_runquiet = true.  Purpose: pin
// oracle/retrack_driver.py (SURVEY.md 8f n6).  The stand-in `coarseTracker->trackNewestCoarse` is the reference's own body of
// CoarseTracker::trackNewestCoarse (CoarseTracker.cpp:750-936) through ref_track_pyramid of oracle/ref_wrap_pyramid.cpp, linked
// into the same library, with every level evaluated by the per-level C callbacks - the pin plugs the SAME tracker oracles into
// this loop and into retrack_driver.track_new_coarse.  What is the reference's: the try loop, minResForAbort = achievedRes, the
// winner test, the achievedRes takeover, the break test and the no-winner fallback (and, below them, everything the n5 harness
// pins).  What is the harness's: the stand-in types (Vec5::Constant, a copy-only SE3, AffLight), which live in a namespace of
// their own so that they cannot collide with ref_wrap_pyramid.cpp's.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include <Eigen/Dense>   // tests/cpp/eigen_stub

typedef void (*CalcResFn)(void* user, int lvl, const double* refToNew16_rowmajor, float new_exposure, const double* aff2, float cutoffTH,
                          double* res6);
typedef void (*CalcGFn)(void* user, int lvl, const double* refToNew16_rowmajor, float new_exposure, const double* aff2,
                        double* H64_rowmajor, double* b8);
extern "C" int ref_track_pyramid(void* user, CalcResFn res, CalcGFn g, int coarsest, double* T16, double* aff2, float new_exposure,
                                 float ref_exposure, const double* ref_aff2, float coarse_cutoff, float mode_a, float mode_b,
                                 const double* min_res5, double* out_last_res5, double* out_flow3, int* counts5, int* repeated_level);

namespace retrack {

typedef Eigen::Matrix<double, 3, 1> Vec3;
struct Vec5 : Eigen::Matrix<double, 5, 1> {
  static Vec5 Constant(double v) { Vec5 m; m.setConstant(v); return m; }
};
struct SE3 {             // the loop only copies poses: a row-major 4x4
  double m[16];
  SE3() { for (int i = 0; i < 16; ++i) m[i] = (i % 5 == 0) ? 1.0 : 0.0; }
};
struct AffLight {        // util/NumType.h:166-171
  AffLight(double a_, double b_) : a(a_), b(b_) {}
  AffLight() : a(0), b(0) {}
  double a, b;
};
struct FrameHessian {};

static bool rgbd_flag = false;
static bool setting_debugout_runquiet = true;
static float setting_reTrackThreshold = 1.5f;

struct TryOut {          // what the stand-in saw of one trackNewestCoarse call
  int ok, repeated_level, counts[5];
  double T[16], aff[2], min_res[5], last_res[5];
};

struct CoarseTracker {   // CoarseTracker::trackNewestCoarse = the reference's body through ref_track_pyramid
  Vec5 lastResiduals;
  Vec3 lastFlowIndicators;
  void* user;
  CalcResFn res;
  CalcGFn g;
  float new_exposure, ref_exposure, coarse_cutoff, mode_a, mode_b;
  const double* ref_aff;
  std::vector<TryOut> seen;
  bool trackNewestCoarse(FrameHessian*, SE3& lastToNew_out, AffLight& aff_g2l_out, int coarsestLvl, Vec5 minResForAbort) {
    TryOut t;
    double a[2] = {aff_g2l_out.a, aff_g2l_out.b}, flow[3];
    for (int i = 0; i < 5; ++i) t.min_res[i] = minResForAbort[i];
    t.ok = ref_track_pyramid(user, res, g, coarsestLvl, lastToNew_out.m, a, new_exposure, ref_exposure, ref_aff, coarse_cutoff, mode_a,
                             mode_b, t.min_res, t.last_res, flow, t.counts, &t.repeated_level);
    aff_g2l_out = AffLight(a[0], a[1]);
    for (int i = 0; i < 5; ++i) lastResiduals[i] = t.last_res[i];
    for (int i = 0; i < 3; ++i) lastFlowIndicators[i] = flow[i];
    for (int i = 0; i < 16; ++i) t.T[i] = lastToNew_out.m[i];
    t.aff[0] = a[0]; t.aff[1] = a[1];
    seen.push_back(t);
    return t.ok != 0;
  }
  bool trackNewestCoarseDense(FrameHessian*, SE3&, AffLight&, int, Vec5) { std::abort(); }   // rgbd_flag is false
};

struct System {
  CoarseTracker* coarseTracker = nullptr;
  Vec5 lastCoarseRMSE;
  int pyrLevelsUsed = 0;
  Vec3 out_flow;
  SE3 out_pose;
  AffLight out_aff;
  bool out_have_one_good = false;
  int out_tries = 0;
  void trackNewCoarse(FrameHessian* fh, std::vector<SE3> const& lastF_2_fh_tries, AffLight aff_last_2_l) {
#include "_ref/gen/retrack.inc"   // FullSystem.cpp:538-617, verbatim (ends with `lastCoarseRMSE = achievedRes;`)
    out_flow = flowVecs;
    out_pose = lastF_2_fh;
    out_aff = aff_g2l;
    out_have_one_good = haveOneGood;
    out_tries = tryIterations;
  }
};

}  // namespace retrack

extern "C" {
// tries16: n_tries row-major 4x4 poses (lastF_2_fh_tries); last_coarse_rmse5 in/out (lastCoarseRMSE).  Returns tryIterations.
// out_*: lastF_2_fh, aff_g2l, flowVecs, haveOneGood, and the index of the last winner (the last try whose ok result is the
// output pose; -1: none).  try_*: n_tries entries of what each trackNewestCoarse call received (minResForAbort) and returned.
int ref_track_new_coarse(void* user, CalcResFn res, CalcGFn g, int coarsest, const double* tries16, int n_tries, const double* aff_last2,
                         float new_exposure, float ref_exposure, const double* ref_aff2, float coarse_cutoff, float mode_a, float mode_b,
                         double* last_coarse_rmse5, float retrack_threshold, double* out_T16, double* out_aff2, double* out_flow3,
                         int* out_have_one_good, int* out_winner, int* try_ok, double* try_T16, double* try_aff2, double* try_min_res5,
                         double* try_last_res5, int* try_counts5, int* try_repeated_level) {
  using namespace retrack;
  setting_reTrackThreshold = retrack_threshold;
  CoarseTracker ct;
  ct.user = user; ct.res = res; ct.g = g;
  ct.new_exposure = new_exposure; ct.ref_exposure = ref_exposure; ct.ref_aff = ref_aff2;
  ct.coarse_cutoff = coarse_cutoff; ct.mode_a = mode_a; ct.mode_b = mode_b;
  System S;
  S.coarseTracker = &ct;
  S.pyrLevelsUsed = coarsest + 1;
  for (int i = 0; i < 5; ++i) S.lastCoarseRMSE[i] = last_coarse_rmse5[i];
  std::vector<SE3> tries((size_t)n_tries);
  for (int k = 0; k < n_tries; ++k)
    for (int i = 0; i < 16; ++i) tries[(size_t)k].m[i] = tries16[16 * k + i];
  FrameHessian fh;
  S.trackNewCoarse(&fh, tries, AffLight(aff_last2[0], aff_last2[1]));
  for (int i = 0; i < 5; ++i) last_coarse_rmse5[i] = S.lastCoarseRMSE[i];
  for (int i = 0; i < 16; ++i) out_T16[i] = S.out_pose.m[i];
  out_aff2[0] = S.out_aff.a; out_aff2[1] = S.out_aff.b;
  for (int i = 0; i < 3; ++i) out_flow3[i] = S.out_flow[i];
  *out_have_one_good = S.out_have_one_good ? 1 : 0;
  *out_winner = -1;
  for (size_t k = 0; k < ct.seen.size(); ++k) {
    const TryOut& t = ct.seen[k];
    bool same = t.ok && S.out_have_one_good && t.aff[0] == S.out_aff.a && t.aff[1] == S.out_aff.b;
    for (int i = 0; i < 16; ++i) same = same && t.T[i] == S.out_pose.m[i];
    if (same) *out_winner = (int)k;
    try_ok[k] = t.ok; try_repeated_level[k] = t.repeated_level;
    for (int i = 0; i < 16; ++i) try_T16[16 * k + i] = t.T[i];
    for (int i = 0; i < 2; ++i) try_aff2[2 * k + i] = t.aff[i];
    for (int i = 0; i < 5; ++i) {
      try_min_res5[5 * k + i] = t.min_res[i]; try_last_res5[5 * k + i] = t.last_res[i]; try_counts5[5 * k + i] = t.counts[i];
    }
  }
  return S.out_tries;
}
}
