// Test infrastructure (never linked into the product): harness around the WHOLE coarse-to-fine body of the REFERENCE's
//   CoarseTracker::trackNewestCoarse      tandem/src/FullSystem/CoarseTracker.cpp:750-936
// cut out of the file where it lies by oracle/ref_build_pyramid.mk (-> oracle/_ref/gen/track_pyramid.inc, git-ignored build
// output) and compiled here, unmodified, against a stand-in for Eigen / Sophus (tests/cpp/eigen_stub) and the members it
// touches.  Purpose: pin oracle/pyramid_driver.py (SURVEY.md 8f n5).  `cudaCoarseTracker` is null, so every level's residual /
// normal-equation evaluation goes through the member calcRes(lvl, ...) / calcGSSSE(lvl, ...), which dispatch to two C
// callbacks with the level number - the pin plugs the SAME per-level tracker objects into this loop and into
// pyramid_driver.track_pyramid.  What is the reference's: the level loop, the cutoff doubling, the LM rules, lastResiduals /
// lastFlowIndicators, the abort test, the repeat-level rule, the affine checks and the fixed-parameter reset.  What is the
// stand-in's: the LDLT solves and SE3::exp (as in oracle/ref_wrap_lm.cpp).
#include <cassert>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <iostream>

#include <Eigen/Dense>   // tests/cpp/eigen_stub

#define PYR_LEVELS 6
#define SCALE_XI_ROT 1.0f      /* HessianBlocks.h:60-66 */
#define SCALE_XI_TRANS 0.5f
#define SCALE_A 10.0f
#define SCALE_B 1000.0f
typedef Eigen::Matrix<double, 8, 8> Mat88;
typedef Eigen::Matrix<double, 8, 1> Vec8;
typedef Eigen::Matrix<double, 7, 1> Vec7;
typedef Eigen::Matrix<double, 6, 1> Vec6;
typedef Eigen::Matrix<double, 5, 1> Vec5;
typedef Eigen::Matrix<double, 3, 1> Vec3;
typedef Eigen::Matrix<double, 2, 1> Vec2;
typedef Eigen::Matrix<float, 2, 1> Vec2f;
typedef Eigen::Matrix<double, 3, 3> Mat33;
typedef Eigen::Matrix<double, 4, 4> Mat44;

// ---- stand-in for Sophus::SE3d (tangent = (upsilon, omega), left-multiplicative update as the loop uses it)
class SE3 {
 public:
  Mat33 R;
  Vec3 t;
  SE3() { R = Mat33::Identity(); t.setZero(); }
  static SE3 exp(const Vec6& xi) {
    const Vec3 ups(xi[0], xi[1], xi[2]), om(xi[3], xi[4], xi[5]);
    const double th = om.norm();
    Mat33 Om; Om.setZero();
    Om(0, 1) = -om[2]; Om(0, 2) = om[1]; Om(1, 0) = om[2]; Om(1, 2) = -om[0]; Om(2, 0) = -om[1]; Om(2, 1) = om[0];
    double A, B, C;
    if (th < 1e-8) { A = 1.0 - th * th / 6; B = 0.5 - th * th / 24; C = 1.0 / 6 - th * th / 120; }
    else { A = std::sin(th) / th; B = (1 - std::cos(th)) / (th * th); C = (th - std::sin(th)) / (th * th * th); }
    const Mat33 Om2 = Om * Om;
    SE3 o;
    Mat33 V;
    for (int i = 0; i < 9; ++i) {
      const double I = (i % 4 == 0) ? 1.0 : 0.0;
      o.R.d[i] = I + A * Om.d[i] + B * Om2.d[i];
      V.d[i] = I + B * Om.d[i] + C * Om2.d[i];
    }
    o.t = V * ups;
    return o;
  }
  SE3 operator*(const SE3& b) const { SE3 o; o.R = R * b.R; o.t = R * b.t + t; return o; }
  Mat44 matrix() const {
    Mat44 m; m.setZero();
    for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) m(r, c) = R(r, c); m(r, 3) = t(r); }
    m(3, 3) = 1;
    return m;
  }
  Vec6 log() const { Vec6 v; v.setZero(); return v; }   // only inside `if (debugPrint)` printouts
};

struct AffLight {   // util/NumType.h:166-192
  AffLight(double a_, double b_) : a(a_), b(b_) {}
  AffLight() : a(0), b(0) {}
  double a, b;
  static Vec2 fromToVecExposure(float exposureF, float exposureT, AffLight g2F, AffLight g2T) {
    if (exposureF == 0 || exposureT == 0) exposureT = exposureF = 1;
    const double a = std::exp(g2T.a - g2F.a) * exposureT / exposureF;
    const double b = g2T.b - a * g2F.b;
    return Vec2(a, b);
  }
  Vec2 vec() { return Vec2(a, b); }
};

typedef void (*CalcResFn)(void* user, int lvl, const double* refToNew16_rowmajor, float new_exposure, const double* aff2, float cutoffTH,
                          double* res6);
typedef void (*CalcGFn)(void* user, int lvl, const double* refToNew16_rowmajor, float new_exposure, const double* aff2,
                        double* H64_rowmajor, double* b8);

struct CudaCoarseTrackerStub {   // never called (cudaCoarseTracker is null), but the level-0 branches must compile
  void setNew(float const*) { std::abort(); }
  Vec6 calcRes(const Mat44&, float, Vec2, float) { std::abort(); }
  void calcG(Mat88&, Vec8&, float, Vec2) { std::abort(); }
};

struct FrameHessian { float ab_exposure = 1; Eigen::Vector3f* dIp[PYR_LEVELS] = {}; };

// ---- settings / members of CoarseTracker the body names (settings.h:116-117: the affine modes are floats)
static float setting_coarseCutoffTH = 20;
static float setting_affineOptModeA = 0, setting_affineOptModeB = 0;
static bool setting_debugout_runquiet = true;
static bool debugPrint = false;

static void row_major(const SE3& T, double* o) {
  const Mat44 M = T.matrix();
  for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) o[4 * r + c] = M(r, c);
}

namespace {
struct Loop {
  CudaCoarseTrackerStub* cudaCoarseTracker = nullptr;
  FrameHessian* newFrame = nullptr;
  FrameHessian* lastRef = nullptr;
  AffLight lastRef_aff_g2l;
  Vec5 lastResiduals;
  Vec3 lastFlowIndicators;
  void* user = nullptr;
  CalcResFn res_cb = nullptr;
  CalcGFn g_cb = nullptr;
  int n_res[5] = {0, 0, 0, 0, 0};
  int prev_lvl = -1, repeated_level = -1;
  float prev_cut = 0;

  // CoarseTracker::calcRes / calcGSSSE of level lvl (CoarseTracker.cpp:376-639), evaluated by the callbacks
  Vec6 calcRes(int lvl, const SE3& refToNew, AffLight aff, float cutoffTH) {
    double T[16], a[2] = {aff.a, aff.b}, r[6];
    row_major(refToNew, T);
    res_cb(user, lvl, T, newFrame->ab_exposure, a, cutoffTH, r);
    ++n_res[lvl];
    // a pass over a level starts at levelCutoffRepeat = 1; the same level starting over after a raised cutoff is the repeat
    if (lvl == prev_lvl && cutoffTH == setting_coarseCutoffTH && prev_cut > setting_coarseCutoffTH) repeated_level = lvl;
    prev_lvl = lvl;
    prev_cut = cutoffTH;
    Vec6 v;
    for (int i = 0; i < 6; ++i) v[i] = r[i];
    return v;
  }
  void calcGSSSE(int lvl, Mat88& H, Vec8& b, const SE3& refToNew, AffLight aff) {
    double T[16], Hm[64], bm[8], a[2] = {aff.a, aff.b};
    row_major(refToNew, T);
    g_cb(user, lvl, T, newFrame->ab_exposure, a, Hm, bm);
    for (int i = 0; i < 8; ++i) { for (int j = 0; j < 8; ++j) H(i, j) = Hm[8 * i + j]; b[i] = bm[i]; }
  }

  bool run(FrameHessian* newFrameHessian, SE3& lastToNew_out, AffLight& aff_g2l_out, int coarsestLvl, Vec5 minResForAbort) {
    lastResiduals.setConstant(NAN);       // :746-747
    lastFlowIndicators.setConstant(1000);
#include "_ref/gen/track_pyramid.inc"   // CoarseTracker.cpp:750-936, verbatim (ends with `return true;`)
  }
};
}  // namespace

extern "C" {
// T16 (row-major 4x4, in/out), aff2 (in/out): lastToNew_out / aff_g2l_out.  Returns trackNewestCoarse's return value.
// out_last_res5 = lastResiduals, out_flow3 = lastFlowIndicators, counts5 = calcRes calls per level, *repeated_level = the
// level the repeat rule ran twice (-1: none).
int ref_track_pyramid(void* user, CalcResFn res, CalcGFn g, int coarsest, double* T16, double* aff2, float new_exposure,
                      float ref_exposure, const double* ref_aff2, float coarse_cutoff, float mode_a, float mode_b,
                      const double* min_res5, double* out_last_res5, double* out_flow3, int* counts5, int* repeated_level) {
  FrameHessian nf, rf;
  nf.ab_exposure = new_exposure; rf.ab_exposure = ref_exposure;
  Loop L;
  L.user = user; L.res_cb = res; L.g_cb = g;
  L.newFrame = &nf; L.lastRef = &rf; L.lastRef_aff_g2l = AffLight(ref_aff2[0], ref_aff2[1]);
  setting_coarseCutoffTH = coarse_cutoff;
  setting_affineOptModeA = mode_a;
  setting_affineOptModeB = mode_b;
  SE3 T;
  for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) T.R(r, c) = T16[4 * r + c]; T.t(r) = T16[4 * r + 3]; }
  AffLight aff(aff2[0], aff2[1]);
  Vec5 minRes;
  for (int i = 0; i < 5; ++i) minRes[i] = min_res5[i];
  const bool ok = L.run(&nf, T, aff, coarsest, minRes);
  row_major(T, T16);
  aff2[0] = aff.a; aff2[1] = aff.b;
  for (int i = 0; i < 5; ++i) { out_last_res5[i] = L.lastResiduals[i]; counts5[i] = L.n_res[i]; }
  for (int i = 0; i < 3; ++i) out_flow3[i] = L.lastFlowIndicators[i];
  *repeated_level = L.repeated_level;
  return ok ? 1 : 0;
}
}
