// Test infrastructure (never linked into the product): harness around code of the REFERENCE,
//   PointFrameResidual::linearize, applyRes          tandem/src/FullSystem/Residuals.cpp:78-274, 306-328
//   FullSystem::linearizeAll_Reductor, applyRes_Reductor, setNewFrameEnergyTH, linearizeAll
//                                                    tandem/src/FullSystem/FullSystemOptimize.cpp:52-210
//   projectPoint (both forms)                        tandem/src/FullSystem/ResidualProjections.h:36-87
//   getInterpolatedElement33, staticPattern          (n8's cut)
// which oracle/ref_build_linearize.mk cuts out of the files where they lie (git-ignored build output) and compiles here,
// unmodified, against stand-ins for the DSO types they touch.  Purpose: pin oracle/linearize_oracle.c against the
// reference's own statements.  The harness runs linearizeAll with multiThreading = false, whose single-thread branch sums
// into a local Vec10: the stand-in Vec10 starts at zero (the reference's Eigen one is uninitialised there, where its reduce
// path zeroes the stats with memset).  deleteOut's stand-in takes the residual out of the point's list without deleting it,
// so the harness can still read a removed residual's fields; dropResidual marks it removed.
#include <algorithm>
#include <cassert>
#include <cmath>
#include <cstring>
#include <functional>
#include <utility>
#include <vector>

#include <Eigen/Dense>         // oracle/ref_shim/linearize_eigen
#include <boost/bind.hpp>      // oracle/ref_shim/boost

#define EIGEN_ALWAYS_INLINE inline
#define EIGEN_STRONG_INLINE inline
#define EIGEN_MAKE_ALIGNED_OPERATOR_NEW
#define PYR_LEVELS 6
#define MAX_RES_PER_POINT 8
#define patternNum 8
#define patternP staticPattern[8]
#define NUM_THREADS 6            // NumType.h:42
#define SCALE_IDEPTH 1.0f        // HessianBlocks.h:59-63
#define SCALE_F 50.0f
#define SCALE_C 50.0f

typedef Eigen::Matrix<float, 2, 1> Vec2f;
typedef Eigen::Matrix<float, 3, 1> Vec3f;
typedef Eigen::Matrix<float, 4, 1> VecCf;
typedef Eigen::Matrix<float, 4, 1> Vec4f;
typedef Eigen::Matrix<float, 6, 1> Vec6f;
typedef Eigen::Matrix<float, 8, 1> VecNRf;
typedef Eigen::Matrix<float, 2, 2> Mat22f;
typedef Eigen::Matrix<float, 3, 3> Mat33f;
typedef Eigen::Matrix<double, 3, 1> Vec3;

namespace dso {

int wG[PYR_LEVELS], hG[PYR_LEVELS];
float wM3G, hM3G;
float setting_huberTH, setting_outlierTHSumComponent, setting_affineOptModeA, setting_affineOptModeB, setting_frameEnergyTHN,
    setting_frameEnergyTHConstWeight, setting_frameEnergyTHFacMedian, setting_overallEnergyTHWeight;

#include "_ref/gen_trace/pattern.inc"
#include "_ref/gen_trace/interp33.inc"

struct Vec10 {   // stand-in: starts at zero
  double d[10] = {};
  double& operator[](int i) { return d[i]; }
};

template <typename Stats>
struct IndexThreadReduce {   // the members linearizeAll touches; runs the whole range on the caller's thread
  Stats stats;
  template <typename F>
  void reduce(F f, int first, int end, int stepSize = 0) {
    stats = Stats();
    f(first, end, &stats, 0);
  }
};

enum ResState { IN = 0, OOB, OUTLIER };   // Residuals.h:47
struct FrameFramePrecalc {   // the members linearize and the reductor read (HessianBlocks.h)
  Mat33f PRE_KRKiTll, PRE_RTll_0;
  Vec3f PRE_KtTll, PRE_tTll_0;
  Vec2f PRE_aff_mode;
  float PRE_b0_mode;
};
struct FrameHessian {
  Eigen::Vector3f* dI;
  int idx;
  float frameEnergyTH;
  std::vector<FrameFramePrecalc> targetPrecalc;
};
struct CalibHessian {   // HessianBlocks.h:397-402, set as setValueScaled sets them
  float value_scaledf[4], value_scaledi[4];
  inline float& fxl() { return value_scaledf[0]; }
  inline float& fyl() { return value_scaledf[1]; }
  inline float& cxl() { return value_scaledf[2]; }
  inline float& cyl() { return value_scaledf[3]; }
  inline float& fxli() { return value_scaledi[0]; }
  inline float& fyli() { return value_scaledi[1]; }
};
struct RawResidualJacobian {   // RawResidualJacobian.h:32-60
  VecNRf resF;
  Vec6f Jpdxi[2];
  VecCf Jpdc[2];
  Vec2f Jpdd;
  VecNRf JIdx[2];
  VecNRf JabF[2];
  Mat22f JIdx2;
  Mat22f JabJIdx;
  Mat22f Jab2;
};
struct EFResidual {   // EnergyFunctionalStructs.h:60-96: the flag applyRes and the reductor use
  bool isActiveAndIsGoodNEW = false;
  int index = 0;
  void takeDataF() {}
  inline const bool& isActive() const { return isActiveAndIsGoodNEW; }
};
struct PointFrameResidual;
struct PointHessian {   // the members the cut functions touch
  float u, v;
  float color[MAX_RES_PER_POINT], weights[MAX_RES_PER_POINT];
  float idepth_scaled, idepth_zero_scaled;
  float maxRelBaseline;
  int numGoodResiduals;
  std::vector<PointFrameResidual*> residuals;
  std::pair<PointFrameResidual*, ResState> lastResiduals[2];
};
struct PointFrameResidual {   // Residuals.h:55-101
  ResState state_state;
  double state_energy;
  ResState state_NewState;
  double state_NewEnergy;
  double state_NewEnergyWithOutlier;
  void setState(ResState s) { state_state = s; }
  PointHessian* point;
  FrameHessian* host;
  FrameHessian* target;
  RawResidualJacobian* J;
  EFResidual* efResidual;
  bool isNew;
  Eigen::Vector2f projectedTo[MAX_RES_PER_POINT];
  Vec3f centerProjectedTo;
  double linearize(CalibHessian* HCalib);
  void applyRes(bool copyJacobians);
  void resetOOB() {   // Residuals.h:92-98
    state_NewEnergy = state_energy = 0;
    state_NewState = ResState::OUTLIER;
    setState(ResState::IN);
  }
};
struct EnergyFunctional {
  std::vector<char>* removed;
  void dropResidual(EFResidual* r) { (*removed)[r->index] = 1; }
};
template <typename T>
inline void deleteOut(std::vector<T*>& v, const int i) {   // the residual stays alive for the harness to read
  v[i] = v.back();
  v.pop_back();
}

class FullSystem {   // the members linearizeAll touches (FullSystem.h)
 public:
  void linearizeAll_Reductor(bool fixLinearization, std::vector<PointFrameResidual*>* toRemove, int min, int max, Vec10* stats, int tid);
  void applyRes_Reductor(bool copyJacobians, int min, int max, Vec10* stats, int tid);
  void setNewFrameEnergyTH();
  Vec3 linearizeAll(bool fixLinearization);
  std::vector<FrameHessian*> frameHessians;
  std::vector<PointFrameResidual*> activeResiduals;
  std::vector<float> allResVec;
  CalibHessian Hcalib;
  EnergyFunctional* ef;
  bool multiThreading = false;
  IndexThreadReduce<Vec10> treadReduce;
};

#include "_ref/gen_activate/projections.inc"
#include "_ref/gen_linearize/linearize.inc"
#include "_ref/gen_linearize/apply_res.inc"
#include "_ref/gen_linearize/linearize_all.inc"

}  // namespace dso

using namespace dso;

extern "C" {

// One optimize()-shaped sequence: frames in frameHessians order (level 0 dI[f]); points; activeResiduals (res_point,
// res_target).  Step s sets every point's idepth_scaled / idepth_zero_scaled (ids / idz + s * n_points), every frame pair's
// precalc (precalc + s * n * n * 27: PRE_KRKiTll, PRE_KtTll, PRE_RTll_0, PRE_tTll_0, PRE_aff_mode, PRE_b0_mode) and the
// frames' frameEnergyTH (frame_th, the newest frame's entry then following each step's setNewFrameEnergyTH), runs
// linearizeAll(fix[s]) and, with apply[s], applyRes_Reductor over every residual.  Outputs per step and residual: the
// state_NewState, state_NewEnergy, state_NewEnergyWithOutlier, centerProjectedTo (NaN where linearize does not set it), the
// Jacobian record, the state_state after the step and removed (the residual went to toRemove); per step and point
// maxRelBaseline and numGoodResiduals; per step lastEnergyP and the newest frame's frameEnergyTH.
void ref_lin_run(int w, int h, int n, const float* const* dI, const float* calib4, const float* settings8, int np, const int* host,
                 const float* u, const float* v, const float* color, const float* weights, const float* mrb, const int* ngood, int m,
                 const int* res_point, const int* res_target, int steps, const int* fix, const int* apply, const float* ids,
                 const float* idz, const float* precalc, const float* frame_th, double* energy, float* new_th, int* new_state,
                 double* new_energy, double* new_energy_wo, float* center, float* J, int* state, int* removed, float* mrb_out,
                 int* ngood_out) {
  wG[0] = w; hG[0] = h;
  wM3G = w - 3; hM3G = h - 3;
  setting_huberTH = settings8[0]; setting_outlierTHSumComponent = settings8[1];
  setting_affineOptModeA = settings8[2]; setting_affineOptModeB = settings8[3];
  setting_frameEnergyTHN = settings8[4]; setting_frameEnergyTHConstWeight = settings8[5];
  setting_frameEnergyTHFacMedian = settings8[6]; setting_overallEnergyTHWeight = settings8[7];
  std::vector<FrameHessian> frames(n);
  FullSystem fs;
  std::vector<char> rem(m, 0);
  EnergyFunctional ef{&rem};
  fs.ef = &ef;
  for (int f = 0; f < n; ++f) {
    frames[f].dI = reinterpret_cast<Eigen::Vector3f*>(const_cast<float*>(dI[f]));
    frames[f].idx = f;
    frames[f].frameEnergyTH = frame_th[f];
    frames[f].targetPrecalc.assign(n, FrameFramePrecalc());
    fs.frameHessians.push_back(&frames[f]);
  }
  fs.Hcalib.value_scaledf[0] = calib4[0]; fs.Hcalib.value_scaledf[1] = calib4[1];
  fs.Hcalib.value_scaledf[2] = calib4[2]; fs.Hcalib.value_scaledf[3] = calib4[3];
  fs.Hcalib.value_scaledi[0] = 1.0f / fs.Hcalib.value_scaledf[0];
  fs.Hcalib.value_scaledi[1] = 1.0f / fs.Hcalib.value_scaledf[1];
  std::vector<PointHessian> pts(np);
  for (int i = 0; i < np; ++i) {
    PointHessian& p = pts[i];
    p.u = u[i]; p.v = v[i];
    for (int k = 0; k < 8; ++k) { p.color[k] = color[8 * i + k]; p.weights[k] = weights[8 * i + k]; }
    p.maxRelBaseline = mrb[i];
    p.numGoodResiduals = ngood[i];
    p.lastResiduals[0].first = p.lastResiduals[1].first = nullptr;
  }
  std::vector<PointFrameResidual> res(m);
  std::vector<RawResidualJacobian> jac(m);
  std::vector<EFResidual> efr(m);
  for (int k = 0; k < m; ++k) {
    PointFrameResidual& r = res[k];
    r.point = &pts[res_point[k]];
    r.host = &frames[host[res_point[k]]];
    r.target = &frames[res_target[k]];
    r.J = &jac[k];
    efr[k].index = k;
    r.efResidual = &efr[k];
    r.isNew = true;
    r.state_NewEnergyWithOutlier = -1;
    r.resetOOB();   // optimize() (FullSystemOptimize.cpp:422-439)
    pts[res_point[k]].residuals.push_back(&r);
    fs.activeResiduals.push_back(&r);
  }
  for (int s = 0; s < steps; ++s) {
    for (int i = 0; i < np; ++i) {
      pts[i].idepth_scaled = ids[(size_t)s * np + i];
      pts[i].idepth_zero_scaled = idz[(size_t)s * np + i];
    }
    for (int a = 0; a < n; ++a)
      for (int b = 0; b < n; ++b) {
        const float* P = precalc + 27 * (((size_t)s * n + a) * n + b);
        FrameFramePrecalc& pc = frames[a].targetPrecalc[b];
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c) { pc.PRE_KRKiTll(r, c) = P[3 * r + c]; pc.PRE_RTll_0(r, c) = P[12 + 3 * r + c]; }
        pc.PRE_KtTll = Vec3f(P[9], P[10], P[11]);
        pc.PRE_tTll_0 = Vec3f(P[21], P[22], P[23]);
        pc.PRE_aff_mode = Vec2f(P[24], P[25]);
        pc.PRE_b0_mode = P[26];
      }
    for (int k = 0; k < m; ++k) res[k].centerProjectedTo = Vec3f(NAN, NAN, NAN);
    Vec3 e = fs.linearizeAll(fix[s] != 0);
    if (apply[s]) {
      Vec10 st;
      fs.applyRes_Reductor(true, 0, (int)fs.activeResiduals.size(), &st, 0);
    }
    energy[s] = e[0];
    new_th[s] = frames[n - 1].frameEnergyTH;
    for (int k = 0; k < m; ++k) {
      const size_t o = (size_t)s * m + k;
      const PointFrameResidual& r = res[k];
      new_state[o] = r.state_NewState;
      new_energy[o] = r.state_NewEnergy;
      new_energy_wo[o] = r.state_NewEnergyWithOutlier;
      for (int c = 0; c < 3; ++c) center[3 * o + c] = r.centerProjectedTo[c];
      float* j = J + 74 * o;
      const RawResidualJacobian& q = jac[k];
      for (int i = 0; i < 8; ++i) j[i] = q.resF[i];
      for (int i = 0; i < 6; ++i) { j[8 + i] = q.Jpdxi[0][i]; j[14 + i] = q.Jpdxi[1][i]; }
      for (int i = 0; i < 4; ++i) { j[20 + i] = q.Jpdc[0][i]; j[24 + i] = q.Jpdc[1][i]; }
      j[28] = q.Jpdd[0]; j[29] = q.Jpdd[1];
      for (int i = 0; i < 8; ++i) { j[30 + i] = q.JIdx[0][i]; j[38 + i] = q.JIdx[1][i]; j[46 + i] = q.JabF[0][i]; j[54 + i] = q.JabF[1][i]; }
      for (int i = 0; i < 4; ++i) { j[62 + i] = q.JIdx2.d[i]; j[66 + i] = q.JabJIdx.d[i]; j[70 + i] = q.Jab2.d[i]; }
      state[o] = r.state_state;
      removed[o] = rem[k];
    }
    for (int i = 0; i < np; ++i) {
      mrb_out[(size_t)s * np + i] = pts[i].maxRelBaseline;
      ngood_out[(size_t)s * np + i] = pts[i].numGoodResiduals;
    }
  }
}

}  // extern "C"
