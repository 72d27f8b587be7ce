// Test infrastructure (never linked into the product): harness around code of the REFERENCE,
//   EFResidual::takeDataF                                   tandem/src/OptimizationBackend/EnergyFunctionalStructs.cpp:39-50
//   AccumulatorXX, AccumulatorX, AccumulatorApprox          MatrixAccumulators.h:36-89, 177-237, 595-972
//   AccumulatedTopHessianSSE (class, addPoint, stitchDoubleInternal)   AccumulatedTopHessian.h:44-166, .cpp:36-162, 241-303
//   AccumulatedSCHessianSSE (class, addPoint, stitchDoubleInternal)    AccumulatedSCHessian.h:42-156, .cpp:34-157
//   EnergyFunctional::accumulateAF_MT, accumulateLF_MT, accumulateSCF_MT, resubstituteF_MT, resubstituteFPt
//                                                           EnergyFunctional.cpp:196-318
// which oracle/ref_build_accumulate.mk cuts out of the files where they lie (git-ignored build output) and compiles here,
// unmodified, against stand-ins for the DSO types they touch.  Purpose: pin oracle/accumulate_oracle.c's TIERS mode against
// the reference's own statements.  The harness runs the single-thread branches (MT = false).
#include <pmmintrin.h>

#include <cassert>
#include <cmath>
#include <cstring>
#include <utility>
#include <vector>

#include <Eigen/Dense>       // oracle/ref_shim/accumulate_eigen
#include <boost/bind.hpp>    // oracle/ref_shim/boost

#define EIGEN_MAKE_ALIGNED_OPERATOR_NEW
#define EIGEN_ALIGN16 alignas(16)
#define NUM_THREADS 6        // NumType.h
#define CPARS 4
#define MAX_RES_PER_POINT 8
#define patternNum 8
#define USE_XI_MODEL 0

typedef Eigen::Matrix<double, Eigen::Dynamic, Eigen::Dynamic> MatXX;
typedef Eigen::Matrix<double, Eigen::Dynamic, 1> VecX;
typedef Eigen::Matrix<float, Eigen::Dynamic, 1> VecXf;
typedef Eigen::Matrix<double, 8, CPARS> Mat8C;
typedef Eigen::Matrix<double, 8, 8> Mat88;
typedef Eigen::Matrix<float, 8, 8> Mat88f;
typedef Eigen::Matrix<double, CPARS, 1> VecC;
typedef Eigen::Matrix<float, CPARS, 1> VecCf;
typedef Eigen::Matrix<double, 8, 1> Vec8;
typedef Eigen::Matrix<float, 8, 1> Vec8f;
typedef Eigen::Matrix<double, 10, 1> Vec10;
typedef Eigen::Matrix<float, 2, 1> Vec2f;
typedef Eigen::Matrix<float, 6, 1> Vec6f;
typedef Eigen::Matrix<float, MAX_RES_PER_POINT, 1> VecNRf;
typedef Eigen::Matrix<float, 1, 8> Mat18f;
typedef Eigen::Matrix<float, 2, 2> Mat22f;
typedef Eigen::Matrix<float, 13, 13> Mat1313f;
typedef Eigen::Matrix<double, 8 + CPARS + 1, 8 + CPARS + 1> MatPCPC;

namespace dso {

template <typename Running>
struct IndexThreadReduce {   // what the cut code names; the harness only runs the MT = false branches
  Running stats;
  template <typename F>
  void reduce(F f, int first, int end, int stepSize = 0) { f(first, end, &stats, 0); }
};

#include "_ref/gen_accumulate/acc_xx.inc"
#include "_ref/gen_accumulate/acc_x.inc"
#include "_ref/gen_accumulate/acc_approx.inc"

class EFPoint;
class EnergyFunctional;
class AccumulatedTopHessianSSE
#include "_ref/gen_accumulate/top_class.inc"
class AccumulatedSCHessianSSE
#include "_ref/gen_accumulate/sc_class.inc"

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
struct PointFrameResidual { RawResidualJacobian* J; };
struct PointHessian { float idepth_hessian, maxRelBaseline, step; };
struct FrameHessian { Vec10 step; };
struct CalibHessian { VecC step; };
class EFResidual {   // EnergyFunctionalStructs.h:51-96: the members the cut code reads
 public:
  RawResidualJacobian* J;
  PointFrameResidual* data;
  int hostIDX, targetIDX;
  VecNRf res_toZeroF;
  Vec8f JpJdF;
  bool isLinearized = false;
  bool isActiveAndIsGoodNEW = false;
  inline const bool& isActive() const { return isActiveAndIsGoodNEW; }
  void takeDataF();
};
class EFPoint {
 public:
  PointHessian* data;
  float priorF, deltaF;
  std::vector<EFResidual*> residualsAll;
  float bdSumF, HdiF, Hdd_accLF, Hdd_accAF, bd_accLF, bd_accAF;
  VecCf Hcd_accLF, Hcd_accAF;
};
class EFFrame {
 public:
  Vec8 prior, delta_prior;
  std::vector<EFPoint*> points;
  FrameHessian* data;
  int idx;
};
class EnergyFunctional {
 public:
  Mat88 *adHost, *adTarget;
  Mat88f *adHostF, *adTargetF;
  Mat18f* adHTdeltaF;
  VecC cPrior;
  VecCf cDeltaF;
  std::vector<EFFrame*> frames;
  std::vector<EFPoint*> allPoints;
  int nFrames, resInA, resInL;
  IndexThreadReduce<Vec10>* red;
  AccumulatedTopHessianSSE *accSSE_top_L, *accSSE_top_A;
  AccumulatedSCHessianSSE* accSSE_bot;
  void accumulateAF_MT(MatXX& H, VecX& b, bool MT);
  void accumulateLF_MT(MatXX& H, VecX& b, bool MT);
  void accumulateSCF_MT(MatXX& H, VecX& b, bool MT);
  void resubstituteF_MT(VecX x, CalibHessian* HCalib, bool MT);
  void resubstituteFPt(const VecCf& xc, Mat18f* xAd, int min, int max, Vec10* stats, int tid);
};

#include "_ref/gen_accumulate/take_data.inc"
#include "_ref/gen_accumulate/top_add.inc"
#include "_ref/gen_accumulate/top_stitch.inc"
#include "_ref/gen_accumulate/sc.inc"
#include "_ref/gen_accumulate/ef.inc"

}  // namespace dso

using namespace dso;

extern "C" {

// One solveSystemF's accumulation and resubstitution.  Jt: per residual the Jacobian record the last applyRes(true) took
// (takeDataF runs here on it for every active residual); active: isActiveAndIsGoodNEW.  ad_host / ad_target: records
// [h + n t], 8x8 row-major; frame_prior / frame_delta_prior n x 8; c_prior 4; c_delta 4; per point prior / delta.
// Outputs: HA, bA, HL, bL, H_sc, b_sc (dim x dim row-major / dim), resInA, per point HdiF, idepth_hessian,
// maxRelBaseline (in: the point's value), and the step of resubstituteF_MT(x).
int ref_acc_run(int n, int np, const int* host, int m, const int* res_point, const int* res_target, const float* Jt,
                const int* active, const double* ad_host, const double* ad_target, const double* frame_prior,
                const double* frame_delta_prior, const double* c_prior, const float* c_delta, const float* prior, const float* delta,
                const double* x, double* HA, double* bA, double* HL, double* bL, double* Hsc, double* bsc, float* hdi, float* idh,
                float* mrb, float* step) {
  const int dim = 8 * n + CPARS;
  // the 74-float records: RawResidualJacobian's members in declaration order, the 2x2 matrices column-major
  std::vector<RawResidualJacobian> taken(m);
  for (int k = 0; k < m; ++k) {
    const float* s = Jt + 74L * k;
    RawResidualJacobian& J = taken[k];
    for (int i = 0; i < 8; ++i) J.resF[i] = s[i];
    for (int i = 0; i < 6; ++i) { J.Jpdxi[0][i] = s[8 + i]; J.Jpdxi[1][i] = s[14 + i]; }
    for (int i = 0; i < 4; ++i) { J.Jpdc[0][i] = s[20 + i]; J.Jpdc[1][i] = s[24 + i]; }
    J.Jpdd[0] = s[28]; J.Jpdd[1] = s[29];
    for (int i = 0; i < 8; ++i) { J.JIdx[0][i] = s[30 + i]; J.JIdx[1][i] = s[38 + i]; J.JabF[0][i] = s[46 + i]; J.JabF[1][i] = s[54 + i]; }
    for (int i = 0; i < 4; ++i) { J.JIdx2.data()[i] = s[62 + i]; J.JabJIdx.data()[i] = s[66 + i]; J.Jab2.data()[i] = s[70 + i]; }
  }
  std::vector<PointFrameResidual> pfr(m);
  std::vector<EFResidual> efr(m);
  std::vector<PointHessian> ph(np);
  std::vector<EFPoint> efp(np);
  std::vector<FrameHessian> fh(n);
  std::vector<EFFrame> eff(n);
  std::vector<Mat88> aH(n * n), aT(n * n);
  std::vector<Mat88f> aHF(n * n), aTF(n * n);
  std::vector<Mat18f> adHT(n * n);
  for (int k = 0; k < n * n; ++k)
    for (int r = 0; r < 8; ++r)
      for (int c = 0; c < 8; ++c) {
        aH[k](r, c) = ad_host[64 * k + 8 * r + c];
        aT[k](r, c) = ad_target[64 * k + 8 * r + c];
        aHF[k](r, c) = (float)aH[k](r, c);   // setAdjointsF: adHostF = adHost.cast<float>()
        aTF[k](r, c) = (float)aT[k](r, c);
      }
  for (int k = 0; k < n * n; ++k) adHT[k].setZero();
  EnergyFunctional ef;
  ef.adHost = aH.data(); ef.adTarget = aT.data(); ef.adHostF = aHF.data(); ef.adTargetF = aTF.data(); ef.adHTdeltaF = adHT.data();
  for (int i = 0; i < CPARS; ++i) { ef.cPrior[i] = c_prior[i]; ef.cDeltaF[i] = c_delta[i]; }
  ef.nFrames = n;
  IndexThreadReduce<Vec10> red;
  ef.red = &red;
  AccumulatedTopHessianSSE topA, topL;
  AccumulatedSCHessianSSE bot;
  ef.accSSE_top_A = &topA; ef.accSSE_top_L = &topL; ef.accSSE_bot = &bot;
  for (int f = 0; f < n; ++f) {
    eff[f].idx = f;
    eff[f].data = &fh[f];
    for (int i = 0; i < 8; ++i) { eff[f].prior[i] = frame_prior[8 * f + i]; eff[f].delta_prior[i] = frame_delta_prior[8 * f + i]; }
    ef.frames.push_back(&eff[f]);
  }
  for (int p = 0; p < np; ++p) {
    ph[p].maxRelBaseline = mrb[p];
    ph[p].idepth_hessian = 0;
    efp[p].data = &ph[p];
    efp[p].priorF = prior[p];
    efp[p].deltaF = delta[p];
    efp[p].HdiF = efp[p].bdSumF = 0;
    eff[host[p]].points.push_back(&efp[p]);
  }
  for (int f = 0; f < n; ++f)
    for (EFPoint* p : eff[f].points) ef.allPoints.push_back(p);   // makeIDX: frames, then their points
  for (int k = 0; k < m; ++k) {
    EFResidual& r = efr[k];
    pfr[k].J = &taken[k];
    r.data = &pfr[k];
    r.J = nullptr;
    r.hostIDX = host[res_point[k]];
    r.targetIDX = res_target[k];
    r.res_toZeroF.setZero();
    r.JpJdF.setZero();
    r.isActiveAndIsGoodNEW = active[k] != 0;
    if (r.isActiveAndIsGoodNEW) r.takeDataF();
    efp[res_point[k]].residualsAll.push_back(&r);
  }
  MatXX HA_, HL_, Hsc_;
  VecX bA_, bL_, bsc_;
  ef.accumulateAF_MT(HA_, bA_, false);
  ef.accumulateLF_MT(HL_, bL_, false);
  ef.accumulateSCF_MT(Hsc_, bsc_, false);
  for (int r = 0; r < dim; ++r) {
    for (int c = 0; c < dim; ++c) {
      HA[r * dim + c] = HA_(r, c); HL[r * dim + c] = HL_(r, c); Hsc[r * dim + c] = Hsc_(r, c);
    }
    bA[r] = bA_[r]; bL[r] = bL_[r]; bsc[r] = bsc_[r];
  }
  for (int p = 0; p < np; ++p) { hdi[p] = efp[p].HdiF; idh[p] = ph[p].idepth_hessian; mrb[p] = ph[p].maxRelBaseline; }
  VecX xv = VecX::Zero(dim);
  for (int i = 0; i < dim; ++i) xv[i] = x[i];
  CalibHessian hc;
  ef.resubstituteF_MT(xv, &hc, false);
  for (int p = 0; p < np; ++p) step[p] = ph[p].step;
  return ef.resInA;
}

}  // extern "C"
