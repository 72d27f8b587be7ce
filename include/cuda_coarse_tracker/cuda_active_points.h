// The active residuals of DSO's window on the device (n12, include/tandem_b200.h): FullSystem::linearizeAll
// (tandem/src/FullSystem/FullSystemOptimize.cpp:142-210) becomes one linearize() call and applyRes_Reductor one applyRes()
// call; load() mirrors optimize()'s activeResiduals list (:422-439).  INTEGRATION.md (2b, n12) shows the call sites.  Owns
// one tdm_active handle; not copyable.
#ifndef TDM_CUDA_ACTIVE_POINTS_H
#define TDM_CUDA_ACTIVE_POINTS_H

#include <Eigen/Dense>

#include <vector>

struct tdm_active;   // include/tandem_b200.h
struct tdm_pyramid;

class CudaActivePoints {
 public:
  // the reference's defaults (util/settings.cpp) for every setting
  CudaActivePoints(int w, int h, int capacity_points, int device = 0);
  ~CudaActivePoints();
  CudaActivePoints(const CudaActivePoints &) = delete;
  CudaActivePoints &operator=(const CudaActivePoints &) = delete;

  // the PointHessian fields linearize reads
  struct Point {
    int host;   // frameHessians index of the point's host
    float u, v;
    float color[8], weights[8];
    float maxRelBaseline;
    int numGoodResiduals;
  };
  // activeResiduals in order: res_point[k] indexes points, res_target[k] is the target's frameHessians index.  Every
  // residual is reset as resetOOB does.  Blocking.
  void load(int n_frames, std::vector<Point> const &points, std::vector<int> const &res_point, std::vector<int> const &res_target);

  // host->targetPrecalc[target]'s members that linearize reads (FrameFramePrecalc::set)
  struct Precalc {
    Eigen::Matrix<float, 3, 3> PRE_KRKiTll;
    Eigen::Matrix<float, 3, 1> PRE_KtTll;
    Eigen::Matrix<float, 3, 3> PRE_RTll_0;
    Eigen::Matrix<float, 3, 1> PRE_tTll_0;
    Eigen::Matrix<float, 2, 1> PRE_aff_mode;
    float PRE_b0_mode;
  };
  struct Result {
    double energy = 0;             // lastEnergyP
    float newFrameEnergyTH = 0;    // frameHessians.back()->frameEnergyTH after setNewFrameEnergyTH
    std::vector<signed char> state_NewState;
    std::vector<float> state_NewEnergy, state_NewEnergyWithOutlier;
    std::vector<Eigen::Matrix<float, 3, 1>> centerProjectedTo;   // NaN: keep the host's value
    std::vector<float> jacobians;   // 74 floats per residual (RawResidualJacobian in declaration order), if asked for
    // fixLinearization only
    std::vector<signed char> state_state;
    std::vector<unsigned char> removed;
    std::vector<float> maxRelBaseline;
    std::vector<int> numGoodResiduals;
  };
  // linearizeAll(fixLinearization) over frames[f]'s level 0; precalc holds n_frames * n_frames entries [host * n + target]
  // (the diagonal is not read); frameEnergyTH per frame; (fxl, fyl, cxl, cyl) is Hcalib's; idepth_scaled /
  // idepth_zero_scaled per point.  Blocking.
  void linearize(std::vector<tdm_pyramid *> const &frames, std::vector<Precalc> const &precalc,
                 std::vector<float> const &frameEnergyTH, float fxl, float fyl, float cxl, float cyl,
                 std::vector<float> const &idepth_scaled, std::vector<float> const &idepth_zero_scaled, bool fixLinearization,
                 Result *out, bool jacobians = true);
  // applyRes_Reductor (asynchronous)
  void applyRes();

  // n13: solveSystemF's accumulators over the data the last applyRes / linearize(fixLinearization) took (takeDataF).
  // The inputs setAdjointsF and setDeltaF leave: adHost / adTarget [h + n * t], each frame's prior and delta_prior, cPrior,
  // cDeltaF, each loaded point's priorF and deltaF.  Dense outputs are row-major with dim = 8 * n_frames + 4, ready for
  // Eigen::Map<MatXX> / Eigen::Map<VecX> (the matrices are returned as std::vector so that this header needs no dynamic
  // Eigen types).
  struct SystemInputs {
    std::vector<Eigen::Matrix<double, 8, 8>> adHost, adTarget;   // n_frames * n_frames each
    std::vector<Eigen::Matrix<double, 8, 1>> prior, delta_prior;   // per frame
    Eigen::Matrix<double, 4, 1> cPrior;
    Eigen::Matrix<float, 4, 1> cDeltaF;
    std::vector<float> priorF, deltaF;   // per loaded point
  };
  struct System {
    int dim = 0;
    std::vector<double> H_top, b_top, H_sc, b_sc;   // HA_top + HL_top, bA_top + bL_top, H_sc, b_sc
    int resInA = 0;
    std::vector<float> HdiF, idepth_hessian;     // per loaded point; 0 where no residual is active
  };
  // accumulateAF_MT + accumulateLF_MT + accumulateSCF_MT (blocking)
  void accumulate(SystemInputs const &in, System *out);
  // resubstituteF_MT's per-point step for the solved x (dim entries) with the last accumulate's adjoints (blocking)
  void resubstitute(std::vector<double> const &x, std::vector<float> *step);

 private:
  tdm_active *handle_ = nullptr;
  int n_frames_ = 0, n_points_ = 0, n_res_ = 0;
};

#endif
