// Drop-in replacement header for tandem/libdr/cuda_coarse_tracker/include/public/cuda_coarse_tracker.h (:9-82)
// implemented over the tandem_b200 C ABI.  Caller: tandem/src/FullSystem/CoarseTracker.cpp:103-106,144,732,777-795,
// 861-887.  The class owns only an opaque handle; callers `new` it, so the layout is ours to define.
#ifndef PBA_CUDA_COARSE_TRACKER_H
#define PBA_CUDA_COARSE_TRACKER_H

#include <Eigen/Dense>

#include <vector>

struct tdm_tracker;   // include/tandem_b200.h
struct tdm_pyramid;
struct tdm_fusion;

class CudaCoarseTracker {
public:
  CudaCoarseTracker(int w, int h, float setting_huberTH, float setting_coarseCutoffTH);

  void setK(int w, int h, float fx, float fy, float cx, float cy);

  ~CudaCoarseTracker();

  void init(int n_max_in = 0);

  void free();

  void setReference(int n_in, float const *pc_u_in, float const *pc_v_in, float const *pc_idepth_in,
                    float const *pc_color_in, float ref_exposure_in, Eigen::Vector2d const &ref_aff_g2l_in);

  void setNew(float const *dInew_in);

  Eigen::Matrix<double, 6, 1> calcRes(Eigen::Matrix<double, 4, 4> const &refToNew, float new_exposure,
                                      Eigen::Vector2d const &aff_g2l, float cutoffTH);

  void calcG(Eigen::Matrix<double, 8, 8> &H_out, Eigen::Matrix<double, 8, 1> &b_out, const float new_exposure,
             const Eigen::Vector2d &aff_g2l);

  // Extension (not in the reference): calcRes + calcG in ONE launch, no warped buffers (SURVEY.md §7 step 7).
  Eigen::Matrix<double, 6, 1> calcResAndG(Eigen::Matrix<double, 4, 4> const &refToNew, float new_exposure,
                                          Eigen::Vector2d const &aff_g2l, float cutoffTH,
                                          Eigen::Matrix<double, 8, 8> &H_out, Eigen::Matrix<double, 8, 1> &b_out);

  // Extension: calcRes of several motion hypotheses (FullSystem::trackNewCoarse tries up to 31, FullSystem.cpp:437-530) in ONE
  // launch and one synchronisation; element k equals calcRes(refToNew[k], new_exposure, aff_g2l[k], cutoffTH) bit for bit.
  std::vector<Eigen::Matrix<double, 6, 1>> calcResBatch(std::vector<Eigen::Matrix<double, 4, 4>> const &refToNew, float new_exposure,
                                                        std::vector<Eigen::Vector2d> const &aff_g2l, float cutoffTH);

  // Extensions for the stages either side of the evaluation (SURVEY.md 8(f) n1-n3; see INTEGRATION.md):
  //  * setNewFromPyramid: setNew from a device-resident FrameHessian::makeImages replacement (tdm_pyramid);
  //  * setReferenceDense: the dense part of CoarseTracker::setCoarseTrackingRef + setReference; the depth map is the
  //    render_index-th map of the last DrFusion::RenderAsync and never leaves the device;
  //  * track: one pyramid level of CoarseTracker::trackNewestCoarse without host round trips.
  void setNewFromPyramid(tdm_pyramid *pyramid, int level);

  int setReferenceDense(tdm_fusion *fusion, int render_index, Eigen::Matrix<double, 4, 4> const &T_depth_to_ref,
                        int tracking_step, bool dense_only, int n_sparse, float const *pc_u, float const *pc_v,
                        float const *pc_idepth, float const *pc_color, float const *idepth0, tdm_pyramid *ref_pyramid,
                        float ref_exposure, Eigen::Vector2d const &ref_aff_g2l);

  struct TrackResult {
    Eigen::Matrix<double, 4, 4> refToNew;
    Eigen::Vector2d aff_g2l;
    Eigen::Matrix<double, 6, 1> res;
    int iterations;
    float levelCutoffRepeat;
  };
  TrackResult track(Eigen::Matrix<double, 4, 4> const &refToNew, Eigen::Vector2d const &aff_g2l, float new_exposure,
                    float coarseCutoffTH, int maxIterations, float lambdaExtrapolationLimit, bool fix_a, bool fix_b);

  // Extension: the body of CoarseTracker::trackNewestCoarse (CoarseTracker.cpp:750-936) in one call, every level on the device
  // with one host wait.  levels[l] is the tracker of pyramid level l (levels.size() - 1 = coarsestLvl), each with setK, a
  // reference and a new image.  affineOptModeA/B = setting_affineOptModeA/B.  Throws std::runtime_error on invalid input.
  struct PyramidTrackResult {
    bool ok;                                       // trackNewestCoarse's return value
    Eigen::Matrix<double, 4, 4> refToNew;          // lastToNew_out (the input when the loop aborted)
    Eigen::Vector2d aff_g2l;                       // aff_g2l_out
    Eigen::Matrix<double, 5, 1> lastResiduals;
    Eigen::Matrix<double, 3, 1> lastFlowIndicators;
    int abortedLevel, repeatedLevel;               // -1: none
    int iterations[5], evaluations[5];
    float levelCutoffRepeat[5];
  };
  static PyramidTrackResult trackPyramid(std::vector<CudaCoarseTracker *> const &levels,
                                         Eigen::Matrix<double, 4, 4> const &refToNew, Eigen::Vector2d const &aff_g2l,
                                         float new_exposure, float coarseCutoffTH, const int maxIterations[5],
                                         float lambdaExtrapolationLimit, float affineOptModeA, float affineOptModeB,
                                         Eigen::Matrix<double, 5, 1> const &minResForAbort);

  // Extension: FullSystem::trackNewCoarse's loop over the motion hypotheses (FullSystem.cpp:538-617, monocular path) in one
  // call: every try is a trackPyramid run from tries[i] and aff_last_2_l with minResForAbort = achievedRes, the winner, takeover
  // and break rules run on the device after each try, and the host waits once.  1..64 tries; reTrackThreshold =
  // setting_reTrackThreshold.  Throws std::runtime_error on invalid input (an empty try list included).
  struct NewCoarseResult {
    Eigen::Matrix<double, 4, 4> lastF_2_fh;
    Eigen::Vector2d aff_g2l;
    Eigen::Matrix<double, 3, 1> flowVecs;
    Eigen::Matrix<double, 5, 1> achievedRes;       // the caller's new lastCoarseRMSE
    bool haveOneGood;
    int tryIterations;
    int winner;                                    // index of the last winning try, -1: none
  };
  static NewCoarseResult trackNewCoarse(std::vector<CudaCoarseTracker *> const &levels,
                                        std::vector<Eigen::Matrix<double, 4, 4>> const &tries, Eigen::Vector2d const &aff_last_2_l,
                                        float new_exposure, float coarseCutoffTH, const int maxIterations[5],
                                        float lambdaExtrapolationLimit, float affineOptModeA, float affineOptModeB,
                                        Eigen::Matrix<double, 5, 1> const &lastCoarseRMSE, float reTrackThreshold);

  // Extension: CoarseTracker::setCoarseTrackingRef including makeCoarseDepthL0 (CoarseTracker.cpp:148-374, :633-733) for the
  // trackers of levels 0..n-1 (the ones trackPyramid takes) in one call: the points the reference's loop uses, in its order
  // (monocular: centerProjectedTo and efPoint->HdiF; rgbd_init: ph->u, ph->v, ph->idepth, ph->idepth_hessian), the colours from
  // the keyframe's pyramid, and, when fusion is not null, the dense append of its render_index-th render.  Every level then
  // holds its reference as after setReference.  Returns pc_n per level; throws std::runtime_error on invalid input.
  static std::vector<int> setCoarseTrackingRef(std::vector<CudaCoarseTracker *> const &levels, bool rgbd_init, int n_points,
                                               float const *pt_u, float const *pt_v, float const *pt_idepth,
                                               float const *pt_hessian, tdm_pyramid *ref_pyramid, tdm_fusion *fusion,
                                               int render_index, Eigen::Matrix<double, 4, 4> const &T_depth_to_ref,
                                               int tracking_step, bool dense_only, float ref_exposure,
                                               Eigen::Vector2d const &ref_aff);
  // Extension: the same, plus makeCoarseDepthL0's undilated level-0 cloud (pc_*_nodia, kept by levels[0]) and
  // get_idepth_quantile(pc_n_nodia, pc_idepth_nodia, quantile_fraction) over it (tandem_backend.cpp:354-361), in the same call:
  // *pc_n_nodia and *depth_quantile receive what FullSystem::deliverDrFrame reads for MVSNet's depth range (NaN when the
  // cloud has no entry at the quantile's index).
  static std::vector<int> setCoarseTrackingRef(std::vector<CudaCoarseTracker *> const &levels, bool rgbd_init, int n_points,
                                               float const *pt_u, float const *pt_v, float const *pt_idepth,
                                               float const *pt_hessian, tdm_pyramid *ref_pyramid, tdm_fusion *fusion,
                                               int render_index, Eigen::Matrix<double, 4, 4> const &T_depth_to_ref,
                                               int tracking_step, bool dense_only, float ref_exposure,
                                               Eigen::Vector2d const &ref_aff, float quantile_fraction, int *pc_n_nodia,
                                               float *depth_quantile);

  void synchronize();

  void startTiming();

  float endTimingMilliseconds();

private:
  tdm_tracker *handle_ = nullptr;
  const int w = 0, h = 0;
  const float setting_huberTH, setting_coarseCutoffTH;
  bool timing_ = false;
  double t_start_ = 0;
};

#endif  // PBA_CUDA_COARSE_TRACKER_H
