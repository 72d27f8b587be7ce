// The immature points of DSO's active keyframes on the device (n8, include/tandem_b200.h): FullSystem::traceNewCoarse
// (tandem/src/FullSystem/FullSystem.cpp:650-691) becomes one trace() call per frame.  Host slot = the keyframe's index among
// the active ones (0..7); INTEGRATION.md shows the call sites.  activatePointsMT's solve (n9) becomes one activate() call, makeNewTraces (n10) one makeNewTraces() call.  Owns one tdm_immature handle; not copyable.
#ifndef TDM_CUDA_IMMATURE_POINTS_H
#define TDM_CUDA_IMMATURE_POINTS_H

#include <Eigen/Dense>

#include <vector>

struct tdm_immature;   // include/tandem_b200.h
struct tdm_pyramid;
class CudaPixelSelector;   // cuda_pixel_selector.h

class CudaImmaturePoints {
 public:
  // the reference's defaults (util/settings.cpp:84-148) for every trace setting
  CudaImmaturePoints(int w, int h, int capacity_per_host, int device = 0);
  ~CudaImmaturePoints();
  CudaImmaturePoints(const CudaImmaturePoints &) = delete;
  CudaImmaturePoints &operator=(const CudaImmaturePoints &) = delete;

  // makeNewTraces (FullSystem.cpp:1629-1646): the constructor for the selected pixels of the new keyframe; returns how many
  // points were kept (those with a finite energyTH, in input order)
  int add(int host_slot, tdm_pyramid *host_pyramid, std::vector<int> const &u, std::vector<int> const &v,
          std::vector<float> const &type);
  // n10: makeNewTraces (FullSystem.cpp:1623-1647) on the device: selector.makeMaps(fh, .., density) and the constructor for
  // every selected pixel, appended in raster order; the map stays on the device.  u / v / type (may be null) receive the
  // kept points.  Returns how many were kept.  Blocking.
  int makeNewTraces(int host_slot, CudaPixelSelector &selector, tdm_pyramid *pyramid, float density, std::vector<int> *u = nullptr,
                    std::vector<int> *v = nullptr, std::vector<float> *type = nullptr);
  // traceNewCoarse: traceOn of every point of the given hosts into the new frame, with KRKi, Kt and aff per host as
  // traceNewCoarse computes them (:655-669).  Asynchronous; get() waits for it.
  void trace(tdm_pyramid *frame_pyramid, std::vector<int> const &host_slots, std::vector<tdm_pyramid *> const &host_pyramids,
             std::vector<Eigen::Matrix<float, 3, 3>> const &KRKi, std::vector<Eigen::Matrix<float, 3, 1>> const &Kt,
             std::vector<Eigen::Matrix<float, 2, 1>> const &aff);
  // the fields activatePointsMT reads (FullSystem.cpp:760-775, 792) of every point of a slot
  struct State {
    std::vector<float> u, v, idepth_min, idepth_max, quality, interval;
    std::vector<int> status;
  };
  State get(int host_slot);
  // after activatePointsMT's compaction (:849-856), with the indices the host set to null
  void remove(int host_slot, std::vector<int> const &indices);
  // the keyframe was marginalised
  void dropHost(int host_slot);

  // n9: host->targetPrecalc[target]'s members that optimizeImmaturePoint reads (FrameFramePrecalc::set)
  struct Precalc {
    Eigen::Matrix<float, 3, 3> PRE_RTll;
    Eigen::Matrix<float, 3, 1> PRE_tTll;
    Eigen::Matrix<float, 2, 1> PRE_aff_mode;
  };
  // result[k] 1 / 0 / -1 as optimizeImmaturePoint returns a PointHessian / 0 / -1, idepth[k] its final currentIdepth,
  // res_state / res_energy[k * n_frames + f] the residual to frame f's state_state / state_energy (-1 / NaN: the host)
  struct Activation {
    int n_frames = 0;
    std::vector<int> result;
    std::vector<float> idepth;
    std::vector<signed char> res_state;
    std::vector<float> res_energy;
  };
  // activatePointsMT_Reductor (FullSystem.cpp:694-703, 819-825) for the toOptimize list: frames are frameHessians in order
  // (frame_slots[f] the frame's slot, -1 for the newest keyframe), precalc holds n_frames * n_frames entries
  // [host * n_frames + target] (the diagonal is not read), (fxl, fyl, cxl, cyl) is Hcalib's.  Candidate k is point
  // cand_index[k] of frame cand_frame[k]'s slot.  Blocking; the set is not changed.
  Activation activate(std::vector<int> const &frame_slots, std::vector<tdm_pyramid *> const &frame_pyramids,
                      std::vector<Precalc> const &precalc, float fxl, float fyl, float cxl, float cyl,
                      std::vector<int> const &cand_frame, std::vector<int> const &cand_index, float min_idepth_h_act = 100.f,
                      int gn_iterations = 3, int min_obs = 1);

 private:
  tdm_immature *handle_ = nullptr;
  int capacity_ = 0;
};

#endif
