// Type-erased interface of the level-0 photometric tracker (tracker.cu).
#pragma once
#include "common.cuh"

namespace tdm {

class TrackerIface {
 public:
  virtual ~TrackerIface() = default;
  virtual void set_k(int w, int h, float fx, float fy, float cx, float cy) = 0;
  virtual void set_reference(int n, const float* u, const float* v, const float* idepth, const float* color,
                             float ref_exposure, const double ref_aff[2]) = 0;
  virtual void set_new(const float* dI) = 0;
  virtual void calc_res(const double* refToNew, float new_exposure, const double aff[2], float cutoffTH, double res6[6]) = 0;
  virtual void calc_res_batch(int n_hyp, const double* refToNew, float new_exposure, const double* aff, float cutoffTH, double* res6) = 0;
  virtual void calc_g(float new_exposure, const double aff[2], double H[64], double b[8]) = 0;
  virtual void calc_res_g(const double* refToNew, float new_exposure, const double aff[2], float cutoffTH, double res6[6],
                          double H[64], double b[8]) = 0;
  virtual void synchronize() = 0;
  virtual void run_resident(int iters, float* ms) = 0;
  // test accessor: the first n entries of the 7 warped arrays of the last calc_res (u, v, dx, dy, idepth, residual, weight)
  virtual void get_warped(int n, float* out /* 7 x n */) = 0;
  // ---- SURVEY 8(f) n1-n3: the stages either side of the evaluation, kept on the device ----
  struct DenseRefArgs {
    const float* depth = nullptr;       // h*w, host or device
    bool depth_on_device = false;
    void* depth_ready = nullptr;        // cudaEvent_t to wait for (device depth), may be null
    const double* T_depth_to_ref = nullptr;   // 4x4 row-major
    int step = 1, dense_only = 1;
    int n_sparse = 0;
    const float *pc_u = nullptr, *pc_v = nullptr, *pc_idepth = nullptr, *pc_color = nullptr;   // n_sparse + 1 entries
    const float* idepth0 = nullptr;     // h*w host, may be null
    const float* ref_gray = nullptr;    // host h*w (stride 1) or device (stride gray_stride)
    bool gray_on_device = false;
    int gray_stride = 1;
    void* gray_ready = nullptr;
    float ref_exposure = 1.f;
    const double* ref_aff = nullptr;
  };
  virtual int set_reference_dense(const DenseRefArgs& a) = 0;
  virtual void get_reference(int n, float* u, float* v, float* idepth, float* color) = 0;
  virtual void set_new_device(const float* d_dI, void* ready_event) = 0;
  virtual int width() const = 0;
  virtual int height() const = 0;
  virtual int device() const = 0;
  void set_new_device_checked(const float* d_dI, void* ready_event, int w, int h, int dev) {
    if (w != width() || h != height()) throw Error("pyramid level size does not match the tracker's image size");
    if (dev != device()) throw Error("pyramid and tracker live on different devices");
    set_new_device(d_dI, ready_event);
  }
  struct TrackArgs {
    const double* refToNew = nullptr;   // 4x4 row-major initial guess
    const double* aff = nullptr;        // (a, b) initial
    float new_exposure = 1.f, coarse_cutoff = 20.f;
    int max_iterations = 10;
    float lambda_extrapolation_limit = 0.001f;
    int fix_a = 0, fix_b = 0;
  };
  struct TrackResult {
    double refToNew[16], aff[2], res[6];
    int iterations, evaluations;
    float cutoff_repeat;
    float device_ms;
  };
  virtual void track(const TrackArgs& a, TrackResult* r) = 0;
  // n5: CoarseTracker::trackNewestCoarse over levels[0..coarsest] (called on levels[0], which runs the loop on its stream)
  struct PyramidArgs {
    const double* refToNew = nullptr;
    const double* aff = nullptr;
    float new_exposure = 1.f, coarse_cutoff = 20.f;
    const int* max_iterations = nullptr;          // [5]
    float lambda_extrapolation_limit = 0.001f;
    float affine_mode_a = 0.f, affine_mode_b = 0.f;
    const double* min_res_for_abort = nullptr;    // [5]
  };
  struct PyramidResult {
    double refToNew[16], aff[2];
    double last_residuals[5], last_flow_indicators[3];
    int ok, aborted_level, repeated_level;
    int iterations[5], evaluations[5];
    float cutoff_repeat[5];
    float device_ms;
  };
  virtual void track_pyramid(TrackerIface* const* levels, int coarsest, const PyramidArgs& a, PyramidResult* r) = 0;
  // n6: FullSystem::trackNewCoarse's loop over the motion hypotheses (one n5 run per try) in one call on levels[0]
  struct NewCoarseArgs {
    const double* tries = nullptr;                // n_tries x 16, row-major lastF_2_fh_tries
    int n_tries = 0;
    const double* aff_last_2_l = nullptr;         // [2]
    float new_exposure = 1.f, coarse_cutoff = 20.f;
    const int* max_iterations = nullptr;          // [5]
    float lambda_extrapolation_limit = 0.001f;
    float affine_mode_a = 0.f, affine_mode_b = 0.f;
    const double* last_coarse_rmse = nullptr;     // [5]
    float retrack_threshold = 1.5f;
  };
  struct TryResult {
    double last_residuals[5];
    int ok, aborted_level, repeated_level;
    int evaluations[5];
  };
  struct NewCoarseResult {
    double refToNew[16], aff[2], achieved_res[5], flow_vecs[3];
    int have_one_good, tries, winner;
    float device_ms;
  };
  virtual void track_new_coarse(TrackerIface* const* levels, int coarsest, const NewCoarseArgs& a, NewCoarseResult* r,
                                TryResult* tries /* r->tries entries, may be null */) = 0;
};

// FrameHessian::makeImages on the device (n2): all pyramid levels of (I, dx, dy) + absSquaredGrad.
class PyramidIface {
 public:
  virtual ~PyramidIface() = default;
  virtual void build(const float* gray_host) = 0;
  virtual void get_level(int lvl, float* dI_host, float* absgrad_host) = 0;
  virtual const float* level_dI(int lvl) const = 0;   // device pointer, float3 per pixel
  virtual void* ready_event() const = 0;              // cudaEvent_t recorded after build()
  virtual int width(int lvl) const = 0;
  virtual int height(int lvl) const = 0;
  virtual int levels() const = 0;
  virtual int device() const = 0;
};
PyramidIface* make_pyramid(int w, int h, int levels, int device);

TrackerIface* make_tracker(int w, int h, float huber, float cutoff, int n_max, int device);

}  // namespace tdm
