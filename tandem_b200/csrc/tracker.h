// Type-erased interface of the level-0 photometric tracker (tracker.cu).
#pragma once
#include "common.cuh"

struct tdm_undistort_settings;

namespace tdm {

class PyramidIface;

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
  // n7: CoarseTracker::setCoarseTrackingRef with makeCoarseDepthL0 for levels[0..n_levels-1] (called on levels[0], which runs
  // it on its stream); pc_n[l] receives each level's count
  struct CoarseRefArgs {
    int n_levels = 1, rgbd_init = 0;
    int n_points = 0;
    const float *pt_u = nullptr, *pt_v = nullptr, *pt_idepth = nullptr, *pt_hessian = nullptr;
    const PyramidIface* ref_pyramid = nullptr;   // colours: level l's dIp[l][i][0]
    const float* depth = nullptr;       // dense map (h*w, host or device), nullptr: none
    bool depth_on_device = false;
    void* depth_ready = nullptr;        // cudaEvent_t to wait for (device depth), may be null
    const double* T_depth_to_ref = nullptr;
    int step = 1, dense_only = 0;
    float ref_exposure = 1.f;
    const double* ref_aff = nullptr;
    float quantile_fraction = 0.f;      // with nodia: the fraction of get_idepth_quantile, in [0, 1]
  };
  // With nodia also the undilated level-0 cloud pc_*_nodia (CoarseTracker.cpp:150-218, kept by levels[0] across calls) and
  // the MVSNet depth range's inverse-depth quantile over it (FullSystem.cpp:1175, tandem_backend.cpp:354-361)
  struct CoarseNodiaResult {
    int pc_n_nodia;
    float idepth_quantile, depth_quantile;   // NaN when the quantile's index is not below pc_n_nodia
  };
  virtual void set_coarse_tracking_ref(TrackerIface* const* levels, const CoarseRefArgs& a, int pc_n[5],
                                       CoarseNodiaResult* nodia /* null: n7 alone */) = 0;
  // the first n entries of levels[0]'s pc_u/v/idepth/color_nodia; an error before the first call with nodia
  virtual void get_coarse_nodia(int n, float* u, float* v, float* idepth, float* color) = 0;
};

// FrameHessian::makeImages on the device (n2): all pyramid levels of (I, dx, dy) + absSquaredGrad.
class PyramidIface {
 public:
  virtual ~PyramidIface() = default;
  virtual void build(const float* gray_host) = 0;
  virtual void get_level(int lvl, float* dI_host, float* absgrad_host) = 0;
  virtual const float* level_dI(int lvl) const = 0;   // device pointer, float3 per pixel
  virtual const float* level_abs(int lvl) const = 0;  // device pointer, absSquaredGrad
  virtual void* ready_event() const = 0;              // cudaEvent_t recorded after build()
  // orders the next build() (and the destructor) after `event` (a cudaEvent_t a reader recorded behind its reads)
  virtual void wait_for(void* event) const = 0;
  virtual int width(int lvl) const = 0;
  virtual int height(int lvl) const = 0;
  virtual int levels() const = 0;
  virtual int device() const = 0;
  // n11: build() from level 0's grey already on the device.  A producer writes it into device_input() (w*h floats) with work
  // enqueued on stream() (a cudaStream_t) and then calls build_device, which records ready_event() as build() does.  d_B
  // (256 floats on the device, or null): the camera's B; absSquaredGrad then carries makeImages' gamma weights.
  virtual float* device_input() = 0;
  virtual void* stream() const = 0;
  virtual void build_device(const float* d_B) = 0;
};
PyramidIface* make_pyramid(int w, int h, int levels, int device);

// n11 (undistort.cu): DSO's per-frame input - PhotometricUndistorter::processFrame, Undistort::undistort's bilinear remap,
// the BGR remap of the dataset reader - into a pyramid (tdm_undistort_frame).
class UndistortIface {
 public:
  virtual ~UndistortIface() = default;
  virtual void get_gamma(float G[256], int* valid) const = 0;
  virtual void set_gamma(const float* Binv) = 0;
  // returns exposure_time; bgr / bgr_out both null or both given
  virtual float frame(const unsigned char* gray, float exposure, float factor, PyramidIface& out, const unsigned char* bgr,
                      unsigned char* bgr_out) = 0;
  virtual int device() const = 0;
};
UndistortIface* make_undistort(const tdm_undistort_settings& s, int device);

// n10 (pixsel.cu): PixelSelector::makeMaps on a pyramid's levels 0..2 (tdm_select_result's layout)
struct SelectResult {
  int num_selected, n2, n3, n4, potential_used, potential_after, reselected, nonuniform_cells;
};
class SelectorIface {
 public:
  virtual ~SelectorIface() = default;
  virtual int potential() const = 0;
  virtual void set_potential(int p) = 0;
  // blocking makeMaps; map_out (host, w*h) may be null
  virtual void make_maps(const PyramidIface& p, float density, int recursions_left, float th_factor, float* map_out,
                         SelectResult* r) = 0;
  // what make_maps and enqueue reject
  virtual void check(const PyramidIface& p, float density, int recursions_left, float th_factor) const = 0;
  // makeMaps on `stream` (a cudaStream_t) after the pyramid's build, the map kept on the device; with emit also
  // makeNewTraces' candidates (candidates()).  The result is copied to host memory that result() reads once the stream has
  // been synchronised; result(commit) then sets the potential to the call's.
  virtual void enqueue(void* stream, const PyramidIface& p, float density, int recursions_left, float th_factor, bool emit) = 0;
  struct Candidates {
    const int* cand;    // u at cand[k], v at cand[stride + k], the type's float bits at cand[2 stride + k]
    int stride;
    const int* count;   // device
  };
  virtual Candidates candidates() const = 0;
  virtual void result(SelectResult* r, bool commit) = 0;
  virtual int width() const = 0;
  virtual int height() const = 0;
  virtual int device() const = 0;
};
SelectorIface* make_selector(int w, int h, const float* settings /* tdm_select_settings */, int device);

// n8 (immature.cu): the immature points of up to 8 host keyframes (slots) and their trace into new frames.  Each field is a
// row of 32-bit words, one per point; status is an int, the others floats.
enum ImmatureRow { IM_U = 0, IM_V, IM_TYPE, IM_ETH, IM_IDMIN, IM_IDMAX, IM_QUALITY, IM_STATUS, IM_UVX, IM_UVY, IM_INTERVAL,
                   IM_COLOR, IM_WEIGHTS = IM_COLOR + 8, IM_GRADH = IM_WEIGHTS + 8, IM_ROWS = IM_GRADH + 4 };
class ImmatureIface {
 public:
  virtual ~ImmatureIface() = default;
  // constructor for n candidate pixels of `host`'s level 0; appends the points with a finite energyTH, returns their number
  virtual int add(int slot, const PyramidIface& host, int n, const int* u, const int* v, const float* type) = 0;
  // traceOn of every point of the given slots into frame's level 0 (asynchronous); KRKi 9, Kt 3, aff 2 per host;
  // host_pyramids (may be null, or hold nulls) are the hosts' pyramids the trace is ordered after and keeps alive
  virtual void trace(const PyramidIface& frame, int n_hosts, const int* slots, const PyramidIface* const* host_pyramids,
                     const float* KRKi, const float* Kt, const float* aff) = 0;
  // n9: optimizeImmaturePoint for every candidate (cand_frame / cand_index) over the frames' level 0 (blocking, one host
  // wait); frame_slots[f] is frame f's slot or -1, precalc n_frames x n_frames x 14, calib4 fxl fyl cxl cyl; outputs may be null
  virtual void activate(int n_frames, const int* frame_slots, const PyramidIface* const* frame_pyramids, const float* precalc,
                        const float* calib4, float min_idepth_h_act, int gn_iterations, int min_obs, int n_cand,
                        const int* cand_frame, const int* cand_index, int* result, float* idepth, signed char* res_state,
                        float* res_energy) = 0;
  // n10: makeNewTraces - makeMaps (recursions 1, thFactor 1) and the constructor for every selected pixel of
  // [3, w-4) x [3, h-4), appended to the slot in raster order (blocking, one host wait); u / v / type (may be null) receive
  // the kept points.  Kept points beyond the slot's free capacity are an error; the set and the potential are then unchanged.
  virtual int make_new_traces(int slot, SelectorIface& sel, const PyramidIface& p, float density, SelectResult* r, int* u, int* v,
                              float* type) = 0;
  virtual int count(int slot) = 0;
  // points first..first+n-1 of a slot, one output per ImmatureRow (null: not wanted); synchronises
  virtual void get(int slot, int first, int n, float* const* rows) = 0;
  virtual void remove(int slot, int n_removed, const int* indices) = 0;
  virtual void drop_host(int slot) = 0;
  virtual void synchronize() = 0;
  virtual int width() const = 0;
  virtual int height() const = 0;
  virtual int device() const = 0;
};
ImmatureIface* make_immature(int w, int h, int capacity_per_host, const float* settings /* tdm_trace_settings */, int device);

// n12 (linearize.cu): the active residuals of one FullSystem::optimize and their linearisation (tdm_active_*)
class ActiveIface {
 public:
  virtual ~ActiveIface() = default;
  // blocking upload; every residual is reset as resetOOB does
  virtual void load(int n_frames, int n_points, const int* host, const float* u, const float* v, const float* color,
                    const float* weights, const float* max_rel_baseline, const int* num_good, int n_res, const int* res_point,
                    const int* res_target) = 0;
  struct Outputs {   // host memory; every pointer may be null
    double* energy = nullptr;
    float* new_frame_energy_th = nullptr;
    signed char* new_state = nullptr;
    float *new_energy = nullptr, *new_energy_with_outlier = nullptr, *center_projected_to = nullptr, *jacobians = nullptr;
    signed char* state = nullptr;       // fix only
    unsigned char* removed = nullptr;   // fix only
    float* max_rel_baseline = nullptr;  // fix only
    int* num_good_residuals = nullptr;  // fix only
  };
  // linearizeAll(fix) over frames[0..n_frames-1]'s level 0 (blocking, one host wait)
  virtual void linearize(const PyramidIface* const* frames, const float* precalc, const float* frame_energy_th, const float* calib4,
                         const float* idepth_scaled, const float* idepth_zero_scaled, int fix, Outputs& o) = 0;
  virtual void apply_res() = 0;   // asynchronous
  virtual void get_state(signed char* state, float* energy) = 0;   // synchronises
  virtual const float* device_jacobians() const = 0;   // n_residuals() x 74 floats
  virtual int n_frames() const = 0;
  virtual int n_residuals() const = 0;
  virtual int device() const = 0;
  // n13 (accumulate.cu): solveSystemF's accumulators over the data the last applyRes(true) took
  struct AccInputs {   // host memory
    const double *ad_host = nullptr, *ad_target = nullptr;                // n x n records [host][target], 8x8 row-major
    const double *frame_prior = nullptr, *frame_delta_prior = nullptr;    // n x 8
    const double* c_prior = nullptr;                                      // 4
    const float* c_delta = nullptr;                                       // 4
    const float *point_prior = nullptr, *point_delta = nullptr;           // per point
  };
  struct AccOutputs {   // host memory; every pointer may be null
    double *H_top = nullptr, *b_top = nullptr, *H_sc = nullptr, *b_sc = nullptr;
    int* n_active = nullptr;
    float *hdi = nullptr, *idepth_hessian = nullptr;
  };
  virtual void accumulate(const AccInputs& in, AccOutputs& o) = 0;    // blocking
  virtual void resubstitute(const double* x, float* step) = 0;        // blocking
  virtual void get_accumulators(double* top, int* top_num, double* acc_e, double* acc_eb, double* acc_d, int* d_num, double* hcc,
                                double* bc) = 0;                      // synchronises
};
ActiveIface* make_active(int w, int h, int capacity_points, const float* settings /* tdm_linearize_settings */, int device);

// the device arrays of an ActiveImpl that the accumulators read
struct ActiveView {
  int n_frames, n_points, n_res;
  bool unique_targets;   // at most one residual per (point, target)
  const int *host, *off, *res_of, *res_target;   // per point; CSR offsets (n_points + 1) and list; per residual
  const float* J;                                // the last linearize's Jacobians
  float* max_rel_baseline;
};
// the taken data and accumulators of one active-residual set (accumulate.cu); every call runs on the set's stream
class AccIface {
 public:
  virtual ~AccIface() = default;
  virtual unsigned char* active() = 0;   // isActiveAndIsGoodNEW per residual
  virtual unsigned char* took() = 0;     // set by each apply for the residuals it took
  virtual void load(const ActiveView& v, const int* host, cudaStream_t st) = 0;   // host: host memory; asynchronous
  virtual void take(const ActiveView& v, cudaStream_t st) = 0;                     // asynchronous, after an apply
  virtual void accumulate(const ActiveView& v, cudaStream_t st, const ActiveIface::AccInputs& in, ActiveIface::AccOutputs& o) = 0;
  virtual void resubstitute(const ActiveView& v, cudaStream_t st, const double* x, float* step) = 0;
  virtual void get_accumulators(const ActiveView& v, cudaStream_t st, double* top, int* top_num, double* acc_e, double* acc_eb,
                                double* acc_d, int* d_num, double* hcc, double* bc) = 0;
};
AccIface* make_acc(int capacity_points);

TrackerIface* make_tracker(int w, int h, float huber, float cutoff, int n_max, int device);

}  // namespace tdm
