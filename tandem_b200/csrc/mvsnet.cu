// CVA-MVSNet engine: host orchestration of the device kernels behind the DrMvsnet call surface.
//
// Reference call path being replaced (SURVEY.md §3.3/§3.4):
//   DrMvsnetImpl::CallAsync      tandem/libdr/dr_mvsnet/src/dr_mvsnet.cpp:125-283  (copy + reorder + K's + H2D)
//   DrMvsnetImpl::CallSequential dr_mvsnet.cpp:285-331                              (module.forward + D2H)
//   CvaMVSNet.forward            cva_mvsnet/models/cva_mvsnet.py:98-184
// Design: one worker thread + one CUDA stream per handle (as the reference), u8 images uploaded from pinned
// memory (6.45 MB instead of 25.8 MB fp32), everything else stays on the device until the four output maps
// are copied back in one pinned D2H.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <atomic>
#include <condition_variable>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <sstream>
#include <thread>
#include <vector>

#include "copy_pool.h"
#include "mvsnet.h"
#include "mvsnet_kernels.cuh"
#include "conv_tc.cuh"
#include "conv_tc_is.cuh"
#include "conv_tc_s2.cuh"
#include "weights.h"

namespace tdm {

namespace {

std::mutex g_slot_mu;
bool g_slot_used[kMaxEngines] = {};
// An engine's index into the constant banks (c_call_params, c_feat_slot, c_conv00), held for the engine's lifetime.
struct EngineSlot {
  int index = -1;
  EngineSlot() {
    std::lock_guard<std::mutex> lk(g_slot_mu);
    for (index = 0; index < kMaxEngines; ++index)
      if (!g_slot_used[index]) { g_slot_used[index] = true; return; }
    throw Error("too many DrMvsnet instances alive in this process (max 8)");
  }
  ~EngineSlot() { std::lock_guard<std::mutex> lk(g_slot_mu); g_slot_used[index] = false; }
  EngineSlot(const EngineSlot&) = delete;
  EngineSlot& operator=(const EngineSlot&) = delete;
};

// ---- small host linear algebra (double) --------------------------------------------------------
void mat4_mul(const double* a, const double* b, double* c) {
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double s = 0;
      for (int k = 0; k < 4; ++k) s += a[i * 4 + k] * b[k * 4 + j];
      c[i * 4 + j] = s;
    }
}
bool mat4_inv(const double* m, double* out) {
  double a[4][8];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) { a[i][j] = m[i * 4 + j]; a[i][4 + j] = (i == j) ? 1.0 : 0.0; }
  for (int c = 0; c < 4; ++c) {
    int piv = c;
    for (int r = c + 1; r < 4; ++r) if (std::fabs(a[r][c]) > std::fabs(a[piv][c])) piv = r;
    if (std::fabs(a[piv][c]) < 1e-300) return false;
    if (piv != c) for (int j = 0; j < 8; ++j) std::swap(a[piv][j], a[c][j]);
    const double d = a[c][c];
    for (int j = 0; j < 8; ++j) a[c][j] /= d;
    for (int r = 0; r < 4; ++r) if (r != c) {
      const double f = a[r][c];
      if (f != 0) for (int j = 0; j < 8; ++j) a[r][j] -= f * a[c][j];
    }
  }
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) out[i * 4 + j] = a[i][4 + j];
  return true;
}
// world->pixel 4x4: rows 0..2 = K * W[:3,:4], row 3 = W[3,:]   (module.py:799-805)
void world_to_pixel(const float* K, const float* c2w, double* P) {
  double c[16], w[16];
  for (int i = 0; i < 16; ++i) c[i] = c2w[i];
  if (!mat4_inv(c, w)) throw Error("cam_to_world is singular");
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j) {
      double s = 0;
      for (int k = 0; k < 3; ++k) s += (double)K[i * 3 + k] * w[k * 4 + j];
      P[i * 4 + j] = s;
    }
  for (int j = 0; j < 4; ++j) P[12 + j] = w[12 + j];
}

struct DevBuf {
  DevPtr<void> p;
  size_t bytes = 0;       // allocation size (with halos)
  size_t alg_bytes = 0;   // algorithmic size C*D*H*W*sizeof(element): what the roofline counts
  int C = 0, D = 0, H = 0, W = 0;
  int pd = 0;             // halo along D (P8 layout, see mvsnet_kernels.cuh)
  int kind = 1;      // 0: fp32 (logits / maps), 1: activation type TA, 2: cost-volume type TV
  bool f32 = false;  // kind == 0
};

struct DevConv {
  int cin = 0, cout = 0, kd = 1, kh = 1, kw = 1;
  bool transposed = false;
  DevPtr<float> w;
  DevPtr<float> bias;
  // tensor-core path (conv_tc.cuh): weights pre-arranged as the canonical K-major B image in the input's 16-bit type
  DevPtr<void> bimg;
  int npad = 0;
  bool tc_ok = false;
  bool tc_deconv = false;  // transposed conv evaluated as a GEMM over the input grid (N = 8 parity classes x cout)
  int nsplit = 1;          // N slices (blockIdx.y) for the 64-channel layers
  bool hilo = false;       // weights carried as hi + lo 16-bit halves (N doubled), see conv_tc.cuh
  bool tc_up2 = false;     // MODE 3: the fused FPN tail, conv3x3 of a nearest-x2 up-sampled map + conv3x3 of a fine map,
                           // on the coarse grid
  bool tc_s2 = false;      // stride-2 conv on the tensor-map (strided TMA) kernel, conv_tc_s2.cuh
  DevPtr<void> bimg_s2;
  int npad_s2 = 0, nsplit_s2 = 1;
  DevPtr<void> bimg_is;  // input-stationary B image (conv_tc_is.cuh): 3x3x3 layers with 1 or 8 output channels
};

struct LaunchRec {
  std::string name;
  double bytes = 0, flops = 0;
  Event e0, e1;
  float ms = 0;
};

}  // namespace

// ================================================================================================
template <typename TA, typename TV>
class MvsnetEngine final : public MvsnetIface {
 public:
  MvsnetEngine(const std::string& path, int device) : device_(device) {
    TDM_CUDA(cudaSetDevice(device_));
    wf_ = load_tdmw(path);
    for (int i = 0; i < 3; ++i) depth_num_[i] = wf_.depth_num[i];
    va_ = wf_.view_aggregation;
    int lo, hi;
    TDM_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    stream_ = make_stream(lo);
    side_stream_ = make_stream(lo);
    ev_fork_ = make_event(cudaEventDisableTiming);
    ev_join_ = make_event(cudaEventDisableTiming);
    for (auto& e : ev_out_) e = make_event(cudaEventDisableTiming);
    ev_in_ = make_event(cudaEventDisableTiming);
    upload_weights();
    worker_ = std::thread([this] { this->loop(); });
  }

  ~MvsnetEngine() override {
    {
      std::unique_lock<std::mutex> lk(mu_);
      cv_done_.wait(lk, [this] { return !busy_; });
      stop_ = true;
    }
    cv_work_.notify_all();
    if (worker_.joinable()) worker_.join();
    cudaSetDevice(device_);
    // consumers of the keyframe handoff may still be reading it: read_handoff returns once their reads are enqueued
    cudaStreamSynchronize(stream_.get());
    for (int i = 0; i < n_ho_release_; ++i) cudaEventSynchronize(ev_ho_release_[i].get());
  }

  void set_option(const std::string& key, int value) override {
    {
      // the worker may be replaying the captured graph: wait for it before the graph is destroyed / options change
      std::unique_lock<std::mutex> lk(mu_);
      cv_done_.wait(lk, [this] { return !busy_; });
    }
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    if (key == "eager_d2h") { eager_d2h_ = value != 0; return; }   // not part of the captured launch sequence
    drop_graph();
    cache_valid_ = false;   // features computed under other options are not reused
    if (key == "filter_all_stages") filter_all_ = value != 0;
    else if (key == "use_graph") use_graph_ = value != 0;
    else if (key == "use_pdl") { TDM_CHECK(value >= 0 && value <= 2, "use_pdl: 0 off, 1 tensor-core kernels, 2 every kernel of the forward"); use_pdl_ = value; }
    else if (key == "pdl_min_smem_kb") { TDM_CHECK(value >= 0 && value <= 225, "pdl_min_smem_kb out of range"); pdl_min_smem_kb_ = value; }
    else if (key == "cv_variant") { TDM_CHECK(value == 3 || value == 4, "cv_variant: 3 (default) or 4"); cv_variant_ = value; }
    else if (key == "tc_smem_kb") { TDM_CHECK(value >= 48 && value <= 225, "tc_smem_kb out of range"); tc_smem_kb_ = value; tc_cache_.clear(); }
    else if ((key.rfind("depth_num_stage", 0) == 0 && key.size() == 16 && key[15] >= '1' && key[15] <= '3') || key == "debug_poison") {
      // depth_num_stageN: override the checkpoint's MODEL.DEPTH_NUM for one stage (BASELINE.json configs[0] uses 32 stage-1
      // hypotheses; CostRegNet is fully convolutional in D).  debug_poison: see alloc.  Both force a re-plan.
      if (key == "debug_poison") {
        debug_poison_ = value != 0;
      } else {
        TDM_CHECK(value == 4 || (value > 0 && value % 8 == 0 && value <= 64), "depth_num must be 4 or a multiple of 8 up to 64");
        depth_num_[key[15] - '1'] = value;
      }
      // the old plan's buffers are sized for the old D: drop them together with the resident window, so that neither
      // run_resident / profile nor a stale logits buffer can be used before the next CallAsync re-plans
      free_plan();
      V_ = H_ = W_ = 0;
      have_inputs_ = false;
    }
    else if (key == "keep_intermediates") keep_ = value != 0;
    else if (key == "use_tc") use_tc_ = value != 0;
    else if (key == "use_is") use_is_ = value != 0;
    else if (key == "fork_fpn") fork_fpn_ = value != 0;
    else if (key == "prob_direct") prob_direct_ = value != 0;
    else if (key == "direct_conv00") direct_conv00_ = value != 0;
    else if (key == "fused_regress") fused_regress_ = value != 0;
    else throw Error("unknown option " + key);
  }

  // "Blocking for last input. Non-blocking for this input." (dr_mvsnet.h:42)
  void call_async(int H, int W, int V, int ref_index, unsigned char* const* bgrs, const float* K3x3x3,
                  float* const* c2ws, float dmin, float dmax, float discard) override {
    check_window(H, W, V, ref_index);
    for (int i = 0; i < V - 1; ++i)
      for (int j = i + 1; j < V; ++j)
        if (bgrs[i] == bgrs[j] || c2ws[i] == c2ws[j])
          throw Error("CallAsync: the same data passed for two views (dr_mvsnet.cpp:153-160)");
    std::unique_lock<std::mutex> lk(mu_);
    wait_idle_for_call(lk);
    TDM_CUDA(cudaSetDevice(device_));
    ensure_plan(V, H, W);
    // copy inputs (owned by the caller only during this call); reference view first (dr_mvsnet.cpp:190-197).  Every view is
    // computed, view vi in slot vi of both pools; the feature cache is emptied.
    cache_valid_ = false;
    std::vector<int> slots(V);
    std::vector<const unsigned char*> srcs(V);
    for (int vi = 0; vi < V; ++vi) {
      view_slot_[vi] = vi;
      slots[vi] = vi;
      srcs[vi] = bgrs[window_view(vi, ref_index)];
    }
    upload_images(V, slots.data(), srcs.data());
    submit(V, ref_index, c2ws, K3x3x3, dmin, dmax, discard, lk);
  }

  // Feature cache.  Pools: plane s of d_bgr_ (u8 image) and of feat1..feat3 (FeatureNet outputs) is slot s, V slots; after
  // a cached call they hold exactly that window's ids.  Ids that left the window are evicted and their slots take the new
  // views, lowest free slot first in window order (reference first).  FeatureNet then runs on the k new views only and its
  // outputs are scattered into their slots; the cost volumes read view v from slot view_slot_[v] (CvParams::plane).
  void call_async_ids(int H, int W, int V, int ref_index, const long long* ids, unsigned char* const* bgrs, const float* K3x3x3,
                      float* const* c2ws, float dmin, float dmax, float discard) override {
    check_window(H, W, V, ref_index);
    for (int i = 0; i < V - 1; ++i)
      for (int j = i + 1; j < V; ++j) {
        if (ids[i] == ids[j]) throw Error("CallAsyncIds: view id " + std::to_string(ids[i]) + " passed for two views");
        if (c2ws[i] == c2ws[j]) throw Error("CallAsync: the same data passed for two views (dr_mvsnet.cpp:153-160)");
      }
    std::unique_lock<std::mutex> lk(mu_);
    wait_idle_for_call(lk);
    // everything below the checks changes state: decide first which views are held (a re-plan empties the pools)
    const bool same_plan = V == V_ && H == H_ && W == W_;
    int held_slot[kMaxSrc + 1];
    for (int vi = 0; vi < V; ++vi) {
      const int view = window_view(vi, ref_index);
      held_slot[vi] = -1;
      if (cache_valid_ && same_plan)
        for (int s = 0; s < V_; ++s)
          if (slot_id_[s] == ids[view]) held_slot[vi] = s;
      if (held_slot[vi] < 0 && !bgrs[view])
        throw Error("CallAsyncIds: no image for view id " + std::to_string(ids[view]) + ", which the handle does not hold");
    }
    TDM_CUDA(cudaSetDevice(device_));
    ensure_plan(V, H, W);
    bool used[kMaxSrc + 1] = {};
    for (int vi = 0; vi < V; ++vi)
      if (held_slot[vi] >= 0) used[held_slot[vi]] = true;
    std::vector<int> slots;
    std::vector<const unsigned char*> srcs;
    int next_free = 0;
    for (int vi = 0; vi < V; ++vi) {
      if (held_slot[vi] < 0) {
        while (used[next_free]) ++next_free;
        held_slot[vi] = next_free;
        used[next_free] = true;
        slots.push_back(next_free);
        srcs.push_back(bgrs[window_view(vi, ref_index)]);
      }
    }
    const int k = (int)slots.size();
    if (k > 0 && k < V) ensure_feature_scratch(k);
    // the new images go into slots that no queued work reads any more: the last forward has finished (the worker is idle)
    // and GetResult's handoff copy of the previous reference image is enqueued on stream_ ahead of these uploads
    upload_images(k, slots.data(), srcs.data());
    for (int vi = 0; vi < V; ++vi) {
      view_slot_[vi] = held_slot[vi];
      slot_id_[held_slot[vi]] = ids[window_view(vi, ref_index)];
    }
    cache_valid_ = true;
    submit(k, ref_index, c2ws, K3x3x3, dmin, dmax, discard, lk, slots.data());
  }

  void feature_cache(long long* ids, int cap, int* n_ids, int* n_computed) override {
    std::unique_lock<std::mutex> lk(mu_);
    cv_done_.wait(lk, [this] { return !busy_; });
    const int n = cache_valid_ ? V_ : 0;
    if (n_ids) *n_ids = n;
    if (n_computed) *n_computed = n_computed_;
    if (ids) {
      TDM_CHECK(cap >= n, "feature_cache: capacity too small");
      for (int view = 0; view < n; ++view) ids[view] = slot_id_[view_slot_[window_index(view, last_ref_index_)]];
    }
  }

  bool ready() override {
    std::lock_guard<std::mutex> lk(mu_);
    return !busy_;
  }
  void wait() override {
    std::unique_lock<std::mutex> lk(mu_);
    cv_done_.wait(lk, [this] { return !busy_; });
  }

  void get_result(float* depth, float* conf, float* depth_dense, float* conf_dense) override {
    std::unique_lock<std::mutex> lk(mu_);
    cv_done_.wait(lk, [this] { return !busy_; });
    if (!worker_error_.empty()) { std::string e = worker_error_; worker_error_.clear(); throw Error(e); }
    if (!has_result_) throw Error("GetResult without a pending result (dr_mvsnet.cpp:100-102)");
    const size_t n = (size_t)H_ * W_;
    float* dst[4] = {depth, conf, depth_dense, conf_dense};
    const char* names[4] = {"s3.depth", "s3.confidence", "s3.depth_dense", "s3.confidence_dense"};
    TDM_CUDA(cudaSetDevice(device_));
    const void* dstv[4] = {depth, conf, depth_dense, conf_dense};
    if (all_page_locked(dstv, 4)) {
      // Page-locked result buffers: the four maps are DMA'd from the device straight into them (they stay on the device
      // until this handle's next forward, which cannot start before this call returns) - no staging copy.
      for (int k = 0; k < 4; ++k)
        TDM_CUDA(cudaMemcpyAsync(dst[k], fbuf(names[k]), n * 4, cudaMemcpyDeviceToHost, stream_.get()));
      TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    } else {
      if (!eager_d2h_) {   // the worker did not copy back: do it now
        for (int k = 0; k < 4; ++k) {
          TDM_CUDA(cudaMemcpyAsync(h_out_.get() + k * n, fbuf(names[k]), n * 4, cudaMemcpyDeviceToHost, stream_.get()));
          TDM_CUDA(cudaEventRecord(ev_out_[k].get(), stream_.get()));
        }
      }
      // each map is copied to caller memory by the pool as soon as its D2H has landed
      std::vector<CopyPool::Job> jobs;
      TDM_CUDA(cudaEventSynchronize(ev_out_[3].get()));   // 4.9 MB over PCIe: ~0.1 ms; simpler than per-map hand-off
      constexpr int kSlices = 2;
      for (int k = 0; k < 4; ++k)
        if (dst[k])
          for (int sl = 0; sl < kSlices; ++sl) {
            const size_t e0 = n * sl / kSlices, e1 = n * (sl + 1) / kSlices;
            jobs.push_back({dst[k] + e0, h_out_.get() + k * n + e0, (e1 - e0) * 4, nullptr});
          }
      CopyPool::shared().run(jobs);
    }
    fill_handoff();
    has_result_ = false;
  }

  void read_handoff(void* stream, const std::function<void(const Handoff&)>& consume) override {
    std::unique_lock<std::mutex> lk(mu_);
    if (!ho_valid_) throw Error("no MVSNet result to integrate: call GetResult first");
    Handoff h;
    h.depth = d_ho_depth_.get();
    h.bgr = d_ho_bgr_.get();
    std::memcpy(h.c2w, ho_c2w_, sizeof(ho_c2w_));
    h.H = ho_H_; h.W = ho_W_; h.device = device_;
    h.ready = (void*)ev_ho_ready_.get();
    try {
      consume(h);
    } catch (...) {
      // consume may have enqueued reads before it failed: mark them too (on another device's stream this fails, and then
      // consume enqueued nothing)
      if (!record_release(stream)) cudaGetLastError();
      throw;
    }
    TDM_CHECK(record_release(stream), "keyframe handoff: cannot record the release event");
  }

  void stage_output(int stage, const std::string& which, float* out, size_t cap) override {
    wait();
    TDM_CHECK(stage >= 1 && stage <= 3, "stage must be 1..3");
    TDM_CUDA(cudaSetDevice(device_));
    const std::string name = "s" + std::to_string(stage) + "." + which;
    auto it = bufs_.find(name);
    if (it == bufs_.end()) throw Error("no such stage output: " + name);
    const size_t n = (size_t)it->second.H * it->second.W;
    TDM_CHECK(cap >= n, "stage_output: capacity too small");
    TDM_CUDA(cudaMemcpy(out, it->second.p.get(), n * 4, cudaMemcpyDeviceToHost));
  }

  // FeatureNet intermediates ("f.*") are those of the last forward, over the views it computed (k planes after a cached call);
  // feat1..feat3 are returned in window order (reference first) whichever pool slots hold the views.
  long long debug_tensor(const std::string& name, float* out, size_t cap, int* dims4) override {
    wait();
    TDM_CUDA(cudaSetDevice(device_));
    auto it = bufs_.find(fk_ < V_ && name.compare(0, 2, "f.") == 0 ? name + "@" + std::to_string(fk_) : name);
    if (it == bufs_.end()) throw Error("no such tensor: " + name);
    const DevBuf& b = it->second;
    const long long npos = (long long)b.D * b.H * b.W;
    const long long n = npos * b.C;
    if (dims4) { dims4[0] = b.C; dims4[1] = b.D; dims4[2] = b.H; dims4[3] = b.W; }
    if (!out) return n;
    TDM_CHECK((long long)cap >= n, "debug_tensor: capacity too small");
    if (b.f32) {
      TDM_CUDA(cudaMemcpy(out, b.p.get(), n * 4, cudaMemcpyDeviceToHost));  // C==1 planar already
      return n;
    }
    const DevPtr<float> tmp = make_dev<float>(n * 4);
    if (b.kind == 2) k_p8_to_planar_f32<TV><<<cdiv(n, 256), 256, 0, stream_.get()>>>(p8<const TV>(b), tmp.get());
    else k_p8_to_planar_f32<TA><<<cdiv(n, 256), 256, 0, stream_.get()>>>(p8<const TA>(b), tmp.get());
    TDM_CUDA(cudaGetLastError());
    TDM_CUDA(cudaMemcpyAsync(out, tmp.get(), n * 4, cudaMemcpyDeviceToHost, stream_.get()));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    if (b.kind == 2 && kVolScale != 1.f)
      for (long long i = 0; i < n; ++i) out[i] *= 1.f / kVolScale;   // report the volume in its own units
    if ((name == "feat1" || name == "feat2" || name == "feat3") && !slots_identity()) {
      const std::vector<float> t(out, out + n);
      const long long plane = (long long)b.H * b.W;
      for (int c = 0; c < b.C; ++c)
        for (int v = 0; v < b.D; ++v)
          std::memcpy(out + ((long long)c * b.D + v) * plane, t.data() + ((long long)c * b.D + view_slot_[v]) * plane, plane * 4);
    }
    return n;
  }

  void run_resident(int iters, float* ms_total, int* launches) override { run_resident_new(V_, iters, ms_total, launches); }

  void run_resident_new(int n_new, int iters, float* ms_total, int* launches) override {
    wait();
    TDM_CHECK(have_inputs_, "run_resident: no window submitted yet");
    TDM_CHECK(n_new >= 1 && n_new <= V_, "run_resident: n_new must be 1..view_num");
    TDM_CUDA(cudaSetDevice(device_));
    int slots[kMaxSrc + 1];
    for (int j = 0; j < n_new; ++j) slots[j] = view_slot_[window_index(V_ - n_new + j, last_ref_index_)];
    if (n_new < V_) ensure_feature_scratch(n_new);
    const Event e0 = make_event(), e1 = make_event();
    TDM_CUDA(cudaEventRecord(e0.get(), stream_.get()));
    for (int i = 0; i < iters; ++i) forward(n_new, slots, false);
    TDM_CUDA(cudaEventRecord(e1.get(), stream_.get()));
    TDM_CUDA(cudaEventSynchronize(e1.get()));
    TDM_CUDA(cudaEventElapsedTime(ms_total, e0.get(), e1.get()));
    if (launches) *launches = launches_per_forward_;
  }

  void* resident_stream() override { return (void*)stream_.get(); }
  int resident_device() const override { return device_; }
  int resident_launch(int iters) override {
    wait();
    TDM_CHECK(have_inputs_, "run_resident: no window submitted yet");
    TDM_CUDA(cudaSetDevice(device_));
    for (int i = 0; i < iters; ++i) forward(V_, nullptr, false);
    return launches_per_forward_;
  }

  std::string profile() override {
    wait();
    TDM_CHECK(have_inputs_, "profile: no window submitted yet");
    TDM_CUDA(cudaSetDevice(device_));
    forward(V_, nullptr, false);  // warm
    recs_.clear();
    forward(V_, nullptr, true);
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    std::ostringstream os;
    for (auto& r : recs_) {
      cudaEventElapsedTime(&r.ms, r.e0.get(), r.e1.get());
      os << r.name << " " << r.ms << " " << (long long)r.bytes << " " << (long long)r.flops << "\n";
    }
    recs_.clear();
    return os.str();
  }

 private:
  // ---------------------------------------------------------------- weights
  void add_conv(const std::string& key, const FoldedConv& fc_in) {
    FoldedConv fc = fc_in;
    if (kVolScale != 1.f && key.size() > 6 && key.compare(key.size() - 6, 6, ".conv0") == 0 && key[0] == 's')
      for (auto& v : fc.w) v *= 1.f / kVolScale;   // the stage's conv0 reads the volume stored as value * kVolScale (exact power of two)
    DevConv dc;
    dc.cin = fc.cin; dc.cout = fc.cout; dc.kd = fc.kd; dc.kh = fc.kh; dc.kw = fc.kw; dc.transposed = fc.transposed;
    dc.w = make_dev<float>(fc.w.size() * 4);
    TDM_CUDA(cudaMemcpy(dc.w.get(), fc.w.data(), fc.w.size() * 4, cudaMemcpyHostToDevice));
    if (!fc.bias.empty()) {
      dc.bias = make_dev<float>(fc.bias.size() * 4);
      TDM_CUDA(cudaMemcpy(dc.bias.get(), fc.bias.data(), fc.bias.size() * 4, cudaMemcpyHostToDevice));
    }
    if (key.size() == 7 && key.compare(2, 5, ".prob") == 0 && key[0] == 's' && fc.w.size() == 216) {
      TDM_CHECK(fc.cin == 8 && fc.cout == 1 && fc.kd == 3 && fc.kh == 3 && fc.kw == 3, "unexpected prob layer shape");
      std::memcpy(prob_w_[key[1] - '1'].w, fc.w.data(), 216 * sizeof(float));   // [tap][cin][1] == [kd][kh][kw][cin]
      have_prob_w_ = true;
    }
    if constexpr (sizeof(TA) == 2) {
      const bool vol_in = key.size() > 6 && key.compare(key.size() - 6, 6, ".conv0") == 0 && key[0] == 's';
      const bool shape_ok = !fc.transposed && fc.kh == 3 && fc.kw == 3 && (fc.kd == 1 || fc.kd == 3) &&
                            (((fc.cin == 8 || fc.cin == 16 || fc.cin == 32) &&
                              (fc.cout == 1 || fc.cout == 8 || fc.cout == 16 || fc.cout == 32)) ||
                             (fc.cin == 64 && fc.cout == 64 && fc.kd == 3));
      if (shape_ok) {
        dc.npad = fc.cout < 16 ? 16 : (fc.cin == 64 ? 32 : fc.cout);
        dc.nsplit = fc.cin == 64 ? 2 : 1;
        dc.hilo = dc.npad <= 32 && fc.cin <= 32 && !(fc.kd == 3 && fc.cin == 32 && fc.cout == 32);
        dc.tc_ok = true;
        if (vol_in) upload_bimgs<TV>(fc, dc); else upload_bimgs<TA>(fc, dc);
      }
      const bool deconv_ok = fc.transposed && fc.kd == 3 && fc.kh == 3 && fc.kw == 3 &&
                             ((fc.cin == 16 && fc.cout == 8) || (fc.cin == 32 && fc.cout == 16) || (fc.cin == 64 && fc.cout == 32));
      if (deconv_ok) {
        dc.nsplit = fc.cin == 64 ? 4 : 1;
        dc.npad = 8 * fc.cout / dc.nsplit;
        dc.tc_ok = dc.tc_deconv = true;
        std::vector<TA> img;
        tc::build_b_image_deconv<TA>(fc.w.data(), fc.cin, fc.cout, img, +from_host<TA>, dc.nsplit);
        dc.bimg = upload(img);
      }
    }
    if constexpr (sizeof(TA) == 2) {
      // stride-2 candidates (the stride itself is only known at launch): 3x3x3 convs of CostRegNet, 5x5 of FeatureNet
      const bool s2_ok = !fc.transposed && fc.kh == fc.kw && (fc.kh == 3 || fc.kh == 5) &&
                         ((fc.kd == 3 && fc.kh == 3 && ((fc.cin == 8 && fc.cout == 16) || (fc.cin == 16 && fc.cout == 32) ||
                                                        (fc.cin == 32 && fc.cout == 64))) ||
                          (fc.kd == 1 && fc.kh == 5 && ((fc.cin == 8 && fc.cout == 16) || (fc.cin == 16 && fc.cout == 32))));
      if (s2_ok) {
        dc.tc_s2 = true;
        dc.nsplit_s2 = fc.cout == 64 ? 2 : 1;
        dc.npad_s2 = fc.cout / dc.nsplit_s2;
        std::vector<std::pair<int, int>> taps;
        short off[tc::kMaxTaps + 1];
        tc::s2_tap_table(fc.kh, 64, 4096, taps, off);   // only the ORDER matters for the B image
        std::vector<TA> img;
        tc::build_b_image_s2<TA>(fc.w.data(), fc.cin, fc.cout, dc.npad_s2, fc.kd, fc.kh, taps, img, +from_host<TA>, dc.nsplit_s2);
        dc.bimg_s2 = upload(img);
      }
    }
    convs_[key] = std::move(dc);
  }

  // Algebraic fusion of the FPN tail for stage 3 (module.py:522-530): feat3 = out3(up2(i2) + skip3(c3) + b3) is linear,
  //   feat3 = [conv3x3(W3) o up2](i2 + b3)  +  conv3x3(W3 . Ws3)(c3)
  // (adding b3 to i2 BEFORE the zero-padded up-sampling reproduces the bias' border behaviour exactly).  Both terms are
  // evaluated in one launch on the coarse grid (k_conv_tc MODE 3), one fp32 accumulator and one rounding per output: 4
  // output parity classes, the 3x3 fine taps of the first pre-summed onto the 3x3 coarse neighbourhood, those of the
  // second placed per coarse tap and sub-position of c3's space-to-depth view.  The 138 MB tensor i3 is never formed.
  void build_fused_fpn() {
    const std::string f = "feature_net.";
    const FoldedConv w3 = fold_conv(wf_, f + "out.stage3.weight", "", "", false);                        // [9][32][8]
    const FoldedConv ws = fold_conv(wf_, f + "skip.stage3.weight", f + "skip.stage3.bias", "", false);   // [1][8][32]
    std::vector<double> b((size_t)9 * 8 * 8, 0.0);   // W3 . Ws3 : [9 fine taps][8][8]
    for (int t = 0; t < 9; ++t)
      for (int ci = 0; ci < 8; ++ci)
        for (int co = 0; co < 8; ++co)
          for (int m = 0; m < 32; ++m) b[((size_t)t * 8 + ci) * 8 + co] += (double)w3.w[((size_t)t * 32 + m) * 8 + co] * (double)ws.w[(size_t)ci * 32 + m];
    // coarse-grid operator [9 coarse taps][64][4 classes * 8]: input channels 0..31 are i2b, 32 + 8 q + c is channel c
    // of c3's sub-position q = (qh, qw).  Fine tap k of parity p reads fine offset p + k - 1 = 2 delta + q.
    FoldedConv a;
    a.cin = 64; a.cout = 32; a.kd = 1; a.kh = 3; a.kw = 3;
    a.w.assign((size_t)9 * 64 * 32, 0.f);
    auto delta = [](int p, int k) { return p + k - 1 < 0 ? -1 : (p + k - 1) / 2; };
    auto sub = [](int p, int k) { return (p + k + 1) % 2; };
    for (int ph = 0; ph < 2; ++ph)
      for (int pw = 0; pw < 2; ++pw)
        for (int kh = 0; kh < 3; ++kh)
          for (int kw = 0; kw < 3; ++kw) {
            const int ta = (delta(ph, kh) + 1) * 3 + (delta(pw, kw) + 1), n0 = (ph * 2 + pw) * 8;
            const int ci0 = 32 + 8 * (sub(ph, kh) * 2 + sub(pw, kw));
            for (int co = 0; co < 8; ++co) {
              for (int m = 0; m < 32; ++m) a.w[((size_t)ta * 64 + m) * 32 + n0 + co] += w3.w[((size_t)(kh * 3 + kw) * 32 + m) * 8 + co];
              for (int c = 0; c < 8; ++c) a.w[((size_t)ta * 64 + ci0 + c) * 32 + n0 + co] = (float)b[((size_t)(kh * 3 + kw) * 8 + c) * 8 + co];
            }
          }
    add_conv("f.fpn3", a);
    DevConv& dc = convs_["f.fpn3"];
    dc.cout = 8;          // real channels per class; N = 4 classes x 8 = npad
    dc.npad = 32;
    dc.hilo = dc.tc_ok = dc.tc_up2 = true;
    upload_bimgs<TA>(a, dc);
    d_bs3_ = make_dev<float>(32 * 4);
    TDM_CUDA(cudaMemcpy(d_bs3_.get(), ws.bias.data(), 32 * 4, cudaMemcpyHostToDevice));
    fused_fpn_ = true;
  }

  template <typename T>
  static DevPtr<void> upload(const std::vector<T>& img) {
    DevPtr<void> p = make_dev(img.size() * sizeof(T));
    TDM_CUDA(cudaMemcpy(p.get(), img.data(), img.size() * sizeof(T), cudaMemcpyHostToDevice));
    return p;
  }
  // B images of the stride-1 kernel and, for the 3x3x3 layers with 1 or 8 output channels, of the input-stationary one
  template <typename TB>
  void upload_bimgs(const FoldedConv& fc, DevConv& dc) {
    std::vector<TB> img;
    tc::build_b_image<TB>(fc.w.data(), fc.cin, fc.cout, dc.npad, fc.kd, img, +from_host<TB>, dc.nsplit, dc.hilo, +to_host<TB>);
    dc.bimg = upload(img);
    if (fc.kd == 3 && (fc.cout == 1 || fc.cout == 8)) {
      tc::build_b_image_is<TB>(fc.w.data(), fc.cin, fc.cout, img, +from_host<TB>, +to_host<TB>);
      dc.bimg_is = upload(img);
    }
  }
  template <typename TB> static TB from_host(float v);
  template <typename TB> static float to_host(TB v) { return (float)v; }

  void upload_weights() {
    const std::string f = "feature_net.";
    if constexpr (kRawInput) {
      // fused pre-processing + conv0.0 (k_conv00_u8): BN-folded fp32 weights of the 3 real input channels -> constant bank
      const FoldedConv c3 = fold_conv(wf_, f + "conv0.0.conv.weight", "", f + "conv0.0.bn", false);   // [9][3][8]
      TDM_CHECK(c3.cin == 3 && c3.cout == 8 && c3.kh == 3 && c3.kw == 3 && c3.kd == 1 && c3.bias.size() == 8, "unexpected conv0.0 shape");
      Conv00Weights cw;
      for (int t = 0; t < 9; ++t)
        for (int ci = 0; ci < 3; ++ci)
          for (int co = 0; co < 8; ++co) cw.w[t * 3 + ci][co] = c3.w[((size_t)t * 3 + ci) * 8 + co];
      for (int co = 0; co < 8; ++co) cw.bias[co] = c3.bias[co];
      TDM_CUDA(cudaMemcpyToSymbol(c_conv00, &cw, sizeof(cw), (size_t)slot_.index * sizeof(Conv00Weights)));
    }
    {
      FoldedConv c00 = fold_conv(wf_, f + "conv0.0.conv.weight", "", f + "conv0.0.bn", false, 8);
      if constexpr (kRawInput)   // the image is stored as exact u8/256 (k_preprocess_bgr<RAW255>): 256/255 lives in the weights
        for (auto& v : c00.w) v = (float)((double)v * (256.0 / 255.0));
      add_conv("f.conv0.0", c00);
    }
    add_conv("f.conv0.1", fold_conv(wf_, f + "conv0.1.conv.weight", "", f + "conv0.1.bn", false));
    for (int b = 1; b <= 2; ++b)
      for (int i = 0; i < 3; ++i) {
        const std::string n = "conv" + std::to_string(b) + "." + std::to_string(i);
        add_conv("f." + n, fold_conv(wf_, f + n + ".conv.weight", "", f + n + ".bn", false));
      }
    add_conv("f.out1", fold_conv(wf_, f + "out.stage1.weight", "", "", false));
    add_conv("f.out2", fold_conv(wf_, f + "out.stage2.weight", "", "", false));
    add_conv("f.out3", fold_conv(wf_, f + "out.stage3.weight", "", "", false));
    add_conv("f.skip2", fold_conv(wf_, f + "skip.stage2.weight", f + "skip.stage2.bias", "", false));
    add_conv("f.skip3", fold_conv(wf_, f + "skip.stage3.weight", f + "skip.stage3.bias", "", false));
    if constexpr (sizeof(TA) == 2) build_fused_fpn();
    for (int s = 1; s <= 3; ++s) {
      const std::string p = "cost_regularization_net.stage" + std::to_string(s) + ".";
      const std::string k = "s" + std::to_string(s) + ".";
      for (int i = 0; i <= 6; ++i) {
        const std::string n = "conv" + std::to_string(i);
        add_conv(k + n, fold_conv(wf_, p + n + ".conv.weight", "", p + n + ".bn", false));
      }
      for (int i : {7, 9, 11}) {
        const std::string n = "conv" + std::to_string(i);
        add_conv(k + n, fold_conv(wf_, p + n + ".conv.weight", "", p + n + ".bn", true));
      }
      add_conv(k + "prob", fold_conv(wf_, p + "prob.weight", "", "", false));
      if (va_) {
        // volume_gates (cva_mvsnet.py:76-83): conv(C->1)+b, BN, ReLU, conv(1->1)+b, BN, ReLU folded to scalars
        const std::string g = "volume_gates.stage" + std::to_string(s) + ".";
        auto bn = [&](const std::string& pre, double& sc, double& sh, double bias) {
          const double ga = wf_.get(pre + ".weight").data[0], be = wf_.get(pre + ".bias").data[0];
          const double mu = wf_.get(pre + ".running_mean").data[0], var = wf_.get(pre + ".running_var").data[0];
          sc = ga / std::sqrt(var + 1e-5);
          sh = (bias - mu) * sc + be;
        };
        double s1, b1, s2, b2;
        bn(g + "1", s1, b1, wf_.get(g + "0.bias").data[0]);
        bn(g + "4", s2, b2, wf_.get(g + "3.bias").data[0]);
        const auto& w1 = wf_.get(g + "0.weight").data;
        Gate& gt = gates_[s - 1];
        gt.C = (int)w1.size();
        for (int c = 0; c < gt.C; ++c) gt.w1[c] = (float)(w1[c] * s1);
        gt.b1 = (float)b1;
        gt.w2 = (float)(wf_.get(g + "3.weight").data[0] * s2);
        gt.b2 = (float)b2;
      }
    }
    select_state_ = make_dev<SelectState>(sizeof(SelectState));
    TDM_CUDA(cudaMemset(select_state_.get(), 0, sizeof(SelectState)));
    h_params_ = make_host<CallParams>(sizeof(CallParams));
    d_params_ = make_dev<CallParams>(sizeof(CallParams));
    h_feat_slot_ = make_host<int>(sizeof(c_feat_slot[0]));
    for (int v = 0; v <= kMaxSrc; ++v) view_slot_[v] = v;
  }

  // ---------------------------------------------------------------- buffers
  // f32: plain fp32 [C][D][H][W] map (logits, depth maps).  Otherwise P8 layout with zero halos; pd3 = 3-D tensor
  // (halo along D as well), vol = cost-volume element type.
  DevBuf& alloc(const std::string& name, int C, int D, int H, int W, bool f32 = false, bool vol = false, bool pd3 = false) {
    DevBuf b;
    b.C = C; b.D = D; b.H = H; b.W = W; b.f32 = f32;
    b.kind = f32 ? 0 : (vol ? 2 : 1);
    const size_t es = f32 ? 4 : (vol ? sizeof(TV) : sizeof(TA));
    b.alg_bytes = (size_t)C * D * H * W * es;
    if (f32) {
      b.bytes = b.alg_bytes;
    } else {
      TDM_CHECK(C % 8 == 0, "P8 layout needs a multiple of 8 channels");
      b.pd = pd3 ? 1 : 0;
      b.bytes = (size_t)(C / 8) * (D + 2 * b.pd) * (H + 2) * (W + 2) * 8 * es + 4096;  // + slack for tile over-reads
    }
    b.p = make_dev(b.bytes);
    TDM_CUDA(cudaMemsetAsync(b.p.get(), 0, b.bytes, stream_.get()));  // halos stay zero forever: kernels only write the interior
    if (debug_poison_) {
      // all-ones bytes are a NaN in fp32, fp16 and bf16: a position the forward should have stored but did not reads as
      // non-finite instead of as a plausible 0 (which a ReLU layer's true output often is).  The P8 interiors and the
      // logits are poisoned; the other fp32 maps are not all written by every forward (depth / confidence / edge of the
      // stages the edge filter skips, thr's spare entry) and keep their zeros.
      if (!f32) {
        const size_t row = (size_t)(W + 2) * 8 * es;
        for (int p = 0; p < (C / 8) * (D + 2 * b.pd); ++p) {
          const int d = p % (D + 2 * b.pd);
          if (d < b.pd || d >= D + b.pd) continue;
          TDM_CUDA(cudaMemset2DAsync((uint8_t*)b.p.get() + ((size_t)p * (H + 2) + 1) * row + 8 * es, row, 0xFF, (size_t)W * 8 * es, H, stream_.get()));
        }
      } else if (name.size() >= 6 && name.compare(name.size() - 6, 6, "logits") == 0) {
        TDM_CUDA(cudaMemsetAsync(b.p.get(), 0xFF, b.bytes, stream_.get()));
      }
    }
    DevBuf& slot = bufs_[name];
    slot = std::move(b);
    return slot;
  }
  template <typename T>
  static P8<T> p8(const DevBuf& b) {
    P8<T> t;
    t.p = (T*)b.p.get();
    t.C = b.C; t.D = b.D; t.H = b.H; t.W = b.W; t.pd = b.pd;
    t.Hp = b.H + 2; t.Wp = b.W + 2;
    t.gs = (long long)(b.D + 2 * b.pd) * t.Hp * t.Wp * 8;
    return t;
  }
  void free_plan() {
    drop_graph();
    tc_cache_.clear();
    bufs_.clear();
    h_bgr_.reset();
    h_out_.reset();
    d_bgr_.reset();
    cache_valid_ = false;
    for (int v = 0; v <= kMaxSrc; ++v) view_slot_[v] = v;
  }
  // FeatureNet's buffers over D views; sfx "" = the whole window (feat1..feat3 are then the feature pool), "@k" = the scratch
  // of a cached forward over k new views
  void alloc_featurenet(int D, const std::string& sfx, int H, int W) {
    alloc("f.img" + sfx, 8, D, H, W);
    alloc("f.c0_0" + sfx, 8, D, H, W);
    alloc("f.c3" + sfx, 8, D, H, W);
    alloc("f.c1_0" + sfx, 16, D, H / 2, W / 2);
    alloc("f.c1_1" + sfx, 16, D, H / 2, W / 2);
    alloc("f.c2" + sfx, 16, D, H / 2, W / 2);
    alloc("f.c2_0" + sfx, 32, D, H / 4, W / 4);
    alloc("f.c2_1" + sfx, 32, D, H / 4, W / 4);
    alloc("f.c1" + sfx, 32, D, H / 4, W / 4);
    alloc("feat1" + sfx, 32, D, H / 4, W / 4);
    alloc("f.i2" + sfx, 32, D, H / 2, W / 2);
    alloc("f.i2b" + sfx, 32, D, H / 2, W / 2);
    alloc("feat2" + sfx, 16, D, H / 2, W / 2);
    alloc("f.i3" + sfx, 32, D, H, W);
    alloc("feat3" + sfx, 8, D, H, W);
  }
  // made once per k and plan (freed with the plan), outside any capture: the forward over k views then replays as its own graph
  void ensure_feature_scratch(int k) {
    if (!bufs_.count("feat1@" + std::to_string(k))) alloc_featurenet(k, "@" + std::to_string(k), H_, W_);
  }
  void ensure_plan(int V, int H, int W) {
    if (V == V_ && H == H_ && W == W_) return;
    free_plan();
    V_ = H_ = W_ = 0;   // no plan until every buffer below exists
    h_bgr_ = make_host<unsigned char>((size_t)V * H * W * 3);
    h_out_ = make_host<float>((size_t)4 * H * W * sizeof(float));
    d_bgr_ = make_dev<unsigned char>((size_t)V * H * W * 3);
    alloc_featurenet(V, "", H, W);
    for (int s = 1; s <= 3; ++s) {
      const std::string k = "s" + std::to_string(s) + ".";
      const int sc = 1 << (3 - s);
      const int Hs = H / sc, Ws = W / sc, D = depth_num_[s - 1];
      const int C = 32 >> (s - 1);
      const bool four = (D == 4);
      TDM_CHECK(D % 2 == 0 && (four || D % 8 == 0), "depth_num must be 4 or a multiple of 8");
      const int D1 = D / 2, D2 = D / 4, D3 = four ? D2 : D / 8;
      alloc(k + "volume", C, D, Hs, Ws, false, true, true);
      alloc(k + "c0", 8, D, Hs, Ws, false, false, true);
      alloc(k + "c1", 16, D1, Hs / 2, Ws / 2, false, false, true);
      alloc(k + "c2", 16, D1, Hs / 2, Ws / 2, false, false, true);
      alloc(k + "c3", 32, D2, Hs / 4, Ws / 4, false, false, true);
      alloc(k + "c4", 32, D2, Hs / 4, Ws / 4, false, false, true);
      alloc(k + "c5", 64, D3, Hs / 8, Ws / 8, false, false, true);
      alloc(k + "c6", 64, D3, Hs / 8, Ws / 8, false, false, true);
      alloc(k + "x7", 32, D2, Hs / 4, Ws / 4, false, false, true);
      alloc(k + "x9", 16, D1, Hs / 2, Ws / 2, false, false, true);
      alloc(k + "x11", 8, D, Hs, Ws, false, false, true);
      alloc(k + "logits", 1, D, Hs, Ws, true);
      for (const char* n : {"depth_dense", "confidence_dense", "depth", "confidence", "edge"})
        alloc(k + n, 1, 1, Hs, Ws, true);
    }
    alloc("thr", 1, 1, 1, 4, true);
    V_ = V; H_ = H; W_ = W;
  }
  float* fbuf(const std::string& n) { return (float*)bufs_.at(n).p.get(); }

  // ---------------------------------------------------------------- launches
  void rec_begin(const std::string& name, double bytes, double flops) {
    ++launch_count_;
    if (!profiling_) return;
    LaunchRec r;
    r.name = name; r.bytes = bytes; r.flops = flops;
    r.e0 = make_event();
    r.e1 = make_event();
    cudaEventRecord(r.e0.get(), stream_.get());
    recs_.push_back(std::move(r));
  }
  void rec_end() {
    if (!profiling_) return;
    cudaEventRecord(recs_.back().e1.get(), stream_.get());
  }
  void rec_cancel() {
    --launch_count_;
    if (!profiling_) return;
    recs_.pop_back();
  }

  template <typename TIn, typename TOut, int CIN, int COUT>
  void conv_inst(const DevBuf& in, const DevConv& c, const DevBuf* res, const DevBuf& out, const ConvGeom& g,
                 const DevBuf* out_b = nullptr, const float* bias_b = nullptr) {
    const long long npos = (long long)g.Do * g.Ho * g.Wo;
    P8<const TOut> r{};
    if (res) r = p8<const TOut>(*res);
    P8<TOut> o{}, ob{};
    float* plain = nullptr;
    if constexpr (COUT == 1) plain = (float*)out.p.get(); else o = p8<TOut>(out);
    if constexpr (COUT != 1) {
      if (out_b) {
        ob = p8<TOut>(*out_b);
        launch_k(k_conv_direct<TIn, TOut, CIN, COUT>, dim3(cdiv(npos, 128)), dim3(128), p8<const TIn>(in), c.w.get(), c.bias.get(), r, o, plain, g, ob, bias_b);
        return;
      }
    }
    if constexpr (COUT >= 16) {
      if (npos < 128ll * 592) {  // too few positions to fill the chip: split the output channels over blockIdx.y
        dim3 grid(cdiv(npos, 128), COUT / 8);
        launch_k(k_conv_direct<TIn, TOut, CIN, COUT, 8>, grid, dim3(128), p8<const TIn>(in), c.w.get(), c.bias.get(), r, o, plain, g, P8<TOut>{}, (const float*)nullptr);
        return;
      }
    }
    launch_k(k_conv_direct<TIn, TOut, CIN, COUT>, dim3(cdiv(npos, 128)), dim3(128), p8<const TIn>(in), c.w.get(), c.bias.get(), r, o, plain, g, P8<TOut>{}, (const float*)nullptr);
  }

  // the other kernels of the forward (all begin with grid_dep_sync()): with use_pdl = 2 they carry the attribute too
  template <typename... KArgs, typename... Args>
  void launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, Args&&... args) {
    if (use_pdl_ < 2) {
      kern<<<grid, block, 0, stream_.get()>>>(static_cast<KArgs>(args)...);
      return;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = 0;
    cfg.stream = stream_.get();
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    TDM_CUDA(cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...));
  }

  // Tensor-core kernels are launched with programmatic stream serialization (PDL): their prologue and weight-image
  // load overlap the tail of the previous kernel (see Ring::start in conv_tc.cuh).  Each kernel's shared-memory limit
  // is raised once, on its first launch.  The block size is read from the instantiation itself: its
  // __launch_bounds__(tc::conv_threads(NWG), 1) is the kernel's maxThreadsPerBlock, i.e. its NWG consumer warpgroups and
  // the producer warp, so the launch cannot disagree with the barrier counts and the producer index compiled into it.
  template <auto Kern, typename... Args>
  void launch_tc(dim3 grid, size_t smem, Args... args) {
    static int threads = 0;
    if (!threads) {
      TDM_CUDA(cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      cudaFuncAttributes fa{};
      TDM_CUDA(cudaFuncGetAttributes(&fa, Kern));
      TDM_CHECK(fa.maxThreadsPerBlock == tc::conv_threads(2) || fa.maxThreadsPerBlock == tc::conv_threads(4),
                "tensor-core conv: unexpected block size " + std::to_string(fa.maxThreadsPerBlock));
      threads = fa.maxThreadsPerBlock;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = dim3(threads);
    // with PDL an early-launched dependent must not stack several CTAs on the few SMs its predecessor left idle (they would
    // compete for those SMs' issue slots while the rest of the GPU waits): ask for enough shared memory that one CTA fills an SM
    cfg.dynamicSmemBytes = use_pdl_ ? std::max(smem, (size_t)pdl_min_smem_kb_ * 1024) : smem;
    cfg.stream = stream_.get();
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = use_pdl_ ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    TDM_CUDA(cudaLaunchKernelEx(&cfg, Kern, args...));
  }

  // Tile plan and input tensor map of one layer's tensor-core launch, made on first use.  Keys: the layer, + "#tail" (prob
  // with the soft-argmin tail), "#is" / "#is#tail" (input-stationary kernel), "#s2" (stride-2 kernel); the output-stationary
  // and stride-2 keys end in "@" + the input's D.
  struct TcCache { tc::Plan plan; tc::PlanS2 plan_s2; CUtensorMap tmap, tmap_res, tmap_out; };
  std::map<std::string, TcCache> tc_cache_;

  template <typename Make>
  const TcCache& tc_cached(const std::string& key, Make make) {
    auto it = tc_cache_.find(key);
    if (it == tc_cache_.end()) it = tc_cache_.emplace(key, make()).first;
    return it->second;
  }

  static void debug_plan(const std::string& wkey, const std::string& what, const tc::Tile& t, int grid, int nsplit, size_t smem) {
    if (std::getenv("TDM_DEBUG_PLAN"))
      fprintf(stderr, "[plan] %-14s %s %dx%dx%d -> R %d TW %d DR %d S %d nch %d tiles %d x nsplit %d smem %zu\n", wkey.c_str(), what.c_str(),
              t.D, t.H, t.W, t.R, t.TW, t.DR, t.S, t.nch, grid, nsplit, smem);
  }

  // tensor map over a P8 input {8 channels, Wp, Hp, channel group * padded planes}; a box is box_w x box_h positions of
  // one plane, every estr-th column / row
  template <typename TIn>
  CUtensorMap p8_tmap(const std::string& wkey, const DevBuf& in, int cg, int iDp, int box_w, int box_h, int estr) {
    CUtensorMap tmap;
    const cuuint64_t dims[4] = {8, (cuuint64_t)(in.W + 2), (cuuint64_t)(in.H + 2), (cuuint64_t)iDp * cg};
    const cuuint64_t strides[3] = {16, (cuuint64_t)(in.W + 2) * 16, (cuuint64_t)(in.W + 2) * (in.H + 2) * 16};
    const cuuint32_t box[4] = {8, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
    const cuuint32_t es[4] = {1, (cuuint32_t)estr, (cuuint32_t)estr, 1};
    const CUtensorMapDataType dt = std::is_same<TIn, __nv_bfloat16>::value ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    const CUresult r = tc::encode_tiled_fn()(&tmap, dt, 4, in.p.get(), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    TDM_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed for " + wkey + " (" + std::to_string((int)r) + ")");
    return tmap;
  }

  // tensor map over the interior of a 3-D P8 output (or skip) tensor {8 channels, W, H, D, channel group} for the output
  // boxes of the transposed convs: box 2 tw columns x 2 r rows x 2 planes x groups channel groups.  Boxes are moved as
  // 16-bit words, fp16 or bf16 alike; elements beyond the interior are zero-filled on loads and skipped on stores, so the
  // halos stay zero.
  CUtensorMap p8_interior_tmap(const std::string& wkey, const DevBuf& t, int tw, int r, int groups) {
    TDM_CHECK(t.pd == 1 && 2 * tw <= 256 && 2 * r <= 256, wkey + ": output box out of the TMA limits");
    CUtensorMap tmap;
    const P8<TA> v = p8<TA>(t);
    TA* base = v.p + ((long long)(v.Hp + 1) * v.Wp + 1) * 8;   // plane 1 (the first interior one), row 1, column 1
    const cuuint64_t dims[5] = {8, (cuuint64_t)t.W, (cuuint64_t)t.H, (cuuint64_t)t.D, (cuuint64_t)(t.C / 8)};
    const cuuint64_t strides[4] = {16, (cuuint64_t)v.Wp * 16, (cuuint64_t)v.Wp * v.Hp * 16, (cuuint64_t)v.gs * 2};
    const cuuint32_t box[5] = {8, (cuuint32_t)(2 * tw), (cuuint32_t)(2 * r), 2, (cuuint32_t)groups};
    const cuuint32_t es[5] = {1, 1, 1, 1, 1};
    const CUresult res = tc::encode_tiled_fn()(&tmap, CU_TENSOR_MAP_DATA_TYPE_UINT16, 5, base, dims, strides, box, es,
                                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                               CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    TDM_CHECK(res == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed for the output box of " + wkey + " (" + std::to_string((int)res) + ")");
    return tmap;
  }

  // input-stationary 3x3x3 stride-1 conv (conv_tc_is.cuh) of a layer with 8 (CPK 16) or 1 (CPK 8, fp32 plain output) channels
  template <typename TIn, int CIN, int CPK, bool PLAIN, typename Tail = tc::NoTail>
  void tc_is_inst(const std::string& wkey, const DevBuf& in, const DevConv& c, const DevBuf& out, bool relu, const Tail& tail = Tail()) {
    const TcCache& tcx = tc_cached(wkey + (Tail::enabled ? "#is#tail" : "#is"), [&] {
      TcCache x{};
      x.plan = tc::make_plan_is(CIN, CPK, in.D, in.H, in.W, (size_t)tc_smem_kb_ * 1024, Tail::enabled);
      tc::Geom& g = x.plan.g;
      TDM_CHECK(!Tail::enabled || g.tiles_d == 1, "the prob tail needs tiles that span all depth planes");
      g.iDp = in.D + 2;
      g.relu = relu ? 1 : 0;
      g.cout = c.cout;
      x.tmap = p8_tmap<TIn>(wkey, in, CIN / 8, g.iDp, g.P, g.R + 2, 1);
      debug_plan(wkey, "IS cin " + std::to_string(CIN) + " N " + std::to_string(3 * CPK) + " in", g, x.plan.grid, 1, x.plan.smem);
      return x;
    });
    const tc::Plan& pl = tcx.plan;
    if (profiling_) recs_.back().name = wkey + "[tc-is]";   // the record conv() opened as "[tc]"
    constexpr int NWG = tc::conv_nwg(0, 3 * CPK, Tail::max_d);
    TDM_CHECK(pl.nwg == NWG, wkey + ": tile plan balanced for another warpgroup count than the kernel's");
    launch_tc<tc::k_conv_tc_is<TIn, TA, CIN, CPK, PLAIN, Tail, NWG>>(dim3(pl.grid), pl.smem, tcx.tmap, (const TIn*)c.bimg_is.get(), (const float*)c.bias.get(),
                                                               PLAIN ? (TA*)nullptr : (TA*)out.p.get(), PLAIN ? (float*)out.p.get() : (float*)nullptr, pl.g, tail);
  }

  template <typename TIn, typename TOut, int CIN, int NPAD, int KD, bool PLAIN, int MODE = 0, bool HILO = false, typename Tail = tc::NoTail>
  void tc_inst(const std::string& wkey, const DevBuf& in, const DevConv& c, const DevBuf* res, const DevBuf& out, bool relu,
               const Tail& tail = Tail()) {
    // res: MODE 1's skip operand (optional), MODE 3's fine input (f.c3)
    TDM_CHECK(MODE == 1 || (MODE == 3) == (res != nullptr), wkey + ": MODE 3 takes a fine input, MODE 0 no residual");
    // FeatureNet layers run over V planes or, with the feature cache, over k: one plan and tensor map per plane count
    const TcCache& tcx = tc_cached(wkey + (Tail::enabled ? "#tail" : "") + "@" + std::to_string(in.D), [&] {
      TcCache x{};
      x.plan = tc::make_plan(CIN, HILO ? 2 * NPAD : NPAD, KD, in.D, in.H, in.W, in.pd, MODE, (size_t)tc_smem_kb_ * 1024,   // tiles live on the INPUT grid
                             Tail::enabled);
      tc::Geom& g = x.plan.g;
      TDM_CHECK(!Tail::enabled || g.tiles_d == 1, "the prob tail needs tiles that span all depth planes");
      g.oHp = out.H + 2; g.oWp = out.W + 2; g.opd = out.pd;
      g.iDp = in.D + 2 * in.pd;
      g.in_gs = p8<const TIn>(in).gs;
      g.relu = relu ? 1 : 0;
      g.has_res = res ? 1 : 0;
      g.cout = c.cout;
      if constexpr (!PLAIN) g.out_gs = p8<TOut>(out).gs;
      x.tmap = p8_tmap<TIn>(wkey, in, MODE == 3 ? 4 : CIN / 8, g.iDp, g.P, g.R + 2, 1);
      x.tmap_res = x.tmap_out = x.tmap;   // read by MODE 1 and 3 only
      if constexpr (MODE == 1) {
        x.tmap_out = p8_interior_tmap(wkey, out, g.TW, g.R, NPAD / 64);
        if (res) x.tmap_res = p8_interior_tmap(wkey, *res, g.TW, g.R, NPAD / 64);
      }
      if constexpr (MODE == 3) x.tmap_res = p8_tmap<TIn>(wkey, *res, 1, res->D, 2 * g.P, 2 * (g.R + 2), 2);
      debug_plan(wkey, "mode " + std::to_string(MODE) + " cin " + std::to_string(CIN) + " N " + std::to_string(HILO ? 2 * NPAD : NPAD) +
                 " kd " + std::to_string(KD) + " in", g, x.plan.grid, c.nsplit, x.plan.smem);
      return x;
    });
    const tc::Plan& pl = tcx.plan;
    TOut* op = nullptr;
    float* plain = nullptr;
    if constexpr (PLAIN) plain = (float*)out.p.get();
    else op = (TOut*)out.p.get();
    constexpr int NWG = tc::conv_nwg(MODE, HILO ? 2 * NPAD : NPAD, Tail::max_d);
    TDM_CHECK(pl.nwg == NWG, wkey + ": tile plan balanced for another warpgroup count than the kernel's");
    // MODE 1: each N slice of NPAD columns is 8 classes x NPAD / 8 channels, whole output channel groups of the box;
    // MODE 3: the epilogue pairs column blocks pw = 0 / 1 of cout = 8
    TDM_CHECK((MODE != 1 || (c.cout == CIN / 2 && c.cout == c.nsplit * NPAD / 8 && NPAD % 64 == 0 && (NPAD == 64 || c.nsplit == 1))) &&
              (MODE != 3 || (c.cout == 8 && c.nsplit == 1)), wkey + ": parity-class layer with an unexpected cout");
    TDM_CHECK(MODE != 1 || (out.pd == 1 && (!res || (res->D == out.D && res->H == out.H && res->W == out.W && res->C == out.C))),
              wkey + ": transposed conv skip / output shapes differ");
    launch_tc<tc::k_conv_tc<TIn, TOut, CIN, NPAD, KD, PLAIN, MODE, HILO, Tail, NWG>>(dim3(pl.grid, c.nsplit), pl.smem, tcx.tmap, tcx.tmap_res, tcx.tmap_out, (const TIn*)c.bimg.get(),
                                                                              (const float*)c.bias.get(), op, plain, pl.g, tail);
  }

  template <int CIN, int NPAD, int KD, int KS>
  void tc_s2_inst(const std::string& wkey, const DevBuf& in, const DevConv& c, const DevBuf& out, bool relu) {
    const TcCache& tcx = tc_cached(wkey + "#s2@" + std::to_string(in.D), [&] {
      TcCache x{};
      x.plan_s2 = tc::make_plan_s2(CIN, NPAD, KD, KS, out.D, out.H, out.W, (size_t)tc_smem_kb_ * 1024);
      tc::GeomS2& g = x.plan_s2.g;
      g.oHp = out.H + 2; g.oWp = out.W + 2; g.opd = out.pd; g.out_gs = p8<TA>(out).gs;
      g.iDp = in.D + 2 * in.pd;
      g.c0 = 1 - KS / 2;
      g.relu = relu ? 1 : 0;
      g.cout = c.cout;
      std::vector<std::pair<int, int>> taps;
      tc::s2_tap_table(KS, g.P, g.slot_pos, taps, g.tap_off);
      x.tmap = p8_tmap<TA>(wkey, in, CIN / 8, g.iDp, 2 * g.P, 2 * g.RR, 2);   // every second column / row per box
      debug_plan(wkey, "S2 cin " + std::to_string(CIN) + " N " + std::to_string(NPAD) + " kd " + std::to_string(KD) + " ks " + std::to_string(KS) + " out",
                 g, x.plan_s2.grid, c.nsplit_s2, x.plan_s2.smem);
      return x;
    });
    const tc::PlanS2& pl = tcx.plan_s2;
    constexpr int NWG = tc::conv_nwg(0, NPAD, 0);
    TDM_CHECK(pl.nwg == NWG, wkey + ": tile plan balanced for another warpgroup count than the kernel's");
    launch_tc<tc::k_conv_tc_s2<TA, TA, CIN, NPAD, KD, KS, NWG>>(dim3(pl.grid, c.nsplit_s2), pl.smem, tcx.tmap, (const TA*)c.bimg_s2.get(),
                                                          (const float*)c.bias.get(), (TA*)out.p.get(), pl.g);
  }

  bool conv_tc_s2_dispatch(const std::string& wkey, const DevBuf& bi, const DevConv& c, const DevBuf& bo, bool relu) {
    if constexpr (sizeof(TA) != 2) {
      return false;
    } else {
      if (bi.kind != 1 || bo.f32) return false;
      if (c.kd == 3 && c.cin == 8) { tc_s2_inst<8, 16, 3, 3>(wkey, bi, c, bo, relu); return true; }
      if (c.kd == 3 && c.cin == 16) { tc_s2_inst<16, 32, 3, 3>(wkey, bi, c, bo, relu); return true; }
      if (c.kd == 3 && c.cin == 32) { tc_s2_inst<32, 32, 3, 3>(wkey, bi, c, bo, relu); return true; }
      if (c.kd == 1 && c.cin == 8) { tc_s2_inst<8, 16, 1, 5>(wkey, bi, c, bo, relu); return true; }
      if (c.kd == 1 && c.cin == 16) { tc_s2_inst<16, 32, 1, 5>(wkey, bi, c, bo, relu); return true; }
      return false;
    }
  }

  // returns true if the tensor-core kernel was launched
  bool conv_tc_dispatch(const std::string& wkey, const DevBuf& bi, const DevConv& c, const DevBuf* rp, const DevBuf& bo, bool relu) {
    if constexpr (sizeof(TA) != 2) {
      return false;
    } else {
      const bool is3d = c.kd == 3;
      if (is3d != (bi.pd == 1)) return false;
      if (c.tc_deconv) {
        if (bo.D != 2 * bi.D || bo.H != 2 * bi.H || bo.W != 2 * bi.W || bi.kind != 1) return false;
        if (c.cin == 16) { tc_inst<TA, TA, 16, 64, 2, false, 1>(wkey, bi, c, rp, bo, relu); return true; }
        if (c.cin == 32) { tc_inst<TA, TA, 32, 128, 2, false, 1>(wkey, bi, c, rp, bo, relu); return true; }
        if (c.cin == 64) { tc_inst<TA, TA, 64, 64, 2, false, 1>(wkey, bi, c, rp, bo, relu); return true; }
        return false;
      }
      if (rp) return false;   // the stride-1 kernel adds no residual
#define TDM_TC(TI, CI, NP, KDV, HL)                                                        \
  if (c.cin == CI && c.npad == NP && c.kd == KDV && c.hilo == HL) {                        \
    tc_inst<TI, TA, CI, NP, KDV, false, 0, HL>(wkey, bi, c, rp, bo, relu);                       \
    return true;                                                                           \
  }
      if (use_is_ && c.bimg_is && !rp) {
        // input-stationary kernel: the stages' conv0 (cost volume in) and prob (fp32 logits out, with fused_regress the
        // softmax / soft-argmin / confidence tail)
        if (bo.f32 && bi.kind == 1 && c.cin == 8 && c.cout == 1) {
          if (tail_req_.stage && fused_regress_) {
            const TailReq& t = tail_req_;
#define TDM_TAIL(MAXD) tc_is_inst<TA, 8, 8, true, RegressTail<MAXD>>(wkey, bi, c, bo, false, RegressTail<MAXD>{t.dsrc, t.depth, t.conf, t.hyp, t.half_range})
            if (t.D <= 8) TDM_TAIL(8); else if (t.D <= 32) TDM_TAIL(32); else if (t.D <= 48) TDM_TAIL(48); else TDM_TAIL(64);
#undef TDM_TAIL
            tail_req_.done = true;
          } else {
            tc_is_inst<TA, 8, 8, true>(wkey, bi, c, bo, false);
          }
          return true;
        }
        if (!bo.f32 && bi.kind == 2 && c.cout == 8) {
          if (c.cin == 32) { tc_is_inst<TV, 32, 16, false>(wkey, bi, c, bo, relu); return true; }
          if (c.cin == 16) { tc_is_inst<TV, 16, 16, false>(wkey, bi, c, bo, relu); return true; }
          if (c.cin == 8) { tc_is_inst<TV, 8, 16, false>(wkey, bi, c, bo, relu); return true; }
        }
      }
      if (bo.f32) {
        if (!(c.cin == 8 && c.cout == 1 && c.kd == 3 && bi.kind == 1 && c.hilo)) return false;
        if (tail_req_.stage && fused_regress_) {
          // softmax / soft-argmin / confidence inside the prob convolution's epilogue: the thread that stored a pixel's D logits
          // finishes the pixel
          const TailReq& t = tail_req_;
#define TDM_TAIL(MAXD)                                                                                           \
  tc_inst<TA, TA, 8, 16, 3, true, 0, true, RegressTail<MAXD>>(wkey, bi, c, nullptr, bo, false,                   \
                                                            RegressTail<MAXD>{t.dsrc, t.depth, t.conf, t.hyp, t.half_range})
          if (t.D <= 8) TDM_TAIL(8); else if (t.D <= 32) TDM_TAIL(32); else if (t.D <= 48) TDM_TAIL(48); else TDM_TAIL(64);
#undef TDM_TAIL
          tail_req_.done = true;
        } else {
          tc_inst<TA, TA, 8, 16, 3, true, 0, true>(wkey, bi, c, nullptr, bo, false);
        }
        return true;
      }
      if (bi.kind == 2) {
        TDM_TC(TV, 32, 16, 3, true) TDM_TC(TV, 16, 16, 3, true) TDM_TC(TV, 8, 16, 3, true)
        return false;
      }
      TDM_TC(TA, 8, 16, 1, true) TDM_TC(TA, 16, 16, 1, true) TDM_TC(TA, 32, 32, 1, true) TDM_TC(TA, 32, 16, 1, true)
      TDM_TC(TA, 16, 16, 3, true) TDM_TC(TA, 32, 32, 3, false) TDM_TC(TA, 64, 32, 3, false)
#undef TDM_TC
      return false;
    }
  }

  // feat3 of the fused FPN tail (build_fused_fpn) from the coarse map `coarse` (f.i2b) and the fine map `fine` (f.c3)
  void conv_fpn3(const std::string& wkey, const std::string& coarse, const std::string& fine, const std::string& out) {
    if constexpr (sizeof(TA) == 2) {
      const DevConv& c = convs_.at(wkey);
      const DevBuf& bi = bufs_.at(coarse);
      const DevBuf& bf = bufs_.at(fine);
      const DevBuf& bo = bufs_.at(out);
      TDM_CHECK(c.tc_up2 && bo.H == 2 * bi.H && bo.W == 2 * bi.W && bo.D == bi.D && bi.C == 32 && bi.pd == 0 &&
                    bf.C == 8 && bf.pd == 0 && bf.D == bo.D && bf.H == bo.H && bf.W == bo.W,
                "conv_fpn3 shape mismatch");
      rec_begin(wkey + "[tc-up2]", (double)bi.alg_bytes + (double)bf.alg_bytes + (double)bo.alg_bytes,
                2.0 * 9 * (32 + 8) * 8 * (double)bo.D * bo.H * bo.W);
      tc_inst<TA, TA, 64, 32, 1, false, 3, true>(wkey, bi, c, &bf, bo, false);
      TDM_CUDA(cudaGetLastError());
      rec_end();
    } else {
      throw Error("conv_fpn3 needs a 16-bit engine");
    }
  }

  // stride s* per axis; 2-D convs pass the view axis as D with kd=1.
  void conv(const std::string& wkey, const std::string& in, const std::string& out, int sd, int sh, int sw,
            bool relu, int res_mode = 0, const std::string& res = "", const std::string& out_b = "",
            const float* bias_b = nullptr) {
    const DevConv& c = convs_.at(wkey);
    const DevBuf& bi = bufs_.at(in);
    const DevBuf& bo = bufs_.at(out);
    TDM_CHECK(bi.C == c.cin && bo.C == c.cout, "conv channel mismatch at " + wkey);
    ConvGeom g;
    g.Di = bi.D; g.Hi = bi.H; g.Wi = bi.W;
    g.Do = bo.D; g.Ho = bo.H; g.Wo = bo.W;
    g.kd = c.kd; g.kh = c.kh; g.kw = c.kw;
    g.sd = sd; g.sh = sh; g.sw = sw;
    g.pd = c.kd / 2; g.ph = c.kh / 2; g.pw = c.kw / 2;
    g.transposed = c.transposed ? 1 : 0;
    g.relu = relu ? 1 : 0;
    g.res_mode = res_mode;
    const double taps = (double)c.kd * c.kh * c.kw;
    const double opos = (double)bo.D * bo.H * bo.W;
    const double macs = c.transposed ? (double)bi.D * bi.H * bi.W * taps * c.cin * c.cout : opos * taps * c.cin * c.cout;
    const double bytes = (double)bi.alg_bytes + (double)bo.alg_bytes + (res_mode ? (double)bufs_.at(res).alg_bytes : 0.0);
    const DevBuf* rp = res_mode ? &bufs_.at(res) : nullptr;
    if constexpr (std::is_same<TA, __half>::value) {
      if (prob_direct_ && have_prob_w_ && bo.f32 && c.cin == 8 && c.cout == 1 && c.kd == 3 && bi.kind == 1 && bi.pd == 1 && bi.W % 4 == 0 &&
          wkey.size() == 7 && wkey.compare(2, 5, ".prob") == 0) {
        rec_begin(wkey + "[direct]", bytes, 2.0 * macs);
        const long long nthr = (long long)bi.D * bi.H * (bi.W / 4);
        k_prob_direct<4><<<cdiv(nthr, 128), 128, 0, stream_.get()>>>(p8<const __half>(bi), (float*)bo.p.get(), prob_w_[wkey[1] - '1']);
        TDM_CUDA(cudaGetLastError());
        rec_end();
        return;
      }
    }
    if (use_tc_ && c.tc_ok && res_mode != 2 && (c.tc_deconv ? (sd == 2 && sh == 2 && sw == 2) : (sd == 1 && sh == 1 && sw == 1))) {
      rec_begin(wkey + "[tc]", bytes, 2.0 * macs);
      if (conv_tc_dispatch(wkey, bi, c, rp, bo, relu)) {
        TDM_CUDA(cudaGetLastError());
        rec_end();
        return;
      }
      rec_cancel();
    }
    if (use_tc_ && c.tc_s2 && res_mode == 0 && sh == 2 && sw == 2 && sd == (c.kd == 3 ? 2 : 1)) {
      rec_begin(wkey + "[tc-s2]", bytes, 2.0 * macs);
      if (conv_tc_s2_dispatch(wkey, bi, c, bo, relu)) {
        TDM_CUDA(cudaGetLastError());
        rec_end();
        return;
      }
      rec_cancel();
    }
    rec_begin(wkey, bytes, 2.0 * macs);
    const DevBuf* obp = out_b.empty() ? nullptr : &bufs_.at(out_b);
#define TDM_CONV_CASE(CI, CO)                                                        \
  if (c.cin == CI && c.cout == CO) {                                                 \
    conv_inst<TA, TA, CI, CO>(bi, c, rp, bo, g, obp, bias_b);                        \
  } else
    if (bo.f32) {
      TDM_CHECK(c.cin == 8 && c.cout == 1 && bi.kind == 1, "fp32 output only for the prob conv");
      conv_inst<TA, float, 8, 1>(bi, c, nullptr, bo, g);
    } else if (bi.kind == 2) {  // stage conv0 reads the cost volume (type TV)
      TDM_CHECK(c.cout == 8 && !res_mode, "volume input only for conv0");
      if (c.cin == 32) conv_inst<TV, TA, 32, 8>(bi, c, rp, bo, g);
      else if (c.cin == 16) conv_inst<TV, TA, 16, 8>(bi, c, rp, bo, g);
      else if (c.cin == 8) conv_inst<TV, TA, 8, 8>(bi, c, rp, bo, g);
      else throw Error("no conv0 instantiation for " + wkey);
    } else
    TDM_CONV_CASE(8, 8) TDM_CONV_CASE(8, 16) TDM_CONV_CASE(16, 16) TDM_CONV_CASE(16, 32)
    TDM_CONV_CASE(32, 32) TDM_CONV_CASE(32, 16) TDM_CONV_CASE(32, 8) TDM_CONV_CASE(8, 32) TDM_CONV_CASE(32, 64)
    TDM_CONV_CASE(64, 64) TDM_CONV_CASE(64, 32) TDM_CONV_CASE(16, 8)
    { throw Error("no conv instantiation for " + wkey); }
#undef TDM_CONV_CASE
    TDM_CUDA(cudaGetLastError());
    rec_end();
  }

  // host side of K1: homographies H = K [R|t]_s^-1 (K [R|t]_r^-1)^-1 in double (module.py:795-808)
  void fill_cv_params(int s, CvParams& p) {
    const std::string k = "s" + std::to_string(s) + ".";
    const DevBuf& vb = bufs_.at(k + "volume");
    std::memset(&p, 0, sizeof(p));
    p.nsrc = V_ - 1; p.D = vb.D; p.H = vb.H; p.W = vb.W;
    for (int v = 0; v < V_; ++v) p.plane[v] = view_slot_[v];
    const float* K = K_ + 9 * (s - 1);
    double Pr[16], Pri[16];
    world_to_pixel(K, c2w_[0], Pr);
    if (!mat4_inv(Pr, Pri)) throw Error("reference projection is singular");
    for (int v = 1; v < V_; ++v) {
      double Ps[16], M[16];
      world_to_pixel(K, c2w_[v], Ps);
      mat4_mul(Ps, Pri, M);
      for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) p.rot[v - 1][i * 3 + j] = (float)M[i * 4 + j];
        p.trans[v - 1][i] = (float)M[i * 4 + 3];
      }
    }
    p.view_aggregation = va_ ? 1 : 0;
    p.vol_scale = kVolScale;
    if (va_) {
      const Gate& g = gates_[s - 1];
      for (int c = 0; c < g.C; ++c) p.gw1[c] = g.w1[c];
      p.gb1 = g.b1; p.gw2 = g.w2; p.gb2 = g.b2;
      float mx = 0.f;
      for (int c = 0; c < g.C; ++c) mx = std::max(mx, std::fabs(g.w1[c]));
      int e = 0;
      if (mx > 0.f && std::isfinite(mx)) std::frexp(mx, &e);      // mx = m * 2^e, m in [0.5, 1)
      p.gw1_scale = std::ldexp(1.f, -e);
      p.dot_unscale = 4096.f / p.gw1_scale;
    }
    p.hyp = hyp_spec(s);
  }

  // everything that depends on the call's poses / depth range / discard percentage -> one pinned struct -> one H2D
  void upload_call_params() {
    for (int s = 1; s <= 3; ++s) {
      fill_cv_params(s, h_params_->cv[s - 1]);
      const HypSpec hs = hyp_spec(s);
      h_params_->hyp[s - 1] = hs;
      h_params_->half_range[s - 1] = ((float)hs.D / 2.f) * hs.interval;
      const DevBuf& d = bufs_.at("s" + std::to_string(s) + ".depth_dense");
      const int n = d.H * d.W;
      // cutoff_index = trunc(H*W*(100-p)/100) in fp32, clamped (module.py:1347-1348)
      const float cf = (float)n * (100.0f - discard_) / 100.0f;
      long long cutoff = (long long)cf;
      cutoff = std::max(0ll, std::min((long long)n - 1, cutoff));
      h_params_->cutoff[s - 1] = (unsigned)cutoff;
    }
    TDM_CUDA(cudaMemcpyAsync(d_params_.get(), h_params_.get(), sizeof(CallParams), cudaMemcpyHostToDevice, stream_.get()));
    TDM_CUDA(cudaMemcpyToSymbolAsync(c_call_params, h_params_.get(), sizeof(CallParams), (size_t)slot_.index * sizeof(CallParams),
                                     cudaMemcpyHostToDevice, stream_.get()));
    TDM_CUDA(cudaMemcpyToSymbolAsync(c_feat_slot, h_feat_slot_.get(), sizeof(c_feat_slot[0]), (size_t)slot_.index * sizeof(c_feat_slot[0]),
                                     cudaMemcpyHostToDevice, stream_.get()));
  }

  void cost_volume(int s) {
    const std::string k = "s" + std::to_string(s) + ".";
    const DevBuf& fb = bufs_.at("feat" + std::to_string(s));
    const DevBuf& vb = bufs_.at(k + "volume");
    const int nsrc = V_ - 1;
    const long long n = (long long)vb.D * vb.H * vb.W;
    rec_begin(k + "cost_volume", (double)fb.alg_bytes + (double)vb.alg_bytes + (s > 1 ? 4.0 * vb.H * vb.W : 0.0),
              (double)n * nsrc * fb.C * 12.0);
    const DminSrc dm = dmin_src(s);
    if constexpr (std::is_same<TA, __half>::value) {
      if (va_) {
        // depth hypotheses per thread: two, four at the 8-channel stage (variant 4: four at every stage); the 32 channels of
        // stage 1 split over two lanes
        const int nd = (cv_variant_ == 4 || fb.C == 8) ? 4 : 2;
        const long long thr = (long long)cdiv(vb.D, nd) * vb.H * vb.W * (fb.C == 32 ? 2 : 1);
        const unsigned grid = (unsigned)cdiv(thr, 128);
        auto go = [&](auto kern) { launch_k(kern, dim3(grid), dim3(128), p8<const __half>(fb), dm, p8<TV>(vb), slot_.index, s - 1); };
        if (fb.C == 32) { if (nd == 2) go(k_cost_volume_va16<TV, 16, 2, 2>); else go(k_cost_volume_va16<TV, 16, 2, 4>); }
        else if (fb.C == 16) { if (nd == 2) go(k_cost_volume_va16<TV, 16, 1, 2>); else go(k_cost_volume_va16<TV, 16, 1, 4>); }
        else if (fb.C == 8) go(k_cost_volume_va16<TV, 8, 1, 4>);
        else throw Error("unsupported feature channels");
        TDM_CUDA(cudaGetLastError());
        rec_end();
        return;
      }
    }
    if (fb.C == 32) k_cost_volume<TA, TV, 16, 2><<<cdiv(2 * n, 128), 128, 0, stream_.get()>>>(p8<const TA>(fb), dm, p8<TV>(vb), slot_.index, s - 1);
    else if (fb.C == 16) k_cost_volume<TA, TV, 16><<<cdiv(n, 128), 128, 0, stream_.get()>>>(p8<const TA>(fb), dm, p8<TV>(vb), slot_.index, s - 1);
    else if (fb.C == 8) k_cost_volume<TA, TV, 8><<<cdiv(n, 128), 128, 0, stream_.get()>>>(p8<const TA>(fb), dm, p8<TV>(vb), slot_.index, s - 1);
    else throw Error("unsupported feature channels");
    TDM_CUDA(cudaGetLastError());
    rec_end();
  }

  // the previous stage's depth map, from which stage s computes the lower end of its hypothesis range where it is consumed
  DminSrc dmin_src(int s) {
    DminSrc d{nullptr, 0, 0};
    if (s <= 1) return d;
    const DevBuf& pd = bufs_.at("s" + std::to_string(s - 1) + ".depth_dense");
    d.prev = (const float*)pd.p.get(); d.ph = pd.H; d.pw = pd.W;
    return d;
  }

  HypSpec hyp_spec(int s) const {
    HypSpec h;
    const float base = (dmax_ - dmin_) / (float)(depth_num_[0] - 1);
    const float ratio = s == 1 ? 1.f : (s == 2 ? 0.5f : 0.25f);
    h.adaptive = s > 1;
    h.dmin = dmin_;
    h.interval = ratio * base;
    h.D = depth_num_[s - 1];
    return h;
  }

  void filter(int s) {
    const std::string k = "s" + std::to_string(s) + ".";
    const DevBuf& d = bufs_.at(k + "depth_dense");
    const int n = d.H * d.W;
    rec_begin(k + "edge_metric+select0", 8.0 * n, 0);
    launch_k(k_edge_metric_select0, dim3(cdiv(n, 256)), dim3(256), fbuf(k + "depth_dense"), fbuf(k + "edge"), d.H, d.W, select_state_.get(), &d_params_->cutoff[s - 1]);
    rec_end();
    rec_begin(k + "percentile", 8.0 * n, 0);
    for (int pass = 1; pass <= 2; ++pass)
      launch_k(k_select_pass, dim3(std::min(cdiv(n, 256 * 8), 2 * kNumSm)), dim3(256), fbuf(k + "edge"), n, select_state_.get(), pass, fbuf("thr") + (s - 1));
    launch_count_ += 1;
    rec_end();
    rec_begin(k + "apply_mask", 20.0 * n, 0);
    launch_k(k_apply_edge_mask, dim3(cdiv(n, 256)), dim3(256), fbuf(k + "edge"), fbuf("thr") + (s - 1), fbuf(k + "depth_dense"),
                                                       fbuf(k + "confidence_dense"), fbuf(k + "depth"),
                                                       fbuf(k + "confidence"), n);
    TDM_CUDA(cudaGetLastError());
    rec_end();
  }

  // Per-call parameters are refreshed in device memory, then the (otherwise argument-invariant) kernel sequence is
  // replayed as a CUDA graph: captured on the second forward of a plan (the first one warms the tensor-map / attribute
  // caches), invalidated by free_plan() and by option changes.  k = the views FeatureNet computes: V (every slot, the
  // identity table) or, for the feature cache, the k views in slots fslots[0..k-1]; one graph per k, the slots are data.
  void forward(int k, const int* fslots, bool profiling) {
    fk_ = k;
    for (int j = 0; j <= kMaxSrc; ++j) h_feat_slot_.get()[j] = k == V_ || j >= k ? j : fslots[j];
    upload_call_params();
    if (profiling || !use_graph_) { forward_launches(profiling); return; }
    FwdGraph& fg = graphs_[k];
    if (fg.exec) { TDM_CUDA(cudaGraphLaunch(fg.exec.get(), stream_.get())); return; }
    if (!fg.warmed) { forward_launches(false); fg.warmed = true; return; }
    cudaGraph_t captured = nullptr;
    TDM_CUDA(cudaStreamBeginCapture(stream_.get(), cudaStreamCaptureModeThreadLocal));
    try {
      forward_launches(false);
    } catch (...) {
      cudaStreamEndCapture(stream_.get(), &captured);
      Graph discarded(captured);
      throw;
    }
    TDM_CUDA(cudaStreamEndCapture(stream_.get(), &captured));
    const Graph graph(captured);
    fg.exec = make_graph_exec(graph.get());
    TDM_CUDA(cudaGraphLaunch(fg.exec.get(), stream_.get()));
  }
  void drop_graph() { graphs_.clear(); }

  // feature cache: FeatureNet output `name` over the fk_ computed views -> their pool slots (c_feat_slot) of `name` over V
  void scatter_features(const std::string& name) {
    if (fk_ == V_) return;
    const DevBuf& src = bufs_.at(name + "@" + std::to_string(fk_));
    const DevBuf& dst = bufs_.at(name);
    TDM_CHECK(src.pd == 0 && dst.pd == 0 && src.C == dst.C && src.H == dst.H && src.W == dst.W, "feature scatter: shape mismatch");
    const int plane_vec = (int)((size_t)(src.H + 2) * (src.W + 2) * 8 * sizeof(TA) / 16);
    rec_begin(name + "[scatter]", 2.0 * src.alg_bytes, 0);
    launch_k(k_scatter_planes, dim3(cdiv(plane_vec, 256), (src.C / 8) * fk_), dim3(256), (const uint4*)src.p.get(), (uint4*)dst.p.get(),
             plane_vec, fk_, V_, slot_.index);
    TDM_CUDA(cudaGetLastError());
    rec_end();
  }

  // The whole graph of cva_mvsnet.py:98-184 on stream_, inputs already in d_bgr_.  FeatureNet runs over the fk_ views of
  // c_feat_slot: all V into feat1..feat3 directly, or (feature cache) fk_ < V views into the "@fk_" scratch, scattered after.
  void forward_launches(bool profiling) {
    profiling_ = profiling;
    launch_count_ = 0;
    const int H = H_, W = W_, k = fk_;
    const std::string fs = k == V_ ? "" : "@" + std::to_string(k);
    auto fb = [&fs](const char* name) { return name + fs; };
    const bool fork = fork_fpn_ && !profiling && k > 0;
    if (k > 0) {   // k == 0: a cached window of held views only, every feature is in the pool
    {
      const long long n = (long long)k * H * W;
      bool fused = false;
      if constexpr (kRawInput) {
        if (direct_conv00_) {
          fused = true;
          rec_begin("f.conv0.0[u8-direct]", 3.0 * n + 8.0 * n * sizeof(TA), 2.0 * 27 * 8 * (double)n);
          launch_k(k_conv00_u8<TA>, dim3(cdiv(W, 32), cdiv(H, 8), k), dim3(256), d_bgr_.get(), p8<TA>(bufs_.at(fb("f.c0_0"))), H, W, slot_.index);
          TDM_CUDA(cudaGetLastError());
          rec_end();
        }
      }
      if (!fused) {
        rec_begin("preprocess", 3.0 * n + 8.0 * n * sizeof(TA), 0);
        k_preprocess_bgr<TA, kRawInput><<<cdiv(n, 256), 256, 0, stream_.get()>>>(d_bgr_.get(), p8<TA>(bufs_.at(fb("f.img"))), k, H * W, slot_.index);
        TDM_CUDA(cudaGetLastError());
        rec_end();
        conv("f.conv0.0", fb("f.img"), fb("f.c0_0"), 1, 1, 1, true);
      }
    }
    conv("f.conv0.1", fb("f.c0_0"), fb("f.c3"), 1, 1, 1, true);
    conv("f.conv1.0", fb("f.c3"), fb("f.c1_0"), 1, 2, 2, true);
    conv("f.conv1.1", fb("f.c1_0"), fb("f.c1_1"), 1, 1, 1, true);
    conv("f.conv1.2", fb("f.c1_1"), fb("f.c2"), 1, 1, 1, true);
    conv("f.conv2.0", fb("f.c2"), fb("f.c2_0"), 1, 2, 2, true);
    conv("f.conv2.1", fb("f.c2_0"), fb("f.c2_1"), 1, 1, 1, true);
    conv("f.conv2.2", fb("f.c2_1"), fb("f.c1"), 1, 1, 1, true);
    // The pyramid's upper outputs (feat2, feat3) are only read by stages 2 and 3, while stage 1 needs feat1 alone and its
    // coarse U-Net levels leave most SMs idle: the FPN tail runs on a second stream, forked here and joined before the
    // stage-2 cost volume (inside the captured graph these are two parallel branches).  Not while profiling: the per-kernel
    // events assume one stream.
    struct SwapBack {   // an exception inside the branch must not leave the engine on the side stream
      Stream &a, &b; bool on;
      ~SwapBack() { if (on) std::swap(a, b); }
    } side{stream_, side_stream_, false};
    if (fork) {
      TDM_CUDA(cudaEventRecord(ev_fork_.get(), stream_.get()));
      TDM_CUDA(cudaStreamWaitEvent(side_stream_.get(), ev_fork_.get(), 0));
      std::swap(stream_, side_stream_);
      side.on = true;
    } else {
      conv("f.out1", fb("f.c1"), fb("feat1"), 1, 1, 1, false);
      scatter_features("feat1");
    }
    if (fused_fpn_ && use_tc_) {
      conv("f.skip2", fb("f.c2"), fb("f.i2"), 1, 1, 1, false, 2, fb("f.c1"), fb("f.i2b"), d_bs3_.get());
      conv("f.out2", fb("f.i2"), fb("feat2"), 1, 1, 1, false);
      conv_fpn3("f.fpn3", fb("f.i2b"), fb("f.c3"), fb("feat3"));
    } else {
      conv("f.skip2", fb("f.c2"), fb("f.i2"), 1, 1, 1, false, 2, fb("f.c1"));
      conv("f.out2", fb("f.i2"), fb("feat2"), 1, 1, 1, false);
      conv("f.skip3", fb("f.c3"), fb("f.i3"), 1, 1, 1, false, 2, fb("f.i2"));
      conv("f.out3", fb("f.i3"), fb("feat3"), 1, 1, 1, false);
    }
    scatter_features("feat2");
    scatter_features("feat3");
    if (fork) {
      TDM_CUDA(cudaEventRecord(ev_join_.get(), stream_.get()));      // stream_ is the side stream here
      std::swap(stream_, side_stream_);
      side.on = false;
      conv("f.out1", fb("f.c1"), fb("feat1"), 1, 1, 1, false);
      scatter_features("feat1");
    }
    }  // k > 0

    for (int s = 1; s <= 3; ++s) {
      const std::string k = "s" + std::to_string(s) + ".";
      const HypSpec hs = hyp_spec(s);
      const DevBuf& dd = bufs_.at(k + "depth_dense");
      if (s == 2 && fork) TDM_CUDA(cudaStreamWaitEvent(stream_.get(), ev_join_.get(), 0));
      cost_volume(s);
      const bool four = hs.D == 4;
      const int s5 = four ? 1 : 2;
      conv(k + "conv0", k + "volume", k + "c0", 1, 1, 1, true);
      conv(k + "conv1", k + "c0", k + "c1", 2, 2, 2, true);
      conv(k + "conv2", k + "c1", k + "c2", 1, 1, 1, true);
      conv(k + "conv3", k + "c2", k + "c3", 2, 2, 2, true);
      conv(k + "conv4", k + "c3", k + "c4", 1, 1, 1, true);
      conv(k + "conv5", k + "c4", k + "c5", s5, 2, 2, true);
      conv(k + "conv6", k + "c5", k + "c6", 1, 1, 1, true);
      conv(k + "conv7", k + "c6", k + "x7", s5, 2, 2, true, 1, k + "c4");
      conv(k + "conv9", k + "x7", k + "x9", 2, 2, 2, true, 1, k + "c2");
      conv(k + "conv11", k + "x9", k + "x11", 2, 2, 2, true, 1, k + "c0");
      {
        TDM_CHECK(hs.D <= 64, "depth_num > 64 unsupported");
        tail_req_ = TailReq{s, hs.D, dmin_src(s), fbuf(k + "depth_dense"), fbuf(k + "confidence_dense"), &d_params_->hyp[s - 1],
                            &d_params_->half_range[s - 1], false};
        conv(k + "prob", k + "x11", k + "logits", 1, 1, 1, false);
        tail_req_.stage = 0;
      }
      if (!tail_req_.done) {
        const int HW = dd.H * dd.W;
        rec_begin(k + "regress", 4.0 * HW * (hs.D + 3), 0);
        const DminSrc dm = dmin_src(s);
        const float* hr = &d_params_->half_range[s - 1];
        if (hs.D <= 8) launch_k(k_regress<8>, dim3(cdiv(HW, 128)), dim3(128), fbuf(k + "logits"), dm, fbuf(k + "depth_dense"), fbuf(k + "confidence_dense"), HW, dd.W, &d_params_->hyp[s - 1], hr);
        else if (hs.D <= 32) launch_k(k_regress<32>, dim3(cdiv(HW, 128)), dim3(128), fbuf(k + "logits"), dm, fbuf(k + "depth_dense"), fbuf(k + "confidence_dense"), HW, dd.W, &d_params_->hyp[s - 1], hr);
        else if (hs.D <= 64) launch_k(k_regress<64>, dim3(cdiv(HW, 128)), dim3(128), fbuf(k + "logits"), dm, fbuf(k + "depth_dense"), fbuf(k + "confidence_dense"), HW, dd.W, &d_params_->hyp[s - 1], hr);
        else throw Error("depth_num > 64 unsupported");
        TDM_CUDA(cudaGetLastError());
        rec_end();
      }
    }
    for (int s = filter_all_ ? 1 : 3; s <= 3; ++s) filter(s);
    launches_per_forward_ = launch_count_;
    profiling_ = false;
  }

  // ---------------------------------------------------------------- worker (DrMvsnetImpl::Loop, dr_mvsnet.cpp:83-93)
  void loop() {
    cudaSetDevice(device_);
    for (;;) {
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_work_.wait(lk, [this] { return stop_ || (busy_ && !started_); });
        if (stop_) return;
        started_ = true;
      }
      std::string err;
      try {
        const size_t n = (size_t)H_ * W_;
        forward(call_k_, call_slots_, false);
        if (eager_d2h_) {
          const char* names[4] = {"s3.depth", "s3.confidence", "s3.depth_dense", "s3.confidence_dense"};
          for (int k = 0; k < 4; ++k) {
            TDM_CUDA(cudaMemcpyAsync(h_out_.get() + k * n, fbuf(names[k]), n * 4, cudaMemcpyDeviceToHost, stream_.get()));
            TDM_CUDA(cudaEventRecord(ev_out_[k].get(), stream_.get()));
          }
        } else {
          TDM_CUDA(cudaEventRecord(ev_out_[0].get(), stream_.get()));   // GetResult copies back itself (page-locked caller buffers)
        }
        wait_event_politely(ev_out_[0].get());   // result "ready" as soon as the first map is home; GetResult waits per map
      } catch (const std::exception& e) {
        err = e.what();
      }
      {
        std::lock_guard<std::mutex> lk(mu_);
        worker_error_ = err;
        has_result_ = err.empty();
        if (!err.empty()) cache_valid_ = false;   // the pool may not hold the features of the ids it lists
        busy_ = false;
        started_ = false;
      }
      cv_done_.notify_all();
    }
  }

  // Keyframe handoff.  Invariant: the handoff buffers are written only by this fill, enqueued on stream_ behind every release
  // event recorded since the previous fill, and freed only after those events have completed; so a consumer's reads, which
  // wait for ev_ho_ready_ and end before their release event, always see exactly the result the last GetResult returned,
  // however far the next window's upload and forward (which overwrite d_bgr_ and s3.depth) have got.  The image is copied
  // from the reference view's pool slot, which is enqueued on stream_ before any later upload into that slot.
  void fill_handoff() {
    const size_t n = (size_t)H_ * W_;
    ho_valid_ = false;
    if (ho_H_ != H_ || ho_W_ != W_) {
      for (int i = 0; i < n_ho_release_; ++i) TDM_CUDA(cudaEventSynchronize(ev_ho_release_[i].get()));
      n_ho_release_ = 0;
      d_ho_depth_.reset(); d_ho_bgr_.reset(); ho_H_ = ho_W_ = 0;
      d_ho_depth_ = make_dev<float>(n * 4);
      d_ho_bgr_ = make_dev<unsigned char>(n * 3);
      ho_H_ = H_; ho_W_ = W_;
    }
    if (!ev_ho_ready_) ev_ho_ready_ = make_event(cudaEventDisableTiming);
    for (int i = 0; i < n_ho_release_; ++i) TDM_CUDA(cudaStreamWaitEvent(stream_.get(), ev_ho_release_[i].get(), 0));
    n_ho_release_ = 0;
    TDM_CUDA(cudaMemcpyAsync(d_ho_depth_.get(), fbuf("s3.depth"), n * 4, cudaMemcpyDeviceToDevice, stream_.get()));
    TDM_CUDA(cudaMemcpyAsync(d_ho_bgr_.get(), d_bgr_.get() + (size_t)view_slot_[0] * n * 3, n * 3, cudaMemcpyDeviceToDevice, stream_.get()));
    TDM_CUDA(cudaEventRecord(ev_ho_ready_.get(), stream_.get()));
    std::memcpy(ho_c2w_, c2w_[0], sizeof(ho_c2w_));
    ho_valid_ = true;
  }
  bool record_release(void* stream) {
    if (cudaSetDevice(device_) != cudaSuccess) return false;
    if (n_ho_release_ == (int)ev_ho_release_.size()) {
      cudaEvent_t e = nullptr;
      if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return false;
      ev_ho_release_.emplace_back(e);
    }
    if (cudaEventRecord(ev_ho_release_[n_ho_release_].get(), (cudaStream_t)stream) != cudaSuccess) return false;
    ++n_ho_release_;
    return true;
  }

  static void check_window(int H, int W, int V, int ref_index) {
    TDM_CHECK(V >= 2 && V <= kMaxSrc + 1, "view_num out of range");
    TDM_CHECK(ref_index >= 0 && ref_index < V, "ref_index out of range");
    TDM_CHECK(H % 32 == 0 && W % 32 == 0, "height and width must be multiples of 32 (three stride-2 levels at 1/4 resolution)");
  }
  // the caller's view at position vi of the reference-first order (dr_mvsnet.cpp:190-197), and back
  static int window_view(int vi, int ref_index) { return vi == 0 ? ref_index : (vi <= ref_index ? vi - 1 : vi); }
  static int window_index(int view, int ref_index) { return view == ref_index ? 0 : (view < ref_index ? view + 1 : view); }

  void wait_idle_for_call(std::unique_lock<std::mutex>& lk) {
    cv_done_.wait(lk, [this] { return !busy_; });
    if (has_result_) throw Error("CallAsync while a result is un-fetched (dr_mvsnet.cpp:315-318)");
    if (!worker_error_.empty()) { std::string e = worker_error_; worker_error_.clear(); throw Error(e); }
  }

  // srcs[j] (H*W*3 u8, owned by the caller only during this call) -> slot slots[j] of d_bgr_
  void upload_images(int n, const int* slots, const unsigned char* const* srcs) {
    const size_t img = (size_t)H_ * W_ * 3;
    if (all_page_locked((const void* const*)srcs, n)) {
      // Page-locked caller images (cudaHostAlloc / cudaHostRegister): DMA straight from them - no staging copy, no copy
      // threads.  The caller owns them only during this call, so the call returns once the seven DMAs have landed
      // (6.45 MB over PCIe gen5: ~0.13 ms, less than the staging memcpy it replaces).
      for (int j = 0; j < n; ++j)
        TDM_CUDA(cudaMemcpyAsync(d_bgr_.get() + (size_t)slots[j] * img, srcs[j], img, cudaMemcpyHostToDevice, stream_.get()));
      TDM_CUDA(cudaEventRecord(ev_in_.get(), stream_.get()));
      TDM_CUDA(cudaEventSynchronize(ev_in_.get()));
    } else {
      // Pageable caller memory: staged through pinned memory.  The staging copy of view v+1 overlaps the DMA of view v (the
      // worker is idle here, so this thread may enqueue on the engine's stream); each view is split into slices copied by the
      // process-wide pool; a slice's H2D is enqueued by whichever thread finished copying it (CUDA stream calls are
      // thread-safe; the order of the DMAs inside the stream does not matter, the forward is enqueued behind all of them).
      std::vector<CopyPool::Job> jobs;
      constexpr int kSlices = 2;
      std::mutex err_mu;
      cudaError_t first_err = cudaSuccess;
      for (int j = 0; j < n; ++j) {
        for (int sl = 0; sl < kSlices; ++sl) {
          const size_t b0 = img * sl / kSlices, b1 = img * (sl + 1) / kSlices;
          unsigned char* hp = h_bgr_.get() + (size_t)slots[j] * img + b0;
          unsigned char* dp = d_bgr_.get() + (size_t)slots[j] * img + b0;
          jobs.push_back({hp, srcs[j] + b0, b1 - b0, [this, hp, dp, b0, b1, &err_mu, &first_err] {
                            cudaSetDevice(device_);   // pool threads start on device 0
                            const cudaError_t e = cudaMemcpyAsync(dp, hp, b1 - b0, cudaMemcpyHostToDevice, stream_.get());
                            if (e != cudaSuccess) { std::lock_guard<std::mutex> lk(err_mu); first_err = e; }
                          }});
        }
      }
      CopyPool::shared().run(jobs);
      TDM_CUDA(first_err);
    }
  }

  // hands the window to the worker: FeatureNet on the k views in slots new_slots[0..k-1] (k == V: every slot)
  void submit(int k, int ref_index, float* const* c2ws, const float* K3x3x3, float dmin, float dmax, float discard,
              std::unique_lock<std::mutex>& lk, const int* new_slots = nullptr) {
    for (int vi = 0; vi < V_; ++vi) std::memcpy(c2w_[vi], c2ws[window_view(vi, ref_index)], 16 * sizeof(float));
    std::memcpy(K_, K3x3x3, 27 * sizeof(float));
    dmin_ = dmin; dmax_ = dmax; discard_ = discard;
    call_k_ = k;
    for (int j = 0; j < k; ++j) call_slots_[j] = new_slots ? new_slots[j] : j;
    n_computed_ = k;
    last_ref_index_ = ref_index;
    busy_ = true;
    have_inputs_ = true;
    lk.unlock();
    cv_work_.notify_all();
  }

  bool slots_identity() const {
    for (int v = 0; v < V_; ++v)
      if (view_slot_[v] != v) return false;
    return true;
  }

  // true when every non-null pointer is page-locked host memory the device can DMA from / into directly
  static bool all_page_locked(const void* const* ptrs, int n) {
    for (int i = 0; i < n; ++i) {
      if (!ptrs[i]) return false;
      cudaPointerAttributes at{};
      if (cudaPointerGetAttributes(&at, ptrs[i]) != cudaSuccess) { cudaGetLastError(); return false; }
      if (at.type != cudaMemoryTypeHost) return false;
    }
    return true;
  }
  // cudaEventSynchronize spins a core for the whole forward; with several handles per GPU and several ranks per host those
  // spinning workers compete with the copy threads and the callers.  Poll with short sleeps instead (<= 20 us late).
  static void wait_event_politely(cudaEvent_t ev) {
    for (;;) {
      const cudaError_t e = cudaEventQuery(ev);
      if (e == cudaSuccess) return;
      if (e != cudaErrorNotReady) TDM_CUDA(e);
      std::this_thread::sleep_for(std::chrono::microseconds(20));
    }
  }

  struct Gate { int C = 0; float w1[64]; float b1 = 0, w2 = 0, b2 = 0; };
  // mixed16: the cost volume is fp16 too, stored x 2^-5 (values reach ~1e4 and fp16 ends at 65504; bf16 has the range but only 8
  // significant bits, which a CPU study found to cost about 1 % of mask IoU on its own)
  static constexpr float kVolScale = (std::is_same<TA, __half>::value && std::is_same<TV, __half>::value) ? 0.03125f : 1.f;
  static constexpr int kNumSm = 132;   // H100 SXM (sm_90a only build)
  static constexpr bool kRawInput = sizeof(TA) == 2;   // 16-bit engines: exact u8/256 input, 256/255 folded into f.conv0.0

  int device_ = 0;
  Stream stream_;
  WeightFile wf_;
  int depth_num_[3];
  bool va_ = false;
  std::map<std::string, DevConv> convs_;
  Gate gates_[3];
  std::map<std::string, DevBuf> bufs_;
  DevPtr<SelectState> select_state_;
  // softmax / soft-argmin / confidence in the epilogue of the tensor-core prob convolution (set_option("fused_regress", 1)):
  // bit-identical to k_regress and three launches fewer, but the consumer threads of a CTA finish their pixels after the last
  // plane with nothing left to overlap, where the stand-alone kernel spreads the same work over 2048 threads per SM. Off.
  bool fused_regress_ = false;
  // the stages' conv0 and prob on the input-stationary kernel (conv_tc_is.cuh); 0: the output-stationary k_conv_tc.
  // Measured on an H100 80GB HBM3 at 400 W (DESIGN.md section 5): the six launches 0.81 -> 0.58 ms, bench value +9 %
  bool use_is_ = true;
  struct TailReq { int stage; int D; DminSrc dsrc; float* depth; float* conf; const HypSpec* hyp; const float* half_range; bool done; };
  TailReq tail_req_{};
  int pdl_min_smem_kb_ = 120;
  int V_ = 0, H_ = 0, W_ = 0;
  HostPtr<unsigned char> h_bgr_;
  DevPtr<unsigned char> d_bgr_;
  HostPtr<float> h_out_;
  Event ev_out_[4];
  Event ev_in_;
  bool eager_d2h_ = true;   // worker copies the four maps into pinned staging right behind the forward (pageable callers);
                            // 0: GetResult copies back itself - for callers that pass page-locked result buffers
  float c2w_[kMaxSrc + 1][16];
  // keyframe handoff (fill_handoff / read_handoff): the last fetched result, kept until the next GetResult
  DevPtr<float> d_ho_depth_;
  DevPtr<unsigned char> d_ho_bgr_;
  float ho_c2w_[16];
  int ho_H_ = 0, ho_W_ = 0;
  bool ho_valid_ = false;
  Event ev_ho_ready_;
  std::vector<Event> ev_ho_release_;   // pool; the first n_ho_release_ were recorded by consumers since the last fill
  int n_ho_release_ = 0;
  float K_[27];
  float dmin_ = 0, dmax_ = 0, discard_ = 0;
  DevPtr<float> d_bs3_;
  HostPtr<CallParams> h_params_;   // pinned
  DevPtr<CallParams> d_params_;
  HostPtr<int> h_feat_slot_;       // pinned [kMaxSrc + 1]: the table c_feat_slot[slot_] the next forward uses
  // feature cache (call_async_ids): slot s of d_bgr_ / feat1..3 holds the view with id slot_id_[s] when cache_valid_; view vi of
  // the last window (reference first) is in slot view_slot_[vi] (the identity after a plain call_async)
  long long slot_id_[kMaxSrc + 1] = {};
  int view_slot_[kMaxSrc + 1];
  bool cache_valid_ = false;
  int last_ref_index_ = 0;
  int n_computed_ = 0;                                 // views FeatureNet computed for the last call
  int call_k_ = 0, call_slots_[kMaxSrc + 1] = {};      // the submitted window's FeatureNet views, for the worker
  int fk_ = 0;                                         // views FeatureNet computes in the forward being enqueued / last enqueued
  struct FwdGraph { GraphExec exec; bool warmed = false; };
  std::map<int, FwdGraph> graphs_;   // one captured forward per FeatureNet view count
  // 4: four depth hypotheses per thread of k_cost_volume_va16 at every stage.  Measured faster than the default 3 on an H100
  // 80GB HBM3 at 700 W (DESIGN.md, "MVSNet variants removed"); off until a change of its own turns it on
  int cv_variant_ = 3;
  // Programmatic dependent launch of the tensor-core kernels: the trigger sits after griddepcontrol.wait (a trigger before it
  // lets the whole chain of later kernels become resident early), and pdl_min_smem_kb_ = 120 keeps one tensor-core CTA per SM.
  bool use_graph_ = true;
  int use_pdl_ = 1;   // 2: the FMA-pipe kernels (cost volume, soft-argmin, edge filter ...) are launched with the attribute as well
  EngineSlot slot_;
  int tc_smem_kb_ = 225;   // shared-memory budget of the tile planner (<= 113 lets two CTAs share an SM)
  bool fused_fpn_ = false;
  bool prob_direct_ = false;  // `prob` (8 -> 1 channels) on the FMA pipes (k_prob_direct) instead of the tensor-core tile; an A/B option and an independent check
  bool have_prob_w_ = false;
  ProbWeights prob_w_[3] = {};
  bool direct_conv00_ = true; // 16-bit engines: pre-processing + conv0.0 fused on the FMA pipes (k_conv00_u8); 0 = preprocess + tensor-core conv
  bool fork_fpn_ = true;      // FPN tail on a second stream / graph branch (A/B: set_option("fork_fpn", 0))
  Stream side_stream_;
  Event ev_fork_, ev_join_;
  bool filter_all_ = false, keep_ = true, use_tc_ = (sizeof(TA) == 2);  // tensor-core convs are the default on 16-bit engines
  bool debug_poison_ = false;  // set_option("debug_poison", 1): activation interiors start as NaN (alloc), for the layer tests
  bool profiling_ = false;
  int launch_count_ = 0, launches_per_forward_ = 0;
  std::vector<LaunchRec> recs_;

  std::thread worker_;
  std::mutex mu_;
  std::condition_variable cv_work_, cv_done_;
  bool busy_ = false, started_ = false, stop_ = false, has_result_ = false, have_inputs_ = false;
  std::string worker_error_;
};

template <> template <> float MvsnetEngine<float, float>::from_host<float>(float v) { return v; }
template <> template <> __half MvsnetEngine<__half, __half>::from_host<__half>(float v) { return __float2half_rn(v); }
template <> template <> __nv_bfloat16 MvsnetEngine<__nv_bfloat16, __nv_bfloat16>::from_host<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

MvsnetIface* make_mvsnet(const std::string& path, int precision, int device) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0)
    throw Error("tandem_b200: no CUDA device visible - this library has no CPU fallback");
  if (precision == 0) return new MvsnetEngine<float, float>(path, device);
  if (precision == 1) return new MvsnetEngine<__half, __half>(path, device);               // mixed16 (fp16 volume x 2^-5)
  if (precision == 2) return new MvsnetEngine<__nv_bfloat16, __nv_bfloat16>(path, device);  // pure bf16
  throw Error("unknown precision");
}


// host-only: the plane-sweep homography of one source view exactly as fill_cv_params computes it (module.py:795-808)
void debug_homography(const float* K3x3, const float* c2w_ref, const float* c2w_src, float* rot9, float* trans3) {
  double Pr[16], Pri[16], Ps[16], M[16];
  world_to_pixel(K3x3, c2w_ref, Pr);
  if (!mat4_inv(Pr, Pri)) throw Error("reference projection is singular");
  world_to_pixel(K3x3, c2w_src, Ps);
  mat4_mul(Ps, Pri, M);
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) rot9[i * 3 + j] = (float)M[i * 4 + j];
    trans3[i] = (float)M[i * 4 + 3];
  }
}

// host-only view of the tensor-core tile planner (no GPU involved; used by the CPU test-suite): the first n (<= 13) of {S, R,
// TW, P, DR, nch, slot_pos, tiles_w, tiles_h, tiles_d, grid, smem_bytes, nwg}; nwg is the consumer-warpgroup count the plan
// was made for, which every launch checks against its kernel's NWG
void debug_conv_plan(int cin, int npad, int kd, int D, int H, int W, int pd, int mode, int smem_kb, long long* out, int n) {
  // mode + 100 = the same mode with tiles that span all D planes (the prob layer with the soft-argmin tail);
  // mode 200 = the input-stationary planner (make_plan_is) with npad = columns per kd block (kd and pd are implied: 3, 1),
  // mode 300 = the same with tiles that span all D planes,
  // mode 400 = the stride-2 planner (make_plan_s2): D, H, W are the OUTPUT dims, pd carries the kernel size (3 or 5)
  if (mode == 400) {
    TDM_CHECK((kd == 1 || kd == 3) && (pd == 3 || pd == 5), "mode 400: kd must be 1 or 3 and pd the kernel size 3 or 5");
    const tc::PlanS2 p = tc::make_plan_s2(cin, npad, kd, pd, D, H, W, (size_t)smem_kb * 1024);
    const tc::GeomS2& g = p.g;
    const long long v[13] = {g.S, g.R, g.TW, g.P, g.DR, g.nch, g.slot_pos, g.tiles_w, g.tiles_h, g.tiles_d, p.grid, (long long)p.smem, p.nwg};
    for (int i = 0; i < n; ++i) out[i] = v[i];
    return;
  }
  const tc::Plan p = mode >= 200 ? tc::make_plan_is(cin, npad, D, H, W, (size_t)smem_kb * 1024, mode == 300)
                                 : tc::make_plan(cin, npad, kd, D, H, W, pd, mode % 100, (size_t)smem_kb * 1024, mode >= 100);
  const tc::Geom& g = p.g;
  const long long v[13] = {g.S, g.R, g.TW, g.P, g.DR, g.nch, g.slot_pos, g.tiles_w, g.tiles_h, g.tiles_d, p.grid, (long long)p.smem, p.nwg};
  for (int i = 0; i < n; ++i) out[i] = v[i];
}

}  // namespace tdm
