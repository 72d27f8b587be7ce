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
#include "conv_tc_s2.cuh"
#include "cost_volume_tma.cuh"
#include "weights.h"

namespace tdm {

namespace {

std::mutex g_slot_mu;
bool g_slot_used[kMaxEngines] = {};
int acquire_slot() {
  std::lock_guard<std::mutex> lk(g_slot_mu);
  for (int i = 0; i < kMaxEngines; ++i)
    if (!g_slot_used[i]) { g_slot_used[i] = true; return i; }
  throw Error("too many DrMvsnet instances alive in this process (max 8)");
}
void release_slot(int i) {
  std::lock_guard<std::mutex> lk(g_slot_mu);
  if (i >= 0 && i < kMaxEngines) g_slot_used[i] = false;
}

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
  void* p = nullptr;
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
  float* w = nullptr;
  float* bias = nullptr;
  // tensor-core path (conv_tc.cuh): weights pre-arranged as the canonical K-major B image in the input's 16-bit type
  void* bimg = nullptr;
  int npad = 0;
  bool tc_ok = false;
  bool tc_deconv = false;  // transposed conv evaluated as a GEMM over the input grid (N = 8 parity classes x cout)
  int nsplit = 1;          // N slices (blockIdx.y) for the 64-channel layers
  bool hilo = false;       // weights carried as hi + lo 16-bit halves (N doubled), see conv_tc.cuh
  bool tc_up2 = false;     // MODE 3: conv3x3 of a nearest-x2 up-sampled map on the coarse grid (fused FPN tail)
  bool tc_s2 = false;      // stride-2 conv on the tensor-map (strided TMA) kernel, conv_tc_s2.cuh
  void* bimg_s2 = nullptr;
  int npad_s2 = 0, nsplit_s2 = 1;
};

struct LaunchRec {
  std::string name;
  double bytes = 0, flops = 0;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
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
    TDM_CUDA(cudaStreamCreateWithPriority(&stream_, cudaStreamNonBlocking, lo));
    TDM_CUDA(cudaStreamCreateWithPriority(&side_stream_, cudaStreamNonBlocking, lo));
    TDM_CUDA(cudaEventCreateWithFlags(&ev_fork_, cudaEventDisableTiming));
    TDM_CUDA(cudaEventCreateWithFlags(&ev_join_, cudaEventDisableTiming));
    slot_ = acquire_slot();
    for (auto& e : ev_out_) TDM_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    TDM_CUDA(cudaEventCreateWithFlags(&ev_in_, cudaEventDisableTiming));
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
    free_plan();
    for (auto& kv : convs_) { cudaFree(kv.second.w); cudaFree(kv.second.bias); cudaFree(kv.second.bimg); cudaFree(kv.second.bimg_s2); }
    if (d_cv_stats_) {
      unsigned st[2] = {0, 0};
      if (std::getenv("TDM_DEBUG_PLAN") && cudaMemcpy(st, d_cv_stats_, sizeof(st), cudaMemcpyDeviceToHost) == cudaSuccess)
        fprintf(stderr, "[cv_tma] (CTA, view) pairs staged by TMA: %u, fallen back to global gathers: %u\n", st[0], st[1]);
      cudaFree(d_cv_stats_);
    }
    if (select_state_) cudaFree(select_state_);
    if (select2_) cudaFree(select2_);
    release_slot(slot_);
    if (d_bs3_) cudaFree(d_bs3_);
    if (h_params_) cudaFreeHost(h_params_);
    if (d_params_) cudaFree(d_params_);
    for (auto& e : ev_out_) if (e) cudaEventDestroy(e);
    if (ev_in_) cudaEventDestroy(ev_in_);
    if (ev_fork_) cudaEventDestroy(ev_fork_);
    if (ev_join_) cudaEventDestroy(ev_join_);
    if (side_stream_) cudaStreamDestroy(side_stream_);
    if (stream_) cudaStreamDestroy(stream_);
  }

  void set_option(const std::string& key, int value) override {
    {
      // the worker may be replaying the captured graph: wait for it before the graph is destroyed / options change
      std::unique_lock<std::mutex> lk(mu_);
      cv_done_.wait(lk, [this] { return !busy_; });
    }
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaStreamSynchronize(stream_));
    if (key == "eager_d2h") { eager_d2h_ = value != 0; return; }   // not part of the captured launch sequence
    drop_graph();
    if (key == "filter_all_stages") filter_all_ = value != 0;
    else if (key == "use_graph") use_graph_ = value != 0;
    else if (key == "use_pdl") { TDM_CHECK(value >= 0 && value <= 2, "use_pdl: 0 off, 1 tensor-core kernels, 2 every kernel of the forward"); use_pdl_ = value; }
    else if (key == "pdl_min_smem_kb") { TDM_CHECK(value >= 0 && value <= 225, "pdl_min_smem_kb out of range"); pdl_min_smem_kb_ = value; }
    else if (key == "cv_variant") { TDM_CHECK(value >= 0 && value <= 5, "cv_variant out of range"); cv_variant_ = value; }
    else if (key == "tc_smem_kb") { TDM_CHECK(value >= 48 && value <= 225, "tc_smem_kb out of range"); tc_smem_kb_ = value; tc_cache_.clear(); s2_cache_.clear(); }
    else if (key.rfind("depth_num_stage", 0) == 0 && key.size() == 16 && key[15] >= '1' && key[15] <= '3') {
      // override the checkpoint's MODEL.DEPTH_NUM for one stage (BASELINE.json configs[0] uses 32 stage-1 hypotheses;
      // CostRegNet is fully convolutional in D).  Forces a re-plan.
      TDM_CHECK(value == 4 || (value > 0 && value % 8 == 0 && value <= 64), "depth_num must be 4 or a multiple of 8 up to 64");
      depth_num_[key[15] - '1'] = value;
      // the old plan's buffers are sized for the old D: drop them together with the resident window, so that neither
      // run_resident / profile nor a stale logits buffer can be used before the next CallAsync re-plans
      free_plan();
      V_ = H_ = W_ = 0;
      have_inputs_ = false;
    }
    else if (key == "keep_intermediates") keep_ = value != 0;
    else if (key == "use_tc") use_tc_ = value != 0;
    else if (key == "fork_fpn") fork_fpn_ = value != 0;
    else if (key == "prob_direct") prob_direct_ = value != 0;
    else if (key == "direct_conv00") direct_conv00_ = value != 0;
    else if (key == "fused_select") fused_select_ = value != 0;
    else if (key == "fused_regress") fused_regress_ = value != 0;
    else if (key == "inline_dmin") inline_dmin_ = value != 0;
    else throw Error("unknown option " + key);
  }

  // "Blocking for last input. Non-blocking for this input." (dr_mvsnet.h:42)
  void call_async(int H, int W, int V, int ref_index, unsigned char* const* bgrs, const float* K3x3x3,
                  float* const* c2ws, float dmin, float dmax, float discard) override {
    TDM_CHECK(V >= 2 && V <= kMaxSrc + 1, "view_num out of range");
    TDM_CHECK(ref_index >= 0 && ref_index < V, "ref_index out of range");
    TDM_CHECK(H % 32 == 0 && W % 32 == 0, "height and width must be multiples of 32 (three stride-2 levels at 1/4 resolution)");
    for (int i = 0; i < V - 1; ++i)
      for (int j = i + 1; j < V; ++j)
        if (bgrs[i] == bgrs[j] || c2ws[i] == c2ws[j])
          throw Error("CallAsync: the same data passed for two views (dr_mvsnet.cpp:153-160)");
    std::unique_lock<std::mutex> lk(mu_);
    cv_done_.wait(lk, [this] { return !busy_; });
    if (has_result_) throw Error("CallAsync while a result is un-fetched (dr_mvsnet.cpp:315-318)");
    if (!worker_error_.empty()) { std::string e = worker_error_; worker_error_.clear(); throw Error(e); }
    TDM_CUDA(cudaSetDevice(device_));
    ensure_plan(V, H, W);
    // copy inputs (owned by the caller only during this call); reference view first (dr_mvsnet.cpp:190-197)
    const size_t img = (size_t)H * W * 3;
    for (int vi = 0; vi < V; ++vi) {
      const int view = vi == 0 ? ref_index : (vi <= ref_index ? vi - 1 : vi);
      std::memcpy(c2w_[vi], c2ws[view], 16 * sizeof(float));
    }
    if (all_page_locked((const void* const*)bgrs, V)) {
      // Page-locked caller images (cudaHostAlloc / cudaHostRegister): DMA straight from them - no staging copy, no copy
      // threads.  The caller owns them only during this call, so the call returns once the seven DMAs have landed
      // (6.45 MB over PCIe gen5: ~0.13 ms, less than the staging memcpy it replaces).
      for (int vi = 0; vi < V; ++vi) {
        const int view = vi == 0 ? ref_index : (vi <= ref_index ? vi - 1 : vi);
        TDM_CUDA(cudaMemcpyAsync(d_bgr_ + (size_t)vi * img, bgrs[view], img, cudaMemcpyHostToDevice, stream_));
      }
      TDM_CUDA(cudaEventRecord(ev_in_, stream_));
      TDM_CUDA(cudaEventSynchronize(ev_in_));
    } else {
      // Pageable caller memory: staged through pinned memory.  The staging copy of view v+1 overlaps the DMA of view v (the
      // worker is idle here, so this thread may enqueue on the engine's stream); each view is split into slices copied by the
      // process-wide pool; a slice's H2D is enqueued by whichever thread finished copying it (CUDA stream calls are
      // thread-safe; the order of the DMAs inside the stream does not matter, the forward is enqueued behind all of them).
      std::vector<CopyPool::Job> jobs;
      constexpr int kSlices = 2;
      std::mutex err_mu;
      cudaError_t first_err = cudaSuccess;
      for (int vi = 0; vi < V; ++vi) {
        const int view = vi == 0 ? ref_index : (vi <= ref_index ? vi - 1 : vi);
        for (int sl = 0; sl < kSlices; ++sl) {
          const size_t b0 = img * sl / kSlices, b1 = img * (sl + 1) / kSlices;
          unsigned char* hp = h_bgr_ + (size_t)vi * img + b0;
          unsigned char* dp = d_bgr_ + (size_t)vi * img + b0;
          jobs.push_back({hp, bgrs[view] + b0, b1 - b0, [this, hp, dp, b0, b1, &err_mu, &first_err] {
                            cudaSetDevice(device_);   // pool threads start on device 0
                            const cudaError_t e = cudaMemcpyAsync(dp, hp, b1 - b0, cudaMemcpyHostToDevice, stream_);
                            if (e != cudaSuccess) { std::lock_guard<std::mutex> lk(err_mu); first_err = e; }
                          }});
        }
      }
      CopyPool::shared().run(jobs);
      TDM_CUDA(first_err);
    }
    std::memcpy(K_, K3x3x3, 27 * sizeof(float));
    dmin_ = dmin; dmax_ = dmax; discard_ = discard;
    busy_ = true;
    have_inputs_ = true;
    lk.unlock();
    cv_work_.notify_all();
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
        TDM_CUDA(cudaMemcpyAsync(dst[k], fbuf(names[k]), n * 4, cudaMemcpyDeviceToHost, stream_));
      TDM_CUDA(cudaStreamSynchronize(stream_));
    } else {
      if (!eager_d2h_) {   // the worker did not copy back: do it now
        for (int k = 0; k < 4; ++k) {
          TDM_CUDA(cudaMemcpyAsync(h_out_ + k * n, fbuf(names[k]), n * 4, cudaMemcpyDeviceToHost, stream_));
          TDM_CUDA(cudaEventRecord(ev_out_[k], stream_));
        }
      }
      // each map is copied to caller memory by the pool as soon as its D2H has landed
      std::vector<CopyPool::Job> jobs;
      TDM_CUDA(cudaEventSynchronize(ev_out_[3]));   // 4.9 MB over PCIe: ~0.1 ms; simpler than per-map hand-off
      constexpr int kSlices = 2;
      for (int k = 0; k < 4; ++k)
        if (dst[k])
          for (int sl = 0; sl < kSlices; ++sl) {
            const size_t e0 = n * sl / kSlices, e1 = n * (sl + 1) / kSlices;
            jobs.push_back({dst[k] + e0, h_out_ + k * n + e0, (e1 - e0) * 4, nullptr});
          }
      CopyPool::shared().run(jobs);
    }
    has_result_ = false;
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
    TDM_CUDA(cudaMemcpy(out, it->second.p, n * 4, cudaMemcpyDeviceToHost));
  }

  long long debug_tensor(const std::string& name, float* out, size_t cap, int* dims4) override {
    wait();
    TDM_CUDA(cudaSetDevice(device_));
    auto it = bufs_.find(name);
    if (it == bufs_.end()) throw Error("no such tensor: " + name);
    const DevBuf& b = it->second;
    const long long npos = (long long)b.D * b.H * b.W;
    const long long n = npos * b.C;
    if (dims4) { dims4[0] = b.C; dims4[1] = b.D; dims4[2] = b.H; dims4[3] = b.W; }
    if (!out) return n;
    TDM_CHECK((long long)cap >= n, "debug_tensor: capacity too small");
    if (b.f32) {
      TDM_CUDA(cudaMemcpy(out, b.p, n * 4, cudaMemcpyDeviceToHost));  // C==1 planar already
      return n;
    }
    float* tmp = nullptr;
    TDM_CUDA(cudaMalloc(&tmp, n * 4));
    if (b.kind == 2) k_p8_to_planar_f32<TV><<<cdiv(n, 256), 256, 0, stream_>>>(p8<const TV>(b), tmp);
    else k_p8_to_planar_f32<TA><<<cdiv(n, 256), 256, 0, stream_>>>(p8<const TA>(b), tmp);
    TDM_CUDA(cudaGetLastError());
    TDM_CUDA(cudaMemcpyAsync(out, tmp, n * 4, cudaMemcpyDeviceToHost, stream_));
    TDM_CUDA(cudaStreamSynchronize(stream_));
    cudaFree(tmp);
    if (b.kind == 2 && kVolScale != 1.f)
      for (long long i = 0; i < n; ++i) out[i] *= 1.f / kVolScale;   // report the volume in its own units
    return n;
  }

  void run_resident(int iters, float* ms_total, int* launches) override {
    wait();
    TDM_CHECK(have_inputs_, "run_resident: no window submitted yet");
    TDM_CUDA(cudaSetDevice(device_));
    cudaEvent_t e0, e1;
    TDM_CUDA(cudaEventCreate(&e0));
    TDM_CUDA(cudaEventCreate(&e1));
    TDM_CUDA(cudaEventRecord(e0, stream_));
    for (int i = 0; i < iters; ++i) forward(false);
    TDM_CUDA(cudaEventRecord(e1, stream_));
    TDM_CUDA(cudaEventSynchronize(e1));
    TDM_CUDA(cudaEventElapsedTime(ms_total, e0, e1));
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (launches) *launches = launches_per_forward_;
  }

  void* resident_stream() override { return (void*)stream_; }
  int resident_device() const override { return device_; }
  int resident_launch(int iters) override {
    wait();
    TDM_CHECK(have_inputs_, "run_resident: no window submitted yet");
    TDM_CUDA(cudaSetDevice(device_));
    for (int i = 0; i < iters; ++i) forward(false);
    return launches_per_forward_;
  }

  std::string profile() override {
    wait();
    TDM_CHECK(have_inputs_, "profile: no window submitted yet");
    TDM_CUDA(cudaSetDevice(device_));
    forward(false);  // warm
    recs_.clear();
    forward(true);
    TDM_CUDA(cudaStreamSynchronize(stream_));
    std::ostringstream os;
    for (auto& r : recs_) {
      cudaEventElapsedTime(&r.ms, r.e0, r.e1);
      cudaEventDestroy(r.e0);
      cudaEventDestroy(r.e1);
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
    TDM_CUDA(cudaMalloc(&dc.w, fc.w.size() * 4));
    TDM_CUDA(cudaMemcpy(dc.w, fc.w.data(), fc.w.size() * 4, cudaMemcpyHostToDevice));
    if (!fc.bias.empty()) {
      TDM_CUDA(cudaMalloc(&dc.bias, fc.bias.size() * 4));
      TDM_CUDA(cudaMemcpy(dc.bias, fc.bias.data(), fc.bias.size() * 4, cudaMemcpyHostToDevice));
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
        if (vol_in) upload_bimg<TV>(fc, dc); else upload_bimg<TA>(fc, dc);
      }
      const bool deconv_ok = fc.transposed && fc.kd == 3 && fc.kh == 3 && fc.kw == 3 &&
                             ((fc.cin == 16 && fc.cout == 8) || (fc.cin == 32 && fc.cout == 16) || (fc.cin == 64 && fc.cout == 32));
      if (deconv_ok) {
        dc.nsplit = fc.cin == 64 ? 4 : 1;
        dc.npad = 8 * fc.cout / dc.nsplit;
        dc.tc_ok = dc.tc_deconv = true;
        std::vector<TA> img;
        auto cvt = [](float v) -> TA { return from_host<TA>(v); };
        if (fc.cin == 16) tc::build_b_image_deconv<TA, 16>(fc.w.data(), fc.cin, fc.cout, img, +cvt);
        else if (fc.cin == 32) tc::build_b_image_deconv<TA, 32>(fc.w.data(), fc.cin, fc.cout, img, +cvt);
        else tc::build_b_image_deconv<TA, 64>(fc.w.data(), fc.cin, fc.cout, img, +cvt, dc.nsplit);
        TDM_CUDA(cudaMalloc(&dc.bimg, img.size() * sizeof(TA)));
        TDM_CUDA(cudaMemcpy(dc.bimg, img.data(), img.size() * sizeof(TA), cudaMemcpyHostToDevice));
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
        auto cvt = [](float v) -> TA { return from_host<TA>(v); };
        tc::build_b_image_s2<TA>(fc.w.data(), fc.cin, fc.cout, dc.npad_s2, fc.kd, fc.kh, taps, img, +cvt, dc.nsplit_s2);
        TDM_CUDA(cudaMalloc(&dc.bimg_s2, img.size() * sizeof(TA)));
        TDM_CUDA(cudaMemcpy(dc.bimg_s2, img.data(), img.size() * sizeof(TA), cudaMemcpyHostToDevice));
      }
    }
    convs_[key] = dc;
  }

  // Algebraic fusion of the FPN tail for stage 3 (module.py:522-530): feat3 = out3(up2(i2) + skip3(c3) + b3) is linear,
  //   feat3 = [conv3x3(W3) o up2](i2 + b3)  +  conv3x3(W3 . Ws3)(c3)
  // (adding b3 to i2 BEFORE the zero-padded up-sampling reproduces the bias' border behaviour exactly).  The first term
  // is evaluated on the coarse grid (4 output parity classes, the 3x3 fine taps pre-summed onto the 3x3 coarse
  // neighbourhood), the second is an 8->8 conv on c3 that adds the first as its residual.  The 138 MB tensor i3 is never
  // formed.
  void build_fused_fpn() {
    const std::string f = "feature_net.";
    const FoldedConv w3 = fold_conv(wf_, f + "out.stage3.weight", "", "", false);                        // [9][32][8]
    const FoldedConv ws = fold_conv(wf_, f + "skip.stage3.weight", f + "skip.stage3.bias", "", false);   // [1][8][32]
    FoldedConv a;   // coarse-grid operator: [9 coarse taps][32][4 classes * 8]
    a.cin = 32; a.cout = 32; a.kd = 1; a.kh = 3; a.kw = 3;
    a.w.assign((size_t)9 * 32 * 32, 0.f);
    auto coarse = [](int p, int k) { return p == 0 ? (k == 0 ? -1 : 0) : (k == 2 ? 1 : 0); };  // fine tap k of parity p -> coarse offset
    for (int ph = 0; ph < 2; ++ph)
      for (int pw = 0; pw < 2; ++pw)
        for (int kh = 0; kh < 3; ++kh)
          for (int kw = 0; kw < 3; ++kw) {
            const int ta = (coarse(ph, kh) + 1) * 3 + (coarse(pw, kw) + 1);
            for (int m = 0; m < 32; ++m)
              for (int co = 0; co < 8; ++co)
                a.w[((size_t)ta * 32 + m) * 32 + (ph * 2 + pw) * 8 + co] += w3.w[((size_t)(kh * 3 + kw) * 32 + m) * 8 + co];
          }
    FoldedConv b;   // W3 . Ws3 : [9][8][8]
    b.cin = 8; b.cout = 8; b.kd = 1; b.kh = 3; b.kw = 3;
    b.w.assign((size_t)9 * 8 * 8, 0.f);
    for (int t = 0; t < 9; ++t)
      for (int ci = 0; ci < 8; ++ci)
        for (int co = 0; co < 8; ++co) {
          double acc = 0;
          for (int m = 0; m < 32; ++m) acc += (double)w3.w[((size_t)t * 32 + m) * 8 + co] * (double)ws.w[(size_t)ci * 32 + m];
          b.w[((size_t)t * 8 + ci) * 8 + co] = (float)acc;
        }
    add_conv("f.out3a", a);
    convs_["f.out3a"].cout = 8;          // real channels per class; N = 4 classes x 8 = npad
    convs_["f.out3a"].tc_up2 = true;
    add_conv("f.out3b", b);
    TDM_CUDA(cudaMalloc(&d_bs3_, 32 * 4));
    TDM_CUDA(cudaMemcpy(d_bs3_, ws.bias.data(), 32 * 4, cudaMemcpyHostToDevice));
    fused_fpn_ = true;
  }

  template <typename TB>
  void upload_bimg(const FoldedConv& fc, DevConv& dc) {
    std::vector<TB> img;
    auto cvt = [](float v) -> TB { return from_host<TB>(v); };
    auto back = [](TB v) -> float { return to_host<TB>(v); };
    if (fc.cin == 8) tc::build_b_image<TB, 8>(fc.w.data(), fc.cin, fc.cout, dc.npad, fc.kd, img, +cvt, 1, dc.hilo, +back);
    else if (fc.cin == 16) tc::build_b_image<TB, 16>(fc.w.data(), fc.cin, fc.cout, dc.npad, fc.kd, img, +cvt, 1, dc.hilo, +back);
    else if (fc.cin == 32) tc::build_b_image<TB, 32>(fc.w.data(), fc.cin, fc.cout, dc.npad, fc.kd, img, +cvt, 1, dc.hilo, +back);
    else tc::build_b_image<TB, 64>(fc.w.data(), fc.cin, fc.cout, dc.npad, fc.kd, img, +cvt, dc.nsplit);
    TDM_CUDA(cudaMalloc(&dc.bimg, img.size() * sizeof(TB)));
    TDM_CUDA(cudaMemcpy(dc.bimg, img.data(), img.size() * sizeof(TB), cudaMemcpyHostToDevice));
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
      TDM_CUDA(cudaMemcpyToSymbol(c_conv00, &cw, sizeof(cw), (size_t)slot_ * sizeof(Conv00Weights)));
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
    TDM_CUDA(cudaMalloc(&select_state_, sizeof(SelectState)));
    TDM_CUDA(cudaMalloc(&select2_, sizeof(SelectState2)));
    TDM_CUDA(cudaMemset(select2_, 0, sizeof(SelectState2)));
    TDM_CUDA(cudaMallocHost(&h_params_, sizeof(CallParams)));
    TDM_CUDA(cudaMalloc(&d_params_, sizeof(CallParams)));
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
    TDM_CUDA(cudaMalloc(&b.p, b.bytes));
    TDM_CUDA(cudaMemsetAsync(b.p, 0, b.bytes, stream_));  // halos stay zero forever: kernels only write the interior
    bufs_[name] = b;
    return bufs_[name];
  }
  template <typename T>
  static P8<T> p8(const DevBuf& b) {
    P8<T> t;
    t.p = (T*)b.p;
    t.C = b.C; t.D = b.D; t.H = b.H; t.W = b.W; t.pd = b.pd;
    t.Hp = b.H + 2; t.Wp = b.W + 2;
    t.gs = (long long)(b.D + 2 * b.pd) * t.Hp * t.Wp * 8;
    return t;
  }
  void free_plan() {
    drop_graph();
    cv_tmap_ok_ = false;
    s2_cache_.clear();
    tc_cache_.clear();
    for (auto& kv : bufs_) cudaFree(kv.second.p);
    bufs_.clear();
    if (h_bgr_) cudaFreeHost(h_bgr_);
    if (h_out_) cudaFreeHost(h_out_);
    if (d_bgr_) cudaFree(d_bgr_);
    h_bgr_ = nullptr; h_out_ = nullptr; d_bgr_ = nullptr;
  }
  void ensure_plan(int V, int H, int W) {
    if (V == V_ && H == H_ && W == W_) return;
    free_plan();
    V_ = V; H_ = H; W_ = W;
    TDM_CUDA(cudaMallocHost(&h_bgr_, (size_t)V * H * W * 3));
    TDM_CUDA(cudaMallocHost(&h_out_, (size_t)4 * H * W * sizeof(float)));
    TDM_CUDA(cudaMalloc(&d_bgr_, (size_t)V * H * W * 3));
    alloc("f.img", 8, V, H, W);
    alloc("f.c0_0", 8, V, H, W);
    alloc("f.c3", 8, V, H, W);
    alloc("f.c1_0", 16, V, H / 2, W / 2);
    alloc("f.c1_1", 16, V, H / 2, W / 2);
    alloc("f.c2", 16, V, H / 2, W / 2);
    alloc("f.c2_0", 32, V, H / 4, W / 4);
    alloc("f.c2_1", 32, V, H / 4, W / 4);
    alloc("f.c1", 32, V, H / 4, W / 4);
    alloc("feat1", 32, V, H / 4, W / 4);
    alloc("f.i2", 32, V, H / 2, W / 2);
    alloc("f.i2b", 32, V, H / 2, W / 2);
    alloc("feat2", 16, V, H / 2, W / 2);
    alloc("f.i3", 32, V, H, W);
    alloc("feat3", 8, V, H, W);
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
      alloc(k + "dmin", 1, 1, Hs, Ws, true);
      for (const char* n : {"depth_dense", "confidence_dense", "depth", "confidence", "edge"})
        alloc(k + n, 1, 1, Hs, Ws, true);
    }
    alloc("thr", 1, 1, 1, 4, true);
  }
  float* fbuf(const std::string& n) { return (float*)bufs_.at(n).p; }

  // ---------------------------------------------------------------- launches
  void rec_begin(const std::string& name, double bytes, double flops) {
    ++launch_count_;
    if (!profiling_) return;
    LaunchRec r;
    r.name = name; r.bytes = bytes; r.flops = flops;
    cudaEventCreate(&r.e0);
    cudaEventCreate(&r.e1);
    cudaEventRecord(r.e0, stream_);
    recs_.push_back(r);
  }
  void rec_end() {
    if (!profiling_) return;
    cudaEventRecord(recs_.back().e1, stream_);
  }
  void rec_cancel() {
    --launch_count_;
    if (!profiling_) return;
    cudaEventDestroy(recs_.back().e0);
    cudaEventDestroy(recs_.back().e1);
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
    if constexpr (COUT == 1) plain = (float*)out.p; else o = p8<TOut>(out);
    if constexpr (COUT != 1) {
      if (out_b) {
        ob = p8<TOut>(*out_b);
        launch_k(k_conv_direct<TIn, TOut, CIN, COUT>, dim3(cdiv(npos, 128)), dim3(128), p8<const TIn>(in), c.w, c.bias, r, o, plain, g, ob, bias_b);
        return;
      }
    }
    if constexpr (COUT >= 16) {
      if (npos < 128ll * 592) {  // too few positions to fill the chip: split the output channels over blockIdx.y
        dim3 grid(cdiv(npos, 128), COUT / 8);
        launch_k(k_conv_direct<TIn, TOut, CIN, COUT, 8>, grid, dim3(128), p8<const TIn>(in), c.w, c.bias, r, o, plain, g, P8<TOut>{}, (const float*)nullptr);
        return;
      }
    }
    launch_k(k_conv_direct<TIn, TOut, CIN, COUT>, dim3(cdiv(npos, 128)), dim3(128), p8<const TIn>(in), c.w, c.bias, r, o, plain, g, P8<TOut>{}, (const float*)nullptr);
  }

  // the other kernels of the forward (all begin with grid_dep_sync()): with use_pdl = 2 they carry the attribute too
  template <typename... KArgs, typename... Args>
  void launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, Args&&... args) {
    if (use_pdl_ < 2) {
      kern<<<grid, block, 0, stream_>>>(static_cast<KArgs>(args)...);
      return;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = 0;
    cfg.stream = stream_;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    TDM_CUDA(cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...));
  }

  // tensor-core kernels are launched with programmatic stream serialization (PDL): their prologue and weight-image
  // load overlap the tail of the previous kernel (see pdl_wait() in conv_tc.cuh)
  template <typename Kern, typename... Args>
  void launch_pdl(Kern kern, dim3 grid, size_t smem, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = dim3(tc::kThreads);
    // with PDL an early-launched dependent must not stack several CTAs on the few SMs its predecessor left idle (they would
    // compete for those SMs' issue slots while the rest of the GPU waits): ask for enough shared memory that one CTA fills an SM
    cfg.dynamicSmemBytes = use_pdl_ ? std::max(smem, (size_t)pdl_min_smem_kb_ * 1024) : smem;
    cfg.stream = stream_;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = use_pdl_ ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    TDM_CUDA(cudaLaunchKernelEx(&cfg, kern, args...));
  }

  struct TcCache { tc::Plan plan; CUtensorMap tmap; };
  std::map<std::string, TcCache> tc_cache_;

  template <typename TIn, typename TOut, int CIN, int NPAD, int KD, bool PLAIN, int MODE = 0, bool HILO = false, typename Tail = tc::NoTail>
  void tc_inst(const std::string& wkey, const DevBuf& in, const DevConv& c, const DevBuf* res, const DevBuf& out, bool relu,
               const Tail& tail = Tail()) {
    const std::string key = wkey + (Tail::enabled ? "#tail" : "");
    auto it = tc_cache_.find(key);
    if (it == tc_cache_.end()) {
      TcCache tcx;
      tcx.plan = tc::make_plan(CIN, HILO ? 2 * NPAD : NPAD, KD, in.D, in.H, in.W, in.pd, MODE, (size_t)tc_smem_kb_ * 1024,   // tiles live on the INPUT grid
                               Tail::enabled);
      tc::Geom& g = tcx.plan.g;
      TDM_CHECK(!Tail::enabled || g.tiles_d == 1, "the prob tail needs tiles that span all depth planes");
      g.oHp = out.H + 2; g.oWp = out.W + 2; g.opd = out.pd;
      g.iDp = in.D + 2 * in.pd;
      g.in_gs = p8<const TIn>(in).gs;
      g.relu = relu ? 1 : 0;
      g.has_res = res ? 1 : 0;
      g.cout = c.cout;
      if constexpr (!PLAIN) {
        g.out_gs = p8<TOut>(out).gs;
        if (res) g.res_gs = p8<const TOut>(*res).gs;
      }
      const cuuint64_t dims[4] = {8, (cuuint64_t)(in.W + 2), (cuuint64_t)(in.H + 2), (cuuint64_t)g.iDp * (CIN / 8)};
      const cuuint64_t strides[3] = {16, (cuuint64_t)(in.W + 2) * 16, (cuuint64_t)(in.W + 2) * (in.H + 2) * 16};
      const cuuint32_t box[4] = {8, (cuuint32_t)g.P, (cuuint32_t)(g.R + 2), 1};
      const cuuint32_t estr[4] = {1, 1, 1, 1};
      const CUtensorMapDataType dt = std::is_same<TIn, __nv_bfloat16>::value ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
      const CUresult r = tc::encode_tiled_fn()(&tcx.tmap, dt, 4, in.p, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      TDM_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed for " + wkey + " (" + std::to_string((int)r) + ")");
      if (std::getenv("TDM_DEBUG_PLAN"))
        fprintf(stderr, "[plan] %-14s mode %d cin %d N %d kd %d in %dx%dx%d -> R %d TW %d DR %d S %d nch %d tiles %d x nsplit %d smem %zu\n", wkey.c_str(), MODE, CIN,
                HILO ? 2 * NPAD : NPAD, KD, in.D, in.H, in.W, g.R, g.TW, g.DR, g.S, g.nch, tcx.plan.grid, c.nsplit, tcx.plan.smem);
      it = tc_cache_.emplace(key, tcx).first;
    }
    const tc::Plan& pl = it->second.plan;
    TOut* op = nullptr;
    float* plain = nullptr;
    const TOut* rp = nullptr;
    if constexpr (PLAIN) {
      plain = (float*)out.p;
    } else {
      op = (TOut*)out.p;
      if (res) rp = (const TOut*)res->p;
    }
    auto kern = tc::k_conv_tc<TIn, TOut, CIN, NPAD, KD, PLAIN, MODE, HILO, Tail>;
    static bool attr_set = false;
    if (!attr_set) {
      TDM_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      attr_set = true;
    }
    launch_pdl(kern, dim3(pl.grid, c.nsplit), pl.smem, it->second.tmap, (const TIn*)c.bimg, (const float*)c.bias, rp, op, plain, pl.g, tail);
  }

  struct S2Cache { tc::PlanS2 plan; CUtensorMap tmap; };
  std::map<std::string, S2Cache> s2_cache_;

  template <int CIN, int NPAD, int KD, int KS>
  void tc_s2_inst(const std::string& wkey, const DevBuf& in, const DevConv& c, const DevBuf& out, bool relu) {
    auto it = s2_cache_.find(wkey);
    if (it == s2_cache_.end()) {
      S2Cache sc;
      sc.plan = tc::make_plan_s2(CIN, NPAD, KD, KS, out.D, out.H, out.W, (size_t)tc_smem_kb_ * 1024);
      tc::GeomS2& g = sc.plan.g;
      const P8<TA> po = p8<TA>(out);
      g.oHp = out.H + 2; g.oWp = out.W + 2; g.opd = out.pd; g.out_gs = po.gs;
      g.ipd = in.pd; g.iDp = in.D + 2 * in.pd;
      g.c0 = 1 - KS / 2;
      g.relu = relu ? 1 : 0;
      g.cout = c.cout;
      std::vector<std::pair<int, int>> taps;
      tc::s2_tap_table(KS, g.P, g.sub_pos, taps, g.tap_off);
      // tensor map over the P8 input: dims {8 ch, Wp, Hp, groups*planes}, every second column / row per box
      const cuuint64_t dims[4] = {8, (cuuint64_t)(in.W + 2), (cuuint64_t)(in.H + 2), (cuuint64_t)g.iDp * (CIN / 8)};
      const cuuint64_t strides[3] = {16, (cuuint64_t)(in.W + 2) * 16, (cuuint64_t)(in.W + 2) * (in.H + 2) * 16};
      const cuuint32_t box[4] = {8, (cuuint32_t)(2 * g.P), (cuuint32_t)(2 * g.RR), 1};
      const cuuint32_t estr[4] = {1, 2, 2, 1};
      const CUtensorMapDataType dt = std::is_same<TA, __nv_bfloat16>::value ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
      const CUresult r = tc::encode_tiled_fn()(&sc.tmap, dt, 4, in.p, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      TDM_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed for " + wkey + " (" + std::to_string((int)r) + ")");
      if (std::getenv("TDM_DEBUG_PLAN"))
        fprintf(stderr, "[plan] %-14s S2 cin %d N %d kd %d ks %d out %dx%dx%d -> R %d TW %d DR %d S %d nch %d tiles %d x nsplit %d smem %zu\n", wkey.c_str(), CIN, NPAD, KD, KS,
                out.D, out.H, out.W, g.R, g.TW, g.DR, g.S, g.nch, sc.plan.grid, c.nsplit_s2, sc.plan.smem);
      it = s2_cache_.emplace(wkey, sc).first;
    }
    auto kern = tc::k_conv_tc_s2<TA, TA, CIN, NPAD, KD, KS>;
    static bool attr_set = false;
    if (!attr_set) {
      TDM_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      attr_set = true;
    }
    const tc::PlanS2& pl = it->second.plan;
    launch_pdl(kern, dim3(pl.grid, c.nsplit_s2), pl.smem, it->second.tmap, (const TA*)c.bimg_s2, (const float*)c.bias, (TA*)out.p, pl.g);
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
#define TDM_TC(TI, CI, NP, KDV, HL)                                                        \
  if (c.cin == CI && c.npad == NP && c.kd == KDV && c.hilo == HL) {                        \
    tc_inst<TI, TA, CI, NP, KDV, false, 0, HL>(wkey, bi, c, rp, bo, relu);                       \
    return true;                                                                           \
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

  void conv_up2(const std::string& wkey, const std::string& in, const std::string& out) {
    if constexpr (sizeof(TA) == 2) {
      const DevConv& c = convs_.at(wkey);
      const DevBuf& bi = bufs_.at(in);
      const DevBuf& bo = bufs_.at(out);
      TDM_CHECK(c.tc_up2 && bo.H == 2 * bi.H && bo.W == 2 * bi.W && bo.D == bi.D, "conv_up2 shape mismatch");
      rec_begin(wkey + "[tc-up2]", (double)bi.alg_bytes + (double)bo.alg_bytes, 2.0 * 9 * 32 * 8 * (double)bo.D * bo.H * bo.W);
      tc_inst<TA, TA, 32, 32, 1, false, 3, true>(wkey, bi, c, nullptr, bo, false);
      TDM_CUDA(cudaGetLastError());
      rec_end();
    } else {
      throw Error("conv_up2 needs a 16-bit engine");
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
        k_prob_direct<4><<<cdiv(nthr, 128), 128, 0, stream_>>>(p8<const __half>(bi), (float*)bo.p, prob_w_[wkey[1] - '1']);
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
    TDM_CUDA(cudaMemcpyAsync(d_params_, h_params_, sizeof(CallParams), cudaMemcpyHostToDevice, stream_));
    TDM_CUDA(cudaMemcpyToSymbolAsync(c_call_params, h_params_, sizeof(CallParams), (size_t)slot_ * sizeof(CallParams),
                                     cudaMemcpyHostToDevice, stream_));
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
    bool done = false;
    if constexpr (std::is_same<TA, __half>::value) {
      if (va_ && cv_variant_ == 5 && fb.C == 8 && vb.D == 8) {
        // A/B: source-view tiles staged in shared memory by TMA (cost_volume_tma.cuh); other stages run variant 3
        if (!cv_tmap_ok_) {
          const cuuint64_t dims[4] = {8, (cuuint64_t)(fb.W + 2), (cuuint64_t)(fb.H + 2), (cuuint64_t)(fb.D + 2 * fb.pd)};
          const cuuint64_t strides[3] = {16, (cuuint64_t)(fb.W + 2) * 16, (cuuint64_t)(fb.W + 2) * (fb.H + 2) * 16};
          const cuuint32_t box[4] = {8, (cuuint32_t)kCvBW, (cuuint32_t)kCvBH, 1};
          const cuuint32_t estr[4] = {1, 1, 1, 1};
          const CUresult r = tc::encode_tiled_fn()(&cv_tmap_, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, fb.p, dims, strides, box, estr,
                                                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
          TDM_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed for the cost-volume source tile");
          if (!d_cv_stats_) { TDM_CUDA(cudaMalloc(&d_cv_stats_, 2 * sizeof(unsigned))); TDM_CUDA(cudaMemset(d_cv_stats_, 0, 2 * sizeof(unsigned))); }
          cv_tmap_ok_ = true;
        }
        k_cost_volume_va16_tma<TV, true><<<dim3(cdiv(vb.W, 16), cdiv(vb.H, 8)), 256, 0, stream_>>>(cv_tmap_, p8<const __half>(fb), dm, p8<TV>(vb), slot_, s - 1, d_cv_stats_);
        TDM_CUDA(cudaGetLastError());
        rec_end();
        return;
      }
      if (va_ && cv_variant_ > 0) {
        done = true;
        const int nd = (cv_variant_ == 2 || cv_variant_ == 4) ? 4 : (fb.C == 8 ? 4 : 2);
        const bool h16 = cv_variant_ >= 3;   // (variant 5 = variant 3 outside stage 3)
        const long long thr = (long long)cdiv(vb.D, nd) * vb.H * vb.W * (fb.C == 32 ? 2 : 1);
        const unsigned grid = (unsigned)cdiv(thr, 128);
        auto go = [&](auto kern) { launch_k(kern, dim3(grid), dim3(128), p8<const __half>(fb), dm, p8<TV>(vb), slot_, s - 1); };
        if (fb.C == 32) {
          if (nd == 2) { if (h16) go(k_cost_volume_va16<TV, 16, 2, 2, true>); else go(k_cost_volume_va16<TV, 16, 2, 2, false>); }
          else         { if (h16) go(k_cost_volume_va16<TV, 16, 2, 4, true>); else go(k_cost_volume_va16<TV, 16, 2, 4, false>); }
        } else if (fb.C == 16) {
          if (nd == 2) { if (h16) go(k_cost_volume_va16<TV, 16, 1, 2, true>); else go(k_cost_volume_va16<TV, 16, 1, 2, false>); }
          else         { if (h16) go(k_cost_volume_va16<TV, 16, 1, 4, true>); else go(k_cost_volume_va16<TV, 16, 1, 4, false>); }
        } else if (fb.C == 8) {
          if (h16) go(k_cost_volume_va16<TV, 8, 1, 4, true>); else go(k_cost_volume_va16<TV, 8, 1, 4, false>);
        } else {
          throw Error("unsupported feature channels");
        }
      }
    }
    if (done) {}
    else if (fb.C == 32) k_cost_volume<TA, TV, 16, 2><<<cdiv(2 * n, 128), 128, 0, stream_>>>(p8<const TA>(fb), dm, p8<TV>(vb), slot_, s - 1);
    else if (fb.C == 16) k_cost_volume<TA, TV, 16><<<cdiv(n, 128), 128, 0, stream_>>>(p8<const TA>(fb), dm, p8<TV>(vb), slot_, s - 1);
    else if (fb.C == 8) k_cost_volume<TA, TV, 8><<<cdiv(n, 128), 128, 0, stream_>>>(p8<const TA>(fb), dm, p8<TV>(vb), slot_, s - 1);
    else throw Error("unsupported feature channels");
    TDM_CUDA(cudaGetLastError());
    rec_end();
  }

  // where stage s takes the lower end of its hypothesis range from: computed in place from the previous stage's depth
  // (inline_dmin_, default) or read from the map k_adaptive_dmin materialised
  DminSrc dmin_src(int s) {
    DminSrc d{nullptr, nullptr, 0, 0};
    if (s <= 1) return d;
    const std::string k = "s" + std::to_string(s) + ".";
    if (!inline_dmin_) { d.map = fbuf(k + "dmin"); return d; }
    const DevBuf& pd = bufs_.at("s" + std::to_string(s - 1) + ".depth_dense");
    d.prev = (const float*)pd.p; d.ph = pd.H; d.pw = pd.W;
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
    if (fused_select_) {
      rec_begin(k + "edge_metric+select0", 8.0 * n, 0);
      launch_k(k_edge_metric_select0, dim3(cdiv(n, 256)), dim3(256), fbuf(k + "depth_dense"), fbuf(k + "edge"), d.H, d.W, select2_, &d_params_->cutoff[s - 1]);
      rec_end();
      rec_begin(k + "percentile", 8.0 * n, 0);
      for (int pass = 1; pass <= 2; ++pass)
        launch_k(k_select_pass, dim3(std::min(cdiv(n, 256 * 8), 2 * kNumSm)), dim3(256), fbuf(k + "edge"), n, select2_, pass, fbuf("thr") + (s - 1));
      launch_count_ += 1;
      rec_end();
    } else {
    rec_begin(k + "edge_metric", 8.0 * n, 0);
    k_edge_metric<<<cdiv(n, 128), 128, 0, stream_>>>(fbuf(k + "depth_dense"), fbuf(k + "edge"), d.H, d.W);
    rec_end();
    rec_begin(k + "percentile", 12.0 * n, 0);
    k_select_init<<<1, 256, 0, stream_>>>(select_state_, &d_params_->cutoff[s - 1]);
    for (int pass = 0; pass < 3; ++pass) {
      k_select_hist<<<std::min(cdiv(n, 256 * 8), 592), 256, 0, stream_>>>(fbuf(k + "edge"), n, select_state_, pass);
      k_select_scan<<<1, 1024, 0, stream_>>>(select_state_, pass, fbuf("thr") + (s - 1));
    }
    launch_count_ += 6;
    rec_end();
    }
    rec_begin(k + "apply_mask", 20.0 * n, 0);
    launch_k(k_apply_edge_mask, dim3(cdiv(n, 256)), dim3(256), fbuf(k + "edge"), fbuf("thr") + (s - 1), fbuf(k + "depth_dense"),
                                                       fbuf(k + "confidence_dense"), fbuf(k + "depth"),
                                                       fbuf(k + "confidence"), n);
    TDM_CUDA(cudaGetLastError());
    rec_end();
  }

  // Per-call parameters are refreshed in device memory, then the (otherwise argument-invariant) kernel sequence is
  // replayed as a CUDA graph: captured on the second forward of a plan (the first one warms the tensor-map / attribute
  // caches), invalidated by free_plan() and by option changes.
  void forward(bool profiling) {
    upload_call_params();
    if (profiling || !use_graph_) { forward_launches(profiling); return; }
    if (graph_exec_) { TDM_CUDA(cudaGraphLaunch(graph_exec_, stream_)); return; }
    if (!warmed_) { forward_launches(false); warmed_ = true; return; }
    cudaGraph_t graph = nullptr;
    TDM_CUDA(cudaStreamBeginCapture(stream_, cudaStreamCaptureModeThreadLocal));
    try {
      forward_launches(false);
    } catch (...) {
      cudaStreamEndCapture(stream_, &graph);
      if (graph) cudaGraphDestroy(graph);
      throw;
    }
    TDM_CUDA(cudaStreamEndCapture(stream_, &graph));
    TDM_CUDA(cudaGraphInstantiate(&graph_exec_, graph, 0));
    cudaGraphDestroy(graph);
    TDM_CUDA(cudaGraphLaunch(graph_exec_, stream_));
  }
  void drop_graph() {
    if (graph_exec_) cudaGraphExecDestroy(graph_exec_);
    graph_exec_ = nullptr;
    warmed_ = false;
  }

  // The whole graph of cva_mvsnet.py:98-184 on stream_, inputs already in d_bgr_.
  void forward_launches(bool profiling) {
    profiling_ = profiling;
    launch_count_ = 0;
    const int V = V_, H = H_, W = W_;
    {
      ViewPtrs vp;
      for (int v = 0; v < V; ++v) vp.v[v] = d_bgr_ + (size_t)v * H * W * 3;
      const long long n = (long long)V * H * W;
      bool fused = false;
      if constexpr (kRawInput) {
        if (direct_conv00_) {
          fused = true;
          rec_begin("f.conv0.0[u8-direct]", 3.0 * n + 8.0 * n * sizeof(TA), 2.0 * 27 * 8 * (double)n);
          launch_k(k_conv00_u8<TA>, dim3(cdiv(W, 32), cdiv(H, 8), V), dim3(256), d_bgr_, p8<TA>(bufs_.at("f.c0_0")), H, W, slot_);
          TDM_CUDA(cudaGetLastError());
          rec_end();
        }
      }
      if (!fused) {
        rec_begin("preprocess", 3.0 * n + 8.0 * n * sizeof(TA), 0);
        k_preprocess_bgr<TA, kRawInput><<<cdiv(n, 256), 256, 0, stream_>>>(vp, p8<TA>(bufs_.at("f.img")), V, H * W);
        TDM_CUDA(cudaGetLastError());
        rec_end();
        conv("f.conv0.0", "f.img", "f.c0_0", 1, 1, 1, true);
      }
    }
    conv("f.conv0.1", "f.c0_0", "f.c3", 1, 1, 1, true);
    conv("f.conv1.0", "f.c3", "f.c1_0", 1, 2, 2, true);
    conv("f.conv1.1", "f.c1_0", "f.c1_1", 1, 1, 1, true);
    conv("f.conv1.2", "f.c1_1", "f.c2", 1, 1, 1, true);
    conv("f.conv2.0", "f.c2", "f.c2_0", 1, 2, 2, true);
    conv("f.conv2.1", "f.c2_0", "f.c2_1", 1, 1, 1, true);
    conv("f.conv2.2", "f.c2_1", "f.c1", 1, 1, 1, true);
    // The pyramid's upper outputs (feat2, feat3) are only read by stages 2 and 3, while stage 1 needs feat1 alone and its
    // coarse U-Net levels leave most SMs idle: the FPN tail runs on a second stream, forked here and joined before the
    // stage-2 cost volume (inside the captured graph these are two parallel branches).  Not while profiling: the per-kernel
    // events assume one stream.
    const bool fork = fork_fpn_ && !profiling;
    struct SwapBack {   // an exception inside the branch must not leave the engine on the side stream
      cudaStream_t &a, &b; bool on;
      ~SwapBack() { if (on) std::swap(a, b); }
    } side{stream_, side_stream_, false};
    if (fork) {
      TDM_CUDA(cudaEventRecord(ev_fork_, stream_));
      TDM_CUDA(cudaStreamWaitEvent(side_stream_, ev_fork_, 0));
      std::swap(stream_, side_stream_);
      side.on = true;
    } else {
      conv("f.out1", "f.c1", "feat1", 1, 1, 1, false);
    }
    if (fused_fpn_ && use_tc_) {
      conv("f.skip2", "f.c2", "f.i2", 1, 1, 1, false, 2, "f.c1", "f.i2b", d_bs3_);
      conv("f.out2", "f.i2", "feat2", 1, 1, 1, false);
      conv_up2("f.out3a", "f.i2b", "feat3");
      conv("f.out3b", "f.c3", "feat3", 1, 1, 1, false, 1, "feat3");
    } else {
      conv("f.skip2", "f.c2", "f.i2", 1, 1, 1, false, 2, "f.c1");
      conv("f.out2", "f.i2", "feat2", 1, 1, 1, false);
      conv("f.skip3", "f.c3", "f.i3", 1, 1, 1, false, 2, "f.i2");
      conv("f.out3", "f.i3", "feat3", 1, 1, 1, false);
    }
    if (fork) {
      TDM_CUDA(cudaEventRecord(ev_join_, stream_));      // stream_ is the side stream here
      std::swap(stream_, side_stream_);
      side.on = false;
      conv("f.out1", "f.c1", "feat1", 1, 1, 1, false);
    }

    for (int s = 1; s <= 3; ++s) {
      const std::string k = "s" + std::to_string(s) + ".";
      const HypSpec hs = hyp_spec(s);
      const DevBuf& dd = bufs_.at(k + "depth_dense");
      if (s == 2 && fork) TDM_CUDA(cudaStreamWaitEvent(stream_, ev_join_, 0));
      if (s > 1 && !inline_dmin_) {
        const DevBuf& pd = bufs_.at("s" + std::to_string(s - 1) + ".depth_dense");
        rec_begin(k + "adaptive_dmin", 4.0 * (pd.H * pd.W + dd.H * dd.W), 0);
        k_adaptive_dmin<<<cdiv(dd.H * dd.W, 256), 256, 0, stream_>>>((const float*)pd.p, pd.H, pd.W, fbuf(k + "dmin"),
                                                                    &d_params_->half_range[s - 1]);
        TDM_CUDA(cudaGetLastError());
        rec_end();
      }
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
        forward(false);
        if (eager_d2h_) {
          const char* names[4] = {"s3.depth", "s3.confidence", "s3.depth_dense", "s3.confidence_dense"};
          for (int k = 0; k < 4; ++k) {
            TDM_CUDA(cudaMemcpyAsync(h_out_ + k * n, fbuf(names[k]), n * 4, cudaMemcpyDeviceToHost, stream_));
            TDM_CUDA(cudaEventRecord(ev_out_[k], stream_));
          }
        } else {
          TDM_CUDA(cudaEventRecord(ev_out_[0], stream_));   // GetResult copies back itself (page-locked caller buffers)
        }
        wait_event_politely(ev_out_[0]);   // result "ready" as soon as the first map is home; GetResult waits per map
      } catch (const std::exception& e) {
        err = e.what();
      }
      {
        std::lock_guard<std::mutex> lk(mu_);
        worker_error_ = err;
        has_result_ = err.empty();
        busy_ = false;
        started_ = false;
      }
      cv_done_.notify_all();
    }
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
  cudaStream_t stream_ = nullptr;
  WeightFile wf_;
  int depth_num_[3];
  bool va_ = false;
  std::map<std::string, DevConv> convs_;
  Gate gates_[3];
  std::map<std::string, DevBuf> bufs_;
  SelectState* select_state_ = nullptr;
  SelectState2* select2_ = nullptr;
  bool inline_dmin_ = true;    // adaptive range's d_min computed where it is consumed (dmin_px) instead of by k_adaptive_dmin (A/B: 0)
  // softmax / soft-argmin / confidence in the epilogue of the tensor-core prob convolution (set_option("fused_regress", 1)):
  // bit-identical to k_regress and three launches fewer, but the consumer threads of a CTA finish their pixels after the last
  // plane with nothing left to overlap, where the stand-alone kernel spreads the same work over 2048 threads per SM. Off.
  bool fused_regress_ = false;
  struct TailReq { int stage; int D; DminSrc dsrc; float* depth; float* conf; const HypSpec* hyp; const float* half_range; bool done; };
  TailReq tail_req_{};
  int pdl_min_smem_kb_ = 120;
  bool fused_select_ = true;   // edge metric + pass 0 in one kernel, passes 1 / 2 with the scan in their last CTA (A/B: set_option("fused_select", 0))
  int V_ = 0, H_ = 0, W_ = 0;
  unsigned char* h_bgr_ = nullptr;
  unsigned char* d_bgr_ = nullptr;
  float* h_out_ = nullptr;
  cudaEvent_t ev_out_[4] = {nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t ev_in_ = nullptr;
  bool eager_d2h_ = true;   // worker copies the four maps into pinned staging right behind the forward (pageable callers);
                            // 0: GetResult copies back itself - for callers that pass page-locked result buffers
  float c2w_[kMaxSrc + 1][16];
  float K_[27];
  float dmin_ = 0, dmax_ = 0, discard_ = 0;
  float* d_bs3_ = nullptr;
  CallParams* h_params_ = nullptr;   // pinned
  CallParams* d_params_ = nullptr;
  cudaGraphExec_t graph_exec_ = nullptr;
  CUtensorMap cv_tmap_{};      // cv_variant 5 (A/B): tiled view of feat3 for the TMA-staged cost volume
  bool cv_tmap_ok_ = false;
  unsigned* d_cv_stats_ = nullptr;
  int cv_variant_ = 3;   // 0: generic cost-volume kernel; 1-4: k_cost_volume_va16 (ND 2/2/4 | 4/4/4, fp32 | fp16 accumulate)
  // Programmatic dependent launch of the tensor-core kernels: the trigger sits after griddepcontrol.wait (a trigger before it
  // lets the whole chain of later kernels become resident early), and pdl_min_smem_kb_ = 120 keeps one tensor-core CTA per SM.
  bool warmed_ = false, use_graph_ = true;
  int use_pdl_ = 1;   // 2: the FMA-pipe kernels (cost volume, soft-argmin, edge filter ...) are launched with the attribute as well
  int slot_ = 0;           // index into c_call_params
  int tc_smem_kb_ = 225;   // shared-memory budget of the tile planner (<= 113 lets two CTAs share an SM)
  bool fused_fpn_ = false;
  bool prob_direct_ = false;  // `prob` (8 -> 1 channels) on the FMA pipes (k_prob_direct) instead of the tensor-core tile; an A/B option and an independent check
  bool have_prob_w_ = false;
  ProbWeights prob_w_[3] = {};
  bool direct_conv00_ = true; // 16-bit engines: pre-processing + conv0.0 fused on the FMA pipes (k_conv00_u8); 0 = preprocess + tensor-core conv
  bool fork_fpn_ = true;      // FPN tail on a second stream / graph branch (A/B: set_option("fork_fpn", 0))
  cudaStream_t side_stream_ = nullptr;
  cudaEvent_t ev_fork_ = nullptr, ev_join_ = nullptr;
  bool filter_all_ = false, keep_ = true, use_tc_ = (sizeof(TA) == 2);  // tensor-core convs are the default on 16-bit engines
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

// host-only view of the tensor-core tile planner (no GPU involved; used by the CPU test-suite): out12 = {S, R, TW, P, DR, nch,
// slot_pos, tiles_w, tiles_h, tiles_d, grid, smem_bytes}
void debug_conv_plan(int cin, int npad, int kd, int D, int H, int W, int pd, int mode, int smem_kb, long long* out12) {
  // mode + 100 = the same mode with tiles that span all D planes (the prob layer with the soft-argmin tail)
  const tc::Plan p = tc::make_plan(cin, npad, kd, D, H, W, pd, mode % 100, (size_t)smem_kb * 1024, mode >= 100);
  const tc::Geom& g = p.g;
  const long long v[12] = {g.S, g.R, g.TW, g.P, g.DR, g.nch, g.slot_pos, g.tiles_w, g.tiles_h, g.tiles_d, p.grid, (long long)p.smem};
  for (int i = 0; i < 12; ++i) out12[i] = v[i];
}

}  // namespace tdm
