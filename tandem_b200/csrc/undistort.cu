// n11: DSO's per-frame input on the device.  PhotometricUndistorter (tandem/src/util/Undistort.cpp:50-179 constructor,
// :213-252 processFrame), Undistort::undistort's bilinear remap (:393-490), the dataset reader's BGR remap
// (DatasetReader.h:354-400) and FullSystem::setGammaFunction (FullSystem.cpp:232-253).  Every float operation is the
// reference's own, correctly rounded and in its order (__f*_rn, no contraction); oracle/undistort_oracle.c restates the same
// statements on the CPU.
//
// Shape.  processFrame works per pixel, so k_undistort applies it at the four taps of each output pixel's bilinear footprint
// (G in shared memory, vignetteMapInv from global memory) and writes level 0's grey straight into the pyramid's input; the
// pyramid's build_device then runs the kernels of tdm_pyramid_build from there, with the gamma weights when asked.  The BGR
// remap rides in the same launch (same table entry, same weights).  One upload of the raw u8 frame (0.3 MB at 640x480)
// replaces the 1.2 MB float image tdm_pyramid_build uploads.
#include <climits>
#include <cstring>
#include <vector>

#include "../../include/tandem_b200.h"
#include "tracker.h"

namespace tdm {

enum Photometric { PH_FACTOR = 0, PH_G = 1, PH_G_VIGNETTE = 2 };
constexpr int kUndistortThreads = 256;

template <int kPh>
__device__ __forceinline__ float photometric(const unsigned char* __restrict__ raw, const float* sG,
                                             const float* __restrict__ vinv, float factor, int j) {
  const unsigned char r = __ldg(raw + j);
  if constexpr (kPh == PH_FACTOR) return __fmul_rn(factor, (float)r);
  if constexpr (kPh == PH_G) return sG[r];
  return __fmul_rn(sG[r], __ldg(vinv + j));
}

// One thread per output pixel.  remap null: passthrough (w == w_org, h == h_org).  bgr_out null: grey only.
template <int kPh, bool kRemap, bool kBgr>
__global__ void __launch_bounds__(kUndistortThreads)
k_undistort(const float2* __restrict__ remap, const unsigned char* __restrict__ raw, const float* __restrict__ G,
            const float* __restrict__ vinv, float factor, float* __restrict__ gray, const unsigned char* __restrict__ bgr,
            unsigned char* __restrict__ bgr_out, int w, int h, int w_org, int h_org) {
  __shared__ float sG[256];
  if constexpr (kPh != PH_FACTOR) {
    sG[threadIdx.x] = G[threadIdx.x];
    __syncthreads();
  }
  const int i = blockIdx.x * kUndistortThreads + threadIdx.x;
  if (i >= w * h) return;
  if constexpr (!kRemap) {
    gray[i] = photometric<kPh>(raw, sG, vinv, factor, i);
    if constexpr (kBgr)
      for (int c = 0; c < 3; ++c) bgr_out[3 * (size_t)i + c] = bgr[3 * (size_t)i + c];
    return;
  }
  const float2 m = remap[i];
  float xx = m.x, yy = m.y;
  // outside (header, n11): xx < 0, yy < 0, (int)xx + 1 > w_org - 1, (int)yy + 1 > h_org - 1, or NaN
  if (!(xx >= 0.f && yy >= 0.f && xx < (float)(w_org - 1) && yy < (float)(h_org - 1))) {
    gray[i] = 0.f;
    if constexpr (kBgr)
      for (int c = 0; c < 3; ++c) bgr_out[3 * (size_t)i + c] = 0;
    return;
  }
  const int xxi = __float2int_rz(xx), yyi = __float2int_rz(yy);
  xx = __fsub_rn(xx, (float)xxi);
  yy = __fsub_rn(yy, (float)yyi);
  const float xxyy = __fmul_rn(xx, yy);
  const float w11 = xxyy, w01 = __fsub_rn(yy, xxyy), w10 = __fsub_rn(xx, xxyy);
  const float w00 = __fadd_rn(__fsub_rn(__fsub_rn(1.f, xx), yy), xxyy);
  const int j = xxi + yyi * w_org;
  // Undistort.cpp:468-471: xxyy * src[1+wOrg] + (yy-xxyy) * src[wOrg] + (xx-xxyy) * src[1] + (1-xx-yy+xxyy) * src[0]
  gray[i] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(w11, photometric<kPh>(raw, sG, vinv, factor, j + 1 + w_org)),
                                          __fmul_rn(w01, photometric<kPh>(raw, sG, vinv, factor, j + w_org))),
                                __fmul_rn(w10, photometric<kPh>(raw, sG, vinv, factor, j + 1))),
                      __fmul_rn(w00, photometric<kPh>(raw, sG, vinv, factor, j)));
  if constexpr (kBgr) {
    for (int c = 0; c < 3; ++c) {
      const unsigned char* s = bgr + 3 * (size_t)j + c;
      const float v = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(w11, (float)s[3 + 3 * w_org]), __fmul_rn(w01, (float)s[3 * w_org])),
                                          __fmul_rn(w10, (float)s[3])),
                                __fmul_rn(w00, (float)s[0]));
      bgr_out[3 * (size_t)i + c] = (unsigned char)__float2int_rz(v);   // static_cast<unsigned char>, v in (-1, 256)
    }
  }
}

template <int kPh, bool kRemap, bool kBgr>
static void launch_undistort_t(cudaStream_t st, const float2* remap, const unsigned char* raw, const float* G, const float* vinv,
                               float factor, float* gray, const unsigned char* bgr, unsigned char* bgr_out, int w, int h,
                               int w_org, int h_org) {
  k_undistort<kPh, kRemap, kBgr><<<cdiv((long long)w * h, kUndistortThreads), kUndistortThreads, 0, st>>>(
      remap, raw, G, vinv, factor, gray, bgr, bgr_out, w, h, w_org, h_org);
}
template <int kPh>
static void launch_undistort_p(cudaStream_t st, const float2* remap, const unsigned char* raw, const float* G, const float* vinv,
                               float factor, float* gray, const unsigned char* bgr, unsigned char* bgr_out, int w, int h,
                               int w_org, int h_org) {
  const int sel = (remap ? 2 : 0) + (bgr_out ? 1 : 0);
  auto f = sel == 0 ? launch_undistort_t<kPh, false, false> : sel == 1 ? launch_undistort_t<kPh, false, true>
         : sel == 2 ? launch_undistort_t<kPh, true, false> : launch_undistort_t<kPh, true, true>;
  f(st, remap, raw, G, vinv, factor, gray, bgr, bgr_out, w, h, w_org, h_org);
}

static bool page_locked(const void* p) {
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return at.type == cudaMemoryTypeHost;
}

class UndistortImpl final : public UndistortIface {
 public:
  UndistortImpl(const tdm_undistort_settings& s, int device) : device_(device) {
    TDM_CHECK(s.w_org > 0 && s.h_org > 0 && s.w > 0 && s.h > 0, "undistort sizes must be positive");
    TDM_CHECK((s.remap_x == nullptr) == (s.remap_y == nullptr), "pass both remap tables or neither (passthrough)");
    TDM_CHECK(s.remap_x || (s.w == s.w_org && s.h == s.h_org), "passthrough needs w == w_org and h == h_org");
    TDM_CHECK(!s.response || (s.n_response >= 256 && s.n_response <= 65536), "n_response outside 256..65536");
    TDM_CHECK(s.photometric_calibration >= 0 && s.photometric_calibration <= 2, "photometric_calibration outside 0..2");
    int nd = 0;
    if (cudaGetDeviceCount(&nd) != cudaSuccess || nd == 0)
      throw Error("tandem_b200: no CUDA device visible - this library has no CPU fallback");
    w_ = s.w; h_ = s.h; w_org_ = s.w_org; h_org_ = s.h_org;
    mode_ = s.photometric_calibration;
    use_exposure_ = s.use_exposure != 0;
    gamma_weights_ = s.gamma_weights != 0;
    const size_t n_org = (size_t)w_org_ * h_org_, n = (size_t)w_ * h_;

    // PhotometricUndistorter::PhotometricUndistorter (Undistort.cpp:50-179) on the caller's arrays
    float G[256] = {};
    std::vector<float> vinv;
    bool response_ok = false;
    if (s.response) {
      const float* r = s.response;
      const int depth = s.n_response;
      response_ok = true;
      for (int i = 0; i < depth - 1; ++i)
        if (r[i + 1] <= r[i]) { response_ok = false; break; }
      if (response_ok) {
        const float mn = r[0], mx = r[depth - 1];
        for (int i = 0; i < 256; ++i) G[i] = (float)(255.0 * (double)(r[i] - mn) / (double)(mx - mn));
        if (mode_ == 0)
          for (int i = 0; i < 256; ++i) G[i] = 255.0f * (float)i / (float)(depth - 1);
      }
    }
    if (response_ok && s.vignette) {
      float maxv = 0.f;
      for (size_t i = 0; i < n_org; ++i)
        if ((float)s.vignette[i] > maxv) maxv = (float)s.vignette[i];
      vinv.resize(n_org);
      for (size_t i = 0; i < n_org; ++i) vinv[i] = 1.0f / ((float)s.vignette[i] / maxv);
      valid_ = true;
    }
    std::memcpy(G_, G, sizeof G_);
    for (int i = 0; i < 256; ++i) B_[i] = (float)i;   // CalibHessian's identity (HessianBlocks.h:392)

    TDM_CUDA(cudaSetDevice(device_));
    uploaded_ = make_event(cudaEventDisableTiming);
    done_ = make_event(cudaEventDisableTiming);
    bgr_done_ = make_event(cudaEventDisableTiming);
    d_G_ = make_dev<float>(256 * 4);
    d_B_ = make_dev<float>(256 * 4);
    TDM_CUDA(cudaMemcpy(d_G_.get(), G_, 256 * 4, cudaMemcpyHostToDevice));
    TDM_CUDA(cudaMemcpy(d_B_.get(), B_, 256 * 4, cudaMemcpyHostToDevice));
    if (valid_ && mode_ == 2) {
      d_vinv_ = make_dev<float>(4 * n_org);
      TDM_CUDA(cudaMemcpy(d_vinv_.get(), vinv.data(), 4 * n_org, cudaMemcpyHostToDevice));
    }
    if (s.remap_x) {
      std::vector<float2> m(n);
      for (size_t i = 0; i < n; ++i) m[i] = make_float2(s.remap_x[i], s.remap_y[i]);
      d_remap_ = make_dev<float2>(sizeof(float2) * n);
      TDM_CUDA(cudaMemcpy(d_remap_.get(), m.data(), sizeof(float2) * n, cudaMemcpyHostToDevice));
    }
    d_raw_ = make_dev<unsigned char>(n_org);
    h_raw_ = make_host<unsigned char>(n_org);
  }
  ~UndistortImpl() override {
    cudaSetDevice(device_);
    cudaEventSynchronize(done_.get());
  }

  void get_gamma(float G[256], int* valid) const override {
    TDM_CHECK(G && valid, "null argument");
    if (valid_) std::memcpy(G, G_, sizeof G_);
    *valid = valid_ ? 1 : 0;
  }

  // FullSystem::setGammaFunction (FullSystem.cpp:232-253)
  void set_gamma(const float* Binv) override {
    if (!Binv) return;
    float B[256];
    std::memcpy(B, B_, sizeof B);
    for (int i = 1; i < 255; i++)
      for (int s = 1; s < 255; s++)
        if (Binv[s] <= (float)i && Binv[s + 1] >= (float)i) {
          B[i] = (float)s + ((float)i - Binv[s]) / (Binv[s + 1] - Binv[s]);
          break;
        }
    B[0] = 0;
    B[255] = 255;
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaEventSynchronize(done_.get()));   // pending frames read d_B_
    TDM_CUDA(cudaMemcpy(d_B_.get(), B, sizeof B, cudaMemcpyHostToDevice));
    std::memcpy(B_, B, sizeof B);
  }

  float frame(const unsigned char* gray, float exposure, float factor, PyramidIface& out, const unsigned char* bgr,
              unsigned char* bgr_out) override {
    TDM_CHECK(gray, "null argument");
    TDM_CHECK((bgr == nullptr) == (bgr_out == nullptr), "pass both bgr and bgr_out or neither");
    TDM_CHECK(out.width(0) == w_ && out.height(0) == h_, "pyramid level 0 size does not match the undistorter's w x h");
    TDM_CHECK(out.device() == device_, "pyramid and undistorter live on different devices");
    TDM_CUDA(cudaSetDevice(device_));
    const size_t n_org = (size_t)w_org_ * h_org_, n = (size_t)w_ * h_;
    const bool want_bgr = bgr != nullptr;
    if (want_bgr && !d_bgr_in_) {
      d_bgr_in_ = make_dev<unsigned char>(3 * n_org);
      d_bgr_out_ = make_dev<unsigned char>(3 * n);
      h_bgr_in_ = make_host<unsigned char>(3 * n_org);
      h_bgr_out_ = make_host<unsigned char>(3 * n);
    }
    const bool pin_gray = page_locked(gray), pin_bgr = want_bgr && page_locked(bgr), pin_out = want_bgr && page_locked(bgr_out);
    cudaStream_t st = (cudaStream_t)out.stream();
    TDM_CUDA(cudaStreamWaitEvent(st, done_.get(), 0));            // the previous frame (maybe on another pyramid) has left our buffers
    if (!pin_gray || (want_bgr && !pin_bgr)) TDM_CUDA(cudaEventSynchronize(uploaded_.get()));   // staging is free
    const unsigned char* g = gray;
    if (!pin_gray) { std::memcpy(h_raw_.get(), gray, n_org); g = h_raw_.get(); }
    TDM_CUDA(cudaMemcpyAsync(d_raw_.get(), g, n_org, cudaMemcpyHostToDevice, st));
    if (want_bgr) {
      const unsigned char* b = bgr;
      if (!pin_bgr) { std::memcpy(h_bgr_in_.get(), bgr, 3 * n_org); b = h_bgr_in_.get(); }
      TDM_CUDA(cudaMemcpyAsync(d_bgr_in_.get(), b, 3 * n_org, cudaMemcpyHostToDevice, st));
    }
    TDM_CUDA(cudaEventRecord(uploaded_.get(), st));

    // processFrame's branch (Undistort.cpp:220)
    const int ph = (!valid_ || exposure <= 0 || mode_ == 0) ? PH_FACTOR : mode_ == 2 ? PH_G_VIGNETTE : PH_G;
    auto launch = ph == PH_FACTOR ? launch_undistort_p<PH_FACTOR> : ph == PH_G ? launch_undistort_p<PH_G>
                                                                               : launch_undistort_p<PH_G_VIGNETTE>;
    launch(st, d_remap_.get(), d_raw_.get(), d_G_.get(), d_vinv_.get(), factor, out.device_input(),
           want_bgr ? d_bgr_in_.get() : nullptr, want_bgr ? d_bgr_out_.get() : nullptr, w_, h_, w_org_, h_org_);
    TDM_CUDA(cudaGetLastError());
    if (want_bgr) {
      TDM_CUDA(cudaMemcpyAsync(pin_out ? bgr_out : h_bgr_out_.get(), d_bgr_out_.get(), 3 * n, cudaMemcpyDeviceToHost, st));
      TDM_CUDA(cudaEventRecord(bgr_done_.get(), st));
    }
    out.build_device(gamma_weights_ ? d_B_.get() : nullptr);
    TDM_CUDA(cudaEventRecord(done_.get(), st));
    if (pin_gray || pin_bgr) TDM_CUDA(cudaEventSynchronize(uploaded_.get()));   // the caller's buffers are ours only during the call
    if (want_bgr) {
      TDM_CUDA(cudaEventSynchronize(bgr_done_.get()));
      if (!pin_out) std::memcpy(bgr_out, h_bgr_out_.get(), 3 * n);
    }
    return use_exposure_ ? exposure : 1.f;
  }
  int device() const override { return device_; }

 private:
  int device_;
  int w_ = 0, h_ = 0, w_org_ = 0, h_org_ = 0, mode_ = 0;
  bool use_exposure_ = false, gamma_weights_ = false, valid_ = false;
  float G_[256] = {}, B_[256] = {};
  Event uploaded_, done_, bgr_done_;
  DevPtr<float> d_G_, d_B_, d_vinv_;
  DevPtr<float2> d_remap_;
  DevPtr<unsigned char> d_raw_, d_bgr_in_, d_bgr_out_;
  HostPtr<unsigned char> h_raw_, h_bgr_in_, h_bgr_out_;
};

UndistortIface* make_undistort(const tdm_undistort_settings& s, int device) { return new UndistortImpl(s, device); }

}  // namespace tdm
