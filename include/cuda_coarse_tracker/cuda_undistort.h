// DSO's per-frame input on the device (n11, include/tandem_b200.h): PhotometricUndistorter::processFrame, Undistort::undistort's
// remap (tandem/src/util/Undistort.cpp), the dataset reader's BGR remap and makeImages' gamma weights, from the raw 8-bit frame
// into the frame's tdm_pyramid.  The camera's gamma state B lives here: FullSystem::setGammaFunction also calls setGamma.
// INTEGRATION.md shows the call sites.  Owns one tdm_undistort handle; not copyable.
#ifndef TDM_CUDA_UNDISTORT_H
#define TDM_CUDA_UNDISTORT_H

struct tdm_undistort;   // include/tandem_b200.h
struct tdm_pyramid;

class CudaUndistort {
 public:
  // Undistort's tables (get_remapX / get_remapY, w*h each; both null: passthrough), the photometric calibration file's first
  // line (n_response floats, or null) and the vignette image (w_org*h_org pixels, or null), and the reference's settings
  // setting_photometricCalibration, setting_useExposure and setting_gammaWeightsPixelSelect.  Every array is copied.
  CudaUndistort(int w_org, int h_org, int w, int h, const float *remapX, const float *remapY, const float *response,
                int n_response, const unsigned short *vignette, int photometricCalibration = 2, bool useExposure = true,
                bool gammaWeights = true, int device = 0);
  ~CudaUndistort();
  CudaUndistort(const CudaUndistort &) = delete;
  CudaUndistort &operator=(const CudaUndistort &) = delete;

  // PhotometricUndistorter::getG(): fills G[256] and returns true when the calibration is valid; false (G untouched) otherwise
  bool getG(float G[256]) const;
  // FullSystem::setGammaFunction(Binv) on this camera's B; null is a no-op
  void setGamma(const float *Binv);
  // Undistort::undistort<unsigned char>(raw, exposure, 0, factor) + makeImages into pyramid (asynchronous, ordered like
  // tdm_pyramid_build); with bgr (w_org*h_org*3) and bgr_out (w*h*3) also the BGR remap, which has landed on return.
  // Returns the frame's exposure_time.
  float undistort(const unsigned char *gray, float exposure, tdm_pyramid *pyramid, float factor = 1,
                  const unsigned char *bgr = nullptr, unsigned char *bgr_out = nullptr);
  tdm_undistort *handle() const { return handle_; }

 private:
  tdm_undistort *handle_ = nullptr;
};

#endif
