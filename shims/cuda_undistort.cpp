// CudaUndistort over the tandem_b200 C ABI.  Errors throw std::runtime_error, as the tracker shim's do.
#include "cuda_coarse_tracker/cuda_undistort.h"

#include <stdexcept>
#include <string>

#include "tandem_b200.h"

static void chk(int rc, const char *where) {
  if (rc != TDM_OK) throw std::runtime_error(std::string(where) + ": " + tdm_last_error());
}

CudaUndistort::CudaUndistort(int w_org, int h_org, int w, int h, const float *remapX, const float *remapY, const float *response,
                             int n_response, const unsigned short *vignette, int photometricCalibration, bool useExposure,
                             bool gammaWeights, int device) {
  tdm_undistort_settings s;
  s.w_org = w_org; s.h_org = h_org; s.w = w; s.h = h;
  s.remap_x = remapX; s.remap_y = remapY;
  s.response = response; s.n_response = n_response;
  s.vignette = vignette;
  s.photometric_calibration = photometricCalibration;
  s.use_exposure = useExposure ? 1 : 0;
  s.gamma_weights = gammaWeights ? 1 : 0;
  chk(tdm_undistort_create(&s, device, &handle_), "CudaUndistort");
}

CudaUndistort::~CudaUndistort() { tdm_undistort_destroy(handle_); }

bool CudaUndistort::getG(float G[256]) const {
  int valid = 0;
  chk(tdm_undistort_get_gamma(handle_, G, &valid), "CudaUndistort::getG");
  return valid != 0;
}

void CudaUndistort::setGamma(const float *Binv) { chk(tdm_undistort_set_gamma(handle_, Binv), "CudaUndistort::setGamma"); }

float CudaUndistort::undistort(const unsigned char *gray, float exposure, tdm_pyramid *pyramid, float factor,
                               const unsigned char *bgr, unsigned char *bgr_out) {
  float t = 0;
  chk(tdm_undistort_frame(handle_, gray, exposure, factor, pyramid, &t, bgr, bgr_out), "CudaUndistort::undistort");
  return t;
}
