// Test infrastructure (never linked into the product): harness around code of the REFERENCE,
//   PhotometricUndistorter, Undistort (class declarations)   tandem/src/util/Undistort.h:40-64, :67-109
//   PhotometricUndistorter's constructor and destructor     tandem/src/util/Undistort.cpp:50-185
//   PhotometricUndistorter::processFrame                    tandem/src/util/Undistort.cpp:213-252
//   Undistort::undistort                                    tandem/src/util/Undistort.cpp:393-490
//   getImageBGR_8UC3_undistort_internal                     tandem/src/util/DatasetReader.h:354-400
//   FullSystem::setGammaFunction                            tandem/src/FullSystem/FullSystem.cpp:232-253
//   CalibHessian::getBGradOnly                              tandem/src/FullSystem/HessianBlocks.h:446-452
//   FrameHessian::makeImages                                tandem/src/FullSystem/HessianBlocks.cpp:128-191
// which oracle/ref_build_undistort.mk cuts out of the files where they lie (sed line ranges -> oracle/_ref/gen_undistort/*.inc,
// git-ignored build output) and compiles here, unmodified, against stand-ins for the DSO types and functions they touch and
// the stand-in Eigen of tests/cpp/eigen_stub.  Purpose: pin oracle/undistort_oracle.c against the reference's own statements.
//
// What the harness adds around the cut:
// - The response goes through a file (the constructor reads it with std::ifstream); the vignette and the BGR frame come from
//   the IOWrap stand-ins, which return the case's buffers.
// - Undistort's destructor and applyBlurNoise are stand-ins (outside the cut); applyBlurNoise returns at once, as the
//   reference's does for benchmark_varBlurNoise == 0.  benchmark_varNoise is 0, so undistort's noise branch never runs and the
//   interpolation helpers it names are stand-ins that are never called.
// - Rows 0 and h-1 of (dx, dy, absSquaredGrad) are never written by makeImages; the harness reports 0 there, the value the
//   library defines (as oracle/ref_wrap_front.cpp does).
#include <cassert>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <iterator>
#include <sstream>
#include <string>
#include <vector>

#include <Eigen/Dense>   // tests/cpp/eigen_stub

namespace Eigen {
typedef Matrix<int, 2, 1> Vector2i;   // Undistort::getSize / getOriginalSize
}

#define PYR_LEVELS 6
#define EIGEN_MAKE_ALIGNED_OPERATOR_NEW
#define EIGEN_STRONG_INLINE inline

namespace dso {

typedef Eigen::Matrix<double, 3, 3> Mat33;
typedef Eigen::Matrix<double, 1, 1> VecX;   // Undistort::parsOrg; the cut never reads it

int setting_photometricCalibration = 2;
bool setting_useExposure = true;
int setting_gammaWeightsPixelSelect = 1;
float benchmark_varNoise = 0, benchmark_varBlurNoise = 0;
int benchmark_noiseGridsize = 3;
int wG[PYR_LEVELS], hG[PYR_LEVELS];
int pyrLevelsUsed = 0;

template <typename T>
class MinimalImage {
 public:
  int w, h;
  T* data;
  MinimalImage(int w_, int h_) : w(w_), h(h_) { data = new T[w * h]; }
  ~MinimalImage() { delete[] data; }
  T& at(int i) { return data[i]; }
};
typedef MinimalImage<unsigned char> MinimalImageB;

class ImageAndExposure {
 public:
  float* image;
  int w, h;
  double timestamp;
  float exposure_time;
  ImageAndExposure(int w_, int h_, double timestamp_ = 0) : w(w_), h(h_), timestamp(timestamp_) {
    image = new float[w * h];
    exposure_time = 1;
  }
  ~ImageAndExposure() { delete[] image; }
  void copyMetaTo(ImageAndExposure& other) { other.exposure_time = exposure_time; }
};

inline float getInterpolatedElement11BiCub(const float*, float, float, int) { return 0; }
inline float getInterpolatedElement(const float*, float, float, int) { return 0; }

namespace IOWrap {
const unsigned short* g_vignette = nullptr;
int g_vignette_bits = 16, g_vw = 0, g_vh = 0;
const unsigned char* g_bgr = nullptr;
MinimalImage<unsigned short>* readImageBW_16U(std::string) {
  if (!g_vignette || g_vignette_bits != 16) return 0;
  auto* m = new MinimalImage<unsigned short>(g_vw, g_vh);
  std::memcpy(m->data, g_vignette, sizeof(unsigned short) * g_vw * g_vh);
  return m;
}
MinimalImageB* readImageBW_8U(std::string) {
  if (!g_vignette || g_vignette_bits != 8) return 0;
  auto* m = new MinimalImageB(g_vw, g_vh);
  for (int i = 0; i < g_vw * g_vh; ++i) m->data[i] = (unsigned char)g_vignette[i];
  return m;
}
unsigned char* readImageBGR_8UC3(std::string, int, int) { return const_cast<unsigned char*>(g_bgr); }
}  // namespace IOWrap

#define private public
#define protected public
#include "_ref/gen_undistort/photometric_class.inc"
#include "_ref/gen_undistort/undistort_class.inc"
#undef private
#undef protected
#include "_ref/gen_undistort/photometric_ctor.inc"
#include "_ref/gen_undistort/process_frame.inc"
#include "_ref/gen_undistort/undistort.inc"

Undistort::~Undistort() {}
void Undistort::applyBlurNoise(float*) const {}
struct HarnessUndistort : Undistort {
  void distortCoordinates(float*, float*, float*, float*, int) const override {}
};

struct CalibHessian {
  float Binv[256];
  float B[256];
#include "_ref/gen_undistort/bgrad.inc"
};
struct FullSystem {
  CalibHessian Hcalib;
  void setGammaFunction(float* BInv);
};
#include "_ref/gen_undistort/set_gamma.inc"

struct FrameHessian {
  Eigen::Vector3f* dI = nullptr;
  Eigen::Vector3f* dIp[PYR_LEVELS] = {};
  float* absSquaredGrad[PYR_LEVELS] = {};
  void makeImages(float* color, CalibHessian* HCalib);
};
#include "_ref/gen_undistort/make_images.inc"

struct ImageFolderReader {
  bool isZipped = false;
  std::vector<std::string> files{"frame"};
  int widthOrg = 0, heightOrg = 0, width = 0, height = 0;
#include "_ref/gen_undistort/bgr.inc"
};

}  // namespace dso

using namespace dso;

namespace {
struct Harness {
  HarnessUndistort u;
  FullSystem fs;
  ImageFolderReader reader;
  std::vector<float> rx, ry;
  int mode, use_exposure, gamma_weights;
};
void apply_settings(const Harness& H) {
  setting_photometricCalibration = H.mode;
  setting_useExposure = H.use_exposure != 0;
  setting_gammaWeightsPixelSelect = H.gamma_weights;
}
}  // namespace

extern "C" {

// remap_x NULL: passthrough.  response (n_response floats) is written to response_file for the constructor; vignette
// (w_org*h_org, vignette_bits 8 or 16) NULL: none.
void* ref_und_create(int w_org, int h_org, int w, int h, const float* remap_x, const float* remap_y, const float* response,
                     int n_response, const unsigned short* vignette, int vignette_bits, int mode, int use_exposure,
                     int gamma_weights, const char* response_file) {
  Harness* H = new Harness;
  H->mode = mode; H->use_exposure = use_exposure; H->gamma_weights = gamma_weights;
  apply_settings(*H);
  std::string file;
  if (response) {
    FILE* f = std::fopen(response_file, "w");
    for (int i = 0; i < n_response; ++i) std::fprintf(f, "%.9g ", response[i]);
    std::fprintf(f, "\n");
    std::fclose(f);
    file = response_file;
  }
  IOWrap::g_vignette = vignette; IOWrap::g_vignette_bits = vignette_bits; IOWrap::g_vw = w_org; IOWrap::g_vh = h_org;
  Undistort& u = H->u;
  u.w = w; u.h = h; u.wOrg = w_org; u.hOrg = h_org;
  u.passthrough = remap_x == nullptr;
  if (remap_x) {
    H->rx.assign(remap_x, remap_x + (size_t)w * h);
    H->ry.assign(remap_y, remap_y + (size_t)w * h);
  }
  u.remapX = H->rx.data(); u.remapY = H->ry.data();
  u.photometricUndist = new PhotometricUndistorter(file, "", vignette ? "vignette" : "", w_org, h_org);
  IOWrap::g_vignette = nullptr;
  for (int i = 0; i < 256; i++) H->fs.Hcalib.Binv[i] = H->fs.Hcalib.B[i] = i;   // HessianBlocks.h:392
  H->reader.widthOrg = w_org; H->reader.heightOrg = h_org; H->reader.width = w; H->reader.height = h;
  return H;
}
void ref_und_destroy(void* h) {
  Harness* H = (Harness*)h;
  delete H->u.photometricUndist;
  delete H;
}
// getG(): returns valid; G receives the 256 entries when valid.  G_member (may be NULL) the member array whatever valid is.
int ref_und_get_gamma(void* h, float* G, float* G_member) {
  Harness* H = (Harness*)h;
  float* g = H->u.photometricUndist->getG();
  if (g) std::memcpy(G, g, 256 * sizeof(float));
  if (G_member) std::memcpy(G_member, H->u.photometricUndist->G, 256 * sizeof(float));
  return g != 0;
}
void ref_und_set_gamma(void* h, float* binv, float* B_out) {
  Harness* H = (Harness*)h;
  H->fs.setGammaFunction(binv);
  std::memcpy(B_out, H->fs.Hcalib.B, sizeof(float) * 256);
}
// Undistort::undistort<unsigned char>, then makeImages of `levels` levels with &Hcalib (dI / absgrad: levels concatenated as
// in oracle/front_oracle.c), and with bgr the BGR remap (passthrough: a copy).
void ref_und_frame(void* h, const unsigned char* gray, float exposure, float factor, const unsigned char* bgr, int levels,
                   float* image_out, float* exposure_time, unsigned char* bgr_out, float* dI_out, float* absgrad_out) {
  Harness* H = (Harness*)h;
  apply_settings(*H);
  Undistort& u = H->u;
  MinimalImageB raw(u.wOrg, u.hOrg);
  std::memcpy(raw.data, gray, (size_t)u.wOrg * u.hOrg);
  ImageAndExposure* r = u.undistort<unsigned char>(&raw, exposure, 0, factor);
  std::memcpy(image_out, r->image, sizeof(float) * u.w * u.h);
  *exposure_time = r->exposure_time;

  pyrLevelsUsed = levels;
  for (int l = 0; l < PYR_LEVELS; ++l) { wG[l] = u.w >> l; hG[l] = u.h >> l; }
  FrameHessian fh;
  fh.makeImages(r->image, &H->fs.Hcalib);
  size_t off = 0;
  for (int l = 0; l < levels; ++l) {
    const size_t n = (size_t)wG[l] * hG[l];
    for (size_t i = 0; i < n; ++i) {
      const bool border = i < (size_t)wG[l] || i >= (size_t)wG[l] * (hG[l] - 1);
      dI_out[3 * (off + i)] = fh.dIp[l][i][0];
      dI_out[3 * (off + i) + 1] = border ? 0.f : fh.dIp[l][i][1];
      dI_out[3 * (off + i) + 2] = border ? 0.f : fh.dIp[l][i][2];
      absgrad_out[off + i] = border ? 0.f : fh.absSquaredGrad[l][i];
    }
    delete[] fh.dIp[l];
    delete[] fh.absSquaredGrad[l];
    off += n;
  }
  delete r;

  if (bgr) {
    if (u.passthrough) {
      std::memcpy(bgr_out, bgr, 3 * (size_t)u.w * u.h);
    } else {
      IOWrap::g_bgr = bgr;
      unsigned char* o = H->reader.getImageBGR_8UC3_undistort_internal(0, u.remapX, u.remapY);
      std::memcpy(bgr_out, o, 3 * (size_t)u.w * u.h);
      std::free(o);
    }
  }
}

}  // extern "C"
