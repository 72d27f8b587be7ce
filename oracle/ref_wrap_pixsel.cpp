// Test infrastructure (never linked into the product): harness around code of the REFERENCE,
//   PixelSelector (class declaration)     tandem/src/FullSystem/PixelSelector2.h:32-66
//   PixelSelector::PixelSelector .. select   tandem/src/FullSystem/PixelSelector2.cpp:41-438
// which oracle/ref_build_pixsel.mk cuts out of the files where they lie (sed line ranges -> oracle/_ref/gen_pixsel/*.inc,
// git-ignored build output) and compiles here, unmodified, against stand-ins for the DSO types they touch and the stand-in
// Eigen of oracle/ref_shim/pixsel_eigen.  Purpose: pin oracle/pixsel_oracle.c against the reference's own statements.
//
// What the harness adds around the cut:
// - thsSmoothed is zero-filled once after construction, so its entries at and beyond w32 * h32 (never written by makeHists,
//   read by select where w % 32 >= 6 or h % 32 >= 4) hold 0, the value the library defines for them.
// - The counts and the potential of every select are recorded where select builds its return value (the Eigen::Vector3i
//   constructor below); the class's private members are opened to the harness for the pattern and thsSmoothed.
// - makeHists runs before every makeMaps, so a new image never meets the reference's pointer-equality cache.
#include <algorithm>
#include <cassert>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include <Eigen/Dense>   // oracle/ref_shim/pixsel_eigen

#define PYR_LEVELS 6
#define EIGEN_MAKE_ALIGNED_OPERATOR_NEW

typedef Eigen::Matrix<float, 2, 1> Vec2f;

namespace dso {
class PixelSelector;
}
namespace {
dso::PixelSelector* g_sel = nullptr;
int g_selects = 0, g_last[4] = {0, 0, 0, 0};
}  // namespace

namespace Eigen {
// select's `return Eigen::Vector3i(n2,n3,n4);` is the only three-int construction in the cut: record it
template <>
Matrix<int, 3, 1>::Matrix(int a, int b, int c);
}  // namespace Eigen

namespace dso {

int wG[PYR_LEVELS], hG[PYR_LEVELS];
float setting_minGradHistCut, setting_minGradHistAdd, setting_gradDownweightPerLevel;
bool setting_selectDirectionDistribution;

struct FrameHessian {
  Eigen::Vector3f* dI;
  float* absSquaredGrad[PYR_LEVELS];
};

// the plot branch of makeMaps (display only; the harness never plots)
struct Vec3b {
  Vec3b() {}
  Vec3b(float, float, float) {}
};
struct MinimalImageB3 {
  Vec3b px;
  MinimalImageB3(int, int) {}
  Vec3b& at(int) { return px; }
  void setPixelCirc(int, int, Vec3b) {}
};
namespace IOWrap {
inline void displayImage(const char*, const MinimalImageB3*, bool = false) {}
}  // namespace IOWrap

#define private public
#include "_ref/gen_pixsel/class.inc"
#undef private
#include "_ref/gen_pixsel/selector.inc"

}  // namespace dso

namespace Eigen {
template <>
Matrix<int, 3, 1>::Matrix(int a, int b, int c) {
  d[0] = a; d[1] = b; d[2] = c;
  g_last[0] = a; g_last[1] = b; g_last[2] = c; g_last[3] = g_sel->currentPotential;
  ++g_selects;
}
}  // namespace Eigen

using namespace dso;

extern "C" {

void* ref_pixsel_create(int w, int h) {
  for (int l = 0; l < PYR_LEVELS; ++l) { wG[l] = w >> l; hG[l] = h >> l; }
  PixelSelector* s = new PixelSelector(w, h);
  std::memset(s->thsSmoothed, 0, sizeof(float) * ((w / 32) * (h / 32) + 100));
  return s;
}
void ref_pixsel_destroy(void* s) { delete (PixelSelector*)s; }
void ref_pixsel_pattern(void* s, int n, unsigned char* out) { std::memcpy(out, ((PixelSelector*)s)->randomPattern, n); }
int ref_pixsel_get_potential(void* s) { return ((PixelSelector*)s)->currentPotential; }
void ref_pixsel_set_potential(void* s, int p) { ((PixelSelector*)s)->currentPotential = p; }

// makeMaps(fh, map_out, density, recursionsLeft, false, thFactor) on level 0 (I, dx, dy) and absSquaredGrad of levels 0..2;
// settings: minGradHistCut, minGradHistAdd, gradDownweightPerLevel, selectDirectionDistribution.  info: n2, n3, n4 and the
// potential of the last select, and how many selects ran.  Returns makeMaps' value.
int ref_pixsel_make_maps(void* sp, int w, int h, float* dI, float* ag0, float* ag1, float* ag2, const float* settings,
                         float density, int recursions_left, float th_factor, float* map_out, int* info) {
  PixelSelector* s = (PixelSelector*)sp;
  for (int l = 0; l < PYR_LEVELS; ++l) { wG[l] = w >> l; hG[l] = h >> l; }
  setting_minGradHistCut = settings[0]; setting_minGradHistAdd = settings[1]; setting_gradDownweightPerLevel = settings[2];
  setting_selectDirectionDistribution = settings[3] != 0.f;
  FrameHessian fh;
  fh.dI = (Eigen::Vector3f*)dI;
  fh.absSquaredGrad[0] = ag0; fh.absSquaredGrad[1] = ag1; fh.absSquaredGrad[2] = ag2;
  g_sel = s;
  g_selects = 0;
  s->makeHists(&fh);
  const int r = s->makeMaps(&fh, map_out, density, recursions_left, false, th_factor);
  s->gradHistFrame = nullptr;
  for (int k = 0; k < 4; ++k) info[k] = g_last[k];
  info[4] = g_selects;
  return r;
}

}  // extern "C"
