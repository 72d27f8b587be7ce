// Test infrastructure (never linked into the product): harness around code of the REFERENCE,
//   ImmaturePoint::ImmaturePoint         tandem/src/FullSystem/ImmaturePoint.cpp:32-61
//   ImmaturePoint::traceOn               tandem/src/FullSystem/ImmaturePoint.cpp:75-414
//   getInterpolatedElement33 / 31 / 33BiLin   tandem/src/util/globalFuncs.h:75-89, 126-140, 166-188
//   staticPattern                        tandem/src/util/settings.cpp:216-266
// which oracle/ref_build_trace.mk cuts out of the files where they lie (sed line ranges -> oracle/_ref/gen_trace/*.inc,
// git-ignored build output) and compiles here, unmodified, against stand-ins for the DSO types they touch and the stand-in
// Eigen of oracle/ref_shim/trace_eigen.  Purpose: pin oracle/trace_oracle.c against the reference's own statements.
// The points of each host slot persist between calls as ImmaturePoint objects, as host->immaturePoints do.  Images are copied
// into buffers with a margin, so a read outside the image stays inside the allocation (the pinned cases have none).
#include <cassert>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <utility>
#include <vector>

#include <Eigen/Dense>   // oracle/ref_shim/trace_eigen

#define EIGEN_ALWAYS_INLINE inline
#define PYR_LEVELS 6
#define MAX_RES_PER_POINT 8
#define patternNum 8
#define patternP staticPattern[8]

typedef Eigen::Matrix<float, 2, 1> Vec2f;
typedef Eigen::Matrix<float, 3, 1> Vec3f;
typedef Eigen::Matrix<float, 2, 2> Mat22f;
typedef Eigen::Matrix<float, 3, 3> Mat33f;

namespace dso {

int wG[PYR_LEVELS], hG[PYR_LEVELS];
float setting_maxPixSearch, setting_trace_stepsize, setting_trace_GNThreshold, setting_trace_extraSlackOnTH,
    setting_trace_slackInterval, setting_trace_minImprovementFactor, setting_huberTH, setting_outlierTH,
    setting_outlierTHSumComponent, setting_overallEnergyTHWeight;
int setting_minTraceTestRadius, setting_trace_GNIterations;

#include "_ref/gen_trace/pattern.inc"
#include "_ref/gen_trace/interp33.inc"
#include "_ref/gen_trace/interp31.inc"
#include "_ref/gen_trace/interp33bilin.inc"

enum ImmaturePointStatus { IPS_GOOD = 0, IPS_OOB, IPS_OUTLIER, IPS_SKIPPED, IPS_BADCONDITION, IPS_UNINITIALIZED };   // ImmaturePoint.h:46-52
struct FrameShell { int id = 0; };
struct FrameHessian {
  Eigen::Vector3f* dI;
  FrameShell* shell;
};
struct CalibHessian {};

class ImmaturePoint {   // the members of ImmaturePoint.h:56-90 that the two functions touch
 public:
  ImmaturePoint(int u_, int v_, FrameHessian* host_, float type, CalibHessian* HCalib);
  ImmaturePointStatus traceOn(FrameHessian* frame, const Mat33f& hostToFrame_KRKi, const Vec3f& hostToFrame_Kt,
                              const Vec2f& hostToFrame_affine, CalibHessian* HCalib, bool debugPrint = false);
  float color[MAX_RES_PER_POINT];
  float weights[MAX_RES_PER_POINT];
  Mat22f gradH;
  float energyTH;
  float u, v;
  FrameHessian* host;
  float quality;
  float my_type;
  float idepth_min;
  float idepth_max;
  ImmaturePointStatus lastTraceStatus;
  Vec2f lastTraceUV;
  float lastTracePixelInterval;
  float idepth_GT;
};

#include "_ref/gen_trace/ctor.inc"
#include "_ref/gen_trace/trace_on.inc"

}  // namespace dso

using namespace dso;

namespace {
std::map<int, std::vector<ImmaturePoint*>> g_points;
FrameShell g_shell;

void set_settings(int w, int h, const float* s) {
  wG[0] = w; hG[0] = h;
  setting_maxPixSearch = s[0]; setting_trace_stepsize = s[1]; setting_trace_GNThreshold = s[2];
  setting_trace_extraSlackOnTH = s[3]; setting_trace_slackInterval = s[4]; setting_trace_minImprovementFactor = s[5];
  setting_huberTH = s[6]; setting_outlierTH = s[7]; setting_outlierTHSumComponent = s[8]; setting_overallEnergyTHWeight = s[9];
  setting_minTraceTestRadius = (int)s[10]; setting_trace_GNIterations = (int)s[11];
}

struct Image {   // level-0 (I, dx, dy) with a margin of rows on both sides
  std::vector<Eigen::Vector3f> buf;
  FrameHessian fh;
  Image(int w, int h, const float* dI) : buf((size_t)w * (h + 8)) {
    for (auto& e : buf) e = Eigen::Vector3f(NAN, NAN, NAN);
    std::memcpy(buf.data() + 4 * (size_t)w, dI, sizeof(float) * 3 * (size_t)w * h);
    fh.dI = buf.data() + 4 * (size_t)w;
    fh.shell = &g_shell;
  }
};
std::map<int, Image*> g_hosts;
}  // namespace

extern "C" {

void ref_trace_reset() {
  for (auto& kv : g_points) for (ImmaturePoint* p : kv.second) delete p;
  g_points.clear();
  for (auto& kv : g_hosts) delete kv.second;
  g_hosts.clear();
}

// FullSystem::makeNewTraces' loop (FullSystem.cpp:1639-1644): construct, keep the points with a finite energyTH
int ref_trace_add(int w, int h, const float* dI, const float* s, int slot, int n, const int* u, const int* v, const float* type) {
  set_settings(w, h, s);
  if (!g_hosts.count(slot)) g_hosts[slot] = new Image(w, h, dI);
  CalibHessian calib;
  int m = 0;
  for (int i = 0; i < n; ++i) {
    ImmaturePoint* p = new ImmaturePoint(u[i], v[i], &g_hosts[slot]->fh, type[i], &calib);
    if (!std::isfinite(p->energyTH)) { delete p; continue; }
    g_points[slot].push_back(p);
    ++m;
  }
  return m;
}

// traceNewCoarse's inner loop (FullSystem.cpp:671-672) for one host slot
void ref_trace_trace(int w, int h, const float* dI, const float* s, int slot, const float* K, const float* Kt, const float* aff) {
  set_settings(w, h, s);
  Image frame(w, h, dI);
  Mat33f KRKi;
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) KRKi(r, c) = K[3 * r + c];
  Vec3f kt(Kt[0], Kt[1], Kt[2]);
  Vec2f af(aff[0], aff[1]);
  CalibHessian calib;
  for (ImmaturePoint* p : g_points[slot]) p->traceOn(&frame.fh, KRKi, kt, af, &calib, false);
}

int ref_trace_count(int slot) { return (int)g_points[slot].size(); }

// point fields (u, v, type, energyTH, color 8, weights 8, gradH 4 row-major) and trace state (idepth_min, idepth_max, quality,
// status, uv 2, interval) of the points of a slot
void ref_trace_get(int slot, float* u, float* v, float* type, float* energyTH, float* color, float* weights, float* gradH,
                   float* idepth_min, float* idepth_max, float* quality, int* status, float* uv, float* interval) {
  const std::vector<ImmaturePoint*>& ps = g_points[slot];
  for (size_t i = 0; i < ps.size(); ++i) {
    const ImmaturePoint* p = ps[i];
    u[i] = p->u; v[i] = p->v; type[i] = p->my_type; energyTH[i] = p->energyTH;
    for (int k = 0; k < 8; ++k) { color[8 * i + k] = p->color[k]; weights[8 * i + k] = p->weights[k]; }
    gradH[4 * i] = p->gradH(0, 0); gradH[4 * i + 1] = p->gradH(0, 1); gradH[4 * i + 2] = p->gradH(1, 0); gradH[4 * i + 3] = p->gradH(1, 1);
    idepth_min[i] = p->idepth_min; idepth_max[i] = p->idepth_max; quality[i] = p->quality; status[i] = (int)p->lastTraceStatus;
    uv[2 * i] = p->lastTraceUV[0]; uv[2 * i + 1] = p->lastTraceUV[1]; interval[i] = p->lastTracePixelInterval;
  }
}

}  // extern "C"
