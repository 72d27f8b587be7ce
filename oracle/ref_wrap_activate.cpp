// Test infrastructure (never linked into the product): harness around code of the REFERENCE,
//   FullSystem::optimizeImmaturePoint    tandem/src/FullSystem/FullSystemOptPoint.cpp:51-205
//   ImmaturePoint::linearizeResidual     tandem/src/FullSystem/ImmaturePoint.cpp:476-543
//   derive_idepth, projectPoint (both)   tandem/src/FullSystem/ResidualProjections.h:36-87
// and, so that the activated points are points the reference itself made and traced, n8's cut of
//   ImmaturePoint::ImmaturePoint / traceOn, getInterpolatedElement33 / 31 / 33BiLin, staticPattern
// which oracle/ref_build_activate.mk cuts out of the files where they lie (git-ignored build output) and compiles here,
// unmodified, against stand-ins for the DSO types they touch and n8's stand-in Eigen.  Purpose: pin
// oracle/activate_oracle.c against the reference's own statements.  The harness passes its own
// ImmaturePointTemporaryResidual array to every call and reads it back afterwards, so state_state / state_energy /
// state_NewState / state_NewEnergy are observable whatever the call returns.
#include <cassert>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <utility>
#include <vector>

#include <Eigen/Dense>   // oracle/ref_shim/trace_eigen

#define EIGEN_ALWAYS_INLINE inline
#define EIGEN_STRONG_INLINE inline
#define EIGEN_MAKE_ALIGNED_OPERATOR_NEW
#define PYR_LEVELS 6
#define MAX_RES_PER_POINT 8
#define patternNum 8
#define patternP staticPattern[8]
#define SCALE_IDEPTH 1.0f   // HessianBlocks.h:59

typedef Eigen::Matrix<float, 2, 1> Vec2f;
typedef Eigen::Matrix<float, 3, 1> Vec3f;
typedef Eigen::Matrix<float, 2, 2> Mat22f;
typedef Eigen::Matrix<float, 3, 3> Mat33f;

namespace dso {

int wG[PYR_LEVELS], hG[PYR_LEVELS];
float wM3G, hM3G;   // globalCalib.cpp:71-72
float setting_maxPixSearch, setting_trace_stepsize, setting_trace_GNThreshold, setting_trace_extraSlackOnTH,
    setting_trace_slackInterval, setting_trace_minImprovementFactor, setting_huberTH, setting_outlierTH,
    setting_outlierTHSumComponent, setting_overallEnergyTHWeight;
int setting_minTraceTestRadius, setting_trace_GNIterations;
float setting_minIdepthH_act;
int setting_GNItsOnPointActivation;

#include "_ref/gen_trace/pattern.inc"
#include "_ref/gen_trace/interp33.inc"
#include "_ref/gen_trace/interp31.inc"
#include "_ref/gen_trace/interp33bilin.inc"

enum ImmaturePointStatus { IPS_GOOD = 0, IPS_OOB, IPS_OUTLIER, IPS_SKIPPED, IPS_BADCONDITION, IPS_UNINITIALIZED };   // ImmaturePoint.h:46-52
enum ResState { IN = 0, OOB, OUTLIER };   // Residuals.h:47
struct FrameShell { int id = 0; };
struct FrameHessian;
struct FrameFramePrecalc {   // the members linearizeResidual reads (HessianBlocks.h)
  Mat33f PRE_RTll;
  Vec3f PRE_tTll;
  Vec2f PRE_aff_mode;
};
struct FrameHessian {
  Eigen::Vector3f* dI;
  FrameShell* shell;
  int idx;
  std::vector<FrameFramePrecalc> targetPrecalc;
};
struct CalibHessian {   // HessianBlocks.h:397-402, set as setValueScaled sets them
  float value_scaledf[4], value_scaledi[4];
  inline float& fxl() { return value_scaledf[0]; }
  inline float& fyl() { return value_scaledf[1]; }
  inline float& cxl() { return value_scaledf[2]; }
  inline float& cyl() { return value_scaledf[3]; }
  inline float& fxli() { return value_scaledi[0]; }
  inline float& fyli() { return value_scaledi[1]; }
};

struct ImmaturePointTemporaryResidual {   // ImmaturePoint.h:35-43
 public:
  ResState state_state;
  double state_energy;
  ResState state_NewState;
  double state_NewEnergy;
  FrameHessian* target;
};

class ImmaturePoint {   // the members of ImmaturePoint.h:56-101 that the cut functions touch
 public:
  ImmaturePoint(int u_, int v_, FrameHessian* host_, float type, CalibHessian* HCalib);
  ImmaturePointStatus traceOn(FrameHessian* frame, const Mat33f& hostToFrame_KRKi, const Vec3f& hostToFrame_Kt,
                              const Vec2f& hostToFrame_affine, CalibHessian* HCalib, bool debugPrint = false);
  double linearizeResidual(CalibHessian* HCalib, const float outlierTHSlack, ImmaturePointTemporaryResidual* tmpRes, float& Hdd,
                           float& bd, float idepth);
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

struct PointHessian;
struct PointFrameResidual {   // the members optimizeImmaturePoint touches (Residuals.h)
  PointFrameResidual(PointHessian* point_, FrameHessian* host_, FrameHessian* target_) : point(point_), host(host_), target(target_) {}
  void setState(ResState s) { state_state = s; }
  PointHessian* point;
  FrameHessian* host;
  FrameHessian* target;
  ResState state_state;
  double state_energy;
  ResState state_NewState;
  double state_NewEnergy;
};
struct PointHessian {   // the members optimizeImmaturePoint touches (HessianBlocks.h:465-...); the constructor keeps what it reads
  enum PtStatus { ACTIVE = 0, INACTIVE, OUTLIER, OOB, MARGINALIZED };
  PointHessian(const ImmaturePoint* const rawPoint, CalibHessian* Hcalib) : host(rawPoint->host), energyTH(rawPoint->energyTH) {}
  ~PointHessian() { for (PointFrameResidual* r : residuals) delete r; }
  void setIdepth(float idepth_) { idepth = idepth_; }
  void setIdepthZero(float idepth_) { idepth_zero = idepth_; }
  void setPointStatus(PtStatus s) { status = s; }
  FrameHessian* host;
  float energyTH;
  float idepth = NAN, idepth_zero = NAN;
  PtStatus status = INACTIVE;
  std::vector<PointFrameResidual*> residuals;
  std::pair<PointFrameResidual*, ResState> lastResiduals[2];
};

class FullSystem {   // the members optimizeImmaturePoint touches (FullSystem.h)
 public:
  PointHessian* optimizeImmaturePoint(ImmaturePoint* point, int minObs, ImmaturePointTemporaryResidual* residuals);
  std::vector<FrameHessian*> frameHessians;
  CalibHessian Hcalib;
  long int statistics_numActivatedPoints = 0;
};

#include "_ref/gen_activate/projections.inc"
#include "_ref/gen_trace/ctor.inc"
#include "_ref/gen_trace/trace_on.inc"
#include "_ref/gen_activate/linearize.inc"
#include "_ref/gen_activate/opt_point.inc"

}  // namespace dso

using namespace dso;

namespace {
std::map<int, std::vector<ImmaturePoint*>> g_points;
FrameShell g_shell;

void set_settings(int w, int h, const float* s) {
  wG[0] = w; hG[0] = h;
  wM3G = w - 3; hM3G = h - 3;
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
    fh.idx = 0;
  }
};
std::map<int, Image*> g_hosts;
}  // namespace

extern "C" {

void ref_act_reset() {
  for (auto& kv : g_points) for (ImmaturePoint* p : kv.second) delete p;
  g_points.clear();
  for (auto& kv : g_hosts) delete kv.second;
  g_hosts.clear();
}

// FullSystem::makeNewTraces' loop (FullSystem.cpp:1639-1644), appended to a slot
int ref_act_add(int w, int h, const float* dI, const float* s, int slot, int n, const int* u, const int* v, const float* type) {
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
void ref_act_trace(int w, int h, const float* dI, const float* s, int slot, const float* K, const float* Kt, const float* aff) {
  set_settings(w, h, s);
  Image frame(w, h, dI);
  Mat33f KRKi;
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) KRKi(r, c) = K[3 * r + c];
  Vec3f kt(Kt[0], Kt[1], Kt[2]);
  Vec2f af(aff[0], aff[1]);
  CalibHessian calib;
  for (ImmaturePoint* p : g_points[slot]) p->traceOn(&frame.fh, KRKi, kt, af, &calib, false);
}

int ref_act_count(int slot) { return (int)g_points[slot].size(); }

// activatePointsMT_Reductor (FullSystem.cpp:694-703) over the candidates: frames in frameHessians order, frame f's points in
// slot frame_slots[f] (-1: none), its level 0 dI[f]; precalc n x n x 14 (PRE_RTll row-major, PRE_tTll, PRE_aff_mode).
// Outputs per candidate: the return (1 PointHessian, 0, -1), the PointHessian's idepth (NaN unless 1), and per frame the
// four residual fields (-1 / NaN in the host's own column).
void ref_act_activate(int w, int h, int n_frames, const float* const* dI, const int* frame_slots, const float* precalc,
                      const float* calib4, float huber, float min_h, int gn_its, int n_cand, const int* cand_frame,
                      const int* cand_index, int min_obs, int* result, float* idepth, int* state, double* energy, int* new_state,
                      double* new_energy) {
  wG[0] = w; hG[0] = h;
  wM3G = w - 3; hM3G = h - 3;
  setting_huberTH = huber;
  setting_minIdepthH_act = min_h;
  setting_GNItsOnPointActivation = gn_its;
  std::vector<Image*> frames(n_frames);
  FullSystem fs;
  for (int f = 0; f < n_frames; ++f) {
    // a host's own image stays the one its points were made on (the same pixels as dI[f])
    frames[f] = frame_slots[f] >= 0 && g_hosts.count(frame_slots[f]) ? g_hosts[frame_slots[f]] : new Image(w, h, dI[f]);
    frames[f]->fh.idx = f;
    frames[f]->fh.targetPrecalc.assign(n_frames, FrameFramePrecalc());
    fs.frameHessians.push_back(&frames[f]->fh);
  }
  for (int f = 0; f < n_frames; ++f)
    for (int t = 0; t < n_frames; ++t) {
      const float* P = precalc + 14 * ((size_t)f * n_frames + t);
      FrameFramePrecalc& pc = frames[f]->fh.targetPrecalc[t];
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) pc.PRE_RTll(r, c) = P[3 * r + c];
      pc.PRE_tTll = Vec3f(P[9], P[10], P[11]);
      pc.PRE_aff_mode = Vec2f(P[12], P[13]);
    }
  fs.Hcalib.value_scaledf[0] = calib4[0]; fs.Hcalib.value_scaledf[1] = calib4[1];
  fs.Hcalib.value_scaledf[2] = calib4[2]; fs.Hcalib.value_scaledf[3] = calib4[3];
  fs.Hcalib.value_scaledi[0] = 1.0f / fs.Hcalib.value_scaledf[0];
  fs.Hcalib.value_scaledi[1] = 1.0f / fs.Hcalib.value_scaledf[1];
  for (int k = 0; k < n_cand; ++k) {
    ImmaturePoint* p = g_points[frame_slots[cand_frame[k]]][cand_index[k]];
    ImmaturePointTemporaryResidual tr[8];
    for (auto& r : tr) { r.state_state = r.state_NewState = OOB; r.state_energy = r.state_NewEnergy = -7; r.target = nullptr; }
    PointHessian* ph = fs.optimizeImmaturePoint(p, min_obs, tr);
    result[k] = ph == (PointHessian*)((long)(-1)) ? -1 : ph ? 1 : 0;
    idepth[k] = result[k] == 1 ? ph->idepth : NAN;
    for (int f = 0, i = 0; f < n_frames; ++f) {
      const size_t o = (size_t)k * n_frames + f;
      if (f == cand_frame[k]) { state[o] = new_state[o] = -1; energy[o] = new_energy[o] = NAN; continue; }
      assert(tr[i].target == &frames[f]->fh);
      state[o] = tr[i].state_state; new_state[o] = tr[i].state_NewState;
      energy[o] = tr[i].state_energy; new_energy[o] = tr[i].state_NewEnergy;
      ++i;
    }
    if (result[k] == 1) {   // the PointHessian the reductor would hand over; its residuals follow the IN columns
      int nin = 0;
      for (int f = 0; f < n_frames; ++f) nin += state[(size_t)k * n_frames + f] == IN;
      if ((int)ph->residuals.size() != nin || ph->idepth != ph->idepth_zero) result[k] = 99;   // flags a harness error
      delete ph;
    }
  }
  for (int f = 0; f < n_frames; ++f)
    if (!(frame_slots[f] >= 0 && g_hosts.count(frame_slots[f]))) delete frames[f];
}

}  // extern "C"
