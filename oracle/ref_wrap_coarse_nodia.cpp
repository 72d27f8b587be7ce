// Test infrastructure (never linked into the product): harness around two function bodies of the REFERENCE,
//   CoarseTracker::makeCoarseDepthL0      tandem/src/FullSystem/CoarseTracker.cpp:148-374
//   get_idepth_quantile                   tandem/src/tandem/tandem_backend.cpp:354-361
// which oracle/ref_build_coarse_nodia.mk cuts out of the files where they lie (sed line ranges -> oracle/_ref/gen_nodia/*.inc,
// git-ignored build output) and compiles here, unmodified, against stand-ins for the DSO classes the first one touches and the
// stand-in Eigen of tests/cpp/eigen_stub.  Purpose: pin oracle/coarse_nodia_oracle.c (the undilated level-0 cloud pc_*_nodia
// and MVSNet's depth-range quantile over it) against the reference's own statements.
// The stand-ins are those of oracle/ref_wrap_coarse_ref.cpp (one FrameHessian holding the points in input order, every
// monocular point with a residual in state IN; buffers allocated per call with one zero element before and behind each
// weight image), except that pc_u/v/idepth/color_nodia live in the caller's buffer and persist across calls, as
// CoarseTracker's members do.
#include <algorithm>
#include <cassert>
#include <cmath>
#include <cstring>
#include <utility>
#include <vector>

#include <Eigen/Dense>   // tests/cpp/eigen_stub

#define PYR_LEVELS 6
typedef Eigen::Matrix<float, 3, 1> Vec3f;

static int pyrLevelsUsed = 0;

enum ResState { IN = 0, OOB, OUTLIER };   // Residuals.h:47
struct EFResidual { bool isActive() const { return true; } };
struct EFPoint { float HdiF; };
struct FrameHessian;
struct PointHessian;
struct PointFrameResidual {
  EFResidual* efResidual;
  FrameHessian* target;
  PointHessian* point;
  Vec3f centerProjectedTo;
};
struct PointHessian {
  float u, v, idepth, idepth_hessian;
  EFPoint* efPoint;
  std::pair<PointFrameResidual*, ResState> lastResiduals[2];
};
struct FrameHessian {
  std::vector<PointHessian*> pointHessians;
  Eigen::Vector3f* dIp[PYR_LEVELS] = {};
};

class CoarseTracker {
 public:
  void makeCoarseDepthL0(std::vector<FrameHessian*> frameHessians, bool rgbd_init);
  int w[PYR_LEVELS], h[PYR_LEVELS];
  float* idepth[PYR_LEVELS];
  float* weightSums[PYR_LEVELS];
  float* weightSums_bak[PYR_LEVELS];
  float *pc_u[PYR_LEVELS], *pc_v[PYR_LEVELS], *pc_idepth[PYR_LEVELS], *pc_color[PYR_LEVELS];
  int pc_n[PYR_LEVELS];
  float *idepth_nodia, *depth_rel_var;
  float *pc_u_nodia, *pc_v_nodia, *pc_idepth_nodia, *pc_color_nodia;
  int pc_n_nodia;
  FrameHessian* lastRef;
};

#include "_ref/gen_nodia/make_coarse_depth.inc"   // CoarseTracker.cpp:148-374, verbatim
#include "_ref/gen_nodia/idepth_quantile.inc"     // tandem_backend.cpp:354-361, verbatim

extern "C" {

// gray: levels concatenated (level l: wl*hl floats, dIp[l][i][0]); pc_nodia: pc_u/v/idepth/color_nodia, 4 x w0*h0 floats,
// read and written; *pc_n_nodia_out receives pc_n_nodia.  The per-level outputs of the call are discarded.
int ref_make_coarse_depth_nodia(int w0, int h0, int levels, int rgbd, int n, const float* pu, const float* pv, const float* pid,
                                const float* phs, const float* gray, float* pc_nodia, int* pc_n_nodia_out) {
  if (levels < 1 || levels > 5) return -1;
  pyrLevelsUsed = levels;
  CoarseTracker ct;
  std::vector<std::vector<float>> bufs;
  std::vector<std::vector<Eigen::Vector3f>> grays(levels);
  size_t off = 0;
  FrameHessian fh;
  for (int l = 0; l < levels; ++l) {
    const int wl = w0 >> l, hl = h0 >> l;
    const size_t nl = (size_t)wl * hl;
    ct.w[l] = wl; ct.h[l] = hl;
    bufs.emplace_back(nl + 2, 0.f); ct.idepth[l] = bufs.back().data() + 1;
    bufs.emplace_back(nl + 2, 0.f); ct.weightSums[l] = bufs.back().data() + 1;
    bufs.emplace_back(nl + 2, 0.f); ct.weightSums_bak[l] = bufs.back().data() + 1;
    bufs.emplace_back(4 * nl, 0.f);
    float* c = bufs.back().data();
    ct.pc_u[l] = c; ct.pc_v[l] = c + nl; ct.pc_idepth[l] = c + 2 * nl; ct.pc_color[l] = c + 3 * nl;
    grays[l].resize(nl);
    for (size_t i = 0; i < nl; ++i) { grays[l][i][0] = gray[off + i]; grays[l][i][1] = grays[l][i][2] = 0; }
    fh.dIp[l] = grays[l].data();
    off += nl;
  }
  const size_t n0 = (size_t)w0 * h0;
  std::vector<float> img(2 * n0, 0.f);
  ct.idepth_nodia = img.data(); ct.depth_rel_var = img.data() + n0;
  ct.pc_u_nodia = pc_nodia; ct.pc_v_nodia = pc_nodia + n0;
  ct.pc_idepth_nodia = pc_nodia + 2 * n0; ct.pc_color_nodia = pc_nodia + 3 * n0;
  ct.lastRef = &fh;
  std::vector<PointHessian> ph(n);
  std::vector<PointFrameResidual> res(n);
  std::vector<EFPoint> ef(n);
  EFResidual efr;
  for (int k = 0; k < n; ++k) {
    ef[k].HdiF = phs[k];
    res[k].efResidual = &efr; res[k].target = &fh; res[k].point = &ph[k];
    res[k].centerProjectedTo = Vec3f(pu[k], pv[k], pid[k]);
    ph[k].u = pu[k]; ph[k].v = pv[k]; ph[k].idepth = pid[k];
    ph[k].idepth_hessian = rgbd ? phs[k] : 1.f;
    ph[k].efPoint = &ef[k];
    ph[k].lastResiduals[0] = std::make_pair(rgbd ? nullptr : &res[k], IN);
    ph[k].lastResiduals[1] = std::make_pair(nullptr, OOB);
    fh.pointHessians.push_back(&ph[k]);
  }
  ct.makeCoarseDepthL0(std::vector<FrameHessian*>{&fh}, rgbd != 0);
  *pc_n_nodia_out = ct.pc_n_nodia;
  return 0;
}

// out[0] = the selected idepth, out[1] = get_idepth_quantile's return value.  NaN for both when (int)(fraction * (float)n) is
// not below n: the reference's nth_element and read are undefined there, so it is not called.
void ref_idepth_quantile(int n, const float* idepth, float fraction, float* out) {
  const int k = (int)(fraction * (float)n);
  out[0] = out[1] = NAN;
  if (n <= 0 || k >= n) return;
  std::vector<float> s(idepth, idepth + n);
  std::nth_element(s.begin(), s.begin() + k, s.end());
  out[0] = s[k];
  out[1] = get_idepth_quantile(n, idepth, fraction);
}

}  // extern "C"
