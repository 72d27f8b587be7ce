// CudaImmaturePoints over the tandem_b200 C ABI.  Errors throw std::runtime_error, as the tracker shim's do.
#include "cuda_coarse_tracker/cuda_immature_points.h"
#include "cuda_coarse_tracker/cuda_pixel_selector.h"

#include <stdexcept>
#include <string>

#include "tandem_b200.h"

static void chk(int rc, const char *where) {
  if (rc != TDM_OK) throw std::runtime_error(std::string(where) + ": " + tdm_last_error());
}

CudaImmaturePoints::CudaImmaturePoints(int w, int h, int capacity_per_host, int device) : capacity_(capacity_per_host) {
  chk(tdm_immature_create(w, h, capacity_per_host, nullptr, device, &handle_), "CudaImmaturePoints");
}

CudaImmaturePoints::~CudaImmaturePoints() { tdm_immature_destroy(handle_); }

int CudaImmaturePoints::add(int host_slot, tdm_pyramid *host_pyramid, std::vector<int> const &u, std::vector<int> const &v,
                            std::vector<float> const &type) {
  if (u.size() != v.size() || u.size() != type.size()) throw std::runtime_error("CudaImmaturePoints::add: sizes differ");
  int n = 0;
  chk(tdm_immature_add(handle_, host_slot, host_pyramid, (int)u.size(), u.data(), v.data(), type.data(), &n),
      "CudaImmaturePoints::add");
  return n;
}

int CudaImmaturePoints::makeNewTraces(int host_slot, CudaPixelSelector &selector, tdm_pyramid *pyramid, float density,
                                      std::vector<int> *u, std::vector<int> *v, std::vector<float> *type) {
  int free = 0, count = 0;
  chk(tdm_immature_get(handle_, host_slot, 0, 0, &count, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                       nullptr, nullptr, nullptr, nullptr, nullptr),
      "CudaImmaturePoints::makeNewTraces");
  free = capacity_ - count;
  std::vector<int> uu(free > 0 ? free : 0), vv(uu.size());
  std::vector<float> tt(uu.size());
  int n = 0;
  chk(tdm_immature_make_new_traces(handle_, host_slot, selector.handle(), pyramid, density, nullptr, &n, uu.data(), vv.data(),
                                   tt.data()),
      "CudaImmaturePoints::makeNewTraces");
  if (u) u->assign(uu.begin(), uu.begin() + n);
  if (v) v->assign(vv.begin(), vv.begin() + n);
  if (type) type->assign(tt.begin(), tt.begin() + n);
  return n;
}

void CudaImmaturePoints::trace(tdm_pyramid *frame_pyramid, std::vector<int> const &host_slots,
                               std::vector<tdm_pyramid *> const &host_pyramids,
                               std::vector<Eigen::Matrix<float, 3, 3>> const &KRKi,
                               std::vector<Eigen::Matrix<float, 3, 1>> const &Kt,
                               std::vector<Eigen::Matrix<float, 2, 1>> const &aff) {
  const size_t n = host_slots.size();
  if (host_pyramids.size() != n || KRKi.size() != n || Kt.size() != n || aff.size() != n)
    throw std::runtime_error("CudaImmaturePoints::trace: sizes differ");
  std::vector<float> k(9 * n), t(3 * n), a(2 * n);
  for (size_t j = 0; j < n; ++j) {
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) k[9 * j + 3 * r + c] = KRKi[j](r, c);
      t[3 * j + r] = Kt[j](r);
    }
    a[2 * j] = aff[j](0);
    a[2 * j + 1] = aff[j](1);
  }
  chk(tdm_immature_trace(handle_, frame_pyramid, (int)n, host_slots.data(), host_pyramids.data(), k.data(), t.data(), a.data()),
      "CudaImmaturePoints::trace");
}

CudaImmaturePoints::State CudaImmaturePoints::get(int host_slot) {
  int n = 0;
  chk(tdm_immature_get(handle_, host_slot, 0, 0, &n, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                       nullptr, nullptr, nullptr, nullptr, nullptr),
      "CudaImmaturePoints::get");
  State s;
  for (auto *f : {&s.u, &s.v, &s.idepth_min, &s.idepth_max, &s.quality, &s.interval}) f->resize(n);
  s.status.resize(n);
  chk(tdm_immature_get(handle_, host_slot, 0, n, nullptr, s.u.data(), s.v.data(), nullptr, nullptr, nullptr, nullptr, nullptr,
                       s.idepth_min.data(), s.idepth_max.data(), s.quality.data(), s.status.data(), nullptr, s.interval.data()),
      "CudaImmaturePoints::get");
  return s;
}

void CudaImmaturePoints::remove(int host_slot, std::vector<int> const &indices) {
  chk(tdm_immature_remove(handle_, host_slot, (int)indices.size(), indices.data()), "CudaImmaturePoints::remove");
}

void CudaImmaturePoints::dropHost(int host_slot) { chk(tdm_immature_drop_host(handle_, host_slot), "CudaImmaturePoints::dropHost"); }

CudaImmaturePoints::Activation CudaImmaturePoints::activate(std::vector<int> const &frame_slots,
                                                            std::vector<tdm_pyramid *> const &frame_pyramids,
                                                            std::vector<Precalc> const &precalc, float fxl, float fyl, float cxl,
                                                            float cyl, std::vector<int> const &cand_frame,
                                                            std::vector<int> const &cand_index, float min_idepth_h_act,
                                                            int gn_iterations, int min_obs) {
  const size_t n = frame_slots.size(), k = cand_frame.size();
  if (frame_pyramids.size() != n || precalc.size() != n * n || cand_index.size() != k)
    throw std::runtime_error("CudaImmaturePoints::activate: sizes differ");
  std::vector<float> pc(14 * n * n);
  for (size_t e = 0; e < n * n; ++e) {
    float *o = pc.data() + 14 * e;
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) o[3 * r + c] = precalc[e].PRE_RTll(r, c);
      o[9 + r] = precalc[e].PRE_tTll(r);
    }
    o[12] = precalc[e].PRE_aff_mode(0);
    o[13] = precalc[e].PRE_aff_mode(1);
  }
  const float calib[4] = {fxl, fyl, cxl, cyl};
  const tdm_activate_settings st = {min_idepth_h_act, gn_iterations, min_obs};
  Activation a;
  a.n_frames = (int)n;
  a.result.resize(k);
  a.idepth.resize(k);
  a.res_state.resize(k * n);
  a.res_energy.resize(k * n);
  chk(tdm_immature_activate(handle_, (int)n, frame_slots.data(), frame_pyramids.data(), pc.data(), calib, &st, (int)k,
                            cand_frame.data(), cand_index.data(), a.result.data(), a.idepth.data(), a.res_state.data(),
                            a.res_energy.data()),
      "CudaImmaturePoints::activate");
  return a;
}
