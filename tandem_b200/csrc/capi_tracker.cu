// extern "C" entry points for the coarse tracker (include/tandem_b200.h).
#include <cmath>
#include <cstring>
#include <vector>

#include "../../include/tandem_b200.h"
#include "capi_common.h"
#include "common.cuh"
#include "fusion.h"
#include "tracker.h"

static_assert(sizeof(tdm_select_result) == sizeof(tdm::SelectResult), "tdm_select_result layout");
static_assert(sizeof(tdm_select_settings) == 16, "tdm_select_settings layout");
static_assert(sizeof(tdm_linearize_settings) == 32, "tdm_linearize_settings layout");

struct tdm_tracker {
  tdm::TrackerIface* impl;
};
struct tdm_pyramid {
  tdm::PyramidIface* impl;
};
struct tdm_immature {
  tdm::ImmatureIface* impl;
};
struct tdm_selector {
  tdm::SelectorIface* impl;
};
struct tdm_undistort {
  tdm::UndistortIface* impl;
};
struct tdm_active {
  tdm::ActiveIface* impl;
};
struct tdm_fusion {   // same layout as in capi_fusion.cu (one pointer)
  tdm::FusionIface* impl;
};

extern "C" {

int tdm_tracker_create(int w, int h, float huber, float cutoff, int n_max, int device, tdm_tracker** out) {
  TDM_API_BEGIN
  TDM_CHECK(out, "null argument");
  *out = new tdm_tracker{tdm::make_tracker(w, h, huber, cutoff, n_max, device)};
  return TDM_OK;
  TDM_API_END
}
void tdm_tracker_destroy(tdm_tracker* t) {
  if (!t) return;
  try { delete t->impl; } catch (...) {}
  delete t;
}
int tdm_tracker_set_k(tdm_tracker* t, int w, int h, float fx, float fy, float cx, float cy) {
  TDM_API_BEGIN
  TDM_CHECK(t, "null handle");
  t->impl->set_k(w, h, fx, fy, cx, cy);
  return TDM_OK;
  TDM_API_END
}
int tdm_tracker_set_reference(tdm_tracker* t, int n, const float* pc_u, const float* pc_v, const float* pc_idepth,
                              const float* pc_color, float ref_exposure, const double ref_aff_g2l[2]) {
  TDM_API_BEGIN
  TDM_CHECK(t && ref_aff_g2l && (n == 0 || (pc_u && pc_v && pc_idepth && pc_color)), "null argument");
  t->impl->set_reference(n, pc_u, pc_v, pc_idepth, pc_color, ref_exposure, ref_aff_g2l);
  return TDM_OK;
  TDM_API_END
}
int tdm_tracker_set_new(tdm_tracker* t, const float* dInew) {
  TDM_API_BEGIN
  TDM_CHECK(t && dInew, "null argument");
  t->impl->set_new(dInew);
  return TDM_OK;
  TDM_API_END
}
int tdm_tracker_calc_res(tdm_tracker* t, const double* refToNew, float new_exposure, const double aff_g2l[2],
                         float cutoffTH, double res6[6]) {
  TDM_API_BEGIN
  TDM_CHECK(t && refToNew && aff_g2l && res6, "null argument");
  t->impl->calc_res(refToNew, new_exposure, aff_g2l, cutoffTH, res6);
  return TDM_OK;
  TDM_API_END
}
int tdm_tracker_calc_g(tdm_tracker* t, float new_exposure, const double aff_g2l[2], double H[64], double b[8]) {
  TDM_API_BEGIN
  TDM_CHECK(t && aff_g2l && H && b, "null argument");
  t->impl->calc_g(new_exposure, aff_g2l, H, b);
  return TDM_OK;
  TDM_API_END
}
int tdm_tracker_calc_res_batch(tdm_tracker* t, int n_hyp, const double* refToNew, float new_exposure, const double* aff_g2l,
                               float cutoffTH, double* res6) {
  TDM_API_BEGIN
  TDM_CHECK(t && refToNew && aff_g2l && res6, "null argument");
  t->impl->calc_res_batch(n_hyp, refToNew, new_exposure, aff_g2l, cutoffTH, res6);
  return TDM_OK;
  TDM_API_END
}
int tdm_tracker_calc_res_g(tdm_tracker* t, const double* refToNew, float new_exposure, const double aff_g2l[2],
                           float cutoffTH, double res6[6], double H[64], double b[8]) {
  TDM_API_BEGIN
  TDM_CHECK(t && refToNew && aff_g2l && res6 && H && b, "null argument");
  t->impl->calc_res_g(refToNew, new_exposure, aff_g2l, cutoffTH, res6, H, b);
  return TDM_OK;
  TDM_API_END
}
int tdm_tracker_synchronize(tdm_tracker* t) {
  TDM_API_BEGIN
  TDM_CHECK(t, "null handle");
  t->impl->synchronize();
  return TDM_OK;
  TDM_API_END
}
int tdm_tracker_run_resident(tdm_tracker* t, int iters, float* ms_total) {
  TDM_API_BEGIN
  TDM_CHECK(t && ms_total, "null argument");
  t->impl->run_resident(iters, ms_total);
  return TDM_OK;
  TDM_API_END
}


/* ---- SURVEY 8(f) n2: image pyramid + gradients on the device ---- */
int tdm_pyramid_create(int w, int h, int levels, int device, tdm_pyramid** out) {
  TDM_API_BEGIN
  TDM_CHECK(out, "null argument");
  *out = new tdm_pyramid{tdm::make_pyramid(w, h, levels, device)};
  return TDM_OK;
  TDM_API_END
}
void tdm_pyramid_destroy(tdm_pyramid* p) {
  if (!p) return;
  try { delete p->impl; } catch (...) {}
  delete p;
}
int tdm_pyramid_build(tdm_pyramid* p, const float* gray) {
  TDM_API_BEGIN
  TDM_CHECK(p && gray, "null argument");
  p->impl->build(gray);
  return TDM_OK;
  TDM_API_END
}
int tdm_pyramid_get_level(tdm_pyramid* p, int level, float* dI, float* abs_squared_grad) {
  TDM_API_BEGIN
  TDM_CHECK(p, "null handle");
  p->impl->get_level(level, dI, abs_squared_grad);
  return TDM_OK;
  TDM_API_END
}
int tdm_tracker_set_new_from_pyramid(tdm_tracker* t, tdm_pyramid* p, int level) {
  TDM_API_BEGIN
  TDM_CHECK(t && p, "null handle");
  TDM_CHECK(level >= 0 && level < p->impl->levels(), "no such pyramid level");
  t->impl->set_new_device_checked(p->impl->level_dI(level), p->impl->ready_event(), p->impl->width(level),
                                  p->impl->height(level), p->impl->device());
  return TDM_OK;
  TDM_API_END
}

/* ---- SURVEY 8(f) n1: dense tracking reference built on the device ---- */
int tdm_tracker_set_reference_dense(tdm_tracker* t, const float* depth, tdm_fusion* depth_from_fusion, int render_index,
                                    const double T_depth_to_ref[16], int tracking_step, int dense_only, int n_sparse,
                                    const float* pc_u, const float* pc_v, const float* pc_idepth, const float* pc_color,
                                    const float* idepth0, const float* ref_gray, tdm_pyramid* ref_gray_from_pyramid,
                                    float ref_exposure, const double ref_aff_g2l[2], int* pc_n) {
  TDM_API_BEGIN
  TDM_CHECK(t && T_depth_to_ref && ref_aff_g2l && pc_n, "null argument");
  TDM_CHECK((depth != nullptr) != (depth_from_fusion != nullptr), "pass exactly one of depth / depth_from_fusion");
  TDM_CHECK((ref_gray != nullptr) != (ref_gray_from_pyramid != nullptr), "pass exactly one of ref_gray / ref_gray_from_pyramid");
  tdm::TrackerIface::DenseRefArgs a;
  if (depth_from_fusion) {
    int dev = -1;
    a.depth = depth_from_fusion->impl->render_depth_device(render_index, &a.depth_ready, &dev);
    a.depth_on_device = true;
    TDM_CHECK(dev == t->impl->device(), "fusion and tracker live on different devices");
  } else {
    a.depth = depth;
  }
  if (ref_gray_from_pyramid) {
    TDM_CHECK(ref_gray_from_pyramid->impl->device() == t->impl->device(), "pyramid and tracker live on different devices");
    TDM_CHECK(ref_gray_from_pyramid->impl->width(0) == t->impl->width() && ref_gray_from_pyramid->impl->height(0) == t->impl->height(),
              "pyramid level 0 does not match the tracker's image size");
    a.ref_gray = ref_gray_from_pyramid->impl->level_dI(0);
    a.gray_on_device = true;
    a.gray_stride = 3;
    a.gray_ready = ref_gray_from_pyramid->impl->ready_event();
  } else {
    a.ref_gray = ref_gray;
  }
  a.T_depth_to_ref = T_depth_to_ref;
  a.step = tracking_step; a.dense_only = dense_only; a.n_sparse = n_sparse;
  a.pc_u = pc_u; a.pc_v = pc_v; a.pc_idepth = pc_idepth; a.pc_color = pc_color;
  a.idepth0 = idepth0; a.ref_exposure = ref_exposure; a.ref_aff = ref_aff_g2l;
  *pc_n = t->impl->set_reference_dense(a);
  return TDM_OK;
  TDM_API_END
}
int tdm_tracker_get_reference(tdm_tracker* t, int n, float* pc_u, float* pc_v, float* pc_idepth, float* pc_color) {
  TDM_API_BEGIN
  TDM_CHECK(t, "null handle");
  t->impl->get_reference(n, pc_u, pc_v, pc_idepth, pc_color);
  return TDM_OK;
  TDM_API_END
}
int tdm_tracker_get_warped(tdm_tracker* t, int n, float* out) {
  TDM_API_BEGIN
  TDM_CHECK(t && out, "null argument");
  t->impl->get_warped(n, out);
  return TDM_OK;
  TDM_API_END
}

/* ---- SURVEY 8(f) n3: one pyramid level's LM loop on the device ---- */
int tdm_tracker_track(tdm_tracker* t, const double refToNew[16], const double aff_g2l[2], float new_exposure,
                      float coarse_cutoff_th, int max_iterations, float lambda_extrapolation_limit, int fix_a, int fix_b,
                      tdm_track_result* out) {
  TDM_API_BEGIN
  TDM_CHECK(t && refToNew && aff_g2l && out, "null argument");
  tdm::TrackerIface::TrackArgs a;
  a.refToNew = refToNew; a.aff = aff_g2l; a.new_exposure = new_exposure; a.coarse_cutoff = coarse_cutoff_th;
  a.max_iterations = max_iterations; a.lambda_extrapolation_limit = lambda_extrapolation_limit; a.fix_a = fix_a; a.fix_b = fix_b;
  tdm::TrackerIface::TrackResult r;
  t->impl->track(a, &r);
  for (int i = 0; i < 16; ++i) out->ref_to_new[i] = r.refToNew[i];
  out->aff_g2l[0] = r.aff[0]; out->aff_g2l[1] = r.aff[1];
  for (int i = 0; i < 6; ++i) out->res[i] = r.res[i];
  out->iterations = r.iterations; out->evaluations = r.evaluations; out->cutoff_repeat = r.cutoff_repeat; out->device_ms = r.device_ms;
  return TDM_OK;
  TDM_API_END
}

/* ---- SURVEY 8(f) n5: CoarseTracker::trackNewestCoarse over all pyramid levels on the device ---- */
int tdm_tracker_track_pyramid(tdm_tracker* const* levels, int coarsest_level, const double refToNew[16], const double aff_g2l[2],
                              float new_exposure, float coarse_cutoff_th, const int max_iterations[5],
                              float lambda_extrapolation_limit, float affine_opt_mode_a, float affine_opt_mode_b,
                              const double min_res_for_abort[5], tdm_track_pyramid_result* out) {
  TDM_API_BEGIN
  TDM_CHECK(levels && refToNew && aff_g2l && max_iterations && min_res_for_abort && out, "null argument");
  TDM_CHECK(coarsest_level >= 0 && coarsest_level <= 4, "coarsest_level must be in 0..4");
  tdm::TrackerIface* impl[5] = {};
  for (int l = 0; l <= coarsest_level; ++l) {
    TDM_CHECK(levels[l], "track_pyramid level " + std::to_string(l) + ": null tracker");
    impl[l] = levels[l]->impl;
  }
  tdm::TrackerIface::PyramidArgs a;
  a.refToNew = refToNew; a.aff = aff_g2l; a.new_exposure = new_exposure; a.coarse_cutoff = coarse_cutoff_th;
  a.max_iterations = max_iterations; a.lambda_extrapolation_limit = lambda_extrapolation_limit;
  a.affine_mode_a = affine_opt_mode_a; a.affine_mode_b = affine_opt_mode_b; a.min_res_for_abort = min_res_for_abort;
  tdm::TrackerIface::PyramidResult r;
  impl[0]->track_pyramid(impl, coarsest_level, a, &r);
  for (int i = 0; i < 16; ++i) out->ref_to_new[i] = r.refToNew[i];
  out->aff_g2l[0] = r.aff[0]; out->aff_g2l[1] = r.aff[1];
  for (int l = 0; l < 5; ++l) {
    out->last_residuals[l] = r.last_residuals[l];
    out->iterations[l] = r.iterations[l]; out->evaluations[l] = r.evaluations[l]; out->cutoff_repeat[l] = r.cutoff_repeat[l];
  }
  for (int i = 0; i < 3; ++i) out->last_flow_indicators[i] = r.last_flow_indicators[i];
  out->ok = r.ok; out->aborted_level = r.aborted_level; out->repeated_level = r.repeated_level; out->device_ms = r.device_ms;
  return TDM_OK;
  TDM_API_END
}

/* ---- SURVEY 8(f) n6: FullSystem::trackNewCoarse's motion-hypothesis loop on the device ---- */
int tdm_tracker_track_new_coarse(tdm_tracker* const* levels, int coarsest_level, const double* tries, int n_tries,
                                 const double aff_last_2_l[2], float new_exposure, float coarse_cutoff_th, const int max_iterations[5],
                                 float lambda_extrapolation_limit, float affine_opt_mode_a, float affine_opt_mode_b,
                                 const double last_coarse_rmse[5], float retrack_threshold, tdm_track_new_coarse_result* out,
                                 tdm_track_try* tries_out) {
  TDM_API_BEGIN
  TDM_CHECK(levels && tries && aff_last_2_l && max_iterations && last_coarse_rmse && out, "null argument");
  TDM_CHECK(n_tries >= 1 && n_tries <= 64, "n_tries must be in 1..64");
  TDM_CHECK(coarsest_level >= 0 && coarsest_level <= 4, "coarsest_level must be in 0..4");
  tdm::TrackerIface* impl[5] = {};
  for (int l = 0; l <= coarsest_level; ++l) {
    TDM_CHECK(levels[l], "track_pyramid level " + std::to_string(l) + ": null tracker");
    impl[l] = levels[l]->impl;
  }
  tdm::TrackerIface::NewCoarseArgs a;
  a.tries = tries; a.n_tries = n_tries; a.aff_last_2_l = aff_last_2_l; a.new_exposure = new_exposure;
  a.coarse_cutoff = coarse_cutoff_th; a.max_iterations = max_iterations; a.lambda_extrapolation_limit = lambda_extrapolation_limit;
  a.affine_mode_a = affine_opt_mode_a; a.affine_mode_b = affine_opt_mode_b; a.last_coarse_rmse = last_coarse_rmse;
  a.retrack_threshold = retrack_threshold;
  tdm::TrackerIface::NewCoarseResult r;
  tdm::TrackerIface::TryResult rec[64];
  impl[0]->track_new_coarse(impl, coarsest_level, a, &r, tries_out ? rec : nullptr);
  for (int i = 0; i < 16; ++i) out->ref_to_new[i] = r.refToNew[i];
  out->aff_g2l[0] = r.aff[0]; out->aff_g2l[1] = r.aff[1];
  for (int l = 0; l < 5; ++l) out->achieved_res[l] = r.achieved_res[l];
  for (int i = 0; i < 3; ++i) out->flow_vecs[i] = r.flow_vecs[i];
  out->have_one_good = r.have_one_good; out->tries = r.tries; out->winner = r.winner; out->device_ms = r.device_ms;
  for (int k = 0; tries_out && k < r.tries; ++k) {
    for (int l = 0; l < 5; ++l) { tries_out[k].last_residuals[l] = rec[k].last_residuals[l]; tries_out[k].evaluations[l] = rec[k].evaluations[l]; }
    tries_out[k].ok = rec[k].ok; tries_out[k].aborted_level = rec[k].aborted_level; tries_out[k].repeated_level = rec[k].repeated_level;
  }
  return TDM_OK;
  TDM_API_END
}

/* ---- SURVEY 8(f) n7: CoarseTracker::setCoarseTrackingRef with makeCoarseDepthL0, every level on the device ---- */
}  // extern "C"

// n7's arguments, checked and passed to levels[0]; nodia (with its fraction) adds the undilated cloud and its quantile
static void coarse_tracking_ref(tdm_tracker* const* levels, int n_levels, int rgbd_init, int n_points, const float* pt_u,
                                const float* pt_v, const float* pt_idepth, const float* pt_hessian, tdm_pyramid* ref_pyramid,
                                const float* depth, tdm_fusion* depth_from_fusion, int render_index, const double T_depth_to_ref[16],
                                int tracking_step, int dense_only, float ref_exposure, const double ref_aff_g2l[2],
                                float quantile_fraction, int pc_n[5], tdm::TrackerIface::CoarseNodiaResult* nodia) {
  TDM_CHECK(levels && ref_pyramid && ref_aff_g2l && pc_n, "null argument");
  TDM_CHECK(n_levels >= 1 && n_levels <= 5, "n_levels must be in 1..5");
  TDM_CHECK(!(depth && depth_from_fusion), "pass at most one of depth / depth_from_fusion");
  TDM_CHECK(!nodia || (std::isfinite(quantile_fraction) && quantile_fraction >= 0.f && quantile_fraction <= 1.f),
            "quantile_fraction must be finite and in [0, 1]");
  tdm::TrackerIface* impl[5] = {};
  for (int l = 0; l < n_levels; ++l) {
    TDM_CHECK(levels[l], "set_coarse_tracking_ref level " + std::to_string(l) + ": null tracker");
    impl[l] = levels[l]->impl;
  }
  tdm::TrackerIface::CoarseRefArgs a;
  a.n_levels = n_levels; a.rgbd_init = rgbd_init != 0; a.n_points = n_points;
  a.pt_u = pt_u; a.pt_v = pt_v; a.pt_idepth = pt_idepth; a.pt_hessian = pt_hessian;
  a.ref_pyramid = ref_pyramid->impl;
  if (depth_from_fusion) {
    TDM_CHECK(T_depth_to_ref, "dense map without T_depth_to_ref");
    int dev = -1;
    a.depth = depth_from_fusion->impl->render_depth_device(render_index, &a.depth_ready, &dev);
    a.depth_on_device = true;
    TDM_CHECK(dev == impl[0]->device(), "fusion and tracker live on different devices");
  } else {
    a.depth = depth;
  }
  a.T_depth_to_ref = T_depth_to_ref; a.step = tracking_step; a.dense_only = dense_only;
  a.ref_exposure = ref_exposure; a.ref_aff = ref_aff_g2l;
  a.quantile_fraction = quantile_fraction;
  impl[0]->set_coarse_tracking_ref(impl, a, pc_n, nodia);
}

extern "C" {

int tdm_tracker_set_coarse_tracking_ref(tdm_tracker* const* levels, int n_levels, int rgbd_init, int n_points, const float* pt_u,
                                        const float* pt_v, const float* pt_idepth, const float* pt_hessian, tdm_pyramid* ref_pyramid,
                                        const float* depth, tdm_fusion* depth_from_fusion, int render_index,
                                        const double T_depth_to_ref[16], int tracking_step, int dense_only, float ref_exposure,
                                        const double ref_aff_g2l[2], int pc_n[5]) {
  TDM_API_BEGIN
  coarse_tracking_ref(levels, n_levels, rgbd_init, n_points, pt_u, pt_v, pt_idepth, pt_hessian, ref_pyramid, depth, depth_from_fusion,
                      render_index, T_depth_to_ref, tracking_step, dense_only, ref_exposure, ref_aff_g2l, 0.f, pc_n, nullptr);
  return TDM_OK;
  TDM_API_END
}

/* ---- n7 + the undilated level-0 cloud and the MVSNet depth range's inverse-depth quantile over it ---- */
int tdm_tracker_set_coarse_tracking_ref_nodia(tdm_tracker* const* levels, int n_levels, int rgbd_init, int n_points,
                                              const float* pt_u, const float* pt_v, const float* pt_idepth, const float* pt_hessian,
                                              tdm_pyramid* ref_pyramid, const float* depth, tdm_fusion* depth_from_fusion,
                                              int render_index, const double T_depth_to_ref[16], int tracking_step, int dense_only,
                                              float ref_exposure, const double ref_aff_g2l[2], float quantile_fraction, int pc_n[5],
                                              tdm_coarse_nodia_result* out) {
  TDM_API_BEGIN
  TDM_CHECK(out, "null argument");
  tdm::TrackerIface::CoarseNodiaResult r{};
  const auto give = [&] { out->pc_n_nodia = r.pc_n_nodia; out->idepth_quantile = r.idepth_quantile; out->depth_quantile = r.depth_quantile; };
  try {
    coarse_tracking_ref(levels, n_levels, rgbd_init, n_points, pt_u, pt_v, pt_idepth, pt_hessian, ref_pyramid, depth,
                        depth_from_fusion, render_index, T_depth_to_ref, tracking_step, dense_only, ref_exposure, ref_aff_g2l,
                        quantile_fraction, pc_n, &r);
  } catch (...) {   // a capacity error: the nodia outputs were computed
    give();
    throw;
  }
  give();
  return TDM_OK;
  TDM_API_END
}
int tdm_tracker_get_coarse_nodia(tdm_tracker* level0, int n, float* u, float* v, float* idepth, float* color) {
  TDM_API_BEGIN
  TDM_CHECK(level0, "null handle");
  level0->impl->get_coarse_nodia(n, u, v, idepth, color);
  return TDM_OK;
  TDM_API_END
}

/* ---- SURVEY 8(f) n8: immature points traced on the device ---- */
int tdm_immature_create(int w, int h, int capacity_per_host, const tdm_trace_settings* settings, int device, tdm_immature** out) {
  TDM_API_BEGIN
  TDM_CHECK(out, "null argument");
  static const tdm_trace_settings defaults = {0.027f, 1.f, 0.1f, 1.2f, 1.5f, 2.f, 9.f, 144.f, 2500.f, 1.f, 2, 3};
  *out = new tdm_immature{tdm::make_immature(w, h, capacity_per_host, (const float*)(settings ? settings : &defaults), device)};
  return TDM_OK;
  TDM_API_END
}
void tdm_immature_destroy(tdm_immature* s) {
  if (!s) return;
  try { delete s->impl; } catch (...) {}
  delete s;
}
int tdm_immature_add(tdm_immature* s, int host_slot, tdm_pyramid* host_pyramid, int n, const int* u, const int* v,
                     const float* type, int* n_added) {
  TDM_API_BEGIN
  TDM_CHECK(s && host_pyramid && n_added, "null argument");
  *n_added = s->impl->add(host_slot, *host_pyramid->impl, n, u, v, type);
  return TDM_OK;
  TDM_API_END
}
int tdm_immature_trace(tdm_immature* s, tdm_pyramid* frame_pyramid, int n_hosts, const int* host_slots,
                       tdm_pyramid* const* host_pyramids, const float* KRKi9, const float* Kt3, const float* aff2) {
  TDM_API_BEGIN
  TDM_CHECK(s && frame_pyramid, "null argument");
  TDM_CHECK(n_hosts >= 0 && n_hosts <= 8, "n_hosts outside 0..8");
  const tdm::PyramidIface* hp[8] = {};
  if (host_pyramids)
    for (int j = 0; j < n_hosts; ++j) hp[j] = host_pyramids[j] ? host_pyramids[j]->impl : nullptr;
  s->impl->trace(*frame_pyramid->impl, n_hosts, host_slots, hp, KRKi9, Kt3, aff2);
  return TDM_OK;
  TDM_API_END
}
int tdm_immature_get(tdm_immature* s, int host_slot, int first, int n, int* count, float* u, float* v, float* type,
                     float* energy_th, float* color, float* weights, float* grad_h, float* idepth_min, float* idepth_max,
                     float* quality, int* status, float* uv, float* interval) {
  TDM_API_BEGIN
  TDM_CHECK(s, "null handle");
  using namespace tdm;
  const bool any = u || v || type || energy_th || color || weights || grad_h || idepth_min || idepth_max || quality || status ||
                   uv || interval;
  std::vector<float> rows(any ? (size_t)IM_ROWS * (n > 0 ? n : 0) : 0);
  float* r[IM_ROWS] = {};
  if (any)
    for (int k = 0; k < IM_ROWS; ++k) r[k] = rows.data() + (size_t)k * n;
  s->impl->get(host_slot, first, n, r);
  if (count) *count = s->impl->count(host_slot);
  if (!any) return TDM_OK;
  auto plain = [&](int row, float* out) { if (out) std::memcpy(out, r[row], 4ull * n); };
  plain(IM_U, u); plain(IM_V, v); plain(IM_TYPE, type); plain(IM_ETH, energy_th); plain(IM_IDMIN, idepth_min);
  plain(IM_IDMAX, idepth_max); plain(IM_QUALITY, quality); plain(IM_INTERVAL, interval);
  if (status) std::memcpy(status, r[IM_STATUS], 4ull * n);
  for (int i = 0; i < n; ++i) {
    for (int k = 0; k < 8; ++k) {
      if (color) color[8 * i + k] = r[IM_COLOR + k][i];
      if (weights) weights[8 * i + k] = r[IM_WEIGHTS + k][i];
    }
    for (int k = 0; k < 4; ++k)
      if (grad_h) grad_h[4 * i + k] = r[IM_GRADH + k][i];
    if (uv) { uv[2 * i] = r[IM_UVX][i]; uv[2 * i + 1] = r[IM_UVY][i]; }
  }
  return TDM_OK;
  TDM_API_END
}
int tdm_immature_remove(tdm_immature* s, int host_slot, int n_removed, const int* indices) {
  TDM_API_BEGIN
  TDM_CHECK(s, "null handle");
  s->impl->remove(host_slot, n_removed, indices);
  return TDM_OK;
  TDM_API_END
}
int tdm_immature_drop_host(tdm_immature* s, int host_slot) {
  TDM_API_BEGIN
  TDM_CHECK(s, "null handle");
  s->impl->drop_host(host_slot);
  return TDM_OK;
  TDM_API_END
}

/* ---- n9: activatePointsMT's optimizeImmaturePoint on the device ---- */
int tdm_immature_activate(tdm_immature* s, int n_frames, const int* frame_slots, tdm_pyramid* const* frame_pyramids,
                          const float* precalc, const float calib4[4], const tdm_activate_settings* settings, int n_cand,
                          const int* cand_frame, const int* cand_index, int* result, float* idepth, signed char* res_state,
                          float* res_energy) {
  TDM_API_BEGIN
  TDM_CHECK(s && frame_slots && frame_pyramids, "null argument");
  TDM_CHECK(n_frames >= 1 && n_frames <= 8, "n_frames outside 1..8");
  static const tdm_activate_settings defaults = {100.f, 3, 1};
  const tdm_activate_settings& st = settings ? *settings : defaults;
  const tdm::PyramidIface* fp[8] = {};
  for (int f = 0; f < n_frames; ++f) {
    TDM_CHECK(frame_pyramids[f], "null argument");
    fp[f] = frame_pyramids[f]->impl;
  }
  s->impl->activate(n_frames, frame_slots, fp, precalc, calib4, st.min_idepth_h_act, st.gn_iterations, st.min_obs, n_cand,
                    cand_frame, cand_index, result, idepth, res_state, res_energy);
  return TDM_OK;
  TDM_API_END
}

/* ---- n10: PixelSelector::makeMaps and makeNewTraces on the device ---- */
int tdm_selector_create(int w, int h, const tdm_select_settings* settings, int device, tdm_selector** out) {
  TDM_API_BEGIN
  TDM_CHECK(out, "null argument");
  static const tdm_select_settings defaults = {0.5f, 7.f, 0.75f, 1};
  *out = new tdm_selector{tdm::make_selector(w, h, (const float*)(settings ? settings : &defaults), device)};
  return TDM_OK;
  TDM_API_END
}
void tdm_selector_destroy(tdm_selector* s) {
  if (!s) return;
  try { delete s->impl; } catch (...) {}
  delete s;
}
int tdm_selector_get_potential(tdm_selector* s, int* potential) {
  TDM_API_BEGIN
  TDM_CHECK(s && potential, "null argument");
  *potential = s->impl->potential();
  return TDM_OK;
  TDM_API_END
}
int tdm_selector_set_potential(tdm_selector* s, int potential) {
  TDM_API_BEGIN
  TDM_CHECK(s, "null handle");
  s->impl->set_potential(potential);
  return TDM_OK;
  TDM_API_END
}
int tdm_selector_make_maps(tdm_selector* s, tdm_pyramid* pyramid, float density, int recursions_left, float th_factor,
                           float* map_out, tdm_select_result* out) {
  TDM_API_BEGIN
  TDM_CHECK(s && pyramid, "null argument");
  s->impl->make_maps(*pyramid->impl, density, recursions_left, th_factor, map_out, reinterpret_cast<tdm::SelectResult*>(out));
  return TDM_OK;
  TDM_API_END
}
int tdm_immature_make_new_traces(tdm_immature* set, int host_slot, tdm_selector* sel, tdm_pyramid* pyramid, float density,
                                 tdm_select_result* out, int* n_added, int* u, int* v, float* type) {
  TDM_API_BEGIN
  TDM_CHECK(set && sel && pyramid, "null argument");
  const int n = set->impl->make_new_traces(host_slot, *sel->impl, *pyramid->impl, density,
                                           reinterpret_cast<tdm::SelectResult*>(out), u, v, type);
  if (n_added) *n_added = n;
  return TDM_OK;
  TDM_API_END
}

/* ---- n11: processFrame, the remap and makeImages' gamma weights on the device ---- */
int tdm_undistort_create(const tdm_undistort_settings* s, int device, tdm_undistort** out) {
  TDM_API_BEGIN
  TDM_CHECK(s && out, "null argument");
  *out = new tdm_undistort{tdm::make_undistort(*s, device)};
  return TDM_OK;
  TDM_API_END
}
void tdm_undistort_destroy(tdm_undistort* u) {
  if (!u) return;
  try { delete u->impl; } catch (...) {}
  delete u;
}
int tdm_undistort_get_gamma(tdm_undistort* u, float G[256], int* valid) {
  TDM_API_BEGIN
  TDM_CHECK(u && G && valid, "null argument");
  u->impl->get_gamma(G, valid);
  return TDM_OK;
  TDM_API_END
}
int tdm_undistort_set_gamma(tdm_undistort* u, const float* Binv) {
  TDM_API_BEGIN
  TDM_CHECK(u, "null handle");
  u->impl->set_gamma(Binv);
  return TDM_OK;
  TDM_API_END
}
int tdm_undistort_frame(tdm_undistort* u, const unsigned char* gray, float exposure, float factor, tdm_pyramid* out,
                        float* exposure_time, const unsigned char* bgr, unsigned char* bgr_out) {
  TDM_API_BEGIN
  TDM_CHECK(u && gray && out, "null argument");
  const float t = u->impl->frame(gray, exposure, factor, *out->impl, bgr, bgr_out);
  if (exposure_time) *exposure_time = t;
  return TDM_OK;
  TDM_API_END
}

/* ---- n12: linearizeAll on the device ---- */
int tdm_active_create(int w, int h, int capacity_points, const tdm_linearize_settings* settings, int device, tdm_active** out) {
  TDM_API_BEGIN
  TDM_CHECK(out, "null argument");
  static const tdm_linearize_settings defaults = {9.f, 2500.f, 1e12f, 1e8f, 0.7f, 0.5f, 1.5f, 1.f};
  *out = new tdm_active{tdm::make_active(w, h, capacity_points, (const float*)(settings ? settings : &defaults), device)};
  return TDM_OK;
  TDM_API_END
}
void tdm_active_destroy(tdm_active* s) {
  if (!s) return;
  try { delete s->impl; } catch (...) {}
  delete s;
}
int tdm_active_load(tdm_active* s, int n_frames, int n_points, const int* point_host, const float* point_u, const float* point_v,
                    const float* color, const float* weights, const float* max_rel_baseline, const int* num_good_residuals,
                    int n_residuals, const int* res_point, const int* res_target) {
  TDM_API_BEGIN
  TDM_CHECK(s, "null handle");
  s->impl->load(n_frames, n_points, point_host, point_u, point_v, color, weights, max_rel_baseline, num_good_residuals, n_residuals,
                res_point, res_target);
  return TDM_OK;
  TDM_API_END
}
int tdm_active_linearize(tdm_active* s, tdm_pyramid* const* frame_pyramids, const float* precalc, const float* frame_energy_th,
                         const float calib4[4], const float* idepth_scaled, const float* idepth_zero_scaled, int fix_linearization,
                         double* energy, float* new_frame_energy_th, signed char* new_state, float* new_energy,
                         float* new_energy_with_outlier, float* center_projected_to, float* jacobians, signed char* state,
                         unsigned char* removed, float* max_rel_baseline, int* num_good_residuals) {
  TDM_API_BEGIN
  TDM_CHECK(s && frame_pyramids, "null argument");
  const tdm::PyramidIface* fp[8] = {};
  const int n = s->impl->n_frames();
  TDM_CHECK(n >= 2, "linearize before load");
  for (int f = 0; f < n; ++f) {
    TDM_CHECK(frame_pyramids[f], "null argument");
    fp[f] = frame_pyramids[f]->impl;
  }
  tdm::ActiveIface::Outputs o;
  o.energy = energy; o.new_frame_energy_th = new_frame_energy_th; o.new_state = new_state; o.new_energy = new_energy;
  o.new_energy_with_outlier = new_energy_with_outlier; o.center_projected_to = center_projected_to; o.jacobians = jacobians;
  o.state = state; o.removed = removed; o.max_rel_baseline = max_rel_baseline; o.num_good_residuals = num_good_residuals;
  s->impl->linearize(fp, precalc, frame_energy_th, calib4, idepth_scaled, idepth_zero_scaled, fix_linearization, o);
  return TDM_OK;
  TDM_API_END
}
int tdm_active_apply_res(tdm_active* s) {
  TDM_API_BEGIN
  TDM_CHECK(s, "null handle");
  s->impl->apply_res();
  return TDM_OK;
  TDM_API_END
}
int tdm_active_get_state(tdm_active* s, signed char* state, float* energy) {
  TDM_API_BEGIN
  TDM_CHECK(s, "null handle");
  s->impl->get_state(state, energy);
  return TDM_OK;
  TDM_API_END
}

/* ---- n13: solveSystemF's accumulators on the device ---- */
int tdm_active_accumulate(tdm_active* s, const double* ad_host, const double* ad_target, const double* frame_prior,
                          const double* frame_delta_prior, const double c_prior[4], const float c_delta[4], const float* point_prior,
                          const float* point_delta, double* H_top, double* b_top, double* H_sc, double* b_sc, int* n_active,
                          float* hdi, float* idepth_hessian) {
  TDM_API_BEGIN
  TDM_CHECK(s, "null handle");
  tdm::ActiveIface::AccInputs in;
  in.ad_host = ad_host; in.ad_target = ad_target; in.frame_prior = frame_prior; in.frame_delta_prior = frame_delta_prior;
  in.c_prior = c_prior; in.c_delta = c_delta; in.point_prior = point_prior; in.point_delta = point_delta;
  tdm::ActiveIface::AccOutputs o;
  o.H_top = H_top; o.b_top = b_top; o.H_sc = H_sc; o.b_sc = b_sc; o.n_active = n_active; o.hdi = hdi; o.idepth_hessian = idepth_hessian;
  s->impl->accumulate(in, o);
  return TDM_OK;
  TDM_API_END
}
int tdm_active_resubstitute(tdm_active* s, const double* x, float* step) {
  TDM_API_BEGIN
  TDM_CHECK(s, "null handle");
  s->impl->resubstitute(x, step);
  return TDM_OK;
  TDM_API_END
}
int tdm_active_get_accumulators(tdm_active* s, double* top, int* top_num, double* acc_e, double* acc_eb, double* acc_d, int* d_num,
                                double* hcc, double* bc) {
  TDM_API_BEGIN
  TDM_CHECK(s, "null handle");
  s->impl->get_accumulators(top, top_num, acc_e, acc_eb, acc_d, d_num, hcc, bc);
  return TDM_OK;
  TDM_API_END
}

}  // extern "C"
