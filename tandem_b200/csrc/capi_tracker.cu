// extern "C" entry points for the coarse tracker (include/tandem_b200.h).
#include "../../include/tandem_b200.h"
#include "capi_common.h"
#include "common.cuh"
#include "fusion.h"
#include "tracker.h"

struct tdm_tracker {
  tdm::TrackerIface* impl;
};
struct tdm_pyramid {
  tdm::PyramidIface* impl;
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

}  // extern "C"
