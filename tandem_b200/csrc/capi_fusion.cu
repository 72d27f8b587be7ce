// extern "C" entry points for the TSDF fusion engine (include/tandem_b200.h).
#include "../../include/tandem_b200.h"
#include "capi_common.h"
#include "common.cuh"
#include "fusion.h"
#include "mvsnet.h"

struct tdm_fusion {
  tdm::FusionIface* impl;
};
struct tdm_mvsnet {   // same layout as in capi_mvsnet.cu (one pointer)
  tdm::MvsnetIface* impl;
};

extern "C" {

int tdm_fusion_create(const tdm_fusion_options* opt, int device, tdm_fusion** out) {
  TDM_API_BEGIN
  TDM_CHECK(opt && out, "null argument");
  *out = new tdm_fusion{tdm::make_fusion(*opt, device)};
  return TDM_OK;
  TDM_API_END
}
void tdm_fusion_destroy(tdm_fusion* h) {
  if (!h) return;
  try { delete h->impl; } catch (...) {}
  delete h;
}
int tdm_fusion_integrate_async(tdm_fusion* h, const unsigned char* bgr, const float* depth, const float* pose) {
  TDM_API_BEGIN
  TDM_CHECK(h && bgr && depth && pose, "null argument");
  h->impl->integrate_async(bgr, depth, pose);
  return TDM_OK;
  TDM_API_END
}
int tdm_fusion_integrate_mvsnet(tdm_fusion* h, tdm_mvsnet* m, const float* pose) {
  TDM_API_BEGIN
  TDM_CHECK(h && m, "null handle");
  tdm::FusionIface* f = h->impl;
  m->impl->read_handoff(f->stream(), [f, pose](const tdm::MvsnetIface::Handoff& ho) {
    f->integrate_device(ho.bgr, ho.depth, ho.H, ho.W, ho.device, ho.ready, pose ? pose : ho.c2w);
  });
  return TDM_OK;
  TDM_API_END
}
int tdm_fusion_render_async(tdm_fusion* h, const float* const* camera_poses, int n_poses) {
  TDM_API_BEGIN
  TDM_CHECK(h && (camera_poses || n_poses == 0), "null argument");
  h->impl->render_async(camera_poses, n_poses);
  return TDM_OK;
  TDM_API_END
}
int tdm_fusion_get_render_result(tdm_fusion* h, unsigned char** bgr_out, float** depth_out, int n_poses) {
  TDM_API_BEGIN
  TDM_CHECK(h && ((bgr_out && depth_out) || n_poses == 0), "null argument");
  h->impl->get_render_result(bgr_out, depth_out, n_poses);
  return TDM_OK;
  TDM_API_END
}
int tdm_fusion_set_slab(tdm_fusion* h, int z_block_lo, int z_block_hi) {
  TDM_API_BEGIN
  TDM_CHECK(h, "null handle");
  h->impl->set_slab(z_block_lo, z_block_hi);
  return TDM_OK;
  TDM_API_END
}
int tdm_fusion_set_interleave(tdm_fusion* h, int rank, int world, int k_blocks, int z0_block) {
  TDM_API_BEGIN
  TDM_CHECK(h, "null handle");
  h->impl->set_interleave(rank, world, k_blocks, z0_block);
  return TDM_OK;
  TDM_API_END
}
int tdm_fusion_peer_export(tdm_fusion* h, tdm_fusion_peer_handle* out) {
  TDM_API_BEGIN
  TDM_CHECK(h && out, "null argument");
  h->impl->peer_export(out);
  return TDM_OK;
  TDM_API_END
}
int tdm_fusion_peer_attach(tdm_fusion* h, const tdm_fusion_peer_handle* all, int world, int rank) {
  TDM_API_BEGIN
  TDM_CHECK(h && all, "null argument");
  h->impl->peer_attach(all, world, rank);
  return TDM_OK;
  TDM_API_END
}
int tdm_fusion_synchronize(tdm_fusion* h) {
  TDM_API_BEGIN
  TDM_CHECK(h, "null handle");
  h->impl->synchronize();
  return TDM_OK;
  TDM_API_END
}
long long tdm_fusion_extract_mesh(tdm_fusion* h, const float lower[3], const float upper[3], float* vert, float* cols,
                                  size_t max_vertices) {
  TDM_API_BEGIN
  TDM_CHECK(h && lower && upper, "null argument");
  return h->impl->extract_mesh_blocking(lower, upper, vert, cols, max_vertices);
  TDM_API_END
}
int tdm_fusion_extract_mesh_async(tdm_fusion* h, const float lower[3], const float upper[3]) {
  TDM_API_BEGIN
  TDM_CHECK(h && lower && upper, "null argument");
  h->impl->extract_mesh_async(lower, upper, true);
  return TDM_OK;
  TDM_API_END
}
long long tdm_fusion_get_mesh(tdm_fusion* h, float* vert, float* cols, size_t max_vertices) {
  TDM_API_BEGIN
  TDM_CHECK(h, "null handle");
  return h->impl->get_mesh(vert, cols, max_vertices, true, /*query_only=*/vert == nullptr && cols == nullptr);
  TDM_API_END
}
int tdm_fusion_last_mesh_ms(tdm_fusion* h, float* ms) {
  TDM_API_BEGIN
  TDM_CHECK(h && ms, "null argument");
  *ms = h->impl->last_mesh_ms();
  return TDM_OK;
  TDM_API_END
}
int tdm_fusion_render_keys_device(tdm_fusion* h, int render_index, long long** keys_dev) {
  TDM_API_BEGIN
  TDM_CHECK(h && keys_dev, "null argument");
  *keys_dev = h->impl->render_keys_device(render_index);
  return TDM_OK;
  TDM_API_END
}
int tdm_fusion_stream(tdm_fusion* h, void** stream_out) {
  TDM_API_BEGIN
  TDM_CHECK(h && stream_out, "null argument");
  *stream_out = h->impl->stream();
  return TDM_OK;
  TDM_API_END
}
int tdm_fusion_unpack_keys(tdm_fusion* h, const long long* keys_dev, float* depth_out, unsigned char* bgr_out) {
  TDM_API_BEGIN
  TDM_CHECK(h && keys_dev && depth_out && bgr_out, "null argument");
  h->impl->unpack_keys(keys_dev, depth_out, bgr_out);
  return TDM_OK;
  TDM_API_END
}
int tdm_debug_mesh_axis_table(float lower, float upper, float voxel_size, int* ints5, float* floats4, int* ranges2, int* bmin_nb, int capacity) {
  TDM_API_BEGIN
  TDM_CHECK(ints5 && floats4 && ranges2 && bmin_nb && capacity > 0, "null argument");
  return tdm::mesh_axis_table(lower, upper, voxel_size, ints5, floats4, ranges2, bmin_nb, capacity);
  TDM_API_END
}
int tdm_debug_hash_slot(int x, int y, int z, int num_buckets, int* reference_expression) {
  TDM_API_BEGIN
  TDM_CHECK(num_buckets > 0, "num_buckets must be positive");
  return tdm::hash_slot_host(x, y, z, num_buckets, reference_expression);
  TDM_API_END
}
int tdm_debug_fast_div_eligible(float voxel_size, float fx, float fy) {
  TDM_API_BEGIN
  return tdm::fast_div_eligible_host(voxel_size, fx, fy);
  TDM_API_END
}
int tdm_fusion_set_option(tdm_fusion* h, const char* name, int value) {
  TDM_API_BEGIN
  TDM_CHECK(h && name, "null argument");
  h->impl->set_option(name, value);
  return TDM_OK;
  TDM_API_END
}
int tdm_fusion_last_alloc_ms(tdm_fusion* h, float* ms) {
  TDM_API_BEGIN
  TDM_CHECK(h && ms, "null argument");
  *ms = h->impl->last_alloc_ms();
  return TDM_OK;
  TDM_API_END
}
int tdm_fusion_get_stats(tdm_fusion* h, tdm_fusion_stats* out) {
  TDM_API_BEGIN
  TDM_CHECK(h && out, "null argument");
  h->impl->get_stats(out);
  return TDM_OK;
  TDM_API_END
}
long long tdm_fusion_dump_blocks(tdm_fusion* h, int* coords, void* voxels, size_t capacity_blocks) {
  TDM_API_BEGIN
  TDM_CHECK(h, "null handle");
  return h->impl->dump_blocks(coords, voxels, capacity_blocks);
  TDM_API_END
}
int tdm_fusion_run_resident(tdm_fusion* h, int iters, float* ms_integrate, float* ms_render) {
  TDM_API_BEGIN
  TDM_CHECK(h && ms_integrate && ms_render, "null argument");
  h->impl->run_resident(iters, ms_integrate, ms_render);
  return TDM_OK;
  TDM_API_END
}

}  // extern "C"
