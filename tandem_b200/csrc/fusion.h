// Type-erased interface of the TSDF fusion engine (fusion.cu).
#pragma once
#include <cfloat>
#include <climits>

#include "../../include/tandem_b200.h"
#include "common.cuh"

namespace tdm {

class FusionIface {
 public:
  virtual ~FusionIface() = default;
  virtual void integrate_async(const unsigned char* bgr, const float* depth, const float* pose) = 0;
  // The same scan from device memory of this handle's device (height x width, as the options): the stream waits for `ready`
  // (a cudaEvent_t) and copies bgr / depth into the scan buffers; every read of them is enqueued on stream() when it returns.
  virtual void integrate_device(const unsigned char* bgr, const float* depth, int height, int width, int device, void* ready,
                                const float* pose) = 0;
  virtual void render_async(const float* const* poses, int n) = 0;
  virtual void get_render_result(unsigned char** bgr, float** depth, int n) = 0;
  virtual void set_slab(int z_block_lo, int z_block_hi) = 0;
  virtual void set_interleave(int rank, int world, int k_blocks, int z0_block) = 0;
  virtual void peer_export(tdm_fusion_peer_handle* out) = 0;
  virtual void peer_attach(const tdm_fusion_peer_handle* all, int world, int rank) = 0;
  virtual void synchronize() = 0;
  virtual void get_stats(tdm_fusion_stats* s) = 0;
  virtual long long dump_blocks(int* coords, void* voxels, size_t cap) = 0;
  virtual void run_resident(int iters, float* ms_int, float* ms_render) = 0;
  // marching cubes (ExtractMeshAsync / GetMeshSync); check_order enforces the reference's call-order state machine
  virtual void extract_mesh_async(const float* lower, const float* upper, bool check_order) = 0;
  virtual long long get_mesh(float* vert, float* cols, size_t max_vertices, bool check_order, bool query_only) = 0;
  virtual long long extract_mesh_blocking(const float* lower, const float* upper, float* vert, float* cols, size_t max_vertices) = 0;
  virtual bool mesh_pending() = 0;
  virtual long long* render_keys_device(int i) = 0;
  virtual void* stream() = 0;   // the CUDA stream all of this handle's work is ordered on (for collectives enqueued behind it)
  virtual void unpack_keys(const long long* keys_dev, float* depth_out, unsigned char* bgr_out) = 0;
  virtual float last_mesh_ms() = 0;
  virtual float last_alloc_ms() = 0;   // k_allocate share of the last run_resident's integrate time (per iteration)
  virtual void set_option(const char* name, int value) = 0;
  // device copy of the i-th depth map of the last RenderAsync + the event recorded behind it (tracker reference, n1)
  virtual const float* render_depth_device(int i, void** ready_event, int* device) = 0;
};

FusionIface* make_fusion(const tdm_fusion_options& o, int device);
int hash_slot_host(int x, int y, int z, int num_buckets, int* reference_expression);
int mesh_axis_table(float lower, float upper, float voxel_size, int* ints5, float* floats4, int* ranges2, int* bmin, int cap);

}  // namespace tdm
