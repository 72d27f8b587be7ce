/* tandem_b200 — C ABI of the H100-native (sm_90a) replacement for TANDEM's libdr (dense per-frame hot path).
 *
 * One opaque handle per object, int return codes (0 = ok, <0 = error, text via tdm_last_error()),
 * no exceptions and no C++/torch types across the boundary, all pointers caller-owned unless stated.
 * Blocking / non-blocking behaviour mirrors the reference classes each group replaces:
 *
 *   tdm_mvsnet_*   <->  class DrMvsnet          tandem/libdr/dr_mvsnet/src/dr_mvsnet/dr_mvsnet.h:36-66
 *   tdm_fusion_*   <->  class DrFusion          tandem/libdr/dr_fusion/src/dr_fusion/dr_fusion.h:44-73
 *   tdm_tracker_*  <->  class CudaCoarseTracker tandem/libdr/cuda_coarse_tracker/include/public/cuda_coarse_tracker.h:9-82
 *
 * The header-compatible C++ shims over this ABI live in include/dr_mvsnet/, include/dr_fusion/ and
 * include/cuda_coarse_tracker/ ; INTEGRATION.md shows how tandem/CMakeLists.txt:118-121 links them.
 */
#ifndef TANDEM_B200_H
#define TANDEM_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TDM_OK 0
#define TDM_ERR (-1)
#define TDM_PRECISION_FP32 0
#define TDM_PRECISION_MIXED16 1 /* fp16 activations, bf16 cost volume (range), fp32 accumulate */
#define TDM_PRECISION_BF16 2    /* bf16 everywhere (accuracy study only: misses the 1e-3 Abs Rel budget) */

/* Thread-local text of the last error raised by any tdm_* call on this thread. */
const char* tdm_last_error(void);
/* Library / build identification: "tandem_b200 <version> sm_90a". */
const char* tdm_version(void);
/* Number of CUDA devices visible (0 on a CPU-only box; never throws). */
int tdm_device_count(void);

/* Page-locked ("pinned") host memory, portable across devices.  Optional: every entry point accepts ordinary pageable
 * memory (staged through the library's own pinned buffers by a small copy pool), but image / result buffers that ARE
 * page-locked - from here, cudaHostAlloc or cudaHostRegister - are detected (cudaPointerGetAttributes) and DMA'd from / into
 * directly, with no staging copy.  The reference does the same staging by hand (tsdf_volume.cu:542-543, dr_mvsnet.cpp:260). */
int tdm_host_alloc_pinned(size_t bytes, void** out);
int tdm_host_free_pinned(void* p);

/* ------------------------------------------------------------------------------------------------
 * CVA-MVSNet (replaces DrMvsnet; dr_mvsnet.h:36-66, implementation dr_mvsnet.cpp:125-331)
 * ---------------------------------------------------------------------------------------------- */
typedef struct tdm_mvsnet tdm_mvsnet;

/* weights_path: a .tdmw container, or the reference's ".../model.pt" path, in which case the sidecar
 * ".../model.tdmw" next to it is loaded (DrMvsnet(char const* filename), dr_mvsnet.cpp:333).
 * precision: activation storage type; accumulation is always fp32. device: CUDA ordinal. */
int tdm_mvsnet_create(const char* weights_path, int precision, int device, tdm_mvsnet** out);
void tdm_mvsnet_destroy(tdm_mvsnet* h);

/* DrMvsnet::CallAsync (dr_mvsnet.h:43-53): "blocking for last input, non-blocking for this input".
 * bgrs[i]: H*W*3 uint8 BGR interleaved, window order, reference view at ref_index; intrinsic: 3x3
 * row-major full resolution (stage K's derived as rows0-1 * 0.25 / 0.5 / 1, dr_mvsnet.cpp:220-247);
 * cam_to_worlds[i]: 4x4 row-major. All inputs are copied before the call returns. */
int tdm_mvsnet_call_async(tdm_mvsnet* h, int height, int width, int view_num, int ref_index,
                          unsigned char* const* bgrs, const float* intrinsic_matrix,
                          float* const* cam_to_worlds, float depth_min, float depth_max,
                          float discard_percentage);
/* Same, with the three per-stage intrinsics given explicitly (9 floats each, stage1..stage3) — the
 * entry the golden-vector tests use, because export_model.py's K's are centre-preserving
 * (cva_mvsnet/models/datasets.py:144-174) while the C++ wrapper's are not. */
int tdm_mvsnet_call_async_k(tdm_mvsnet* h, int height, int width, int view_num, int ref_index,
                            unsigned char* const* bgrs, const float* intrinsics_stage123,
                            float* const* cam_to_worlds, float depth_min, float depth_max,
                            float discard_percentage);
/* Extension: CallAsync with a feature cache.  view_ids[i] names view i (a caller-chosen keyframe id, e.g. DSO's
 * FrameShell::id).  The handle keeps, per id of the last such call, the view's image and its FeatureNet outputs on the
 * device, and runs FeatureNet only for the ids it does not hold; ids that left the window are evicted.  The result is
 * the one tdm_mvsnet_call_async gives for the same images.  bgrs[i] may be NULL for an id the handle holds; a non-NULL
 * bgrs[i] of a held id is ignored (the id wins: the cached image and features are used).  intrinsics: the 3x3
 * full-resolution K as in tdm_mvsnet_call_async, or with stage_k != 0 the 27 floats of tdm_mvsnet_call_async_k.
 * Errors, with nothing launched and the cache unchanged: a NULL image for an id the handle does not hold (every id, when
 * the size or view_num differs from the last call's), the same id twice, and every tdm_mvsnet_call_async
 * error.  tdm_mvsnet_call_async / _call_async_k, a new size or view_num and any tdm_mvsnet_set_option except eager_d2h
 * empty the cache. */
int tdm_mvsnet_call_async_ids(tdm_mvsnet* h, int height, int width, int view_num, int ref_index, const long long* view_ids,
                              unsigned char* const* bgrs, const float* intrinsics, int stage_k,
                              float* const* cam_to_worlds, float depth_min, float depth_max, float discard_percentage);
/* The feature cache after the last call (waits for it): *n_ids receives the number of ids held (view_num after a
 * tdm_mvsnet_call_async_ids, 0 after a plain call), view_ids (capacity >= *n_ids, or NULL with capacity 0) those ids in
 * the last window's order, *n_computed the views FeatureNet computed for the last call.  n_ids / n_computed may be NULL. */
int tdm_mvsnet_feature_cache(tdm_mvsnet* h, long long* view_ids, int capacity, int* n_ids, int* n_computed);
/* DrMvsnet::GetResult (blocking). Copies the stage-3 maps (H*W floats each; any pointer may be NULL)
 * into caller memory: depth/confidence are edge-filtered, *_dense unfiltered (dr_mvsnet.cpp:296-329).
 * Calling it twice without a new CallAsync is an error, as in the reference (dr_mvsnet.cpp:100-102). */
int tdm_mvsnet_get_result(tdm_mvsnet* h, float* depth, float* confidence, float* depth_dense,
                          float* confidence_dense);
int tdm_mvsnet_ready(tdm_mvsnet* h); /* 1 ready, 0 busy  (DrMvsnet::Ready) */
int tdm_mvsnet_wait(tdm_mvsnet* h);  /* DrMvsnet::Wait */

/* Options (call before the first call_async): filter_all_stages=1 also edge-filters stages 1 and 2
 * (the Python model does, cva_mvsnet.py:165-173; the C++ consumer only reads stage 3).
 * keep_intermediates=1 keeps every layer output alive for tdm_mvsnet_debug_tensor. */
int tdm_mvsnet_set_option(tdm_mvsnet* h, const char* key, int value);
/* Stage outputs of the last finished call: which = "depth"|"confidence"|"depth_dense"|"confidence_dense"|"edge". */
int tdm_mvsnet_stage_output(tdm_mvsnet* h, int stage /*1..3*/, const char* which, float* out, size_t capacity);
/* Test hook: copy a named intermediate of the last call as planar fp32 [C][D][H][W]; dims4 receives C,D,H,W.
 * feat1..feat3 hold every view of the window in window order (reference first); the other FeatureNet tensors ("f.*")
 * hold only the views the last forward computed (after a cached call: its new views, in window order).
 * Returns the number of floats written, or <0. */
long long tdm_mvsnet_debug_tensor(tdm_mvsnet* h, const char* name, float* out, size_t capacity, int* dims4);

/* Device-resident measurement: re-runs the forward of the last submitted window `iters` times on the
 * handle's stream with inputs already in HBM (no H2D/D2H inside), timed with CUDA events on that stream.
 * ms_total receives the elapsed milliseconds; launches (optional) the kernel launches per forward. */
int tdm_mvsnet_run_resident(tdm_mvsnet* h, int iters, float* ms_total, int* launches);
/* Same, with FeatureNet recomputing only the last n_new (1..view_num) views of the last window (window order) and the
 * others read from the feature pool: the device time of a window that adds n_new keyframes to the cache. */
int tdm_mvsnet_run_resident_new(tdm_mvsnet* h, int n_new, int iters, float* ms_total, int* launches);
/* Same clock over n handles of one device: iters_total forwards issued round-robin, each handle on its own stream (the
 * windows are independent, so their kernels may overlap on the GPU); ms_total spans first launch .. last completion. */
int tdm_mvsnet_run_resident_multi(tdm_mvsnet* const* hs, int n, int iters_total, float* ms_total, int* launches);
/* Host-only introspection (no GPU needed): the plane-sweep homography of one source view as the cost-volume kernel receives it
 * (homo_warping, cva_mvsnet/models/module.py:795-808): M = K [R|t]_src^-1 (K [R|t]_ref^-1)^-1, rot = M[:3,:3], trans = M[:3,3];
 * a reference pixel (x, y) at depth d lands at rot (x, y, 1)^T d + trans in the source image. K row-major 3x3, poses row-major
 * 4x4 cam->world. */
int tdm_debug_homography(const float* K3x3, const float* c2w_ref, const float* c2w_src, float* rot9, float* trans3);
/* Host-only introspection (no GPU needed): the tile plan the tensor-core convolution planner picks for a layer - cin, N columns of
 * the MMA (npad, doubled for hi/lo weights), kd (1: 2-D over planes, 3: 3-D, 2: transposed-as-GEMM), the grid D x H x W the
 * tiles live on, pd (D halo), mode (0 stride-1, 1 transposed, 3 up2; +100: tiles span all D planes; 200: input-stationary 3x3x3
 * planner with npad = columns per kd block, 300: the same with tiles that span all D planes), shared-memory budget in KB.
 * Mode 400 is the stride-2 planner: kd is 1 or 3, D x H x W is the OUTPUT grid and pd carries the kernel size (3 or 5); its
 * "slot positions" are the positions of one of the four parity sub-tiles.
 * out12 = {ring slots, tile rows, tile cols, pitch, planes per tile, 128-row chunks per plane, slot positions, tiles_w,
 * tiles_h, tiles_d, grid, shared-memory bytes}. */
int tdm_debug_conv_plan(int cin, int npad, int kd, int D, int H, int W, int pd, int mode, int smem_kb, long long* out12);
/* The same plan with an explicit output count: writes the first n (1..13) values of out12 followed by the consumer
 * warpgroups of the kernel the plan is made for (the count its tile cost was balanced for). */
int tdm_debug_conv_plan_n(int cin, int npad, int kd, int D, int H, int W, int pd, int mode, int smem_kb, long long* out, int n);
/* Per-kernel CUDA-event timing of one resident forward: writes lines "name ms algorithmic_bytes flops\n"
 * into buf (NUL terminated). Returns bytes written or <0. */
long long tdm_mvsnet_profile(tdm_mvsnet* h, char* buf, size_t capacity);

/* ------------------------------------------------------------------------------------------------
 * TSDF fusion (replaces DrFusion; dr_fusion.h:18-73, implementation dr_fusion/src/tsdfvh/tsdf_volume.cu)
 * ---------------------------------------------------------------------------------------------- */
typedef struct tdm_fusion tdm_fusion;
typedef struct tdm_fusion_options { /* field-for-field DrFusionOptions, dr_fusion.h:18-36 */
  float voxel_size;
  int num_buckets;
  int bucket_size;
  int num_blocks;
  int block_size;
  int max_sdf_weight;
  float truncation_distance;
  float max_sensor_depth;
  float min_sensor_depth;
  int num_render_streams;
  float fx, fy, cx, cy;
  int height, width;
} tdm_fusion_options;

int tdm_fusion_create(const tdm_fusion_options* opt, int device, tdm_fusion** out);
void tdm_fusion_destroy(tdm_fusion* h);
/* DrFusion::IntegrateScanAsync (dr_fusion.h:50): bgr H*W*3 u8, depth H*W f32 metric z-depth, pose 4x4
 * row-major cam->world; inputs are copied into pinned staging before returning (tsdf_volume.cu:542-543). */
int tdm_fusion_integrate_async(tdm_fusion* h, const unsigned char* bgr, const float* depth, const float* pose);
/* Extension: IntegrateScanAsync of the result the last tdm_mvsnet_get_result of m returned, read on the device
 * (tandem_backend.cpp:166 passes that result's depth, the window's reference BGR image and its cam_to_world; the
 * reference's IntegrateScanAsync, tsdf_volume.cu:515-598, then uploads both images again).  Integrates the filtered
 * stage-3 depth and the reference view's BGR image - the bytes tdm_mvsnet_get_result wrote and the caller passed to
 * tdm_mvsnet_call_async - with pose, or with the window's reference cam_to_world when pose is NULL: the volume is the one
 * tdm_fusion_integrate_async builds from the same inputs, bit for bit.
 * get_result keeps that result on the device (a device-to-device copy on the engine's stream) until the next get_result, so
 * the call may come after the next window's call_async, as in TANDEM; the same result may be integrated again, into this
 * or other fusion handles.  Same call order as tdm_fusion_integrate_async; returns once the work is enqueued (no host
 * synchronisation).  Either handle may be destroyed right after the call.  Errors, with nothing launched: a null handle,
 * no result fetched from m yet, a fusion height / width that differs from the window's, handles on different devices, a
 * singular pose, the wrong call order. */
int tdm_fusion_integrate_mvsnet(tdm_fusion* h, tdm_mvsnet* m, const float* pose);
/* DrFusion::RenderAsync (dr_fusion.h:52): n_poses must equal num_render_streams (tsdf_volume.cu:643-648). */
int tdm_fusion_render_async(tdm_fusion* h, const float* const* camera_poses, int n_poses);
/* DrFusion::GetRenderResult (dr_fusion.h:54): pointers into a pinned double buffer owned by the handle,
 * valid until the next get_render_result (tsdf_volume.cu:710-732). bgr_out/depth_out: arrays of n_poses. */
int tdm_fusion_get_render_result(tdm_fusion* h, unsigned char** bgr_out, float** depth_out, int n_poses);
int tdm_fusion_synchronize(tdm_fusion* h);
/* Multi-GPU extension (not in the reference; SURVEY.md 8e): restrict this instance to the Z-slab of voxel blocks with
 * z_block_lo <= block.z < z_block_hi (block = 8 voxels; pass the owned range widened by one halo block so that trilinear
 * reads never cross ranks). Every rank integrates the same (broadcast) scans; renders are combined by a per-pixel
 * nearest-hit reduction (tandem_b200/parallel.py: reduce_nearest_hit). Call before the first scan. */
int tdm_fusion_set_slab(tdm_fusion* h, int z_block_lo, int z_block_hi);
/* Interleaved variant of the Z-slab partition: block row z is owned by rank ((z - z0_block) div k_blocks) mod world; every rank
 * additionally stores one halo block row on either side of each of its slabs.  Thin interleaved slabs balance the PER-FRAME work
 * (allocation, integration, ray-cast samples) over the ranks for any view direction - contiguous slabs only balance memory - at
 * the price of (k_blocks + 2) / k_blocks redundant integration.  Same exchange step as set_slab.  Call before the first scan. */
int tdm_fusion_set_interleave(tdm_fusion* h, int rank, int world, int k_blocks, int z0_block);
/* Pixel-partitioned ray-cast over the Z-slab-partitioned volume (the fused compute + transfer form of the exchange): every rank
 * exports its hash table and voxel pool (tdm_fusion_peer_export: raw pointers for instances of one process, CUDA IPC handles for
 * other processes), the handles of all ranks are gathered by the caller (e.g. torch.distributed.all_gather_object) and attached
 * (tdm_fusion_peer_attach: cudaIpcOpenMemHandle -> NVLink P2P mapping).  From then on RenderAsync renders only the 8x8 pixel
 * tiles t with t mod world == rank, but marches them through the WHOLE volume, reading each voxel from the rank that owns its
 * block row (local HBM or P2P loads inside the ray-cast kernel) - bit-identical to the single-volume render, occluders in other
 * slabs included; foreign tiles carry the "miss" key, so the same MIN all-reduce (slab_exchange mode) assembles the image.
 * Needs contiguous slabs in rank order WITHOUT halo rows (set_slab(owned_lo, owned_hi)), and the caller must order every rank's
 * ray-cast behind every rank's integration of the same scan (a stream-ordered barrier, tandem_b200.parallel.stream_barrier). */
typedef struct tdm_fusion_peer_handle {
  unsigned long long keys_ptr, ptrs_ptr, voxels_ptr;   /* device pointers (meaningful inside the exporting process) */
  long long pid;
  int device, num_buckets, bucket_size, slab_lo, slab_hi, reserved;
  unsigned char ipc_keys[64], ipc_ptrs[64], ipc_voxels[64];   /* cudaIpcMemHandle_t */
} tdm_fusion_peer_handle;
int tdm_fusion_peer_export(tdm_fusion* h, tdm_fusion_peer_handle* out);
int tdm_fusion_peer_attach(tdm_fusion* h, const tdm_fusion_peer_handle* all_ranks, int world, int rank);
/* The one exchange step of the slab-partitioned ray-cast, on the device: tdm_fusion_render_keys_device packs render
 * `render_index` of the last RenderAsync into height*width int64 keys (depth bits << 24 | b | g<<8 | r<<16; miss = +inf) in a
 * DEVICE buffer owned by the handle (stream synchronised on return) - the caller all-reduces it with MIN over the ranks
 * (NCCL, in place) - tdm_fusion_unpack_keys turns reduced keys back into a depth map and a bgr image in HOST buffers. */
int tdm_fusion_render_keys_device(tdm_fusion* h, int render_index, long long** keys_dev);
int tdm_fusion_unpack_keys(tdm_fusion* h, const long long* keys_dev, float* depth_out, unsigned char* bgr_out);
/* The CUDA stream (cudaStream_t) all work of this handle is ordered on.  With tdm_fusion_set_option(h, "slab_exchange", 1)
 * the ray-cast writes the keys itself (no pack kernel, no per-slab D2H, GetRenderResult does not wait) and
 * tdm_fusion_render_keys_device returns without a host sync: the caller enqueues its MIN all-reduce ON THIS STREAM (e.g.
 * torch.cuda.ExternalStream + torch.distributed, or ncclAllReduce directly) and tdm_fusion_unpack_keys behind it - one
 * host sync per frame, in unpack_keys. */
int tdm_fusion_stream(tdm_fusion* h, void** stream_out);
/* Mesh (dr_fusion.h:56-68; TsdfVolume::ExtractMeshAsync / GetMeshSync / ExtractMesh, tsdf_volume.cu:739-839; kernel
 * marching_cubes/mesh_extractor.cu:244-265): marching cubes over the cells of the box [lower, upper) at voxel spacing.
 * Output layout of GetMeshSync: vertices as xyz float triples, colours as rgb float triples in [0,1], 3 consecutive
 * vertices per triangle (no index buffer). Triangle ORDER is unspecified (the reference appends with atomicAdd).
 *   tdm_fusion_extract_mesh_async = ExtractMeshAsync: launches the extraction on the fusion stream and returns; only legal
 *     where IntegrateScanAsync is legal (tsdf_volume.cu:760-763) and not twice in a row (:769-772);
 *   tdm_fusion_get_mesh = GetMeshSync: waits, copies 3*triangles vertices out, returns the vertex count (error if it exceeds
 *     max_vertices, :796-799); with vert == cols == NULL it waits and returns the count only, the mesh stays pending;
 *   tdm_fusion_extract_mesh = TsdfVolume::ExtractMesh (blocking, no call-order check; DrFusion::GetMesh / SaveMeshToFile);
 *     with vert == cols == NULL it only returns the vertex count and keeps the mesh on the device, so that the next call
 *     (with buffers of that size) copies it out without extracting again. */
long long tdm_fusion_extract_mesh(tdm_fusion* h, const float lower[3], const float upper[3],
                                  float* vert, float* cols, size_t max_vertices);
int tdm_fusion_extract_mesh_async(tdm_fusion* h, const float lower[3], const float upper[3]);
long long tdm_fusion_get_mesh(tdm_fusion* h, float* vert, float* cols, size_t max_vertices);
/* Host-only introspection (no GPU needed): the per-axis cell table the mesh extractor uploads for one axis of a box - per cell
 * the voxel indices {gMA, gMB, gPA, gPB, gC} (ints5), {wM, wP, cM, cP} (floats4), and per voxel block {first cell, #cells}
 * (ranges2, bmin_nb = {first block, #blocks}). Returns the number of cells (mesh_extractor.cu:248-261 arithmetic). */
int tdm_debug_mesh_axis_table(float lower, float upper, float voxel_size, int* ints5, float* floats4, int* ranges2, int* bmin_nb, int capacity);
/* Host-only introspection (no GPU needed): the bucket the voxel-hashing kernels compute for block (x, y, z) - a division-free
 * remainder (precomputed ceil(2^64 / num_buckets)) - and, in *reference_expression when non-NULL, the reference's expression
 * ((x * 73856093) ^ (y * 19349669) ^ (z * 83492791)) % num_buckets, + num_buckets when negative (hash_table.cu:157-168). */
int tdm_debug_hash_slot(int x, int y, int z, int num_buckets, int* reference_expression);
/* Device time (CUDA events) of the last extraction: classify + scan + emit. */
int tdm_fusion_last_mesh_ms(tdm_fusion* h, float* ms);
/* Introspection for parity tests and the roofline: counters of the last integrate / render. */
typedef struct tdm_fusion_stats {
  long long allocated_blocks;      /* total blocks in the map */
  long long visible_blocks;        /* blocks integrated in the last scan */
  long long dropped_blocks;        /* bucket overflows (never allocated), cumulative */
  long long candidate_blocks;      /* distinct blocks touched by the last allocation pass */
} tdm_fusion_stats;
int tdm_fusion_get_stats(tdm_fusion* h, tdm_fusion_stats* out);
/* Dump the block map: xyz int triples (sorted lexicographically) into coords (capacity in blocks) and,
 * if voxels != NULL, 512 voxels per block as {float sdf; uint8 c0,c1,c2; uint8 weight} (8 B each). */
long long tdm_fusion_dump_blocks(tdm_fusion* h, int* coords, void* voxels, size_t capacity_blocks);
/* Device-resident measurement of integrate+render for the last submitted scan/pose (sums over iters);
 * tdm_fusion_last_alloc_ms: the allocation kernel's share of ms_integrate, per iteration. */
int tdm_fusion_run_resident(tdm_fusion* h, int iters, float* ms_integrate, float* ms_render);
int tdm_fusion_last_alloc_ms(tdm_fusion* h, float* ms);
/* Options.  "raycast_shared" (default 1: the production ray-cast, index arithmetic shared between the nine voxel reads of a
 * sample, one block lookup per distinct block; 0: the comparator shaped after the reference's sampler, one hash lookup per
 * voxel read) and "fast_div" (constant-divisor FMA division in the production ray-cast, exhaustively checked correctly
 * rounded; default 0) leave every rendered bit unchanged; "slab_clip" / "slab_exchange" (Z-slab volumes, see above).  Any
 * other name fails with "unknown fusion option". */
int tdm_fusion_set_option(tdm_fusion* h, const char* name, int value);

/* ------------------------------------------------------------------------------------------------
 * Coarse tracker, pyramid level 0 (replaces CudaCoarseTracker; cuda_coarse_tracker.h:9-82)
 * ---------------------------------------------------------------------------------------------- */
typedef struct tdm_tracker tdm_tracker;
int tdm_tracker_create(int w, int h, float setting_huberTH, float setting_coarseCutoffTH, int n_max,
                       int device, tdm_tracker** out);
void tdm_tracker_destroy(tdm_tracker* t);
int tdm_tracker_set_k(tdm_tracker* t, int w, int h, float fx, float fy, float cx, float cy);
int tdm_tracker_set_reference(tdm_tracker* t, int n, const float* pc_u, const float* pc_v,
                              const float* pc_idepth, const float* pc_color, float ref_exposure,
                              const double ref_aff_g2l[2]);
int tdm_tracker_set_new(tdm_tracker* t, const float* dInew /* h*w*3: (I,dx,dy) interleaved */);
/* calcRes: refToNew 4x4 row-major double; res6 = [E, numTermsInE, flowT, 0, flowRT, saturatedRatio]. */
int tdm_tracker_calc_res(tdm_tracker* t, const double* refToNew, float new_exposure,
                         const double aff_g2l[2], float cutoffTH, double res6[6]);
/* calcG: H 8x8 row-major, b 8; uses the warped buffers of the last calc_res (tdm_tracker_calc_res_g, _calc_res_batch and
 * _track write none and leave what calcG refers to unchanged; before any calc_res it fails). */
int tdm_tracker_calc_g(tdm_tracker* t, float new_exposure, const double aff_g2l[2], double H[64], double b[8]);
/* Fused single-launch calcRes+calcG (no warped buffers), same outputs. */
int tdm_tracker_calc_res_g(tdm_tracker* t, const double* refToNew, float new_exposure,
                           const double aff_g2l[2], float cutoffTH, double res6[6], double H[64], double b[8]);
/* Extension (SURVEY 8e: the tracker's only parallel axis): calcRes of n_hyp (<= 64) independent motion hypotheses - the poses
 * FullSystem::trackNewCoarse tries one after the other (FullSystem.cpp:437-530) - in ONE launch and one synchronisation.
 * refToNew: n_hyp x 16, aff_g2l: n_hyp x 2, res6: n_hyp x 6; hypothesis k's result equals tdm_tracker_calc_res on that pose bit
 * for bit.  Does not disturb the buffers of the last calc_res (calc_g still refers to them). */
int tdm_tracker_calc_res_batch(tdm_tracker* t, int n_hyp, const double* refToNew, float new_exposure, const double* aff_g2l,
                               float cutoffTH, double* res6);
int tdm_tracker_synchronize(tdm_tracker* t);
int tdm_tracker_run_resident(tdm_tracker* t, int iters, float* ms_total);
/* Test accessor (not for hot paths): copies the first n (<= n_max) entries of the seven per-point arrays the last calc_res
 * wrote - u, v, dx, dy, idepth, residual, huber weight; zero at every point not accepted - to out (7 x n, array-major).
 * Synchronises the tracker's stream. */
int tdm_tracker_get_warped(tdm_tracker* t, int n, float* out);

/* ------------------------------------------------------------------------------------------------
 * SURVEY.md 8(f) "next" rows: the host stages either side of the evaluation, moved onto the device.  These entry
 * points have no counterpart in the reference's class (they replace code ABOVE its boundary); INTEGRATION.md shows
 * the three call sites in CoarseTracker.cpp / HessianBlocks.cpp that would switch to them.
 * ---------------------------------------------------------------------------------------------- */
/* n2  FrameHessian::makeImages (tandem/src/FullSystem/HessianBlocks.cpp:128-191): grey pyramid by 2x2 means +
 *     central-difference gradients for `levels` levels (level l is (w>>l) x (h>>l), globalCalib.cpp:84-85).
 *     build() uploads the w*h grey image (1.2 MB instead of the 3.7 MB float3 image setNew uploads) and is asynchronous;
 *     get_level() copies one level back (dI: (I,dx,dy) float3 per pixel; abs_squared_grad: dx^2+dy^2, no gamma weights). */
typedef struct tdm_pyramid tdm_pyramid;
int tdm_pyramid_create(int w, int h, int levels, int device, tdm_pyramid** out);
void tdm_pyramid_destroy(tdm_pyramid* p);
int tdm_pyramid_build(tdm_pyramid* p, const float* gray);
int tdm_pyramid_get_level(tdm_pyramid* p, int level, float* dI, float* abs_squared_grad);
/* setNew (cuda_coarse_tracker.cpp:99-102) without the host round trip: device-to-device from a pyramid level whose size
 * equals the tracker's (a tracker instance per level puts levels 1..3 of CoarseTracker.cpp:774 on the GPU as well). */
int tdm_tracker_set_new_from_pyramid(tdm_tracker* t, tdm_pyramid* p, int level);

/* n1  the dense part of CoarseTracker::setCoarseTrackingRef (tandem/src/FullSystem/CoarseTracker.cpp:655-732) followed by
 *     setReference: forward-warps the dense depth map (host pointer, or the render_index-th map of the last
 *     tdm_fusion_render_async - device resident, no PCIe hop) with T_depth_to_ref = ref.camToWorld^-1 * depth.camToWorld
 *     (row-major), keeps the nearest depth per target pixel, and appends the hit pixels in raster order behind the
 *     n_sparse sparse points of makeCoarseDepthL0.  pc_* hold n_sparse + 1 entries: the extra one is the slot the
 *     reference's `++pc_n` skips (CoarseTracker.cpp:717-722) and is uploaded as is; NULL is allowed when n_sparse == 0.
 *     idepth0 (h*w, the sparse inverse-depth image idepth[0]) may be NULL.  The grey values of the reference keyframe
 *     come from ref_gray (h*w floats) or from level 0 of a pyramid.  *pc_n receives the reference's pc_n[0]. */
int tdm_tracker_set_reference_dense(tdm_tracker* t, const float* depth, tdm_fusion* depth_from_fusion, int render_index,
                                    const double T_depth_to_ref[16], int tracking_step, int dense_only, int n_sparse,
                                    const float* pc_u, const float* pc_v, const float* pc_idepth, const float* pc_color,
                                    const float* idepth0, const float* ref_gray, tdm_pyramid* ref_gray_from_pyramid,
                                    float ref_exposure, const double ref_aff_g2l[2], int* pc_n);
/* Reads the first n reference points back (tests, debugging). Any output pointer may be NULL. */
int tdm_tracker_get_reference(tdm_tracker* t, int n, float* pc_u, float* pc_v, float* pc_idepth, float* pc_color);

/* n3  one pyramid level of CoarseTracker::trackNewestCoarse (CoarseTracker.cpp:761-916) without host round trips:
 *     initial evaluation with cutoff doubling (:775-790), then up to max_iterations damped Gauss-Newton steps with the
 *     reference's accept / lambda / extrapolation / termination rules; fix_a / fix_b = setting_affineOptModeA/B < 0.
 *     Blocking; the caller keeps the coarse-to-fine logic (repeat a level when cutoff_repeat > 1, abort thresholds). */
typedef struct tdm_track_result {
  double ref_to_new[16];   /* row-major */
  double aff_g2l[2];
  double res[6];           /* resOld of the accepted state: E, numTermsInE, flow T, 0, flow RT, saturated ratio */
  int iterations;          /* executed LM iterations */
  int evaluations;         /* fused residual + normal-equation evaluations launched */
  float cutoff_repeat;     /* levelCutoffRepeat */
  float device_ms;         /* CUDA-event time of the whole loop */
} tdm_track_result;
int tdm_tracker_track(tdm_tracker* t, const double refToNew[16], const double aff_g2l[2], float new_exposure,
                      float coarse_cutoff_th, int max_iterations, float lambda_extrapolation_limit, int fix_a, int fix_b,
                      tdm_track_result* out);

/* n5  CoarseTracker::trackNewestCoarse (CoarseTracker.cpp:750-936) for one motion hypothesis, all levels on the device
 *     with one host wait: levels[l] is the tracker of pyramid level l, (w0>>l) x (h0>>l), each with setK, a reference and a
 *     new image (setNewFromPyramid); the loop runs on levels[0]'s stream after the pending work of every level's stream.
 *     Per level coarsest_level..0: lambda = 0.01, cutoff doubling while > 60 % of the residuals saturate, the LM iterations
 *     of tdm_tracker_track (max_iterations[l]), lastResiduals[l] = sqrtf(E / numTermsInE), abort (ok = 0, pose unchanged)
 *     when it exceeds 1.5 * min_res_for_abort[l] (NaN never aborts), and one repeat of the first level whose cutoff had to
 *     be raised.  Then the affine checks of :923-931 with setting_affineOptModeA/B (< 0: that parameter is fixed and, if
 *     ok, reported as 0).  Levels > 0 are evaluated with the GPU definitions of calcRes / calcG (DESIGN.md, n5).
 *     Blocking.  Invalid input (missing setK / reference / new image, wrong level sizes, different devices,
 *     coarsest_level outside 0..4, max_iterations outside 0..200) is an error and launches nothing. */
typedef struct tdm_track_pyramid_result {
  double ref_to_new[16];        /* lastToNew_out (row-major); unchanged from the input when the loop aborted */
  double aff_g2l[2];            /* aff_g2l_out, after the "mode < 0 -> 0" rule of :934-935 */
  double last_residuals[5];     /* CoarseTracker::lastResiduals, NaN for levels not reached */
  double last_flow_indicators[3];
  int ok;                       /* trackNewestCoarse's return value */
  int aborted_level;            /* level whose residual exceeded 1.5 * min_res_for_abort, else -1 */
  int repeated_level;           /* level run twice by the repeat rule (:911-915), else -1 */
  int iterations[5], evaluations[5];   /* per level, summed over both passes of a repeated level */
  float cutoff_repeat[5];       /* largest levelCutoffRepeat of each level's passes */
  float device_ms;
} tdm_track_pyramid_result;
int tdm_tracker_track_pyramid(tdm_tracker* const* levels, int coarsest_level, const double refToNew[16], const double aff_g2l[2],
                              float new_exposure, float coarse_cutoff_th, const int max_iterations[5],
                              float lambda_extrapolation_limit, float affine_opt_mode_a, float affine_opt_mode_b,
                              const double min_res_for_abort[5], tdm_track_pyramid_result* out);

/* n6  FullSystem::trackNewCoarse (tandem/src/FullSystem/FullSystem.cpp:538-617), monocular path: the loop over the motion
 *     hypotheses the caller built (lastF_2_fh_tries, :420-536), every try an n5 run, all on the device with one host wait.
 *     Try i starts from tries[i] (n_tries x 16, row-major) and aff_last_2_l with min_res_for_abort = achievedRes as it stands
 *     (all NaN for the first try).  After each try, statement for statement: a winner (ok, lastResiduals[0] finite as a float
 *     and not >= achievedRes[0]) gives the pose, aff and lastFlowIndicators; once one has won, every level of achievedRes takes
 *     over the try's lastResiduals where it is not finite (as a float) or larger; the loop stops when
 *     achievedRes[0] < last_coarse_rmse[0] * retrack_threshold (setting_reTrackThreshold).  Without a winner the pose is
 *     tries[0], the aff aff_last_2_l and the flow (0, 0, 0).  The other arguments and the level requirements are those of
 *     tdm_tracker_track_pyramid.  Blocking.  Invalid input (everything tdm_tracker_track_pyramid rejects, n_tries outside 1..64,
 *     null arrays) is an error and launches nothing.  tries_out, when not NULL, receives `tries` records. */
typedef struct tdm_track_try {
  double last_residuals[5];     /* lastResiduals after the try, NaN for levels it did not reach */
  int ok;                       /* trackNewestCoarse's return value */
  int aborted_level, repeated_level;   /* as in tdm_track_pyramid_result, -1: none */
  int evaluations[5];
} tdm_track_try;
typedef struct tdm_track_new_coarse_result {
  double ref_to_new[16];        /* lastF_2_fh (row-major) */
  double aff_g2l[2];            /* aff_g2l */
  double achieved_res[5];       /* achievedRes: the caller's new lastCoarseRMSE (:617) */
  double flow_vecs[3];          /* flowVecs */
  int have_one_good;
  int tries;                    /* tryIterations: tries run */
  int winner;                   /* index of the last winning try, -1: none (not in the reference) */
  float device_ms;
} tdm_track_new_coarse_result;
int tdm_tracker_track_new_coarse(tdm_tracker* const* levels, int coarsest_level, const double* tries, int n_tries,
                                 const double aff_last_2_l[2], float new_exposure, float coarse_cutoff_th, const int max_iterations[5],
                                 float lambda_extrapolation_limit, float affine_opt_mode_a, float affine_opt_mode_b,
                                 const double last_coarse_rmse[5], float retrack_threshold, tdm_track_new_coarse_result* out,
                                 tdm_track_try* tries_out);

/* n7  CoarseTracker::setCoarseTrackingRef (tandem/src/FullSystem/CoarseTracker.cpp:633-733) including makeCoarseDepthL0
 *     (:148-374), for the trackers of levels 0..n_levels-1 ((w0>>l) x (h0>>l), as tdm_tracker_track_pyramid expects them) in
 *     one call on levels[0]'s stream.  The points are the ones the reference uses, in its order (frameHessians x
 *     pointHessians): rgbd_init == 0, those passing the lastResiduals[0] / ResState::IN test of :157 with pt_u/v/idepth =
 *     centerProjectedTo[0..2] and pt_hessian = efPoint->HdiF; rgbd_init == 1, ph->u, ph->v, ph->idepth, ph->idepth_hessian.
 *     Scatter (several points on one pixel are summed in input order), 2x2 sum pyramid, dilation, normalise-and-compact per
 *     level with the colours dIp[l][i][0] of ref_pyramid; then, with a dense map (host `depth` or the render_index-th render of
 *     depth_from_fusion, as in tdm_tracker_set_reference_dense; both NULL: none) n1's dense append behind level 0's points.
 *     Like the reference's arrays, a tracker's reference arrays persist across calls: slot pc_n[l] keeps the last candidate the
 *     reference wrote there and rejected, or what it held before.  Every level then holds pc_n[l] points with ref_exposure and
 *     ref_aff_g2l, as after setReference.  Blocking, one host wait; ordered after the pending work of every level's stream, the
 *     pyramid's build and the render.  Invalid input (null handles or arrays that are needed, n_levels outside 1..5, wrong level
 *     sizes, no setK on level 0, a pyramid with fewer levels or another level-0 size, different devices, a point whose rounded
 *     pixel - (int)(u + 0.5f) monocular, (int)(u + 0.5) RGB-D - lies outside the level-0 image) is an error and launches
 *     nothing.  A level whose n_max cannot hold its points and the slot behind them is an error found after the launch; every
 *     level's reference is then empty. */
int tdm_tracker_set_coarse_tracking_ref(tdm_tracker* const* levels, int n_levels, int rgbd_init, int n_points, const float* pt_u,
                                        const float* pt_v, const float* pt_idepth, const float* pt_hessian, tdm_pyramid* ref_pyramid,
                                        const float* depth, tdm_fusion* depth_from_fusion, int render_index,
                                        const double T_depth_to_ref[16], int tracking_step, int dense_only, float ref_exposure,
                                        const double ref_aff_g2l[2], int pc_n[5]);

/* n7 + nodia  tdm_tracker_set_coarse_tracking_ref, and in the same call on the same stream with the same host wait the rest of
 *     makeCoarseDepthL0's level-0 output that FullSystem::deliverDrFrame reads for every MVSNet window (FullSystem.cpp:1175):
 *     the undilated cloud pc_u/v/idepth/color_nodia (CoarseTracker.cpp:150-218) - candidates are the pixels of
 *     [2,w-2) x [2,h-2) with a point, accepted when their colour is finite and their unweighted idepth sum > 0 (monocular;
 *     RGB-D leaves the sums 0) - and get_idepth_quantile over it (tandem_backend.cpp:354-361): the idepth at index
 *     (int)(quantile_fraction * (float)pc_n_nodia) in sorted order and 1.0f / it.  The cloud lives in levels[0] and persists
 *     across calls like the reference's arrays: slot pc_n_nodia keeps the last rejected candidate behind the last accepted
 *     one, or what it held before.  Plain tdm_tracker_set_coarse_tracking_ref calls leave it alone.  Both quantile values are
 *     NaN when that index is not below pc_n_nodia (no accepted pixel, or quantile_fraction 1), where the reference reads
 *     outside its vector.  quantile_fraction outside [0, 1] or not finite, or a null `out`, is an error and launches nothing;
 *     everything else as tdm_tracker_set_coarse_tracking_ref.  `out` is filled even when a level's n_max turns out too small. */
typedef struct tdm_coarse_nodia_result {
  int pc_n_nodia;             /* CoarseTracker::pc_n_nodia */
  float idepth_quantile;      /* the selected pc_idepth_nodia value */
  float depth_quantile;       /* get_idepth_quantile's return value: MVSNet's depth_max is 3 * this (FullSystem.cpp:1180) */
} tdm_coarse_nodia_result;
int tdm_tracker_set_coarse_tracking_ref_nodia(tdm_tracker* const* levels, int n_levels, int rgbd_init, int n_points,
                                              const float* pt_u, const float* pt_v, const float* pt_idepth, const float* pt_hessian,
                                              tdm_pyramid* ref_pyramid, const float* depth, tdm_fusion* depth_from_fusion,
                                              int render_index, const double T_depth_to_ref[16], int tracking_step, int dense_only,
                                              float ref_exposure, const double ref_aff_g2l[2], float quantile_fraction, int pc_n[5],
                                              tdm_coarse_nodia_result* out);
/* Reads the first n entries (0..w*h) of level0's pc_u/v/idepth/color_nodia back (tests, dumps); any output pointer may be
 * NULL.  An error before the first tdm_tracker_set_coarse_tracking_ref_nodia call with level0 as levels[0]. */
int tdm_tracker_get_coarse_nodia(tdm_tracker* level0, int n, float* u, float* v, float* idepth, float* color);

#ifdef __cplusplus
}
#endif
#endif /* TANDEM_B200_H */
