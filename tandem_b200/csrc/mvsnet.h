// Type-erased interface of the CVA-MVSNet engine (implemented in mvsnet.cu for fp32 and bf16 storage).
#pragma once
#include <functional>
#include <string>

namespace tdm {

class MvsnetIface {
 public:
  // The result the last GetResult returned, kept on the engine's device until the next GetResult (the keyframe handoff to the
  // TSDF, tdm_fusion_integrate_mvsnet): filtered stage-3 depth, the reference view's BGR and its cam_to_world.
  struct Handoff {
    const float* depth;          // H*W
    const unsigned char* bgr;    // H*W*3, the reference view's image
    float c2w[16];
    int H, W, device;
    void* ready;                 // cudaEvent_t recorded behind the copy that filled the buffers
  };
  virtual ~MvsnetIface() = default;
  virtual void set_option(const std::string& key, int value) = 0;
  // K3x3x3: three row-major 3x3 intrinsics, stage1..stage3.
  virtual void call_async(int H, int W, int V, int ref_index, unsigned char* const* bgrs, const float* K3x3x3,
                          float* const* c2ws, float dmin, float dmax, float discard) = 0;
  // Feature cache (tdm_mvsnet_call_async_ids): views are named by caller ids; FeatureNet runs only for the ids the handle does
  // not hold, whose bgrs[i] must be non-null (the bgrs of held ids are ignored).
  virtual void call_async_ids(int H, int W, int V, int ref_index, const long long* ids, unsigned char* const* bgrs,
                              const float* K3x3x3, float* const* c2ws, float dmin, float dmax, float discard) = 0;
  // ids held (the last cached call's window, in its order; none after a plain call_async) and the views the last call computed
  virtual void feature_cache(long long* ids, int cap, int* n_ids, int* n_computed) = 0;
  virtual bool ready() = 0;
  virtual void wait() = 0;
  virtual void get_result(float* depth, float* conf, float* depth_dense, float* conf_dense) = 0;
  // Calls consume(handoff) under the engine's lock.  consume enqueues every read of the handoff on `stream` (a cudaStream_t
  // of the handoff's device) behind handoff.ready; the engine then records a release event on `stream` that the next
  // GetResult's fill and the destructor wait for.  Throws when no result has been fetched yet.
  virtual void read_handoff(void* stream, const std::function<void(const Handoff&)>& consume) = 0;
  virtual void stage_output(int stage, const std::string& which, float* out, size_t cap) = 0;
  virtual long long debug_tensor(const std::string& name, float* out, size_t cap, int* dims4) = 0;
  virtual void run_resident(int iters, float* ms_total, int* launches) = 0;
  // the last window's forward with FeatureNet recomputing only its last n_new views (window order), the others read from the pool
  virtual void run_resident_new(int n_new, int iters, float* ms_total, int* launches) = 0;
  virtual std::string profile() = 0;
  // building blocks of tdm_mvsnet_run_resident_multi (several engines of one device timed together)
  virtual void* resident_stream() = 0;                 // cudaStream_t
  virtual int resident_device() const = 0;
  virtual int resident_launch(int iters) = 0;          // enqueue iters forwards, no synchronisation; returns launches per forward
};

MvsnetIface* make_mvsnet(const std::string& weights_path, int precision, int device);
void debug_homography(const float* K3x3, const float* c2w_ref, const float* c2w_src, float* rot9, float* trans3);
void debug_conv_plan(int cin, int npad, int kd, int D, int H, int W, int pd, int mode, int smem_kb, long long* out, int n);

}  // namespace tdm
