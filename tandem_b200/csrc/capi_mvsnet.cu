// extern "C" entry points for the MVSNet engine + library-wide helpers (include/tandem_b200.h).
#include <vector>
#include <cstring>
#include <string>

#include "../../include/tandem_b200.h"
#include "capi_common.h"
#include "common.cuh"
#include "mvsnet.h"

namespace tdm {
static thread_local std::string g_last_error;
void set_last_error(const std::string& s) { g_last_error = s; }
}  // namespace tdm

struct tdm_mvsnet {
  tdm::MvsnetIface* impl;
};

extern "C" {

const char* tdm_last_error(void) { return tdm::g_last_error.c_str(); }
const char* tdm_version(void) { return "tandem_b200 0.1.0 sm_90a"; }
int tdm_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int tdm_host_alloc_pinned(size_t bytes, void** out) {
  TDM_API_BEGIN
  TDM_CHECK(out && bytes > 0, "null argument");
  TDM_CUDA(cudaHostAlloc(out, bytes, cudaHostAllocPortable));
  return TDM_OK;
  TDM_API_END
}
int tdm_host_free_pinned(void* p) {
  TDM_API_BEGIN
  if (p) TDM_CUDA(cudaFreeHost(p));
  return TDM_OK;
  TDM_API_END
}

int tdm_debug_homography(const float* K3x3, const float* c2w_ref, const float* c2w_src, float* rot9, float* trans3) {
  TDM_API_BEGIN
  TDM_CHECK(K3x3 && c2w_ref && c2w_src && rot9 && trans3, "null argument");
  tdm::debug_homography(K3x3, c2w_ref, c2w_src, rot9, trans3);
  return TDM_OK;
  TDM_API_END
}

int tdm_debug_conv_plan(int cin, int npad, int kd, int D, int H, int W, int pd, int mode, int smem_kb, long long* out12) {
  TDM_API_BEGIN
  TDM_CHECK(out12 && cin >= 8 && npad >= 8 && (kd == 1 || kd == 2 || kd == 3) && D > 0 && H > 0 && W > 0, "bad argument");
  tdm::debug_conv_plan(cin, npad, kd, D, H, W, pd, mode, smem_kb, out12);
  return TDM_OK;
  TDM_API_END
}

int tdm_mvsnet_create(const char* weights_path, int precision, int device, tdm_mvsnet** out) {
  TDM_API_BEGIN
  TDM_CHECK(weights_path && out, "null argument");
  *out = new tdm_mvsnet{tdm::make_mvsnet(weights_path, precision, device)};
  return TDM_OK;
  TDM_API_END
}
void tdm_mvsnet_destroy(tdm_mvsnet* h) {
  if (!h) return;
  try { delete h->impl; } catch (...) {}
  delete h;
}
int tdm_mvsnet_call_async_k(tdm_mvsnet* h, int height, int width, int view_num, int ref_index,
                            unsigned char* const* bgrs, const float* Ks, float* const* c2ws, float dmin,
                            float dmax, float discard) {
  TDM_API_BEGIN
  TDM_CHECK(h && bgrs && Ks && c2ws, "null argument");
  h->impl->call_async(height, width, view_num, ref_index, bgrs, Ks, c2ws, dmin, dmax, discard);
  return TDM_OK;
  TDM_API_END
}
int tdm_mvsnet_call_async(tdm_mvsnet* h, int height, int width, int view_num, int ref_index,
                          unsigned char* const* bgrs, const float* K, float* const* c2ws, float dmin,
                          float dmax, float discard) {
  TDM_API_BEGIN
  TDM_CHECK(h && bgrs && K && c2ws, "null argument");
  // K_stage3 = K, K_stage2 rows 0-1 * 0.5, K_stage1 rows 0-1 * 0.25 (dr_mvsnet.cpp:220-247, incl. its TODO)
  float Ks[27];
  const float sc[3] = {0.25f, 0.5f, 1.0f};
  for (int s = 0; s < 3; ++s)
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j)
        Ks[s * 9 + i * 3 + j] = (i < 2) ? (float)((double)sc[s] * (double)K[i * 3 + j]) : K[i * 3 + j];
  h->impl->call_async(height, width, view_num, ref_index, bgrs, Ks, c2ws, dmin, dmax, discard);
  return TDM_OK;
  TDM_API_END
}
int tdm_mvsnet_get_result(tdm_mvsnet* h, float* depth, float* confidence, float* depth_dense, float* confidence_dense) {
  TDM_API_BEGIN
  TDM_CHECK(h, "null handle");
  h->impl->get_result(depth, confidence, depth_dense, confidence_dense);
  return TDM_OK;
  TDM_API_END
}
int tdm_mvsnet_ready(tdm_mvsnet* h) {
  TDM_API_BEGIN
  TDM_CHECK(h, "null handle");
  return h->impl->ready() ? 1 : 0;
  TDM_API_END
}
int tdm_mvsnet_wait(tdm_mvsnet* h) {
  TDM_API_BEGIN
  TDM_CHECK(h, "null handle");
  h->impl->wait();
  return TDM_OK;
  TDM_API_END
}
int tdm_mvsnet_set_option(tdm_mvsnet* h, const char* key, int value) {
  TDM_API_BEGIN
  TDM_CHECK(h && key, "null argument");
  h->impl->set_option(key, value);
  return TDM_OK;
  TDM_API_END
}
int tdm_mvsnet_stage_output(tdm_mvsnet* h, int stage, const char* which, float* out, size_t capacity) {
  TDM_API_BEGIN
  TDM_CHECK(h && which && out, "null argument");
  h->impl->stage_output(stage, which, out, capacity);
  return TDM_OK;
  TDM_API_END
}
long long tdm_mvsnet_debug_tensor(tdm_mvsnet* h, const char* name, float* out, size_t capacity, int* dims4) {
  TDM_API_BEGIN
  TDM_CHECK(h && name, "null argument");
  return h->impl->debug_tensor(name, out, capacity, dims4);
  TDM_API_END
}
int tdm_mvsnet_run_resident(tdm_mvsnet* h, int iters, float* ms_total, int* launches) {
  TDM_API_BEGIN
  TDM_CHECK(h && ms_total, "null argument");
  h->impl->run_resident(iters, ms_total, launches);
  return TDM_OK;
  TDM_API_END
}
int tdm_mvsnet_run_resident_multi(tdm_mvsnet* const* hs, int n, int iters_total, float* ms_total, int* launches) {
  TDM_API_BEGIN
  TDM_CHECK(hs && ms_total && n >= 1 && n <= 16 && iters_total >= 1, "bad argument");
  for (int j = 0; j < n; ++j) TDM_CHECK(hs[j] && hs[j]->impl->resident_device() == hs[0]->impl->resident_device(), "handles must share a device");
  TDM_CUDA(cudaSetDevice(hs[0]->impl->resident_device()));
  std::vector<cudaStream_t> st(n);
  for (int j = 0; j < n; ++j) st[j] = (cudaStream_t)hs[j]->impl->resident_stream();
  hs[0]->impl->resident_launch(0);   // drains every engine's worker before the clock starts
  for (int j = 1; j < n; ++j) hs[j]->impl->resident_launch(0);
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& e : ev) TDM_CUDA(cudaEventCreate(&e));
  TDM_CUDA(cudaEventRecord(ev[0], st[0]));
  for (int j = 1; j < n; ++j) TDM_CUDA(cudaStreamWaitEvent(st[j], ev[0], 0));
  int nl = 0;
  for (int it = 0; it < iters_total; ++it) nl = hs[it % n]->impl->resident_launch(1);   // round robin, one stream per engine
  for (int j = 1; j < n; ++j) {
    TDM_CUDA(cudaEventRecord(ev[j], st[j]));
    TDM_CUDA(cudaStreamWaitEvent(st[0], ev[j], 0));
  }
  TDM_CUDA(cudaEventRecord(ev[n], st[0]));
  TDM_CUDA(cudaEventSynchronize(ev[n]));
  TDM_CUDA(cudaEventElapsedTime(ms_total, ev[0], ev[n]));
  for (auto& e : ev) cudaEventDestroy(e);
  if (launches) *launches = nl;
  return TDM_OK;
  TDM_API_END
}
long long tdm_mvsnet_profile(tdm_mvsnet* h, char* buf, size_t capacity) {
  TDM_API_BEGIN
  TDM_CHECK(h && buf && capacity > 0, "null argument");
  std::string s = h->impl->profile();
  if (s.size() + 1 > capacity) s.resize(capacity - 1);
  std::memcpy(buf, s.c_str(), s.size() + 1);
  return (long long)s.size();
  TDM_API_END
}

}  // extern "C"
