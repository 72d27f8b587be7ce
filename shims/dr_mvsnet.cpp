// class DrMvsnet over the tandem_b200 C ABI (replaces tandem/libdr/dr_mvsnet/src/dr_mvsnet.cpp).
// Error convention of the reference: print to std::cerr and exit(EXIT_FAILURE) (dr_mvsnet.cpp:101-102,157,315-318).
#include "dr_mvsnet/dr_mvsnet.h"

#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <vector>

#include "tandem_b200.h"

class DrMvsnetImpl {
 public:
  tdm_mvsnet* h = nullptr;
  int height = 0, width = 0;
};

static void die(const char* where) {
  std::cerr << "ERROR: " << where << ": " << tdm_last_error() << std::endl;
  exit(EXIT_FAILURE);
}

// The reference constructor has no precision / device argument (dr_mvsnet.h:38), so the two choices a deployment may want
// come from the environment: TDM_PRECISION = mixed16 (default; benchmark precision) | fp32 (parity engine, Abs Rel 2e-6 vs
// the reference's fp32 model) | bf16, and TDM_DEVICE = CUDA ordinal (default 0).  Documented in INTEGRATION.md.
static int env_precision() {
  const char* p = getenv("TDM_PRECISION");
  if (!p || !*p || !strcmp(p, "mixed16")) return TDM_PRECISION_MIXED16;
  if (!strcmp(p, "fp32")) return TDM_PRECISION_FP32;
  if (!strcmp(p, "bf16")) return TDM_PRECISION_BF16;
  std::cerr << "ERROR: DrMvsnet: TDM_PRECISION must be mixed16, fp32 or bf16 (got '" << p << "')" << std::endl;
  exit(EXIT_FAILURE);
}
static int env_device() {
  const char* d = getenv("TDM_DEVICE");
  return d && *d ? atoi(d) : 0;
}

DrMvsnet::DrMvsnet(char const* filename) {
  impl = new DrMvsnetImpl();
  if (tdm_mvsnet_create(filename, env_precision(), env_device(), &impl->h) != TDM_OK) die("DrMvsnet::DrMvsnet");
}

DrMvsnet::~DrMvsnet() {
  tdm_mvsnet_destroy(impl->h);  // waits for in-flight work and joins the worker (dr_mvsnet.cpp:28-38)
  delete impl;
}

void DrMvsnet::CallAsync(int height, int width, int view_num, int ref_index, unsigned char** bgrs,
                         float const* intrinsic_matrix, float** cam_to_worlds, float depth_min, float depth_max,
                         float discard_percentage, bool debug_print) {
  if (debug_print)
    printf("--- DrMvsnet::CallAsync --- W=%d, H=%d, view_num=%d, ref_index=%d, depth_min=%f, depth_max=%f, discard=%f\n",
           width, height, view_num, ref_index, depth_min, depth_max, discard_percentage);
  impl->height = height;
  impl->width = width;
  if (tdm_mvsnet_call_async(impl->h, height, width, view_num, ref_index, bgrs, intrinsic_matrix, cam_to_worlds, depth_min,
                            depth_max, discard_percentage) != TDM_OK)
    die("DrMvsnet::CallAsync");
}

void DrMvsnet::CallAsync(int height, int width, int view_num, int ref_index, std::vector<long long> const& view_ids,
                         unsigned char** bgrs, float const* intrinsic_matrix, float** cam_to_worlds, float depth_min,
                         float depth_max, float discard_percentage, bool debug_print) {
  if (debug_print)
    printf("--- DrMvsnet::CallAsync (feature cache) --- W=%d, H=%d, view_num=%d, ref_index=%d, depth_min=%f, depth_max=%f, discard=%f\n",
           width, height, view_num, ref_index, depth_min, depth_max, discard_percentage);
  if ((int)view_ids.size() != view_num) {
    std::cerr << "ERROR: DrMvsnet::CallAsync: " << view_ids.size() << " view ids for " << view_num << " views" << std::endl;
    exit(EXIT_FAILURE);
  }
  impl->height = height;
  impl->width = width;
  if (tdm_mvsnet_call_async_ids(impl->h, height, width, view_num, ref_index, view_ids.data(), bgrs, intrinsic_matrix, 0,
                                cam_to_worlds, depth_min, depth_max, discard_percentage) != TDM_OK)
    die("DrMvsnet::CallAsync");
}

DrMvsnetOutput* DrMvsnet::GetResult() {
  DrMvsnetOutput* out = new DrMvsnetOutput(impl->height, impl->width);
  if (tdm_mvsnet_get_result(impl->h, out->depth, out->confidence, out->depth_dense, out->confidence_dense) != TDM_OK)
    die("DrMvsnet::GetResult");
  return out;  // ownership is the caller's (TandemBackend never frees it, SURVEY.md Appendix B.7; not our business)
}

void DrMvsnet::Wait() {
  if (tdm_mvsnet_wait(impl->h) != TDM_OK) die("DrMvsnet::Wait");
}

bool DrMvsnet::Ready() { return tdm_mvsnet_ready(impl->h) == 1; }

tdm_mvsnet* DrMvsnet::handle() const { return impl->h; }

// ---- known-answer test on the converted golden container -------------------------------------------------------
// sample_inputs.bin (tools/convert_sample_inputs.py): "TDMS0001", i32 V,H,W, f32 K[9] (stage 3), f32 dmin,dmax,discard,
// f32 c2w[V*16], u8 bgr[V*H*W*3] (window order, reference at V-2), f32 depth[H*W], f32 confidence[H*W] (stage 3 filtered).
bool test_dr_mvsnet(DrMvsnet& model, char const* filename_inputs, bool print, int repetitions, char const* out_folder) {
  (void)out_folder;
  std::ifstream f(filename_inputs, std::ios::binary);
  if (!f) { std::cerr << "test_dr_mvsnet: cannot open " << filename_inputs << std::endl; return false; }
  char magic[8];
  f.read(magic, 8);
  if (std::memcmp(magic, "TDMS0001", 8) != 0) { std::cerr << "test_dr_mvsnet: bad container" << std::endl; return false; }
  int32_t V, H, W;
  f.read((char*)&V, 4); f.read((char*)&H, 4); f.read((char*)&W, 4);
  float K[9], dmin, dmax, discard;
  f.read((char*)K, 36); f.read((char*)&dmin, 4); f.read((char*)&dmax, 4); f.read((char*)&discard, 4);
  std::vector<float> c2w((size_t)V * 16);
  f.read((char*)c2w.data(), c2w.size() * 4);
  std::vector<unsigned char> bgr((size_t)V * H * W * 3);
  f.read((char*)bgr.data(), bgr.size());
  std::vector<float> depth_ref((size_t)H * W), conf_ref((size_t)H * W);
  f.read((char*)depth_ref.data(), depth_ref.size() * 4);
  f.read((char*)conf_ref.data(), conf_ref.size() * 4);
  if (!f) { std::cerr << "test_dr_mvsnet: truncated container" << std::endl; return false; }
  std::vector<unsigned char*> bp(V);
  std::vector<float*> cp(V);
  for (int v = 0; v < V; ++v) { bp[v] = bgr.data() + (size_t)v * H * W * 3; cp[v] = c2w.data() + (size_t)v * 16; }
  const int ref_index = V - 2;  // dr_mvsnet.cpp:405
  bool ok = true;
  double t_sum = 0;
  const int warmup = 5;         // dr_mvsnet.cpp:468
  for (int rep = 0; rep < repetitions + warmup; ++rep) {
    auto t0 = std::chrono::high_resolution_clock::now();
    model.CallAsync(H, W, V, ref_index, bp.data(), K, cp.data(), dmin, dmax, discard, false);
    DrMvsnetOutput* out = model.GetResult();
    double ms = std::chrono::duration<double, std::milli>(std::chrono::high_resolution_clock::now() - t0).count();
    if (rep >= warmup) t_sum += ms;
    double ed = 0, ec = 0;
    for (size_t i = 0; i < depth_ref.size(); ++i) {
      ed += std::fabs(out->depth[i] - depth_ref[i]);
      ec += std::fabs(out->confidence[i] - conf_ref[i]);
    }
    ed /= depth_ref.size(); ec /= depth_ref.size();
    const double atol = 1e-2;   // dr_mvsnet.cpp:508-513
    if (!(ed < atol) || !(ec < atol)) ok = false;
    if (print) printf("test_dr_mvsnet rep %d: depth mean-abs %.3e, confidence mean-abs %.3e, %.2f ms\n", rep, ed, ec, ms);
    delete out;
  }
  if (print && repetitions > 0) printf("test_dr_mvsnet: CallAsync+GetResult %.2f ms avg over %d reps\n", t_sum / repetitions, repetitions);
  return ok;
}
