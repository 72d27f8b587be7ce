// Test infrastructure: C entry points around the REFERENCE's own `class DrFusion`
// (tandem/libdr/dr_fusion/src/dr_fusion/dr_fusion.h), compiled unmodified from /root/reference by
// oracle/ref_build.mk into oracle/_ref/libdr_fusion_ref.so.  Used only by tests (-m gpu) to pin our CPU oracle and
// CUDA path against the reference (oracle/gen_reference_pins.py) and as a GPU baseline (tools/bench_fusion_tracker.py).
#include <cstdlib>
#include <cstring>
#include <vector>

#include "dr_fusion/dr_fusion.h"

extern "C" {

void* ref_fusion_create(const DrFusionOptions* o) { return new DrFusion(*o); }
void ref_fusion_destroy(void* h) { delete static_cast<DrFusion*>(h); }
void ref_fusion_integrate(void* h, unsigned char* bgr, float* depth, const float* pose) {
  static_cast<DrFusion*>(h)->IntegrateScanAsync(bgr, depth, pose);
}
// renders one pose and copies the result out (height*width*3 u8, height*width f32)
void ref_fusion_render(void* h, const float* pose, unsigned char* bgr_out, float* depth_out, int npx) {
  DrFusion* f = static_cast<DrFusion*>(h);
  f->RenderAsync({pose});
  std::vector<unsigned char*> b;
  std::vector<float*> d;
  f->GetRenderResult(b, d);
  std::memcpy(bgr_out, b[0], (size_t)npx * 3);
  std::memcpy(depth_out, d[0], (size_t)npx * 4);
}
void ref_fusion_sync(void* h) { static_cast<DrFusion*>(h)->Synchronize(); }

}  // extern "C"

// DrFusion::GetMesh (dr_fusion.cpp:95-149) - vertices / colours copied out, the reference's mallocs released
extern "C" long long ref_fusion_get_mesh(void* h, float* lower, float* upper, float* vert, float* cols, long long cap_vertices) {
  DrMesh m = static_cast<DrFusion*>(h)->GetMesh(lower, upper);
  const long long n = (long long)m.num;
  const long long k = n < cap_vertices ? n : cap_vertices;
  if (k > 0 && vert && cols) {
    std::memcpy(vert, m.vert, (size_t)k * 3 * sizeof(float));
    std::memcpy(cols, m.cols, (size_t)k * 3 * sizeof(float));
  }
  free(m.vert);
  free(m.cols);
  return n;
}
