// DrMvsnet -> DrFusion keyframe chain through the header-compatible C++ shims, in TandemBackendImpl::CallSequential's order
// (tandem_backend.cpp:137-200): GetResult(k-1) -> CallAsync(k) -> IntegrateScanAsync(*mvsnet) of window k-1 -> RenderAsync ->
// GetRenderResult.  The integration uses the device-side overload DrFusion::IntegrateScanAsync(DrMvsnet const&, nullptr).
// Run by tests/test_keyframe_handoff_gpu.py, which writes the input sequence and compares the renders with the host path.
//
// input  "TDMK0001", i32 n_frames, V, H, W, f32 K[9], dmin, dmax, discard, then per frame f32 c2w[16] + u8 bgr[H*W*3];
//        window k = frames k .. k+V-1 with the reference at V-2 (FullSystem.cpp:1127)
// output per integrated window: f32 render depth[H*W] + u8 render bgr[H*W*3], rendered at that window's reference pose
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <vector>

#include "dr_fusion/dr_fusion.h"
#include "dr_mvsnet/dr_mvsnet.h"

int main(int argc, char** argv) {
  if (argc < 4) { printf("usage: shim_keyframe <weights.tdmw> <frames.bin> <renders.bin>\n"); return 2; }
  std::ifstream f(argv[2], std::ios::binary);
  char magic[8];
  f.read(magic, 8);
  if (!f || std::memcmp(magic, "TDMK0001", 8) != 0) { printf("bad input container\n"); return 2; }
  int32_t n, V, H, W;
  f.read((char*)&n, 4); f.read((char*)&V, 4); f.read((char*)&H, 4); f.read((char*)&W, 4);
  float K[9], dmin, dmax, discard;
  f.read((char*)K, 36); f.read((char*)&dmin, 4); f.read((char*)&dmax, 4); f.read((char*)&discard, 4);
  const size_t img = (size_t)H * W * 3;
  std::vector<float> c2w((size_t)n * 16);
  std::vector<unsigned char> bgr((size_t)n * img);
  for (int i = 0; i < n; ++i) {
    f.read((char*)&c2w[(size_t)i * 16], 64);
    f.read((char*)&bgr[(size_t)i * img], img);
  }
  if (!f) { printf("truncated input container\n"); return 2; }

  DrMvsnet mvsnet(argv[1]);
  DrFusionOptions o{};   // the test's host path uses the same options
  o.voxel_size = 0.01f; o.num_buckets = 100003; o.bucket_size = 10; o.num_blocks = 200000; o.block_size = 8;
  o.max_sdf_weight = 64; o.truncation_distance = 0.04f; o.max_sensor_depth = 10.f; o.min_sensor_depth = 0.1f;
  o.num_render_streams = 1; o.fx = K[0]; o.fy = K[4]; o.cx = K[2]; o.cy = K[5]; o.height = H; o.width = W;
  DrFusion fusion(o);
  std::ofstream out(argv[3], std::ios::binary);

  const int nw = n - V + 1, ref = V - 2;
  for (int k = 0; k <= nw; ++k) {
    DrMvsnetOutput* result = nullptr;
    if (k > 0) result = mvsnet.GetResult();
    if (k < nw) {
      std::vector<unsigned char*> bp(V);
      std::vector<float*> cp(V);
      for (int v = 0; v < V; ++v) { bp[v] = &bgr[(size_t)(k + v) * img]; cp[v] = &c2w[(size_t)(k + v) * 16]; }
      mvsnet.CallAsync(H, W, V, ref, bp.data(), K, cp.data(), dmin, dmax, discard);
    }
    if (result) {
      fusion.IntegrateScanAsync(mvsnet, nullptr);
      const float* pose = &c2w[(size_t)(k - 1 + ref) * 16];
      fusion.RenderAsync({pose});
      std::vector<unsigned char*> rb;
      std::vector<float*> rd;
      fusion.GetRenderResult(rb, rd);
      out.write((const char*)rd[0], (std::streamsize)H * W * 4);
      out.write((const char*)rb[0], (std::streamsize)img);
      delete result;
    }
  }
  out.close();
  printf("shim_keyframe: %d windows integrated\n", nw);
  return out ? 0 : 1;
}
