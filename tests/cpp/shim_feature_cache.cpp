// A sliding keyframe window through the header-compatible DrMvsnet shim's feature-cache overload,
// DrMvsnet::CallAsync(..., std::vector<long long> const& view_ids, ...), in TandemBackendImpl::CallSequential's order
// (GetResult(k-1) -> CallAsync(k)).  Each keyframe's id is its frame index and its image is passed only in the window that
// adds it (NULL for the ids the handle holds).  Run by tests/test_mvsnet_feature_cache_gpu.py, which writes the input
// sequence and compares the maps with tdm_mvsnet_call_async on a fresh handle.
//
// input  "TDMK0001", i32 n_frames, V, H, W, f32 K[9], dmin, dmax, discard, then per frame f32 c2w[16] + u8 bgr[H*W*3];
//        window k = frames k .. k+V-1 with the reference at V-2 (FullSystem.cpp:1127)
// output per window: f32 depth[H*W], confidence[H*W], depth_dense[H*W], confidence_dense[H*W]
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <vector>

#include "dr_mvsnet/dr_mvsnet.h"

int main(int argc, char** argv) {
  if (argc < 4) { printf("usage: shim_feature_cache <weights.tdmw> <frames.bin> <maps.bin>\n"); return 2; }
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
  std::ofstream out(argv[3], std::ios::binary);
  const int nw = n - V + 1, ref = V - 2;
  for (int k = 0; k <= nw; ++k) {
    if (k > 0) {
      DrMvsnetOutput* r = mvsnet.GetResult();
      for (const float* m : {r->depth, r->confidence, r->depth_dense, r->confidence_dense})
        out.write((const char*)m, (std::streamsize)H * W * 4);
      delete r;
    }
    if (k < nw) {
      std::vector<long long> ids(V);
      std::vector<unsigned char*> bp(V);
      std::vector<float*> cp(V);
      for (int v = 0; v < V; ++v) {
        ids[v] = k + v;
        // the first window brings every image; later ones only the keyframe they add
        bp[v] = (k == 0 || v == V - 1) ? &bgr[(size_t)(k + v) * img] : nullptr;
        cp[v] = &c2w[(size_t)(k + v) * 16];
      }
      mvsnet.CallAsync(H, W, V, ref, ids, bp.data(), K, cp.data(), dmin, dmax, discard);
    }
  }
  out.close();
  printf("shim_feature_cache: %d windows\n", nw);
  return out ? 0 : 1;
}
