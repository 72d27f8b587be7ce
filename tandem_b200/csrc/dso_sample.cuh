// Device helpers shared by the kernels that restate DSO's per-point code (immature.cu: n8 / n9, linearize.cu: n12): the
// correctly rounded float operations (no contraction), the residual pattern and the bilinear sample of a (I, dx, dy) image.
#pragma once
#include <cuda_runtime.h>

namespace tdm {
namespace {

__constant__ int c_pattern[8][2] = {{0, -2}, {-1, -1}, {1, -1}, {-2, 0}, {0, 0}, {2, 0}, {-1, 1}, {0, 2}};   // staticPattern[8]

__device__ __forceinline__ float fm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fs(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fd(float a, float b) { return __fdiv_rn(a, b); }

// (int)x in 0..w-2 and (int)y in 0..h-2: the 2x2 footprint lies in the image.  Outside it a sample is a non-finite hit.
__device__ __forceinline__ bool inside(float x, float y, int w, int h) {
  return x > -1.f && y > -1.f && x < (float)(w - 1) && y < (float)(h - 1);
}

// getInterpolatedElement33 (globalFuncs.h:75-89), components 0..C-1 (C = 1: getInterpolatedElement31, :126-140)
template <int C>
__device__ __forceinline__ void interp(const float* __restrict__ dI, float x, float y, int w, float* out) {
  const int ix = (int)x, iy = (int)y;
  const float dx = fs(x, (float)ix), dy = fs(y, (float)iy), dxdy = fm(dx, dy);
  const float* bp = dI + 3 * ((long long)ix + (long long)iy * w);
  const float w0 = dxdy, w1 = fs(dy, dxdy), w2 = fs(dx, dxdy), w3 = fa(fs(fs(1.f, dx), dy), dxdy);
#pragma unroll
  for (int k = 0; k < C; ++k)
    out[k] = fa(fa(fa(fm(w0, __ldg(bp + 3 * (1 + w) + k)), fm(w1, __ldg(bp + 3 * w + k))), fm(w2, __ldg(bp + 3 + k))),
                fm(w3, __ldg(bp + k)));
}

}  // namespace
}  // namespace tdm
