// Tensor-core convolution: im2col-free implicit GEMM on Hopper's warpgroup MMA (wgmma), fed by tiled TMA.  Replaces
// cuDNN's per-layer library calls of the reference (module.forward, dr_mvsnet.cpp:294) for every stride-1 3x3(x3)
// convolution of FeatureNet / CostRegNet (module.py:496-531, 577-600).
//
// Formulation ("flattened zero-haloed planes"): activations are P8, i.e. [C/8][D+2][H+2][W+2][8] with zero halos
// (mvsnet_kernels.cuh).  A CTA owns an output tile of R rows x TW columns x DR planes.  For every input plane it
// needs, (R+2) row segments of TW+2 positions per channel group are copied by TMA into a shared-memory tile of pitch
// P = TW+2 positions.  Flattening (row, col) -> l = row*P + col makes every tap (kh,kw) a CONSTANT shift kh*P + kw of
// l, so the A operand of tap (kd,kh,kw) for the 64 output positions l0..l0+63 is the same shared-memory tile read
// through a descriptor whose start address is advanced by (l0 + kh*P + kw)*16 bytes:
//   K-major, no-swizzle canonical layout  ((8,m),(8,2)) : ((16 B, SBO = 128 B), (2 B, LBO))
//   rows = positions (16 B apart), SBO = 8 positions, LBO = distance between the two 8-channel halves of a K=16 step
//   (the next channel group's plane for CIN >= 16, the next tap's shift for CIN == 8).
// Outputs computed for the 2 pad columns of each row are garbage and masked in the epilogue (utilisation TW/(TW+2)).
// B (weights, all taps) is pre-arranged on the host in the same canonical core-matrix order and stays resident.
//
// Roles (288 threads): warpgroups 0 and 1 consume, warp 8 produces (one lane issues the TMA copies).  A plane's
// 64-position sub-chunks alternate between the two consumer warpgroups; each accumulates its sub-chunk in registers
// (m64nNk16, one instruction per K=16 step) and runs the epilogue (bias / ReLU / skip / store) straight from the
// accumulator fragment, so one warpgroup's epilogue overlaps the other's MMAs.
#pragma once
#include <cuda.h>

#include <cmath>
#include <vector>

#include "common.cuh"
#include "mvsnet_kernels.cuh"

namespace tdm {
namespace tc {

struct Geom {
  int D, H, W;            // output == input dims (stride 1, pad 1)
  int Hp, Wp;             // H+2, W+2
  int pd;                 // 1: 3-D conv (KD = 3, halo planes exist), 0: 2-D conv over independent planes (KD = 1)
  long long in_gs, out_gs, res_gs;   // channel-group strides in elements
  int R, TW, DR;          // tile: rows, cols, output planes
  int P;                  // TW + 2
  int nch;                // 128-position chunks per plane = ceil(R*P / 128), each two 64-position wgmma sub-chunks
  int slot_pos;           // positions per (ring slot, channel group)
  int tiles_w, tiles_h, tiles_d;
  int relu, has_res;
  int cout;               // real output channels (<= NPAD)
  int S;                  // ring slots
  int oHp, oWp, opd;      // padded dims / D halo of the OUTPUT tensor (differs from the input in deconv mode)
  int iDp;                // padded plane count of the input: tensor-map dim 3 = channel_group * iDp + plane
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must abort the kernel (trap -> launch error), never hang the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try(bar, parity))
    if (clock64() - t0 > 4000000000ll) __trap();   // ~2 s at 1.9 GHz: no legitimate wait in these kernels is that long
}
// 1-D TMA bulk copy global -> shared, completion counted on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// wgmma shared-memory matrix descriptor (sm_90): start[0,14) lbo[16,30) sbo[32,46), all in 16-byte units; base offset 0,
// layout type 0 (no swizzle).  SBO is always 128 B (8 rows of 16 B), so the high word is a constant.
constexpr uint32_t kDescHi = 128u >> 4;
__device__ __forceinline__ uint64_t desc(uint32_t start16, uint32_t lbo16) {
  return ((uint64_t)kDescHi << 32) | (uint64_t)((start16 & 0x3FFFu) | (lbo16 << 16));
}

// D[64 x N] (+)= A[64 x 16] * B[16 x N], both operands K-major in shared memory, fp32 accumulators in registers.
// Fragment: d[4j + 2i + e] is row (warp % 4) * 16 + lane / 4 + 8i, column 8j + 2 * (lane % 4) + e.
template <int N, typename T> __device__ __forceinline__ void wgmma(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t acc);
template <> __device__ __forceinline__ void wgmma<16, __half>(float (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma<16, __nv_bfloat16>(float (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma<32, __half>(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma<32, __nv_bfloat16>(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma<64, __half>(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma<64, __nv_bfloat16>(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma<128, __half>(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma<128, __nv_bfloat16>(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// Tiled TMA load of one box of a 4-D tensor map (SASS: UTMALDG); out-of-bounds elements are zero-filled.
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* tmap, int x0, int x1, int x2, int x3, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];" ::"r"(
          smem_u32(dst)),
      "l"(tmap), "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(smem_u32(bar))
      : "memory");
}

// Programmatic dependent launch: a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may start
// while its predecessor drains; everything before pdl_wait() (barrier init, the weight image load) overlaps the
// predecessor's tail, everything that touches activations comes after it.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

constexpr int kConsumerWG = 2;                       // consumer warpgroups (warps 0..7)
constexpr int kThreads = 128 * kConsumerWG + 32;     // + the producer warp
constexpr int kProducerWarp = 4 * kConsumerWG;

// One 64-position sub-chunk of one output plane: every (kd, K=16 step) is one wgmma.  aoff(b) is the A offset of step b
// inside an input plane's ring slot, alo(b) its LBO (16-byte units); B block (kd, b) starts at b_base16 + (kd*NBLK+b)*N*2.
template <int N, typename T, int KD, int NBLK, typename AOff, typename ALbo>
__device__ __forceinline__ void mma_subchunk(float (&acc)[N / 2], const uint32_t (&slot16)[KD], uint32_t sub16, uint32_t b_base16,
                                             uint32_t b_lbo16, AOff aoff, ALbo alo) {
  wgmma_fence();
#pragma unroll
  for (int kd = 0; kd < KD; ++kd) {
#pragma unroll
    for (int b = 0; b < NBLK; ++b) {
      const uint64_t ad = desc(slot16[kd] + sub16 + aoff(b), alo(b));
      const uint64_t bd = desc(b_base16 + (uint32_t)((kd * NBLK + b) * N * 2), b_lbo16);
      wgmma<N, T>(acc, ad, bd, (kd | b) != 0 ? 1u : 0u);
    }
  }
  wgmma_commit();
  wgmma_wait_all();
}

// Two consecutive channels of an 8-channel group: one 4-byte store / load.
template <typename T> __device__ __forceinline__ void store2(T* p, float x0, float x1) {
  T v[2] = {from_f<T>(x0), from_f<T>(x1)};
  *reinterpret_cast<uint32_t*>(p) = *reinterpret_cast<const uint32_t*>(v);
}
template <typename T> __device__ __forceinline__ void load2(const T* p, float& x0, float& x1) {
  const uint32_t u = __ldg(reinterpret_cast<const unsigned int*>(p));
  const T* v = reinterpret_cast<const T*>(&u);
  x0 = to_f<T>(v[0]); x1 = to_f<T>(v[1]);
}

// Per-pixel tail of the OUT_PLAIN (prob) instantiation: with tiles that span all D planes (make_plan(full_depth)) the thread
// that stored a pixel's D logits is the same for every plane, so once the tile's last plane is stored it can finish the
// pixel (softmax / soft-argmin / confidence, module.py:1116-1133) without another launch.  NoTail = plain convolution.
struct NoTail {
  static constexpr bool enabled = false;
  __device__ __forceinline__ void operator()(const float*, int, int, int, int) const {}
};

// blocks of B per kd plane: one block = one K=16 MMA step = NPAD x 16 elements in canonical order
// MODE 0: 3x3 stencil per plane (9 taps).  MODE 1: transposed conv k3 s2 p1 op1 as a GEMM over the INPUT grid: 2x2 taps
// per plane at offsets {0,1}^2 (stencil positions (1..2,1..2)), 2 planes, N = 8 output parity classes x COUT.
template <int CIN, int MODE = 0> constexpr int blocks_per_kd() { return MODE == 1 ? 4 * (CIN / 16) : (CIN >= 16 ? 9 * (CIN / 16) : 5); }  // MODE 3 == MODE 0 geometry

// OUT_PLAIN: fp32 [D][H][W] (prob conv).
// HILO: the B image carries every weight twice, as W_hi = round16(W) in columns [0,NPAD) and W_lo = round16(W - W_hi)
// in columns [NPAD, 2*NPAD); the MMA runs with N = 2*NPAD and the epilogue adds the two halves, which restores ~fp32
// weight precision at the cost of a wider N.
template <typename TIn, typename TOut, int CIN, int NPAD, int KD, bool OUT_PLAIN, int MODE = 0, bool HILO = false, typename Tail = NoTail>
__global__ void __launch_bounds__(kThreads, 1)
k_conv_tc(const __grid_constant__ CUtensorMap tmap /*P8 input: {8, Wp, Hp, groups*planes}, box {8, P, R+2, 1}*/,
          const TIn* __restrict__ bimg /*host-arranged B image*/, const float* __restrict__ bias,
          const TOut* __restrict__ res, TOut* __restrict__ out, float* __restrict__ plain_out, const __grid_constant__ Geom g,
          const __grid_constant__ Tail tail) {
  static_assert(!Tail::enabled || OUT_PLAIN, "a per-pixel tail only exists for the single-channel fp32 output");
  constexpr int CG = CIN / 8;
  constexpr int NBLK = blocks_per_kd<CIN, MODE>();
  constexpr int NMMA = HILO ? 2 * NPAD : NPAD;   // instruction N
  static_assert(!(HILO && MODE == 1), "hi/lo weights are not wired for the 3-D transposed-conv epilogue");
  // MODE 3: 2-D "conv3x3 of a nearest-x2 up-sampled map" evaluated on the COARSE grid: 9 taps, N = 4 output parity
  // classes x COUT (the 3x3 fine taps collapse onto 2x2 coarse neighbours; weights pre-summed on the host).
  constexpr int B_BYTES = KD * NBLK * NMMA * 32;
  constexpr int PLANE0 = MODE == 1 ? 1 : 0;
  constexpr bool CLASS_EPI = MODE == 1 || MODE == 3;   // deconv reads input planes d and d+1 (padded indices d+1, d+2)

  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* sB = smem;
  uint8_t* sA = smem + ((B_BYTES + 127) / 128) * 128;
  const uint32_t cg_bytes = (uint32_t)g.slot_pos * 16u;
  const uint32_t slot_bytes = cg_bytes * CG;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sA + (size_t)slot_bytes * g.S);
  uint64_t* full = bars;                 // [S]
  uint64_t* empty = bars + 8;            // [S]
  uint64_t* b_full = bars + 16;

  // N-slicing (blockIdx.y): wide outputs (CIN = 64 layers, whose full B image would not fit shared memory) are split into
  // slices of NPAD columns, each with its own contiguous B image; slice ns produces output columns [ns*NPAD, (ns+1)*NPAD).
  const int ns = blockIdx.y;
  bimg += (size_t)ns * (B_BYTES / sizeof(TIn));
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // provably warp-uniform (uniform datapath)
  const int lane = threadIdx.x & 31;
  int tile = blockIdx.x;
  const int tw = tile % g.tiles_w; tile /= g.tiles_w;
  const int th = tile % g.tiles_h; tile /= g.tiles_h;
  const int td = tile;
  const int w0 = tw * g.TW, h0 = th * g.R, d0 = td * g.DR;
  const int ndo = min(g.DR, g.D - d0);             // output planes of this tile
  const int nin = ndo + KD - 1;                    // input planes to stream

  if (threadIdx.x == 0) {
    for (int s = 0; s < g.S; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4 * kConsumerWG); }
    mbar_init(b_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(b_full, B_BYTES);          // weights do not depend on the previous kernel: fetch them before pdl_wait
    bulk_g2s(sB, bimg, B_BYTES, b_full);
  }
  __syncthreads();
  pdl_wait();   // from here on activations written by the previous kernel are read and our outputs are written
  // trigger the dependents only now: a trigger BEFORE the wait lets the whole chain of later kernels become resident early (each
  // one's prologue would trigger the next), and their idle CTAs then hold the shared memory the running kernel's tiles need
  if (threadIdx.x == 0) pdl_launch_dependents();

  if (warp == kProducerWarp) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      // one tiled TMA per (plane, channel group): box = (R+2) rows x P positions, rows / columns beyond the tensor are
      // zero-filled by the TMA engine, so partial tiles need no special casing
      const uint32_t box_bytes = (uint32_t)g.P * (uint32_t)(g.R + 2) * 16u;
      for (int rp = 0; rp < nin; ++rp) {
        const int slot = rp % g.S;
        if (rp >= g.S) mbar_wait(&empty[slot], ((rp / g.S) - 1) & 1);
        mbar_expect_tx(&full[slot], box_bytes * CG);
        const int pp = d0 + rp + PLANE0;  // padded plane index (pd == 1: plane d-1+kd+1; pd == 0: plane d)
#pragma unroll 1
        for (int cg = 0; cg < CG; ++cg)
          tma_load_4d(sA + (size_t)slot * slot_bytes + (size_t)cg * cg_bytes, &tmap, 0, w0, h0, cg * g.iDp + pp, &full[slot]);
      }
    }
    return;
  }
  // ===================== consumers: MMA + epilogue =====================
  const int wg = warp >> 2, wq = warp & 3;
  const int P = g.P;
  const uint32_t cgb16 = cg_bytes >> 4;
  // A offset / LBO of K=16 step b inside a ring slot, in 16-byte units
  auto aoff = [&](int b) -> uint32_t {
    if constexpr (MODE == 1) {
      const int t = b / (CIN / 16), j = b % (CIN / 16);
      return (uint32_t)(2 * j) * cgb16 + (uint32_t)((1 + t / 2) * P + (1 + t % 2));
    } else if constexpr (CIN >= 16) {
      const int t = b / (CIN / 16), j = b % (CIN / 16);
      return (uint32_t)(2 * j) * cgb16 + (uint32_t)((t / 3) * P + (t % 3));
    } else {
      // taps are paired (0,1)(2,3)(4,5)(6,7)(7*,8): the 5th step re-reads tap 7 against zero weights so that no K slice
      // ever touches shared memory outside the copied tile
      const int t0 = b < 4 ? 2 * b : 7;
      return (uint32_t)((t0 / 3) * P + (t0 % 3));
    }
  };
  auto alo = [&](int b) -> uint32_t {
    if constexpr (MODE == 1 || CIN >= 16) {
      return cgb16;
    } else {
      const int t0 = b < 4 ? 2 * b : 7, t1 = b < 4 ? 2 * b + 1 : 8;
      return (uint32_t)(((t1 / 3) - (t0 / 3)) * P + (t1 % 3) - (t0 % 3));
    }
  };
  const uint32_t sB16 = smem_u32(sB) >> 4, sA16 = smem_u32(sA) >> 4;
  const uint32_t b_lbo16 = (uint32_t)(NMMA * 16 >> 4);
  const int nsub = 2 * g.nch;                      // 64-position sub-chunks per plane
  mbar_wait(b_full, 0);
  int next_wait = 0;
  for (int od = 0; od < ndo; ++od) {
    while (next_wait <= od + KD - 1) {
      mbar_wait(&full[next_wait % g.S], (next_wait / g.S) & 1);
      ++next_wait;
    }
    uint32_t slot16[KD];
#pragma unroll
    for (int kd = 0; kd < KD; ++kd) slot16[kd] = sA16 + (uint32_t)((od + kd) % g.S) * (slot_bytes >> 4);
    const int d = d0 + od;
    for (int sc = wg; sc < nsub; sc += kConsumerWG) {
      float acc[NMMA / 2];
      mma_subchunk<NMMA, TIn, KD, NBLK>(acc, slot16, (uint32_t)sc * 64u, sB16, b_lbo16, aoff, alo);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int l = sc * 64 + wq * 16 + (lane >> 2) + 8 * i;
        const int hh = l / P, ww = l - hh * P;
        const int h = h0 + hh, w = w0 + ww;
        if (!(hh < g.R && ww < g.TW && h < g.H && w < g.W)) continue;
        if constexpr (OUT_PLAIN) {
          if ((lane & 3) == 0) {
            float x = acc[2 * i];
            if constexpr (HILO) x += acc[4 * (NPAD / 8) + 2 * i];
            plain_out[((long long)d * g.H + h) * g.W + w] = x + (bias ? bias[0] : 0.f);
          }
        } else {
#pragma unroll
          for (int j = 0; j < NPAD / 8; ++j) {
            const int n = ns * NPAD + 8 * j + 2 * (lane & 3);
            float x[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              x[e] = acc[4 * j + 2 * i + e];
              if constexpr (HILO) x[e] += acc[4 * (j + NPAD / 8) + 2 * i + e];
            }
            long long pos;
            int co;
            if constexpr (CLASS_EPI) {
              // N = 8 (MODE 1) or 4 (MODE 3) parity classes x COUT: class (pd,ph,pw) of input position (d,h,w) is output (2d+pd, 2h+ph, 2w+pw)
              const int cls = n / g.cout;
              co = n % g.cout;
              const int od2 = MODE == 1 ? 2 * d + (cls >> 2) : d, oh2 = 2 * h + ((cls >> 1) & 1), ow2 = 2 * w + (cls & 1);
              pos = ((((long long)(od2 + g.opd)) * g.oHp + (oh2 + 1)) * g.oWp + (ow2 + 1)) * 8;
            } else {
              co = n;
              if (ns * NPAD + 8 * j >= g.cout) continue;
              pos = ((((long long)(d + g.pd)) * g.Hp + (h + 1)) * g.Wp + (w + 1)) * 8;
            }
            const long long e0 = pos + (co >> 3) * g.out_gs + (co & 7);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              x[e] += bias ? bias[co + e] : 0.f;
              if (g.relu) x[e] = fmaxf(x[e], 0.f);
            }
            if (g.has_res) {
              float r0, r1;
              load2<TOut>(res + pos + (co >> 3) * g.res_gs + (co & 7), r0, r1);
              x[0] += r0; x[1] += r1;
            }
            store2<TOut>(out + e0, x[0], x[1]);
          }
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[od % g.S]);   // oldest input plane of od no longer read by this warp -> producer may refill
  }
  if constexpr (Tail::enabled) {
    // ndo == D (host-checked): this thread wrote all D logits of its pixels itself (program order makes them visible to it)
    if ((lane & 3) == 0) {
      for (int sc = wg; sc < nsub; sc += kConsumerWG)
        for (int i = 0; i < 2; ++i) {
          const int l = sc * 64 + wq * 16 + (lane >> 2) + 8 * i;
          const int hh = l / P, ww = l - hh * P;
          const int h = h0 + hh, w = w0 + ww;
          if (hh < g.R && ww < g.TW && h < g.H && w < g.W) tail(plain_out, h * g.W + w, w, h, g.H * g.W);
        }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
template <int CIN> inline size_t b_image_elems(int npad, int kd) { return (size_t)kd * blocks_per_kd<CIN>() * npad * 16; }

// w: folded fp32 weights [tap][cin][cout] (tap = (kd*3+kh)*3+kw).  Writes the canonical K-major no-swizzle image:
// block(kd,b) = [k half (2)][n/8][n%8][8 k-elements]
// nsplit > 1: the image holds nsplit consecutive slice images, slice s covering output channels [s*npad, (s+1)*npad).
template <typename T, int CIN>
inline void build_b_image(const float* w, int cin, int cout, int npad, int kd_n, std::vector<T>& img, T (*cvt)(float),
                          int nsplit = 1, bool hilo = false, float (*back)(T) = nullptr) {
  constexpr int NBLK = blocks_per_kd<CIN>();
  const int nmma = hilo ? 2 * npad : npad;
  const size_t slice = (size_t)kd_n * NBLK * nmma * 16;
  img.assign(slice * nsplit, cvt(0.f));
  for (int kd = 0; kd < kd_n; ++kd)
    for (int b = 0; b < NBLK; ++b)
      for (int half = 0; half < 2; ++half)
        for (int nn = 0; nn < cout; ++nn)
          for (int e = 0; e < 8; ++e) {
            const int n = nn % npad;
            T* simg = img.data() + slice * (nn / npad);
            int tap9, ci;
            if (CIN >= 16) { tap9 = b / (CIN / 16); ci = (b % (CIN / 16)) * 16 + half * 8 + e; }
            else { tap9 = b < 4 ? 2 * b + half : (half == 0 ? -1 : 8); ci = e; }  // block 4 = (zero, tap 8)
            if (tap9 < 0 || tap9 >= 9 || ci >= cin) continue;
            const int tap = kd * 9 + tap9;
            const float val = w[((size_t)tap * cin + ci) * cout + nn];
            T* blk = simg + ((size_t)(kd * NBLK + b) * 2 + half) * (nmma / 8) * 64;
            const T hi = cvt(val);
            blk[(n / 8) * 64 + (n % 8) * 8 + e] = hi;
            if (hilo) {
              const int n2 = npad + n;
              blk[(n2 / 8) * 64 + (n2 % 8) * 8 + e] = cvt(val - back(hi));
            }
          }
}

// Transposed conv (k3 s2 p1 op1) B image: w is the gather-form folded weight [tap27][cin][cout] (tap index = kernel index
// of the ConvTranspose3d).  Per axis, output parity p and input offset t (0 = same index, 1 = next index) select the
// kernel index: p=0:t=0 -> k=1 ; p=1:t=0 -> k=2, t=1 -> k=0 ; (p=0,t=1) contributes nothing.
template <typename T, int CIN>
inline void build_b_image_deconv(const float* w, int cin, int cout, std::vector<T>& img, T (*cvt)(float), int nsplit = 1) {
  constexpr int NBLK = blocks_per_kd<CIN, 1>();
  const int npad = 8 * cout / nsplit;
  const size_t slice = (size_t)2 * NBLK * npad * 16;
  img.assign(slice * nsplit, cvt(0.f));
  auto kidx = [](int p, int t) { return p == 0 ? (t == 0 ? 1 : -1) : (t == 0 ? 2 : 0); };
  for (int td = 0; td < 2; ++td)
    for (int b = 0; b < NBLK; ++b)
      for (int half = 0; half < 2; ++half)
        for (int cls = 0; cls < 8; ++cls)
          for (int co = 0; co < cout; ++co)
            for (int e = 0; e < 8; ++e) {
              const int t = b / (CIN / 16), j = b % (CIN / 16);
              const int ci = j * 16 + half * 8 + e;
              const int th = t / 2, tw = t % 2;
              const int kd = kidx(cls >> 2, td), kh = kidx((cls >> 1) & 1, th), kw = kidx(cls & 1, tw);
              if (kd < 0 || kh < 0 || kw < 0 || ci >= cin) continue;
              const int nfull = cls * cout + co, n = nfull % npad;
              T* simg = img.data() + slice * (nfull / npad);
              const float val = w[((size_t)((kd * 3 + kh) * 3 + kw) * cin + ci) * cout + co];
              simg[(((size_t)(td * NBLK + b) * 2 + half) * (npad / 8) + n / 8) * 64 + (n % 8) * 8 + e] = cvt(val);
            }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    TDM_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr));
    TDM_CHECK(p != nullptr && qr == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available from the driver");
    fn = (EncodeTiledFn)p;
  }
  return fn;
}

struct Plan {
  Geom g;
  int grid;
  size_t smem;
};

inline Plan make_plan(int cin, int npad, int kd, int D, int H, int W, int pd, int mode = 0, size_t smem_limit = 225 * 1024,
                      bool full_depth = false /* tiles span all D planes (the prob layer's soft-argmin tail needs a pixel's D logits in one CTA) */) {
  Plan p{};
  Geom& g = p.g;
  g.D = D; g.H = H; g.W = W; g.Hp = H + 2; g.Wp = W + 2; g.pd = pd;
  const int cg = cin / 8;
  const int nblk = mode == 1 ? 4 * (cin / 16) : (cin >= 16 ? 9 * (cin / 16) : 5);
  const size_t bbytes = (((size_t)kd * nblk * npad * 32) + 127) / 128 * 128;
  // Search (ring depth, tile width, tile rows, planes per tile) for the cheapest feasible tiling.
  // cost = L2 bytes per useful output position (halo re-reads in h, w and d)
  //        x MMA rows issued per useful position (pad columns, partial last chunk)
  //        x wave quantisation on the 132 SMs of an H100 SXM (one CTA per SM: time ~ ceil(T/132) tile-times for T tiles)
  double best_cost = 1e30;
  int bestR = 0, bestTW = 0, bestS = 0, bestDR = 0;
  const int s_hi = kd == 3 ? 4 : 3, s_lo = kd == 3 ? 3 : 2;   // kd == 2 (deconv): 2 live + 1 prefetch
  for (int S = s_hi; S >= s_lo; --S) {
    for (int tiles_w = 1; tiles_w <= 20; ++tiles_w) {
      const int TW = (W + tiles_w - 1) / tiles_w;
      if (TW + 2 > 256) continue;               // TMA box dims <= 256
      if (tiles_w > 1 && TW < 30) break;
      const int tw_n = (W + TW - 1) / TW;
      const int P = TW + 2;
      for (int R = 1; R <= 32 && R <= H; ++R) {
        const int nch = (R * P + 127) / 128;
        const int slot_pos = (std::max((R + 2) * P, nch * 128 + 2 * P + 2) + 8 + 7) / 8 * 8;
        const size_t smem = bbytes + (size_t)S * cg * slot_pos * 16 + 256;
        if (smem > smem_limit) break;
        const int th_n = (H + R - 1) / R;
        for (int dsplit = 1; dsplit <= (full_depth ? 1 : D); ++dsplit) {
          const int DR = (D + dsplit - 1) / dsplit;
          if (kd >= 2 && DR < 2 && D >= 2) break;
          const int td_n = (D + DR - 1) / DR;
          const double T = (double)tw_n * th_n * td_n;
          const double amp = (double)(R + 2) / R * (double)P / TW * (kd == 3 ? (double)(DR + 2) / DR : (kd == 2 ? (double)(DR + 1) / DR : 1.0));
          // estimated kernel time in clocks: waves x (per-CTA fixed cost + instruction stream), inflated by halo re-reads.
          // The constants are a model (instruction cost growing with N, a fixed per-CTA prologue, fill and drain), not
          // a measurement; they only rank tilings against each other.
          const double clk_mma = mode == 1 ? 35.0 + 0.45 * npad : 45.0 + 0.35 * npad;
          const double tile_clk = 8500.0 + (double)DR * nch * nblk * kd * clk_mma;
          const double cost = std::ceil(T / 132.0) * tile_clk * (1.0 + 0.25 * (amp - 1.0)) * (S == s_hi ? 1.0 : 1.05);
          if (cost < best_cost - 1e-9) { best_cost = cost; bestR = R; bestTW = TW; bestS = S; bestDR = DR; }
          if (T > 4000) break;
        }
      }
    }
    if (bestR > 0 && S == s_hi) break;
  }
  if (bestR == 0 && smem_limit < 225 * 1024) return make_plan(cin, npad, kd, D, H, W, pd, mode, 225 * 1024, full_depth);   // soft limit
  TDM_CHECK(bestR > 0, "conv_tc: no tile fits shared memory");
  g.S = bestS; g.R = bestR; g.TW = bestTW; g.P = bestTW + 2; g.DR = bestDR;
  g.nch = (g.R * g.P + 127) / 128;
  g.slot_pos = (std::max((g.R + 2) * g.P, g.nch * 128 + 2 * g.P + 2) + 8 + 7) / 8 * 8;   // 128-byte aligned TMA destinations
  g.tiles_w = (W + g.TW - 1) / g.TW;
  g.tiles_h = (H + g.R - 1) / g.R;
  g.tiles_d = (D + g.DR - 1) / g.DR;
  p.grid = g.tiles_w * g.tiles_h * g.tiles_d;
  p.smem = bbytes + (size_t)g.S * cg * g.slot_pos * 16 + 256;
  return p;
}

}  // namespace tc
}  // namespace tdm
