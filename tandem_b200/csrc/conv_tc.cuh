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
// Roles (128 * NWG + 32 threads): warpgroups 0 .. NWG-1 consume, warp 4 * NWG produces (one lane issues the TMA copies).
// NWG is 4 (544 threads) where the instantiation fits 96 registers without spills, else 2 (288 threads); see conv_nwg.
// A plane's 64-position sub-chunks are dealt round-robin to the consumer warpgroups; each accumulates its sub-chunk in
// registers (m64nNk16, one instruction per K=16 step), waits for the chain and runs the epilogue (bias / ReLU / skip /
// store) straight from the accumulator fragment, so one warpgroup's drain and epilogue overlap the other warpgroups' MMAs.
//
// This file also holds what the stride-2 (conv_tc_s2.cuh) and input-stationary (conv_tc_is.cuh) kernels share with
// k_conv_tc: the TMA ring and its prologue, the tile decode, the fragment-row -> pixel map, the bias registers, the
// per-pixel tail loop, the wgmma wrappers, the K-step pairing of taps, the B-image index and the tile search.
#pragma once
#include <cuda.h>

#include <climits>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "mvsnet_kernels.cuh"

namespace tdm {
namespace tc {

// A tiling of a D x H x W grid of positions (the output grid; for the transposed / up-2 modes of k_conv_tc the input
// grid) into tiles of R rows x TW columns x DR planes, and the TMA ring that feeds them.
struct Tile {
  int D, H, W;
  int S;                  // ring slots (input planes in flight)
  int R, TW, DR;          // tile: rows, cols, planes
  int P;                  // row pitch of a TMA box in shared memory, TW + halo
  int nch;                // 128-position chunks per plane = ceil(R*P / 128), each two 64-position wgmma sub-chunks
  int slot_pos;           // positions per TMA box destination in a slot: a channel group's plane, or one of its 4 parity
                          // sub-tiles in the stride-2 kernel
  int tiles_w, tiles_h, tiles_d;
};

struct Geom : Tile {
  int Hp, Wp;             // H+2, W+2
  int pd;                 // 1: 3-D conv (KD = 3, halo planes exist), 0: 2-D conv over independent planes (KD = 1)
  long long in_gs, out_gs;   // channel-group strides in elements
  int relu, has_res;         // has_res: MODE 1 adds its skip operand
  int cout;               // real output channels (<= NPAD)
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
// One asm body per N: TY is the PTX type of the 16-bit operands ("f16" / "bf16"), IA / IB / IP the operand numbers of
// the two descriptors and of the accumulate flag.
template <int N, typename T> __device__ __forceinline__ void wgmma(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t acc);
#define TDM_WGMMA_ASM(N, TY, REGS, IA, IB, IP, ...)                                                                       \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #IP ", 0;\n\t"                                                    \
               "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." TY "." TY " {" REGS "}, %" #IA ", %" #IB                 \
               ", p, 1, 1, 0, 0;\n\t}"                                                                                   \
               : __VA_ARGS__                                                                                             \
               : "l"(a), "l"(b), "r"(acc))
#define TDM_WGMMA(N, REGS, IA, IB, IP, ...)                                                                                  \
  template <> __device__ __forceinline__ void wgmma<N, __half>(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t acc) {        \
    TDM_WGMMA_ASM(N, "f16", REGS, IA, IB, IP, __VA_ARGS__);                                                                  \
  }                                                                                                                         \
  template <> __device__ __forceinline__ void wgmma<N, __nv_bfloat16>(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t acc) { \
    TDM_WGMMA_ASM(N, "bf16", REGS, IA, IB, IP, __VA_ARGS__);                                                                 \
  }
TDM_WGMMA(16, "%0,%1,%2,%3,%4,%5,%6,%7", 8, 9, 10,
          "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]))
TDM_WGMMA(32, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15", 16, 17, 18,
          "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]))
TDM_WGMMA(64, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31", 32, 33, 34,
          "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]))
TDM_WGMMA(128, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63", 64, 65, 66,
          "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]))
// N = 24 / 48: the input-stationary kernel's three 8- / 16-column kd blocks (conv_tc_is.cuh)
TDM_WGMMA(24, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11", 12, 13, 14,
          "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]))
TDM_WGMMA(48, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23", 24, 25, 26,
          "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]))
#undef TDM_WGMMA
#undef TDM_WGMMA_ASM
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Orders an accumulator fragment against the asynchronous wgmma that writes it: the compiler may not move a read of d
// above the wait_group that precedes this fence, nor a write below the wgmma issue that follows it.
template <int NR> __device__ __forceinline__ void fence_frag(float (&d)[NR]) {
#pragma unroll
  for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Tiled TMA load of one box of a 4-D tensor map (SASS: UTMALDG); out-of-bounds elements are zero-filled.
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* tmap, int x0, int x1, int x2, int x3, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];" ::"r"(
          smem_u32(dst)),
      "l"(tmap), "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(smem_u32(bar))
      : "memory");
}
// The same for a 5-D tensor map, and its reverse: a whole box shared -> global (SASS: UTMASTG), elements beyond the
// tensor are not written.  Stores are tracked in bulk groups: commit closes one, wait_read(0) returns once every
// committed store has finished reading shared memory, so that its source may be overwritten (or the CTA exit).
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* tmap, int x0, int x1, int x2, int x3, int x4, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];" ::"r"(
          smem_u32(dst)),
      "l"(tmap), "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(x4), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* tmap, const void* src, int x0, int x1, int x2, int x3, int x4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(tmap),
               "r"(smem_u32(src)), "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(x4)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// Makes this thread's generic-proxy writes to shared memory visible to later TMA (async-proxy) reads of it
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Programmatic dependent launch: a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may start
// while its predecessor drains (see Ring::start for what runs before pdl_wait()).
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// Consumer warpgroups (warps 0 .. 4*NWG-1; warp 4*NWG produces) of one instantiation, fixed at build time.  Four keep up
// to four MMA chains in flight per SM, so that one warpgroup's drain and epilogue are covered by three others' MMAs.  At
// 544 threads (17 warps, five of them on one SM sub-partition) ptxas allows 96 registers per thread; two warpgroups (288
// threads, 168 registers) remain only where that cap spills (-Xptxas -v, DESIGN.md section 5): the prob layer's
// soft-argmin tail for more than 32 planes (RegressTail<48 / 64>), and the N = 64 transposed convs (MODE 1: conv11 and
// the conv7 slices).  Those build at 58 registers with four since their skip operand comes through the shared-memory
// output box, but their tile plans, and with them the launch situations the layer tests are built around
// (oracle/mvsnet_layers.py WINDOWS), are those of two warpgroups; the N = 128 one (conv9) runs four.
// mode: k_conv_tc's MODE (0 for the stride-2 and input-stationary kernels); n: instruction N; tail_d: Tail::max_d, 0
// without a tail.  The planners read the same function with their full-depth tile's D for tail_d (D <= 32 exactly when
// the tail's bucket max_d is), so their warpgroup balance matches the kernel they plan for.
__host__ __device__ constexpr int conv_nwg(int mode, int n, int tail_d) { return (mode == 1 && n <= 64) || tail_d > 32 ? 2 : 4; }
// Most 128-position chunks per input plane of a transposed-conv (MODE 1) tile: its consumers keep the output-box offsets
// of their fragment rows in registers, 2 * ceil(2 * kDeconvMaxCh / NWG) of them
constexpr int kDeconvMaxCh = 8;
__host__ __device__ constexpr int conv_threads(int nwg) { return 128 * nwg + 32; }
// Tile-time factor of a plane's 2*nch sub-chunks dealt round-robin to nwg warpgroups: the last round may leave some idle
inline double wg_balance(int nch, int nwg) { return (double)((2 * nch + nwg - 1) / nwg * nwg) / (2 * nch); }

// ---------------------------------------------------------------------------------------------------------------
// K-step pairing of taps, shared by the kernels' A descriptors and the host B images
// ---------------------------------------------------------------------------------------------------------------
// One K=16 MMA step covers two 8-channel K halves.  CIN >= 16: step b reads tap b / (CIN/16) in both halves, channels
// (b % (CIN/16)) * 16 + 8 * half.  CIN == 8: half h of step b reads tap 2b + h, so taps pair as (0,1)(2,3)...; an odd
// last tap is paired with its predecessor, whose half carries zero weights, so that no K slice ever reads shared memory
// outside the copied tile.  ntaps = taps per input plane (9: 3x3 stencil, 4: transposed conv, KS*KS: stride 2).
__host__ __device__ constexpr int ksteps(int cin, int ntaps) { return cin >= 16 ? ntaps * (cin / 16) : (ntaps + 1) / 2; }
__host__ __device__ constexpr int kstep_tap(int cin, int ntaps, int b, int half) {
  return cin >= 16 ? b / (cin / 16) : (2 * b + 1 < ntaps ? 2 * b + half : ntaps - 2 + half);
}
__host__ __device__ constexpr int kstep_ch(int cin, int b, int half) { return cin >= 16 ? (b % (cin / 16)) * 16 + 8 * half : 0; }
// false for the zero-weight half of an odd last pair
__host__ __device__ constexpr bool kstep_live(int cin, int ntaps, int b, int half) { return cin >= 16 || half == 1 || 2 * b + 1 < ntaps; }

// A offset / LBO (16-byte units) of K=16 step b inside a ring slot; off(t) is tap t's position offset, cgb16 the
// distance between two channel groups
template <int CIN, int NTAPS, typename TapOff>
__device__ __forceinline__ uint32_t kstep_aoff(int b, uint32_t cgb16, TapOff off) {
  return (uint32_t)(kstep_ch(CIN, b, 0) / 8) * cgb16 + (uint32_t)off(kstep_tap(CIN, NTAPS, b, 0));
}
template <int CIN, int NTAPS, typename TapOff>
__device__ __forceinline__ uint32_t kstep_alo(int b, uint32_t cgb16, TapOff off) {
  if constexpr (CIN >= 16) return cgb16;
  else return (uint32_t)(off(kstep_tap(CIN, NTAPS, b, 1)) - off(kstep_tap(CIN, NTAPS, b, 0)));
}

// ---------------------------------------------------------------------------------------------------------------
// The TMA ring
// ---------------------------------------------------------------------------------------------------------------
// Shared memory: [B image, 128-byte aligned][S slots of slot_bytes][full[S] at +0, empty[S] at +8, b_full at +16 (8-byte
// barriers, S <= 8; k_conv_tc's MODE 1 adds its output-box barriers at +17 .. +20), 256 bytes][MODE 1: two output
// boxes].  Input plane rp goes to slot rp % S; full[s] counts its TMA bytes, empty[s] the 4 * NWG consumer warps'
// releases of it.
template <int NWG>
struct Ring {
  uint8_t* a;             // slot 0
  uint32_t slot_bytes;
  int S;
  uint64_t* bars;
  int waited;             // consumer: planes 0 .. waited-1 have landed

  // Carves shared memory and runs the prologue: barrier init, then the weight image fetch, then pdl_wait(), then the
  // trigger.  The weights do not depend on the previous kernel, so their copy overlaps its tail; from pdl_wait() on,
  // activations written by the previous kernel are read and outputs are written.  The dependents are triggered only
  // after the wait: a trigger BEFORE it lets the whole chain of later kernels become resident early (each one's
  // prologue would trigger the next), and their idle CTAs then hold the shared memory the running kernel's tiles need.
  __device__ __forceinline__ static Ring start(uint8_t* smem, uint32_t b_bytes, const void* bimg, uint32_t slot_bytes, int S) {
    Ring r{smem + (b_bytes + 127) / 128 * 128, slot_bytes, S, nullptr, 0};
    r.bars = reinterpret_cast<uint64_t*>(r.a + (size_t)slot_bytes * S);
    if (threadIdx.x == 0) {
      for (int s = 0; s < S; ++s) { mbar_init(r.full(s), 1); mbar_init(r.empty(s), 4 * NWG); }
      mbar_init(r.bars + 16, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      mbar_expect_tx(r.bars + 16, b_bytes);
      bulk_g2s(smem, bimg, b_bytes, r.bars + 16);
    }
    __syncthreads();
    pdl_wait();
    if (threadIdx.x == 0) pdl_launch_dependents();
    return r;
  }
  __device__ __forceinline__ uint64_t* full(int s) const { return bars + s; }
  __device__ __forceinline__ uint64_t* empty(int s) const { return bars + 8 + s; }

  // Producer (one lane): input planes 0 .. nin-1, each into its slot once the consumers released the slot's previous
  // plane; boxes(dst, rp, bar) issues plane rp's TMA boxes into dst, tx_bytes in all.
  template <typename Boxes> __device__ __forceinline__ void produce(int nin, uint32_t tx_bytes, Boxes boxes) const {
    for (int rp = 0; rp < nin; ++rp) {
      const int slot = rp % S;
      if (rp >= S) mbar_wait(empty(slot), ((rp / S) - 1) & 1);
      mbar_expect_tx(full(slot), tx_bytes);
      boxes(a + (size_t)slot * slot_bytes, rp, full(slot));
    }
  }

  // Consumers: the weight image, every input plane up to `plane`, the shared address (16-byte units) of a plane's slot,
  // and the release of a plane this warp no longer reads (the producer may refill its slot once all consumer warps released it).
  __device__ __forceinline__ void wait_weights() const { mbar_wait(bars + 16, 0); }
  __device__ __forceinline__ void wait(int plane) {
    for (; waited <= plane; ++waited) mbar_wait(full(waited % S), (waited / S) & 1);
  }
  __device__ __forceinline__ uint32_t slot16(int plane) const { return (smem_u32(a) >> 4) + (uint32_t)(plane % S) * (slot_bytes >> 4); }
  __device__ __forceinline__ void release(int plane) const {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(empty(plane % S));
  }
};

// First output position (w0, h0, d0) and plane count of this CTA's tile
struct TileOrigin { int w0, h0, d0, ndo; };
__device__ __forceinline__ TileOrigin tile_origin(const Tile& t) {
  int tile = blockIdx.x;
  const int tw = tile % t.tiles_w; tile /= t.tiles_w;
  const int th = tile % t.tiles_h; tile /= t.tiles_h;
  return {tw * t.TW, th * t.R, tile * t.DR, min(t.DR, t.D - tile * t.DR)};
}

// Pixel (h, w) of fragment row half i, i.e. of tile position l + 8i, where l = sub-chunk * 64 + (warp % 4) * 16 + lane / 4;
// false for the pad columns and positions beyond the grid
__device__ __forceinline__ bool frag_pixel(const Tile& t, const TileOrigin& o, int l, int i, int& h, int& w) {
  int hh = l / t.P, ww = l - hh * t.P;   // row half 1 is 8 positions on: one division serves both halves
  if (i) {
    ww += 8;
    while (ww >= t.P) { ww -= t.P; ++hh; }
  }
  h = o.h0 + hh; w = o.w0 + ww;
  return hh < t.R && ww < t.TW && h < t.H && w < t.W;
}

// The tile (row, column) of a consumer thread's two fragment row halves, carried across its sub-chunks of a plane.  Sub-chunk
// wg + (k + 1) * NWG lies STEP = 64 * NWG positions after wg + k * NWG, so each half advances by STEP / P rows and STEP % P
// columns with one wrap: the two divisions of frag_pixel happen once per CTA, and no register depends on the chunk count.
// in(i) is frag_pixel's test (pad columns and positions beyond the grid are out).
template <int NWG>
struct FragRows {
  int hh[2], ww[2];
  int dq, dr;             // STEP / P, STEP % P
  int hlim, wlim;         // rows / columns of the tile inside the grid
  __device__ __forceinline__ FragRows(const Tile& t, const TileOrigin& o, int wg, int wq, int lane) {
    constexpr int STEP = 64 * NWG;
    dq = STEP / t.P;
    dr = STEP - dq * t.P;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int l = wg * 64 + wq * 16 + (lane >> 2) + 8 * i;
      hh[i] = l / t.P;
      ww[i] = l - hh[i] * t.P;
    }
    hlim = min(t.R, t.H - o.h0);
    wlim = min(t.TW, t.W - o.w0);
  }
  __device__ __forceinline__ bool in(int i) const { return hh[i] < hlim && ww[i] < wlim; }
  __device__ __forceinline__ void next(int P) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      hh[i] += dq;
      ww[i] += dr;
      if (ww[i] >= P) { ww[i] -= P; ++hh[i]; }
    }
  }
};

// This thread's bias values, loaded once per CTA: bv[j][e] is added to fragment column 8j + 2 * (lane % 4) + e, i.e.
// output column n0 + 8j + 2 * (lane % 4) + e (for CLASS, parity class x cout + channel); zero beyond cout
template <bool CLASS, int NB>
__device__ __forceinline__ void load_bias(float (&bv)[NB][2], const float* bias, int n0, int cout, int lane) {
#pragma unroll
  for (int j = 0; j < NB; ++j) {
    const int n = n0 + 8 * j + 2 * (lane & 3);
    const int co = CLASS ? n % cout : n;
    const bool live = bias && (CLASS || n0 + 8 * j < cout);
#pragma unroll
    for (int e = 0; e < 2; ++e) bv[j][e] = live ? bias[co + e] : 0.f;
  }
}

// Per-pixel tail of the single-channel fp32 (prob) convolution: with tiles that span all D planes the thread that stored a
// pixel's D logits is the same for every plane, so once the tile's last plane is stored it can finish the pixel
// (softmax / soft-argmin / confidence, module.py:1116-1133) without another launch.  NoTail = plain convolution.
struct NoTail {
  static constexpr bool enabled = false;
  static constexpr int max_d = 0;
  __device__ __forceinline__ void operator()(const float*, int, int, int, int) const {}
};
// Runs the tail over this thread's pixels once the tile is stored.  ndo == D (host-checked): the thread wrote all D
// logits of its pixels itself (program order makes them visible to it).
template <int NWG, typename Tail>
__device__ __forceinline__ void run_tail(const Tail& tail, float* plain_out, const Tile& t, const TileOrigin& o, int wg, int wq, int lane) {
  if ((lane & 3) == 0) {
    for (int sc = wg; sc < 2 * t.nch; sc += NWG)
      for (int i = 0; i < 2; ++i) {
        // each row half decoded on its own: carried over from half 0, its pixel would stay live across the tail call, and
        // RegressTail<64> already sits at the register cap
        int h, w;
        if (frag_pixel(t, o, sc * 64 + wq * 16 + (lane >> 2) + 8 * i, 0, h, w)) tail(plain_out, h * t.W + w, w, h, t.H * t.W);
      }
  }
}

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

// Two consecutive channels of an 8-channel group: one 4-byte store / load (the load is split into its issue, a plain
// 4-byte __ldg, and unpack2, so that it can be issued early).
template <typename T> __device__ __forceinline__ uint32_t pack2(float x0, float x1) {
  T v[2] = {from_f<T>(x0), from_f<T>(x1)};
  return *reinterpret_cast<const uint32_t*>(v);
}
template <typename T> __device__ __forceinline__ void store2(T* p, float x0, float x1) {
  *reinterpret_cast<uint32_t*>(p) = pack2<T>(x0, x1);
}
template <typename T> __device__ __forceinline__ void unpack2(uint32_t u, float& x0, float& x1) {
  const T* v = reinterpret_cast<const T*>(&u);
  x0 = to_f<T>(v[0]); x1 = to_f<T>(v[1]);
}

// Tap t of the 3x3 stencil (MODE 0 / 3): position offset inside a ring slot of pitch P
__device__ __forceinline__ int stencil_off(int t, int P) { return (t / 3) * P + (t % 3); }

// OUT_PLAIN: fp32 [D][H][W] (prob conv).
// HILO: the B image carries every weight twice, as W_hi = round16(W) in columns [0,NPAD) and W_lo = round16(W - W_hi)
// in columns [NPAD, 2*NPAD); the MMA runs with N = 2*NPAD and the epilogue adds the two halves, which restores ~fp32
// weight precision at the cost of a wider N.
// MODE 0: 3x3 stencil per plane (9 taps).  MODE 1: transposed conv k3 s2 p1 op1 as a GEMM over the INPUT grid: 2x2 taps
// per plane at offsets {0,1}^2 (stencil positions (1..2,1..2)), 2 planes, N = 8 output parity classes x COUT.
// MODE 3: the fused FPN tail, out = conv3x3(up2(x)) + conv3x3(y) for a map x on the COARSE grid and y on the fine one,
// evaluated on the coarse grid: 9 coarse taps, N = 4 output parity classes x COUT.  Fine tap k of output parity p reads
// fine offset p + k - 1 = 2 * delta + q, i.e. coarse offset delta in {-1, 0, 1} and sub-position q in {0, 1}.  Channel
// groups 0 .. 3 of a ring slot are x (tmap); groups 4 .. 7 are the four parity sub-tiles (qh, qw) of y's 8 channels
// (tmap_res, every second fine row and column), so y's term is a 3x3 coarse-grid conv over 32 space-to-depth channels
// like x's (weights pre-summed and placed per class, coarse tap and sub-position on the host).
// NWG: consumer warpgroups, conv_nwg(MODE, instruction N, Tail::max_d).
template <typename TIn, typename TOut, int CIN, int NPAD, int KD, bool OUT_PLAIN, int MODE, bool HILO, typename Tail, int NWG>
__global__ void __launch_bounds__(conv_threads(NWG), 1)
k_conv_tc(const __grid_constant__ CUtensorMap tmap /*P8 input: {8, Wp, Hp, groups*planes}, box {8, P, R+2, 1}*/,
          const __grid_constant__ CUtensorMap tmap_res /*MODE 1: skip operand, see OutBox; MODE 3: the fine input,
                                                          box {8, 2P, 2(R+2), 1} with element strides 2 in W and H*/,
          const __grid_constant__ CUtensorMap tmap_out /*MODE 1: output*/,
          const TIn* __restrict__ bimg /*host-arranged B image*/, const float* __restrict__ bias,
          TOut* __restrict__ out, float* __restrict__ plain_out, const __grid_constant__ Geom g, const __grid_constant__ Tail tail) {
  static_assert(!Tail::enabled || OUT_PLAIN, "a per-pixel tail only exists for the single-channel fp32 output");
  static_assert(MODE != 3 || (CIN == 64 && KD == 1), "MODE 3 streams 4 coarse and 4 fine sub-tile channel groups");
  constexpr int CG = CIN / 8;
  constexpr int CG_TMAP = MODE == 3 ? 4 : CG;     // channel groups from tmap; MODE 3 loads the rest from tmap_res
  constexpr int NTAPS = MODE == 1 ? 4 : 9;
  constexpr int NBLK = ksteps(CIN, NTAPS);
  constexpr int NMMA = HILO ? 2 * NPAD : NPAD;   // instruction N
  static_assert(!(HILO && MODE == 1), "hi/lo weights are not wired for the 3-D transposed-conv epilogue");
  constexpr int B_BYTES = KD * NBLK * NMMA * 32;
  constexpr int PLANE0 = MODE == 1 ? 1 : 0;
  constexpr bool CLASS_EPI = MODE == 1 || MODE == 3;   // deconv reads input planes d and d+1 (padded indices d+1, d+2)

  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t cg_bytes = (uint32_t)g.slot_pos * 16u;
  // N-slicing (blockIdx.y): wide outputs (CIN = 64 layers, whose full B image would not fit shared memory) are split into
  // slices of NPAD columns, each with its own contiguous B image; slice ns produces output columns [ns*NPAD, (ns+1)*NPAD).
  const int ns = blockIdx.y;
  Ring<NWG> ring = Ring<NWG>::start(smem, B_BYTES, bimg + (size_t)ns * (B_BYTES / sizeof(TIn)), cg_bytes * CG, g.S);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // provably warp-uniform (uniform datapath)
  const int lane = threadIdx.x & 31;
  const TileOrigin o = tile_origin(g);
  const int nin = o.ndo + KD - 1;                  // input planes to stream

  // MODE 1 output boxes: input plane d of the tile yields output planes 2d, 2d + 1, rows 2h0 .. 2h0 + 2R - 1 and columns
  // 2w0 .. 2w0 + 2TW - 1.  Its box holds them for the OBG output channel groups of this N slice, in P8 order
  // [group][2][2R][2TW][8]; the skip operand comes in by TMA into the box, the consumers turn it into the output in
  // place, and the producer stores the box by TMA.  Two boxes alternate, so that plane od + 1 never waits for od's store.
  constexpr int OBG = MODE == 1 ? NPAD / 64 : 1;
  const uint32_t obox_bytes = MODE == 1 ? 128u * (uint32_t)(g.R * g.TW * OBG) : 0u;
  uint8_t* const obox0 = reinterpret_cast<uint8_t*>(ring.bars) + 256;
  uint64_t* const obox_full = ring.bars + 17;     // [2] skip operand landed (or the box is free, without one)
  uint64_t* const obox_filled = ring.bars + 19;   // [2] the 4 * NWG consumer warps wrote their outputs
  if constexpr (MODE == 1) {
    if (threadIdx.x == 0) {
      for (int b = 0; b < 2; ++b) { mbar_init(obox_full + b, 1); mbar_init(obox_filled + b, 4 * NWG); }
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
  }

  if (warp == 4 * NWG) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      // one tiled TMA per (plane, channel group): box = (R+2) rows x P positions, rows / columns beyond the tensor are
      // zero-filled by the TMA engine, so partial tiles need no special casing
      const uint32_t box_bytes = (uint32_t)g.P * (uint32_t)(g.R + 2) * 16u;
      auto boxes = [&](uint8_t* dst, int rp, uint64_t* bar) {
        const int pp = o.d0 + rp + PLANE0;  // padded plane index (pd == 1: plane d-1+kd+1; pd == 0: plane d)
#pragma unroll 1
        for (int cg = 0; cg < CG_TMAP; ++cg) tma_load_4d(dst + (size_t)cg * cg_bytes, &tmap, 0, o.w0, o.h0, cg * g.iDp + pp, bar);
        if constexpr (MODE == 3) {
          // box position (i, j) is coarse (h0 - 1 + i, w0 - 1 + j), like the coarse boxes; in sub-tile (qh, qw) it holds
          // fine (2 (h0 - 1 + i) + qh, 2 (w0 - 1 + j) + qw), padded coordinates from (2 h0 - 1 + qh, 2 w0 - 1 + qw)
#pragma unroll 1
          for (int q = 0; q < 4; ++q)
            tma_load_4d(dst + (size_t)(CG_TMAP + q) * cg_bytes, &tmap_res, 0, 2 * o.w0 - 1 + (q & 1), 2 * o.h0 - 1 + (q >> 1), pp, bar);
        }
      };
      if constexpr (MODE == 1) {
        // input planes, skip boxes and output stores interleaved: plane od's consumers need input planes od, od + 1 and
        // box od % 2; the box of od + 2 is refilled once od's store has read it.  Skip and output tensor maps cover
        // the interior of the P8 tensors: rows / columns beyond the grid read as zero and are never written.
        const int og = OBG == 1 ? ns : 0;   // first output channel group of this slice
        auto fill = [&](int od) {
          uint64_t* bar = obox_full + (od & 1);
          if (g.has_res) {
            mbar_expect_tx(bar, obox_bytes);
            tma_load_5d(obox0 + (size_t)(od & 1) * obox_bytes, &tmap_res, 0, 2 * o.w0, 2 * o.h0, 2 * (o.d0 + od), og, bar);
          } else {
            mbar_arrive(bar);
          }
        };
        int rp = 0;
        auto feed = [&](int upto) {
          for (; rp < upto && rp < nin; ++rp) {
            const int slot = rp % g.S;
            if (rp >= g.S) mbar_wait(ring.empty(slot), ((rp / g.S) - 1) & 1);
            mbar_expect_tx(ring.full(slot), box_bytes * CG);
            boxes(ring.a + (size_t)slot * ring.slot_bytes, rp, ring.full(slot));
          }
        };
        feed(g.S);
        fill(0);
        if (o.ndo > 1) fill(1);
        for (int od = 0; od < o.ndo; ++od) {
          mbar_wait(obox_filled + (od & 1), (od >> 1) & 1);
          tma_store_5d(&tmap_out, obox0 + (size_t)(od & 1) * obox_bytes, 0, 2 * o.w0, 2 * o.h0, 2 * (o.d0 + od), og);
          bulk_commit();
          feed(od + 1 + g.S);   // the consumers released plane od before they signalled its box
          if (od + 2 < o.ndo) {
            bulk_wait_read0();
            fill(od + 2);
          }
        }
        bulk_wait_read0();
      } else {
        ring.produce(nin, box_bytes * CG, boxes);
      }
    }
    return;
  }
  // ===================== consumers: MMA + epilogue =====================
  const int wg = warp >> 2, wq = warp & 3;
  const int P = g.P;
  const uint32_t cgb16 = cg_bytes >> 4;
  auto tap_off = [&](int t) -> int {
    if constexpr (MODE == 1) return (1 + t / 2) * P + (1 + t % 2);
    else return stencil_off(t, P);
  };
  auto aoff = [&](int b) -> uint32_t { return kstep_aoff<CIN, NTAPS>(b, cgb16, tap_off); };
  auto alo = [&](int b) -> uint32_t { return kstep_alo<CIN, NTAPS>(b, cgb16, tap_off); };
  const uint32_t sB16 = smem_u32(smem) >> 4;
  const uint32_t b_lbo16 = (uint32_t)(NMMA * 16 >> 4);
  const int nsub = 2 * g.nch;                      // 64-position sub-chunks per plane
  ring.wait_weights();
  // 16-bit outputs of MODE 0 / 3: fragment row half i of a sub-chunk stores at element fr.hh[i] * orow + fr.ww[i] * OCOL
  // of its plane's base pointer (ob below), i.e. at P8 position (h + 1, w + 1) of pixel (h, w) in MODE 0, and at output
  // (2h + 1, 2w + 1), class (0, 0), in MODE 3.  MODE 3's N = 4 parity classes x 8 channels (cout = 8, nsplit = 1: the host
  // checks both) make column block j class (ph, pw) = (j >> 1, j & 1), channels 2 * (lane % 4) + e, of output
  // (d, 2h + ph, 2w + pw).
  static_assert(MODE != 3 || NPAD == 32, "MODE 3 writes 4 parity classes of 8 channels");
  constexpr int OCOL = MODE == 3 ? 16 : 8;
  const int orow = MODE == 3 ? 16 * g.oWp : 8 * g.Wp;
  const FragRows<NWG> fr0(g, o, wg, wq, lane);
  // bias in registers, except for N = 128, whose 32 more registers would spill: it loads them in the epilogue.  MODE 1
  // slice ns holds output channels ns * CPS .. + CPS - 1 of all 8 classes (build_b_image_deconv): column n is class
  // n / CPS, channel ns * CPS + n % CPS.
  constexpr bool BIAS_REG = NPAD <= 64;
  constexpr int CPS = NPAD / 8;
  const float* const bias_s = MODE == 1 && bias ? bias + ns * CPS : bias;
  float bv[OUT_PLAIN || !BIAS_REG ? 1 : NPAD / 8][2];
  if constexpr (OUT_PLAIN) bv[0][0] = bias ? bias[0] : 0.f;
  else if constexpr (BIAS_REG && MODE == 1) load_bias<true>(bv, bias_s, 0, CPS, lane);
  else if constexpr (BIAS_REG) load_bias<CLASS_EPI>(bv, bias, ns * NPAD, g.cout, lane);
  // PAIR_EPI (MODE 3) moves whole 32-byte sectors.  Classes pw = 0 and pw = 1 of one (ph, output channel group) are
  // column blocks 2k and 2k + 1 (cout = 8; the host checks it), and their output pixels 2w and 2w + 1 are adjacent: 32
  // bytes per input position.  Lanes q and q ^ 1 of a fragment row swap one packed word, so that lane q writes 8
  // contiguous bytes, channels 4 * (q >> 1) .. +3 of class pw = q & 1.  A warp access then covers its 8 positions'
  // 32-byte runs in full, where two 4-byte accesses per lane filled half of each sector apiece.
  constexpr bool PAIR_EPI = MODE == 3;
  const int pq = lane & 1;
  // MODE 1: box element offset of this lane's channels 2q, 2q + 1 of class 0 for fragment row half i of this
  // warpgroup's k-th sub-chunk (sub-chunk wg + k * NWG), -1 for pad columns and rows beyond the tile; decoded once per
  // CTA.  Class (pd, ph, pw) and channel group c of the slice add c * 2 * PD_STR + pd * PD_STR + ph * PH_STR + pw * 8.
  constexpr int MAXSC = MODE == 1 ? (2 * kDeconvMaxCh + NWG - 1) / NWG : 1;
  int boff[MAXSC][2];
  const int PH_STR = 16 * g.TW, PD_STR = 32 * g.R * g.TW;
  if constexpr (MODE == 1) {
#pragma unroll
    for (int k = 0; k < MAXSC; ++k)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int l = (wg + k * NWG) * 64 + wq * 16 + (lane >> 2) + 8 * i;
        const int hh = l / P, ww = l - hh * P;
        boff[k][i] = hh < g.R && ww < g.TW ? (4 * hh * g.TW + 2 * ww) * 8 + 2 * (lane & 3) : -1;
      }
  }
  for (int od = 0; od < o.ndo; ++od) {
    ring.wait(od + KD - 1);
    uint32_t slot16[KD];
#pragma unroll
    for (int kd = 0; kd < KD; ++kd) slot16[kd] = ring.slot16(od + kd);
    const int d = o.d0 + od;
    TOut* const box = reinterpret_cast<TOut*>(obox0 + (size_t)(od & 1) * obox_bytes);
    if constexpr (MODE == 1) mbar_wait(obox_full + (od & 1), (od >> 1) & 1);
    // this lane's first element of tile position (0, 0) in output plane d (MODE 0: + column block 0 of the N slice)
    TOut* ob = nullptr;
    if constexpr (MODE == 3)
      ob = out + (((long long)(d + g.opd) * g.oHp + 2 * o.h0 + 1) * g.oWp + 2 * o.w0 + 1) * 8 + 8 * pq + 4 * ((lane & 3) >> 1);
    else if constexpr (MODE == 0 && !OUT_PLAIN)
      ob = out + (((long long)(d + g.pd) * g.Hp + o.h0 + 1) * g.Wp + o.w0 + 1) * 8 + (ns * NPAD / 8) * g.out_gs + 2 * (lane & 3);
    FragRows<NWG> fr = fr0;
#pragma unroll 1
    for (int k = 0; wg + k * NWG < nsub; ++k) {
      const int sc = wg + k * NWG;
      float acc[NMMA / 2];
      mma_subchunk<NMMA, TIn, KD, NBLK>(acc, slot16, (uint32_t)sc * 64u, sB16, b_lbo16, aoff, alo);
      if constexpr (MODE == 1) {
        // acc + bias -> ReLU -> + skip -> one rounding, in place in the box
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          int bo = boff[0][i];
#pragma unroll
          for (int kk = 1; kk < MAXSC; ++kk)
            if (k == kk) bo = boff[kk][i];
          if (bo < 0) continue;
#pragma unroll
          for (int j = 0; j < NPAD / 8; ++j) {
            const int cls = j / OBG, c = j % OBG;
            uint32_t* const p = reinterpret_cast<uint32_t*>(box + bo + (2 * c + (cls >> 2)) * PD_STR + ((cls >> 1) & 1) * PH_STR + (cls & 1) * 8);
            float x[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              x[e] = acc[4 * j + 2 * i + e];
              if constexpr (BIAS_REG) x[e] += bv[j][e];
              else x[e] += bias_s ? __ldg(bias_s + (8 * j + 2 * (lane & 3)) % CPS + e) : 0.f;
              if (g.relu) x[e] = fmaxf(x[e], 0.f);
            }
            if (g.has_res) {
              float r0, r1;
              unpack2<TOut>(*p, r0, r1);
              x[0] += r0; x[1] += r1;
            }
            *p = pack2<TOut>(x[0], x[1]);
          }
        }
        continue;
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        if constexpr (OUT_PLAIN) {
          int h, w;
          if (!frag_pixel(g, o, sc * 64 + wq * 16 + (lane >> 2), i, h, w) || (lane & 3) != 0) continue;
          float x = acc[2 * i];
          if constexpr (HILO) x += acc[4 * (NPAD / 8) + 2 * i];
          plain_out[((long long)d * g.H + h) * g.W + w] = x + bv[0][0];
          continue;
        }
        const bool in = fr.in(i);
        if (!in && !PAIR_EPI) continue;   // PAIR_EPI: every lane takes part in the word exchange
        TOut* const op = ob + (fr.hh[i] * orow + fr.ww[i] * OCOL);
        if constexpr (PAIR_EPI) {
#pragma unroll
          for (int k2 = 0; k2 < NPAD / 16; ++k2) {
            uint32_t v[2];
#pragma unroll
            for (int p = 0; p < 2; ++p) {
              const int j = 2 * k2 + p;
              float x[2];
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                x[e] = acc[4 * j + 2 * i + e];
                if constexpr (HILO) x[e] += acc[4 * (j + NPAD / 8) + 2 * i + e];
                x[e] += bv[j][e];
                if (g.relu) x[e] = fmaxf(x[e], 0.f);
              }
              v[p] = pack2<TOut>(x[0], x[1]);
            }
            const uint32_t own = pq ? v[1] : v[0], other = __shfl_xor_sync(0xffffffffu, pq ? v[0] : v[1], 1);
            if (in) *reinterpret_cast<uint2*>(op + k2 * 8 * g.oWp) = pq ? make_uint2(other, own) : make_uint2(own, other);
          }
        } else {
#pragma unroll
          for (int j = 0; j < NPAD / 8; ++j) {
            if (ns * NPAD + 8 * j >= g.cout) continue;
            float x[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              x[e] = acc[4 * j + 2 * i + e];
              if constexpr (HILO) x[e] += acc[4 * (j + NPAD / 8) + 2 * i + e];
            }
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              if constexpr (BIAS_REG) x[e] += bv[j][e];
              else x[e] += bias ? bias[ns * NPAD + 8 * j + 2 * (lane & 3) + e] : 0.f;
              if (g.relu) x[e] = fmaxf(x[e], 0.f);
            }
            store2<TOut>(op + j * g.out_gs, x[0], x[1]);
          }
        }
      }
      fr.next(P);
    }
    if constexpr (MODE == 1) {
      // this warp's outputs of plane od are in the box: hand it to the producer's TMA store
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(obox_filled + (od & 1));
    }
    ring.release(od);   // oldest input plane of od
  }
  if constexpr (Tail::enabled) run_tail<NWG>(tail, plain_out, g, o, wg, wq, lane);
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
// Canonical K-major no-swizzle index of B element (K half, column n, k element e) of K=16 block blk, in an image of
// ncols columns: block = [k half (2)][n/8][n%8][8 k-elements]
inline size_t b_index(int blk, int half, int n, int e, int ncols) {
  return (((size_t)blk * 2 + half) * (ncols / 8) + n / 8) * 64 + (n % 8) * 8 + e;
}

// w: folded fp32 weights [tap][cin][cout] (tap = (kd*3+kh)*3+kw).  Writes the canonical K-major no-swizzle image.
// nsplit > 1: the image holds nsplit consecutive slice images, slice s covering output channels [s*npad, (s+1)*npad).
template <typename T>
inline void build_b_image(const float* w, int cin, int cout, int npad, int kd_n, std::vector<T>& img, T (*cvt)(float),
                          int nsplit = 1, bool hilo = false, float (*back)(T) = nullptr) {
  const int nblk = ksteps(cin, 9);
  const int nmma = hilo ? 2 * npad : npad;
  const size_t slice = (size_t)kd_n * nblk * nmma * 16;
  img.assign(slice * nsplit, cvt(0.f));
  for (int kd = 0; kd < kd_n; ++kd)
    for (int b = 0; b < nblk; ++b)
      for (int half = 0; half < 2; ++half)
        for (int nn = 0; nn < cout; ++nn)
          for (int e = 0; e < 8; ++e) {
            const int n = nn % npad;
            T* simg = img.data() + slice * (nn / npad);
            const int tap9 = kstep_tap(cin, 9, b, half), ci = kstep_ch(cin, b, half) + e;
            if (!kstep_live(cin, 9, b, half) || ci >= cin) continue;
            const float val = w[((size_t)(kd * 9 + tap9) * cin + ci) * cout + nn];
            const T hi = cvt(val);
            simg[b_index(kd * nblk + b, half, n, e, nmma)] = hi;
            if (hilo) simg[b_index(kd * nblk + b, half, npad + n, e, nmma)] = cvt(val - back(hi));
          }
}

// Transposed conv (k3 s2 p1 op1) B image: w is the gather-form folded weight [tap27][cin][cout] (tap index = kernel index
// of the ConvTranspose3d).  Per axis, output parity p and input offset t (0 = same index, 1 = next index) select the
// kernel index: p=0:t=0 -> k=1 ; p=1:t=0 -> k=2, t=1 -> k=0 ; (p=0,t=1) contributes nothing.
// nsplit > 1: slice s holds output channels s * cout / nsplit .. + cout / nsplit - 1 of all 8 classes, column
// cls * cout / nsplit + channel % (cout / nsplit), so that each slice writes whole output channel groups.
template <typename T>
inline void build_b_image_deconv(const float* w, int cin, int cout, std::vector<T>& img, T (*cvt)(float), int nsplit = 1) {
  const int nblk = ksteps(cin, 4);
  const int npad = 8 * cout / nsplit;
  const size_t slice = (size_t)2 * nblk * npad * 16;
  img.assign(slice * nsplit, cvt(0.f));
  auto kidx = [](int p, int t) { return p == 0 ? (t == 0 ? 1 : -1) : (t == 0 ? 2 : 0); };
  for (int td = 0; td < 2; ++td)
    for (int b = 0; b < nblk; ++b)
      for (int half = 0; half < 2; ++half)
        for (int cls = 0; cls < 8; ++cls)
          for (int co = 0; co < cout; ++co)
            for (int e = 0; e < 8; ++e) {
              const int t = kstep_tap(cin, 4, b, half), ci = kstep_ch(cin, b, half) + e;
              const int th = t / 2, tw = t % 2;
              const int kd = kidx(cls >> 2, td), kh = kidx((cls >> 1) & 1, th), kw = kidx(cls & 1, tw);
              if (kd < 0 || kh < 0 || kw < 0 || ci >= cin) continue;
              const int cps = cout / nsplit, n = cls * cps + co % cps;   // slice co / cps: channels co / cps * cps .. + cps - 1
              T* simg = img.data() + slice * (co / cps);
              const float val = w[((size_t)((kd * 3 + kh) * 3 + kw) * cin + ci) * cout + co];
              simg[b_index(td * nblk + b, half, n, e, npad)] = cvt(val);
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

// Positions a TMA box of R + halo rows of pitch P occupies in a ring slot: the box itself, and at least as far as the
// A reads of the last 128-position chunk reach (its taps start up to halo * (P + 1) positions on), plus 8, rounded up
// to 8 (128-byte aligned TMA destinations).
inline int box_positions(int R, int P, int halo) {
  const int nch = (R * P + 127) / 128;
  return (std::max((R + halo) * P, nch * 128 + halo * (P + 1)) + 8 + 7) / 8 * 8;
}

// What the tile search of one kernel depends on, apart from its halo amplification and clocks per tile
struct TileLimits {
  int s_hi, s_lo;         // ring depth range; the deepest that fits is preferred
  int halo;               // a tile reads R + halo rows of P = TW + halo positions per input plane
  int boxes;              // TMA boxes per channel group and plane
  int p_max;              // TMA box limit on P
  int tw_min;             // narrowest tile width when W is split
  int nch_max;            // most 128-position chunks per plane
  int dr_min;             // fewest planes per tile (when D >= 2)
  bool full_depth;        // tiles span all D planes (the prob layer's soft-argmin tail needs a pixel's D logits in one CTA)
  int out_box = 0;        // shared-memory bytes of output boxes per tile position (R x TW), 0 without them.  They count
                          // against the 225 KB an SM offers, not against a lower budget (see plan_tiles)
  int tw_max = INT_MAX;   // widest tile
  int whole_rounds = 0;   // > 0: a plane of more than one chunk deals its 2 * nch sub-chunks in whole rounds of this many
                          // warpgroups (no warpgroup idles through the last round)
};

struct Plan {
  Geom g;
  int grid;
  size_t smem;
  int nwg;                // consumer warpgroups the tiling was balanced for (conv_nwg); the launch checks its kernel's NWG
};

// Searches (ring depth, tile width, tile rows, planes per tile) for the cheapest tiling whose B image (b_bytes), ring
// slots and barriers fit smem_limit.
// cost = L2 bytes per useful output position (halo re-reads in h, w and d: amp(R, TW, P, DR))
//        x MMA rows issued per useful position (pad columns, partial last chunk)
//        x wave quantisation on the 132 SMs of an H100 SXM (one CTA per SM: time ~ ceil(T/132) tile-times for T tiles)
// tile_clk(DR, nch) is the estimated time of one tile in clocks: a per-CTA fixed cost + the instruction stream.  Its
// constants are a model (instruction cost growing with N, a fixed per-CTA prologue, fill and drain), not a measurement;
// they only rank tilings against each other; callers scale it by wg_balance for the kernel's consumer warpgroups.  A limit
// below 225 KB is soft: if nothing fits it, 225 KB is searched.  It bounds the B image and the ring; output boxes
// (TileLimits::out_box) count against the 225 KB only.
template <typename Amp, typename Clk>
inline Tile plan_tiles(int D, int H, int W, int cg, size_t b_bytes, size_t smem_limit, const TileLimits& lim, Amp amp, Clk tile_clk,
                       size_t& smem_out) {
  auto box_bytes = [&](int R, int P) { return (size_t)lim.out_box * R * (P - lim.halo); };
  auto smem_of = [&](int S, int R, int P) {
    return b_bytes + (size_t)S * cg * lim.boxes * box_positions(R, P, lim.halo) * 16 + 256 + box_bytes(R, P);
  };
  double best_cost = 1e30;
  int bestR = 0, bestTW = 0, bestS = 0, bestDR = 0;
  for (int S = lim.s_hi; S >= lim.s_lo; --S) {
    for (int tiles_w = 1; tiles_w <= 20; ++tiles_w) {
      const int TW = (W + tiles_w - 1) / tiles_w;
      if (TW + lim.halo > lim.p_max || TW > lim.tw_max) continue;
      if (tiles_w > 1 && TW < lim.tw_min) break;
      const int tw_n = (W + TW - 1) / TW;
      const int P = TW + lim.halo;
      for (int R = 1; R <= 32 && R <= H; ++R) {
        const int nch = (R * P + 127) / 128;
        if (nch > lim.nch_max) break;
        if (smem_of(S, R, P) - box_bytes(R, P) > smem_limit || smem_of(S, R, P) > 225 * 1024) break;
        if (lim.whole_rounds && nch > 1 && (2 * nch) % lim.whole_rounds) continue;
        const int th_n = (H + R - 1) / R;
        for (int dsplit = 1; dsplit <= (lim.full_depth ? 1 : D); ++dsplit) {
          const int DR = (D + dsplit - 1) / dsplit;
          if (DR < lim.dr_min && D >= 2) break;
          const int td_n = (D + DR - 1) / DR;
          const double T = (double)tw_n * th_n * td_n;
          const double cost = std::ceil(T / 132.0) * tile_clk(DR, nch) * (1.0 + 0.25 * (amp(R, TW, P, DR) - 1.0)) * (S == lim.s_hi ? 1.0 : 1.05);
          if (cost < best_cost - 1e-9) { best_cost = cost; bestR = R; bestTW = TW; bestS = S; bestDR = DR; }
          if (T > 4000) break;
        }
      }
    }
    if (bestR > 0 && S == lim.s_hi) break;
  }
  if (bestR == 0 && smem_limit < 225 * 1024) return plan_tiles(D, H, W, cg, b_bytes, 225 * 1024, lim, amp, tile_clk, smem_out);
  TDM_CHECK(bestR > 0, "conv_tc: no tile fits shared memory");
  Tile t{};
  t.D = D; t.H = H; t.W = W;
  t.S = bestS; t.R = bestR; t.TW = bestTW; t.P = bestTW + lim.halo; t.DR = bestDR;
  t.nch = (t.R * t.P + 127) / 128;
  t.slot_pos = box_positions(t.R, t.P, lim.halo);
  t.tiles_w = (W + t.TW - 1) / t.TW;
  t.tiles_h = (H + t.R - 1) / t.R;
  t.tiles_d = (D + t.DR - 1) / t.DR;
  smem_out = smem_of(t.S, t.R, t.P);
  return t;
}

inline size_t b_image_bytes(int kd, int nblk, int ncols) { return (((size_t)kd * nblk * ncols * 32) + 127) / 128 * 128; }

inline Plan make_plan(int cin, int npad, int kd, int D, int H, int W, int pd, int mode = 0, size_t smem_limit = 225 * 1024,
                      bool full_depth = false /* tiles span all D planes (the prob layer's soft-argmin tail) */) {
  Plan p{};
  const int nblk = ksteps(cin, mode == 1 ? 4 : 9);
  const int s_hi = kd == 3 ? 4 : 3, s_lo = kd == 3 ? 3 : 2;   // kd == 2 (deconv): 2 live + 1 prefetch
  TileLimits lim{s_hi, s_lo, 2, 1, 256, 30, INT_MAX, kd >= 2 ? 2 : 1, full_depth};
  if (mode == 1) {
    // two output boxes of npad / 64 channel groups, 8 output positions of 16 bytes per input position; a box spans 2 TW
    // columns (TMA box dimensions <= 256)
    lim.out_box = 2 * (npad / 64) * 128;
    lim.tw_max = 128;
    lim.nch_max = kDeconvMaxCh;
    // with four warpgroups an odd chunk count leaves two of them idle for one chain per plane, and the plane's box store
    // waits for the slowest warpgroup: tiles of 1 or an even number of chunks only
    lim.whole_rounds = conv_nwg(1, npad, 0);
  }
  // the fused FPN tail (MODE 3, CIN 64) also loads the fine input's parity sub-tiles: boxes of 2P columns (TMA box
  // dimensions <= 256)
  if (mode == 3 && cin == 64) lim.p_max = 128;
  auto amp = [&](int R, int TW, int P, int DR) {
    return (double)(R + 2) / R * (double)P / TW * (kd == 3 ? (double)(DR + 2) / DR : (kd == 2 ? (double)(DR + 1) / DR : 1.0));
  };
  const int nwg = conv_nwg(mode, npad, full_depth ? D : 0);
  auto tile_clk = [&](int DR, int nch) {
    const double clk_mma = mode == 1 ? 35.0 + 0.45 * npad : 45.0 + 0.35 * npad;
    return (8500.0 + (double)DR * nch * nblk * kd * clk_mma) * wg_balance(nch, nwg);
  };
  static_cast<Tile&>(p.g) = plan_tiles(D, H, W, cin / 8, b_image_bytes(kd, nblk, npad), smem_limit, lim, amp, tile_clk, p.smem);
  p.g.Hp = H + 2; p.g.Wp = W + 2; p.g.pd = pd;
  p.grid = p.g.tiles_w * p.g.tiles_h * p.g.tiles_d;
  p.nwg = nwg;
  return p;
}

}  // namespace tc
}  // namespace tdm
