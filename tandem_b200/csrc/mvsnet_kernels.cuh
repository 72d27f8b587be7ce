// CVA-MVSNet device kernels, generation 1 ("direct" path): fp32 accumulation, one thread per output
// position.  These kernels are the parity baseline for every layer; the wgmma implicit-GEMM
// kernels (conv_tc.cuh) replace the convolutions layer by layer and are validated against these and
// against the CPU oracle.
//
// Activation layout "P8" (shared with the tensor-core path): channel-group-planar with zero halos,
//     [C/8][D+2*pd][H+2][W+2][8]          (pd = 1 for volumes, 0 for the view axis of 2-D maps)
// so one position of one channel group is a 16-byte (16-bit types) vector, a row segment of a group
// is contiguous (1-D TMA bulk copies), and every 3x3x3 tap is a constant address shift inside a
// plane.  Halos are zeroed once at allocation; kernels only ever write the interior.
//
// Reference semantics restated here (never the reference's code):
//   FeatureNet / Conv2d+BN+ReLU      cva_mvsnet/models/module.py:496-531, 104-110
//   homography warp + aggregation    module.py:764-908, 1068-1110 ; gates cva_mvsnet.py:76-83
//   CostRegNet (Conv3d / Deconv3d)   module.py:577-600, 213-219, 272-278
//   softmax / expectation / conf     module.py:1116-1133
//   adaptive hypotheses              cva_mvsnet.py:143-147, module.py:1503-1565
//   edge filter                      module.py:1320-1361
#pragma once
#include <type_traits>

#include "common.cuh"

namespace tdm {

// Programmatic dependent launch (mvsnet.cu launch_pdl / launch_k): first statement of every kernel of the forward.  Launched with
// cudaLaunchAttributeProgrammaticStreamSerialization the grid may become resident while its predecessor still runs; it must not touch
// memory before griddepcontrol.wait (= predecessor complete and visible).  The trigger right behind the wait lets the NEXT kernel's
// launch latency / prologue overlap this grid (one kernel of look-ahead).  Launched normally, both instructions are no-ops apart from
// the trigger, which still lets a tensor-core successor set up its barriers and weight image early.
__device__ __forceinline__ void grid_dep_sync() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}


template <typename T>
struct P8 {
  T* p;
  int C, D, H, W;   // logical dims
  int pd;           // halo along D (0 or 1); H and W always carry a halo of 1
  int Hp, Wp;       // H+2, W+2
  long long gs;     // elements between channel groups = (D+2pd)*Hp*Wp*8
  __device__ __forceinline__ long long pos(int d, int h, int w) const {
    return ((((long long)(d + pd)) * Hp + (h + 1)) * Wp + (w + 1)) * 8;
  }
};

// ------------------------------------------------------------------------------------------------
// a1: u8 BGR HWC (window order) -> T [V][H][W][4] RGB/255 (+ zero 4th channel), reference view first.
// Replaces the scalar CPU loop + 25.8 MB pageable H2D of dr_mvsnet.cpp:190-217,260.
// ------------------------------------------------------------------------------------------------
struct ViewPtrs {
  const unsigned char* v[16];
};

// RAW255: the 16-bit engines store u8/256 - exact in fp16 / bf16 (8 significant bits, power-of-two scale) - and fold the
// remaining 256/255 of dr_mvsnet.cpp:203-210 into the first convolution's weights (which keeps the weights' magnitude, so
// their hi/lo halves stay in the normal fp16 range): the network input carries no rounding error at all, where u8/255
// rounded to 16 bit would inject a relative error of up to 2^-11 into every feature.  The fp32 parity engine divides as the
// reference does.
template <typename T, bool RAW255 = false>
__global__ void k_preprocess_bgr(ViewPtrs src, P8<T> out, int V, int HW) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)V * HW) return;
  int v = (int)(i / HW);
  int p = (int)(i - (long long)v * HW);
  const unsigned char* s = src.v[v] + 3ll * p;
  float o[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (RAW255) {
    o[0] = (float)s[2] * 0.00390625f; o[1] = (float)s[1] * 0.00390625f; o[2] = (float)s[0] * 0.00390625f;
  } else {
    o[0] = __fdiv_rn((float)s[2], 255.0f);
    o[1] = __fdiv_rn((float)s[1], 255.0f);
    o[2] = __fdiv_rn((float)s[0], 255.0f);
  }
  store_vec<T, 8>(out.p + out.pos(v, p / out.W, p % out.W), o);
}

// ------------------------------------------------------------------------------------------------
// a1 + the first FeatureNet layer in one kernel (16-bit engines): conv0.0 is 3 -> 8 channels, 3x3 (module.py:500) - 216 MACs per
// pixel, nothing for the FMA pipes - while the generic route costs two full-resolution round trips: k_preprocess_bgr writes a
// zero-padded 8-channel 16-bit image (5 of 8 channels are padding: 34 MB for 6.45 MB of pixels) that the tensor-core conv reads
// back.  Here every thread owns one pixel: the u8 BGR tile (+1 halo, zero outside the image = the conv's zero padding) is
// staged in shared memory, x = u8 / 255 is formed in fp32 exactly as dr_mvsnet.cpp:203-210 does, the 27 x 8 products run as
// FFMA against BN-folded fp32 weights held in the constant bank (uniform operands, no load instructions), bias + ReLU, one
// 16-byte store.  (Dividing inside the 27-tap loop instead of at staging time cost 65 us instead of the ~20 us of the FMAs.)  No 16-bit rounding of the input or of the weights at all.
// ------------------------------------------------------------------------------------------------
struct Conv00Weights {
  float w[27][8];   // [tap = kh*3+kw][cin = R,G,B][cout] flattened as [(tap*3 + cin)][cout]
  float bias[8];
};
__constant__ Conv00Weights c_conv00[8 /* kMaxEngines */];

template <typename T>
__global__ void __launch_bounds__(256) k_conv00_u8(const unsigned char* __restrict__ bgr /*[V][H][W][3], reference view first*/, P8<T> out, int H, int W, int slot) {
  grid_dep_sync();
  constexpr int TX = 32, TY = 8;
  __shared__ float tile[TY + 2][(TX + 2) * 3];   // x = u8 / 255 formed ONCE per input value (IEEE division, dr_mvsnet.cpp:203-210)
  const Conv00Weights& cw = c_conv00[slot];
  const int v = blockIdx.z;
  const int x0 = blockIdx.x * TX, y0 = blockIdx.y * TY;
  const unsigned char* img = bgr + (size_t)v * H * W * 3;
  for (int i = threadIdx.x; i < (TY + 2) * (TX + 2); i += 256) {
    const int ty = i / (TX + 2), tx = i - ty * (TX + 2);
    const int yy = y0 + ty - 1, xx = x0 + tx - 1;
    float b = 0.f, g = 0.f, r = 0.f;
    if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
      const unsigned char* s = img + 3ll * ((long long)yy * W + xx);
      b = __fdiv_rn((float)s[0], 255.0f); g = __fdiv_rn((float)s[1], 255.0f); r = __fdiv_rn((float)s[2], 255.0f);
    }
    tile[ty][3 * tx] = r; tile[ty][3 * tx + 1] = g; tile[ty][3 * tx + 2] = b;   // network channel order is RGB
  }
  __syncthreads();
  const int lx = threadIdx.x % TX, ly = threadIdx.x / TX;
  const int x = x0 + lx, y = y0 + ly;
  if (x >= W || y >= H) return;
  float acc[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) acc[c] = cw.bias[c];
#pragma unroll
  for (int kh = 0; kh < 3; ++kh)
#pragma unroll
    for (int kw = 0; kw < 3; ++kw)
#pragma unroll
      for (int ci = 0; ci < 3; ++ci) {
        const float xin = tile[ly + kh][3 * (lx + kw) + ci];
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[c] = fmaf(xin, cw.w[(kh * 3 + kw) * 3 + ci][c], acc[c]);
      }
#pragma unroll
  for (int c = 0; c < 8; ++c) acc[c] = fmaxf(acc[c], 0.f);
  store_vec<T, 8>(out.p + out.pos(v, y, x), acc);
}

// ------------------------------------------------------------------------------------------------
// Generic direct convolution / transposed convolution, channels-last.
// ------------------------------------------------------------------------------------------------
struct ConvGeom {
  int Di, Hi, Wi;
  int Do, Ho, Wo;
  int kd, kh, kw;
  int sd, sh, sw;
  int pd, ph, pw;
  int transposed;  // 0: conv, 1: transposed conv evaluated as a gather over output positions
  int relu;
  int res_mode;    // 0 none; 1 same-shape residual added after the activation; 2 residual is the
                   // nearest-neighbour x2 up-sampling (h,w) of a half-resolution tensor (FPN top-down)
};

// COUT_T output channels per thread (COUT_T == COUT: one thread owns a position; COUT_T == 8: blockIdx.y selects the
// 8-channel group, used for the small low-resolution layers where positions alone cannot fill 132 SMs).
template <typename TIn, typename TOut, int CIN, int COUT, int COUT_T = COUT>
__global__ void __launch_bounds__(128)
k_conv_direct(const P8<const TIn> in, const float* __restrict__ wgt /*[taps][CIN][COUT]*/,
              const float* __restrict__ bias /*[COUT] or null*/, const P8<const TOut> res,
              const P8<TOut> out, float* __restrict__ plain_out /*COUT==1: fp32 [D][H][W]*/, ConvGeom g,
              const P8<TOut> out_b = P8<TOut>{}, const float* __restrict__ bias_b = nullptr /*optional 2nd output = out + bias_b*/) {
  grid_dep_sync();
  constexpr int SLICE = CIN * COUT_T;
  constexpr int TAPS_PER_STAGE = (SLICE >= 4096) ? 1 : (4096 / SLICE);
  __shared__ __align__(16) float ws[TAPS_PER_STAGE * SLICE];
  const int co0 = blockIdx.y * COUT_T;

  const long long npos = (long long)g.Do * g.Ho * g.Wo;
  const long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const bool active = p < npos;
  int ow = 0, oh = 0, od = 0;
  if (active) {
    ow = (int)(p % g.Wo);
    long long t = p / g.Wo;
    oh = (int)(t % g.Ho);
    od = (int)(t / g.Ho);
  }
  float acc[COUT_T];
#pragma unroll
  for (int c = 0; c < COUT_T; ++c) acc[c] = 0.f;

  const int ntaps = g.kd * g.kh * g.kw;
  for (int t0 = 0; t0 < ntaps; t0 += TAPS_PER_STAGE) {
    const int nt = min(TAPS_PER_STAGE, ntaps - t0);
    __syncthreads();
    if constexpr (COUT_T == COUT) {
      for (int i = threadIdx.x; i < nt * SLICE; i += blockDim.x) ws[i] = wgt[(long long)t0 * SLICE + i];
    } else {
      for (int i = threadIdx.x; i < nt * SLICE; i += blockDim.x)
        ws[i] = wgt[((long long)t0 * CIN + i / COUT_T) * COUT + co0 + (i % COUT_T)];
    }
    __syncthreads();
    if (!active) continue;
    for (int tt = 0; tt < nt; ++tt) {
      const int t = t0 + tt;
      const int kw_ = t % g.kw;
      const int kh_ = (t / g.kw) % g.kh;
      const int kd_ = t / (g.kw * g.kh);
      int id, ih, iw;
      bool ok = true;
      if (!g.transposed) {
        id = od * g.sd - g.pd + kd_;
        ih = oh * g.sh - g.ph + kh_;
        iw = ow * g.sw - g.pw + kw_;
      } else {
        int nd = od + g.pd - kd_, nh = oh + g.ph - kh_, nw = ow + g.pw - kw_;
        ok = (nd % g.sd == 0) && (nh % g.sh == 0) && (nw % g.sw == 0) && nd >= 0 && nh >= 0 && nw >= 0;
        id = nd / g.sd; ih = nh / g.sh; iw = nw / g.sw;
      }
      ok = ok && id >= 0 && id < g.Di && ih >= 0 && ih < g.Hi && iw >= 0 && iw < g.Wi;
      if (!ok) continue;
      const TIn* ip = in.p + in.pos(id, ih, iw);
      const float* wt = ws + tt * SLICE;
      constexpr int CH = 8;
      static_assert(CIN % 8 == 0, "P8 layout: channel count must be a multiple of 8");
#pragma unroll 1
      for (int c0 = 0; c0 < CIN; c0 += CH) {
        float x[CH];
        load_vec<TIn, CH>(ip + (c0 >> 3) * in.gs, x);
#pragma unroll
        for (int ci = 0; ci < CH; ++ci) {
          const float* wr = wt + (c0 + ci) * COUT_T;
#pragma unroll
          for (int co = 0; co < COUT_T; ++co) acc[co] = fmaf(x[ci], wr[co], acc[co]);
        }
      }
    }
  }
  if (!active) return;
#pragma unroll
  for (int c = 0; c < COUT_T; ++c) {
    float v = acc[c] + (bias ? bias[co0 + c] : 0.f);
    if (g.relu) v = fmaxf(v, 0.f);
    acc[c] = v;
  }
  if constexpr (COUT == 1) {
    plain_out[p] = acc[0];
  } else {
    if (g.res_mode != 0) {
      const long long rp = g.res_mode == 1 ? res.pos(od, oh, ow) : res.pos(od, oh >> 1, ow >> 1);
#pragma unroll
      for (int c0 = 0; c0 < COUT_T; c0 += 8) {
        float r[8];
        load_vec<TOut, 8>(res.p + rp + ((co0 + c0) >> 3) * res.gs, r);
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[c0 + c] += r[c];
      }
    }
    const long long op = out.pos(od, oh, ow);
#pragma unroll
    for (int c0 = 0; c0 < COUT_T; c0 += 8) {
      float o8[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) o8[c] = acc[c0 + c];
      store_vec<TOut, 8>(out.p + op + ((co0 + c0) >> 3) * out.gs, o8);
      if (bias_b) {
#pragma unroll
        for (int c = 0; c < 8; ++c) o8[c] += bias_b[co0 + c0 + c];
        store_vec<TOut, 8>(out_b.p + op + ((co0 + c0) >> 3) * out_b.gs, o8);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// a7 tail: the `prob` layer (Conv3d 8 -> 1, 3x3x3, no bias / BN, module.py:577-600) as a direct fp32 convolution.
// With one output channel a tensor-core tile spends 15 of its 16 N columns on padding while streaming the same A operand,
// so this layer is cheaper on the FMA pipes: one thread owns PX consecutive outputs of a row, loads the PX+2 input vectors
// (8 fp16 channels = 16 B each) of each of the 9 (kd, kh) rows once with 128-bit loads (zero halos: no bounds tests), and
// multiplies them with weights that arrive as a __grid_constant__ kernel parameter, i.e. as constant-bank operands of the
// FFMAs (no weight loads at all).  fp32 accumulation with the fp32 BN-free weights of the checkpoint.
// The 864 FFMA + 432 conversions per thread are expected to lose to the tensor-core tile even at 1/16 utilisation, so this
// kernel is OFF by default (set_option("prob_direct", 1)) and serves as an independent check.
// ------------------------------------------------------------------------------------------------
struct ProbWeights {
  float w[27 * 8];   // [kd][kh][kw][cin]
};

template <int PX>
__global__ void __launch_bounds__(128)
k_prob_direct(P8<const __half> in, float* __restrict__ logits /*[D][H][W]*/, const __grid_constant__ ProbWeights Wt) {
  const int S = in.W / PX;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int s = idx % S;
  const int t = idx / S;
  const int h = t % in.H, d = t / in.H;
  if (d >= in.D) return;
  float acc[PX];
#pragma unroll
  for (int i = 0; i < PX; ++i) acc[i] = 0.f;
  // element offset of (d-1, h-1, w0-1); every tap row is a constant shift from it
  const unsigned base = (unsigned)((((d + in.pd - 1) * in.Hp + h) * in.Wp + s * PX) * 8);
  const unsigned plane = (unsigned)(in.Hp * in.Wp * 8), row = (unsigned)(in.Wp * 8);
#pragma unroll
  for (int kd = 0; kd < 3; ++kd) {
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const uint4* rp = reinterpret_cast<const uint4*>(in.p + base + kd * plane + kh * row);
      float x[PX + 2][8];
#pragma unroll
      for (int q = 0; q < PX + 2; ++q) {
        const uint4 v = __ldg(rp + q);
        const __half2* hv = reinterpret_cast<const __half2*>(&v);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(hv[j]);
          x[q][2 * j] = f.x;
          x[q][2 * j + 1] = f.y;
        }
      }
#pragma unroll
      for (int kw = 0; kw < 3; ++kw)
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const float wv = Wt.w[((kd * 3 + kh) * 3 + kw) * 8 + c];
#pragma unroll
          for (int i = 0; i < PX; ++i) acc[i] = fmaf(x[i + kw][c], wv, acc[i]);
        }
    }
  }
  float* op = logits + ((size_t)d * in.H + h) * in.W + s * PX;
  if constexpr (PX == 4) {
    *reinterpret_cast<float4*>(op) = make_float4(acc[0], acc[1], acc[2], acc[3]);
  } else {
#pragma unroll
    for (int i = 0; i < PX; ++i) op[i] = acc[i];
  }
}

// ------------------------------------------------------------------------------------------------
// a3/a4: depth hypotheses.  Stage 1: d_j = dmin + interval*j.  Later stages: per-pixel dmin map from
// the bilinear (align_corners=False) x2 up-sampling of the previous stage's dense depth.
// ------------------------------------------------------------------------------------------------
struct HypSpec {
  int adaptive;    // 0 uniform, 1 adaptive
  float dmin;      // uniform
  float interval;  // stage interval (ratio * base)
  int D;
};

__device__ __forceinline__ float hyp_value(const HypSpec& h, float dmin_px, int j) {
  if (!h.adaptive) return h.dmin + h.interval * (float)j;
  const float dmax = dmin_px + (float)h.D * h.interval;
  const float lin = (float)j / (float)h.D;  // torch.linspace(0,1,D+1)[j], exact for power-of-two D
  return dmin_px + (dmax - dmin_px) * lin;
}

// a4 without a kernel of its own (round 2): the lower end of a pixel's adaptive hypothesis range, d_min = max(up2(depth_prev) -
// half_range, 1e-3) with up2 = bilinear x2, align_corners=False (cva_mvsnet.py:143-147, module.py:1503-1565), evaluated where it
// is consumed - the cost-volume kernel's prologue and the regression - from the previous stage's depth map (4 L2-resident
// loads).  Explicit fma / mul intrinsics: every consumer must see bit-identical hypotheses.  map != nullptr reads the
// materialised map instead (k_adaptive_dmin, kept for the A/B and the fp32 parity engine's layer-wise tests).
struct DminSrc {
  const float* map;    // [H][W] or null
  const float* prev;   // [ph][pw] depth of the previous stage
  int ph, pw;
};
__device__ __forceinline__ float dmin_px(const DminSrc& s, int pix, int x, int y, float half_range) {
  if (s.map) return s.map[pix];
  const float sy = fmaxf(__fmaf_rn(0.5f, (float)y + 0.5f, -0.5f), 0.f), sx = fmaxf(__fmaf_rn(0.5f, (float)x + 0.5f, -0.5f), 0.f);
  const int y0 = (int)sy, x0 = (int)sx;
  const int y1 = min(y0 + 1, s.ph - 1), x1 = min(x0 + 1, s.pw - 1);
  const float ly = sy - (float)y0, lx = sx - (float)x0;
  const float hy = 1.f - ly, hx = 1.f - lx;
  const float t0 = __fmaf_rn(lx, s.prev[y0 * s.pw + x1], __fmul_rn(hx, s.prev[y0 * s.pw + x0]));
  const float t1 = __fmaf_rn(lx, s.prev[y1 * s.pw + x1], __fmul_rn(hx, s.prev[y1 * s.pw + x0]));
  const float up = __fmaf_rn(ly, t1, __fmul_rn(hy, t0));
  return fmaxf(up - half_range, 0.001f);
}

__global__ void k_adaptive_dmin(const float* __restrict__ prev /*[h][w]*/, int h, int w,
                                float* __restrict__ dmin /*[2h][2w]*/, const float* __restrict__ half_range_p) {
  const float half_range = *half_range_p;
  const int H = 2 * h, W = 2 * w;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H * W) return;
  const int y = i / W, x = i - y * W;
  float sy = fmaxf(0.5f * ((float)y + 0.5f) - 0.5f, 0.f);
  float sx = fmaxf(0.5f * ((float)x + 0.5f) - 0.5f, 0.f);
  int y0 = (int)sy, x0 = (int)sx;
  int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
  float ly = sy - (float)y0, lx = sx - (float)x0;
  float hy = 1.f - ly, hx = 1.f - lx;
  float up = hy * (hx * prev[y0 * w + x0] + lx * prev[y0 * w + x1]) +
             ly * (hx * prev[y1 * w + x0] + lx * prev[y1 * w + x1]);
  dmin[i] = fmaxf(up - half_range, 0.001f);
}

// ------------------------------------------------------------------------------------------------
// K1 (a5+a6): fused plane-sweep cost volume with view aggregation.  One thread per (d,h,w) voxel,
// w fastest: all sources are warped, differenced, gated and accumulated in registers and the final
// volume is written exactly once; the per-view warped volumes of the reference never exist.
// ------------------------------------------------------------------------------------------------
constexpr int kMaxSrc = 15;
// Per-call parameters (homographies, depth range, filter rank) live in ONE device buffer that is refreshed by a small
// async copy before every forward, so that the kernel arguments never change and the whole forward replays as a CUDA
// graph.
// fp16 volumes saturate instead of overflowing to inf (65504 * 32 = 2.1e6 in volume units; largest value seen: 9.5e3)
template <typename TV> __device__ __forceinline__ float vol_store(float v) {
  if constexpr (std::is_same<TV, __half>::value) return fminf(v, 65504.f);
  else return v;
}

struct CvParams {
  int nsrc, D, H, W;
  float rot[kMaxSrc][9];
  float trans[kMaxSrc][3];
  float gw1[64];       // folded gate layer 1 weights (per channel)
  float gb1, gw2, gb2; // folded scalars
  float gw1_scale;     // power of two with max|gw1| * gw1_scale in [0.5, 1): keeps the fp16 copy of gw1 in the normal range
  float dot_unscale;   // 4096 / gw1_scale: undoes the fp16 path's operand scaling of the gate's dot product
  int view_aggregation;
  HypSpec hyp;
  float vol_scale;     // the volume is STORED as value * vol_scale (1 for fp32 / bf16 volumes; 2^-5 for the fp16 volume of the
                       // mixed16 engine, whose conv0 weights carry the inverse): a power of two, i.e. exact
};

// C = channels handled by ONE thread; CSPLIT adjacent lanes share a voxel and split its channels (C*CSPLIT in total):
// halves the register footprint of the 32-channel stage (222 -> ~127 regs, 12 % -> 37 % occupancy) at the price of
// one warp shuffle per view for the gate's dot product and duplicated (cheap) geometry.
struct CallParams {
  CvParams cv[3];
  HypSpec hyp[3];
  float half_range[3];
  unsigned cutoff[3];
};

// One slot per engine instance (several DrMvsnet handles may be in flight on a device); refreshed stream-ordered with
// cudaMemcpyToSymbolAsync before each forward.  Constant memory keeps the homographies as uniform operands of the inner
// loops (reading them through a global pointer or shared memory would add loads to the cost-volume kernel's inner loop).
constexpr int kMaxEngines = 8;
__constant__ CallParams c_call_params[kMaxEngines];

template <typename T, typename TV, int C, int CSPLIT = 1>
__global__ void __launch_bounds__(128)
k_cost_volume(P8<const T> feats /*views on the D axis, ref first*/, const DminSrc dsrc,
              P8<TV> vol, int slot, int stage /*per-call parameters: c_call_params[slot].cv[stage] (graph-replayable)*/) {
  const CvParams& p = c_call_params[slot].cv[stage];
  const long long n = (long long)p.D * p.H * p.W;
  long long i = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / CSPLIT;
  const int part = threadIdx.x % CSPLIT;          // which slice of the channels this lane owns
  const bool active = i < n;
  if (!active) i = n - 1;                          // keep the lane alive for the shuffles; its store is masked
  feats.p += (long long)part * (C / 8) * feats.gs;
  vol.p += (long long)part * (C / 8) * vol.gs;
  const float* gw1 = p.gw1 + part * C;
  const int x = (int)(i % p.W);
  const int y = (int)((i / p.W) % p.H);
  const int d = (int)(i / ((long long)p.W * p.H));
  const float depth = hyp_value(p.hyp, p.hyp.adaptive ? dmin_px(dsrc, y * p.W + x, x, y, c_call_params[slot].half_range[stage]) : 0.f, d);

  float ref[C];
  {
    const T* rp = feats.p + feats.pos(0, y, x);
#pragma unroll
    for (int c0 = 0; c0 < C; c0 += 8) {
      float t8[8];
      load_vec<T, 8>(rp + (c0 >> 3) * feats.gs, t8);
#pragma unroll
      for (int c = 0; c < 8; ++c) ref[c0 + c] = t8[c];
    }
  }
  float acc[C];
#pragma unroll
  for (int c = 0; c < C; ++c) acc[c] = 0.f;
  float sum[C], sq[C];
  if (!p.view_aggregation) {
#pragma unroll
    for (int c = 0; c < C; ++c) { sum[c] = ref[c]; sq[c] = ref[c] * ref[c]; }
  }
  const float fx = (float)x, fy = (float)y;
  const float half_w = 0.5f * (float)(p.W - 1), half_h = 0.5f * (float)(p.H - 1);

  for (int s = 0; s < p.nsrc; ++s) {
    const float* R = p.rot[s];
    const float* t = p.trans[s];
    const float rx = R[0] * fx + R[1] * fy + R[2];
    const float ry = R[3] * fx + R[4] * fy + R[5];
    const float rz = R[6] * fx + R[7] * fy + R[8];
    const float qx = rx * depth + t[0];
    const float qy = ry * depth + t[1];
    const float qz = rz * depth + t[2];
    float warped[C];
#pragma unroll
    for (int c = 0; c < C; ++c) warped[c] = 0.f;
    if constexpr (sizeof(T) == 2) {
      // 16-bit engines: one reciprocal instead of the reference's four IEEE divisions (the normalise / un-normalise
      // round trip of grid_sample is the identity up to 1 ulp), and no per-tap bounds tests: the P8 layout carries a
      // zero halo of one position, which IS grid_sample's zeros padding for every sample with -1 <= ix < W, -1 <= iy < H.
      const float inv = __frcp_rn(qz);
      const float ix = qx * inv, iy = qy * inv;
      if (!(qz < 0.001f) && ix >= -1.f && iy >= -1.f && ix < (float)p.W && iy < (float)p.H) {
        const float x0f = floorf(ix), y0f = floorf(iy);
        const float ax = ix - x0f, ay = iy - y0f;
        const float w00 = (1.f - ax) * (1.f - ay), w01 = ax * (1.f - ay), w10 = (1.f - ax) * ay, w11 = ax * ay;
        const T* tp = feats.p + feats.pos(s + 1, (int)y0f, (int)x0f);
        const int row = feats.Wp * 8;
        if constexpr (std::is_same<T, __half>::value) {
          // fp16 features: the 4-tap interpolation runs as packed HFMA2 (2 channels per instruction) and only the result is
          // widened to fp32 - 48 instead of 128 instructions per 16 channels.  The extra rounding (<= 2^-11 relative, the
          // same size as the storage quantisation of the features themselves) is covered by the Abs Rel tests.
          const __half2 h00 = __float2half2_rn(w00), h01 = __float2half2_rn(w01), h10 = __float2half2_rn(w10), h11 = __float2half2_rn(w11);
#pragma unroll
          for (int c0 = 0; c0 < C; c0 += 8) {
            const T* tq = tp + (c0 >> 3) * feats.gs;
            const uint4 q00 = __ldg(reinterpret_cast<const uint4*>(tq)), q01 = __ldg(reinterpret_cast<const uint4*>(tq + 8));
            const uint4 q10 = __ldg(reinterpret_cast<const uint4*>(tq + row)), q11 = __ldg(reinterpret_cast<const uint4*>(tq + row + 8));
            const __half2* a00 = reinterpret_cast<const __half2*>(&q00);
            const __half2* a01 = reinterpret_cast<const __half2*>(&q01);
            const __half2* a10 = reinterpret_cast<const __half2*>(&q10);
            const __half2* a11 = reinterpret_cast<const __half2*>(&q11);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const __half2 r = __hfma2(a11[k], h11, __hfma2(a10[k], h10, __hfma2(a01[k], h01, __hmul2(a00[k], h00))));
              const float2 rf = __half22float2(r);
              warped[c0 + 2 * k] = rf.x;
              warped[c0 + 2 * k + 1] = rf.y;
            }
          }
        } else {
#pragma unroll
          for (int c0 = 0; c0 < C; c0 += 8) {
            const T* tq = tp + (c0 >> 3) * feats.gs;
            float f00[8], f01[8], f10[8], f11[8];
            load_vec<T, 8>(tq, f00);
            load_vec<T, 8>(tq + 8, f01);
            load_vec<T, 8>(tq + row, f10);
            load_vec<T, 8>(tq + row + 8, f11);
#pragma unroll
            for (int c = 0; c < 8; ++c)
              warped[c0 + c] = fmaf(f11[c], w11, fmaf(f10[c], w10, fmaf(f01[c], w01, f00[c] * w00)));
          }
        }
      }
    } else {
    const float u = qx / qz, v = qy / qz;
    // grid_sample(align_corners=True) round trip through normalised coordinates
    const float gx = u / half_w - 1.f, gy = v / half_h - 1.f;
    const float ix = ((gx + 1.f) * 0.5f) * (float)(p.W - 1);
    const float iy = ((gy + 1.f) * 0.5f) * (float)(p.H - 1);
    const bool finite = (ix == ix) && (iy == iy) && fabsf(ix) < 1e8f && fabsf(iy) < 1e8f;
    if (finite && !(qz < 0.001f)) {
      const float x0f = floorf(ix), y0f = floorf(iy);
      const int x0 = (int)x0f, y0 = (int)y0f;
      const float ax = ix - x0f, ay = iy - y0f;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int xx = x0 + (k & 1), yy = y0 + (k >> 1);
        const float wgt = ((k & 1) ? ax : 1.f - ax) * ((k >> 1) ? ay : 1.f - ay);
        if (xx >= 0 && xx < p.W && yy >= 0 && yy < p.H) {
          const T* tp = feats.p + feats.pos(s + 1, yy, xx);
#pragma unroll
          for (int c0 = 0; c0 < C; c0 += 8) {
            float f[8];
            load_vec<T, 8>(tp + (c0 >> 3) * feats.gs, f);
#pragma unroll
            for (int c = 0; c < 8; ++c) warped[c0 + c] = fmaf(f[c], wgt, warped[c0 + c]);
          }
        }
      }
    }
    }  // exact (fp32 parity) path
    if (p.view_aggregation) {
      float dot = 0.f;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const float df = warped[c] - ref[c];
        warped[c] = df * df;
        dot = fmaf(gw1[c], warped[c], dot);
      }
      if constexpr (CSPLIT == 2) dot += __shfl_xor_sync(0xffffffffu, dot, 1);
      const float h1 = fmaxf(dot + p.gb1, 0.f);
      const float g = fmaxf(fmaf(p.gw2, h1, p.gb2), 0.f) + 1.f;
#pragma unroll
      for (int c = 0; c < C; ++c) acc[c] = fmaf(g, warped[c], acc[c]);
    } else {
#pragma unroll
      for (int c = 0; c < C; ++c) { sum[c] += warped[c]; sq[c] = fmaf(warped[c], warped[c], sq[c]); }
    }
  }
  if (p.view_aggregation) {
    const float dv = (float)p.nsrc;
    if constexpr (sizeof(T) == 2) {
      const float idv = 1.f / dv;
#pragma unroll
      for (int c = 0; c < C; ++c) acc[c] *= idv;
    } else {
#pragma unroll
      for (int c = 0; c < C; ++c) acc[c] = acc[c] / dv;
    }
  } else {
    const float nv = (float)(p.nsrc + 1);
#pragma unroll
    for (int c = 0; c < C; ++c) { const float m = sum[c] / nv; acc[c] = sq[c] / nv - m * m; }
  }
  if (active) {
    const long long op = vol.pos(d, y, x);
#pragma unroll
    for (int c0 = 0; c0 < C; c0 += 8) {
      float o8[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) o8[c] = vol_store<TV>(acc[c0 + c] * p.vol_scale);
      store_vec<TV, 8>(vol.p + op + (c0 >> 3) * vol.gs, o8);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// a6': view-aggregation cost volume, fp16 features (the mixed16 engine's kernel; k_cost_volume above stays the exact fp32
// parity path and the variance path).  The generic kernel is instruction-issue bound (ncu: 60-82 % issue slots, ~160
// instructions per (voxel, view) sample at C = 8, DRAM 1-4 %), so this one removes instructions:
//  * one thread owns ND consecutive depth hypotheses of a pixel: the view's R*[x y 1]^T, its constant-bank loads and the
//    gate weights are shared by ND samples, and the ND samples walk along the epipolar line (L1 locality);
//  * packed fp16 math up to the squared difference: the bilinear chain starts from -ref, so it yields (warped - ref)
//    directly; all fp16 operands carry a 1/64 scale (weights and ref; exact, a power of two) so the square, scaled by
//    1/4096, cannot overflow before |warped - ref| = 16376 (features are fp16 themselves; max seen 115);
//  * the gate's dot product runs in HFMA2 against a normalised fp16 copy of gw1 and is un-scaled in fp32;
//  * accumulation over views stays fp32 (ACC16 = false) as packed FFMA2, or fp16 (ACC16 = true, study variant);
//  * rcp.approx instead of the IEEE reciprocal, 32-bit element offsets.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float rcp_approx(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
// two independent correctly rounded FMAs (Hopper has no paired fp32 FMA instruction)
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

template <typename TV, int C /*channels of one thread*/, int CSPLIT, int ND, bool ACC16>
__global__ void __launch_bounds__(128)
k_cost_volume_va16(P8<const __half> feats, const DminSrc dsrc, P8<TV> vol, int slot, int stage) {
  grid_dep_sync();
  const CvParams& p = c_call_params[slot].cv[stage];
  constexpr float kS = 1.f / 64.f;
  const int HW = p.H * p.W;
  const int ngrp = (p.D + ND - 1) / ND;
  const int n = ngrp * HW;
  int i = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) / CSPLIT);
  const int part = threadIdx.x % CSPLIT;
  const bool active = i < n;
  if (!active) i = n - 1;                          // keep the lane alive for the shuffles; its stores are masked
  const int dg = i / HW, pix = i - dg * HW;
  const int y = pix / p.W, x = pix - y * p.W;
  const int d0 = dg * ND;
  const __half* fbase = feats.p + (size_t)part * (C / 8) * feats.gs;
  const int fgs = (int)feats.gs;

  __half2 nref[C / 2], gwh[C / 2];
  {
    const __half* rp = fbase + feats.pos(0, y, x);
    const __half2 ms = __float2half2_rn(-kS);
#pragma unroll
    for (int c0 = 0; c0 < C; c0 += 8) {
      const uint4 q = __ldg(reinterpret_cast<const uint4*>(rp + (size_t)(c0 >> 3) * feats.gs));
      const __half2* h = reinterpret_cast<const __half2*>(&q);
#pragma unroll
      for (int k = 0; k < 4; ++k) nref[c0 / 2 + k] = __hmul2(h[k], ms);
    }
#pragma unroll
    for (int k = 0; k < C / 2; ++k)
      gwh[k] = __floats2half2_rn(p.gw1[part * C + 2 * k] * p.gw1_scale, p.gw1[part * C + 2 * k + 1] * p.gw1_scale);
  }
  float depth[ND];
  {
    const float dmn = p.hyp.adaptive ? dmin_px(dsrc, pix, x, y, c_call_params[slot].half_range[stage]) : 0.f;
#pragma unroll
    for (int k = 0; k < ND; ++k) depth[k] = hyp_value(p.hyp, dmn, min(d0 + k, p.D - 1));
  }
  float2 acc[ND][C / 2];
  __half2 acch[ND][C / 2];
#pragma unroll
  for (int k = 0; k < ND; ++k)
#pragma unroll
    for (int c = 0; c < C / 2; ++c) { acc[k][c] = make_float2(0.f, 0.f); acch[k][c] = __float2half2_rn(0.f); }

  const float fx = (float)x, fy = (float)y, Wf = (float)p.W, Hf = (float)p.H;
  const int row = feats.Wp * 8;
  for (int s = 0; s < p.nsrc; ++s) {
    const float* R = p.rot[s];
    const float* t = p.trans[s];
    const float rx = R[0] * fx + R[1] * fy + R[2];
    const float ry = R[3] * fx + R[4] * fy + R[5];
    const float rz = R[6] * fx + R[7] * fy + R[8];
    const float t0 = t[0], t1 = t[1], t2 = t[2];
    const int vbase = ((s + 1 + feats.pd) * feats.Hp + 1) * feats.Wp + 1;
#pragma unroll
    for (int k = 0; k < ND; ++k) {
      const float qx = fmaf(rx, depth[k], t0), qy = fmaf(ry, depth[k], t1), qz = fmaf(rz, depth[k], t2);
      const float inv = rcp_approx(qz);
      const float ix = qx * inv, iy = qy * inv;
      __half2 df[C / 2];
      if (!(qz < 0.001f) && ix >= -1.f && iy >= -1.f && ix < Wf && iy < Hf) {
        const float x0f = floorf(ix), y0f = floorf(iy);
        const float ax = ix - x0f, ay = iy - y0f;
        const float wy1 = ay * kS, wy0 = fmaf(-ay, kS, kS), wx0 = 1.f - ax;
        const __half2 h00 = __float2half2_rn(wx0 * wy0), h01 = __float2half2_rn(ax * wy0);
        const __half2 h10 = __float2half2_rn(wx0 * wy1), h11 = __float2half2_rn(ax * wy1);
        const __half* tp = fbase + (size_t)(unsigned)((vbase + (int)y0f * feats.Wp + (int)x0f) * 8);
#pragma unroll
        for (int c0 = 0; c0 < C; c0 += 8) {
          const __half* tq = tp + (c0 >> 3) * fgs;
          const uint4 q00 = __ldg(reinterpret_cast<const uint4*>(tq)), q01 = __ldg(reinterpret_cast<const uint4*>(tq + 8));
          const uint4 q10 = __ldg(reinterpret_cast<const uint4*>(tq + row)), q11 = __ldg(reinterpret_cast<const uint4*>(tq + row + 8));
          const __half2* a00 = reinterpret_cast<const __half2*>(&q00);
          const __half2* a01 = reinterpret_cast<const __half2*>(&q01);
          const __half2* a10 = reinterpret_cast<const __half2*>(&q10);
          const __half2* a11 = reinterpret_cast<const __half2*>(&q11);
#pragma unroll
          for (int j = 0; j < 4; ++j)
            df[c0 / 2 + j] = __hfma2(a11[j], h11, __hfma2(a10[j], h10, __hfma2(a01[j], h01, __hfma2(a00[j], h00, nref[c0 / 2 + j]))));
        }
      } else {
#pragma unroll
        for (int c = 0; c < C / 2; ++c) df[c] = nref[c];     // grid_sample's zeros padding: warped = 0
      }
      __half2 dh = __float2half2_rn(0.f);
#pragma unroll
      for (int c = 0; c < C / 2; ++c) {
        df[c] = __hmul2(df[c], df[c]);                       // (warped - ref)^2 / 4096
        dh = __hfma2(df[c], gwh[c], dh);
      }
      const float2 dl = __half22float2(dh);
      float dot = dl.x + dl.y;
      if constexpr (CSPLIT == 2) dot += __shfl_xor_sync(0xffffffffu, dot, 1);
      const float h1 = fmaxf(fmaf(dot, p.dot_unscale, p.gb1), 0.f);
      const float g = fmaxf(fmaf(p.gw2, h1, p.gb2), 0.f) + 1.f;
      if constexpr (ACC16) {
        const __half2 gh = __float2half2_rn(g);
#pragma unroll
        for (int c = 0; c < C / 2; ++c) acch[k][c] = __hfma2(df[c], gh, acch[k][c]);
      } else {
        const float2 g2 = make_float2(g, g);
#pragma unroll
        for (int c = 0; c < C / 2; ++c) acc[k][c] = ffma2(__half22float2(df[c]), g2, acc[k][c]);
      }
    }
  }
  if (active) {
    const float sc = 4096.f / (float)p.nsrc * p.vol_scale;
    TV* vbase_p = vol.p + (size_t)part * (C / 8) * vol.gs;
#pragma unroll
    for (int k = 0; k < ND; ++k) {
      if (d0 + k < p.D) {
        const long long op = vol.pos(d0 + k, y, x);
#pragma unroll
        for (int c0 = 0; c0 < C; c0 += 8) {
          float o8[8];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 v = ACC16 ? __half22float2(acch[k][c0 / 2 + j]) : acc[k][c0 / 2 + j];
            o8[2 * j] = vol_store<TV>(v.x * sc);
            o8[2 * j + 1] = vol_store<TV>(v.y * sc);
          }
          store_vec<TV, 8>(vbase_p + op + (size_t)(c0 >> 3) * vol.gs, o8);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// a8: softmax over D + soft-argmin depth + 4-neighbour confidence, one thread per pixel.
// ------------------------------------------------------------------------------------------------
template <int MAXD, bool L2_LOADS>
__device__ __forceinline__ void regress_px(const float* __restrict__ logits /*[D][H][W]*/, const DminSrc& dsrc,
                                           float* __restrict__ depth, float* __restrict__ conf, int HW, int i, int x, int y,
                                           const HypSpec& hyp, float half_range) {
  const int D = hyp.D;
  float l[MAXD];
  float m = -INFINITY;
#pragma unroll
  for (int j = 0; j < MAXD; ++j)
    if (j < D) { l[j] = L2_LOADS ? __ldcg(logits + (long long)j * HW + i) : logits[(long long)j * HW + i]; m = fmaxf(m, l[j]); }
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < MAXD; ++j)
    if (j < D) { l[j] = expf(l[j] - m); s += l[j]; }
  const float dm = hyp.adaptive ? dmin_px(dsrc, i, x, y, half_range) : 0.f;
  float dsum = 0.f, isum = 0.f;
#pragma unroll
  for (int j = 0; j < MAXD; ++j)
    if (j < D) {
      l[j] = l[j] / s;
      dsum = fmaf(l[j], hyp_value(hyp, dm, j), dsum);
      isum = fmaf(l[j], (float)j, isum);
    }
  int idx = min(max((int)isum, 0), D - 1);
  float c = 0.f;
#pragma unroll
  for (int j = 0; j < MAXD; ++j)
    if (j < D && j >= idx - 1 && j <= idx + 2) c += l[j];
  depth[i] = dsum;
  conf[i] = c;
}

template <int MAXD>
__global__ void k_regress(const float* __restrict__ logits /*[D][H][W]*/, const DminSrc dsrc,
                          float* __restrict__ depth, float* __restrict__ conf, int HW, int W, const HypSpec* __restrict__ hyp_p,
                          const float* __restrict__ half_range_p) {
  grid_dep_sync();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= HW) return;
  regress_px<MAXD, false>(logits, dsrc, depth, conf, HW, i, i % W, i / W, *hyp_p, *half_range_p);
}

// the same arithmetic as the tail of the tensor-core prob convolution (conv_tc_is.cuh, Tail): the epilogue thread that stored
// a pixel's D logits finishes the pixel, reading its own stores back from L2 (bit-identical to k_regress by construction)
template <int MAXD>
struct RegressTail {
  static constexpr bool enabled = true;
  DminSrc dsrc;
  float* depth;
  float* conf;
  const HypSpec* hyp;
  const float* half_range;
  __device__ __forceinline__ void operator()(const float* logits, int i, int x, int y, int HW) const {
    regress_px<MAXD, true>(logits, dsrc, depth, conf, HW, i, x, y, *hyp, *half_range);
  }
};

// ------------------------------------------------------------------------------------------------
// K4 (a9): edge filter.  (1) per-pixel 15-th smallest |window - centre| over a zero padded 5x5
// window; (2) exact k-th order statistic of the H*W edge values by a 3-pass radix select on the
// float bit patterns (all values >= 0 so the unsigned order equals the float order);
// (3) zero depth/confidence where edge > threshold.
// ------------------------------------------------------------------------------------------------
__global__ void k_edge_metric(const float* __restrict__ depth, float* __restrict__ edge, int H, int W) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H * W) return;
  const int y = i / W, x = i - y * W;
  const float c = depth[i];
  float e[25];
#pragma unroll
  for (int dy = -2; dy <= 2; ++dy)
#pragma unroll
    for (int dx = -2; dx <= 2; ++dx) {
      const int yy = y + dy, xx = x + dx;
      const float v = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? depth[yy * W + xx] : 0.f;
      e[(dy + 2) * 5 + dx + 2] = fabsf(v - c);
    }
  // partial selection: after pass k the k smallest are in e[0..k]
#pragma unroll
  for (int k = 0; k < 15; ++k) {
#pragma unroll
    for (int j = k + 1; j < 25; ++j) {
      const float a = e[k], b = e[j];
      e[k] = fminf(a, b);
      e[j] = fmaxf(a, b);
    }
  }
  edge[i] = e[14];
}

struct SelectState {
  unsigned prefix;   // bits decided so far (high bits)
  unsigned k;        // remaining rank inside the current prefix bucket
  unsigned hist[2048];
};

__global__ void k_select_init(SelectState* st, const unsigned* __restrict__ k) {
  for (int i = threadIdx.x; i < 2048; i += blockDim.x) st->hist[i] = 0;
  if (threadIdx.x == 0) { st->prefix = 0; st->k = *k; }
}

// pass p: 0 -> bits 31..21 (11), 1 -> bits 20..10 (11), 2 -> bits 9..0 (10)
__global__ void k_select_hist(const float* __restrict__ v, int n, SelectState* st, int pass) {
  __shared__ unsigned h[2048];
  for (int i = threadIdx.x; i < 2048; i += blockDim.x) h[i] = 0;
  __syncthreads();
  const unsigned prefix = st->prefix;
  const int shift = pass == 0 ? 21 : (pass == 1 ? 10 : 0);
  const unsigned hi_mask = pass == 0 ? 0u : (pass == 1 ? 0xFFE00000u : 0xFFFFFC00u);
  const unsigned bmask = pass == 2 ? 0x3FFu : 0x7FFu;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned b = __float_as_uint(v[i]);
    if ((b & hi_mask) == prefix) atomicAdd(&h[(b >> shift) & bmask], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2048; i += blockDim.x)
    if (h[i]) atomicAdd(&st->hist[i], h[i]);
}

// one block of 1024 threads: parallel prefix over the 2048 bins, the thread whose bin pair contains rank k publishes
__global__ void __launch_bounds__(1024) k_select_scan(SelectState* st, int pass, float* thr_out) {
  __shared__ unsigned wsum[32];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int shift = pass == 0 ? 21 : (pass == 1 ? 10 : 0);
  const unsigned a = st->hist[2 * t], b = st->hist[2 * t + 1];
  const unsigned k = st->k, prefix = st->prefix;
  unsigned incl = a + b;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned n = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += n;
  }
  if (lane == 31) wsum[w] = incl;
  __syncthreads();
  unsigned off = 0;
  for (int i = 0; i < w; ++i) off += wsum[i];
  const unsigned excl = off + incl - (a + b);
  __syncthreads();   // everybody has read st->hist / st->k before they are overwritten
  st->hist[2 * t] = 0;
  st->hist[2 * t + 1] = 0;
  int bin = -1;
  unsigned nk = 0;
  if (k >= excl && k < excl + a) { bin = 2 * t; nk = k - excl; }
  else if (k >= excl + a && k < excl + a + b) { bin = 2 * t + 1; nk = k - excl - a; }
  if (bin >= 0) {
    const unsigned np = prefix | ((unsigned)bin << shift);
    st->k = nk;
    st->prefix = np;
    if (pass == 2) *thr_out = __uint_as_float(np);
  }
}

// ---- fused percentile select (round 2): 4 launches instead of 9 --------------------------------------------------------
// The exact k-th order statistic of the edge map is still a 3-pass radix select over the float bit patterns (11 + 11 + 10
// bits), but every pass is ONE launch: the CTAs histogram their share into shared memory, merge into the global histogram,
// and the LAST CTA to finish (ticket) scans the 2048 bins, narrows (prefix, k) for the next pass and re-zeroes the histogram.
// Pass 0 rides on the edge-metric kernel itself (the values are in registers there).  State between passes lives in SelectState;
// its histogram and ticket are zero whenever no select is in flight (zeroed at allocation and by every pass' last CTA).
struct SelectState2 {
  unsigned prefix, k, ticket, pad;
  unsigned hist[2048];
};

// blockDim.x == 256.  Called by every thread of the last CTA of pass `pass`.
__device__ __forceinline__ void select_scan_last_cta(SelectState2* st, int pass, unsigned k_in, unsigned prefix_in, float* thr_out) {
  __shared__ unsigned wsum[8];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int shift = pass == 0 ? 21 : (pass == 1 ? 10 : 0);
  unsigned c[8], tot = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) { c[j] = __ldcg(&st->hist[8 * t + j]); tot += c[j]; }
  unsigned incl = tot;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned n = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += n;
  }
  if (lane == 31) wsum[w] = incl;
  __syncthreads();
  unsigned off = 0;
  for (int i = 0; i < w; ++i) off += wsum[i];
  unsigned excl = off + incl - tot;
#pragma unroll
  for (int j = 0; j < 8; ++j) st->hist[8 * t + j] = 0;
  if (k_in >= excl && k_in < excl + tot) {            // exactly one thread
    unsigned kk = k_in - excl;
    int bin = 8 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (kk < c[j]) { bin = 8 * t + j; break; }
      kk -= c[j];
    }
    const unsigned np = prefix_in | ((unsigned)bin << shift);
    st->k = kk;
    st->prefix = np;
    if (pass == 2) *thr_out = __uint_as_float(np);
  }
  if (t == 0) st->ticket = 0;
}

// shared by the three passes: merge the CTA's shared-memory histogram, elect the last CTA, let it scan
__device__ __forceinline__ void select_finish_pass(SelectState2* st, unsigned* h /*shared [2048]*/, int pass, unsigned k_in, unsigned prefix_in,
                                                   float* thr_out) {
  __shared__ bool is_last;
  __syncthreads();
  for (int i = threadIdx.x; i < 2048; i += blockDim.x)
    if (h[i]) atomicAdd(&st->hist[i], h[i]);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(&st->ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (is_last) {
    __threadfence();
    select_scan_last_cta(st, pass, k_in, prefix_in, thr_out);
  }
}

// a9 edge metric + pass 0 of the percentile select (bits 31..21)
__global__ void __launch_bounds__(256) k_edge_metric_select0(const float* __restrict__ depth, float* __restrict__ edge, int H, int W,
                                                             SelectState2* st, const unsigned* __restrict__ cutoff) {
  grid_dep_sync();
  __shared__ unsigned h[2048];
  for (int i = threadIdx.x; i < 2048; i += blockDim.x) h[i] = 0;
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < H * W) {
    const int y = i / W, x = i - y * W;
    const float c = depth[i];
    float e[25];
#pragma unroll
    for (int dy = -2; dy <= 2; ++dy)
#pragma unroll
      for (int dx = -2; dx <= 2; ++dx) {
        const int yy = y + dy, xx = x + dx;
        const float v = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? depth[yy * W + xx] : 0.f;
        e[(dy + 2) * 5 + dx + 2] = fabsf(v - c);
      }
#pragma unroll
    for (int k = 0; k < 15; ++k) {
#pragma unroll
      for (int j = k + 1; j < 25; ++j) {
        const float a = e[k], b = e[j];
        e[k] = fminf(a, b);
        e[j] = fmaxf(a, b);
      }
    }
    edge[i] = e[14];
    atomicAdd(&h[__float_as_uint(e[14]) >> 21], 1u);
  }
  select_finish_pass(st, h, 0, *cutoff, 0u, nullptr);
}

// passes 1 (bits 20..10) and 2 (bits 9..0)
__global__ void __launch_bounds__(256) k_select_pass(const float* __restrict__ v, int n, SelectState2* st, int pass, float* thr_out) {
  grid_dep_sync();
  __shared__ unsigned h[2048];
  for (int i = threadIdx.x; i < 2048; i += blockDim.x) h[i] = 0;
  const unsigned prefix = st->prefix, k_in = st->k;      // written by the previous pass' last CTA (kernel boundary in between)
  __syncthreads();
  const int shift = pass == 1 ? 10 : 0;
  const unsigned hi_mask = pass == 1 ? 0xFFE00000u : 0xFFFFFC00u;
  const unsigned bmask = pass == 2 ? 0x3FFu : 0x7FFu;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned b = __float_as_uint(v[i]);
    if ((b & hi_mask) == prefix) atomicAdd(&h[(b >> shift) & bmask], 1u);
  }
  select_finish_pass(st, h, pass, k_in, prefix, thr_out);
}

__global__ void k_apply_edge_mask(const float* __restrict__ edge, const float* __restrict__ thr,
                                  const float* __restrict__ depth_dense, const float* __restrict__ conf_dense,
                                  float* __restrict__ depth, float* __restrict__ conf, int n) {
  grid_dep_sync();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool m = edge[i] > *thr;
  depth[i] = m ? 0.f : depth_dense[i];
  conf[i] = m ? 0.f : conf_dense[i];
}

// layout helper for tests: channels-last T -> planar fp32 [C][N]
template <typename T>
__global__ void k_p8_to_planar_f32(const P8<const T> in, float* __restrict__ out) {
  const long long npos = (long long)in.D * in.H * in.W;
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= npos * in.C) return;
  const int c = (int)(i / npos);
  long long pos = i - (long long)c * npos;
  const int w = (int)(pos % in.W);
  pos /= in.W;
  const int h = (int)(pos % in.H);
  const int d = (int)(pos / in.H);
  out[i] = to_f<T>(in.p[in.pos(d, h, w) + (c >> 3) * in.gs + (c & 7)]);
}

}  // namespace tdm
