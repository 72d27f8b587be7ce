// n10: DSO's pixel selection on the device (PixelSelector, tandem/src/FullSystem/PixelSelector2.cpp:41-438): the random
// pattern of the constructor (:41-56), makeHists (:78-141), select (:295-438) and makeMaps (:142-291), on a tdm_pyramid's
// levels 0..2, plus the candidate list of makeNewTraces (FullSystem.cpp:1634-1646) that immature.cu constructs from.  Every
// float operation is the reference's own, correctly rounded and in its order (__f*_rn, no contraction); oracle/pixsel_oracle.c
// restates the same statements on the CPU.
//
// Shape (DESIGN.md, n10).  select's visiting order carries one serial dependency: the direction of every block is
// directions[randomPattern[n2] & 0xF], n2 the number of cells (pot x pot) that made a level-2 selection earlier.  A level-3 or
// level-4 selection never moves n2, and a cell selects under direction d iff one of its pixels passes the level-0 threshold
// with a non-zero score under d.  So
//   k_mask   one thread per cell: the 16-bit mask of the directions under which the cell selects;
//   k_chain  one warp walks the cells in visiting order, 32 at a time: cells with mask 0 or 0xFFFF have fixed increments
//            (a popcount), the others are resolved one by one from the pattern (its prefix in shared memory); it leaves n2 at
//            the start of every level-4 block;
//   k_pick   one warp per level-4 block: from that n2 and the masks, each cell's direction and selection, then the type-1,
//            type-2 and type-4 pixels as first maxima in visiting order (warp reductions);
//   k_decide one thread: makeMaps' re-selection decision.  The host enqueues recursionsLeft + 1 rounds; once a round has
//            decided to keep its selection the later rounds return at once, so a call has one host wait.
// The subsample and makeNewTraces' list rank the selections in raster order (row counts, a scan, ballots within a row).
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>

#include <cub/block/block_scan.cuh>

#include "tracker.h"

namespace tdm {

namespace {

__device__ __forceinline__ float fm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fs(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fd(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ int cdiv_d(int a, int b) { return (int)(((long long)a + b - 1) / b); }

// select's directions (:312-328): double literals converted to float, as Vec2f's constructor converts them
__constant__ float c_dirs[16][2] = {{0, 1.0000},       {0.3827, 0.9239},  {0.1951, 0.9808},  {0.9239, 0.3827},
                                    {0.7071, 0.7071},  {0.3827, -0.9239}, {0.8315, 0.5556},  {0.8315, -0.5556},
                                    {0.5556, -0.8315}, {0.9808, 0.1951},  {0.9239, -0.3827}, {0.7071, -0.7071},
                                    {0.5556, 0.8315},  {0.9808, -0.1951}, {1.0000, 0.0000},  {0.1951, -0.9808}};

constexpr int kThreads = 256, kGrid = 528;   // grid-stride kernels: every item is computed alone, so any grid gives the same
constexpr int kRpShared = 32768;             // k_chain's shared prefix of the pattern

struct SelSettings {   // tdm_select_settings
  float cut, add, dw1;
  int dir_dist;
};

// the state of one call, on the device
struct SelState {
  int pot, rec_left, active, reselected;   // active: the next round selects
  int n[3], pot_used, nonuniform;
  int subsample, charTH, num_have, dropped;
  int pot_after, n_cand;
};

struct Img {
  const float* dI;   // level 0, (I, dx, dy)
  const float *ag0, *ag1, *ag2;
  const float* ths;  // thsSmoothed, w32 * h32
  const unsigned char* rp;
  float* map;
  int w, h;
};

// thsSmoothed[(xf>>5) + (yf>>5) * w32]; a flat index at or beyond w32 * h32 reads 0 (the reference's array is uninitialised
// there)
__device__ __forceinline__ float th_at(const Img& I, int xf, int yf) {
  const int w32 = I.w / 32, h32 = I.h / 32, i = (xf >> 5) + (yf >> 5) * w32;
  return i < w32 * h32 ? __ldg(I.ths + i) : 0.f;
}
__device__ __forceinline__ float score(float dx, float dy, int d) {
  return fabsf(fa(fm(dx, c_dirs[d][0]), fm(dy, c_dirs[d][1])));
}
__device__ __forceinline__ bool tested(int xf, int yf, int w, int h) { return !(xf < 4 || xf >= w - 5 || yf < 4 || yf > h - 4); }

// makeHists, first half: one block per full 32 x 32 cell; ths = computeHistQuantil(hist, cut) + add
__global__ void __launch_bounds__(kThreads) k_hist(const float* __restrict__ ag0, int w, int h, SelSettings S, float* __restrict__ ths) {
  __shared__ int hist[91];
  const int w32 = w / 32, x = blockIdx.x % w32, y = blockIdx.x / w32;
  for (int i = threadIdx.x; i < 91; i += blockDim.x) hist[i] = 0;
  __syncthreads();
  for (int k = threadIdx.x; k < 1024; k += blockDim.x) {
    const int it = (k & 31) + 32 * x, jt = (k >> 5) + 32 * y;
    if (it > w - 2 || jt > h - 2 || it < 1 || jt < 1) continue;
    const float s = __fsqrt_rn(ag0[it + (size_t)jt * w]);
    int g = s < 49.f ? (int)s : 48;   // a non-finite gradient (the pyramid makes none) counts as the clamp
    if (g > 48) g = 48;
    atomicAdd(&hist[g + 1], 1);
    atomicAdd(&hist[0], 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int th = (int)fa(fm((float)hist[0], S.cut), 0.5f), q = 90;   // computeHistQuantil, :66-75
    for (int i = 0; i < 90; i++) {
      th -= hist[i + 1];
      if (th < 0) { q = i; break; }
    }
    ths[blockIdx.x] = fa((float)q, S.add);
  }
}

// makeHists, second half: thsSmoothed = (mean of the up-to-9 neighbours)^2, summed in the reference's order
__global__ void k_smooth(const float* __restrict__ ths, int w32, int h32, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= w32 * h32) return;
  const int x = c % w32, y = c / w32;
  float sum = 0.f, num = 0.f;
  auto add = [&](int i) { num = fa(num, 1.f); sum = fa(sum, ths[i]); };
  if (x > 0) {
    if (y > 0) add(x - 1 + (y - 1) * w32);
    if (y < h32 - 1) add(x - 1 + (y + 1) * w32);
    add(x - 1 + y * w32);
  }
  if (x < w32 - 1) {
    if (y > 0) add(x + 1 + (y - 1) * w32);
    if (y < h32 - 1) add(x + 1 + (y + 1) * w32);
    add(x + 1 + y * w32);
  }
  if (y > 0) add(x + (y - 1) * w32);
  if (y < h32 - 1) add(x + (y + 1) * w32);
  add(x + y * w32);
  out[c] = fm(fd(sum, num), fd(sum, num));
}

// per cell (pot x pot from the origin, clipped), the directions under which it makes a level-2 selection; clears the map
__global__ void __launch_bounds__(kThreads) k_mask(const SelState* __restrict__ st, Img I, SelSettings S, float thF,
                                                   uint16_t* __restrict__ mask) {
  if (!st->active) return;
  const int pot = st->pot, w = I.w, h = I.h, cw = cdiv_d(w, pot), ch = cdiv_d(h, pot);
  const long long ncell = (long long)cw * ch, npix = (long long)w * h;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < std::max(ncell, npix); i += (long long)gridDim.x * blockDim.x) {
    if (i < npix) I.map[i] = 0.f;
    if (i >= ncell) continue;
    const int x0 = (int)(i % cw) * pot, y0 = (int)(i / cw) * pot;
    const int x1 = (int)std::min<long long>((long long)x0 + pot, w), y1 = (int)std::min<long long>((long long)y0 + pot, h);
    unsigned m = 0;
    for (int yf = y0; yf < y1 && m != 0xFFFFu; ++yf)
      for (int xf = x0; xf < x1 && m != 0xFFFFu; ++xf) {
        if (!tested(xf, yf, w, h)) continue;
        const size_t idx = xf + (size_t)yf * w;
        if (!(__ldg(I.ag0 + idx) > fm(th_at(I, xf, yf), thF))) continue;
        if (!S.dir_dist) { m = 0xFFFFu; break; }   // the score is ag0 > 0
        const float dx = __ldg(I.dI + 3 * idx + 1), dy = __ldg(I.dI + 3 * idx + 2);
#pragma unroll
        for (int d = 0; d < 16; ++d)
          if (score(dx, dy, d) > 0.f) m |= 1u << d;
      }
    mask[i] = (uint16_t)m;
  }
}

// n2 at the start of every level-4 block.  One warp; lanes 0-15 hold the 16 cells of one level-4 block in visiting order
// (level-3 blocks in raster order, cells in raster order within each), lanes 16-31 those of the next block.
__global__ void __launch_bounds__(kThreads) k_chain(SelState* __restrict__ st, const uint16_t* __restrict__ mask,
                                                    const unsigned char* __restrict__ rp, int w, int h, int* __restrict__ n2b4) {
  if (!st->active) return;
  __shared__ __align__(16) unsigned char srp[kRpShared];
  const int pot = st->pot, cw = cdiv_d(w, pot), ch = cdiv_d(h, pot), bw = cdiv_d(cw, 4), bh = cdiv_d(ch, 4);
  // n2 stays below the number of cells: only that prefix of the pattern can be read
  const int pre = (int)std::min<long long>(std::min<long long>((long long)w * h, (long long)cw * ch), kRpShared);
  for (int i = threadIdx.x; i < pre / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(srp)[i] = __ldg(reinterpret_cast<const uint4*>(rp) + i);
  for (int i = pre / 16 * 16 + threadIdx.x; i < pre; i += blockDim.x) srp[i] = rp[i];
  __syncthreads();
  if (threadIdx.x >= 32) return;
  const int lane = threadIdx.x;
  const int nb = bw * bh, z = lane & 15;
  const int ox = 2 * ((z >> 2) & 1) + (z & 1), oy = 2 * (z >> 3) + ((z >> 1) & 1);
  int n2 = 0, nonuni_cells = 0;
  for (int b0 = 0; b0 < nb; b0 += 2) {
    const int b = b0 + (lane >> 4), gx = 4 * (b % bw) + ox, gy = 4 * (b / bw) + oy;
    const unsigned m = (b < nb && gx < cw && gy < ch) ? mask[gx + (size_t)gy * cw] : 0u;
    unsigned nonuni = __ballot_sync(0xffffffffu, m != 0u && m != 0xFFFFu);
    unsigned sel = __ballot_sync(0xffffffffu, m == 0xFFFFu);
    nonuni_cells += __popc(nonuni);
    while (nonuni) {
      const int j = __ffs(nonuni) - 1;
      const int n2j = n2 + __popc(sel & ((1u << j) - 1u));
      const int d = (n2j < pre ? srp[n2j] : __ldg(rp + n2j)) & 0xF;
      if ((__shfl_sync(0xffffffffu, m, j) >> d) & 1u) sel |= 1u << j;
      nonuni &= nonuni - 1u;
    }
    if (lane == 0) n2b4[b0] = n2;
    if (lane == 16 && b0 + 1 < nb) n2b4[b0 + 1] = n2 + __popc(sel & 0xFFFFu);
    n2 += __popc(sel);
  }
  if (lane == 0) {
    st->n[0] = n2; st->n[1] = 0; st->n[2] = 0;
    st->nonuniform = nonuni_cells;
  }
}

// The first maximum of a candidate's value v (> 0) in visiting order `key` over the warp: (value, key, pixel)
struct Best {
  float v;
  long long key;
  int idx;
};
__device__ __forceinline__ void offer(Best& b, float v, long long key, int idx) {
  if (v > b.v || (v == b.v && v > 0.f && key < b.key)) { b.v = v; b.key = key; b.idx = idx; }
}
__device__ __forceinline__ Best warp_best(Best b) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float v = __shfl_xor_sync(0xffffffffu, b.v, o);
    const long long key = __shfl_xor_sync(0xffffffffu, b.key, o);
    const int idx = __shfl_xor_sync(0xffffffffu, b.idx, o);
    offer(b, v, key, idx);
  }
  return b;
}

// select's loop (:339-434) for one level-4 block per warp, from the block's n2.  By (b)-(e) of DESIGN.md (n10): cell z
// (visiting order) has direction rp[n2_z] and selects iff its mask holds that direction, its pixel the first maximum in
// raster order; a level-3 block without a type-1 cell selects the first maximum of its pixels in visiting order under its
// cells' direction; the level-4 block, without a type-1 or type-2 selection, the first maximum of all its pixels.  Each is a
// warp reduction over (value, visiting-order key), ties to the smaller key, as the strict > keeps the first.
constexpr int kPickThreads = 128;
__global__ void __launch_bounds__(kPickThreads) k_pick(SelState* __restrict__ st, Img I, SelSettings S, float thF,
                                                       const uint16_t* __restrict__ mask, const int* __restrict__ n2b4) {
  if (!st->active) return;
  const int lane = threadIdx.x & 31;
  const int pot = st->pot, w = I.w, h = I.h, w1 = w / 2, w2 = w / 4;
  const int cw = cdiv_d(w, pot), ch = cdiv_d(h, pot), bw = cdiv_d(cw, 4), nb = bw * cdiv_d(ch, 4);
  const float dw1 = S.dw1, dw2 = fm(dw1, dw1);
  int c3 = 0, c4 = 0;
  for (int b = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); b < nb; b += (int)((gridDim.x * blockDim.x) >> 5)) {
    // the 16 cells in visiting order: direction and selection, by the chain from the block's n2
    const int z = lane & 15, gx = 4 * (b % bw) + 2 * ((z >> 2) & 1) + (z & 1), gy = 4 * (b / bw) + 2 * (z >> 3) + ((z >> 1) & 1);
    const bool exists = gx < cw && gy < ch;
    const unsigned m = exists ? mask[gx + (size_t)gy * cw] : 0u;
    int n2 = n2b4[b], dirs = 0;   // lane z < 16 keeps its cell's direction
    unsigned selected = 0;
    for (int k = 0; k < 16; ++k) {
      const int d = __ldg(I.rp + n2) & 0xF;
      const unsigned mk = __shfl_sync(0xffffffffu, m, k);
      if (lane == k) dirs = d;
      if ((mk >> d) & 1u) { selected |= 1u << k; ++n2; }
    }
    // type 1: per selected cell, the first maximum in raster order
    for (unsigned sm = selected; sm; sm &= sm - 1u) {
      const int k = __ffs(sm) - 1, d = __shfl_sync(0xffffffffu, dirs, k);
      const int cx = __shfl_sync(0xffffffffu, gx, k) * pot, cy = __shfl_sync(0xffffffffu, gy, k) * pot;
      const int mx = std::min(pot, w - cx), npx = mx * std::min(pot, h - cy);
      Best bb{0.f, 0, -1};
      for (int q = lane; q < npx; q += 32) {
        const int xf = cx + q % mx, yf = cy + q / mx, idx = xf + w * yf;
        if (!tested(xf, yf, w, h)) continue;
        const float ag0 = __ldg(I.ag0 + idx);
        if (!(ag0 > fm(th_at(I, xf, yf), thF))) continue;
        offer(bb, S.dir_dist ? score(__ldg(I.dI + 3 * (size_t)idx + 1), __ldg(I.dI + 3 * (size_t)idx + 2), d) : ag0, q, idx);
      }
      bb = warp_best(bb);
      if (lane == 0) I.map[bb.idx] = 1.f;
    }
    // type 2: per level-3 block without a type-1 cell, the first maximum in visiting order under its cells' direction
    int any23 = selected != 0u;
    for (int s3 = 0; s3 < 4; ++s3) {
      if ((selected >> (4 * s3)) & 0xFu) continue;
      const int d = __shfl_sync(0xffffffffu, dirs, 4 * s3);
      Best bb{0.f, 0, -1};
      for (int k = 4 * s3; k < 4 * s3 + 4; ++k) {
        const int cgx = __shfl_sync(0xffffffffu, gx, k), cgy = __shfl_sync(0xffffffffu, gy, k);
        if (cgx >= cw || cgy >= ch) continue;
        const int cx = cgx * pot, cy = cgy * pot, mx = std::min(pot, w - cx), npx = mx * std::min(pot, h - cy);
        for (int q = lane; q < npx; q += 32) {
          const int xf = cx + q % mx, yf = cy + q / mx, idx = xf + w * yf;
          if (!tested(xf, yf, w, h)) continue;
          const float th1 = fm(th_at(I, xf, yf), dw1);
          const float ag1 = __ldg(I.ag1 + (xf >> 1) + (yf >> 1) * w1);   // (int)(xf*0.5f+0.25f), exact
          if (!(ag1 > fm(th1, thF))) continue;
          offer(bb, S.dir_dist ? score(__ldg(I.dI + 3 * (size_t)idx + 1), __ldg(I.dI + 3 * (size_t)idx + 2), d) : ag1,
                ((long long)k << 40) | q, idx);
        }
      }
      bb = warp_best(bb);
      if (bb.idx >= 0) {
        any23 = 1;
        if (lane == 0) { I.map[bb.idx] = 2.f; ++c3; }
      }
    }
    // type 4: without a type-1 or type-2 selection, the first maximum of the block in visiting order
    if (!any23) {
      const int d = __shfl_sync(0xffffffffu, dirs, 0);
      Best bb{0.f, 0, -1};
      for (int k = 0; k < 16; ++k) {
        const int cgx = __shfl_sync(0xffffffffu, gx, k), cgy = __shfl_sync(0xffffffffu, gy, k);
        if (cgx >= cw || cgy >= ch) continue;
        const int cx = cgx * pot, cy = cgy * pot, mx = std::min(pot, w - cx), npx = mx * std::min(pot, h - cy);
        for (int q = lane; q < npx; q += 32) {
          const int xf = cx + q % mx, yf = cy + q / mx, idx = xf + w * yf;
          if (!tested(xf, yf, w, h)) continue;
          const float th2 = fm(fm(th_at(I, xf, yf), dw1), dw2);
          const float ag2 = __ldg(I.ag2 + (xf >> 2) + (yf >> 2) * w2);   // (int)(xf*0.25f+0.125), exact
          if (!(ag2 > fm(th2, thF))) continue;
          offer(bb, S.dir_dist ? score(__ldg(I.dI + 3 * (size_t)idx + 1), __ldg(I.dI + 3 * (size_t)idx + 2), d) : ag2,
                ((long long)k << 40) | q, idx);
        }
      }
      bb = warp_best(bb);
      if (bb.idx >= 0 && lane == 0) { I.map[bb.idx] = 4.f; ++c4; }
    }
  }
  if (c3) atomicAdd(&st->n[1], c3);
  if (c4) atomicAdd(&st->n[2], c4);
}

// (int)x as x86-64's cvttss2si computes it, the reference's build: INT_MIN where the value has no int (NaN, out of range)
__device__ __forceinline__ int to_int(float x) { return (x >= -2147483648.f && x < 2147483648.f) ? (int)x : INT_MIN; }

// makeMaps' decision after a select (:190-257)
__global__ void k_decide(SelState* __restrict__ st, float numWant) {
  if (!st->active) return;
  const int pot = st->pot;
  const float numHave = (float)(st->n[0] + st->n[1] + st->n[2]);
  const float quotia = fd(numWant, numHave);
  const float K = fm(fm(numHave, (float)(pot + 1)), (float)(pot + 1));
  int ideal = to_int(fs(__fsqrt_rn(fd(K, numWant)), 1.f));
  if (ideal < 1) ideal = 1;
  if (st->rec_left > 0 && quotia > 1.25f && pot > 1) {
    if (ideal >= pot) ideal = pot - 1;
    st->pot = ideal; st->rec_left--; st->reselected = 1;
    return;
  }
  if (st->rec_left > 0 && quotia < 0.25f) {
    if (ideal <= pot) ideal = pot + 1;
    st->pot = ideal; st->rec_left--; st->reselected = 1;
    return;
  }
  st->active = 0;
  st->pot_used = pot;
  st->num_have = (int)numHave;
  st->subsample = (double)quotia < 0.95;
  st->charTH = st->subsample ? (int)(unsigned char)fm(255.f, quotia) : 255;
  st->pot_after = ideal;
}

// selections per row
__global__ void k_rowcount(const float* __restrict__ map, int w, int h, int* __restrict__ cnt) {
  const int y = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (y >= h) return;
  int c = 0;
  for (int x0 = 0; x0 < w; x0 += 32) {
    const int x = x0 + lane;
    c += __popc(__ballot_sync(0xffffffffu, x < w && map[x + (size_t)y * w] != 0.f));
  }
  if (lane == 0) cnt[y] = c;
}

// exclusive scan of n ints in one block; *total (may be null) receives the sum
__global__ void __launch_bounds__(1024) k_scan(const int* __restrict__ in, int* __restrict__ out, int n, int* __restrict__ total) {
  using Scan = cub::BlockScan<int, 1024>;
  __shared__ typename Scan::TempStorage tmp;
  int base = 0;
  for (int c0 = 0; c0 < n; c0 += 1024) {
    const int i = c0 + threadIdx.x;
    int v = i < n ? in[i] : 0, pos, tot;
    Scan(tmp).ExclusiveSum(v, pos, tot);
    if (i < n) out[i] = base + pos;
    base += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0 && total) *total = base;
}

// makeMaps' subsample (:231-249): the k-th selection in raster order is dropped when randomPattern[k] > charTH.  keep[y]
// receives the number of row y's kept selections makeNewTraces constructs (x in [3, w-4), y in [3, h-4)).
__global__ void k_subsample(SelState* __restrict__ st, float* __restrict__ map, const unsigned char* __restrict__ rp, int w, int h,
                            const int* __restrict__ rowbase, int* __restrict__ keep) {
  const int y = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (y >= h) return;
  const bool sub = st->subsample;
  const int charTH = st->charTH;
  const bool row_in = y >= 3 && y < h - 4;
  int rank = rowbase[y], kept = 0, dropped = 0;
  for (int x0 = 0; x0 < w; x0 += 32) {
    const int x = x0 + lane;
    const bool s = x < w && map[x + (size_t)y * w] != 0.f;
    const unsigned b = __ballot_sync(0xffffffffu, s);
    bool k = s;
    if (s && sub && __ldg(rp + rank + __popc(b & ((1u << lane) - 1u))) > charTH) {
      map[x + (size_t)y * w] = 0.f;
      k = false;
      ++dropped;
    }
    kept += __popc(__ballot_sync(0xffffffffu, k && row_in && x >= 3 && x < w - 4));
    rank += __popc(b);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) dropped += __shfl_xor_sync(0xffffffffu, dropped, o);
  if (lane == 0) {
    keep[y] = kept;
    if (dropped) atomicAdd(&st->dropped, dropped);
  }
}

// makeNewTraces' candidates in raster order: u at cand[k], v at cand[stride + k], the type's bits at cand[2 stride + k]
__global__ void k_emit(const float* __restrict__ map, int w, int h, const int* __restrict__ keepbase, int* __restrict__ cand, int stride) {
  const int y = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (y < 3 || y >= h - 4) return;
  int pos = keepbase[y];
  for (int x0 = 0; x0 < w; x0 += 32) {
    const int x = x0 + lane;
    const float t = x < w ? map[x + (size_t)y * w] : 0.f;
    const bool k = t != 0.f && x >= 3 && x < w - 4;
    const unsigned b = __ballot_sync(0xffffffffu, k);
    if (k) {
      const int p = pos + __popc(b & ((1u << lane) - 1u));
      cand[p] = x; cand[stride + p] = y; cand[2 * stride + p] = __float_as_int(t);
    }
    pos += __popc(b);
  }
}

// glibc's rand() after srand(seed) (random_r.c, TYPE_3: degree 31, separation 3, 310 discarded calls), restated so the library
// never touches the process's rand state: r_0 = seed, r_i = 16807 r_(i-1) mod (2^31 - 1) for i < 31, r_31..33 = r_0..2,
// r_i = r_(i-31) + r_(i-3) mod 2^32 from i = 34; call k returns r_(344+k) >> 1.
void glibc_rand_bytes(unsigned seed, size_t n, unsigned char* out) {
  uint32_t ring[34];
  int32_t word = (int32_t)seed;
  ring[0] = (uint32_t)word;
  for (int i = 1; i < 31; ++i) {
    const int32_t hi = word / 127773, lo = word % 127773;   // Schrage's method, as srandom_r computes it
    word = 16807 * lo - 2836 * hi;
    if (word < 0) word += 2147483647;
    ring[i] = (uint32_t)word;
  }
  for (int i = 31; i < 34; ++i) ring[i] = ring[i - 31];
  for (size_t i = 34; i < 344 + n; ++i) {
    const uint32_t v = ring[(i - 31) % 34] + ring[(i - 3) % 34];
    ring[i % 34] = v;
    if (i >= 344) out[i - 344] = (unsigned char)((v >> 1) & 0xFF);
  }
}

constexpr int kMaxRecursions = 16;

class SelectorImpl final : public SelectorIface {
 public:
  SelectorImpl(int w, int h, const float* settings, int device) : w_(w), h_(h), device_(device) {
    int nd = 0;
    if (cudaGetDeviceCount(&nd) != cudaSuccess || nd == 0)
      throw Error("tandem_b200: no CUDA device visible - this library has no CPU fallback");
    TDM_CHECK(w / 32 >= 1 && h / 32 >= 1, "pixel selector: w / 32 and h / 32 must be at least 1");
    TDM_CHECK(settings, "null argument");
    std::memcpy(&s_, settings, sizeof s_);
    TDM_CHECK(std::isfinite(s_.cut) && s_.cut >= 0.f && s_.cut <= 0.99f && std::isfinite(s_.add) && std::isfinite(s_.dw1) &&
                  (s_.dir_dist == 0 || s_.dir_dist == 1),
              "bad selection settings");
    TDM_CUDA(cudaSetDevice(device_));
    const size_t n = (size_t)w * h, nb4 = (size_t)cdiv(w, 4) * cdiv(h, 4), cells32 = (size_t)(w / 32) * (h / 32);
    stream_ = make_stream(0);
    done_ = make_event(cudaEventDisableTiming);
    d_rp_ = make_dev<unsigned char>(n);
    d_ths_raw_ = make_dev<float>(4 * cells32);
    d_ths_ = make_dev<float>(4 * cells32);
    d_mask_ = make_dev<uint16_t>(2 * n);
    d_n2b4_ = make_dev<int>(4 * nb4);
    d_map_ = make_dev<float>(4 * n);
    d_rows_ = make_dev<int>(4ull * 4 * h);
    d_cand_ = make_dev<int>(12 * n);
    d_st_ = make_dev<SelState>(sizeof(SelState));
    h_st_ = make_host<SelState>(sizeof(SelState));
    h_rp_ = make_host<unsigned char>(n);
    glibc_rand_bytes(3141592u, n, h_rp_.get());   // PixelSelector::PixelSelector: std::srand(3141592)
    TDM_CUDA(cudaMemcpyAsync(d_rp_.get(), h_rp_.get(), n, cudaMemcpyHostToDevice, stream_.get()));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
  }
  ~SelectorImpl() override {
    cudaSetDevice(device_);
    cudaStreamSynchronize(stream_.get());
  }

  int potential() const override { return potential_; }
  void set_potential(int p) override {
    TDM_CHECK(p >= 1, "the potential must be at least 1");
    potential_ = p;
  }
  int width() const override { return w_; }
  int height() const override { return h_; }
  int device() const override { return device_; }

  void check(const PyramidIface& p, float density, int recursions_left, float th_factor) const override {
    TDM_CHECK(p.levels() >= 3, "pixel selection needs a pyramid of at least 3 levels");
    TDM_CHECK(p.width(0) == w_ && p.height(0) == h_, "pyramid level 0 is not the selector's image size");
    TDM_CHECK(p.device() == device_, "pyramid and pixel selector live on different devices");
    TDM_CHECK(std::isfinite(density) && density >= 0.f, "density must be finite and not negative");
    TDM_CHECK(recursions_left >= 0 && recursions_left <= kMaxRecursions, "recursions_left outside 0..16");
    TDM_CHECK(std::isfinite(th_factor) && th_factor > 0.f, "th_factor must be finite and positive");
  }

  void enqueue(void* stream, const PyramidIface& p, float density, int recursions_left, float th_factor, bool emit) override {
    cudaStream_t s = (cudaStream_t)stream;
    const int w32 = w_ / 32, h32 = h_ / 32;
    SelState init{};
    init.pot = potential_; init.rec_left = recursions_left; init.active = 1;
    *h_st_ = init;
    TDM_CUDA(cudaMemcpyAsync(d_st_.get(), h_st_.get(), sizeof(SelState), cudaMemcpyHostToDevice, s));
    TDM_CUDA(cudaStreamWaitEvent(s, (cudaEvent_t)p.ready_event(), 0));
    const Img I{p.level_dI(0), p.level_abs(0), p.level_abs(1), p.level_abs(2), d_ths_.get(), d_rp_.get(), d_map_.get(), w_, h_};
    k_hist<<<w32 * h32, kThreads, 0, s>>>(I.ag0, w_, h_, s_, d_ths_raw_.get());
    k_smooth<<<cdiv(w32 * h32, 128), 128, 0, s>>>(d_ths_raw_.get(), w32, h32, d_ths_.get());
    for (int r = 0; r <= recursions_left; ++r) {
      k_mask<<<kGrid, kThreads, 0, s>>>(d_st_.get(), I, s_, th_factor, d_mask_.get());
      k_chain<<<1, kThreads, 0, s>>>(d_st_.get(), d_mask_.get(), d_rp_.get(), w_, h_, d_n2b4_.get());
      k_pick<<<kGrid, kPickThreads, 0, s>>>(d_st_.get(), I, s_, th_factor, d_mask_.get(), d_n2b4_.get());
      k_decide<<<1, 1, 0, s>>>(d_st_.get(), density);
    }
    int* cnt = d_rows_.get();
    int* base = cnt + h_;
    int* keep = base + h_;
    int* keepbase = keep + h_;
    const int rb = cdiv(h_, kThreads / 32);
    k_rowcount<<<rb, kThreads, 0, s>>>(d_map_.get(), w_, h_, cnt);
    k_scan<<<1, 1024, 0, s>>>(cnt, base, h_, nullptr);
    k_subsample<<<rb, kThreads, 0, s>>>(d_st_.get(), d_map_.get(), d_rp_.get(), w_, h_, base, keep);
    if (emit) {
      k_scan<<<1, 1024, 0, s>>>(keep, keepbase, h_, &d_st_.get()->n_cand);
      k_emit<<<rb, kThreads, 0, s>>>(d_map_.get(), w_, h_, keepbase, d_cand_.get(), w_ * h_);
    }
    TDM_CUDA(cudaGetLastError());
    TDM_CUDA(cudaMemcpyAsync(h_st_.get(), d_st_.get(), sizeof(SelState), cudaMemcpyDeviceToHost, s));
  }
  Candidates candidates() const override { return Candidates{d_cand_.get(), w_ * h_, &d_st_.get()->n_cand}; }

  void result(SelectResult* r, bool commit) override {
    const SelState& st = *h_st_;
    r->num_selected = st.num_have - st.dropped;
    r->n2 = st.n[0]; r->n3 = st.n[1]; r->n4 = st.n[2];
    r->potential_used = st.pot_used;
    r->potential_after = st.pot_after;
    r->reselected = st.reselected;
    r->nonuniform_cells = st.nonuniform;
    if (commit) potential_ = st.pot_after;
  }

  void make_maps(const PyramidIface& p, float density, int recursions_left, float th_factor, float* map_out,
                 SelectResult* r) override {
    check(p, density, recursions_left, th_factor);
    TDM_CUDA(cudaSetDevice(device_));
    enqueue(stream_.get(), p, density, recursions_left, th_factor, false);
    if (map_out)
      TDM_CUDA(cudaMemcpyAsync(map_out, d_map_.get(), 4ull * w_ * h_, cudaMemcpyDeviceToHost, stream_.get()));
    // a later build or destroy of the pyramid waits for the selection
    TDM_CUDA(cudaEventRecord(done_.get(), stream_.get()));
    p.wait_for(done_.get());
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    SelectResult tmp;
    result(r ? r : &tmp, true);
  }

 private:
  int w_, h_, device_;
  SelSettings s_;
  int potential_ = 3;   // PixelSelector::currentPotential
  Stream stream_;
  Event done_;
  DevPtr<unsigned char> d_rp_;
  HostPtr<unsigned char> h_rp_;
  DevPtr<float> d_ths_raw_, d_ths_, d_map_;
  DevPtr<uint16_t> d_mask_;
  DevPtr<int> d_n2b4_, d_rows_, d_cand_;
  DevPtr<SelState> d_st_;
  HostPtr<SelState> h_st_;
};

}  // namespace

static_assert(sizeof(SelSettings) == 4 * 4, "tdm_select_settings layout");
static_assert(sizeof(SelectResult) == 8 * 4, "tdm_select_result layout");

SelectorIface* make_selector(int w, int h, const float* settings, int device) { return new SelectorImpl(w, h, settings, device); }

}  // namespace tdm
