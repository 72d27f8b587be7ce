// Voxel-hashed TSDF fusion behind the DrFusion call surface (dr_fusion.h:44-73).
//
// Reference being replaced (SURVEY.md §2.2, §8 a11-a13, Appendix A.2):
//   AllocateFromDepthKernel  tandem/libdr/dr_fusion/src/tsdfvh/tsdf_volume.cu:317-434 (+ hash_table.cu:80-115)
//   IntegrateScanKernel      tsdf_volume.cu:436-513 (+ :303-315, voxel.h:29-53)
//   GenerateRgbDepthKernel   tsdf_volume.cu:600-632 (+ GetInterpolatedVoxel :161-289)
// Design (not a port):
//   K5 allocate : one thread per depth PIXEL (the reference sizes its grid by the 10 M hash entries), lock-free
//                 insert with a single 64-bit CAS on the packed block key (no lock state, no duplicate blocks),
//                 every new block appended to a compact block list.
//   K6 integrate: a visibility pass compacts the blocks in view, persistent CTAs stride over that list (the reference
//                 scans all 10 M entries, free ones included), 256 threads x 2 voxels, one 128-bit load + store per
//                 thread, no per-voxel re-hash.
//   K7 ray-cast : one thread per pixel in 8x8 tiles, sphere tracing clipped to the bounding box of everything ever
//                 allocated; per-axis index arithmetic shared by the nine voxel reads of a sample, ONE hash probe per
//                 distinct voxel block of a sample (one-entry pointer cache in front), division-free bucket index,
//                 colour blend only for the final hit.  Every sample sits where the reference's march puts it.
//                 k_raycast (option "raycast_shared" = 0) is the comparator: the reference's sampler voxel by voxel, one
//                 hash probe per voxel read; the production kernel must render the same volume bit for bit.
// The hash function, bucket structure (full bucket -> block dropped), voxel record (8 B) and all geometry are
// the reference's; geometry that decides integers uses __f*_rn intrinsics so it is bit-identical to the CPU
// oracle (oracle/tsdf_oracle.c) which evaluates the same expressions without FMA contraction.
#include <unistd.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

#include "fusion.h"
#include "mat4.h"

namespace tdm {

namespace {

constexpr unsigned long long kEmptyKey = ~0ull;
constexpr int kKeyBias = 1 << 20;

struct Mat4 { float m[16]; };

struct FusionDev {
  tdm_fusion_options o;
  unsigned long long* keys;  // [num_buckets*bucket_size], kEmptyKey = free
  int* ptrs;                 // block index per entry
  uint2* voxels;             // [num_blocks*512] {sdf bits, c0|c1<<8|c2<<16|w<<24}
  int4* list;                // compact list of allocated blocks (x,y,z,ptr)
  int* bbox;                 // [6] block-coordinate bounding box (min xyz, max xyz) of EVERY block any scan's rays walked through -
                             // also other ranks' blocks: each rank walks all rays, so the box is replicated knowledge
  int* counters;             // [0] #blocks allocated, [1] dropped, [2] visible (last scan), [3] new this scan
  int slab_lo, slab_hi;      // Z-slab partition (block z in [slab_lo, slab_hi) is kept; SURVEY.md 8e), default: everything
  float r_vs, r_fx, r_fy;    // RN(1 / voxel_size), RN(1 / fx), RN(1 / fy) for cdiv_ (ray-cast only)
  float half_vs;             // RN(voxel_size / 2.0f): the sampler's half-voxel shift (tsdf_volume.cu:166), a per-volume constant
  unsigned long long mod_magic;   // ceil(2^64 / num_buckets): exact 32-bit remainder without a division (fast_umod)
  unsigned mod_c32;               // 2^32 mod num_buckets
  // Interleaved Z-slab partition (il_k > 0): block z belongs to rank ((z - il_z0) div il_k) mod il_world; a rank STORES its own
  // blocks plus one halo block on either side of each of its slabs.  Thin interleaved slabs keep the per-frame work of every
  // rank proportional to 1 / world for ANY view direction (contiguous slabs only balance memory: a camera looking along a slab
  // leaves the other ranks idle), at the price of (il_k + 2) / il_k redundant integration.
  int il_k, il_world, il_rank, il_z0;
  // Peer view of a Z-slab-partitioned volume (pixel-partitioned ray-cast, SURVEY.md 8e): the hash tables and voxel pools of ALL
  // ranks, mapped into this device's address space (CUDA IPC over NVLink P2P, or plain pointers for instances of one process).
  // Block row z is read from the rank that OWNS it: pr_lo[r] <= z < pr_hi[r].  pr_world == 0: not attached.
  const unsigned long long* pr_keys[8];
  const int* pr_ptrs[8];
  const uint2* pr_voxels[8];
  int pr_lo[8], pr_hi[8];
  int pr_world, pr_rank;
};

__device__ __forceinline__ int il_owner(const FusionDev& d, int bz) {
  int g = bz - d.il_z0;
  g = g >= 0 ? g / d.il_k : -((-g + d.il_k - 1) / d.il_k);   // floor division
  int o = g % d.il_world;
  return o < 0 ? o + d.il_world : o;
}
__device__ __forceinline__ bool slab_stores(const FusionDev& d, int bz) {   // does this rank keep block row bz (own or halo)?
  if (d.il_k > 0) return il_owner(d, bz) == d.il_rank || il_owner(d, bz - 1) == d.il_rank || il_owner(d, bz + 1) == d.il_rank;
  return bz >= d.slab_lo && bz < d.slab_hi;
}

__device__ __forceinline__ float mul_(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add_(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub_(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float div_(float a, float b) { return __fdiv_rn(a, b); }

// Correctly rounded x / d for a divisor that is constant over the kernel, from its correctly rounded reciprocal r = RN(1/d):
//   q0 = RN(x r);  e = x - q0 d (exact, one FMA);  q = RN(q0 + e r)
// is RN(x / d) whenever no intermediate under- / overflows and d's significand is not all ones (Markstein's theorem for
// FMA division; tests/test_abi.py::test_constant_division_is_correctly_rounded checks it exhaustively for d = 0.01f and on 1e8
// random pairs).  Outside the safe range, and for the excluded divisors (FAST is then false on the host), the IEEE division
// is used.  3 instructions instead of the ~25 of div.rn.f32's software expansion; the ray-cast does 11 such divisions per
// sample (by voxel_size, fx, fy), a third of its instruction count.  Results are bit-identical to div_ by construction.
template <bool FAST>
__device__ __forceinline__ float cdiv_(float x, float d, float r) {
  if constexpr (!FAST) return __fdiv_rn(x, d);
  const float ax = fabsf(x);
  if (!(ax > 1e-18f && ax < 1e18f)) return __fdiv_rn(x, d);   // zeros, denormal-range and huge values, NaN
  const float q0 = __fmul_rn(x, r);
  const float e = __fmaf_rn(-q0, d, x);
  return __fmaf_rn(e, r, q0);
}

__device__ __forceinline__ float3 xform(const Mat4& T, float3 v) {  // matrix_utils.h:914-921 (w == 1)
  const float* m = T.m;
  float3 r;
  r.x = add_(add_(add_(mul_(m[0], v.x), mul_(m[1], v.y)), mul_(m[2], v.z)), mul_(m[3], 1.0f));
  r.y = add_(add_(add_(mul_(m[4], v.x), mul_(m[5], v.y)), mul_(m[6], v.z)), mul_(m[7], 1.0f));
  r.z = add_(add_(add_(mul_(m[8], v.x), mul_(m[9], v.y)), mul_(m[10], v.z)), mul_(m[11], 1.0f));
  return r;
}
__device__ __forceinline__ float norm3(float3 v) {
  return __fsqrt_rn(add_(add_(mul_(v.x, v.x), mul_(v.y, v.y)), mul_(v.z, v.z)));
}
__device__ __forceinline__ float3 get_point3d(const tdm_fusion_options& o, int i, float depth) {  // utils.h:93-101
  const int v = i / o.width, u = i - o.width * v;
  float3 p;
  p.z = depth;
  p.x = div_(mul_(sub_((float)u, o.cx), p.z), o.fx);
  p.y = div_(mul_(sub_((float)v, o.cy), p.z), o.fy);
  return p;
}
// the same with the pixel terms (u - cx), (v - cy) - loop invariants of a ray - computed once by the caller (same operations)
template <bool FAST>
__device__ __forceinline__ float3 get_point3d_px(const FusionDev& d, float ucx /* sub_(u, cx) */, float vcy /* sub_(v, cy) */, float depth) {
  float3 p;
  p.z = depth;
  p.x = cdiv_<FAST>(mul_(ucx, p.z), d.o.fx, d.r_fx);
  p.y = cdiv_<FAST>(mul_(vcy, p.z), d.o.fy, d.r_fy);
  return p;
}
__device__ __forceinline__ int2 project(const tdm_fusion_options& o, float3 p) {  // utils.h:103-108
  const float x = add_(div_(mul_(o.fx, p.x), p.z), o.cx);
  const float y = add_(div_(mul_(o.fy, p.y), p.z), o.cy);
  return make_int2(__float2int_rz(roundf(x)), __float2int_rz(roundf(y)));
}
__device__ __forceinline__ int sgn(float n) { return (n > 0) - (n < 0); }

__device__ __forceinline__ unsigned long long pack_key(int x, int y, int z) {
  return (unsigned long long)(unsigned)(x + kKeyBias) | ((unsigned long long)(unsigned)(y + kKeyBias) << 21) |
         ((unsigned long long)(unsigned)(z + kKeyBias) << 42);
}
// u mod n for any 32-bit u and n from the precomputed M = ceil(2^64 / n) (Lemire, Kaser, Kurz, "Faster remainder by direct
// computation", 2019: exact whenever M has at least 64 fractional bits for 32-bit operands): fraction = M * u mod 2^64,
// remainder = floor(fraction * n / 2^64).  ~8 integer instructions instead of the ~25 of the runtime `%` expansion.
__host__ __device__ __forceinline__ unsigned fast_umod(unsigned u, unsigned n, unsigned long long M) {
  const unsigned long long frac = M * (unsigned long long)u;
#ifdef __CUDA_ARCH__
  return (unsigned)__umul64hi(frac, (unsigned long long)n);
#else
  return (unsigned)(((unsigned __int128)frac * n) >> 64);
#endif
}
// hash_table.cu:157-168: ((x * 73856093) ^ (y * 19349669) ^ (z * 83492791)) % num_buckets on ints, + num_buckets if negative -
// i.e. the mathematical (floor) modulus of the SIGNED 32-bit hash h.  With u = (unsigned)h: h = u - 2^32 [h < 0], so
// h mod n = (u mod n - [h < 0] * (2^32 mod n)) mod n.  tests/test_abi.py pins it against Python's % on ints.
__host__ __device__ __forceinline__ int hash_slot(int x, int y, int z, int num_buckets, unsigned long long magic, unsigned c32) {
  const int h = (int)((unsigned)x * 73856093u) ^ (int)((unsigned)y * 19349669u) ^ (int)((unsigned)z * 83492791u);
  int r = (int)fast_umod((unsigned)h, (unsigned)num_buckets, magic);
  if (h < 0) { r -= (int)c32; if (r < 0) r += num_buckets; }
  return r;
}
__device__ __forceinline__ long long hash_bucket(const FusionDev& d, int x, int y, int z) {
  return (long long)hash_slot(x, y, z, d.o.num_buckets, d.mod_magic, d.mod_c32) * d.o.bucket_size;
}

__device__ void insert_block(const FusionDev& d, int x, int y, int z) {
  if (x <= -kKeyBias || x >= kKeyBias || y <= -kKeyBias || y >= kKeyBias || z <= -kKeyBias || z >= kKeyBias) return;
  if (!slab_stores(d, z)) return;   // another rank's Z-slab
  const unsigned long long key = pack_key(x, y, z);
  const long long b = hash_bucket(d, x, y, z);
  for (int i = 0; i < d.o.bucket_size; ++i) {
    unsigned long long cur = d.keys[b + i];
    if (cur == key) return;
    if (cur == kEmptyKey) {
      cur = atomicCAS(&d.keys[b + i], kEmptyKey, key);
      if (cur == key) return;           // somebody else inserted the same block
      if (cur == kEmptyKey) {           // we own the slot: take a voxel block and publish it in the list
        const int ptr = atomicAdd(&d.counters[0], 1);
        if (ptr >= d.o.num_blocks) {    // heap exhausted (heap.cu:16-18 aborts; we drop and count)
          atomicAdd(&d.counters[1], 1);
          d.ptrs[b + i] = -1;
          return;
        }
        d.ptrs[b + i] = ptr;
        d.list[ptr] = make_int4(x, y, z, ptr);
        atomicAdd(&d.counters[3], 1);
        return;
      }
      // slot taken by a different block in the meantime: keep scanning
    }
  }
  atomicAdd(&d.counters[1], 1);  // bucket full: block dropped (hash_table.cu:103-115 returns without allocating)
}

__device__ __forceinline__ int find_in(const unsigned long long* __restrict__ keys, const int* __restrict__ ptrs, const FusionDev& d,
                                       int x, int y, int z) {  // hash_table.cu:141-155
  if (x <= -kKeyBias || x >= kKeyBias || y <= -kKeyBias || y >= kKeyBias || z <= -kKeyBias || z >= kKeyBias) return -1;
  const unsigned long long key = pack_key(x, y, z);
  const long long b = hash_bucket(d, x, y, z);
  for (int i = 0; i < d.o.bucket_size; ++i) {
    const unsigned long long k = keys[b + i];
    if (k == key) return ptrs[b + i];
    if (k == kEmptyKey) return -1;   // inserts fill a bucket front to back and nothing is ever removed: a free slot ends the search
  }
  return -1;
}
__device__ __forceinline__ int find_block(const FusionDev& d, int x, int y, int z) { return find_in(d.keys, d.ptrs, d, x, y, z); }

// ---------------------------------------------------------------------------------------------- K5
__global__ void __launch_bounds__(128) k_allocate(FusionDev d, const float* __restrict__ depth, Mat4 T) {
  const tdm_fusion_options& o = d.o;
  const int n = o.height * o.width;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float dz = depth[i];
  if (dz < o.min_sensor_depth || dz > o.max_sensor_depth) return;
  const float bs = mul_((float)o.block_size, o.voxel_size);
  const float3 start = make_float3(T.m[3], T.m[7], T.m[11]);
  const float3 p = xform(T, get_point3d(o, i, dz));
  if (p.x == 0 && p.y == 0 && p.z == 0) return;
  const float3 dd = make_float3(sub_(p.x, start.x), sub_(p.y, start.y), sub_(p.z, start.z));
  const float dn = norm3(dd);
  const float3 dir = make_float3(div_(dd.x, dn), div_(dd.y, dn), div_(dd.z, dn));
  const float len = add_(dn, o.truncation_distance);
  const float3 end = make_float3(add_(start.x, mul_(dir.x, len)), add_(start.y, mul_(dir.y, len)), add_(start.z, mul_(dir.z, len)));
  int3 bp = make_int3((int)floorf(div_(start.x, bs)), (int)floorf(div_(start.y, bs)), (int)floorf(div_(start.z, bs)));
  const int3 be = make_int3((int)floorf(div_(end.x, bs)), (int)floorf(div_(end.y, bs)), (int)floorf(div_(end.z, bs)));
  const int3 step = make_int3(sgn(dir.x), sgn(dir.y), sgn(dir.z));
  const float3 dt = make_float3(dir.x != 0 ? fabsf(div_(bs, dir.x)) : FLT_MAX, dir.y != 0 ? fabsf(div_(bs, dir.y)) : FLT_MAX,
                                dir.z != 0 ? fabsf(div_(bs, dir.z)) : FLT_MAX);
  const float3 bd = make_float3(mul_(add_((float)bp.x, (float)step.x), bs), mul_(add_((float)bp.y, (float)step.y), bs),
                                mul_(add_((float)bp.z, (float)step.z), bs));
  float3 mt = make_float3(dir.x != 0 ? div_(sub_(bd.x, start.x), dir.x) : FLT_MAX,
                          dir.y != 0 ? div_(sub_(bd.y, start.y), dir.y) : FLT_MAX,
                          dir.z != 0 ? div_(sub_(bd.z, start.z), dir.z) : FLT_MAX);
  int3 diff = make_int3(0, 0, 0);
  bool neg = false;
  if (bp.x != be.x && dir.x < 0) { diff.x--; neg = true; }
  if (bp.y != be.y && dir.y < 0) { diff.y--; neg = true; }
  if (bp.z != be.z && dir.z < 0) { diff.z--; neg = true; }
  {
    // Replicated bounding box of everything the scans' rays touch (own and foreign blocks alike): the DDA is monotone per axis,
    // so the ray's blocks lie in the box spanned by its first and last block (+-1 for the `neg` pre-step).  Plain read first:
    // after the first few rays of a scan almost no atomic is issued.
    const int lo[3] = {min(bp.x, be.x) - 1, min(bp.y, be.y) - 1, min(bp.z, be.z) - 1};
    const int hi[3] = {max(bp.x, be.x) + 1, max(bp.y, be.y) + 1, max(bp.z, be.z) + 1};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (lo[a] < d.bbox[a]) atomicMin(&d.bbox[a], lo[a]);
      if (hi[a] > d.bbox[3 + a]) atomicMax(&d.bbox[3 + a], hi[a]);
    }
  }
  insert_block(d, bp.x, bp.y, bp.z);
  if (neg) { bp.x += diff.x; bp.y += diff.y; bp.z += diff.z; insert_block(d, bp.x, bp.y, bp.z); }
  int guard = 0;
  while ((bp.x != be.x || bp.y != be.y || bp.z != be.z) && guard++ < 100000) {
    if (mt.x < mt.y) {
      if (mt.x < mt.z) { bp.x += step.x; mt.x = add_(mt.x, dt.x); } else { bp.z += step.z; mt.z = add_(mt.z, dt.z); }
    } else {
      if (mt.y < mt.z) { bp.y += step.y; mt.y = add_(mt.y, dt.y); } else { bp.z += step.z; mt.z = add_(mt.z, dt.z); }
    }
    insert_block(d, bp.x, bp.y, bp.z);
  }
}

// ---------------------------------------------------------------------------------------------- K6
__device__ __forceinline__ uint2 combine(uint2 v, float nsdf, const unsigned char* col, int max_w) {  // voxel.h:29-53
  const float w = (float)(v.y >> 24);
  const float wn = add_(w, 1.0f);
  unsigned out = 0;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float cur = (float)((v.y >> (8 * c)) & 0xFF);
    const float m = div_(add_(mul_(cur, w), mul_((float)col[c], 1.0f)), wn);
    out |= ((unsigned)m & 0xFF) << (8 * c);
  }
  const float sdf = div_(add_(mul_(__uint_as_float(v.x), w), mul_(nsdf, 1.0f)), wn);
  int nw = (int)(v.y >> 24) + 1;
  if (nw > max_w) nw = max_w;
  return make_uint2(__float_as_uint(sdf), out | ((unsigned)nw << 24));
}

// Only ~10 % of the allocated blocks are in view of a scan, and the map grows with every keyframe, so the visibility test runs
// once per block in its own kernel (thread per block, warp-aggregated append to a compact list) and the voxel update visits
// the visible blocks only.
__global__ void __launch_bounds__(256) k_visible(FusionDev d, Mat4 Ti, int* __restrict__ vis_list) {
  const tdm_fusion_options& o = d.o;
  const int nblocks = min(d.counters[0], o.num_blocks);
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  bool vis = false;
  if (b < nblocks) {
    const int4 e = d.list[b];
    const float vs = o.voxel_size;
    const float3 pos = make_float3(mul_(mul_((float)e.x, vs), 8.0f), mul_(mul_((float)e.y, vs), 8.0f), mul_(mul_((float)e.z, vs), 8.0f));
    const float3 pc = xform(Ti, pos);
    if (!(pc.z < 0)) {
      const double half = 0.5 * (double)vs * 8.0;  // double as written in the reference (tsdf_volume.cu:460-463)
      const float3 ctr = make_float3((float)((double)pc.x + half), (float)((double)pc.y + half), (float)((double)pc.z + half));
      const int2 px = project(o, ctr);
      vis = px.x >= 0 && px.y >= 0 && px.x < o.width && px.y < o.height;
    }
  }
  const unsigned m = __ballot_sync(0xffffffffu, vis);
  if (m) {
    const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
    int base = 0;
    if (lane == leader) base = atomicAdd(&d.counters[2], __popc(m));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (vis) vis_list[base + __popc(m & ((1u << lane) - 1u))] = b;
  }
}

__global__ void __launch_bounds__(256)
k_integrate_list(FusionDev d, const unsigned char* __restrict__ bgr, const float* __restrict__ depth, Mat4 Ti, const int* __restrict__ vis_list) {
  const tdm_fusion_options& o = d.o;
  const int nvis = d.counters[2];
  const float vs = o.voxel_size, tau = o.truncation_distance;
  for (int k = blockIdx.x; k < nvis; k += gridDim.x) {
    const int4 e = d.list[vis_list[k]];
    const float3 pos = make_float3(mul_(mul_((float)e.x, vs), 8.0f), mul_(mul_((float)e.y, vs), 8.0f), mul_(mul_((float)e.z, vs), 8.0f));
    const int t = threadIdx.x;
    const int bx = t >> 5, by = (t >> 2) & 7, bz0 = (t & 3) * 2;
    uint4* vp = reinterpret_cast<uint4*>(d.voxels + (size_t)e.w * 512 + bx * 64 + by * 8 + bz0);
    uint4 raw = *vp;
    uint2 vox[2] = {make_uint2(raw.x, raw.y), make_uint2(raw.z, raw.w)};
    bool dirty = false;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const float3 vw = make_float3(add_(pos.x, mul_((float)bx, vs)), add_(pos.y, mul_((float)by, vs)),
                                    add_(pos.z, mul_((float)(bz0 + q), vs)));
      const float3 vc = xform(Ti, vw);
      if (vc.z == 0.0f) continue;
      const int2 px = project(o, vc);
      if (!(px.x >= 0 && px.y >= 0 && px.x < o.width && px.y < o.height)) continue;
      const int idx = px.y * o.width + px.x;
      const float dz = depth[idx];
      if (dz <= 0 || dz < o.min_sensor_depth || dz > o.max_sensor_depth) continue;
      const float sd = norm3(get_point3d(o, idx, dz)), vd = norm3(vc);
      float nsdf;
      if (vd > sub_(sd, tau) && vd < add_(sd, tau) && dz < o.max_sensor_depth) nsdf = sub_(sd, vd);
      else if (vd < sub_(sd, tau)) nsdf = tau;
      else continue;
      vox[q] = combine(vox[q], nsdf, bgr + 3 * (size_t)idx, o.max_sdf_weight);
      dirty = true;
    }
    if (dirty) *vp = make_uint4(vox[0].x, vox[0].y, vox[1].x, vox[1].y);
  }
}

// ---------------------------------------------------------------------------------------------- K7
// Per-ray last-block caches in front of the hash table.
//  Cache1: the block index, for the reference-shaped comparator k_raycast.
struct Cache1 {
  int x, y, z, ptr;
  __device__ __forceinline__ void init() { x = y = z = INT_MIN; ptr = -1; }
  __device__ __forceinline__ int find(const FusionDev& d, int bx, int by, int bz) {
    if (bx != x || by != y || bz != z) { x = bx; y = by; z = bz; ptr = find_block(d, bx, by, bz); }
    return ptr;
  }
};
// Cache1 holding the block's BASE POINTER: a hit costs the three compares only (ncu: re-deriving voxels + ptr * 512 on every
// hit was 4.5 % of the ray-cast's instructions).  Used by the production ray-cast.
struct Cache1P {
  int x, y, z;
  const uint2* base;
  __device__ __forceinline__ void init() { x = y = z = INT_MIN; base = nullptr; }
  __device__ __forceinline__ const uint2* block(const FusionDev& d, int bx, int by, int bz) {
    if (bx != x || by != y || bz != z) {
      x = bx; y = by; z = bz;
      const int p = find_block(d, bx, by, bz);
      base = p < 0 ? nullptr : d.voxels + (size_t)p * 512;
    }
    return base;
  }
  __device__ __forceinline__ bool holds(int bx, int by, int bz) const { return bx == x && by == y && bz == z; }
  __device__ __forceinline__ const uint2* held(const FusionDev&) const { return base; }
};
// Last-block cache over the PEER view: the block is looked up in the table of the rank that owns its z row and its voxels are
// read from that rank's pool - local HBM for this rank's own rows, NVLink P2P loads for the others.
struct CachePeer {
  int x, y, z;
  const uint2* base;
  __device__ __forceinline__ void init() { x = y = z = INT_MIN; base = nullptr; }
  __device__ __forceinline__ const uint2* block(const FusionDev& d, int bx, int by, int bz) {
    if (bx != x || by != y || bz != z) {
      x = bx; y = by; z = bz;
      base = nullptr;
      int r = 0;
      while (r < d.pr_world - 1 && bz >= d.pr_hi[r]) ++r;     // contiguous slabs in rank order
      if (bz >= d.pr_lo[r] && bz < d.pr_hi[r]) {
        const int p = find_in(d.pr_keys[r], d.pr_ptrs[r], d, bx, by, bz);
        if (p >= 0) base = d.pr_voxels[r] + (size_t)p * 512;
      }
    }
    return base;
  }
  __device__ __forceinline__ bool holds(int bx, int by, int bz) const { return bx == x && by == y && bz == z; }
  __device__ __forceinline__ const uint2* held(const FusionDev&) const { return base; }
};
__device__ __forceinline__ uint2 get_voxel(const FusionDev& d, float3 p, Cache1& bc) {  // tsdf_volume.cu:109-159
  const float s = d.o.voxel_size;
  const int gx = (int)add_(div_(p.x, s), mul_((float)sgn(p.x), 0.5f));
  const int gy = (int)add_(div_(p.y, s), mul_((float)sgn(p.y), 0.5f));
  const int gz = (int)add_(div_(p.z, s), mul_((float)sgn(p.z), 0.5f));
  const int ptr = bc.find(d, gx >> 3, gy >> 3, gz >> 3);  // floor division by the block size 8
  if (ptr < 0) return make_uint2(0u, 0u);
  return __ldg(d.voxels + (size_t)ptr * 512 + (gx & 7) * 64 + (gy & 7) * 8 + (gz & 7));
}

__device__ uint2 get_interpolated(const FusionDev& d, float3 p, Cache1& bc) {  // tsdf_volume.cu:161-289
  const uint2 v0 = get_voxel(d, p, bc);
  if ((v0.y >> 24) == 0) return v0;
  const float s = d.o.voxel_size;
  const float hs = div_(s, 2.0f);
  const float3 pd = make_float3(sub_(p.x, hs), sub_(p.y, hs), sub_(p.z, hs));
  const float3 vp = make_float3(div_(p.x, s), div_(p.y, s), div_(p.z, s));
  const float wx = sub_(vp.x, floorf(vp.x)), wy = sub_(vp.y, floorf(vp.y)), wz = sub_(vp.z, floorf(vp.z));
  float dist = 0.f, cf[3] = {0.f, 0.f, 0.f};
  // corner order of the reference: 000,100,010,001,110,011,101,111
  const int ox[8] = {0, 1, 0, 0, 1, 0, 1, 1}, oy[8] = {0, 0, 1, 0, 1, 1, 0, 1}, oz[8] = {0, 0, 0, 1, 0, 1, 1, 1};
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float3 q = make_float3(add_(pd.x, ox[k] ? s : 0.f), add_(pd.y, oy[k] ? s : 0.f), add_(pd.z, oz[k] ? s : 0.f));
    uint2 v = get_voxel(d, q, bc);
    if ((v.y >> 24) == 0) v = v0;
    const float w = mul_(mul_(ox[k] ? wx : sub_(1.f, wx), oy[k] ? wy : sub_(1.f, wy)), oz[k] ? wz : sub_(1.f, wz));
    dist = add_(dist, mul_(w, __uint_as_float(v.x)));
#pragma unroll
    for (int c = 0; c < 3; ++c) cf[c] = add_(cf[c], mul_(w, (float)((v.y >> (8 * c)) & 0xFF)));
  }
  unsigned col = 0;
#pragma unroll
  for (int c = 0; c < 3; ++c) col |= ((unsigned)cf[c] & 0xFF) << (8 * c);
  return make_uint2(__float_as_uint(dist), col | (v0.y & 0xFF000000u));
}

// get_interpolated with the index arithmetic shared between the nine voxel reads (same values, same order of the fp32
// operations that produce the result -> bit-identical).  WorldToGlobalVoxel is separable per axis, so a sample needs three
// divisions per axis (the sample itself, and the two dual-cell corners) instead of three per voxel read; and when the eight
// corners are index-adjacent and sit inside one voxel block (two thirds of all samples) they are read from ONE block lookup at
// constant offsets.  ncu on the one-lookup-per-voxel form: 502 M warp instructions per 640x480 render, 18 % of them FP32.
__device__ __forceinline__ int w2g_axis(float q /* = x / s */, float x) {   // tsdf_volume.cu:109-113, division hoisted
  // sgn(x) * 0.5f is exactly +-0.5f, or +0.f for x == 0 and NaN: two selects instead of two set-compares, a subtraction, an
  // int -> float conversion and a multiplication (ncu: this line and sgn() were 10 % of the ray-cast's instructions)
  const float h = x > 0.f ? 0.5f : (x < 0.f ? -0.5f : 0.f);
  return (int)add_(q, h);
}
template <class Cache>
__device__ __forceinline__ uint2 voxel_at(const FusionDev& d, int gx, int gy, int gz, Cache& bc) {
  const uint2* blk = bc.block(d, gx >> 3, gy >> 3, gz >> 3);
  if (!blk) return make_uint2(0u, 0u);
  return __ldg(blk + (gx & 7) * 64 + (gy & 7) * 8 + (gz & 7));
}
// COLOR = false: the marching steps only consume the interpolated sdf and the centre voxel's weight; the colour blend (8 corners
// x 3 channels of unpack / convert / multiply-add: a fifth of the sample's instructions) is only evaluated for the final hit.
template <class Cache, bool COLOR, bool FAST>
__device__ uint2 get_interpolated_shared(const FusionDev& d, float3 p, Cache& bc) {
  const float s = d.o.voxel_size, rs = d.r_vs;
  const float3 vp = make_float3(cdiv_<FAST>(p.x, s, rs), cdiv_<FAST>(p.y, s, rs), cdiv_<FAST>(p.z, s, rs));
  const uint2 v0 = voxel_at(d, w2g_axis(vp.x, p.x), w2g_axis(vp.y, p.y), w2g_axis(vp.z, p.z), bc);
  if ((v0.y >> 24) == 0) return v0;
  const float hs = d.half_vs;   // = div_(s, 2.0f), hoisted to the host (IEEE division there too)
  const float3 pd = make_float3(sub_(p.x, hs), sub_(p.y, hs), sub_(p.z, hs));
  const float wx = sub_(vp.x, floorf(vp.x)), wy = sub_(vp.y, floorf(vp.y)), wz = sub_(vp.z, floorf(vp.z));
  const float ux = sub_(1.f, wx), uy = sub_(1.f, wy), uz = sub_(1.f, wz);
  // the two voxel indices per axis that the corners pd + {0, s} round to
  const float ax0 = add_(pd.x, 0.f), ax1 = add_(pd.x, s), ay0 = add_(pd.y, 0.f), ay1 = add_(pd.y, s), az0 = add_(pd.z, 0.f), az1 = add_(pd.z, s);
  const int gx0 = w2g_axis(cdiv_<FAST>(ax0, s, rs), ax0), gx1 = w2g_axis(cdiv_<FAST>(ax1, s, rs), ax1);
  const int gy0 = w2g_axis(cdiv_<FAST>(ay0, s, rs), ay0), gy1 = w2g_axis(cdiv_<FAST>(ay1, s, rs), ay1);
  const int gz0 = w2g_axis(cdiv_<FAST>(az0, s, rs), az0), gz1 = w2g_axis(cdiv_<FAST>(az1, s, rs), az1);
  uint2 c[8];   // corner order of the reference: 000,100,010,001,110,011,101,111
  const bool one_block = gx1 == gx0 + 1 && gy1 == gy0 + 1 && gz1 == gz0 + 1 && (gx0 & 7) != 7 && (gy0 & 7) != 7 && (gz0 & 7) != 7;
  if (one_block) {
    const uint2* blk = bc.block(d, gx0 >> 3, gy0 >> 3, gz0 >> 3);
    if (!blk) {
#pragma unroll
      for (int k = 0; k < 8; ++k) c[k] = make_uint2(0u, 0u);
    } else {
      const uint2* b = blk + (gx0 & 7) * 64 + (gy0 & 7) * 8 + (gz0 & 7);
      c[0] = __ldg(b); c[1] = __ldg(b + 64); c[2] = __ldg(b + 8); c[3] = __ldg(b + 1);
      c[4] = __ldg(b + 72); c[5] = __ldg(b + 9); c[6] = __ldg(b + 65); c[7] = __ldg(b + 73);
    }
  } else {
    // The eight corners span at most two block rows per axis.  Reading them corner by corner through the one-entry cache
    // ping-pongs between the blocks (order 000,100,010,001,...: up to seven hash probes per sample, and - SIMT - every warp
    // has lanes on this path at every step: ncu counted ~600 warp instructions per marching step, two thirds of them probes).
    // Here every DISTINCT block is looked up once: P_ijk = block (bx_i, by_j, bz_k), and a combination that does not cross
    // a block face on some axis re-uses the pointer of its neighbour (typical sample: one axis crosses -> one new probe).
    // Pure memoisation of find_block on a volume that is constant during the render -> bit-identical.
    const int bx0 = gx0 >> 3, bx1 = gx1 >> 3, by0 = gy0 >> 3, by1 = gy1 >> 3, bz0 = gz0 >> 3, bz1 = gz1 >> 3;
    const bool cx = bx1 != bx0, cy = by1 != by0, cz = bz1 != bz0;
    const int ox0 = (gx0 & 7) * 64, ox1 = (gx1 & 7) * 64, oy0 = (gy0 & 7) * 8, oy1 = (gy1 & 7) * 8, oz0 = gz0 & 7, oz1 = gz1 & 7;
    auto rd = [](const uint2* blk, int off) { return blk ? __ldg(blk + off) : make_uint2(0u, 0u); };
    // A = block of the 0-side corner, Z = block of the 1-side corner.  With ONE crossing axis (87 % of these samples) every
    // corner lies in A or Z; only samples that cross two or three faces need more probes.  (Each bc.block call site is
    // executed by the warp whenever ANY lane needs it - the ordering below keeps the rarely needed sites rarely executed.)
    // (the one-entry cache holds the centre voxel's block, which is A or Z: when it is Z, keep it before A's lookup evicts it)
    const bool any = cx || cy || cz, zheld = any && bc.holds(bx1, by1, bz1);
    const uint2* pZh = zheld ? bc.held(d) : nullptr;
    const uint2* pA = bc.block(d, bx0, by0, bz0);
    const uint2* pZ = !any ? pA : (zheld ? pZh : bc.block(d, bx1, by1, bz1));
    const uint2* p100 = !cx ? pA : ((!cy && !cz) ? pZ : bc.block(d, bx1, by0, bz0));
    const uint2* p010 = !cy ? pA : ((!cx && !cz) ? pZ : bc.block(d, bx0, by1, bz0));
    const uint2* p001 = !cz ? pA : ((!cx && !cy) ? pZ : bc.block(d, bx0, by0, bz1));
    const uint2* p110 = !cz ? pZ : (!cx ? p010 : (!cy ? p100 : bc.block(d, bx1, by1, bz0)));
    const uint2* p101 = !cy ? pZ : (!cx ? p001 : (!cz ? p100 : bc.block(d, bx1, by0, bz1)));
    const uint2* p011 = !cx ? pZ : (!cy ? p001 : (!cz ? p010 : bc.block(d, bx0, by1, bz1)));
    c[0] = rd(pA, ox0 + oy0 + oz0);   c[1] = rd(p100, ox1 + oy0 + oz0); c[2] = rd(p010, ox0 + oy1 + oz0);
    c[3] = rd(p001, ox0 + oy0 + oz1); c[4] = rd(p110, ox1 + oy1 + oz0); c[5] = rd(p011, ox0 + oy1 + oz1);
    c[6] = rd(p101, ox1 + oy0 + oz1); c[7] = rd(pZ, ox1 + oy1 + oz1);
  }
  float dist = 0.f, cf[3] = {0.f, 0.f, 0.f};
  const int ox[8] = {0, 1, 0, 0, 1, 0, 1, 1}, oy[8] = {0, 0, 1, 0, 1, 1, 0, 1}, oz[8] = {0, 0, 0, 1, 0, 1, 1, 1};
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    uint2 v = c[k];
    if ((v.y >> 24) == 0) v = v0;
    const float w = mul_(mul_(ox[k] ? wx : ux, oy[k] ? wy : uy), oz[k] ? wz : uz);
    dist = add_(dist, mul_(w, __uint_as_float(v.x)));
    if constexpr (COLOR) {
#pragma unroll
      for (int q = 0; q < 3; ++q) cf[q] = add_(cf[q], mul_(w, (float)((v.y >> (8 * q)) & 0xFF)));
    }
  }
  unsigned col = 0;
  if constexpr (COLOR) {
#pragma unroll
    for (int q = 0; q < 3; ++q) col |= ((unsigned)cf[q] & 0xFF) << (8 * q);
  }
  return make_uint2(__float_as_uint(dist), col | (v0.y & 0xFF000000u));
}

// one ray per thread, shared-index sampling (the default ray-cast).  The kernel is latency-bound (a step is one long dependent
// chain: divide -> convert -> address -> load -> interpolate -> next t) and rays differ a lot in length, so small CTAs (8x8
// pixels, 20 CTAs per SM requested, which holds the kernel at 48 registers) at high residency balance better than 16x16,
// 16x8 or 8x4 ones (DESIGN.md, "TSDF variants removed").
// SLAB (Z-slab partition, SURVEY.md 8e): this rank stores only the blocks z in [slab_lo, slab_hi), so every sample whose
// trilinear neighbourhood lies outside that z range reads "no voxel" (weight 0) and advances the ray by exactly tau.  Those
// samples are not taken: before the ray enters the slab's z range `cur` is advanced by the same fp32 additions (cur += tau)
// without touching memory, and once the ray has left the range it can never hit again (world z is monotone along a ray), so
// it ends as a miss.  The samples that ARE taken sit at the same positions as in the unclipped march of this slab volume ->
// bit-identical slab renders at 1/N of the sampling work per rank.  keys != nullptr: the packed nearest-hit key
// (depth bits << 24 | colour, miss = +inf) is written straight from the ray's registers (the exchange step's operand).
__device__ __forceinline__ long long pack_hit_key(float depth, unsigned bgr24) {
  const long long bits = depth > 0.f ? (long long)__float_as_uint(depth) : 0x7F800000ll;
  return (bits << 24) | (long long)(depth > 0.f ? (bgr24 & 0xFFFFFFu) : 0u);
}
// PEER (pixel-partitioned ray-cast over a Z-slab-partitioned volume): this rank renders the pixel tiles t with t mod world ==
// rank, marching through the WHOLE volume; every voxel is read from the rank that owns its block row (CachePeer: local HBM or
// NVLink P2P).  Each sample therefore sees exactly the voxels of the un-partitioned volume at exactly the same positions: the
// union of the ranks' tiles is bit-identical to the single-volume render, occluders in other slabs included.  Foreign tiles
// get the "miss" key, so the same MIN all-reduce assembles the image.
// FAST: constant-divisor division (cdiv_), bit-identical to the IEEE division (option "fast_div", off by default).
template <bool SLAB, bool FAST, bool PEER>
__global__ void __launch_bounds__(64, 20)
k_raycast_shared(FusionDev d, Mat4 T, unsigned char* __restrict__ bgr_out, float* __restrict__ depth_out, long long* __restrict__ keys) {
  const tdm_fusion_options& o = d.o;
  const int x = blockIdx.x * 8 + (threadIdx.x % 8);
  const int y = blockIdx.y * 8 + (threadIdx.x / 8);
  if (x >= o.width || y >= o.height) return;
  const int i = y * o.width + x;
  const float ucx = sub_((float)x, o.cx), vcy = sub_((float)y, o.cy);   // get_point3d's pixel terms (utils.h:93-101)
  if constexpr (PEER) {
    if ((int)((blockIdx.y * gridDim.x + blockIdx.x) % (unsigned)d.pr_world) != d.pr_rank) {   // another rank's tile
      bgr_out[3 * i] = bgr_out[3 * i + 1] = bgr_out[3 * i + 2] = 0;
      depth_out[i] = 0.f;
      if (keys) keys[i] = pack_hit_key(0.f, 0u);
      return;
    }
  }
  typename std::conditional<PEER, CachePeer, Cache1P>::type bc;
  bc.init();
  float cur = 0.f;
  float t_exit = FLT_MAX;
  {
    // Clip the march to the bounding box of everything any scan ever allocated (d.bbox, replicated on every rank): outside it
    // every sample reads "no voxel" and advances by tau, so the leading ones are replaced by the same fp32 additions without
    // memory accesses and the trailing ones by an immediate miss - bit-identical, and it stops (a) rays that look out of the
    // mapped region and (b), in a Z-slab rank, rays that have passed an occluder stored on ANOTHER rank and would otherwise
    // march on to max_sensor_depth through this rank's empty space.
    // ray in world space: P(cur) = O + cur * D (linear model of xform(T, get_point3d(i, cur)); slack: 1 block + 2.5 voxels)
    const float ux = ((float)x - o.cx) / o.fx, uy = ((float)y - o.cy) / o.fy;
    const float s8 = 8.f * o.voxel_size, slack = 10.5f * o.voxel_size;
    float t_in = 0.f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float D = T.m[4 * a] * ux + T.m[4 * a + 1] * uy + T.m[4 * a + 2], O = T.m[4 * a + 3];
      const float lo = (float)d.bbox[a] * s8 - slack, hi = (float)(d.bbox[3 + a] + 1) * s8 + slack;
      if (fabsf(D) < 1e-12f) {
        if (O < lo || O > hi) t_in = FLT_MAX;
      } else {
        const float t0 = (lo - O) / D, t1 = (hi - O) / D;
        t_in = fmaxf(t_in, fminf(t0, t1));
        t_exit = fminf(t_exit, fmaxf(t0, t1));
      }
    }
    while (cur < t_in && cur < o.max_sensor_depth) cur = add_(cur, o.truncation_distance);
  }
  if (SLAB && d.il_k == 0) {
    // world z of the sample at ray parameter cur: zw = a * cur + b (linear model of xform(T, get_point3d(i, cur)).z; its
    // rounding differs from the exact evaluation by ~1e-6 m, covered by the half-voxel slack below).  A sample reads voxels
    // within +-1.5 voxels of its own position, a block b holds the voxels [8b - 0.5, 8b + 7.5) * s.
    const float a = T.m[8] * ((float)x - o.cx) / o.fx + T.m[9] * ((float)y - o.cy) / o.fy + T.m[10], b = T.m[11];
    const float s = o.voxel_size;
    const float zlo = ((float)d.slab_lo * 8.f - 2.5f) * s, zhi = ((float)d.slab_hi * 8.f + 2.5f) * s;
    float t_enter = 0.f;
    if (fabsf(a) < 1e-12f) {
      if (b < zlo || b > zhi) t_enter = FLT_MAX;                     // parallel to the slab and outside it
    } else {
      const float t0 = (zlo - b) / a, t1 = (zhi - b) / a;
      t_enter = fminf(t0, t1);
      t_exit = fminf(t_exit, fmaxf(t0, t1));
    }
    while (cur < t_enter && cur < o.max_sensor_depth) cur = add_(cur, o.truncation_distance);   // what the skipped samples would do
  }
  int guard = 0;
  bool hit = false;
  float il_a = 0.f, il_b = 0.f;
  if constexpr (SLAB) {
    if (d.il_k > 0) {   // interleaved slabs: sample world z / voxel_size = il_a * cur + il_b (linear model, 2.5-voxel slack below)
      il_a = (T.m[8] * ((float)x - o.cx) / o.fx + T.m[9] * ((float)y - o.cy) / o.fy + T.m[10]) / o.voxel_size;
      il_b = T.m[11] / o.voxel_size;
    }
  }
  while (cur < o.max_sensor_depth && guard++ < 100000) {
    if constexpr (SLAB) {
      if (d.il_k > 0) {
        // a sample reads voxels within +-1.5 voxels of its position; skip it (advance by tau, exactly what a sample that finds
        // no voxel does) unless one of the block rows it can touch is stored on this rank
        const float zv = fmaf(il_a, cur, il_b);
        const int b0 = (int)floorf(zv - 2.5f) >> 3, b1 = (int)floorf(zv + 2.5f) >> 3;
        if (!slab_stores(d, b0) && !slab_stores(d, b1)) { cur = add_(cur, o.truncation_distance); continue; }
      }
    }
    if (cur > t_exit) break;
    const uint2 v = get_interpolated_shared<decltype(bc), false, FAST>(d, xform(T, get_point3d_px<FAST>(d, ucx, vcy, cur)), bc);
    const unsigned w = v.y >> 24;
    const float sdf = __uint_as_float(v.x);
    cur = add_(cur, w == 0 ? o.truncation_distance : sdf);
    if (w != 0 && sdf < o.voxel_size) { hit = true; break; }
  }
  // (un-clipped march: a ray that runs out of range ends with cur >= max_sensor_depth; the slab march may also stop behind the slab)
  if (hit && cur < o.max_sensor_depth) {
    const uint2 v = get_interpolated_shared<decltype(bc), true, FAST>(d, xform(T, get_point3d_px<FAST>(d, ucx, vcy, cur)), bc);
    bgr_out[3 * i] = v.y & 0xFF; bgr_out[3 * i + 1] = (v.y >> 8) & 0xFF; bgr_out[3 * i + 2] = (v.y >> 16) & 0xFF;
    depth_out[i] = cur;
    if (keys) keys[i] = pack_hit_key(cur, v.y);
  } else {
    bgr_out[3 * i] = bgr_out[3 * i + 1] = bgr_out[3 * i + 2] = 0;
    depth_out[i] = 0.f;
    if (keys) keys[i] = pack_hit_key(0.f, 0u);
  }
}

// The comparator (option "raycast_shared" = 0): the reference's march and sampler (tsdf_volume.cu:600-632, 161-289) restated
// voxel by voxel - one hash probe per voxel read behind a last-block cache, IEEE divisions, sgn().  Every production variant of
// k_raycast_shared must render the same volume bit for bit (tests/test_fusion_gpu.py::test_raycast_is_bit_identical_to_reference_sampler).
__global__ void __launch_bounds__(256)
k_raycast(FusionDev d, Mat4 T, unsigned char* __restrict__ bgr_out, float* __restrict__ depth_out) {
  const tdm_fusion_options& o = d.o;
  const int x = blockIdx.x * 16 + (threadIdx.x & 15);
  const int y = blockIdx.y * 16 + (threadIdx.x >> 4);
  if (x >= o.width || y >= o.height) return;
  const int i = y * o.width + x;
  Cache1 bc;
  bc.init();
  float cur = 0.f;
  int guard = 0;
  while (cur < o.max_sensor_depth && guard++ < 100000) {
    const uint2 v = get_interpolated(d, xform(T, get_point3d(o, i, cur)), bc);
    const unsigned w = v.y >> 24;
    const float sdf = __uint_as_float(v.x);
    cur = add_(cur, w == 0 ? o.truncation_distance : sdf);
    if (w != 0 && sdf < o.voxel_size) break;
  }
  if (cur < o.max_sensor_depth) {
    const uint2 v = get_interpolated(d, xform(T, get_point3d(o, i, cur)), bc);
    bgr_out[3 * i] = v.y & 0xFF; bgr_out[3 * i + 1] = (v.y >> 8) & 0xFF; bgr_out[3 * i + 2] = (v.y >> 16) & 0xFF;
    depth_out[i] = cur;
  } else {
    bgr_out[3 * i] = bgr_out[3 * i + 1] = bgr_out[3 * i + 2] = 0;
    depth_out[i] = 0.f;
  }
}

// Slab-partitioned ray-cast (SURVEY.md 8e): per-pixel key = depth bits << 24 | b | g << 8 | r << 16, a miss = +inf, so that the
// per-pixel MIN over ranks (one NCCL all-reduce on these device buffers) keeps the nearest hit and its colour.
__global__ void k_pack_hits(const float* __restrict__ depth, const unsigned char* __restrict__ bgr, long long* __restrict__ keys, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float d = depth[i];
  const long long bits = d > 0.f ? (long long)__float_as_uint(d) : 0x7F800000ll;
  keys[i] = (bits << 24) | (long long)bgr[3 * i] | ((long long)bgr[3 * i + 1] << 8) | ((long long)bgr[3 * i + 2] << 16);
}
__global__ void k_unpack_hits(const long long* __restrict__ keys, float* __restrict__ depth, unsigned char* __restrict__ bgr, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long k = keys[i];
  const unsigned bits = (unsigned)(k >> 24);
  const bool miss = bits == 0x7F800000u;
  depth[i] = miss ? 0.f : __uint_as_float(bits);
  bgr[3 * i] = miss ? 0 : (unsigned char)(k & 0xFF);
  bgr[3 * i + 1] = miss ? 0 : (unsigned char)((k >> 8) & 0xFF);
  bgr[3 * i + 2] = miss ? 0 : (unsigned char)((k >> 16) & 0xFF);
}

__global__ void k_fill_keys(unsigned long long* keys, int* ptrs, long long n) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) { keys[i] = kEmptyKey; ptrs[i] = -1; }
}

#include "mesh.cuh"

// ---- host side of the mesh extractor: the per-axis tables (same fp32 expression sequence as the reference) ----
inline int w2g1_host(float x, float s) {   // one axis of WorldToGlobalVoxel, tsdf_volume.cu:109-113
  const float sg = (float)((x > 0) - (x < 0));
  return (int)(x / s + sg * 0.5f);
}
inline int floor_div8(int v) { return v >> 3; }

struct MeshAxisHost {
  std::vector<MeshAxisCell> cells;
  std::vector<int2> ranges;
  int bmin = 0, nb = 0;
};

MeshAxisHost build_mesh_axis(float lower, float upper, float s) {
  MeshAxisHost A;
  const float ext = fabsf(lower - upper) / s;                 // mesh_extractor.cu:248-252
  TDM_CHECK(ext == ext && ext < 4.0e6f && fabsf(lower) < 1.0e5f && fabsf(upper) < 1.0e5f, "mesh bounding box too large");
  const int n = (int)ext;
  if (n <= 0) return A;
  const float h = s / 2.0f;
  A.cells.resize(n);
  for (int i = 0; i < n; ++i) {
    MeshAxisCell c;
    const float pos = std::fmaf((float)i, s, lower);          // mesh_extractor.cu:258-261 (contracted by the reference's nvcc)
    c.cM = pos + (-h);                                        // :143-144 (M = -P)
    c.cP = pos + h;
    const float pdM = c.cM - h, pdP = c.cP - h;               // :28-30
    const float vpM = c.cM / s, vpP = c.cP / s;               // :31
    c.wM = vpM - floorf(vpM);                                 // :32-34
    c.wP = vpP - floorf(vpP);
    c.gMA = w2g1_host(pdM + 0.0f, s); c.gMB = w2g1_host(pdM + s, s);
    c.gPA = w2g1_host(pdP + 0.0f, s); c.gPB = w2g1_host(pdP + s, s);
    c.gC = w2g1_host(pos, s);
    A.cells[i] = c;
    const int blk = floor_div8(c.gMA);
    const int lo = std::min(std::min(c.gMA, c.gMB), std::min(std::min(c.gPA, c.gPB), c.gC));
    const int hi = std::max(std::max(c.gMA, c.gMB), std::max(std::max(c.gPA, c.gPB), c.gC));
    TDM_CHECK(lo >= blk * 8 && hi < blk * 8 + kMeshTile, "mesh: voxel reach of a cell exceeds the staged tile");
    TDM_CHECK(i == 0 || c.gMA >= A.cells[i - 1].gMA, "mesh: voxel index is not monotone in the cell index");
  }
  A.bmin = floor_div8(A.cells[0].gMA);
  A.nb = floor_div8(A.cells[n - 1].gMA) - A.bmin + 1;
  A.ranges.assign(A.nb, make_int2(0, 0));
  for (int i = 0; i < n; ++i) {
    int2& r = A.ranges[floor_div8(A.cells[i].gMA) - A.bmin];
    if (r.y == 0) r.x = i;
    r.y++;
  }
  return A;
}

}  // namespace

// ================================================================================================
class FusionImpl final : public FusionIface {
 public:
  FusionImpl(const tdm_fusion_options& o, int device) : device_(device) {
    int nd = 0;
    if (cudaGetDeviceCount(&nd) != cudaSuccess || nd == 0)
      throw Error("tandem_b200: no CUDA device visible - this library has no CPU fallback");
    TDM_CHECK(o.block_size == 8, "block_size must be 8 (the voxel block layout is 8x8x8 as in FullSystem.cpp:259-276)");
    TDM_CHECK(o.num_buckets > 0 && o.bucket_size > 0 && o.num_blocks > 0, "bad hash table options");
    TDM_CHECK(o.height > 0 && o.width > 0 && o.num_render_streams >= 0, "bad image options");
    TDM_CHECK(o.max_sdf_weight > 0 && o.max_sdf_weight <= 255, "max_sdf_weight must fit the u8 voxel weight");
    TDM_CUDA(cudaSetDevice(device_));
    d_.o = o;
    d_.slab_lo = INT_MIN;
    d_.slab_hi = INT_MAX;
    d_.il_k = 0; d_.il_world = 1; d_.il_rank = 0; d_.il_z0 = 0;
    d_.pr_world = 0; d_.pr_rank = 0;
    {
      // reciprocals for cdiv_: host IEEE division = correctly rounded (the file is built with -ffp-contract=off, no fast-math)
      volatile float one = 1.0f;
      d_.r_vs = one / o.voxel_size; d_.r_fx = one / o.fx; d_.r_fy = one / o.fy;
      volatile float two = 2.0f;
      d_.half_vs = o.voxel_size / two;
      auto ok = [](float d) {
        unsigned u;
        std::memcpy(&u, &d, 4);
        const unsigned ex = (u >> 23) & 0xFF, man = u & 0x7FFFFF;
        return d > 0.f && ex > 40 && ex < 214 && man != 0x7FFFFF;   // 2^-87 < d < 2^87, significand not all ones
      };
      fast_div_ok_ = ok(o.voxel_size) && ok(o.fx) && ok(o.fy);
      // div.rn.f32's fast path is already ~8 instructions and the ray-cast is latency-, not issue-bound.  Kept as an A/B option
      // (bit-identical), off by default; DESIGN.md ("TSDF variants removed") records its timings.
      const char* e = getenv("TDM_FAST_DIV");
      fast_div_ = fast_div_ok_ && e && e[0] == '1';
    }
    n_entries_ = (long long)o.num_buckets * o.bucket_size;
    d_.mod_magic = 0xFFFFFFFFFFFFFFFFull / (unsigned long long)o.num_buckets + 1ull;
    d_.mod_c32 = (unsigned)((1ull << 32) % (unsigned long long)o.num_buckets);
    int lo, hi;
    TDM_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    stream_ = make_stream(lo);  // low priority as tsdf_volume.cu:64-75
    keys_ = make_dev<unsigned long long>(n_entries_ * 8); d_.keys = keys_.get();
    ptrs_ = make_dev<int>(n_entries_ * 4); d_.ptrs = ptrs_.get();
    voxels_ = make_dev<uint2>((size_t)o.num_blocks * 512 * 8); d_.voxels = voxels_.get();
    list_ = make_dev<int4>((size_t)o.num_blocks * sizeof(int4)); d_.list = list_.get();
    counters_ = make_dev<int>(8 * sizeof(int)); d_.counters = counters_.get();
    bbox_ = make_dev<int>(6 * sizeof(int)); d_.bbox = bbox_.get();
    {
      const int init[6] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN};
      TDM_CUDA(cudaMemcpy(d_.bbox, init, sizeof(init), cudaMemcpyHostToDevice));
    }
    d_vis_list_ = make_dev<int>((size_t)o.num_blocks * sizeof(int));
    TDM_CUDA(cudaMemsetAsync(d_.voxels, 0, (size_t)o.num_blocks * 512 * 8, stream_.get()));
    TDM_CUDA(cudaMemsetAsync(d_.counters, 0, 8 * sizeof(int), stream_.get()));
    k_fill_keys<<<cdiv(n_entries_, 256), 256, 0, stream_.get()>>>(d_.keys, d_.ptrs, n_entries_);
    TDM_CUDA(cudaGetLastError());
    const size_t npx = (size_t)o.height * o.width;
    h_bgr_in_ = make_host<unsigned char>(npx * 3);
    h_depth_in_ = make_host<float>(npx * 4);
    d_bgr_in_ = make_dev<unsigned char>(npx * 3);
    d_depth_in_ = make_dev<float>(npx * 4);
    const int ns = std::max(1, o.num_render_streams);
    for (int half = 0; half < 2; ++half) {
      h_bgr_out_[half] = make_host<unsigned char>(npx * 3 * ns);
      h_depth_out_[half] = make_host<float>(npx * 4 * ns);
      std::memset(h_bgr_out_[half].get(), 0, npx * 3 * ns);     // "slab_exchange" mode never writes them: GetRenderResult then hands out
      std::memset(h_depth_out_[half].get(), 0, npx * 4 * ns);   // all-miss images rather than uninitialised memory
    }
    d_bgr_out_ = make_dev<unsigned char>(npx * 3 * ns);
    d_depth_out_ = make_dev<float>(npx * 4 * ns);
    h_counters_ = make_host<int>(8 * sizeof(int));
    ev_int_ = make_event(cudaEventDisableTiming);
    ev_render_ = make_event(cudaEventDisableTiming);
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    render_poses_.resize(ns);
  }

  ~FusionImpl() override {
    cudaSetDevice(device_);
    cudaStreamSynchronize(stream_.get());
    for (void* q : ipc_opened_) cudaIpcCloseMemHandle(q);
  }

  // IntegrateScanAsync, tsdf_volume.cu:515-598
  void integrate_async(const unsigned char* bgr, const float* depth, const float* pose) override {
    if (next_ != kIntegrate)
      throw Error("call order is IntegrateScanAsync -> RenderAsync -> GetRenderResult (tsdf_volume.cu:520-525)");
    TDM_CUDA(cudaSetDevice(device_));
    const size_t npx = (size_t)d_.o.height * d_.o.width;
    std::memcpy(pose_.m, pose, 64);
    if (!inv4_f32(pose_.m, pose_inv_.m)) throw Error("camera pose is singular");
    auto page_locked = [](const void* p) {
      cudaPointerAttributes at{};
      if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
      return at.type == cudaMemoryTypeHost;
    };
    if (page_locked(bgr) && page_locked(depth)) {
      // page-locked caller buffers: DMA straight from them; they are only ours during this call (tsdf_volume.cu:542-543
      // copies before returning), so wait for the two DMAs (2.15 MB, ~45 us) - cheaper than the staging memcpy it replaces
      TDM_CUDA(cudaMemcpyAsync(d_bgr_in_.get(), bgr, npx * 3, cudaMemcpyHostToDevice, stream_.get()));
      TDM_CUDA(cudaMemcpyAsync(d_depth_in_.get(), depth, npx * 4, cudaMemcpyHostToDevice, stream_.get()));
      TDM_CUDA(cudaEventRecord(ev_int_.get(), stream_.get()));
      launch_integrate();
      TDM_CUDA(cudaEventSynchronize(ev_int_.get()));
    } else {
      TDM_CUDA(cudaEventSynchronize(ev_int_.get()));  // previous scan has left the pinned staging buffers
      std::memcpy(h_bgr_in_.get(), bgr, npx * 3);
      std::memcpy(h_depth_in_.get(), depth, npx * 4);
      TDM_CUDA(cudaMemcpyAsync(d_bgr_in_.get(), h_bgr_in_.get(), npx * 3, cudaMemcpyHostToDevice, stream_.get()));
      TDM_CUDA(cudaMemcpyAsync(d_depth_in_.get(), h_depth_in_.get(), npx * 4, cudaMemcpyHostToDevice, stream_.get()));
      launch_integrate();
    }
    TDM_CUDA(cudaEventRecord(ev_int_.get(), stream_.get()));
    have_scan_ = true;
    ++volume_epoch_;   // a pending mesh extracted before this scan no longer describes the volume
    next_ = kRender;
  }

  // IntegrateScanAsync from device memory (the MVSNet keyframe handoff, tdm_fusion_integrate_mvsnet): the same scan buffers
  // and the same launch_integrate as above, filled device to device; no host synchronisation.  Checks everything before
  // anything is enqueued.
  void integrate_device(const unsigned char* bgr, const float* depth, int height, int width, int device, void* ready,
                        const float* pose) override {
    if (next_ != kIntegrate)
      throw Error("call order is IntegrateScanAsync -> RenderAsync -> GetRenderResult (tsdf_volume.cu:520-525)");
    TDM_CHECK(device == device_, "the MVSNet handle and the fusion live on different devices");
    TDM_CHECK(height == d_.o.height && width == d_.o.width, "the MVSNet window's height / width differ from the fusion's");
    Mat4 p, pinv;
    std::memcpy(p.m, pose, 64);
    if (!inv4_f32(p.m, pinv.m)) throw Error("camera pose is singular");
    TDM_CUDA(cudaSetDevice(device_));
    const size_t npx = (size_t)d_.o.height * d_.o.width;
    TDM_CUDA(cudaStreamWaitEvent(stream_.get(), (cudaEvent_t)ready, 0));
    TDM_CUDA(cudaMemcpyAsync(d_bgr_in_.get(), bgr, npx * 3, cudaMemcpyDeviceToDevice, stream_.get()));
    TDM_CUDA(cudaMemcpyAsync(d_depth_in_.get(), depth, npx * 4, cudaMemcpyDeviceToDevice, stream_.get()));
    pose_ = p;
    pose_inv_ = pinv;
    launch_integrate();
    TDM_CUDA(cudaEventRecord(ev_int_.get(), stream_.get()));
    have_scan_ = true;
    ++volume_epoch_;
    next_ = kRender;
  }

  // RenderAsync, tsdf_volume.cu:634-700
  void render_async(const float* const* poses, int n) override {
    if (next_ != kRender) throw Error("call order is IntegrateScanAsync -> RenderAsync -> GetRenderResult (tsdf_volume.cu:635-640)");
    if (n != d_.o.num_render_streams) throw Error("RenderAsync: number of poses must equal num_render_streams (tsdf_volume.cu:643-648)");
    TDM_CUDA(cudaSetDevice(device_));
    for (int i = 0; i < n; ++i) std::memcpy(render_poses_[i].m, poses[i], 64);
    launch_render(n, true);
    TDM_CUDA(cudaEventRecord(ev_render_.get(), stream_.get()));
    n_rendered_ = n;
    next_ = kGet;
  }

  // GetRenderResult, tsdf_volume.cu:702-737
  void get_render_result(unsigned char** bgr, float** depth, int n) override {
    if (next_ != kGet) throw Error("call order is IntegrateScanAsync -> RenderAsync -> GetRenderResult (tsdf_volume.cu:703-708)");
    if (n != n_rendered_) throw Error("GetRenderResult: wrong number of outputs");
    TDM_CUDA(cudaSetDevice(device_));
    if (!slab_exchange_) TDM_CUDA(cudaEventSynchronize(ev_render_.get()));   // exchange mode: nothing was copied back, nothing to wait for
    const size_t npx = (size_t)d_.o.height * d_.o.width;
    for (int i = 0; i < n; ++i) {
      bgr[i] = h_bgr_out_[free_half_].get() + (size_t)i * npx * 3;
      depth[i] = h_depth_out_[free_half_].get() + (size_t)i * npx;
    }
    free_half_ ^= 1;  // the returned half stays valid until the next GetRenderResult (tsdf_volume.cu:719-732)
    next_ = kIntegrate;
  }

  void set_slab(int z_lo, int z_hi) override {
    TDM_CHECK(z_lo < z_hi, "empty slab");
    TDM_CHECK(!have_scan_, "set_slab must be called before the first scan");
    d_.slab_lo = z_lo;
    d_.slab_hi = z_hi;
  }

  // Peer view (pixel-partitioned ray-cast): export this instance's tables, attach everybody's.
  void peer_export(tdm_fusion_peer_handle* out) override {
    TDM_CUDA(cudaSetDevice(device_));
    std::memset(out, 0, sizeof(*out));
    out->keys_ptr = (unsigned long long)(uintptr_t)d_.keys;
    out->ptrs_ptr = (unsigned long long)(uintptr_t)d_.ptrs;
    out->voxels_ptr = (unsigned long long)(uintptr_t)d_.voxels;
    out->device = device_;
    out->pid = (long long)getpid();
    out->num_buckets = d_.o.num_buckets; out->bucket_size = d_.o.bucket_size;
    out->slab_lo = d_.slab_lo; out->slab_hi = d_.slab_hi;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    TDM_CUDA(cudaIpcGetMemHandle((cudaIpcMemHandle_t*)out->ipc_keys, d_.keys));
    TDM_CUDA(cudaIpcGetMemHandle((cudaIpcMemHandle_t*)out->ipc_ptrs, d_.ptrs));
    TDM_CUDA(cudaIpcGetMemHandle((cudaIpcMemHandle_t*)out->ipc_voxels, d_.voxels));
  }
  void peer_attach(const tdm_fusion_peer_handle* all, int world, int rank) override {
    TDM_CHECK(world >= 1 && world <= 8 && rank >= 0 && rank < world, "peer_attach: world must be 1..8");
    TDM_CHECK(d_.il_k == 0, "the peer view needs contiguous Z-slabs (set_slab), not the interleaved partition");
    TDM_CUDA(cudaSetDevice(device_));
    for (int r = 0; r < world; ++r) {
      const tdm_fusion_peer_handle& h = all[r];
      TDM_CHECK(h.num_buckets == d_.o.num_buckets && h.bucket_size == d_.o.bucket_size, "peer_attach: hash table geometry differs between ranks");
      TDM_CHECK(r == 0 || h.slab_lo == all[r - 1].slab_hi, "peer_attach: slabs must be contiguous in rank order and WITHOUT halo rows");
      void *k = nullptr, *p = nullptr, *v = nullptr;
      if (r == rank) {
        k = d_.keys; p = d_.ptrs; v = d_.voxels;
      } else if (h.pid == (long long)getpid()) {      // another instance of this process (tests; single-process multi-GPU)
        k = (void*)(uintptr_t)h.keys_ptr; p = (void*)(uintptr_t)h.ptrs_ptr; v = (void*)(uintptr_t)h.voxels_ptr;
        if (h.device != device_) {
          int can = 0;
          TDM_CUDA(cudaDeviceCanAccessPeer(&can, device_, h.device));
          TDM_CHECK(can, "peer_attach: no peer access between the two devices");
          const cudaError_t e = cudaDeviceEnablePeerAccess(h.device, 0);
          if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) TDM_CUDA(e);
          cudaGetLastError();
        }
      } else {                                         // another process: CUDA IPC (maps the peer's allocation over NVLink / PCIe P2P)
        TDM_CUDA(cudaIpcOpenMemHandle(&k, *(const cudaIpcMemHandle_t*)h.ipc_keys, cudaIpcMemLazyEnablePeerAccess));
        TDM_CUDA(cudaIpcOpenMemHandle(&p, *(const cudaIpcMemHandle_t*)h.ipc_ptrs, cudaIpcMemLazyEnablePeerAccess));
        TDM_CUDA(cudaIpcOpenMemHandle(&v, *(const cudaIpcMemHandle_t*)h.ipc_voxels, cudaIpcMemLazyEnablePeerAccess));
        ipc_opened_.push_back(k); ipc_opened_.push_back(p); ipc_opened_.push_back(v);
      }
      d_.pr_keys[r] = (const unsigned long long*)k; d_.pr_ptrs[r] = (const int*)p; d_.pr_voxels[r] = (const uint2*)v;
      d_.pr_lo[r] = h.slab_lo; d_.pr_hi[r] = h.slab_hi;
    }
    d_.pr_world = world; d_.pr_rank = rank;
  }

  void set_interleave(int rank, int world, int k_blocks, int z0_block) override {
    TDM_CHECK(world >= 1 && rank >= 0 && rank < world && k_blocks >= 1, "bad interleave parameters");
    TDM_CHECK(!have_scan_, "set_interleave must be called before the first scan");
    if (world == 1) return;   // one rank stores everything
    d_.il_k = k_blocks; d_.il_world = world; d_.il_rank = rank; d_.il_z0 = z0_block;
    d_.slab_lo = INT_MIN + 1;   // marks the volume as partitioned (mesh extraction refuses, ray-cast takes the SLAB path)
  }

  void synchronize() override {
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
  }

  void get_stats(tdm_fusion_stats* s) override {
    fetch_counters();
    s->allocated_blocks = std::min(h_counters_.get()[0], d_.o.num_blocks);
    s->dropped_blocks = h_counters_.get()[1];
    s->visible_blocks = h_counters_.get()[2];
    s->candidate_blocks = h_counters_.get()[3];
  }

  long long dump_blocks(int* coords, void* voxels, size_t cap) override {
    fetch_counters();
    const long long n = std::min(h_counters_.get()[0], d_.o.num_blocks);
    if (!coords) return n;
    std::vector<int4> list((size_t)n);
    TDM_CUDA(cudaMemcpy(list.data(), d_.list, (size_t)n * sizeof(int4), cudaMemcpyDeviceToHost));
    std::sort(list.begin(), list.end(), [](const int4& a, const int4& b) {
      if (a.x != b.x) return a.x < b.x;
      if (a.y != b.y) return a.y < b.y;
      return a.z < b.z;
    });
    const long long m = std::min<long long>(n, (long long)cap);
    for (long long k = 0; k < m; ++k) {
      coords[3 * k] = list[k].x; coords[3 * k + 1] = list[k].y; coords[3 * k + 2] = list[k].z;
      if (voxels)
        TDM_CUDA(cudaMemcpy((char*)voxels + (size_t)k * 4096, d_.voxels + (size_t)list[k].w * 512, 4096, cudaMemcpyDeviceToHost));
    }
    return n;
  }

  // ExtractMeshAsync, tsdf_volume.cu:759-779 (+ MeshExtractor::ExtractMesh, mesh_extractor.cu:267-282)
  void extract_mesh_async(const float* lower, const float* upper, bool check_order) override {
    if (check_order && next_ != kIntegrate)
      throw Error("Please call this function after GetRenderResult (tsdf_volume.cu:760-763)");
    if (mesh_kind_ == kMeshAsync) throw Error("ExtractMeshAsync called twice without GetMeshSync (tsdf_volume.cu:769-772)");
    start_mesh(lower, upper);
    mesh_kind_ = kMeshAsync;   // only once everything is enqueued: a failed call leaves no half-started extraction behind
  }

  // GetMeshSync, tsdf_volume.cu:781-839: vertices as xyz triples, colours as rgb triples, 3 per triangle
  long long get_mesh(float* vert, float* cols, size_t max_vertices, bool check_order, bool query_only) override {
    if (check_order && next_ != kIntegrate)
      throw Error("Please call this function after GetRenderResult (tsdf_volume.cu:782-785)");
    if (mesh_kind_ != kMeshAsync) throw Error("GetMeshSync without ExtractMeshAsync (tsdf_volume.cu:787-790)");
    if (!query_only) mesh_kind_ = kMeshNone;   // consumed even if the copy-out below fails (the reference exits there)
    return finish_mesh(vert, cols, max_vertices, query_only);
  }

  // TsdfVolume::ExtractMesh (blocking, tsdf_volume.cu:739-757).  The reference runs it on an extractor of its own, so it
  // never disturbs an ExtractMeshAsync/GetMeshSync pair; here both share the device buffers, hence a blocking call while an
  // asynchronous result is un-fetched is rejected instead of silently consuming it.  A count-only query (vert == cols ==
  // nullptr) keeps the mesh on the device; it is re-used by the following copy call only for the identical box and an
  // unchanged volume, anything else extracts again.
  long long extract_mesh_blocking(const float* lower, const float* upper, float* vert, float* cols, size_t max_vertices) override {
    if (mesh_kind_ == kMeshAsync)
      throw Error("ExtractMesh (GetMesh / SaveMeshToFile) while an ExtractMeshAsync result is pending: call GetMeshSync first");
    const bool query_only = vert == nullptr && cols == nullptr;
    bool reuse = mesh_kind_ == kMeshBlocking && mesh_epoch_ == volume_epoch_;
    for (int a = 0; a < 3 && reuse; ++a) reuse = mesh_lower_[a] == lower[a] && mesh_upper_[a] == upper[a];
    if (!reuse) {
      mesh_kind_ = kMeshNone;
      start_mesh(lower, upper);
      mesh_kind_ = kMeshBlocking;
    }
    if (!query_only) mesh_kind_ = kMeshNone;
    return finish_mesh(vert, cols, max_vertices, query_only);
  }
  float last_mesh_ms() override { return mesh_ms_; }
  float last_alloc_ms() override { return last_alloc_ms_; }
  void set_option(const char* name, int value) override {
    const std::string n(name);
    if (n == "raycast_shared") raycast_shared_ = value != 0;
    else if (n == "slab_clip") slab_clip_ = value != 0;
    else if (n == "fast_div") fast_div_ = value != 0 && fast_div_ok_;
    else if (n == "slab_exchange") slab_exchange_ = value != 0;
    else throw Error("unknown fusion option " + n);
  }
  bool mesh_pending() override { return mesh_kind_ != kMeshNone; }

  const float* render_depth_device(int i, void** ready_event, int* device) override {
    TDM_CHECK(i >= 0 && i < n_rendered_, "render_depth_device: no such render");
    if (ready_event) *ready_event = (void*)ev_render_.get();
    if (device) *device = device_;
    return d_depth_out_.get() + (size_t)i * d_.o.height * d_.o.width;
  }
  // slab exchange step: device buffer of packed nearest-hit keys of render i (valid until the next call), stream synchronised
  long long* render_keys_device(int i) override {
    TDM_CHECK(i >= 0 && i < n_rendered_, "render_keys_device: no such render");
    TDM_CUDA(cudaSetDevice(device_));
    const int npx = d_.o.height * d_.o.width;
    if (slab_exchange_) {   // the ray-cast wrote the keys itself; no extra kernel, no host sync: the caller's collective is
      TDM_CHECK(i == 0 && d_hit_keys_, "slab exchange mode packs render 0 only");   // enqueued on stream() behind it
      return d_hit_keys_.get();
    }
    if (!d_hit_keys_) d_hit_keys_ = make_dev<long long>((size_t)npx * sizeof(long long));
    k_pack_hits<<<cdiv(npx, 256), 256, 0, stream_.get()>>>(d_depth_out_.get() + (size_t)i * npx, d_bgr_out_.get() + (size_t)i * npx * 3, d_hit_keys_.get(), npx);
    TDM_CUDA(cudaGetLastError());
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
    return d_hit_keys_.get();
  }
  void* stream() override { return (void*)stream_.get(); }
  void unpack_keys(const long long* keys_dev, float* depth_out, unsigned char* bgr_out) override {
    TDM_CUDA(cudaSetDevice(device_));
    const int npx = d_.o.height * d_.o.width;
    if (!d_unpack_depth_) {   // set last: the pair is complete once it is
      DevPtr<float> depth = make_dev<float>((size_t)npx * 4);
      d_unpack_bgr_ = make_dev<unsigned char>((size_t)npx * 3);
      d_unpack_depth_ = std::move(depth);
    }
    k_unpack_hits<<<cdiv(npx, 256), 256, 0, stream_.get()>>>(keys_dev, d_unpack_depth_.get(), d_unpack_bgr_.get(), npx);
    TDM_CUDA(cudaGetLastError());
    TDM_CUDA(cudaMemcpyAsync(depth_out, d_unpack_depth_.get(), (size_t)npx * 4, cudaMemcpyDeviceToHost, stream_.get()));
    TDM_CUDA(cudaMemcpyAsync(bgr_out, d_unpack_bgr_.get(), (size_t)npx * 3, cudaMemcpyDeviceToHost, stream_.get()));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
  }
  void run_resident(int iters, float* ms_int, float* ms_render) override {
    TDM_CHECK(have_scan_, "run_resident: no scan submitted yet");
    TDM_CUDA(cudaSetDevice(device_));
    const Event e0 = make_event(), e1 = make_event(), e2 = make_event(), split = make_event();
    float ti = 0, tr = 0, ta = 0;
    const int n = std::max(1, d_.o.num_render_streams);
    if (render_poses_.empty()) render_poses_.resize(1);
    for (int it = 0; it < iters; ++it) {
      TDM_CUDA(cudaEventRecord(e0.get(), stream_.get()));
      launch_integrate(split.get());
      TDM_CUDA(cudaEventRecord(e1.get(), stream_.get()));
      launch_render(n, false);
      TDM_CUDA(cudaEventRecord(e2.get(), stream_.get()));
      TDM_CUDA(cudaEventSynchronize(e2.get()));
      float a, b, c;
      TDM_CUDA(cudaEventElapsedTime(&a, e0.get(), e1.get()));
      TDM_CUDA(cudaEventElapsedTime(&b, e1.get(), e2.get()));
      TDM_CUDA(cudaEventElapsedTime(&c, e0.get(), split.get()));
      ti += a; tr += b; ta += c;
    }
    *ms_int = ti; *ms_render = tr;
    last_alloc_ms_ = ta / std::max(iters, 1);
  }

 private:
  // split (run_resident only) is recorded between the allocation and the visibility pass
  void launch_integrate(cudaEvent_t split = nullptr) {
    const int npx = d_.o.height * d_.o.width;
    TDM_CUDA(cudaMemsetAsync(d_.counters + 2, 0, 2 * sizeof(int), stream_.get()));
    k_allocate<<<cdiv(npx, 128), 128, 0, stream_.get()>>>(d_, d_depth_in_.get(), pose_);
    TDM_CUDA(cudaGetLastError());
    if (split) TDM_CUDA(cudaEventRecord(split, stream_.get()));
    k_visible<<<cdiv(d_.o.num_blocks, 256), 256, 0, stream_.get()>>>(d_, pose_inv_, d_vis_list_.get());
    TDM_CUDA(cudaGetLastError());
    k_integrate_list<<<132 * 8, 256, 0, stream_.get()>>>(d_, d_bgr_in_.get(), d_depth_in_.get(), pose_inv_, d_vis_list_.get());
    TDM_CUDA(cudaGetLastError());
  }
  void launch_render(int n, bool copy_back) {
    const size_t npx = (size_t)d_.o.height * d_.o.width;
    const dim3 grid8(cdiv(d_.o.width, 8), cdiv(d_.o.height, 8));
    const bool peer = d_.pr_world > 1;
    const bool slab = !peer && (d_.slab_lo != INT_MIN || d_.slab_hi != INT_MAX) && slab_clip_;
    for (int i = 0; i < n; ++i) {
      unsigned char* bo = d_bgr_out_.get() + (size_t)i * npx * 3;
      float* dout_i = d_depth_out_.get() + (size_t)i * npx;
      long long* keys = nullptr;
      if (slab_exchange_ && raycast_shared_ && i == 0) {   // k_raycast writes no keys
        if (!d_hit_keys_) d_hit_keys_ = make_dev<long long>(npx * sizeof(long long));
        keys = d_hit_keys_.get();
      }
      const Mat4& T = render_poses_[i];
      if (!raycast_shared_) k_raycast<<<dim3(cdiv(d_.o.width, 16), cdiv(d_.o.height, 16)), 256, 0, stream_.get()>>>(d_, T, bo, dout_i);
      else if (peer) k_raycast_shared<false, false, true><<<grid8, 64, 0, stream_.get()>>>(d_, T, bo, dout_i, keys);
      else if (slab && fast_div_) k_raycast_shared<true, true, false><<<grid8, 64, 0, stream_.get()>>>(d_, T, bo, dout_i, keys);
      else if (slab) k_raycast_shared<true, false, false><<<grid8, 64, 0, stream_.get()>>>(d_, T, bo, dout_i, keys);
      else if (fast_div_) k_raycast_shared<false, true, false><<<grid8, 64, 0, stream_.get()>>>(d_, T, bo, dout_i, keys);
      else k_raycast_shared<false, false, false><<<grid8, 64, 0, stream_.get()>>>(d_, T, bo, dout_i, keys);
      TDM_CUDA(cudaGetLastError());
    }
    if (copy_back && !slab_exchange_) {   // slab exchange mode: the per-slab render is only an operand of the exchange step
      TDM_CUDA(cudaMemcpyAsync(h_bgr_out_[free_half_].get(), d_bgr_out_.get(), npx * 3 * n, cudaMemcpyDeviceToHost, stream_.get()));
      TDM_CUDA(cudaMemcpyAsync(h_depth_out_[free_half_].get(), d_depth_out_.get(), npx * 4 * n, cudaMemcpyDeviceToHost, stream_.get()));
    }
  }
  static constexpr int kMeshGrid = 132 * 8;   // 8 CTAs per SM of an H100 SXM
  // count + scan + emit + total on stream_ (no host sync)
  void launch_mesh_all() {
    TDM_CUDA(cudaEventRecord(ev_mesh0_.get(), stream_.get()));
    k_mesh<false><<<kMeshGrid, 256, 0, stream_.get()>>>(d_, mesh_axes_, d_mesh_counts_.get(), nullptr, 0, nullptr, nullptr);
    TDM_CUDA(cudaGetLastError());
    k_mesh_scan<<<1, 1024, 0, stream_.get()>>>(d_mesh_counts_.get(), d_mesh_offsets_.get(), d_.counters, d_.o.num_blocks, d_mesh_total_.get());
    TDM_CUDA(cudaGetLastError());
    launch_mesh_emit();
    TDM_CUDA(cudaMemcpyAsync(h_mesh_total_.get(), d_mesh_total_.get(), sizeof(int), cudaMemcpyDeviceToHost, stream_.get()));
    TDM_CUDA(cudaEventRecord(ev_mesh1_.get(), stream_.get()));
  }
  void start_mesh(const float* lower, const float* upper) {
    TDM_CUDA(cudaSetDevice(device_));
    const int nblk = d_.o.num_blocks;
    if (!d_mesh_counts_) {   // set last: the group is complete once it is
      DevPtr<int> counts = make_dev<int>((size_t)nblk * sizeof(int));
      d_mesh_offsets_ = make_dev<int>((size_t)nblk * sizeof(int));
      d_mesh_total_ = make_dev<int>(sizeof(int));
      h_mesh_total_ = make_host<int>(sizeof(int));
      ev_mesh0_ = make_event();
      ev_mesh1_ = make_event();
      d_mesh_counts_ = std::move(counts);
    }
    // per-axis tables -> one device buffer: [cells x | cells y | cells z | ranges x | ranges y | ranges z]
    MeshAxisHost A[3];
    size_t bytes = 0;
    bool empty = false;
    for (int a = 0; a < 3; ++a) {
      A[a] = build_mesh_axis(lower[a], upper[a], d_.o.voxel_size);
      empty = empty || A[a].cells.empty();
      bytes += A[a].cells.size() * sizeof(MeshAxisCell) + A[a].ranges.size() * sizeof(int2) + 64;
      mesh_lower_[a] = lower[a];
      mesh_upper_[a] = upper[a];
    }
    TDM_CHECK(d_.slab_lo == INT_MIN && d_.slab_hi == INT_MAX,
              "mesh extraction of a Z-slab-partitioned volume is not supported (cells at slab faces would be emitted by two ranks)");
    mesh_empty_ = empty;
    mesh_epoch_ = volume_epoch_;
    *h_mesh_total_ = 0;
    if (empty) return;
    if (bytes > mesh_tables_cap_) {
      d_mesh_tables_.reset();
      mesh_tables_cap_ = 0;
      d_mesh_tables_ = make_dev<char>(bytes);
      mesh_tables_cap_ = bytes;
    }
    std::vector<char> host(bytes, 0);
    size_t off = 0;
    for (int a = 0; a < 3; ++a) {
      const size_t nb = A[a].cells.size() * sizeof(MeshAxisCell);
      std::memcpy(host.data() + off, A[a].cells.data(), nb);
      mesh_axes_.cells[a] = reinterpret_cast<const MeshAxisCell*>(d_mesh_tables_.get() + off);
      off += (nb + 15) / 16 * 16;
    }
    for (int a = 0; a < 3; ++a) {
      const size_t nb = A[a].ranges.size() * sizeof(int2);
      std::memcpy(host.data() + off, A[a].ranges.data(), nb);
      mesh_axes_.brange[a] = reinterpret_cast<const int2*>(d_mesh_tables_.get() + off);
      off += (nb + 15) / 16 * 16;
      mesh_axes_.bmin[a] = A[a].bmin;
      mesh_axes_.nb[a] = A[a].nb;
    }
    TDM_CUDA(cudaMemcpyAsync(d_mesh_tables_.get(), host.data(), off, cudaMemcpyHostToDevice, stream_.get()));  // pageable: staged before return
    if (!d_mesh_vert_) {   // first estimate (72 B per triangle, 2 M triangles = 151 MB); finish_mesh grows it when the count says so
      const char* init = getenv("TDM_MESH_INIT_TRIS");
      grow_mesh_buffers(init && atoll(init) > 0 ? atoll(init) : (1 << 21));
    }
    launch_mesh_all();
  }
  // waits for the extraction, grows the output buffers if the count says so, copies out; returns the vertex count
  long long finish_mesh(float* vert, float* cols, size_t max_vertices, bool query_only) {
    if (mesh_empty_) { mesh_ms_ = 0.f; return 0; }
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaEventSynchronize(ev_mesh1_.get()));
    TDM_CUDA(cudaEventElapsedTime(&mesh_ms_, ev_mesh0_.get(), ev_mesh1_.get()));
    long long ntri = *h_mesh_total_;
    // (also for a count-only query: the count handed out must be the count of the mesh the copy call will deliver)
    // First estimate too small: grow and run the extraction again.  The per-block counts / offsets of the first run are
    // only valid for the volume they were counted on; scans may have been integrated since ExtractMeshAsync (the call-order
    // state machine allows a whole Integrate -> Render -> GetRenderResult cycle in between), so count + scan + emit are all
    // redone, and once more should the newer volume need even more room.
    for (int attempt = 0; ntri > mesh_cap_tris_; ++attempt) {
      TDM_CHECK(attempt < 4, "mesh output kept outgrowing its buffers");
      grow_mesh_buffers(ntri + ntri / 4);
      launch_mesh_all();
      TDM_CUDA(cudaEventSynchronize(ev_mesh1_.get()));
      float again = 0.f;
      TDM_CUDA(cudaEventElapsedTime(&again, ev_mesh0_.get(), ev_mesh1_.get()));
      mesh_ms_ += again;
      ntri = *h_mesh_total_;
      mesh_epoch_ = volume_epoch_;
    }
    if (query_only) return 3 * ntri;
    const long long nv = 3 * ntri;
    if ((unsigned long long)nv > (unsigned long long)max_vertices)
      throw Error("Did not provide enough storage for mesh. (tsdf_volume.cu:796-799)");
    if (nv > 0) {
      TDM_CHECK(vert && cols, "null mesh output buffers");
      TDM_CUDA(cudaMemcpy(vert, d_mesh_vert_.get(), (size_t)nv * 3 * sizeof(float), cudaMemcpyDeviceToHost));
      TDM_CUDA(cudaMemcpy(cols, d_mesh_cols_.get(), (size_t)nv * 3 * sizeof(float), cudaMemcpyDeviceToHost));
    }
    return nv;
  }
  void grow_mesh_buffers(long long tris) {
    d_mesh_vert_.reset(); d_mesh_cols_.reset();
    mesh_cap_tris_ = 0;
    d_mesh_vert_ = make_dev<float>((size_t)tris * 9 * sizeof(float));
    d_mesh_cols_ = make_dev<float>((size_t)tris * 9 * sizeof(float));
    mesh_cap_tris_ = (int)std::min<long long>(tris, INT_MAX);
  }
  void launch_mesh_emit() {
    k_mesh<true><<<kMeshGrid, 256, 0, stream_.get()>>>(d_, mesh_axes_, d_mesh_counts_.get(), d_mesh_offsets_.get(), mesh_cap_tris_, d_mesh_vert_.get(), d_mesh_cols_.get());
    TDM_CUDA(cudaGetLastError());
  }
  void fetch_counters() {
    TDM_CUDA(cudaSetDevice(device_));
    TDM_CUDA(cudaMemcpyAsync(h_counters_.get(), d_.counters, 8 * sizeof(int), cudaMemcpyDeviceToHost, stream_.get()));
    TDM_CUDA(cudaStreamSynchronize(stream_.get()));
  }

  enum Next { kIntegrate, kRender, kGet };
  int device_;
  FusionDev d_{};
  long long n_entries_ = 0;
  Stream stream_;
  DevPtr<unsigned long long> keys_;   // the hash table and voxel pool d_ points at
  DevPtr<int> ptrs_, counters_, bbox_;
  DevPtr<uint2> voxels_;
  DevPtr<int4> list_;
  Event ev_int_, ev_render_;
  HostPtr<unsigned char> h_bgr_in_;
  DevPtr<unsigned char> d_bgr_in_;
  HostPtr<float> h_depth_in_;
  DevPtr<float> d_depth_in_;
  HostPtr<unsigned char> h_bgr_out_[2];
  HostPtr<float> h_depth_out_[2];
  DevPtr<unsigned char> d_bgr_out_;
  DevPtr<float> d_depth_out_;
  HostPtr<int> h_counters_;
  int free_half_ = 0;
  Mat4 pose_{}, pose_inv_{};
  std::vector<Mat4> render_poses_;
  int n_rendered_ = 0;
  bool have_scan_ = false;
  Next next_ = kIntegrate;
  bool raycast_shared_ = true;   // false: the reference-shaped comparator k_raycast
  bool fast_div_ok_ = false, fast_div_ = false;   // constant-divisor division in the ray-cast (cdiv_): bit-identical, 3 instructions per division
  std::vector<void*> ipc_opened_;   // peers' allocations mapped with cudaIpcOpenMemHandle (closed in the destructor)
  bool slab_clip_ = true;        // Z-slab volumes: rays are only sampled inside the slab's z range (bit-identical, see k_raycast_shared)
  bool slab_exchange_ = false;   // Z-slab volumes: the ray-cast emits packed nearest-hit keys for the exchange step, the per-slab
                                 // render is not copied back and GetRenderResult does not wait (tandem_b200.parallel)
  DevPtr<int> d_vis_list_;
  float last_alloc_ms_ = 0.f;
  DevPtr<long long> d_hit_keys_;
  DevPtr<float> d_unpack_depth_;
  DevPtr<unsigned char> d_unpack_bgr_;
  // mesh extraction state
  DevPtr<char> d_mesh_tables_;
  size_t mesh_tables_cap_ = 0;
  MeshAxes mesh_axes_{};
  DevPtr<int> d_mesh_counts_, d_mesh_offsets_, d_mesh_total_;
  HostPtr<int> h_mesh_total_;
  DevPtr<float> d_mesh_vert_, d_mesh_cols_;
  int mesh_cap_tris_ = 0;
  Event ev_mesh0_, ev_mesh1_;
  enum MeshKind { kMeshNone, kMeshAsync, kMeshBlocking };
  MeshKind mesh_kind_ = kMeshNone;   // who owns the extraction sitting in the device buffers
  bool mesh_empty_ = false;
  float mesh_lower_[3] = {0, 0, 0}, mesh_upper_[3] = {0, 0, 0};
  unsigned long long volume_epoch_ = 0, mesh_epoch_ = 0;   // scans integrated so far / at the time of the extraction
  float mesh_ms_ = 0.f;
};

FusionIface* make_fusion(const tdm_fusion_options& o, int device) { return new FusionImpl(o, device); }

// host-only view of the hash function the kernels use (division-free remainder) beside the reference's expression
int hash_slot_host(int x, int y, int z, int num_buckets, int* reference_expression) {
  if (num_buckets <= 0) return -1;
  const unsigned long long magic = 0xFFFFFFFFFFFFFFFFull / (unsigned long long)num_buckets + 1ull;
  const unsigned c32 = (unsigned)((1ull << 32) % (unsigned long long)num_buckets);
  if (reference_expression) {   // hash_table.cu:157-168 as written
    const int a = (int)((unsigned)x * 73856093u), b = (int)((unsigned)y * 19349669u), c = (int)((unsigned)z * 83492791u);
    int r = (a ^ b ^ c) % num_buckets;
    if (r < 0) r += num_buckets;
    *reference_expression = r;
  }
  return hash_slot(x, y, z, num_buckets, magic, c32);
}

// host-only view of the mesh extractor's per-axis table (no GPU involved; used by the CPU test-suite)
int mesh_axis_table(float lower, float upper, float voxel_size, int* ints5, float* floats4, int* ranges2, int* bmin, int cap) {
  const MeshAxisHost A = build_mesh_axis(lower, upper, voxel_size);
  const int n = (int)A.cells.size();
  for (int i = 0; i < n && i < cap; ++i) {
    const MeshAxisCell& c = A.cells[i];
    ints5[5 * i] = c.gMA; ints5[5 * i + 1] = c.gMB; ints5[5 * i + 2] = c.gPA; ints5[5 * i + 3] = c.gPB; ints5[5 * i + 4] = c.gC;
    floats4[4 * i] = c.wM; floats4[4 * i + 1] = c.wP; floats4[4 * i + 2] = c.cM; floats4[4 * i + 3] = c.cP;
  }
  for (int b = 0; b < A.nb && b < cap; ++b) { ranges2[2 * b] = A.ranges[b].x; ranges2[2 * b + 1] = A.ranges[b].y; }
  if (bmin) { bmin[0] = A.bmin; bmin[1] = A.nb; }
  return n;
}

}  // namespace tdm
