// Marching-cubes mesh extraction behind DrFusion::ExtractMeshAsync / GetMeshSync / GetMesh (SURVEY.md §8f row n4).
// Included by fusion.cu inside namespace tdm { namespace { ... } } (uses FusionDev, find_block, the __f*_rn helpers).
//
// Reference being replaced:
//   ExtractMeshKernel / ExtractMeshAtPosition   tandem/libdr/dr_fusion/src/marching_cubes/mesh_extractor.cu:137-265
//   TrilinearInterpolation / VertexInterpolation mesh_extractor.cu:24-104, 106-135
//   Mesh::AppendTriangle (atomicAdd append)      marching_cubes/mesh.cu:21-24
//   TsdfVolume::GetMeshSync (host copy loop)     tsdfvh/tsdf_volume.cu:781-839
// The reference brute-forces every cell of the bounding box (10 m cube at 1 cm = 1e9 cells, tandem_backend.cpp:80-81)
// with 65 hash probes per surviving cell, appends 72-byte triangles to managed memory through one global atomic and
// re-packs them on the host one triangle at a time.
//
// Design (block-sparse, two passes, no global atomics):
//   * every quantity a cell needs is SEPARABLE per axis (cell position, the +-s/2 corner coordinates, the two voxel
//     indices and the trilinear weight of each corner sample, the centre voxel index), so the host evaluates three small
//     per-axis tables once per call with exactly the reference's fp32 expression sequence;
//   * a cell can only emit triangles if the FIRST voxel its p000 sample reads is allocated (mesh_extractor.cu:146-149
//     fails otherwise), and that voxel index is monotone in the cell index, so every allocated voxel block owns a
//     contiguous box of cells: one CTA per block of the compact block list, nothing else is visited;
//   * the CTA stages the 12^3 voxel neighbourhood (its block + the 7 positive neighbours, 8 hash probes per block instead
//     of 65 per cell) in shared memory, classifies its <= 9^3 cells, and
//     pass 1 writes the block's triangle count, a single-CTA scan turns counts into offsets, pass 2 re-classifies and
//     writes vertices / colours straight in the GetMeshSync layout (xyz and rgb float triples) at deterministic offsets.
// Arithmetic: identical sequence to oracle/tsdf_oracle.c (fmaf where the reference's nvcc build contracts a*b+c,
// __f*_rn everywhere else) -> the triangle set is bit-identical to the oracle's.
#pragma once

#include "mc_tables.h"

struct MeshAxisCell {   // one cell index along one axis
  int gMA, gMB;         // voxel indices read by the corner sample at pos - s/2 (pos_dual + 0, pos_dual + s)
  int gPA, gPB;         // ... at pos + s/2
  int gC;               // voxel index of the cell position itself (colour lookup, mesh_extractor.cu:200)
  float wM, wP;         // trilinear weight frac(corner / s) of the two corner samples
  float cM, cP;         // corner coordinates pos -+ s/2
};

struct MeshAxes {
  const MeshAxisCell* cells[3];
  const int2* brange[3];   // per block coordinate b - bmin[a]: {first cell, #cells} whose gMA lies in block b
  int bmin[3], nb[3];
};

constexpr int kMeshTile = 12;                 // voxels per axis staged per block (8 + reach of 3, +1 slack)
constexpr int kMeshTileVox = kMeshTile * kMeshTile * kMeshTile;
constexpr unsigned long long kMeshEdgeA = 0x321076543210ull;   // edge e joins corners A[e] -> B[e] (mesh_extractor.cu:203-237)
constexpr unsigned long long kMeshEdgeB = 0x765447650321ull;
// cube corners in the reference's bit order (mesh_extractor.cu:188-196): 010,110,100,000,011,111,101,001
constexpr unsigned kMeshCornerX = 0x66, kMeshCornerY = 0x33, kMeshCornerZ = 0xF0;   // bit c = 1 -> the +s/2 side

struct MeshCellCtx {
  int ox[4], oy[4], oz[4];   // tile offsets of the 4 voxel indices per axis: [side*2 + {A,B}], pre-multiplied
  float wx[2], wy[2], wz[2];
};

// dist of the eight cube corners + cube index; false if any of the 64 voxel reads has weight 0 (mesh_extractor.cu:24-104)
__device__ __forceinline__ bool mesh_classify(const uint2* __restrict__ tile, const MeshCellCtx& c, float (&dist)[8], int& cube) {
  cube = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int sx = (kMeshCornerX >> k) & 1, sy = (kMeshCornerY >> k) & 1, sz = (kMeshCornerZ >> k) & 1;
    const float wx = c.wx[sx], wy = c.wy[sy], wz = c.wz[sz];
    const float ux = sub_(1.0f, wx), uy = sub_(1.0f, wy), uz = sub_(1.0f, wz);
    float d = 0.0f;
    // sample order of the reference: 000,100,010,001,110,011,101,111
    constexpr int qx[8] = {0, 1, 0, 0, 1, 0, 1, 1}, qy[8] = {0, 0, 1, 0, 1, 1, 0, 1}, qz[8] = {0, 0, 0, 1, 0, 1, 1, 1};
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const uint2 v = tile[c.ox[sx * 2 + qx[q]] + c.oy[sy * 2 + qy[q]] + c.oz[sz * 2 + qz[q]]];
      if ((v.y >> 24) == 0) return false;
      const float W = mul_(mul_(qx[q] ? wx : ux, qy[q] ? wy : uy), qz[q] ? wz : uz);
      d = __fmaf_rn(W, __uint_as_float(v.x), d);
    }
    dist[k] = d;
    if (d < 0.0f) cube |= 1 << k;
  }
  return true;
}

__device__ __forceinline__ int mesh_tri_count(unsigned long long tri) {
  int n = 0;
#pragma unroll
  for (int k = 0; k < 15; k += 3) n += ((tri >> (4 * k)) & 0xF) != 0xF;
  return n;
}

template <bool EMIT>
__global__ void __launch_bounds__(256)
k_mesh(FusionDev d, MeshAxes ax, int* __restrict__ counts, const int* __restrict__ offsets, int capacity_tris,
       float* __restrict__ vert, float* __restrict__ cols) {
  __shared__ uint2 tile[kMeshTileVox];
  __shared__ int sptr[8];
  __shared__ int swarp[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nblocks = min(d.counters[0], d.o.num_blocks);
  for (int b = blockIdx.x; b < nblocks; b += gridDim.x) {
    if (EMIT && counts[b] == 0) continue;
    const int4 e = d.list[b];
    const int bx = e.x - ax.bmin[0], by = e.y - ax.bmin[1], bz = e.z - ax.bmin[2];
    int2 rx = make_int2(0, 0), ry = rx, rz = rx;
    if (bx >= 0 && bx < ax.nb[0] && by >= 0 && by < ax.nb[1] && bz >= 0 && bz < ax.nb[2]) {
      rx = ax.brange[0][bx]; ry = ax.brange[1][by]; rz = ax.brange[2][bz];
    }
    const int ncell = rx.y * ry.y * rz.y;
    if (ncell == 0) {
      if (!EMIT && tid == 0) counts[b] = 0;
      continue;
    }
    __syncthreads();   // the previous block's tile is no longer read
    if (tid < 8) sptr[tid] = tid == 0 ? e.w : find_block(d, e.x + (tid >> 2), e.y + ((tid >> 1) & 1), e.z + (tid & 1));
    __syncthreads();
    int neg = 0;
    for (int t = tid; t < kMeshTileVox; t += 256) {
      const int tx = t / (kMeshTile * kMeshTile), ty = (t / kMeshTile) % kMeshTile, tz = t % kMeshTile;
      const int ptr = sptr[(tx >> 3) * 4 + (ty >> 3) * 2 + (tz >> 3)];
      const uint2 v = ptr < 0 ? make_uint2(0u, 0u) : __ldg(d.voxels + (size_t)ptr * 512 + (tx & 7) * 64 + (ty & 7) * 8 + (tz & 7));
      tile[t] = v;
      neg |= (v.y >> 24) != 0 && __uint_as_float(v.x) < 0.0f;
    }
    // Every corner distance is a chain of fma(W, sdf, acc) with W >= 0: if no observed voxel of the neighbourhood is negative,
    // every distance is >= +0, the cube index is 0 and the block emits nothing - skip it (most blocks of the viewing frustum
    // are free space with sdf = +truncation).  The all-negative case is NOT skipped (a -0 sum would read as "not below").
    if (!__syncthreads_or(neg)) {
      if (!EMIT && tid == 0) counts[b] = 0;
      continue;
    }
    const int t0x = e.x * 8, t0y = e.y * 8, t0z = e.z * 8;
    int running = EMIT ? offsets[b] : 0;   // EMIT: first triangle slot of this round; COUNT: per-thread sum
    for (int base = 0; base < ncell; base += 256) {
      const int cell = base + tid;
      int ntri = 0, cube = 0;
      float dist[8];
      MeshCellCtx c;
      MeshAxisCell cx, cy, cz;
      unsigned long long tri = ~0ull;
      if (cell < ncell) {
        const int ix = cell % rx.y, iy = (cell / rx.y) % ry.y, iz = cell / (rx.y * ry.y);
        cx = ax.cells[0][rx.x + ix]; cy = ax.cells[1][ry.x + iy]; cz = ax.cells[2][rz.x + iz];
        c.ox[0] = (cx.gMA - t0x) * kMeshTile * kMeshTile; c.ox[1] = (cx.gMB - t0x) * kMeshTile * kMeshTile;
        c.ox[2] = (cx.gPA - t0x) * kMeshTile * kMeshTile; c.ox[3] = (cx.gPB - t0x) * kMeshTile * kMeshTile;
        c.oy[0] = (cy.gMA - t0y) * kMeshTile; c.oy[1] = (cy.gMB - t0y) * kMeshTile;
        c.oy[2] = (cy.gPA - t0y) * kMeshTile; c.oy[3] = (cy.gPB - t0y) * kMeshTile;
        c.oz[0] = cz.gMA - t0z; c.oz[1] = cz.gMB - t0z; c.oz[2] = cz.gPA - t0z; c.oz[3] = cz.gPB - t0z;
        c.wx[0] = cx.wM; c.wx[1] = cx.wP; c.wy[0] = cy.wM; c.wy[1] = cy.wP; c.wz[0] = cz.wM; c.wz[1] = cz.wP;
        if (mesh_classify(tile, c, dist, cube)) {
          tri = kMcTri[cube];
          ntri = mesh_tri_count(tri);
        }
      }
      if (!EMIT) {
        running += ntri;
        continue;
      }
      // exclusive scan of ntri over the 256 threads of this round
      int incl = ntri;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      __syncthreads();   // swarp of the previous round consumed
      if (lane == 31) swarp[warp] = incl;
      __syncthreads();
      int before = 0, total = 0;
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        const int s = swarp[w];
        if (w < warp) before += s;
        total += s;
      }
      int slot = running + before + incl - ntri;
      running += total;
      if (ntri == 0) continue;
      const uint2 vc = tile[(cx.gC - t0x) * kMeshTile * kMeshTile + (cy.gC - t0y) * kMeshTile + (cz.gC - t0z)];
      const float r = div_((float)((vc.y >> 16) & 0xFF), 255.f), g = div_((float)((vc.y >> 8) & 0xFF), 255.f),
                  bl = div_((float)(vc.y & 0xFF), 255.f);   // GetMeshSync writes colour z,y,x = R,G,B (tsdf_volume.cu:805-807)
      for (int k = 0; k < 15; ++k) {
        const int ed = (int)((tri >> (4 * k)) & 0xF);
        if (ed == 0xF) break;
        if (slot + k / 3 >= capacity_tris) break;   // output buffer too small: the host re-runs with a larger one
        const int ca = (int)((kMeshEdgeA >> (4 * ed)) & 0xF), cb = (int)((kMeshEdgeB >> (4 * ed)) & 0xF);
        const float ax_ = (kMeshCornerX >> ca) & 1 ? cx.cP : cx.cM, ay_ = (kMeshCornerY >> ca) & 1 ? cy.cP : cy.cM,
                    az_ = (kMeshCornerZ >> ca) & 1 ? cz.cP : cz.cM;
        const float bx_ = (kMeshCornerX >> cb) & 1 ? cx.cP : cx.cM, by_ = (kMeshCornerY >> cb) & 1 ? cy.cP : cy.cM,
                    bz_ = (kMeshCornerZ >> cb) & 1 ? cz.cP : cz.cM;
        float d1 = 0.f, d2 = 0.f;
#pragma unroll
        for (int q = 0; q < 8; ++q) {   // register-resident select instead of a dynamically indexed array
          if (q == ca) d1 = dist[q];
          if (q == cb) d2 = dist[q];
        }
        float px, py, pz;
        if (fabsf(sub_(0.0f, d1)) < 0.00001f) { px = ax_; py = ay_; pz = az_; }            // mesh_extractor.cu:113-115
        else if (fabsf(sub_(0.0f, d2)) < 0.00001f) { px = bx_; py = by_; pz = bz_; }
        else if (fabsf(sub_(d1, d2)) < 0.00001f) { px = ax_; py = ay_; pz = az_; }
        else {
          const float mu = div_(sub_(0.0f, d1), sub_(d2, d1));
          px = __fmaf_rn(mu, sub_(bx_, ax_), ax_); py = __fmaf_rn(mu, sub_(by_, ay_), ay_); pz = __fmaf_rn(mu, sub_(bz_, az_), az_);
        }
        const size_t o = ((size_t)slot * 3 + k) * 3;   // vertex index = 3*triangle + k%3, and k/3 advances the triangle
        vert[o] = px; vert[o + 1] = py; vert[o + 2] = pz;
        cols[o] = r; cols[o + 1] = g; cols[o + 2] = bl;
      }
    }
    if (!EMIT) {
      // block total
      int v = running;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      __syncthreads();
      if (lane == 0) swarp[warp] = v;
      __syncthreads();
      if (tid == 0) {
        int t = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) t += swarp[w];
        counts[b] = t;
      }
    }
  }
}

// exclusive scan of the per-block triangle counts (<= num_blocks ints), one CTA; total -> out_total[0]
__global__ void __launch_bounds__(1024) k_mesh_scan(const int* __restrict__ counts, int* __restrict__ offsets, const int* __restrict__ n_ptr,
                                                    int n_cap, int* __restrict__ out_total) {
  __shared__ int ssum[1024];
  const int n = min(*n_ptr, n_cap);
  const int tid = threadIdx.x;
  const int per = (n + 1023) / 1024;
  const int lo = min(tid * per, n), hi = min(lo + per, n);
  int s = 0;
  for (int i = lo; i < hi; ++i) s += counts[i];
  ssum[tid] = s;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const int v = tid >= o ? ssum[tid - o] : 0;
    __syncthreads();
    ssum[tid] += v;
    __syncthreads();
  }
  int run = ssum[tid] - s;
  for (int i = lo; i < hi; ++i) { offsets[i] = run; run += counts[i]; }
  if (tid == 1023) out_total[0] = ssum[1023];
}
