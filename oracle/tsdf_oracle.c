/* ORACLE (test infrastructure - never linked into, or called by, the product library).
 *
 * Sequential CPU restatement of TANDEM's voxel-hashed TSDF (libdr/dr_fusion, a ReFusion derivative):
 *   coordinate maps        tsdfvh/tsdf_volume.cu:103-145
 *   GetVoxel / trilinear   tsdf_volume.cu:147-159, 161-289
 *   UpdateVoxel / Combine  tsdf_volume.cu:303-315, tsdfvh/voxel.h:29-53
 *   allocation DDA         tsdf_volume.cu:317-434, hash_table.cu:80-115 (AllocateBlock), :157-168 (Hash)
 *   integrate              tsdf_volume.cu:436-513
 *   ray-cast               tsdf_volume.cu:600-632
 *   GetPoint3d / Project   utils/utils.h:93-108
 * PARITY UNPINNED: the reference ships no golden data or test for DrFusion (SURVEY.md §4), and its CUDA code
 * cannot run in the build container.  This file therefore *defines* the deterministic semantics we hold the
 * CUDA path to (SURVEY.md Appendix B): blocks are allocated in pixel-raster / DDA order with the reference's
 * bucket hash (a full bucket drops the block), free hash entries are not integrated, every voxel of a block is
 * updated at most once per scan.  fp32 arithmetic is evaluated without FMA contraction (compile with
 * -ffp-contract=off); the CUDA kernels use __f*_rn intrinsics for the same expressions so that the integer
 * decisions (pixel indices, voxel indices, weights) are bit-identical.
 * Deviations from the letter of the reference, all documented in DESIGN.md: the camera-pose inverse is a
 * 2x2-sub-determinant fp32 inverse (not the 16-cofactor one, matrix_utils.h:958-1080); a voxel whose camera
 * z is exactly 0 is skipped (the reference divides by it); a NaN depth pixel is ignored (the reference's allocation DDA
 * never ends on one).
 */
#include <math.h>
#include <float.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { float x, y, z; } f3;
typedef struct { int x, y, z; } i3;
typedef struct { float sdf; unsigned char c[3]; unsigned char w; } Voxel; /* 8 bytes, voxel.h:13-21 */

typedef struct {
  float voxel_size; int num_buckets, bucket_size, num_blocks, block_size, max_sdf_weight;
  float truncation_distance, max_sensor_depth, min_sensor_depth; int num_render_streams;
  float fx, fy, cx, cy; int height, width;
} Options; /* == DrFusionOptions, dr_fusion.h:18-36 */

typedef struct { i3 pos; int ptr; } Entry; /* hash_entry.h; ptr -1 = free */

typedef struct {
  Options o;
  Entry* entries; long n_entries;
  Voxel* voxels;  /* num_blocks * 512 */
  int heap_next;
  long allocated, dropped, last_visible, last_candidates;
  unsigned char* touched; /* per-voxel flag for the ray-cast distinct-voxel counter */
  long last_render_distinct_voxels;
} Tsdf;

/* ---- float4x4 helpers (row-major), fp32 ---- */
static f3 xform(const float* m, f3 v) { /* matrix_utils.h:914-921: w assumed 1 */
  f3 r;
  r.x = m[0] * v.x + m[1] * v.y + m[2] * v.z + m[3] * 1.0f;
  r.y = m[4] * v.x + m[5] * v.y + m[6] * v.z + m[7] * 1.0f;
  r.z = m[8] * v.x + m[9] * v.y + m[10] * v.z + m[11] * 1.0f;
  return r;
}
/* general 4x4 inverse through 2x2 sub-determinants, fp32 (same routine as tandem_b200/csrc/mat4.h) */
static int inv4(const float* m, float* o) {
  float s0 = m[0] * m[5] - m[4] * m[1], s1 = m[0] * m[6] - m[4] * m[2], s2 = m[0] * m[7] - m[4] * m[3];
  float s3 = m[1] * m[6] - m[5] * m[2], s4 = m[1] * m[7] - m[5] * m[3], s5 = m[2] * m[7] - m[6] * m[3];
  float c5 = m[10] * m[15] - m[14] * m[11], c4 = m[9] * m[15] - m[13] * m[11], c3 = m[9] * m[14] - m[13] * m[10];
  float c2 = m[8] * m[15] - m[12] * m[11], c1 = m[8] * m[14] - m[12] * m[10], c0 = m[8] * m[13] - m[12] * m[9];
  float det = s0 * c5 - s1 * c4 + s2 * c3 + s3 * c2 - s4 * c1 + s5 * c0;
  if (det == 0.0f) return 0;
  float id = 1.0f / det;
  o[0] = (m[5] * c5 - m[6] * c4 + m[7] * c3) * id;
  o[1] = (-m[1] * c5 + m[2] * c4 - m[3] * c3) * id;
  o[2] = (m[13] * s5 - m[14] * s4 + m[15] * s3) * id;
  o[3] = (-m[9] * s5 + m[10] * s4 - m[11] * s3) * id;
  o[4] = (-m[4] * c5 + m[6] * c2 - m[7] * c1) * id;
  o[5] = (m[0] * c5 - m[2] * c2 + m[3] * c1) * id;
  o[6] = (-m[12] * s5 + m[14] * s2 - m[15] * s1) * id;
  o[7] = (m[8] * s5 - m[10] * s2 + m[11] * s1) * id;
  o[8] = (m[4] * c4 - m[5] * c2 + m[7] * c0) * id;
  o[9] = (-m[0] * c4 + m[1] * c2 - m[3] * c0) * id;
  o[10] = (m[12] * s4 - m[13] * s2 + m[15] * s0) * id;
  o[11] = (-m[8] * s4 + m[9] * s2 - m[11] * s0) * id;
  o[12] = (-m[4] * c3 + m[5] * c1 - m[6] * c0) * id;
  o[13] = (m[0] * c3 - m[1] * c1 + m[2] * c0) * id;
  o[14] = (-m[12] * s3 + m[13] * s1 - m[14] * s0) * id;
  o[15] = (m[8] * s3 - m[9] * s1 + m[10] * s0) * id;
  return 1;
}

static float norm3(f3 v) { return sqrtf(v.x * v.x + v.y * v.y + v.z * v.z); } /* utils.h:44-46 */
static int sgn(float n) { return (n > 0) - (n < 0); }

static f3 get_point3d(const Options* o, int i, float depth) { /* utils.h:93-101 */
  int v = i / o->width, u = i - o->width * v;
  f3 p;
  p.z = depth;
  p.x = ((float)u - o->cx) * p.z / o->fx;
  p.y = ((float)v - o->cy) * p.z / o->fy;
  return p;
}
static int to_int_sat(float f) { /* CUDA float->int conversion semantics (saturating, NaN -> 0) */
  if (f != f) return 0;
  if (f >= 2147483648.0f) return 2147483647;
  if (f <= -2147483648.0f) return (-2147483647 - 1);
  return (int)f;
}
static void project(const Options* o, f3 p, int* px, int* py) { /* utils.h:103-108 */
  float x = (o->fx * p.x) / p.z + o->cx;
  float y = (o->fy * p.y) / p.z + o->cy;
  *px = to_int_sat(roundf(x));
  *py = to_int_sat(roundf(y));
}

/* ---- hash (hash_table.cu:157-168): int32 wrap-around arithmetic ---- */
static long hash_bucket(const Tsdf* t, i3 p) {
  int32_t a = (int32_t)((uint32_t)p.x * 73856093u), b = (int32_t)((uint32_t)p.y * 19349669u),
          c = (int32_t)((uint32_t)p.z * 83492791u);
  int32_t r = (a ^ b ^ c) % t->o.num_buckets;
  if (r < 0) r += t->o.num_buckets;
  return (long)r * t->o.bucket_size;
}
static int find_entry(const Tsdf* t, i3 p) { /* hash_table.cu:141-155 */
  long b = hash_bucket(t, p);
  for (int i = 0; i < t->o.bucket_size; ++i) {
    const Entry* e = &t->entries[b + i];
    if (e->ptr != -1 && e->pos.x == p.x && e->pos.y == p.y && e->pos.z == p.z) return e->ptr;
  }
  return -1;
}
static void allocate_block(Tsdf* t, i3 p) { /* hash_table.cu:80-115, sequential semantics */
  long b = hash_bucket(t, p);
  long free_idx = -1;
  for (int i = 0; i < t->o.bucket_size; ++i) {
    Entry* e = &t->entries[b + i];
    if (e->ptr != -1 && e->pos.x == p.x && e->pos.y == p.y && e->pos.z == p.z) return;
    if (free_idx < 0 && e->ptr == -1) free_idx = b + i;
  }
  if (free_idx < 0 || t->heap_next >= t->o.num_blocks) { t->dropped++; return; }
  t->entries[free_idx].pos = p;
  t->entries[free_idx].ptr = t->heap_next++;
  t->allocated++;
}

/* ---- coordinate maps (tsdf_volume.cu:109-145) ---- */
static float signf_(float v) { return (float)((v > 0) - (v < 0)); }
static i3 world_to_global_voxel(const Tsdf* t, f3 p) {
  i3 r;
  float s = t->o.voxel_size;
  r.x = (int)(p.x / s + signf_(p.x) * 0.5f);
  r.y = (int)(p.y / s + signf_(p.y) * 0.5f);
  r.z = (int)(p.z / s + signf_(p.z) * 0.5f);
  return r;
}
static int fdiv(int v, int b) { return v < 0 ? (v - b + 1) / b : v / b; }
static int pmod(int v, int b) { int m = v % b; return m < 0 ? m + b : m; }

static Voxel get_voxel(Tsdf* t, f3 p) { /* tsdf_volume.cu:147-159 */
  i3 g = world_to_global_voxel(t, p);
  int B = t->o.block_size;
  i3 blk = {fdiv(g.x, B), fdiv(g.y, B), fdiv(g.z, B)};
  int ptr = find_entry(t, blk);
  Voxel v;
  if (ptr < 0) { memset(&v, 0, sizeof v); return v; }
  long idx = (long)ptr * B * B * B + pmod(g.x, B) * B * B + pmod(g.y, B) * B + pmod(g.z, B);
  if (t->touched) t->touched[idx] = 1;
  return t->voxels[idx];
}

static Voxel get_interpolated(Tsdf* t, f3 p) { /* tsdf_volume.cu:161-289 */
  Voxel v0 = get_voxel(t, p);
  if (v0.w == 0) return v0;
  float s = t->o.voxel_size;
  f3 pd = {p.x - s / 2.0f, p.y - s / 2.0f, p.z - s / 2.0f};
  f3 vp = {p.x / s, p.y / s, p.z / s};
  float wx = vp.x - floorf(vp.x), wy = vp.y - floorf(vp.y), wz = vp.z - floorf(vp.z);
  float dist = 0.0f, cf[3] = {0, 0, 0};
  /* corner order of the reference: 000,100,010,001,110,011,101,111 */
  static const int ox[8] = {0, 1, 0, 0, 1, 0, 1, 1}, oy[8] = {0, 0, 1, 0, 1, 1, 0, 1}, oz[8] = {0, 0, 0, 1, 0, 1, 1, 1};
  for (int k = 0; k < 8; ++k) {
    f3 q = {pd.x + (ox[k] ? s : 0.0f), pd.y + (oy[k] ? s : 0.0f), pd.z + (oz[k] ? s : 0.0f)};
    Voxel v = get_voxel(t, q);
    const Voxel* src = (v.w == 0) ? &v0 : &v;
    float w = (ox[k] ? wx : 1.0f - wx) * (oy[k] ? wy : 1.0f - wy) * (oz[k] ? wz : 1.0f - wz);
    dist += w * src->sdf;
    for (int c = 0; c < 3; ++c) cf[c] = cf[c] + w * (float)src->c[c];
  }
  Voxel r;
  r.w = v0.w;
  r.sdf = dist;
  for (int c = 0; c < 3; ++c) r.c[c] = (unsigned char)cf[c];
  return r;
}

static void combine(Voxel* a, float sdf, const unsigned char* col, int max_w) { /* voxel.h:29-53, voxel.weight == 1 */
  float w = (float)a->w;
  for (int c = 0; c < 3; ++c) a->c[c] = (unsigned char)(((float)a->c[c] * w + (float)col[c] * 1.0f) / (w + 1.0f));
  a->sdf = (a->sdf * w + sdf * 1.0f) / (w + 1.0f);
  int nw = a->w + 1;
  a->w = (unsigned char)(nw > max_w ? max_w : nw);
}

/* ================= public API (ctypes) ================= */
Tsdf* tsdf_oracle_create(const Options* o) {
  Tsdf* t = (Tsdf*)calloc(1, sizeof(Tsdf));
  t->o = *o;
  t->n_entries = (long)o->num_buckets * o->bucket_size;
  t->entries = (Entry*)malloc(sizeof(Entry) * t->n_entries);
  for (long i = 0; i < t->n_entries; ++i) { t->entries[i].pos.x = t->entries[i].pos.y = t->entries[i].pos.z = 0; t->entries[i].ptr = -1; }
  long nv = (long)o->num_blocks * o->block_size * o->block_size * o->block_size;
  t->voxels = (Voxel*)calloc(nv, sizeof(Voxel));
  return t;
}
void tsdf_oracle_destroy(Tsdf* t) { if (!t) return; free(t->entries); free(t->voxels); free(t->touched); free(t); }

static void allocate_from_depth(Tsdf* t, const float* depth, const float* T) { /* tsdf_volume.cu:317-434 */
  const Options* o = &t->o;
  float bs = (float)o->block_size * o->voxel_size;
  f3 start = {T[3], T[7], T[11]};
  long before = t->allocated;
  int n = o->height * o->width;
  for (int i = 0; i < n; ++i) {
    /* documented deviation: NaN depth is rejected (the reference's `< min || > max` lets it into a DDA that never ends) */
    if (!(depth[i] >= o->min_sensor_depth && depth[i] <= o->max_sensor_depth)) continue;
    f3 pu = get_point3d(o, i, depth[i]);
    f3 p = xform(T, pu);
    if (p.x == 0 && p.y == 0 && p.z == 0) continue;
    f3 d = {p.x - start.x, p.y - start.y, p.z - start.z};
    float dn = norm3(d);
    f3 dir = {d.x / dn, d.y / dn, d.z / dn};
    float sd = dn; /* distance(start, point) */
    float len = sd + o->truncation_distance;
    f3 end = {start.x + dir.x * len, start.y + dir.y * len, start.z + dir.z * len};
    i3 bp = {(int)floorf(start.x / bs), (int)floorf(start.y / bs), (int)floorf(start.z / bs)};
    i3 be = {(int)floorf(end.x / bs), (int)floorf(end.y / bs), (int)floorf(end.z / bs)};
    i3 step = {sgn(dir.x), sgn(dir.y), sgn(dir.z)};
    f3 dt = {dir.x != 0 ? fabsf(bs / dir.x) : FLT_MAX, dir.y != 0 ? fabsf(bs / dir.y) : FLT_MAX,
             dir.z != 0 ? fabsf(bs / dir.z) : FLT_MAX};
    f3 bd = {((float)bp.x + (float)step.x) * bs, ((float)bp.y + (float)step.y) * bs, ((float)bp.z + (float)step.z) * bs};
    f3 mt = {dir.x != 0 ? (bd.x - start.x) / dir.x : FLT_MAX, dir.y != 0 ? (bd.y - start.y) / dir.y : FLT_MAX,
             dir.z != 0 ? (bd.z - start.z) / dir.z : FLT_MAX};
    i3 diff = {0, 0, 0};
    int neg = 0;
    if (bp.x != be.x && dir.x < 0) { diff.x--; neg = 1; }
    if (bp.y != be.y && dir.y < 0) { diff.y--; neg = 1; }
    if (bp.z != be.z && dir.z < 0) { diff.z--; neg = 1; }
    allocate_block(t, bp);
    if (neg) { bp.x += diff.x; bp.y += diff.y; bp.z += diff.z; allocate_block(t, bp); }
    int guard = 0;
    while ((bp.x != be.x || bp.y != be.y || bp.z != be.z) && guard++ < 100000) {
      if (mt.x < mt.y) {
        if (mt.x < mt.z) { bp.x += step.x; mt.x += dt.x; } else { bp.z += step.z; mt.z += dt.z; }
      } else {
        if (mt.y < mt.z) { bp.y += step.y; mt.y += dt.y; } else { bp.z += step.z; mt.z += dt.z; }
      }
      allocate_block(t, bp);
    }
  }
  t->last_candidates = t->allocated - before;
}

static void integrate(Tsdf* t, const unsigned char* bgr, const float* depth, const float* T, const float* Ti) {
  const Options* o = &t->o; /* tsdf_volume.cu:436-513 */
  int B = o->block_size;
  float vs = o->voxel_size, tau = o->truncation_distance;
  long vis = 0;
  for (long e = 0; e < t->n_entries; ++e) {
    if (t->entries[e].ptr == -1) continue; /* Appendix B.2: free entries are not integrated */
    i3 bp = t->entries[e].pos;
    f3 pos = {(float)bp.x * vs * (float)B, (float)bp.y * vs * (float)B, (float)bp.z * vs * (float)B};
    f3 pc = xform(Ti, pos);
    if (pc.z < 0) continue;
    double half = 0.5 * (double)vs * (double)B; /* double arithmetic as written, tsdf_volume.cu:460-463 */
    f3 ctr = {(float)((double)pc.x + half), (float)((double)pc.y + half), (float)((double)pc.z + half)};
    int px, py;
    project(o, ctr, &px, &py);
    if (!(px >= 0 && py >= 0 && px < o->width && py < o->height)) continue;
    vis++;
    Voxel* blk = t->voxels + (long)t->entries[e].ptr * B * B * B;
    for (int bx = 0; bx < B; ++bx)
      for (int by = 0; by < B; ++by)
        for (int bz = 0; bz < B; ++bz) {
          f3 vw = {pos.x + (float)bx * vs, pos.y + (float)by * vs, pos.z + (float)bz * vs};
          f3 vc = xform(Ti, vw);
          if (vc.z == 0.0f) continue; /* documented deviation: the reference divides by zero here */
          project(o, vc, &px, &py);
          if (!(px >= 0 && py >= 0 && px < o->width && py < o->height)) continue;
          int idx = py * o->width + px;
          float dz = depth[idx];
          if (!(dz > 0 && dz >= o->min_sensor_depth && dz <= o->max_sensor_depth)) continue; /* NaN fails it */
          f3 p3 = get_point3d(o, idx, dz);
          float sd = norm3(p3), vd = norm3(vc);
          float nsdf;
          if (vd > sd - tau && vd < sd + tau && dz < o->max_sensor_depth) nsdf = sd - vd;
          else if (vd < sd - tau) nsdf = tau;
          else continue;
          /* UpdateVoxel re-derives the voxel from the world position (tsdf_volume.cu:303-315) */
          f3 back = xform(T, vc);
          i3 g = world_to_global_voxel(t, back);
          i3 gb = {fdiv(g.x, B), fdiv(g.y, B), fdiv(g.z, B)};
          int ptr = find_entry(t, gb);
          if (ptr < 0) continue;
          Voxel* tgt = t->voxels + (long)ptr * B * B * B + pmod(g.x, B) * B * B + pmod(g.y, B) * B + pmod(g.z, B);
          (void)blk;
          combine(tgt, nsdf, bgr + 3 * idx, o->max_sdf_weight);
        }
  }
  t->last_visible = vis;
}

int tsdf_oracle_integrate(Tsdf* t, const unsigned char* bgr, const float* depth, const float* pose) {
  float Ti[16];
  if (!inv4(pose, Ti)) return -1;
  allocate_from_depth(t, depth, pose);
  integrate(t, bgr, depth, pose, Ti);
  return 0;
}

void tsdf_oracle_render(Tsdf* t, const float* pose, unsigned char* bgr_out, float* depth_out) { /* :600-632 */
  const Options* o = &t->o;
  long nv = (long)o->num_blocks * o->block_size * o->block_size * o->block_size;
  if (!t->touched) t->touched = (unsigned char*)calloc(nv, 1); else memset(t->touched, 0, nv);
  int n = o->height * o->width;
  for (int i = 0; i < n; ++i) {
    float cur = 0;
    int guard = 0;
    while (cur < o->max_sensor_depth && guard++ < 100000) {
      f3 p = xform(pose, get_point3d(o, i, cur));
      Voxel v = get_interpolated(t, p);
      if (v.w == 0) cur += o->truncation_distance; else cur += v.sdf;
      if (v.w != 0 && v.sdf < o->voxel_size) break;
    }
    if (cur < o->max_sensor_depth) {
      f3 p = xform(pose, get_point3d(o, i, cur));
      Voxel v = get_interpolated(t, p);
      bgr_out[3 * i] = v.c[0]; bgr_out[3 * i + 1] = v.c[1]; bgr_out[3 * i + 2] = v.c[2];
      depth_out[i] = cur;
    } else {
      bgr_out[3 * i] = bgr_out[3 * i + 1] = bgr_out[3 * i + 2] = 0;
      depth_out[i] = 0.0f;
    }
  }
  long cnt = 0;
  for (long k = 0; k < nv; ++k) cnt += t->touched[k];
  t->last_render_distinct_voxels = cnt;
}

void tsdf_oracle_stats(const Tsdf* t, long* out5) {
  out5[0] = t->allocated; out5[1] = t->last_visible; out5[2] = t->dropped; out5[3] = t->last_candidates;
  out5[4] = t->last_render_distinct_voxels;
}

static int cmp_i3(const void* a, const void* b) {
  const int* p = (const int*)a; const int* q = (const int*)b;
  for (int k = 0; k < 3; ++k) if (p[k] != q[k]) return p[k] < q[k] ? -1 : 1;
  return 0;
}
/* dump blocks sorted by (x,y,z): coords[3*n], voxels[n*512] (may be NULL). returns n */
long tsdf_oracle_dump(const Tsdf* t, int* coords, Voxel* voxels, long cap) {
  int B3 = t->o.block_size * t->o.block_size * t->o.block_size;
  long n = 0;
  int* tmp = (int*)malloc(sizeof(int) * 4 * (t->allocated + 1));
  for (long e = 0; e < t->n_entries; ++e) if (t->entries[e].ptr != -1) {
    tmp[4 * n] = t->entries[e].pos.x; tmp[4 * n + 1] = t->entries[e].pos.y; tmp[4 * n + 2] = t->entries[e].pos.z;
    tmp[4 * n + 3] = t->entries[e].ptr; n++;
  }
  qsort(tmp, n, 4 * sizeof(int), cmp_i3);
  long m = n < cap ? n : cap;
  for (long k = 0; k < m; ++k) {
    coords[3 * k] = tmp[4 * k]; coords[3 * k + 1] = tmp[4 * k + 1]; coords[3 * k + 2] = tmp[4 * k + 2];
    if (voxels) memcpy(voxels + k * B3, t->voxels + (long)tmp[4 * k + 3] * B3, sizeof(Voxel) * B3);
  }
  free(tmp);
  return n;
}

/* ================= marching cubes (SURVEY.md 8f row n4) =================
 * Restates ExtractMeshKernel / ExtractMeshAtPosition / TrilinearInterpolation / VertexInterpolation
 * (marching_cubes/mesh_extractor.cu:24-104, 106-135, 137-243, 244-265) and the vertex / colour layout of
 * TsdfVolume::GetMeshSync (tsdf_volume.cu:781-839): brute force over every cell of the bounding box in linear cell
 * order (x fastest), so the oracle's output order is the reference's for a single thread; the reference appends with
 * atomicAdd (mesh.cu:21-24), i.e. its order is arbitrary -> tests compare sorted triangle sets.
 * Where the reference's nvcc build (default -fmad=true) contracts a*b+c, this restatement calls fmaf() explicitly
 * (the file is built with -ffp-contract=off, so nothing else is fused): the cell position i*s+lower
 * (mesh_extractor.cu:258-261), the trilinear accumulation distance += W*sdf (:41-96) and the edge vertex
 * p1+mu*(p2-p1) (:121-123).  The CUDA kernel uses the same fmaf / __f*_rn sequence, so the two are bit-identical.
 */
#include "mc_tables.h"

static int w2g1(float x, float s) { return (int)(x / s + signf_(x) * 0.5f); } /* one axis of tsdf_volume.cu:109-113 */

static Voxel voxel_at(Tsdf* t, int gx, int gy, int gz) { /* tsdf_volume.cu:115-159 from a global voxel index */
  int B = t->o.block_size;
  i3 blk = {fdiv(gx, B), fdiv(gy, B), fdiv(gz, B)};
  int ptr = find_entry(t, blk);
  Voxel v;
  if (ptr < 0) { memset(&v, 0, sizeof v); return v; }
  return t->voxels[(long)ptr * B * B * B + pmod(gx, B) * B * B + pmod(gy, B) * B + pmod(gz, B)];
}

/* mesh_extractor.cu:24-104 - false as soon as one of the eight voxels has weight 0; only the distance is consumed */
static int mesh_trilinear(Tsdf* t, f3 p, float* dist_out) {
  float s = t->o.voxel_size;
  float h = s / 2.0f;
  f3 pd = {p.x - h, p.y - h, p.z - h};
  f3 vp = {p.x / s, p.y / s, p.z / s};
  float wx = vp.x - floorf(vp.x), wy = vp.y - floorf(vp.y), wz = vp.z - floorf(vp.z);
  static const int ox[8] = {0, 1, 0, 0, 1, 0, 1, 1}, oy[8] = {0, 0, 1, 0, 1, 1, 0, 1}, oz[8] = {0, 0, 0, 1, 0, 1, 1, 1};
  float dist = 0.0f;
  for (int k = 0; k < 8; ++k) {
    f3 q = {pd.x + (ox[k] ? s : 0.0f), pd.y + (oy[k] ? s : 0.0f), pd.z + (oz[k] ? s : 0.0f)};
    Voxel v = voxel_at(t, w2g1(q.x, s), w2g1(q.y, s), w2g1(q.z, s));
    if (v.w == 0) return 0;
    float W = ((ox[k] ? wx : 1.0f - wx) * (oy[k] ? wy : 1.0f - wy)) * (oz[k] ? wz : 1.0f - wz);
    dist = fmaf(W, v.sdf, dist);
  }
  *dist_out = dist;
  return 1;
}

/* cube corners in the reference's bit order (mesh_extractor.cu:188-196): 010,110,100,000,011,111,101,001 */
static const int kCornerX[8] = {0, 1, 1, 0, 0, 1, 1, 0}, kCornerY[8] = {1, 1, 0, 0, 1, 1, 0, 0}, kCornerZ[8] = {0, 0, 0, 0, 1, 1, 1, 1};
static const int kEdgeA[12] = {0, 1, 2, 3, 4, 5, 6, 7, 0, 1, 2, 3}, kEdgeB[12] = {1, 2, 3, 0, 5, 6, 7, 4, 4, 5, 6, 7}; /* :203-237 */

static float lerp_axis(float mu, float a, float b) { return fmaf(mu, b - a, a); } /* mesh_extractor.cu:121-123 */

/* vert/cols: xyz / rgb float triples per vertex (three vertices per triangle), cap in vertices. returns #vertices */
long tsdf_oracle_extract_mesh(Tsdf* t, const float* lower, const float* upper, float* vert, float* cols, long cap) {
  float s = t->o.voxel_size;
  int n[3];
  for (int a = 0; a < 3; ++a) n[a] = to_int_sat(fabsf(lower[a] - upper[a]) / s); /* :248-252 */
  long nv = 0;
  float h = s / 2.0f;
  for (int iz = 0; iz < n[2]; ++iz)
    for (int iy = 0; iy < n[1]; ++iy)
      for (int ix = 0; ix < n[0]; ++ix) {
        f3 pos = {fmaf((float)ix, s, lower[0]), fmaf((float)iy, s, lower[1]), fmaf((float)iz, s, lower[2])};
        /* cheap reject first (result-neutral): the p000 sample's first voxel must exist (it is tested first, :146-149) */
        f3 cp[8];
        float d[8];
        /* evaluation order of the reference: 000,100,010,001,110,011,101,111 -> our corner ids 3,2,0,7,1,4,6,5 */
        static const int order[8] = {3, 2, 0, 7, 1, 4, 6, 5};
        int ok = 1;
        for (int k = 0; k < 8 && ok; ++k) {
          int c = order[k];
          cp[c].x = pos.x + (kCornerX[c] ? h : -h);
          cp[c].y = pos.y + (kCornerY[c] ? h : -h);
          cp[c].z = pos.z + (kCornerZ[c] ? h : -h);
          ok = mesh_trilinear(t, cp[c], &d[c]);
        }
        if (!ok) continue;
        int cube = 0;
        for (int c = 0; c < 8; ++c) if (d[c] < 0.0f) cube |= 1 << c;
        uint64_t tri = kMcTri[cube];
        if ((tri & 0xF) == 0xF) continue; /* edgeTable[cubeindex] == 0 */
        Voxel vc = voxel_at(t, w2g1(pos.x, s), w2g1(pos.y, s), w2g1(pos.z, s)); /* :200 */
        float col[3] = {(float)vc.c[2] / 255.f, (float)vc.c[1] / 255.f, (float)vc.c[0] / 255.f}; /* GetMeshSync: z,y,x */
        for (int k = 0; k < 15; ++k) {
          int e = (int)((tri >> (4 * k)) & 0xF);
          if (e == 0xF) break;
          int a = kEdgeA[e], b = kEdgeB[e];
          f3 p;
          float d1 = d[a], d2 = d[b];
          if (fabsf(0.0f - d1) < 0.00001f) p = cp[a];
          else if (fabsf(0.0f - d2) < 0.00001f) p = cp[b];
          else if (fabsf(d1 - d2) < 0.00001f) p = cp[a];
          else {
            float mu = (0.0f - d1) / (d2 - d1);
            p.x = lerp_axis(mu, cp[a].x, cp[b].x); p.y = lerp_axis(mu, cp[a].y, cp[b].y); p.z = lerp_axis(mu, cp[a].z, cp[b].z);
          }
          if (nv < cap) {
            vert[3 * nv] = p.x; vert[3 * nv + 1] = p.y; vert[3 * nv + 2] = p.z;
            cols[3 * nv] = col[0]; cols[3 * nv + 1] = col[1]; cols[3 * nv + 2] = col[2];
          }
          nv++;
        }
      }
  return nv;
}
