/* CPU oracle of n10 (test infrastructure only): DSO's pixel selection restated in C, statement for statement.
 *   pattern     PixelSelector::PixelSelector's random pattern   tandem/src/FullSystem/PixelSelector2.cpp:41-56
 *               (std::srand(3141592), then rand() & 0xFF per pixel; glibc's TYPE_3 additive feedback generator is restated
 *               here, so nothing touches the process-global rand state)
 *   make_hists  PixelSelector::makeHists    :66-141
 *   select      PixelSelector::select       :295-438
 *   make_maps   PixelSelector::makeMaps     :142-291 (without the plot branch)
 * Inputs are the pinned pyramid definition (front_oracle.c): level 0 (I, dx, dy) and absSquaredGrad of levels 0..2, no
 * gamma weights (a linear response).  Two reads of memory the reference never writes are defined here as the device defines
 * them: level 2's last row is 0 (as front_oracle.c leaves it), and a thsSmoothed index at or beyond w32 * h32 reads 0.
 * fp32 without contraction (oracle/pixsel_oracle.mk). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* rand() after srand(seed) of glibc (random_r.c, TYPE_3: degree 31, separation 3, 310 discarded outputs) */
void pixsel_oracle_pattern(unsigned int seed, int n, unsigned char* out) {
  int32_t r[34];
  r[0] = (int32_t)seed;
  for (int i = 1; i < 31; ++i) {
    /* 16807 * r mod (2^31 - 1) by Schrage's method, as srandom_r computes it */
    const int32_t hi = r[i - 1] / 127773, lo = r[i - 1] % 127773;
    int32_t word = 16807 * lo - 2836 * hi;
    if (word < 0) word += 2147483647;
    r[i] = word;
  }
  /* the sequence r_i: r_31..33 = r_0..2, r_i = r_(i-31) + r_(i-3) (mod 2^32) from i = 34; call k returns r_(344+k) >> 1 */
  uint32_t ring[34];
  for (int i = 0; i < 31; ++i) ring[i] = (uint32_t)r[i];
  for (int i = 31; i < 34; ++i) ring[i] = ring[i - 31];
  for (long long i = 34; i < 344 + (long long)n; ++i) {
    const uint32_t v = ring[(i - 31) % 34] + ring[(i - 3) % 34];
    ring[i % 34] = v;
    if (i >= 344) out[i - 344] = (unsigned char)((v >> 1) & 0xFF);
  }
}

/* select's directions (:312-328): double literals converted to float, as Vec2f's constructor converts them */
static const float kDirs[16][2] = {{0, 1.0000},      {0.3827, 0.9239},  {0.1951, 0.9808},  {0.9239, 0.3827},
                                   {0.7071, 0.7071}, {0.3827, -0.9239}, {0.8315, 0.5556},  {0.8315, -0.5556},
                                   {0.5556, -0.8315}, {0.9808, 0.1951}, {0.9239, -0.3827}, {0.7071, -0.7071},
                                   {0.5556, 0.8315}, {0.9808, -0.1951}, {1.0000, 0.0000},  {0.1951, -0.9808}};

/* settings: setting_minGradHistCut, setting_minGradHistAdd, setting_gradDownweightPerLevel, setting_selectDirectionDistribution */
typedef struct {
  float cut, add, dw1;
  int dir_dist;
} Settings;

static int hist_quantil(const int* hist, float below) {   /* computeHistQuantil, :66-75 */
  int th = hist[0] * below + 0.5f;
  for (int i = 0; i < 90; i++) {
    th -= hist[i + 1];
    if (th < 0) return i;
  }
  return 90;
}

/* thsSmoothed (w32 * h32 floats) */
void pixsel_oracle_make_hists(int w, int h, const float* ag0, const float* settings, float* ths_smoothed) {
  const int w32 = w / 32, h32 = h / 32;
  float* ths = (float*)malloc(sizeof(float) * w32 * h32);
  int hist0[91];
  for (int y = 0; y < h32; y++)
    for (int x = 0; x < w32; x++) {
      const float* map0 = ag0 + 32 * x + 32 * y * w;
      memset(hist0, 0, sizeof hist0);
      for (int j = 0; j < 32; j++)
        for (int i = 0; i < 32; i++) {
          int it = i + 32 * x;
          int jt = j + 32 * y;
          if (it > w - 2 || jt > h - 2 || it < 1 || jt < 1) continue;
          const float s = sqrtf(map0[i + j * w]);
          int g = s < 49.f ? (int)s : 48;   /* a non-finite gradient (never made by the pyramid) counts as the clamp */
          if (g > 48) g = 48;
          hist0[g + 1]++;
          hist0[0]++;
        }
      ths[x + y * w32] = hist_quantil(hist0, settings[0]) + settings[1];
    }
  for (int y = 0; y < h32; y++)
    for (int x = 0; x < w32; x++) {
      float sum = 0, num = 0;
      if (x > 0) {
        if (y > 0) { num++; sum += ths[x - 1 + (y - 1) * w32]; }
        if (y < h32 - 1) { num++; sum += ths[x - 1 + (y + 1) * w32]; }
        num++; sum += ths[x - 1 + (y)*w32];
      }
      if (x < w32 - 1) {
        if (y > 0) { num++; sum += ths[x + 1 + (y - 1) * w32]; }
        if (y < h32 - 1) { num++; sum += ths[x + 1 + (y + 1) * w32]; }
        num++; sum += ths[x + 1 + (y)*w32];
      }
      if (y > 0) { num++; sum += ths[x + (y - 1) * w32]; }
      if (y < h32 - 1) { num++; sum += ths[x + (y + 1) * w32]; }
      num++; sum += ths[x + y * w32];
      ths_smoothed[x + y * w32] = (sum / num) * (sum / num);
    }
  free(ths);
}

typedef struct {
  int w, h;
  const float *dI, *ag0, *ag1, *ag2, *ths;
  const unsigned char* rp;
  Settings s;
} Frame;

static float th_at(const Frame* F, int xf, int yf) {
  const int w32 = F->w / 32, h32 = F->h / 32, i = (xf >> 5) + (yf >> 5) * w32;
  return i < w32 * h32 ? F->ths[i] : 0.f;
}

/* select, :295-438.  *ties counts the pixels whose score tied the running best (> 0) at some level. */
static void select_(const Frame* F, float* map_out, int pot, float thFactor, int n[3], int* ties) {
  const int w = F->w, h = F->h, w1 = w / 2, w2 = w / 4;
  const float dw1 = F->s.dw1, dw2 = dw1 * dw1;
  memset(map_out, 0, sizeof(float) * w * h);
  int n3 = 0, n2 = 0, n4 = 0;
  for (int y4 = 0; y4 < h; y4 += (4 * pot))
    for (int x4 = 0; x4 < w; x4 += (4 * pot)) {
      int my3 = 4 * pot < h - y4 ? 4 * pot : h - y4;
      int mx3 = 4 * pot < w - x4 ? 4 * pot : w - x4;
      int bestIdx4 = -1; float bestVal4 = 0;
      const float* dir4 = kDirs[F->rp[n2] & 0xF];
      for (int y3 = 0; y3 < my3; y3 += (2 * pot))
        for (int x3 = 0; x3 < mx3; x3 += (2 * pot)) {
          int x34 = x3 + x4, y34 = y3 + y4;
          int my2 = 2 * pot < h - y34 ? 2 * pot : h - y34;
          int mx2 = 2 * pot < w - x34 ? 2 * pot : w - x34;
          int bestIdx3 = -1; float bestVal3 = 0;
          const float* dir3 = kDirs[F->rp[n2] & 0xF];
          for (int y2 = 0; y2 < my2; y2 += pot)
            for (int x2 = 0; x2 < mx2; x2 += pot) {
              int x234 = x2 + x34, y234 = y2 + y34;
              int my1 = pot < h - y234 ? pot : h - y234;
              int mx1 = pot < w - x234 ? pot : w - x234;
              int bestIdx2 = -1; float bestVal2 = 0;
              const float* dir2 = kDirs[F->rp[n2] & 0xF];
              for (int y1 = 0; y1 < my1; y1 += 1)
                for (int x1 = 0; x1 < mx1; x1 += 1) {
                  int idx = x1 + x234 + w * (y1 + y234);
                  int xf = x1 + x234, yf = y1 + y234;
                  if (xf < 4 || xf >= w - 5 || yf < 4 || yf > h - 4) continue;
                  float pixelTH0 = th_at(F, xf, yf);
                  float pixelTH1 = pixelTH0 * dw1;
                  float pixelTH2 = pixelTH1 * dw2;
                  const float dx = F->dI[3 * idx + 1], dy = F->dI[3 * idx + 2];
                  float ag0 = F->ag0[idx];
                  if (ag0 > pixelTH0 * thFactor) {
                    float dirNorm = fabsf(dx * dir2[0] + dy * dir2[1]);
                    if (!F->s.dir_dist) dirNorm = ag0;
                    if (dirNorm > bestVal2) { bestVal2 = dirNorm; bestIdx2 = idx; bestIdx3 = -2; bestIdx4 = -2; }
                    else if (dirNorm == bestVal2 && bestVal2 > 0) ++*ties;
                  }
                  if (bestIdx3 == -2) continue;
                  float ag1 = F->ag1[(int)(xf * 0.5f + 0.25f) + (int)(yf * 0.5f + 0.25f) * w1];
                  if (ag1 > pixelTH1 * thFactor) {
                    float dirNorm = fabsf(dx * dir3[0] + dy * dir3[1]);
                    if (!F->s.dir_dist) dirNorm = ag1;
                    if (dirNorm > bestVal3) { bestVal3 = dirNorm; bestIdx3 = idx; bestIdx4 = -2; }
                    else if (dirNorm == bestVal3 && bestVal3 > 0) ++*ties;
                  }
                  if (bestIdx4 == -2) continue;
                  float ag2 = F->ag2[(int)(xf * 0.25f + 0.125) + (int)(yf * 0.25f + 0.125) * w2];
                  if (ag2 > pixelTH2 * thFactor) {
                    float dirNorm = fabsf(dx * dir4[0] + dy * dir4[1]);
                    if (!F->s.dir_dist) dirNorm = ag2;
                    if (dirNorm > bestVal4) { bestVal4 = dirNorm; bestIdx4 = idx; }
                    else if (dirNorm == bestVal4 && bestVal4 > 0) ++*ties;
                  }
                }
              if (bestIdx2 > 0) { map_out[bestIdx2] = 1; bestVal3 = 1e10; n2++; }
            }
          if (bestIdx3 > 0) { map_out[bestIdx3] = 2; bestVal4 = 1e10; n3++; }
        }
      if (bestIdx4 > 0) { map_out[bestIdx4] = 4; n4++; }
    }
  n[0] = n2; n[1] = n3; n[2] = n4;
}

/* The cells (pot x pot, aligned to the image origin) whose level-2 selection depends on the direction they get: some
 * direction selects and another does not (DESIGN.md, n10). */
static int nonuniform_cells(const Frame* F, int pot, float thFactor) {
  const int w = F->w, h = F->h;
  int count = 0;
  for (int y0 = 0; y0 < h; y0 += pot)
    for (int x0 = 0; x0 < w; x0 += pot) {
      unsigned mask = 0;
      for (int yf = y0; yf < y0 + pot && yf < h; ++yf)
        for (int xf = x0; xf < x0 + pot && xf < w; ++xf) {
          if (xf < 4 || xf >= w - 5 || yf < 4 || yf > h - 4) continue;
          const int idx = xf + yf * w;
          if (!(F->ag0[idx] > th_at(F, xf, yf) * thFactor)) continue;
          for (int d = 0; d < 16; ++d)
            if (!F->s.dir_dist || fabsf(F->dI[3 * idx + 1] * kDirs[d][0] + F->dI[3 * idx + 2] * kDirs[d][1]) > 0) mask |= 1u << d;
        }
      count += mask != 0 && mask != 0xFFFFu;
    }
  return count;
}

/* (int)x as x86-64's cvttss2si computes it: INT_MIN where the value has no int (NaN, out of range) */
static int to_int(float x) { return (x >= -2147483648.f && x < 2147483648.f) ? (int)x : (-2147483647 - 1); }

/* makeMaps, :142-291.  *potential is currentPotential (in and out).  info: n2, n3, n4 of the final select, the potential it
 * used, whether the call re-selected, ties, non-uniform cells of the final select, selects run.  Returns numHaveSub. */
int pixsel_oracle_make_maps(int w, int h, const float* dI, const float* ag0, const float* ag1, const float* ag2,
                            const float* ths_smoothed, const unsigned char* pattern, const float* settings, int* potential,
                            float density, int recursionsLeft, float thFactor, float* map_out, int* info) {
  Frame F = {w, h, dI, ag0, ag1, ag2, ths_smoothed, pattern, {settings[0], settings[1], settings[2], settings[3] != 0.f}};
  float numHave = 0;
  float numWant = density;
  float quotia;
  int idealPotential = *potential;
  int n[3];
  info[4] = 0; info[5] = 0; info[7] = 0;
  for (;;) {
    const int currentPotential = *potential;
    int ties = 0;
    select_(&F, map_out, currentPotential, thFactor, n, &ties);
    info[0] = n[0]; info[1] = n[1]; info[2] = n[2]; info[3] = currentPotential; info[5] += ties;
    info[6] = nonuniform_cells(&F, currentPotential, thFactor);
    info[7]++;
    numHave = n[0] + n[1] + n[2];
    quotia = numWant / numHave;
    float K = numHave * (currentPotential + 1) * (currentPotential + 1);
    idealPotential = to_int(sqrtf(K / numWant) - 1);
    if (idealPotential < 1) idealPotential = 1;
    if (recursionsLeft > 0 && quotia > 1.25 && currentPotential > 1) {
      if (idealPotential >= currentPotential) idealPotential = currentPotential - 1;
      *potential = idealPotential;
      recursionsLeft--;
      info[4] = 1;
      continue;
    } else if (recursionsLeft > 0 && quotia < 0.25) {
      if (idealPotential <= currentPotential) idealPotential = currentPotential + 1;
      *potential = idealPotential;
      recursionsLeft--;
      info[4] = 1;
      continue;
    }
    break;
  }
  int numHaveSub = numHave;
  if (quotia < 0.95) {
    int wh = w * h;
    int rn = 0;
    unsigned char charTH = 255 * quotia;
    for (int i = 0; i < wh; i++) {
      if (map_out[i] != 0) {
        if (pattern[rn] > charTH) {
          map_out[i] = 0;
          numHaveSub--;
        }
        rn++;
      }
    }
  }
  *potential = idealPotential;
  return numHaveSub;
}
