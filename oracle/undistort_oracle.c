/* ORACLE (test infrastructure - never linked into, or called by, the product library).
 *
 * Plain-C restatement of DSO's per-frame input (n11), statement for statement:
 *   undistort_oracle_create     PhotometricUndistorter's constructor      tandem/src/util/Undistort.cpp:50-179
 *                               (G must increase; normalised in double, stored as float; photometricCalibration 0: linear;
 *                               vignette / its maximum, inverted; valid only with response and vignette)
 *   undistort_oracle_set_gamma  FullSystem::setGammaFunction              tandem/src/FullSystem/FullSystem.cpp:232-253
 *   undistort_oracle_frame      processFrame + Undistort::undistort       Undistort.cpp:213-252, :393-490
 *   undistort_oracle_bgr        the dataset reader's BGR remap            tandem/src/util/DatasetReader.h:354-400
 *   undistort_oracle_make_images  FrameHessian::makeImages with its gamma weights (HessianBlocks.cpp:128-191, getBGradOnly
 *                               HessianBlocks.h:446-452): front_oracle.c's pyramid, then absSquaredGrad of [w, w*(h-1)) of
 *                               every level times gw * gw, which is the reference's `dabs_l[idx] *= gw*gw`.
 * PINNED against the reference's own statements by oracle/ref_build_undistort.mk + oracle/ref_wrap_undistort.cpp
 * (tests/golden/reference_pins_undistort.npz).  Library definitions where the reference is undefined (include/tandem_b200.h,
 * n11): a remap entry with xx < 0, yy < 0, (int)xx + 1 > w_org - 1 or (int)yy + 1 > h_org - 1 gives 0; (int)(I + 0.5f) of a
 * non-finite or out-of-range I is INT_MIN, as x86's cvttss2si gives it.
 */
#include <limits.h>

#include "front_oracle.c"

/* Returns valid.  G[256] receives the normalised G whenever the response is well formed; vinv (w_org*h_org) the inverted
 * vignette when valid.  response NULL: not valid. */
int undistort_oracle_create(const float* response, int n_response, const unsigned short* vignette, int n_pix, int mode,
                            float* G, float* vinv) {
  if (!response) return 0;
  for (int i = 0; i < n_response - 1; i++)
    if (response[i + 1] <= response[i]) return 0;
  const float min = response[0], max = response[n_response - 1];
  for (int i = 0; i < 256; i++) G[i] = 255.0 * (response[i] - min) / (max - min);
  if (mode == 0)
    for (int i = 0; i < 256; i++) G[i] = 255.0f * i / (float)(n_response - 1);
  if (!vignette) return 0;
  float maxV = 0;
  for (int i = 0; i < n_pix; i++)
    if (vignette[i] > maxV) maxV = vignette[i];
  for (int i = 0; i < n_pix; i++) vinv[i] = 1.0f / (vignette[i] / maxV);
  return 1;
}

/* B (256) in and out. */
void undistort_oracle_set_gamma(const float* Binv, float* B) {
  for (int i = 1; i < 255; i++)
    for (int s = 1; s < 255; s++)
      if (Binv[s] <= i && Binv[s + 1] >= i) {
        B[i] = s + (i - Binv[s]) / (Binv[s + 1] - Binv[s]);
        break;
      }
  B[0] = 0;
  B[255] = 255;
}

static int outside(float xx, float yy, int w_org, int h_org) {
  return !(xx >= 0 && yy >= 0 && xx < w_org - 1 && yy < h_org - 1);
}

/* processFrame into scratch (w_org*h_org floats), then the remap into out (w*h); remap_x NULL: passthrough.  Returns
 * exposure_time. */
float undistort_oracle_frame(const unsigned char* raw, int w_org, int h_org, int w, int h, const float* remap_x,
                             const float* remap_y, int valid, int mode, int use_exposure, const float* G, const float* vinv,
                             float exposure, float factor, float* scratch, float* out) {
  const int wh = w_org * h_org;
  if (!valid || exposure <= 0 || mode == 0) {
    for (int i = 0; i < wh; i++) scratch[i] = factor * raw[i];
  } else {
    for (int i = 0; i < wh; i++) scratch[i] = G[raw[i]];
    if (mode == 2)
      for (int i = 0; i < wh; i++) scratch[i] *= vinv[i];
  }
  if (!remap_x) {
    memcpy(out, scratch, sizeof(float) * (size_t)w * h);
  } else {
    for (int idx = w * h - 1; idx >= 0; idx--) {
      float xx = remap_x[idx], yy = remap_y[idx];
      if (outside(xx, yy, w_org, h_org)) {
        out[idx] = 0;
        continue;
      }
      const int xxi = xx, yyi = yy;
      xx -= xxi;
      yy -= yyi;
      const float xxyy = xx * yy;
      const float* src = scratch + xxi + yyi * w_org;
      out[idx] = xxyy * src[1 + w_org] + (yy - xxyy) * src[w_org] + (xx - xxyy) * src[1] + (1 - xx - yy + xxyy) * src[0];
    }
  }
  return use_exposure ? exposure : 1;
}

void undistort_oracle_bgr(const unsigned char* in, int w_org, int h_org, int w, int h, const float* remap_x,
                          const float* remap_y, unsigned char* out) {
  if (!remap_x) {
    memcpy(out, in, 3 * (size_t)w * h);
    return;
  }
  for (int idx = w * h - 1; idx >= 0; idx--) {
    float xx = remap_x[idx], yy = remap_y[idx];
    if (outside(xx, yy, w_org, h_org)) {
      out[3 * idx] = out[3 * idx + 1] = out[3 * idx + 2] = 0;
      continue;
    }
    const int xxi = xx, yyi = yy;
    xx -= xxi;
    yy -= yyi;
    const float xxyy = xx * yy;
    for (int c = 0; c < 3; ++c) {
      const unsigned char* src = in + (3 * xxi + c) + 3 * yyi * w_org;
      const float v = xxyy * src[3 + 3 * w_org] + (yy - xxyy) * src[3 * w_org] + (xx - xxyy) * src[3] + (1 - xx - yy + xxyy) * src[0];
      out[3 * idx + c] = (unsigned char)(int)v;   /* v in (-1, 256): truncation toward 0, as static_cast<unsigned char> */
    }
  }
}

/* CalibHessian::getBGradOnly with the x86 conversion of (int)(color + 0.5f) */
static float bgrad(const float* B, float color) {
  const float v = color + 0.5f;
  int c = (v >= -2147483648.f && v < 2147483648.f) ? (int)v : INT_MIN;
  if (c < 5) c = 5;
  if (c > 250) c = 250;
  return B[c + 1] - B[c];
}

/* front_oracle_make_images' layout; B NULL: no gamma weights. */
void undistort_oracle_make_images(const float* color, int w, int h, int levels, const float* B, float* dI, float* absgrad) {
  front_oracle_make_images(color, w, h, levels, dI, absgrad);
  if (!B) return;
  size_t off = 0;
  for (int lvl = 0; lvl < levels; ++lvl) {
    const int wl = w >> lvl, hl = h >> lvl;
    for (int idx = wl; idx < wl * (hl - 1); idx++) {
      const float gw = bgrad(B, dI[3 * (off + idx)]);
      absgrad[off + idx] *= gw * gw;
    }
    off += (size_t)wl * hl;
  }
}
