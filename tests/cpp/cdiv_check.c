/* Test helper (CPU): the 3-instruction constant-divisor quotient used by the TSDF ray-cast (cdiv_ in tandem_b200/csrc/fusion.cu)
 * against IEEE division.  q0 = RN(x r), e = x - q0 d (exact FMA), q = RN(q0 + e r), r = RN(1/d). */
#include <math.h>
#include <stdint.h>
#include <string.h>

static inline float cdiv(float x, float d, float r) {
  const float ax = fabsf(x);
  if (!(ax > 1e-18f && ax < 1e18f)) return x / d;
  const float q0 = x * r;
  const float e = fmaf(-q0, d, x);
  return fmaf(e, r, q0);
}
static inline uint32_t bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float from_bits(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

/* every positive float x in [lo, hi] (and its negation) against divisor d; returns the number of mismatches */
long cdiv_check_exhaustive(float d, float lo, float hi) {
  volatile float one = 1.0f;
  const float r = one / d;
  long bad = 0;
  for (uint32_t u = bits(lo); u <= bits(hi); ++u) {
    const float x = from_bits(u);
    if (bits(cdiv(x, d, r)) != bits(x / d)) ++bad;
    if (bits(cdiv(-x, d, r)) != bits(-x / d)) ++bad;
  }
  return bad;
}
/* n random x against the fixed divisor d: random sign and significand, exponent uniform in 2^[-40, 40); returns mismatches */
long cdiv_check_random_x(float d, uint64_t seed, long n) {
  uint64_t s = seed * 0x9E3779B97F4A7C15ull + 1;
  volatile float one = 1.0f;
  const float r = one / d;
  long bad = 0;
  for (long i = 0; i < n; ++i) {
    s ^= s << 13; s ^= s >> 7; s ^= s << 17;
    const uint32_t a = (uint32_t)s;
    const uint32_t xe = 127 - 40 + (uint32_t)(s >> 32) % 80;
    const float x = from_bits((a & 0x80000000u) | (xe << 23) | (a & 0x7FFFFF));
    if (bits(cdiv(x, d, r)) != bits(x / d)) ++bad;
  }
  return bad;
}
/* n random (x, d) pairs: x log-uniform in [1e-6, 1e6] with random sign, d log-uniform in [1e-4, 1e4]; returns mismatches */
long cdiv_check_random(uint64_t seed, long n) {
  uint64_t s = seed * 0x9E3779B97F4A7C15ull + 1;
  long bad = 0;
  volatile float one = 1.0f;
  for (long i = 0; i < n; ++i) {
    s ^= s << 13; s ^= s >> 7; s ^= s << 17;
    const uint32_t a = (uint32_t)s, b = (uint32_t)(s >> 32);
    /* exponents: x in 2^[-20, 20), d in 2^[-13, 13); mantissas random */
    const uint32_t xe = 127 - 20 + (a >> 23) % 40, de = 127 - 13 + (b >> 23) % 26;
    float x = from_bits((xe << 23) | (a & 0x7FFFFF));
    const float d = from_bits((de << 23) | (b & 0x7FFFFF));
    if ((b & 0x7FFFFF) == 0x7FFFFF) continue;   /* all-ones significands are excluded on the host (fast_div_ok_) */
    if (a & 0x80000000u) x = -x;
    const float r = one / d;
    if (bits(cdiv(x, d, r)) != bits(x / d)) ++bad;
  }
  return bad;
}
