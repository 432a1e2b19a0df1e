// atanf, atan2f and asinf as the host's libm computes them, for the host and the device.
//
// The planner (geometry.cpp: Projector::lookupInput) maps a direction to an equirectangular input with atan2f and asinf
// from the system libm.  The per-frame orientation path (oriented_view.h) has to reproduce those results bit for bit on
// the device, so these are ports of the library's code, operation for operation.
//
// Which library: GNU libc 2.39 (Ubuntu 2.39-0ubuntu8.5), x86-64, libm.so.6.  There, asinf, atan2f and atanf are plain
// symbols (not ifuncs: the CPU's features do not select among variants as they do for sinf, cosf and tan), and their code
// has no FMA instruction.  The sequences below were read from `objdump -d` of __asinf_finite, __atan2f_finite and atanf,
// the constants from the .rodata words those functions load, and the wrappers asinf / atan2f (the compat wrappers, which
// are the default symbol versions) for what they add around them.  Every value is a float, every operation one IEEE
// single-precision + - * / or square root, round to nearest even: the fdlibm algorithms, with glibc's compiler having
// folded the coefficient tables into immediate loads (so atanf keeps no local array, and on the device uses no stack).
// tests/test_oriented.py compiles this header for the host and compares asinf and atanf with the library over all 2^32
// inputs, atan2f over 10^8 seeded pairs and the special values.
//
// On the device every operation is an explicit __f*_rn intrinsic (nvcc would contract a*b+c into an FMA), on the host a
// plain operator (host code is compiled with -ffp-contract=off).  The only difference left is the bit pattern of a NaN
// result: the device's is canonical.  Nothing downstream reads a NaN's payload (quantizeAxis maps every NaN to INT_MIN).
#pragma once

#include <cstdint>
#include <cstring>

#include "flat_view.h"

namespace t360 {

T360_HD float fSqrt(float a) {
#ifdef __CUDA_ARCH__
  return __fsqrt_rn(a);
#else
  return std::sqrt(a);
#endif
}
T360_HD uint32_t floatBits(float f) {
#ifdef __CUDA_ARCH__
  return __float_as_uint(f);
#else
  uint32_t u;
  std::memcpy(&u, &f, sizeof(u));
  return u;
#endif
}
T360_HD float bitsFloat(uint32_t u) {
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  std::memcpy(&f, &u, sizeof(f));
  return f;
#endif
}

// atanf (fdlibm s_atanf.c): argument reduction to |x| < 7/16 around atan(0.5), atan(1), atan(1.5) and atan(inf), then an
// odd polynomial split into even and odd halves in w = x^4.
T360_HD float libmAtanf(float x) {
  const uint32_t hx = floatBits(x), ix = hx & 0x7fffffffu;
  const bool neg = static_cast<int32_t>(hx) < 0;
  if (ix > 0x4bffffffu) {  // |x| >= 2^24 or NaN
    if (ix > 0x7f800000u) return fAdd(x, x);
    return neg ? fSub(-0x1.921fb4p+0f, 0x1.4442d0p-24f) : fAdd(0x1.4442d0p-24f, 0x1.921fb4p+0f);
  }
  float hi = 0.0f, lo = 0.0f;
  bool reduced = true;
  if (ix <= 0x3edfffffu) {         // |x| < 0.4375
    if (ix <= 0x30ffffffu) return x;  // |x| < 2^-29 (the library only raises inexact / underflow here)
    reduced = false;
  } else {
    x = bitsFloat(ix);
    if (ix > 0x3f97ffffu) {
      if (ix > 0x401bffffu) {  // 2.4375 <= |x| < 2^24
        hi = 0x1.921fb4p+0f; lo = 0x1.4442d0p-24f;
        x = fDiv(-1.0f, x);
      } else {                 // 1.1875 <= |x| < 2.4375
        hi = 0x1.f730bcp-1f; lo = 0x1.281f68p-25f;
        x = fDiv(fSub(x, 1.5f), fAdd(fMul(x, 1.5f), 1.0f));
      }
    } else if (ix > 0x3f2fffffu) {  // 0.6875 <= |x| < 1.1875
      hi = 0x1.921fb4p-1f; lo = 0x1.4442d0p-25f;
      x = fDiv(fSub(x, 1.0f), fAdd(x, 1.0f));
    } else {                        // 0.4375 <= |x| < 0.6875
      hi = 0x1.dac670p-2f; lo = 0x1.586ed2p-28f;
      x = fDiv(fSub(fAdd(x, x), 1.0f), fAdd(x, 2.0f));
    }
  }
  const float z = fMul(x, x), w = fMul(z, z);
  float s1 = fAdd(fMul(0x1.0ad3aep-6f, w), 0x1.97b4b2p-5f);
  s1 = fAdd(fMul(s1, w), 0x1.10d66ap-4f);
  s1 = fAdd(fMul(s1, w), 0x1.745cdcp-4f);
  s1 = fAdd(fMul(s1, w), 0x1.24924ap-3f);
  s1 = fMul(fAdd(fMul(s1, w), 0x1.555556p-2f), z);
  float s2 = fSub(fMul(-0x1.2b4442p-5f, w), 0x1.dde2d6p-5f);
  s2 = fSub(fMul(s2, w), 0x1.3b0f2ap-4f);
  s2 = fSub(fMul(s2, w), 0x1.c71c70p-4f);
  s2 = fMul(fSub(fMul(s2, w), 0x1.99999ap-3f), w);
  const float r = fMul(fAdd(s1, s2), x);
  if (!reduced) return fSub(x, r);
  const float a = fSub(hi, fSub(fSub(r, lo), x));
  return neg ? -a : a;
}

// atan2f (fdlibm e_atan2f.c, with the wrapper, which only sets errno around it when the library's _LIB_VERSION is POSIX)
T360_HD float libmAtan2f(float y, float x) {
  constexpr float kTiny = 0x1.4484c0p-100f, kPi = 0x1.921fb6p+1f, kPio2 = 0x1.921fb6p+0f, kPio4 = 0x1.921fb6p-1f;
  const uint32_t hx = floatBits(x), hy = floatBits(y), ix = hx & 0x7fffffffu, iy = hy & 0x7fffffffu;
  // x + y on x86 returns x quieted when both are NaN; the compiler may swap the operands of a + b, so spell it out
  if (ix > 0x7f800000u) return fAdd(x, x);
  if (iy > 0x7f800000u) return fAdd(y, y);
  if (hx == 0x3f800000u) return libmAtanf(y);
  const int m = static_cast<int>(((hy >> 31) & 1u) | ((hx >> 30) & 2u));  // 2 * sign(x) + sign(y)
  if (iy == 0) {
    if (m == 2) return fAdd(kTiny, kPi);
    if (m == 3) return fSub(-kPi, kTiny);
    return y;
  }
  const bool yNeg = static_cast<int32_t>(hy) < 0;
  if (ix == 0) return yNeg ? fSub(-kPio2, kTiny) : fAdd(kTiny, kPio2);
  if (ix == 0x7f800000u) {
    if (iy == 0x7f800000u) {
      switch (m) {
        case 0: return fAdd(kTiny, kPio4);
        case 1: return fSub(-kPio4, kTiny);
        case 2: return fAdd(fMul(3.0f, kPio4), kTiny);
        default: return fSub(fMul(-3.0f, kPio4), kTiny);
      }
    }
    switch (m) {
      case 0: return 0.0f;
      case 1: return -0.0f;
      case 2: return fAdd(kTiny, kPi);
      default: return fSub(-kPi, kTiny);
    }
  }
  if (iy == 0x7f800000u) return yNeg ? fSub(-kPio2, kTiny) : fAdd(kTiny, kPio2);
  const int32_t d = static_cast<int32_t>(iy) - static_cast<int32_t>(ix), k = d >> 23;
  float z;
  if (d > 0x1e7fffff) z = fSub(kPio2, 0x1.777a5cp-25f);  // |y / x| > 2^60: pi/2 + pi_lo/2
  else if (static_cast<int32_t>(hx) < 0 && k < -60) z = 0.0f;
  else z = libmAtanf(bitsFloat(floatBits(fDiv(y, x)) & 0x7fffffffu));
  switch (m) {
    case 0: return z;
    case 1: return -z;
    case 2: return fSub(kPi, fAdd(z, 0x1.777a5cp-24f));  // pi - (z - pi_lo)
    default: return fSub(fAdd(z, 0x1.777a5cp-24f), kPi);
  }
}

// asinf (e_asinf.c: the Cephes polynomial with fdlibm's argument reduction), with the wrapper's domain error: |x| > 1
// returns the default NaN (__kernel_standard_f), a NaN returns itself quieted.
T360_HD float libmAsinf(float x) {
  constexpr float kPio2Hi = 0x1.921fb6p+0f, kPio2Lo = -0x1.777a5cp-25f, kPio4Hi = 0x1.921fb6p-1f;
  const uint32_t hx = floatBits(x), ix = hx & 0x7fffffffu;
  const bool neg = static_cast<int32_t>(hx) <= 0;
  if (ix == 0x3f800000u) return fAdd(fMul(x, kPio2Lo), fMul(x, kPio2Hi));
  if (ix > 0x3f800000u) {
    if (ix > 0x7f800000u) {
      const float z = fSub(x, x);
      return fDiv(z, z);
    }
    return bitsFloat(0x7fc00000u);
  }
  auto poly = [](float t) {
    float p = fAdd(fMul(0x1.596d28p-5f, t), 0x1.8c283cp-6f);
    p = fAdd(fMul(p, t), 0x1.747e4ap-5f);
    p = fAdd(fMul(p, t), 0x1.3301e4p-4f);
    p = fAdd(fMul(p, t), 0x1.5555c8p-3f);
    return fMul(p, t);
  };
  if (ix <= 0x3effffffu) {            // |x| < 0.5
    if (ix <= 0x31ffffffu) return x;  // |x| < 2^-27
    return fAdd(x, fMul(poly(fMul(x, x)), x));
  }
  const float t = fMul(fSub(1.0f, bitsFloat(ix)), 0.5f);
  const float p = poly(t), s = fSqrt(t);
  float r;
  if (ix > 0x3f799999u) {  // |x| > 0.975
    const float h = fAdd(fMul(p, s), s);
    r = fSub(kPio2Hi, fAdd(0x1.777a5cp-25f, fAdd(h, h)));  // pio2_hi - (2 (s + s p) - pio2_lo)
  } else {
    const float df = bitsFloat(floatBits(s) & 0xfffff000u);
    const float c = fDiv(fSub(t, fMul(df, df)), fAdd(s, df));
    const float q = fSub(kPio4Hi, fAdd(df, df));
    const float pp = fSub(fMul(fAdd(s, s), p), fSub(kPio2Lo, fAdd(c, c)));
    r = fSub(kPio4Hi, fSub(pp, q));
  }
  return neg ? -r : r;
}

}  // namespace t360
