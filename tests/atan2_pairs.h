// The atan2f argument pairs both libm gates draw: tests/libm_gate.cpp (the host build of libmAtan2f against glibc) and
// tests/twin_gate.cu (its device build against its host build).  Index-based, so a pair depends only on (seed, i) and
// both gates see the same pairs whatever their thread or grid layout.  Compiles for the host and the device.
#pragma once

#include <cstdint>

#include "libm_ports.h"

namespace t360gate {

// splitmix64's output function: a counter-based hash, z -> a well-mixed 64-bit word
T360_HD uint64_t mix64(uint64_t z) {
  z += 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

// +-0, subnormals, the extreme normals, +-inf, NaNs, and the arguments at atanf's range splits (7/16, 11/16, 19/16,
// 39/16, 2^24, 2^-29) and at 1 and 0.5: kAtan2Specials values, the second half the first negated
constexpr int kAtan2Specials = 56;
T360_HD uint32_t atan2Special(int k) {
  const uint32_t base[kAtan2Specials / 2] = {
      0x00000000u, 0x00000001u, 0x00000002u, 0x003fffffu, 0x007fffffu, 0x00800000u, 0x00800001u, 0x3f800000u, 0x3f7fffffu, 0x3f800001u,
      0x3ee00000u, 0x3edfffffu, 0x3f300000u, 0x3f2fffffu, 0x3f980000u, 0x3f97ffffu, 0x401c0000u, 0x401bffffu, 0x4c000000u, 0x4bffffffu,
      0x31000000u, 0x30ffffffu, 0x7f7fffffu, 0x7f800000u, 0x7fc00000u, 0x7f800001u, 0x7fffffffu, 0x3f000000u};
  return k < kAtan2Specials / 2 ? base[k] : base[k - kAtan2Specials / 2] | 0x80000000u;
}

// pair k < kAtan2Specials^2 of the cross product of the special values: (y, x) bit patterns
T360_HD void atan2SpecialPair(int k, uint32_t* yb, uint32_t* xb) {
  *yb = atan2Special(k / kAtan2Specials);
  *xb = atan2Special(k % kAtan2Specials);
}

// pair i of stream `seed`: every fourth an arbitrary pair of bit patterns, the rest y = x * r with |r| near atanf's range
// splits (7/16, 11/16, 19/16, 39/16), near 1 and 0.5, and near the 2^+-60 / 2^24 / 2^-29 cut-offs, nudged by up to 32
// ulps either way, with a random sign
T360_HD void atan2RandomPair(uint64_t seed, uint64_t i, uint32_t* yb, uint32_t* xb) {
  const uint64_t r = mix64(mix64(seed) ^ i);
  const uint32_t a = static_cast<uint32_t>(r), b = static_cast<uint32_t>(r >> 32);
  if ((i & 3) == 0) {
    *yb = a;
    *xb = b;
    return;
  }
  const float ratios[] = {0.4375f, 0.6875f, 1.1875f, 2.4375f, 1.0f, 0.5f, 0x1p24f, 0x1p60f, 0x1p-60f, 0x1p-29f};
  // x: any finite float of moderate exponent; y = x * ratio, nudged by a few ulps either way
  const float x = t360::bitsFloat((a & 0x807fffffu) | ((100u + (a >> 23) % 56u) << 23));
  const float ratio = ratios[(b >> 8) % (sizeof(ratios) / sizeof(ratios[0]))];
  const int nudge = static_cast<int>(b & 0x3f) - 32;
  const uint32_t y = t360::floatBits(t360::fMul(x, ratio)) + static_cast<uint32_t>(nudge);
  *yb = (y & 0x7fffffffu) | ((b >> 16 & 1u) << 31);
  *xb = t360::floatBits(x);
}

}  // namespace t360gate
