// Compares the host build of csrc/libm_ports.h with the system libm bit for bit (tests/test_oriented.py builds and runs
// it): asinf and atanf over every float bit pattern, atan2f over seeded random pairs and every pair of special values.
// Prints each mismatch (up to a limit) and the totals; exits 1 on any mismatch.
//
//   libm_gate <threads> <atan2f pairs> <seed>
#include <math.h>

#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <thread>
#include <vector>

#include "libm_ports.h"

namespace {

std::atomic<unsigned long long> gMismatches{0};
std::atomic<int> gPrinted{0};

void report(const char* fn, uint32_t a, uint32_t b, uint32_t want, uint32_t got) {
  gMismatches.fetch_add(1);
  if (gPrinted.fetch_add(1) < 40)
    std::printf("MISMATCH %s(0x%08x, 0x%08x): libm 0x%08x port 0x%08x\n", fn, a, b, want, got);
}

void checkUnary(const char* fn, float (*libm)(float), float (*port)(float), uint64_t begin, uint64_t end) {
  for (uint64_t u = begin; u < end; ++u) {
    const float x = t360::bitsFloat(static_cast<uint32_t>(u));
    const uint32_t want = t360::floatBits(libm(x)), got = t360::floatBits(port(x));
    if (want != got) report(fn, static_cast<uint32_t>(u), 0, want, got);
  }
}

void checkPair(uint32_t yb, uint32_t xb) {
  const float y = t360::bitsFloat(yb), x = t360::bitsFloat(xb);
  const uint32_t want = t360::floatBits(atan2f(y, x)), got = t360::floatBits(t360::libmAtan2f(y, x));
  if (want != got) report("atan2f", yb, xb, want, got);
}

uint64_t splitmix(uint64_t& s) {
  uint64_t z = (s += 0x9e3779b97f4a7c15ull);
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

// n pairs from stream `seed`: a quarter arbitrary bit patterns, the rest y = x * r with |r| near atanf's range splits
// (7/16, 11/16, 19/16, 39/16), near 1, and near the 2^+-60 / 2^24 cut-offs, with random signs
void randomPairs(uint64_t seed, uint64_t n) {
  static const float kRatios[] = {0.4375f, 0.6875f, 1.1875f, 2.4375f, 1.0f, 0.5f, 0x1p24f, 0x1p60f, 0x1p-60f, 0x1p-29f};
  uint64_t s = seed;
  for (uint64_t i = 0; i < n; ++i) {
    const uint64_t r = splitmix(s);
    const uint32_t a = static_cast<uint32_t>(r), b = static_cast<uint32_t>(r >> 32);
    if ((i & 3) == 0) {
      checkPair(a, b);
      continue;
    }
    // x: any finite float of moderate exponent; y = x * ratio, nudged by a few ulps either way
    const float x = t360::bitsFloat((a & 0x807fffffu) | ((100u + (a >> 23) % 56u) << 23));
    const float ratio = kRatios[(b >> 8) % (sizeof(kRatios) / sizeof(kRatios[0]))];
    const int nudge = static_cast<int>(b & 0x3f) - 32;
    const uint32_t yb = t360::floatBits(x * ratio) + static_cast<uint32_t>(nudge);
    checkPair((yb & 0x7fffffffu) | ((b >> 16 & 1u) << 31), t360::floatBits(x));
  }
}

}  // namespace

int main(int argc, char** argv) {
  const int threads = argc > 1 ? std::atoi(argv[1]) : 8;
  const unsigned long long pairs = argc > 2 ? std::strtoull(argv[2], nullptr, 10) : 100000000ull;
  const unsigned long long seed = argc > 3 ? std::strtoull(argv[3], nullptr, 10) : 1;

  // every combination of the special values
  std::vector<uint32_t> special = {0x00000000u, 0x00000001u, 0x00000002u, 0x003fffffu, 0x007fffffu, 0x00800000u, 0x00800001u,
                                   0x3f800000u, 0x3f7fffffu, 0x3f800001u, 0x3ee00000u, 0x3edfffffu, 0x3f300000u, 0x3f2fffffu,
                                   0x3f980000u, 0x3f97ffffu, 0x401c0000u, 0x401bffffu, 0x4c000000u, 0x4bffffffu, 0x31000000u,
                                   0x30ffffffu, 0x7f7fffffu, 0x7f800000u, 0x7fc00000u, 0x7f800001u, 0x7fffffffu, 0x3f000000u};
  const size_t base = special.size();
  for (size_t i = 0; i < base; ++i) special.push_back(special[i] | 0x80000000u);
  for (uint32_t y : special)
    for (uint32_t x : special) checkPair(y, x);

  std::vector<std::thread> pool;
  const uint64_t total = 1ull << 32, chunk = total / threads + 1;
  for (int t = 0; t < threads; ++t) {
    pool.emplace_back([=] {
      const uint64_t b = t * chunk, e = b + chunk < total ? b + chunk : total;
      checkUnary("asinf", asinf, t360::libmAsinf, b, e);
      checkUnary("atanf", atanf, t360::libmAtanf, b, e);
      randomPairs(seed * 1000003ull + t, pairs / threads + (static_cast<unsigned long long>(t) < pairs % threads ? 1 : 0));
    });
  }
  for (auto& th : pool) th.join();
  std::printf("asinf: 2^32 inputs, atanf: 2^32 inputs, atan2f: %llu random + %zu special pairs; %llu mismatches\n", pairs,
              special.size() * special.size(), gMismatches.load());
  return gMismatches.load() ? 1 : 0;
}
