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

#include "atan2_pairs.h"
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

// pairs [begin, end) of stream `seed` (atan2_pairs.h)
void randomPairs(uint64_t seed, uint64_t begin, uint64_t end) {
  for (uint64_t i = begin; i < end; ++i) {
    uint32_t y, x;
    t360gate::atan2RandomPair(seed, i, &y, &x);
    checkPair(y, x);
  }
}

}  // namespace

int main(int argc, char** argv) {
  const int threads = argc > 1 ? std::atoi(argv[1]) : 8;
  const unsigned long long pairs = argc > 2 ? std::strtoull(argv[2], nullptr, 10) : 100000000ull;
  const unsigned long long seed = argc > 3 ? std::strtoull(argv[3], nullptr, 10) : 1;

  // every combination of the special values
  for (int k = 0; k < t360gate::kAtan2Specials * t360gate::kAtan2Specials; ++k) {
    uint32_t y, x;
    t360gate::atan2SpecialPair(k, &y, &x);
    checkPair(y, x);
  }

  std::vector<std::thread> pool;
  const uint64_t total = 1ull << 32, chunk = total / threads + 1;
  for (int t = 0; t < threads; ++t) {
    pool.emplace_back([=] {
      const uint64_t b = t * chunk, e = b + chunk < total ? b + chunk : total;
      checkUnary("asinf", asinf, t360::libmAsinf, b, e);
      checkUnary("atanf", atanf, t360::libmAtanf, b, e);
      randomPairs(seed, pairs * t / threads, pairs * (t + 1) / threads);
    });
  }
  for (auto& th : pool) th.join();
  std::printf("asinf: 2^32 inputs, atanf: 2^32 inputs, atan2f: %llu random + %d special pairs; %llu mismatches\n", pairs,
              t360gate::kAtan2Specials * t360gate::kAtan2Specials, gMismatches.load());
  return gMismatches.load() ? 1 : 0;
}
