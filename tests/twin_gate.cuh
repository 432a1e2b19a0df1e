// Host / device twin gates: the device build of float functions of the per-frame position chains (csrc/flat_view.h,
// libm_ports.h, oriented_view.h) against their host build, the one the planner and the host twins run.  This header is
// the harness every gate shares (tests/*twin_gate.cu); tests/test_twin_gates.py builds each gate with the library's own
// nvcc flags (transform360_b200/build.py: ARCH, -O3, HOST_FLAGS) and runs it.
//
// A probe is a T360_HD function of an index i: it draws its inputs from (probe, i) alone -- a Draw, a splitmix64 stream
// seeded with a hash of (the gate's seed, probe, i) -- calls one twin function or chain, and packs the result into the
// gate's kOut 32-bit words.  The same probe code runs in a kernel on the device and in a thread pool on the host.  Tiers:
// a fullOnly probe takes every 32-bit pattern and runs in the full gate only; the others draw structured families
// (arbitrary bit patterns, special values, values a few ulps either side of each branch threshold and realistic values)
// or run whole chains over seeded geometries.
//
// Comparison: integer words compare raw, float words bit for bit (-0 against +0 included), with one exception: every NaN
// equals every NaN (each probe writes a NaN float as 0x7fc00000, fw).  x86 propagates a NaN's payload and sm_90 returns
// the canonical NaN; no record depends on a payload (roundHalfEven maps every NaN to INT_MIN).  There is no other
// exception.
//
// Each half sums a 64-bit mix of (probe, i, words) over each block of 2^20 inputs: an order-independent fingerprint.  The
// host compares the fingerprints; for up to 16 mismatching blocks per probe both halves re-evaluate the block element by
// element, and at most 20 lines `probe i input-bits host-bits device-bits` are printed, then the probes that mismatch.  A
// mismatching block that is not re-evaluated counts as one mismatch.  The last line is `<P> probes, <N> inputs, <M>
// mismatches`; the exit status is 1 on any mismatch.
//
//   gate [--threads T] [--shift S]     the full gate (2^S times fewer inputs per probe; a fullOnly probe samples one
//                                      pattern in 2^S)
//   gate --host-only [--threads T]     the host half of the probes that are not fullOnly at 2^20 inputs each, per-probe
//                                      fingerprints printed; no CUDA runtime call
//   gate --self-test [--threads T]     the host half against a copy of itself with one bit of one word flipped (kFlip)
//   gate --ledger [--threads T]        `class <probe> <class> <count>`: how many of the --host-only inputs (a prefix of
//                                      the full gate's) reach each input class a probe names and marks with CLASS
//
// A gate is a type G with
//   kSeed, kOut, kProbes, and kInfo[kProbes], a ProbeInfo per probe;
//   template <int P> static T360_HD void probe(const Data&, uint64_t i, Words<kOut>&), which finds the words zeroed;
//   HostData makeData(), its shared data built on the host; Data view(const HostData&, int shift), the view a probe
//   reads on the host; Data deviceData(const HostData&, Data, Uploads&), the same view of device copies;
//   kFlip, the self-test's flipped probe, element, word and bit.
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <atomic>
#include <chrono>
#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <string>
#include <thread>
#include <type_traits>
#include <utility>
#include <vector>

#include "atan2_pairs.h"
#include "oriented_view.h"

namespace t360gate {

constexpr uint64_t kBlock = 1ull << 20;

// ---- inputs -----------------------------------------------------------------------------------------------------------
// The draws of one (probe, i): a splitmix64 stream from a hash of (seed, probe, i), so inputs do not depend on the order
// or the thread that evaluates them.  Every float it makes is exact (integer scaling by powers of two) or made with the
// twin operations, so both halves see the same bits.
struct Draw {
  uint64_t s;
  T360_HD Draw(uint64_t seed, int probe, uint64_t i) : s(mix64(seed ^ (static_cast<uint64_t>(probe) << 56) ^ mix64(i))) {}
  T360_HD uint32_t u32() {
    s += 0x9e3779b97f4a7c15ull;
    return static_cast<uint32_t>(mix64(s) >> 32);
  }
  T360_HD int below(int n) { return static_cast<int>(u32() % static_cast<uint32_t>(n)); }
  T360_HD bool coin() { return u32() & 1u; }
  T360_HD float unit() { return static_cast<float>(u32() >> 8) * 0x1p-24f; }  // [0, 1), exact
  T360_HD float range(float a, float b) { return t360::fAdd(a, t360::fMul(t360::fSub(b, a), unit())); }
  T360_HD float sign(float v) { return coin() ? -v : v; }
  T360_HD float bits() { return t360::bitsFloat(u32()); }
  // +-0, +-1, +-0.5, +-inf, NaN, a subnormal, the largest float, a tiny normal
  T360_HD float special() {
    const uint32_t v[] = {0x00000000u, 0x3f800000u, 0x3f000000u, 0x7f800000u, 0x7fc00000u, 0x00000001u, 0x007fffffu, 0x7f7fffffu, 0x00800000u};
    return sign(t360::bitsFloat(v[below(9)]));
  }
  // a component of a ray or differential: mostly realistic, sometimes tiny, exactly zero or special
  T360_HD float component(float scale) {
    const int c = below(16);
    if (c == 0) return sign(0.0f);
    if (c == 1) return special();
    if (c == 2) return sign(t360::fMul(range(0.0f, 1.0f), 1e-6f));
    return t360::fMul(range(-1.0f, 1.0f), scale);
  }
};
// a ray or differential of three components (x, y, z drawn in that order)
T360_HD t360::SphereVec drawVec(Draw& d, float scale) { return t360::SphereVec{d.component(scale), d.component(scale), d.component(scale)}; }

struct HostRng {  // host-only draws for building a gate's shared data (double, libm: not part of any probe's inputs)
  uint64_t s;
  uint64_t next() { return mix64(s++); }
  double uniform(double a, double b) { return a + (b - a) * static_cast<double>(next() >> 11) * 0x1p-53; }
  int below(int n) { return static_cast<int>(next() % static_cast<uint64_t>(n)); }
};

// ---- outputs ----------------------------------------------------------------------------------------------------------
T360_HD uint32_t fw(float f) { return f != f ? 0x7fc00000u : t360::floatBits(f); }  // the canonical word of a float result
T360_HD uint32_t iw(int v) { return static_cast<uint32_t>(v); }

template <int N>
struct Words {
  uint32_t in[4];   // the inputs a drill-down prints
  uint32_t out[N];  // the compared words
  uint64_t cls;     // ledger classes (host only)
};

// CLASS(k, cond): the element is in ledger class k of its probe (the k-th name of ProbeInfo::classes)
#ifdef __CUDA_ARCH__
#define CLASS(k, cond) ((void)0)
#else
#define CLASS(k, cond) (w.cls |= (cond) ? (1ull << (k)) : 0ull)
#endif

struct ProbeInfo {
  const char* name;
  const char* classes;  // the ledger's class names in CLASS order, space-separated ("-": not a class of this probe)
  uint64_t inputs;      // in the full gate
  bool fullOnly;        // every 32-bit pattern, run in the full gate only
};

struct Flip {  // the self-test's flipped bit
  int probe;
  uint64_t element;
  int word, bit;
};

template <int N>
T360_HD uint64_t elementMix(int p, uint64_t i, const uint32_t* out) {
  uint64_t h = mix64((static_cast<uint64_t>(p) << 56) ^ i);
  for (int k = 0; k < N; ++k) h = mix64(h ^ (static_cast<uint64_t>(out[k]) << (k & 1 ? 32 : 0)) ^ static_cast<uint64_t>(k));
  return h;
}

template <class G, int P>
T360_HD void evaluate(const typename G::Data& D, uint64_t i, Words<G::kOut>& w) {
  w = Words<G::kOut>{};
  G::template probe<P>(D, i, w);
}

// f(std::integral_constant<int, P>{}) for P == p: a probe index chosen at run time, the probe's code at compile time
template <class F, int... P>
void withProbe(int p, F&& f, std::integer_sequence<int, P...>) {
  ((p == P ? f(std::integral_constant<int, P>{}) : void()), ...);
}
template <class G, class F>
void withProbe(int p, F&& f) {
  withProbe(p, f, std::make_integer_sequence<int, G::kProbes>());
}

// ---- the device half --------------------------------------------------------------------------------------------------
template <class G, int P>
__global__ void __launch_bounds__(256) fingerprintKernel(typename G::Data D, uint64_t inputs, uint64_t firstBlock, unsigned long long* fp) {
  const uint64_t block = firstBlock + blockIdx.x, begin = block * kBlock, end = begin + kBlock < inputs ? begin + kBlock : inputs;
  unsigned long long sum = 0;
  Words<G::kOut> w;
  for (uint64_t i = begin + threadIdx.x; i < end; i += blockDim.x) {
    evaluate<G, P>(D, i, w);
    sum += elementMix<G::kOut>(P, i, w.out);
  }
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_down_sync(0xffffffffu, sum, o);
  __shared__ unsigned long long warpSum[8];
  if ((threadIdx.x & 31) == 0) warpSum[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; ++k) sum += warpSum[k];
    fp[block] = sum;
  }
}
template <class G, int P>
__global__ void wordsKernel(typename G::Data D, uint64_t begin, uint64_t count, uint32_t* out) {
  for (uint64_t k = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; k < count; k += gridDim.x * static_cast<uint64_t>(blockDim.x)) {
    Words<G::kOut> w;
    evaluate<G, P>(D, begin + k, w);
    for (int q = 0; q < G::kOut; ++q) out[G::kOut * k + q] = w.out[q];
  }
}

#define CUDA_OK(x)                                                                          \
  do {                                                                                      \
    const cudaError_t e_ = (x);                                                             \
    if (e_ != cudaSuccess) {                                                                \
      std::fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
      std::exit(2);                                                                         \
    }                                                                                       \
  } while (0)

// Device copies of a gate's host vectors, freed together
struct Uploads {
  std::vector<void*> copies;
  template <class T>
  T* operator()(const std::vector<T>& v) {
    T* d = nullptr;
    CUDA_OK(cudaMalloc(&d, v.size() * sizeof(T)));
    CUDA_OK(cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    copies.push_back(d);
    return d;
  }
  ~Uploads() {
    for (void* d : copies) cudaFree(d);
  }
};

// ---- the host half ----------------------------------------------------------------------------------------------------
using ProbeList = std::vector<std::pair<int, uint64_t>>;  // (probe, inputs)

inline uint64_t blocksOf(uint64_t inputs) { return (inputs + kBlock - 1) / kBlock; }
inline uint64_t blockEnd(uint64_t b, uint64_t inputs) { return std::min(inputs, (b + 1) * kBlock); }

// fn(p, block, inputs) over every block of the given probes on `threads` threads, one block at a time per thread
inline void forBlocks(int threads, const ProbeList& probes, const std::function<void(int, uint64_t, uint64_t)>& fn) {
  std::vector<std::array<uint64_t, 3>> tasks;  // probe, block, inputs
  for (auto [p, inputs] : probes)
    for (uint64_t b = 0; b < blocksOf(inputs); ++b) tasks.push_back({static_cast<uint64_t>(p), b, inputs});
  std::atomic<size_t> next{0};
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; ++t)
    pool.emplace_back([&] {
      for (size_t k; (k = next.fetch_add(1)) < tasks.size();) fn(static_cast<int>(tasks[k][0]), tasks[k][1], tasks[k][2]);
    });
  for (auto& th : pool) th.join();
}

// the host build of probe p: one out-of-line copy per probe, called through a pointer
template <class G>
auto hostProbe(int p) {
  void (*f)(const typename G::Data&, uint64_t, Words<G::kOut>&) = nullptr;
  withProbe<G>(p, [&](auto P) { f = &evaluate<G, decltype(P)::value>; });
  return f;
}

// fn(i, words) for every element i in [begin, end) of probe p, evaluated on the host
template <class G, class F>
void forElements(const typename G::Data& D, int p, uint64_t begin, uint64_t end, F&& fn) {
  const auto probe = hostProbe<G>(p);
  Words<G::kOut> w;
  for (uint64_t i = begin; i < end; ++i) {
    probe(D, i, w);
    fn(i, w);
  }
}

template <class G>
void hostWords(const typename G::Data& D, int p, uint64_t begin, uint64_t count, std::vector<uint32_t>& words) {
  words.assign(G::kOut * count, 0);
  forElements<G>(D, p, begin, begin + count, [&](uint64_t i, const Words<G::kOut>& w) { std::memcpy(&words[G::kOut * (i - begin)], w.out, sizeof(w.out)); });
}

// The host half's fingerprints of every probe in `probes`, computed together so the thread pool stays busy
template <class G>
std::vector<std::vector<uint64_t>> hostFingerprints(const typename G::Data& D, int threads, const ProbeList& probes) {
  std::vector<std::vector<uint64_t>> fp(G::kProbes);
  for (auto [p, inputs] : probes) fp[p].assign(blocksOf(inputs), 0);
  forBlocks(threads, probes, [&](int p, uint64_t b, uint64_t inputs) {
    uint64_t sum = 0;
    forElements<G>(D, p, b * kBlock, blockEnd(b, inputs), [&](uint64_t i, const Words<G::kOut>& w) { sum += elementMix<G::kOut>(p, i, w.out); });
    fp[p][b] = sum;
  });
  return fp;
}

// A half gives the block fingerprints of a probe and, for a drill-down, the words of one block.
struct Half {
  std::function<void(int p, uint64_t inputs, std::vector<uint64_t>& fp)> fingerprints;
  std::function<void(int p, uint64_t begin, uint64_t count, std::vector<uint32_t>& words)> words;
};

inline std::string hexWords(const uint32_t* w, int n) {
  std::string s;
  char buf[16];
  for (int k = 0; k < n; ++k) {
    std::snprintf(buf, sizeof(buf), k ? ":%08x" : "%08x", w[k]);
    s += buf;
  }
  return s;
}

// Compares the host half's fingerprints with the other half's, drills into mismatching blocks; returns the mismatches
template <class G>
uint64_t compare(const typename G::Data& D, const ProbeList& probes, const std::vector<std::vector<uint64_t>>& hostFp, const Half& other,
                 uint64_t* totalInputs) {
  constexpr int N = G::kOut;
  uint64_t mismatches = 0;
  int printed = 0;
  std::string failing;
  for (auto [p, inputs] : probes) {
    const uint64_t before = mismatches;
    *totalInputs += inputs;
    std::vector<uint64_t> fp;
    other.fingerprints(p, inputs, fp);
    int drilled = 0;
    for (uint64_t b = 0; b < hostFp[p].size(); ++b) {
      if (hostFp[p][b] == fp[b]) continue;
      if (drilled++ >= 16) {
        ++mismatches;
        continue;
      }
      const uint64_t begin = b * kBlock, count = blockEnd(b, inputs) - begin;
      std::vector<uint32_t> hw, ow;
      hostWords<G>(D, p, begin, count, hw);
      other.words(p, begin, count, ow);
      for (uint64_t k = 0; k < count; ++k) {
        if (std::memcmp(&hw[N * k], &ow[N * k], N * 4) == 0) continue;
        ++mismatches;
        if (printed++ < 20) {
          Words<N> w;
          hostProbe<G>(p)(D, begin + k, w);
          std::printf("%s %" PRIu64 " %s %s %s\n", G::kInfo[p].name, begin + k, hexWords(w.in, 4).c_str(), hexWords(&hw[N * k], N).c_str(),
                      hexWords(&ow[N * k], N).c_str());
        }
      }
    }
    if (mismatches > before) failing += std::string(" ") + G::kInfo[p].name;
  }
  if (!failing.empty()) std::printf("mismatching probes:%s\n", failing.c_str());
  return mismatches;
}

// ---- the gate ---------------------------------------------------------------------------------------------------------
template <class G>
int runGate(int argc, char** argv) {
  constexpr int N = G::kOut;
  int threads = static_cast<int>(std::thread::hardware_concurrency());
  int shift = 0;
  std::string mode = "full";
  for (int a = 1; a < argc; ++a) {
    const std::string s = argv[a];
    if (s == "--threads" && a + 1 < argc) threads = std::atoi(argv[++a]);
    else if (s == "--shift" && a + 1 < argc) shift = std::atoi(argv[++a]);
    else if (s == "--host-only" || s == "--self-test" || s == "--ledger") mode = s.substr(2);
    else {
      std::fprintf(stderr, "usage: %s [--threads T] [--shift S] [--host-only | --self-test | --ledger]\n", argv[0]);
      return 2;
    }
  }
  threads = std::max(1, threads);
  const typename G::HostData H = G::makeData();
  const typename G::Data hostD = G::view(H, shift);

  ProbeList probes;
  for (int p = 0; p < G::kProbes; ++p) {
    if (mode != "full" && G::kInfo[p].fullOnly) continue;
    uint64_t n = mode == "full" ? std::max<uint64_t>(G::kInfo[p].inputs >> shift, 1) : std::min(G::kInfo[p].inputs, kBlock);
    if (mode == "self-test" && p == G::kFlip.probe) n = std::max(n, (G::kFlip.element / kBlock + 1) * kBlock);
    probes.push_back({p, n});
  }

  if (mode == "ledger") {
    std::vector<std::array<std::atomic<uint64_t>, 64>> counts(G::kProbes);
    forBlocks(threads, probes, [&](int p, uint64_t b, uint64_t inputs) {
      uint64_t local[64] = {};
      forElements<G>(hostD, p, b * kBlock, blockEnd(b, inputs), [&](uint64_t, const Words<N>& w) {
        for (int k = 0; k < 64; ++k) local[k] += (w.cls >> k) & 1u;
      });
      for (int k = 0; k < 64; ++k) counts[p][k] += local[k];
    });
    for (auto [p, inputs] : probes) {
      const std::string names = G::kInfo[p].classes;
      size_t at = 0;
      for (int k = 0; at < names.size(); ++k) {
        const size_t sp = names.find(' ', at);
        const std::string name = names.substr(at, sp == std::string::npos ? std::string::npos : sp - at);
        at = sp == std::string::npos ? names.size() : sp + 1;
        if (name != "-") std::printf("class %s %s %" PRIu64 "\n", G::kInfo[p].name, name.c_str(), counts[p][k].load());
      }
    }
    return 0;
  }

  const auto t0 = std::chrono::steady_clock::now();
  const std::vector<std::vector<uint64_t>> hostFp = hostFingerprints<G>(hostD, threads, probes);
  const double hostSeconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();

  if (mode == "host-only") {
    for (auto [p, inputs] : probes) {
      uint64_t h = 0;
      for (uint64_t f : hostFp[p]) h = mix64(h ^ f);
      std::printf("fingerprint %s %" PRIu64 " %016" PRIx64 "\n", G::kInfo[p].name, inputs, h);
    }
    std::printf("host %.1f s on %d threads\n", hostSeconds, threads);
    return 0;
  }

  uint64_t totalInputs = 0, mismatches = 0;
  if (mode == "self-test") {
    // the other half: the host half with one bit flipped, its fingerprints taken from its words so the drill-down's
    // words and the fingerprints' are checked against each other for every probe
    constexpr Flip f = G::kFlip;
    Half flipped;
    flipped.words = [&](int p, uint64_t begin, uint64_t count, std::vector<uint32_t>& words) {
      hostWords<G>(hostD, p, begin, count, words);
      if (p == f.probe && f.element >= begin && f.element < begin + count) words[N * (f.element - begin) + f.word] ^= 1u << f.bit;
    };
    flipped.fingerprints = [&](int p, uint64_t inputs, std::vector<uint64_t>& out) {
      out.assign(blocksOf(inputs), 0);
      for (uint64_t b = 0; b < out.size(); ++b) {
        const uint64_t begin = b * kBlock, count = blockEnd(b, inputs) - begin;
        std::vector<uint32_t> words;
        flipped.words(p, begin, count, words);
        for (uint64_t k = 0; k < count; ++k) out[b] += elementMix<N>(p, begin + k, &words[N * k]);
      }
    };
    mismatches = compare<G>(hostD, probes, hostFp, flipped, &totalInputs);
    std::printf("self-test: flipped %s %" PRIu64 " word %d bit %d\n", G::kInfo[f.probe].name, f.element, f.word, f.bit);
  } else {
    Uploads uploads;
    const typename G::Data devD = G::deviceData(H, hostD, uploads);
    unsigned long long* dFp = nullptr;
    uint32_t* dWords = nullptr;
    uint64_t maxBlocks = 0;
    for (auto [p, inputs] : probes) maxBlocks = std::max(maxBlocks, blocksOf(inputs));
    CUDA_OK(cudaMalloc(&dFp, maxBlocks * sizeof(unsigned long long)));
    CUDA_OK(cudaMalloc(&dWords, N * kBlock * sizeof(uint32_t)));
    cudaEvent_t e0, e1;
    CUDA_OK(cudaEventCreate(&e0));
    CUDA_OK(cudaEventCreate(&e1));
    float deviceMs = 0.0f;
    Half device;
    device.fingerprints = [&](int p, uint64_t inputs, std::vector<uint64_t>& out) {
      const uint64_t blocks = blocksOf(inputs);
      CUDA_OK(cudaEventRecord(e0));
      withProbe<G>(p, [&](auto P) {
        for (uint64_t b = 0; b < blocks; b += 65535) {
          fingerprintKernel<G, decltype(P)::value><<<static_cast<unsigned>(std::min<uint64_t>(65535, blocks - b)), 256>>>(devD, inputs, b, dFp);
          CUDA_OK(cudaGetLastError());
        }
      });
      CUDA_OK(cudaEventRecord(e1));
      CUDA_OK(cudaEventSynchronize(e1));
      float ms;
      CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
      deviceMs += ms;
      out.resize(blocks);
      CUDA_OK(cudaMemcpy(out.data(), dFp, blocks * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    };
    device.words = [&](int p, uint64_t begin, uint64_t count, std::vector<uint32_t>& words) {
      withProbe<G>(p, [&](auto P) { wordsKernel<G, decltype(P)::value><<<1024, 256>>>(devD, begin, count, dWords); });
      CUDA_OK(cudaGetLastError());
      words.resize(N * count);
      CUDA_OK(cudaMemcpy(words.data(), dWords, N * count * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    };
    mismatches = compare<G>(hostD, probes, hostFp, device, &totalInputs);
    std::printf("device %.1f s, host %.1f s on %d threads\n", deviceMs / 1000.0, hostSeconds, threads);
    cudaFree(dFp); cudaFree(dWords);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
  }
  std::printf("%zu probes, %" PRIu64 " inputs, %" PRIu64 " mismatches\n", probes.size(), totalInputs, mismatches);
  return mismatches ? 1 : 0;
}

}  // namespace t360gate
