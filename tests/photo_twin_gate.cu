// Host / device twin gate of the lens photometry: the device build of the float function it adds (oriented_view.h:
// lensGain, the falloff and the gain's quantisation) and of the chains that call it (lensPhotoPosition, lensPhotoPoint,
// lensPhotoSample) against their host build, the one T360B200_lensPhotoMaps runs.  tests/test_photo_twins.py builds it
// with the library's own nvcc flags (transform360_b200/build.py: ARCH, -O3, HOST_FLAGS) and runs it.  Its design is
// tests/twin_gate.cu's and tests/mip_twin_gate.cu's: hash-drawn inputs, per-block order-independent fingerprints, element
// re-evaluation of mismatching blocks, floats compared bit for bit (every NaN written as 0x7fc00000).
// Probes:
//   lensGain           lensHit<true> of drawn directions and lenses, then lensGain with drawn falloffs and gains; the
//                      ledger's classes: r = 0 (a ray on the lens axis), theta = thetaMax (the lens's bound set to the
//                      ray's own theta), V near the refusal bound (v1 = -(1 - e) / r^2, e down to 2^-20), Gq at its clamp
//                      (G >= 16), and rays the lens does not cover;
//   lensPhotoPosition  drawn rig directions, hard (both = false and true) and feathered seams;
//   lensPhotoSample<BARREL> / <plain>: 2^24 (geometry, pixel) samples each over seeded contexts, rigs and photometries.
//
//   photo_twin_gate [--threads T] [--shift S]     the full gate (2^S times fewer inputs per probe)
//   photo_twin_gate --host-only [--threads T]     the host half at 2^20 inputs per probe, fingerprints printed; no CUDA call
//   photo_twin_gate --self-test [--threads T]     the host half against a copy of itself with one bit of one word flipped
//   photo_twin_gate --ledger [--threads T]        per-probe counts of the classes above over the --host-only inputs
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
#include <utility>
#include <vector>

#include "atan2_pairs.h"
#include "oriented_view.h"

using namespace t360;
using t360gate::mix64;

namespace {

constexpr int kBlockShift = 20;
constexpr uint64_t kBlock = 1ull << kBlockShift;
constexpr uint64_t kSeed = 20261019ull;
constexpr int kOut = 6;

struct Draw {
  uint64_t s;
  T360_HD Draw(int probe, uint64_t i) : s(mix64(kSeed ^ (static_cast<uint64_t>(probe) << 56) ^ mix64(i))) {}
  T360_HD uint32_t u32() {
    s += 0x9e3779b97f4a7c15ull;
    return static_cast<uint32_t>(mix64(s) >> 32);
  }
  T360_HD int below(int n) { return static_cast<int>(u32() % static_cast<uint32_t>(n)); }
  T360_HD bool coin() { return u32() & 1u; }
  T360_HD float unit() { return static_cast<float>(u32() >> 8) * 0x1p-24f; }  // [0, 1), exact
  T360_HD float range(float a, float b) { return fAdd(a, fMul(fSub(b, a), unit())); }
  T360_HD float sign(float v) { return coin() ? -v : v; }
  T360_HD float special() {  // +-0, +-1, +-0.5, +-inf, NaN, a subnormal, the largest float, a tiny normal
    const uint32_t v[] = {0x00000000u, 0x3f800000u, 0x3f000000u, 0x7f800000u, 0x7fc00000u, 0x00000001u, 0x007fffffu, 0x7f7fffffu, 0x00800000u};
    return sign(bitsFloat(v[below(9)]));
  }
  // a component of a ray or differential: mostly realistic, sometimes tiny, exactly zero or special
  T360_HD float component(float scale) {
    const int c = below(16);
    if (c == 0) return sign(0.0f);
    if (c == 1) return special();
    if (c == 2) return sign(fMul(range(0.0f, 1.0f), 1e-6f));
    return fMul(range(-1.0f, 1.0f), scale);
  }
};

T360_HD uint32_t fw(float f) { return f != f ? 0x7fc00000u : floatBits(f); }
T360_HD uint32_t iw(int v) { return static_cast<uint32_t>(v); }

struct Words {
  uint32_t in[4];
  uint32_t out[kOut];
  uint32_t cls;  // ledger classes (host only)
};

// ---- data the probes share (host-built, copied to the device) --------------------------------------------------------
struct ChainGeo {
  SphereGeometry g;  // a lens rig's output geometry (mono, equirect-like input fields)
  Rotation r;
  float seam;        // seamScale (0: the hard seam)
  bool both;
  bool barrel;
  int colOffset, rowOffset;  // of its sphere tables in GateData::tables (-1: none)
};
struct GateData {
  const LensRigModel* rig;
  int nRig, nRigAxis;  // [0, nRigAxis): lenses along +-z (rho = 0 reachable)
  const LensPhotoPlane* photo;
  int nPhoto;
  const ChainGeo* geo;
  int nGeo;
  const float* tables;  // every geometry's sphere tables, back to back
};

T360_HD SphereVec drawVec(Draw& d, float scale) { return SphereVec{d.component(scale), d.component(scale), d.component(scale)}; }

enum Probe { kGain, kPosition, kSampleBarrel, kSamplePlain, kProbes };
struct ProbeInfo {
  const char* name;
  uint64_t inputs;
};
const ProbeInfo kInfo[kProbes] = {
    {"lensGain", 1ull << 28}, {"lensPhotoPosition", 1ull << 26}, {"lensPhotoSample<BARREL>", 1ull << 24}, {"lensPhotoSample<plain>", 1ull << 24}};
const char* const kGainClasses[] = {"r0", "thetaMax", "nearBound", "clamp", "uncovered"};
enum { kClsR0 = 1, kClsThetaMax = 2, kClsNearBound = 4, kClsClamp = 8, kClsUncovered = 16 };

template <int P>
T360_HD void probe(const GateData& D, uint64_t i, Words& w) {
  Draw d(P, i);
  for (uint32_t& o : w.out) o = 0;
  for (uint32_t& o : w.in) o = 0;
  w.cls = 0;
  if constexpr (P == kGain) {
    const bool axis = d.below(8) == 0;
    LensModel L = D.rig[axis ? d.below(D.nRigAxis) : d.below(D.nRig)].lens[0];
    SphereVec t = axis ? SphereVec{d.sign(0.0f), d.sign(0.0f), d.range(0.1f, 2.0f)} : drawVec(d, 1.0f);
    const int cls = d.below(4);
    if (cls == 1) {  // the lens's bound exactly at this ray's theta
      const LensHitR h = lensHit<true>(L, t, lensRow(L.m + 6, t), 1000, 1000);
      if (h.theta == h.theta) L.thetaMax = h.theta;
    }
    const LensHitR h = lensHit<true>(L, t, lensRow(L.m + 6, t), 16 + d.below(8000), 16 + d.below(8000));
    float v[3] = {d.range(-0.3f, 0.1f), d.range(-0.05f, 0.05f), d.range(-0.005f, 0.005f)};
    float gain = d.coin() ? d.range(0.001f, 8.0f) : d.range(0.9f, 1.1f);
    if (cls == 2 && h.covered && h.r > 0.0f) {  // V near 0: v1 = -(1 - e) / r^2
      const float e = fDiv(1.0f, static_cast<float>(1u << d.below(21)));
      v[0] = fDiv(fSub(e, 1.0f), fMul(h.r, h.r));
      v[1] = v[2] = 0.0f;
    }
    if (cls == 3) {  // G >= 16 and around it
      gain = d.range(7.0f, 8.0f);
      v[0] = fDiv(d.range(-0.75f, -0.4f), fAdd(fMul(h.r == h.r ? h.r : 1.0f, h.r == h.r ? h.r : 1.0f), 1e-3f));
    }
    const int gq = lensGain(h, v, gain);
    w.in[0] = floatBits(t.x); w.in[1] = floatBits(t.y); w.in[2] = floatBits(v[0]); w.in[3] = floatBits(gain);
    w.out[0] = iw(gq); w.out[1] = fw(h.r); w.out[2] = fw(h.theta); w.out[3] = iw(h.covered);
    if (!h.covered) w.cls |= kClsUncovered;
    if (h.covered && h.r == 0.0f) w.cls |= kClsR0;
    if (h.covered && h.theta == L.thetaMax) w.cls |= kClsThetaMax;
    if (cls == 2 && h.covered && h.r > 0.0f && gq > 0) w.cls |= kClsNearBound;
    if (gq == 65535) w.cls |= kClsClamp;
  } else if constexpr (P == kPosition) {
    const bool axis = d.below(4) == 0;
    const LensRigModel& rig = D.rig[axis ? d.below(D.nRigAxis) : d.below(D.nRig)];
    SphereVec t = drawVec(d, 1.0f);
    if (axis) t = SphereVec{d.sign(0.0f), d.sign(0.0f), d.sign(d.range(0.1f, 2.0f))};
    const LensPhotoPlane& c = D.photo[d.below(D.nPhoto)];
    const float s = rig.numLenses > 1 && d.coin() ? d.range(0.3f, 30.0f) : 0.0f;
    const bool both = d.coin();
    const int inW = 16 + d.below(8000), inH = 16 + d.below(8000);
    float p0[2], p1[2];
    int g0, g1;
    bool overlap;
    const int wt = lensPhotoPosition(rig, s, both, c, t, inW, inH, p0, p1, &g0, &g1, &overlap);
    w.in[0] = floatBits(t.x); w.in[1] = floatBits(t.y); w.in[2] = floatBits(t.z); w.in[3] = floatBits(s);
    w.out[0] = fw(p0[0]); w.out[1] = fw(p0[1]); w.out[2] = fw(p1[0]); w.out[3] = fw(p1[1]);
    w.out[4] = iw(wt) | iw(overlap) << 9 | iw(both) << 10; w.out[5] = iw(g0) | iw(g1) << 16;
  } else {
    int k = d.below(D.nGeo);
    while (D.geo[k].barrel != (P == kSampleBarrel)) k = d.below(D.nGeo);  // (the kernels' instantiation for the layout)
    const ChainGeo& e = D.geo[k];
    const LensRigModel& rig = D.rig[d.below(D.nRig)];
    const LensPhotoPlane& c = D.photo[d.below(D.nPhoto)];
    const float* colTab = e.colOffset < 0 ? nullptr : D.tables + e.colOffset;
    const float* rowTab = e.rowOffset < 0 ? nullptr : D.tables + e.rowOffset;
    const int row = d.below(e.g.mapH), col = d.below(e.g.mapW);
    const float s = rig.numLenses > 1 ? e.seam : 0.0f;
    int32_t r0[2], r1[2];
    int g0, g1;
    bool overlap;
    const int wt = P == kSampleBarrel ? lensPhotoSample<true>(e.g, e.r, rig, s, e.both, c, colTab, rowTab, row, col, r0, r1, &g0, &g1, &overlap)
                                      : lensPhotoSample<false>(e.g, e.r, rig, s, e.both, c, colTab, rowTab, row, col, r0, r1, &g0, &g1, &overlap);
    w.in[0] = iw(row); w.in[1] = iw(col); w.in[2] = iw(k); w.in[3] = floatBits(s);
    w.out[0] = iw(r0[0]); w.out[1] = iw(r0[1]); w.out[2] = iw(r1[0]); w.out[3] = iw(r1[1]);
    w.out[4] = iw(wt) | iw(overlap) << 9; w.out[5] = iw(g0) | iw(g1) << 16;
  }
}

using ProbeFn = void (*)(const GateData&, uint64_t, Words&);
template <int... P>
constexpr std::array<ProbeFn, sizeof...(P)> probeTable(std::integer_sequence<int, P...>) {
  return {&probe<P>...};
}
const auto kHostProbe = probeTable(std::make_integer_sequence<int, kProbes>());

T360_HD uint64_t elementMix(int p, uint64_t i, const uint32_t* out) {
  uint64_t h = mix64((static_cast<uint64_t>(p) << 56) ^ i);
  for (int k = 0; k < kOut; ++k) h = mix64(h ^ (static_cast<uint64_t>(out[k]) << (k & 1 ? 32 : 0)) ^ static_cast<uint64_t>(k));
  return h;
}

// ---- the device half --------------------------------------------------------------------------------------------------
template <int P>
__global__ void __launch_bounds__(256) fingerprintKernel(GateData D, uint64_t inputs, uint64_t firstBlock, unsigned long long* fp) {
  const uint64_t block = firstBlock + blockIdx.x, begin = block * kBlock, end = begin + kBlock < inputs ? begin + kBlock : inputs;
  unsigned long long sum = 0;
  Words w;
  for (uint64_t i = begin + threadIdx.x; i < end; i += blockDim.x) {
    probe<P>(D, i, w);
    sum += elementMix(P, i, w.out);
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
template <int P>
__global__ void wordsKernel(GateData D, uint64_t begin, uint64_t count, uint32_t* out) {
  for (uint64_t k = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; k < count; k += gridDim.x * static_cast<uint64_t>(blockDim.x)) {
    Words w;
    probe<P>(D, begin + k, w);
    for (int q = 0; q < kOut; ++q) out[kOut * k + q] = w.out[q];
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

using LaunchFp = void (*)(const GateData&, uint64_t, uint64_t, uint64_t, unsigned long long*);
using LaunchWords = void (*)(const GateData&, uint64_t, uint64_t, uint32_t*);
template <int P>
void launchFp(const GateData& D, uint64_t inputs, uint64_t first, uint64_t blocks, unsigned long long* fp) {
  fingerprintKernel<P><<<static_cast<unsigned>(blocks), 256>>>(D, inputs, first, fp);
  CUDA_OK(cudaGetLastError());
}
template <int P>
void launchWords(const GateData& D, uint64_t begin, uint64_t count, uint32_t* out) {
  wordsKernel<P><<<1024, 256>>>(D, begin, count, out);
  CUDA_OK(cudaGetLastError());
}
template <int... P>
constexpr std::array<LaunchFp, sizeof...(P)> fpTable(std::integer_sequence<int, P...>) { return {&launchFp<P>...}; }
template <int... P>
constexpr std::array<LaunchWords, sizeof...(P)> wordsTable(std::integer_sequence<int, P...>) { return {&launchWords<P>...}; }

// ---- the shared data --------------------------------------------------------------------------------------------------
struct HostData {
  std::vector<LensRigModel> rig;
  std::vector<LensPhotoPlane> photo;
  std::vector<ChainGeo> geo;
  std::vector<float> tables;
  int nRigAxis = 0;
};

struct HostRng {  // host-only draws for building the shared data (double, libm: not part of any probe's inputs)
  uint64_t s;
  uint64_t next() { return mix64(s++); }
  double uniform(double a, double b) { return a + (b - a) * static_cast<double>(next() >> 11) * 0x1p-53; }
  int below(int n) { return static_cast<int>(next() % static_cast<uint64_t>(n)); }
};

HostData makeData() {
  HostData H;
  HostRng g{kSeed * 7919};
  auto angle = [&] { return g.below(4) == 0 ? static_cast<float>(90 * g.below(4)) : static_cast<float>(g.uniform(-180, 180)); };
  // rigs: lenses along +-z first (their axes reach rho = 0 exactly), then rotated ones
  auto lens = [&](bool axisAligned, bool back) {
    LensModel L{};
    if (axisAligned) {
      const float m[9] = {back ? -1.0f : 1.0f, 0, 0, 0, -1.0f, 0, 0, 0, back ? -1.0f : 1.0f};
      std::memcpy(L.m, m, sizeof(m));
    } else {
      const Rotation r = rotationFromAngles(angle(), angle(), angle());
      const float m[9] = {r.xx, r.xy, r.xz, r.yx, r.yy, r.yz, r.zx, r.zy, r.zz};
      std::memcpy(L.m, m, sizeof(m));
    }
    L.ax = static_cast<float>(g.uniform(0.1, 0.5));
    L.bx = static_cast<float>(g.uniform(0.3, 0.7));
    L.ay = static_cast<float>(g.uniform(0.1, 0.5));
    L.by = static_cast<float>(g.uniform(0.3, 0.7));
    for (float& k : L.k) k = static_cast<float>(g.uniform(-0.05, 0.05));
    L.thetaMax = g.below(3) == 0 ? static_cast<float>(M_PI) : static_cast<float>(g.uniform(0.5, M_PI));
    return L;
  };
  for (int pass = 0; pass < 2; ++pass) {
    for (int k = 0; k < 64; ++k) {
      LensRigModel rig{};
      rig.numLenses = 1 + k % 2;
      rig.lens[0] = lens(pass == 0, false);
      if (rig.numLenses == 2) rig.lens[1] = lens(pass == 0, true);
      H.rig.push_back(rig);
    }
    if (pass == 0) H.nRigAxis = static_cast<int>(H.rig.size());
  }
  // photometries: the identity, then drawn falloffs, gains, offsets and pivots
  for (int k = 0; k < 64; ++k) {
    LensPhotoPlane c{};
    c.pivot = k == 0 ? 16 : (g.below(2) ? 128 : g.below(256));
    for (int i = 0; i < 2; ++i) {
      c.v[i][0] = k == 0 ? 0.0f : static_cast<float>(g.uniform(-0.2, 0.05));
      c.v[i][1] = k == 0 ? 0.0f : static_cast<float>(g.uniform(-0.02, 0.03));
      c.v[i][2] = k == 0 ? 0.0f : static_cast<float>(g.uniform(-0.002, 0.002));
      c.gain[i] = k == 0 ? 1.0f : static_cast<float>(g.uniform(0.01, 8.0));
      c.offset[i] = k == 0 ? 0 : g.below(2049) - 1024;
    }
    H.photo.push_back(c);
  }
  // geometries: every sphere output layout (barrel included), odd and even sizes, K = 1, 2, 4, 8, hard and feathered seams
  const int layouts[] = {LAYOUT_CUBEMAP_32, LAYOUT_CUBEMAP_23_OFFCENTER, LAYOUT_EAC_32, LAYOUT_EQUIRECT, LAYOUT_BARREL, LAYOUT_BARREL_SPLIT};
  for (int k = 0; k < 96; ++k) {
    FrameTransformContext c{};
    c.output_layout = static_cast<Layout>(layouts[k % 6]);
    c.input_layout = LAYOUT_EQUIRECT;
    c.input_stereo_format = c.output_stereo_format = STEREO_FORMAT_MONO;
    c.expand_coef = g.below(2) ? 1.0f : static_cast<float>(g.uniform(1.0, 1.2));
    c.input_expand_coef = 1.0f;
    c.width_scale_factor = c.height_scale_factor = 1.0f;
    c.vflip = g.below(2);
    if (g.below(3) == 0) { c.fixed_cube_offcenter_x = static_cast<float>(g.uniform(-0.3, 0.3)); c.fixed_cube_offcenter_z = static_cast<float>(g.uniform(-0.3, 0.3)); }
    ChainGeo e{};
    e.g = sphereGeometry(c, 8 + g.below(1500), 8 + g.below(1500), 16 + g.below(8000), 16 + g.below(8000), 1 << (k / 6) % 4);
    e.r = rotationFromAngles(angle(), angle(), angle());
    e.seam = g.below(2) ? 0.0f : static_cast<float>(1.0 / (2.0 * g.uniform(0.01, 180) * M_PI / 180.0));
    e.both = g.below(2);
    e.barrel = barrelLayout(c.output_layout);
    const std::vector<float> t = buildSphereTables(e.g);
    e.colOffset = t.empty() ? -1 : static_cast<int>(H.tables.size());
    e.rowOffset = t.empty() ? -1 : e.colOffset + static_cast<int>(sphereTableRowOffset(e.g));
    H.tables.insert(H.tables.end(), t.begin(), t.end());
    H.geo.push_back(e);
  }
  if (H.tables.empty()) H.tables.push_back(0.0f);
  return H;
}

GateData view(const HostData& H) {
  return GateData{H.rig.data(), static_cast<int>(H.rig.size()), H.nRigAxis, H.photo.data(), static_cast<int>(H.photo.size()),
                  H.geo.data(), static_cast<int>(H.geo.size()), H.tables.data()};
}

template <class T>
T* upload(const std::vector<T>& v) {
  T* d = nullptr;
  CUDA_OK(cudaMalloc(&d, v.size() * sizeof(T)));
  CUDA_OK(cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  return d;
}

// ---- the halves -------------------------------------------------------------------------------------------------------
struct Half {
  std::function<void(int p, uint64_t inputs, std::vector<uint64_t>& fp)> fingerprints;
  std::function<void(int p, uint64_t begin, uint64_t count, std::vector<uint32_t>& words)> words;
};

uint64_t blocksOf(uint64_t inputs) { return (inputs + kBlock - 1) / kBlock; }

uint64_t hostBlock(const GateData& D, int p, uint64_t b, uint64_t inputs) {
  const uint64_t begin = b * kBlock, end = std::min(inputs, begin + kBlock);
  uint64_t sum = 0;
  Words w;
  for (uint64_t i = begin; i < end; ++i) {
    kHostProbe[p](D, i, w);
    sum += elementMix(p, i, w.out);
  }
  return sum;
}

void hostWords(const GateData& D, int p, uint64_t begin, uint64_t count, std::vector<uint32_t>& words) {
  words.assign(kOut * count, 0);
  Words w;
  for (uint64_t k = 0; k < count; ++k) {
    kHostProbe[p](D, begin + k, w);
    std::memcpy(&words[kOut * k], w.out, sizeof(w.out));
  }
}

// The host half's block fingerprints of every probe, the blocks of all probes dealt to `threads` threads
std::vector<std::vector<uint64_t>> hostFingerprints(const GateData& D, int threads, const std::vector<std::pair<int, uint64_t>>& probes) {
  std::vector<std::vector<uint64_t>> fp(kProbes);
  std::vector<std::array<uint64_t, 3>> tasks;  // probe, block, inputs
  for (auto [p, inputs] : probes) {
    fp[p].assign(blocksOf(inputs), 0);
    for (uint64_t b = 0; b < blocksOf(inputs); ++b) tasks.push_back({static_cast<uint64_t>(p), b, inputs});
  }
  std::atomic<size_t> next{0};
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; ++t)
    pool.emplace_back([&] {
      for (size_t k; (k = next.fetch_add(1)) < tasks.size();) {
        const int p = static_cast<int>(tasks[k][0]);
        fp[p][tasks[k][1]] = hostBlock(D, p, tasks[k][1], tasks[k][2]);
      }
    });
  for (auto& th : pool) th.join();
  return fp;
}

std::string hexWords(const uint32_t* w, int n) {
  std::string s;
  char buf[16];
  for (int k = 0; k < n; ++k) {
    std::snprintf(buf, sizeof(buf), k ? ":%08x" : "%08x", w[k]);
    s += buf;
  }
  return s;
}

// Compares the host half's fingerprints with the other half's, drills into mismatching blocks; returns the mismatches
uint64_t compare(const GateData& D, const std::vector<std::pair<int, uint64_t>>& probes, const std::vector<std::vector<uint64_t>>& hostFp,
                 const Half& other, uint64_t* totalInputs) {
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
      const uint64_t begin = b * kBlock, count = std::min(inputs, begin + kBlock) - begin;
      std::vector<uint32_t> hw, ow;
      hostWords(D, p, begin, count, hw);
      other.words(p, begin, count, ow);
      for (uint64_t k = 0; k < count; ++k) {
        if (std::memcmp(&hw[kOut * k], &ow[kOut * k], kOut * 4) == 0) continue;
        ++mismatches;
        if (printed++ < 20) {
          Words w;
          kHostProbe[p](D, begin + k, w);
          std::printf("%s %" PRIu64 " %s %s %s\n", kInfo[p].name, begin + k, hexWords(w.in, 4).c_str(), hexWords(&hw[kOut * k], kOut).c_str(),
                      hexWords(&ow[kOut * k], kOut).c_str());
        }
      }
    }
    if (mismatches > before) failing += std::string(" ") + kInfo[p].name;
  }
  if (!failing.empty()) std::printf("mismatching probes:%s\n", failing.c_str());
  return mismatches;
}

double seconds(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

}  // namespace

int main(int argc, char** argv) {
  int threads = static_cast<int>(std::thread::hardware_concurrency());
  int shift = 0;
  std::string mode = "full";
  for (int a = 1; a < argc; ++a) {
    const std::string s = argv[a];
    if (s == "--threads" && a + 1 < argc) threads = std::atoi(argv[++a]);
    else if (s == "--shift" && a + 1 < argc) shift = std::atoi(argv[++a]);
    else if (s == "--host-only" || s == "--self-test" || s == "--ledger") mode = s.substr(2);
    else {
      std::fprintf(stderr, "usage: photo_twin_gate [--threads T] [--shift S] [--host-only | --self-test | --ledger]\n");
      return 2;
    }
  }
  threads = std::max(1, threads);
  const HostData H = makeData();
  const GateData hostD = view(H);

  std::vector<std::pair<int, uint64_t>> probes;
  for (int p = 0; p < kProbes; ++p) probes.push_back({p, mode == "full" ? std::max<uint64_t>(kInfo[p].inputs >> shift, 1) : kBlock});

  if (mode == "ledger") {  // the lensGain classes over the --host-only inputs
    uint64_t counts[5] = {};
    Words w;
    for (uint64_t i = 0; i < kBlock; ++i) {
      probe<kGain>(hostD, i, w);
      for (int c = 0; c < 5; ++c) counts[c] += (w.cls >> c) & 1u;
    }
    for (int c = 0; c < 5; ++c) std::printf("ledger %s %s %" PRIu64 "\n", kInfo[kGain].name, kGainClasses[c], counts[c]);
    return 0;
  }

  auto t0 = std::chrono::steady_clock::now();
  const std::vector<std::vector<uint64_t>> hostFp = hostFingerprints(hostD, threads, probes);
  const double hostSeconds = seconds(t0);

  if (mode == "host-only") {
    for (auto [p, inputs] : probes) {
      uint64_t h = 0;
      for (uint64_t f : hostFp[p]) h = mix64(h ^ f);
      std::printf("fingerprint %s %" PRIu64 " %016" PRIx64 "\n", kInfo[p].name, inputs, h);
    }
    std::printf("host %.1f s on %d threads\n", hostSeconds, threads);
    return 0;
  }

  uint64_t totalInputs = 0, mismatches = 0;
  if (mode == "self-test") {
    // the other half: the host half with bit 3 of word 5 (a gain) of one lensPhotoSample<plain> element flipped
    const int fp = kSamplePlain, fword = 5, fbit = 3;
    const uint64_t fi = kBlock / 2 + 4321;
    Half flipped;
    flipped.words = [&](int p, uint64_t begin, uint64_t count, std::vector<uint32_t>& words) {
      hostWords(hostD, p, begin, count, words);
      if (p == fp && fi >= begin && fi < begin + count) words[kOut * (fi - begin) + fword] ^= 1u << fbit;
    };
    flipped.fingerprints = [&](int p, uint64_t inputs, std::vector<uint64_t>& out) {
      if (p != fp) {
        out = hostFp[p];
        return;
      }
      out.assign(blocksOf(inputs), 0);
      for (uint64_t b = 0; b < out.size(); ++b) {
        const uint64_t begin = b * kBlock, count = std::min(inputs, begin + kBlock) - begin;
        std::vector<uint32_t> words;
        flipped.words(p, begin, count, words);
        for (uint64_t k = 0; k < count; ++k) out[b] += elementMix(p, begin + k, &words[kOut * k]);
      }
    };
    mismatches = compare(hostD, probes, hostFp, flipped, &totalInputs);
    std::printf("self-test: flipped %s %" PRIu64 " word %d bit %d\n", kInfo[fp].name, fi, fword, fbit);
  } else {
    GateData devD = hostD;
    LensRigModel* dRig = upload(H.rig);
    LensPhotoPlane* dPhoto = upload(H.photo);
    ChainGeo* dGeo = upload(H.geo);
    float* dTables = upload(H.tables);
    devD.rig = dRig; devD.photo = dPhoto; devD.geo = dGeo; devD.tables = dTables;
    constexpr auto launchFps = fpTable(std::make_integer_sequence<int, kProbes>());
    constexpr auto launchW = wordsTable(std::make_integer_sequence<int, kProbes>());
    unsigned long long* dFp = nullptr;
    uint32_t* dWords = nullptr;
    uint64_t maxBlocks = 0;
    for (auto [p, inputs] : probes) maxBlocks = std::max(maxBlocks, blocksOf(inputs));
    CUDA_OK(cudaMalloc(&dFp, maxBlocks * sizeof(unsigned long long)));
    CUDA_OK(cudaMalloc(&dWords, kOut * kBlock * sizeof(uint32_t)));
    cudaEvent_t e0, e1;
    CUDA_OK(cudaEventCreate(&e0));
    CUDA_OK(cudaEventCreate(&e1));
    float deviceMs = 0.0f;
    Half device;
    device.fingerprints = [&](int p, uint64_t inputs, std::vector<uint64_t>& out) {
      const uint64_t blocks = blocksOf(inputs);
      CUDA_OK(cudaEventRecord(e0));
      for (uint64_t b = 0; b < blocks; b += 65535) launchFps[p](devD, inputs, b, std::min<uint64_t>(65535, blocks - b), dFp);
      CUDA_OK(cudaEventRecord(e1));
      CUDA_OK(cudaEventSynchronize(e1));
      float ms;
      CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
      deviceMs += ms;
      out.resize(blocks);
      CUDA_OK(cudaMemcpy(out.data(), dFp, blocks * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    };
    device.words = [&](int p, uint64_t begin, uint64_t count, std::vector<uint32_t>& words) {
      launchW[p](devD, begin, count, dWords);
      words.resize(kOut * count);
      CUDA_OK(cudaMemcpy(words.data(), dWords, kOut * count * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    };
    mismatches = compare(hostD, probes, hostFp, device, &totalInputs);
    std::printf("device %.1f s, host %.1f s on %d threads\n", deviceMs / 1000.0, hostSeconds, threads);
    cudaFree(dFp); cudaFree(dWords); cudaFree(dRig); cudaFree(dPhoto); cudaFree(dGeo); cudaFree(dTables);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
  }
  std::printf("%zu probes, %" PRIu64 " inputs, %" PRIu64 " mismatches\n", probes.size(), totalInputs, mismatches);
  return mismatches ? 1 : 0;
}
