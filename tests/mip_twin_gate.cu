// Host / device twin gate of the anti-aliased camera views: the device build of every float function the footprint adds
// (oriented_view.h: cameraXY, modelRay, rayDifferential, equirectJacobian, cubeInputFace, cubeJacobian, lensJacobian,
// mipLevelOf, mipScale, mipCameraPoint, mipCameraSample) against its host build, the one T360B200_cameraMipMaps runs.
// tests/test_mip_twins.py builds it with the library's own nvcc flags (transform360_b200/build.py: ARCH, -O3, HOST_FLAGS)
// and runs it.  Its design is tests/twin_gate.cu's:
//   - a probe is a T360_HD function of an index i: it draws its inputs from a splitmix64 stream seeded with a hash of
//     (seed, probe, i), calls one twin function or chain, and packs the result into at most six 32-bit words.  The same
//     probe code runs in a kernel on the device and in a thread pool on the host;
//   - each half sums a 64-bit mix of (probe, i, words) over each block of 2^20 inputs, an order-independent fingerprint.
//     The host compares them; for up to 16 mismatching blocks per probe both halves re-evaluate the block element by
//     element, and at most 20 lines `probe i input-bits host-bits device-bits` are printed.  The last line is
//     `<P> probes, <N> inputs, <M> mismatches`; the exit status is 1 on any mismatch;
//   - float words compare bit for bit (-0 against +0 included); every NaN is written as 0x7fc00000 (no record depends on a
//     payload), and nothing else is excused.
// Probes:
//   mipLevelOf         every 32-bit pattern of rho^2 (as a.a; b.b, the top level and the bias drawn): level and weight;
//   rayDifferential    each model's differential at drawn (X, Y) and half steps, cameras from cameraConstants;
//   equirectJacobian   drawn rays (near-pole, axis and arbitrary) and differentials, every input re-pack;
//   cubeJacobian       cubeInputFace of the normalised ray and the quotient rule on that face;
//   lensJacobian       drawn rig directions, rays on a lens axis (rho = 0, both signs of Z) included;
//   mipScale           drawn positions and level ratios;
//   mipCameraPoint / mipCameraSample, LENS = false and true: 2^24 (geometry, pixel) samples each over seeded contexts,
//   cameras of every model, rigs, maxLevel and lodBias.
//
//   mip_twin_gate [--threads T] [--shift S]     the full gate (2^S times fewer inputs per probe)
//   mip_twin_gate --host-only [--threads T]     the host half at 2^20 inputs per probe, fingerprints printed; no CUDA call
//   mip_twin_gate --self-test [--threads T]     the host half against a copy of itself with one bit of one word flipped
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
constexpr uint64_t kSeed = 20261018ull;
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
};

// ---- data the probes share (host-built, copied to the device) --------------------------------------------------------
struct ChainGeo {
  SphereGeometry g;  // a camera view's geometry (rig: mono, equirect-like input fields)
  MipGeometry m;
  int bias;
};
struct GateData {
  const RectilinearCamera* cam;
  int nCam;
  const LensRigModel* rig;
  int nRig, nRigAxis;  // [0, nRigAxis): lenses along +-z (rho = 0 reachable)
  const ChainGeo* ctxGeo;
  int nCtxGeo;
  const ChainGeo* lensGeo;
  int nLensGeo;
};

T360_HD SphereVec drawVec(Draw& d, float scale) { return SphereVec{d.component(scale), d.component(scale), d.component(scale)}; }

enum Probe { kLod, kRayDiff, kEquirect, kCube, kLens, kScale, kPointCtx, kPointLens, kSampleCtx, kSampleLens, kProbes };
struct ProbeInfo {
  const char* name;
  uint64_t inputs;
};
const ProbeInfo kInfo[kProbes] = {
    {"mipLevelOf", 1ull << 32},       {"rayDifferential", 1ull << 26}, {"equirectJacobian", 1ull << 26}, {"cubeJacobian", 1ull << 26},
    {"lensJacobian", 1ull << 26},     {"mipScale", 1ull << 26},        {"mipCameraPoint<ctx>", 1ull << 24},
    {"mipCameraPoint<lens>", 1ull << 24}, {"mipCameraSample<ctx>", 1ull << 24}, {"mipCameraSample<lens>", 1ull << 24},
};

template <int P>
T360_HD void probe(const GateData& D, uint64_t i, Words& w) {
  Draw d(P, i);
  for (uint32_t& o : w.out) o = 0;
  for (uint32_t& o : w.in) o = 0;
  if constexpr (P == kLod) {
    const float aa = bitsFloat(static_cast<uint32_t>(i));
    const float bb = d.below(4) == 0 ? d.special() : (d.coin() ? 0.0f : bitsFloat(d.u32() & 0x7fffffffu));
    const int top = d.below(kMipMaxLevels + 1), bias = d.below(2049) - 1024;
    int wt;
    const int level = mipLevelOf(aa, bb, top, bias, &wt);
    w.in[0] = floatBits(aa); w.in[1] = floatBits(bb); w.in[2] = iw(top); w.in[3] = iw(bias);
    w.out[0] = iw(level); w.out[1] = iw(wt);
  } else if constexpr (P == kRayDiff) {
    const RectilinearCamera& c = D.cam[d.below(D.nCam)];
    const float X = d.below(8) == 0 ? d.sign(d.coin() ? 1.0f : 0.0f) : d.range(-1.0f, 1.0f);
    const float Y = d.below(8) == 0 ? d.sign(d.coin() ? 1.0f : 0.0f) : d.range(-1.0f, 1.0f);
    const float h = d.coin() ? fDiv(1.0f, static_cast<float>(1 + d.below(8192))) : d.range(0.0f, 0.01f);
    const SphereVec r = d.coin() ? rayDifferential(c, fSub(X, h), Y, fAdd(X, h), Y) : rayDifferential(c, X, fSub(Y, h), X, fAdd(Y, h));
    w.in[0] = floatBits(X); w.in[1] = floatBits(Y); w.in[2] = floatBits(h); w.in[3] = iw(c.model);
    w.out[0] = fw(r.x); w.out[1] = fw(r.y); w.out[2] = fw(r.z);
  } else if constexpr (P == kEquirect) {
    SphereGeometry g{};
    g.inW = 16 + d.below(16000); g.inH = 8 + d.below(8000);
    g.packLR = d.below(3) == 0; g.packTB = !g.packLR && d.coin();
    SphereVec t = drawVec(d, 1.0f);
    if (d.below(8) == 0) { t.x = fMul(t.x, 1e-4f); t.z = fMul(t.z, 1e-4f); }  // near a pole
    const SphereVec r = drawVec(d, 0.01f);
    float du, dv;
    equirectJacobian(g, t, r, &du, &dv);
    w.in[0] = floatBits(t.x); w.in[1] = floatBits(t.y); w.in[2] = floatBits(t.z); w.in[3] = iw(g.inW);
    w.out[0] = fw(du); w.out[1] = fw(dv);
  } else if constexpr (P == kCube) {
    SphereGeometry g{};
    g.inW = 16 + d.below(16000); g.inH = 8 + d.below(8000);
    g.packLR = d.below(3) == 0; g.packTB = !g.packLR && d.coin();
    g.inputExpand = d.coin() ? 1.0f : d.range(1.0f, 1.1f);
    SphereVec t = drawVec(d, 1.0f);
    if (d.below(8) == 0) t.x = t.z;  // on a face edge
    const SphereVec r = drawVec(d, 0.01f);
    const float n = fSqrt(fAdd(fAdd(fMul(t.x, t.x), fMul(t.y, t.y)), fMul(t.z, t.z)));
    const int f = cubeInputFace(fDiv(t.x, n), fDiv(t.y, n), fDiv(t.z, n));
    float du = 0.0f, dv = 0.0f;
    if (f >= 0) cubeJacobian(g, f, t, r, &du, &dv);
    w.in[0] = floatBits(t.x); w.in[1] = floatBits(t.y); w.in[2] = floatBits(t.z); w.in[3] = floatBits(r.x);
    w.out[0] = iw(f); w.out[1] = fw(du); w.out[2] = fw(dv);
  } else if constexpr (P == kLens) {
    const bool axis = d.below(4) == 0;
    const LensRigModel& rig = D.rig[axis ? d.below(D.nRigAxis) : d.below(D.nRig)];
    SphereVec t = drawVec(d, 1.0f);
    if (axis) t = SphereVec{d.sign(0.0f), d.sign(0.0f), d.sign(d.range(0.1f, 2.0f))};  // rho = 0 on either lens's axis
    const SphereVec rx = drawVec(d, 0.01f), ry = drawVec(d, 0.01f);
    const int inW = 16 + d.below(8000), inH = 16 + d.below(8000);
    float a[2], b[2];
    lensJacobian(rig, t, rx, ry, inW, inH, a, b);
    w.in[0] = floatBits(t.x); w.in[1] = floatBits(t.y); w.in[2] = floatBits(t.z); w.in[3] = iw(inW);
    w.out[0] = fw(a[0]); w.out[1] = fw(a[1]); w.out[2] = fw(b[0]); w.out[3] = fw(b[1]);
  } else if constexpr (P == kScale) {
    const float p = d.below(8) == 0 ? d.special() : d.range(-10.0f, 20000.0f);
    const int l = 1 + d.below(kMipMaxLevels), n = 16 + d.below(16000);
    int m = n;
    for (int k = 0; k < l; ++k) m = (m + 1) / 2;
    const float s = d.coin() ? fDiv(static_cast<float>(m), static_cast<float>(n)) : d.range(0.001f, 1.0f);
    w.in[0] = floatBits(p); w.in[1] = floatBits(s);
    w.out[0] = fw(mipScale(p, s));
  } else {
    constexpr bool LENS = P == kPointLens || P == kSampleLens;
    const ChainGeo& e = LENS ? D.lensGeo[d.below(D.nLensGeo)] : D.ctxGeo[d.below(D.nCtxGeo)];
    const RectilinearCamera& c = D.cam[d.below(D.nCam)];
    const LensRigModel& rig = D.rig[d.below(D.nRig)];
    const int row = d.below(e.g.mapH), col = d.below(e.g.mapW);
    w.in[0] = iw(row); w.in[1] = iw(col); w.in[2] = iw(c.model); w.in[3] = iw(e.m.top);
    int wt;
    if constexpr (P == kPointCtx || P == kPointLens) {
      float p0[2], p1[2];
      const int level = mipCameraPoint<LENS>(e.g, c, rig, e.m, e.bias, row, col, p0, p1, &wt);
      w.out[0] = fw(p0[0]); w.out[1] = fw(p0[1]); w.out[2] = fw(p1[0]); w.out[3] = fw(p1[1]); w.out[4] = iw(level); w.out[5] = iw(wt);
    } else {
      int32_t r0[2], r1[2] = {0, 0};
      const int level = mipCameraSample<LENS>(e.g, c, rig, e.m, e.bias, row, col, r0, r1, &wt);
      w.out[0] = iw(r0[0]); w.out[1] = iw(r0[1]); w.out[2] = iw(r1[0]); w.out[3] = iw(r1[1]); w.out[4] = iw(level); w.out[5] = iw(wt);
    }
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
  std::vector<RectilinearCamera> cam;
  std::vector<LensRigModel> rig;
  std::vector<ChainGeo> ctxGeo, lensGeo;
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
  // cameras of every model over its range, with the library's constants
  auto pose = [&](int model, double hfov, double vfov, double d) {
    H.cam.push_back(cameraConstants(model, static_cast<float>(d), angle(), angle(), angle(), static_cast<float>(hfov), static_cast<float>(vfov)));
  };
  for (int k = 0; k < 128; ++k) {
    pose(kCameraPinhole, g.uniform(1, 179), g.uniform(1, 179), 0);
    pose(kCameraEquidistant, g.uniform(1, 360), g.uniform(1, 360), 0);
    pose(kCameraStereographic, g.uniform(1, 359), g.uniform(1, 359), 0);
    const double d = g.uniform(0, 1), top = d < 1 ? 2.0 * std::acos(-d) * 180.0 / M_PI : 359.0;
    pose(kCameraPannini, g.uniform(1, std::min(359.0, top - 0.01)), g.uniform(1, 179), d);
  }
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
  // geometries: context inputs (equirect and cube map, every stereo format and output split, odd and even sizes, K = 1,
  // 2, 4, 8) and rigs (mono), each with a maxLevel in 1..8 and a bias
  const StereoFormat stereo[] = {STEREO_FORMAT_MONO, STEREO_FORMAT_LR, STEREO_FORMAT_TB};
  for (int k = 0; k < 384; ++k) {
    const bool rigInput = k % 4 == 3;
    FrameTransformContext c{};
    c.output_layout = LAYOUT_CUBEMAP_32;
    c.input_layout = !rigInput && g.below(3) == 0 ? LAYOUT_CUBEMAP_32 : LAYOUT_EQUIRECT;
    c.input_stereo_format = rigInput ? STEREO_FORMAT_MONO : stereo[(k / 4) % 3];
    c.output_stereo_format = rigInput ? STEREO_FORMAT_MONO : stereo[(k / 12) % 3];
    c.vflip = (k / 36) % 2;
    c.expand_coef = 1.0f;
    c.input_expand_coef = rigInput || g.below(2) == 0 ? 1.0f : static_cast<float>(g.uniform(1.0, 1.1));
    const int K = 1 << (k / 2) % 4;
    ChainGeo e{};
    e.g = sphereGeometry(c, 8 + g.below(2000), 8 + g.below(2000), 8 + g.below(16000), 8 + g.below(8000), K);
    e.m = mipGeometry(e.g, 1 + g.below(kMipMaxLevels));
    e.bias = g.below(2049) - 1024;
    (rigInput ? H.lensGeo : H.ctxGeo).push_back(e);
  }
  return H;
}

GateData view(const HostData& H) {
  return GateData{H.cam.data(), static_cast<int>(H.cam.size()), H.rig.data(), static_cast<int>(H.rig.size()), H.nRigAxis,
                  H.ctxGeo.data(), static_cast<int>(H.ctxGeo.size()), H.lensGeo.data(), static_cast<int>(H.lensGeo.size())};
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
    else if (s == "--host-only" || s == "--self-test") mode = s.substr(2);
    else {
      std::fprintf(stderr, "usage: mip_twin_gate [--threads T] [--shift S] [--host-only | --self-test]\n");
      return 2;
    }
  }
  threads = std::max(1, threads);
  const HostData H = makeData();
  const GateData hostD = view(H);

  std::vector<std::pair<int, uint64_t>> probes;
  for (int p = 0; p < kProbes; ++p) probes.push_back({p, mode == "full" ? std::max<uint64_t>(kInfo[p].inputs >> shift, 1) : kBlock});

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
    // the other half: the host half with bit 5 of word 4 (the level) of one mipCameraSample<lens> element flipped
    const int fp = kSampleLens, fword = 4, fbit = 5;
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
    RectilinearCamera* dCam = upload(H.cam);
    LensRigModel* dRig = upload(H.rig);
    ChainGeo* dCtx = upload(H.ctxGeo);
    ChainGeo* dLens = upload(H.lensGeo);
    devD.cam = dCam; devD.rig = dRig; devD.ctxGeo = dCtx; devD.lensGeo = dLens;
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
    cudaFree(dFp); cudaFree(dWords); cudaFree(dCam); cudaFree(dRig); cudaFree(dCtx); cudaFree(dLens);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
  }
  std::printf("%zu probes, %" PRIu64 " inputs, %" PRIu64 " mismatches\n", probes.size(), totalInputs, mismatches);
  return mismatches ? 1 : 0;
}
