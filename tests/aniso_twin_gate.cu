// Twin gate of the anisotropic camera views: the device build of every float function the probes add (oriented_view.h:
// anisoLevelOf, anisoFootprint, anisoCameraPoint, anisoCameraSample) against its host build, the one
// T360B200_cameraAnisoMaps runs.  The harness, its comparison rule and its modes are tests/twin_gate.cuh's.  Probes:
//   anisoLevelOf       drawn a.a and b.b (every bit pattern of a.a, b.b from equal, exact multiples of 256 levels apart,
//                      0, denormal, inf / NaN or arbitrary), top level, bias and log2 maxProbes: level, weight and e; the
//                      ledger's classes: aa == bb, lambda_maj - lambda_min an exact non-zero multiple of 256, a zero and
//                      a denormal axis, an infinite or NaN axis (a pole), and e clamped by maxProbes;
//   anisoFootprint<ctx> / <lens>: 2^24 (geometry, pixel) samples each over seeded contexts, cameras of every model, rigs,
//                      maxLevel 0..8, lodBias and maxProbes; the ledger's classes: probes on the column and on the row axis;
//   anisoCameraPoint / anisoCameraSample, LENS = false and true: a drawn probe k < N of the same samples; the ledger's
//                      classes: the first and last probes on different cube faces (ctx) or closer lenses (lens).
#include "twin_gate.cuh"

using namespace t360;
using namespace t360gate;

namespace {

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
  int nRig;
  const ChainGeo* ctxGeo;
  int nCtxGeo;
  const ChainGeo* lensGeo;
  int nLensGeo;
};

// lambda256 of x as anisoLevelOf takes it (for the ledger)
T360_HD int lambdaOf(float x) { return (static_cast<int32_t>(floatBits(x)) - 0x3f800000) >> 16; }

#ifndef __CUDA_ARCH__
// The rotated ray of probe k of footprint f, as anisoCameraPoint takes it (for the ledger: host only)
SphereVec probeRay(const RectilinearCamera& c, const MipGeometry& m, const AnisoFootprint& f, int k) {
  if (f.e == 0) return f.t;
  const int n = 1 << f.e;
  const float o = fDiv(static_cast<float>(2 * k + 1 - n), static_cast<float>(n));
  return f.rows ? rotateHD(c.r, modelRay(c, f.X, fAdd(f.Y, fMul(o, m.halfY)))) : rotateHD(c.r, modelRay(c, fAdd(f.X, fMul(o, m.halfX)), f.Y));
}
int faceOf(const SphereVec& t) {
  const float n = fSqrt(fAdd(fAdd(fMul(t.x, t.x), fMul(t.y, t.y)), fMul(t.z, t.z)));
  return cubeInputFace(fDiv(t.x, n), fDiv(t.y, n), fDiv(t.z, n));
}
int closerLens(const LensRigModel& rig, const SphereVec& t) {
  const float z0 = lensRow(rig.lens[0].m + 6, t);
  return rig.numLenses > 1 && lensRow(rig.lens[1].m + 6, t) > z0 ? 1 : 0;
}
#endif

struct AnisoGate {
  static constexpr uint64_t kSeed = 20261022ull;
  static constexpr int kOut = 9;
  enum Probe { kLod, kFootCtx, kFootLens, kPointCtx, kPointLens, kSampleCtx, kSampleLens, kProbes };
  static constexpr ProbeInfo kInfo[kProbes] = {
      {"anisoLevelOf", "equal multipleOf256 zero denormal infNaN clamped", 1ull << 28},
      {"anisoFootprint<ctx>", "columnAxis rowAxis", 1ull << 24},
      {"anisoFootprint<lens>", "columnAxis rowAxis", 1ull << 24},
      {"anisoCameraPoint<ctx>", "faceChange", 1ull << 24},
      {"anisoCameraPoint<lens>", "lensChange", 1ull << 24},
      {"anisoCameraSample<ctx>", "faceChange", 1ull << 24},
      {"anisoCameraSample<lens>", "lensChange", 1ull << 24},
  };
  // bit 3 of word 6 (the level, weight and probe count) of an anisoCameraSample<lens> element
  static constexpr Flip kFlip = {kSampleLens, kBlock / 2 + 2718, 6, 3};

  using Data = GateData;
  struct HostData {
    std::vector<RectilinearCamera> cam;
    std::vector<LensRigModel> rig;
    std::vector<ChainGeo> ctxGeo, lensGeo;
  };
  template <int P>
  static T360_HD void probe(const Data& D, uint64_t i, Words<kOut>& w);
  static HostData makeData();
  static Data view(const HostData& H, int) {
    return GateData{H.cam.data(), static_cast<int>(H.cam.size()), H.rig.data(), static_cast<int>(H.rig.size()), H.ctxGeo.data(),
                    static_cast<int>(H.ctxGeo.size()), H.lensGeo.data(), static_cast<int>(H.lensGeo.size())};
  }
  static Data deviceData(const HostData& H, Data D, Uploads& up) {
    D.cam = up(H.cam); D.rig = up(H.rig); D.ctxGeo = up(H.ctxGeo); D.lensGeo = up(H.lensGeo);
    return D;
  }
};

template <int P>
T360_HD void AnisoGate::probe(const GateData& D, uint64_t i, Words<kOut>& w) {
  Draw d(kSeed, P, i);
  if constexpr (P == kLod) {
    const float aa = bitsFloat(d.u32() & 0x7fffffffu);
    float bb;
    switch (d.below(8)) {
      case 0: bb = aa; break;
      case 1: bb = bitsFloat(floatBits(aa) + (static_cast<uint32_t>(d.below(8)) << 24)); break;  // 4^k aa: 256 k apart
      case 2: bb = 0.0f; break;
      case 3: bb = bitsFloat(1u + d.u32() % 0x7fffffu); break;  // denormal
      case 4: bb = d.special(); break;
      default: bb = bitsFloat(d.u32() & 0x7fffffffu);
    }
    float x = aa, y = bb;
    if (d.coin()) { x = bb; y = aa; }
    const int top = d.below(kMipMaxLevels + 1), bias = d.below(2049) - 1024, maxLog2 = d.below(5);
    int wt, e;
    const int level = anisoLevelOf(x, y, top, bias, maxLog2, &wt, &e);
    w.in[0] = floatBits(x); w.in[1] = floatBits(y); w.in[2] = iw(top | maxLog2 << 8); w.in[3] = iw(bias);
    w.out[0] = iw(level); w.out[1] = iw(wt); w.out[2] = iw(e);
    const float inf = bitsFloat(0x7f800000u);
    const bool finite = x < inf && y < inf;
    const int diff = finite ? lambdaOf(x > y ? x : y) - lambdaOf(x > y ? y : x) : 0;
    CLASS(0, x == y);
    CLASS(1, finite && diff > 0 && diff % 256 == 0);
    CLASS(2, x == 0.0f || y == 0.0f);
    CLASS(3, (x > 0.0f && floatBits(x) < 0x800000u) || (y > 0.0f && floatBits(y) < 0x800000u));
    CLASS(4, !finite);
    CLASS(5, finite && ((diff + 255) >> 8) > maxLog2);
  } else {
    constexpr bool LENS = P == kFootLens || P == kPointLens || P == kSampleLens;
    const ChainGeo& e = LENS ? D.lensGeo[d.below(D.nLensGeo)] : D.ctxGeo[d.below(D.nCtxGeo)];
    const RectilinearCamera& c = D.cam[d.below(D.nCam)];
    const LensRigModel& rig = D.rig[d.below(D.nRig)];
    const int row = d.below(e.g.mapH), col = d.below(e.g.mapW), maxLog2 = d.below(5);
    w.in[0] = iw(row); w.in[1] = iw(col); w.in[2] = iw(c.model | maxLog2 << 8); w.in[3] = iw(e.m.top);
    const AnisoFootprint f = anisoFootprint<LENS>(e.g, c, rig, e.m, e.bias, maxLog2, row, col);
    const uint32_t shared = iw(f.level) | iw(f.w) << 8 | iw(f.e) << 16 | iw(f.rows) << 20 | iw(f.eye) << 21;
    if constexpr (P == kFootCtx || P == kFootLens) {
      w.out[0] = fw(f.X); w.out[1] = fw(f.Y); w.out[2] = fw(f.t.x); w.out[3] = fw(f.t.y); w.out[4] = fw(f.t.z); w.out[5] = shared;
      CLASS(0, f.e > 0 && !f.rows);
      CLASS(1, f.e > 0 && f.rows);
    } else {
      const int k = d.below(1 << f.e);
      w.in[3] = iw(e.m.top | k << 8);
      if constexpr (P == kPointCtx || P == kPointLens) {
        float p0[2], p1[2];
        anisoCameraPoint<LENS>(e.g, c, rig, e.m, f, k, p0, p1);
        w.out[0] = fw(p0[0]); w.out[1] = fw(p0[1]); w.out[2] = fw(p1[0]); w.out[3] = fw(p1[1]);
      } else {
        int32_t r0[2], r1[2] = {0, 0};
        anisoCameraSample<LENS>(e.g, c, rig, e.m, f, k, r0, r1);
        w.out[0] = iw(r0[0]); w.out[1] = iw(r0[1]); w.out[2] = iw(r1[0]); w.out[3] = iw(r1[1]);
      }
      w.out[6] = shared;
#ifndef __CUDA_ARCH__
      if (f.e > 0) {
        const SphereVec first = probeRay(c, e.m, f, 0), last = probeRay(c, e.m, f, (1 << f.e) - 1);
        if constexpr (LENS) CLASS(0, closerLens(rig, first) != closerLens(rig, last));
        else CLASS(0, e.g.cubeInput && faceOf(first) != faceOf(last));
      }
#endif
    }
  }
}

AnisoGate::HostData AnisoGate::makeData() {
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
    pose(kCameraEquirect, g.uniform(1, 360), g.uniform(1, 180), 0);
  }
  // rigs of one and two lenses (a back-to-back pair and arbitrary rotations)
  auto lens = [&](bool back, bool rotated) {
    LensModel L{};
    const Rotation r = rotated ? rotationFromAngles(angle(), angle(), angle()) : rotationFromAngles(back ? 180.0f : 0.0f, 0.0f, 0.0f);
    const float m[9] = {r.xx, r.xy, r.xz, -r.yx, -r.yy, -r.yz, r.zx, r.zy, r.zz};
    std::memcpy(L.m, m, sizeof(m));
    L.ax = static_cast<float>(g.uniform(0.1, 0.5));
    L.bx = static_cast<float>(g.uniform(0.3, 0.7));
    L.ay = static_cast<float>(g.uniform(0.1, 0.5));
    L.by = static_cast<float>(g.uniform(0.3, 0.7));
    for (float& k : L.k) k = static_cast<float>(g.uniform(-0.05, 0.05));
    L.thetaMax = g.below(3) == 0 ? static_cast<float>(M_PI) : static_cast<float>(g.uniform(1.2, M_PI));
    return L;
  };
  for (int k = 0; k < 128; ++k) {
    LensRigModel rig{};
    rig.numLenses = 1 + k % 2;
    const bool rotated = k % 4 >= 2;
    rig.lens[0] = lens(false, rotated);
    if (rig.numLenses == 2) rig.lens[1] = lens(true, rotated);
    H.rig.push_back(rig);
  }
  // geometries: context inputs (equirect and cube map, every stereo format and output split, odd and even sizes, K = 1,
  // 2, 4, 8) and rigs (mono), each with a maxLevel in 0..8 (0: the probes supersample level 0) and a bias
  const StereoFormat stereo[] = {STEREO_FORMAT_MONO, STEREO_FORMAT_LR, STEREO_FORMAT_TB};
  for (int k = 0; k < 384; ++k) {
    const bool rigInput = k % 4 == 3;
    FrameTransformContext c{};
    c.output_layout = LAYOUT_CUBEMAP_32;
    c.input_layout = !rigInput && g.below(2) == 0 ? LAYOUT_CUBEMAP_32 : LAYOUT_EQUIRECT;
    c.input_stereo_format = rigInput ? STEREO_FORMAT_MONO : stereo[(k / 4) % 3];
    c.output_stereo_format = rigInput ? STEREO_FORMAT_MONO : stereo[(k / 12) % 3];
    c.vflip = (k / 36) % 2;
    c.expand_coef = 1.0f;
    c.input_expand_coef = rigInput || g.below(2) == 0 ? 1.0f : static_cast<float>(g.uniform(1.0, 1.1));
    const int K = 1 << (k / 2) % 4;
    ChainGeo e{};
    e.g = sphereGeometry(c, 8 + g.below(1000), 8 + g.below(1000), 8 + g.below(16000), 8 + g.below(8000), K);
    e.m = mipGeometry(e.g, g.below(kMipMaxLevels + 1));
    e.bias = g.below(2049) - 1024;
    (rigInput ? H.lensGeo : H.ctxGeo).push_back(e);
  }
  return H;
}

}  // namespace

int main(int argc, char** argv) { return runGate<AnisoGate>(argc, argv); }
