// Twin gate of the per-frame position chains: the device build of every float function of csrc/flat_view.h, libm_ports.h
// and oriented_view.h that the per-frame kernels call, against its host build, the one the planner runs.  The harness,
// its comparison rule and its modes are tests/twin_gate.cuh's.  Three tiers:
//   A. every 32-bit pattern (fullOnly; under --shift, patternA samples one in 2^S): libmAtanf, libmAsinf, fSqrt, sincCos,
//      truncToInt, roundHalfEven, quantizeAxis (K = 1, 2, 4, 8);
//   B. structured families (arbitrary bit patterns, special values, values a few ulps either side of each branch threshold
//      and realistic values): libmAtan2f, pixelCentre, toPixel, rotateHD, rayToSphereHD, warpOffCentreHD, sphereInputHD,
//      lensPosition, lensBlendPosition, cameraRay (equidistant, stereographic, Pannini: the pinhole ray is not part of
//      cameraRay, rectilinearPoint builds it, and tier C covers it);
//   C. whole chains over geometries from sphereGeometry() of seeded contexts with their buildSphereTables tables:
//      flatSample, sphereSample, lensSample, lensBlendSample and rectilinearSample in every instantiation the kernels use.
#include "twin_gate.cuh"

using namespace t360;
using namespace t360gate;

namespace {

// ---- data the structured probes and the chains share (host-built, copied to the device) ------------------------------
struct GeoEntry {
  SphereGeometry g;
  uint32_t colTab, rowTab;  // offsets into GateData::tab
};
struct GateData {
  const Rotation* rot;
  int nRot, nRotReal;  // [0, nRotReal): rotationFromAngles; the rest raw matrices with +-0 and +-1 entries
  const LensRigModel* rig;
  int nRig, nRig2;  // [0, nRig2): two-lens rigs
  const RectilinearCamera* cam;
  int nCam, nCamPinhole;  // [0, nCamPinhole): pinhole cameras, then the other models
  const GeoEntry* geo;
  int nGeo, nGeoPlain;  // [0, nGeoPlain): layouts other than the barrels
  const float* tab;
  int shift;
};

// ---- tier A: every bit pattern ----------------------------------------------------------------------------------------
T360_HD uint32_t patternA(const GateData& D, uint64_t i) {
  if (D.shift == 0) return static_cast<uint32_t>(i);
  return static_cast<uint32_t>((i << D.shift) | (mix64(i) & ((1ull << D.shift) - 1)));
}

constexpr int kToPixelPlanes = 4;
T360_HD int toPixelWidth(int k) { return k == 0 ? 1 : k == 1 ? 3 : k == 2 ? 1920 : 7679; }  // odd and even plane widths
constexpr uint64_t kToPixelFloats = 0x7f800002ull;  // the floats in [-1, 2]: +0 .. 2 and -0 .. -1

// ---- tier B -----------------------------------------------------------------------------------------------------------
T360_HD SphereVec drawVec(Draw& r, float lo, float hi) { return SphereVec{r.range(lo, hi), r.range(lo, hi), r.range(lo, hi)}; }

// q for rotateHD and the off-centre warp: random, axis-aligned with signed zeros, random with signed-zero components, or
// arbitrary bit patterns
T360_HD SphereVec drawQ(Draw& r) {
  switch (r.below(4)) {
    case 0: return drawVec(r, -2.0f, 2.0f);
    case 1: {
      float c[3] = {r.sign(0.0f), r.sign(0.0f), r.sign(0.0f)};
      c[r.below(3)] = r.sign(r.coin() ? 1.0f : 0.5f);
      return SphereVec{c[0], c[1], c[2]};
    }
    case 2: {
      SphereVec q = drawVec(r, -1.0f, 1.0f);
      if (r.coin()) q.x = r.sign(0.0f);
      if (r.coin()) q.y = r.sign(0.0f);
      if (r.coin()) q.z = r.sign(0.0f);
      return q;
    }
    default: return SphereVec{r.coin() ? r.bits() : r.special(), r.coin() ? r.bits() : r.special(), r.coin() ? r.bits() : r.special()};
  }
}

// an offset of the off-centre eye: inside the sphere, outside it, or with zero components
T360_HD SphereVec drawOffset(Draw& r) {
  const float m = r.coin() ? 0.9f : 2.0f;
  SphereVec o = drawVec(r, -m, m);
  if (r.below(4) == 0) o.y = 0.0f;
  if (r.below(8) == 0) o.x = r.sign(0.0f);
  return o;
}

// the direction t the input lookup maps: random, the branch cut (t.x = +-0, t.z < 0), exact poles, close to the seam (the
// barrel clamp), NaN components, subnormal and non-unit vectors, a component exactly +-0.5 after normalisation with
// another equal to it (|gx| or |gy| exactly 1 on a cube input; with subnormal squares, also on the face picked),
// axis-aligned with signed zeros
T360_HD SphereVec drawDirection(Draw& r, int kind) {
  switch (kind) {
    case 0: return drawVec(r, -1.0f, 1.0f);
    case 1: return SphereVec{r.sign(0.0f), r.range(-1.0f, 1.0f), -r.range(0.0f, 1.0f)};
    case 2: return SphereVec{r.sign(0.0f), r.sign(r.range(0.001f, 4.0f)), r.sign(0.0f)};
    case 3: return SphereVec{r.sign(bitsFloat(0x2f800000u + (r.u32() >> 6))), r.range(-0.5f, 0.5f), -r.range(0.5f, 1.0f)};
    case 4: {
      SphereVec t = drawVec(r, -1.0f, 1.0f);
      (r.coin() ? t.x : (r.coin() ? t.y : t.z)) = bitsFloat(0x7fc00000u | r.u32());
      return t;
    }
    case 5: {
      const float s = bitsFloat((r.u32() & 0x807fffffu) | (static_cast<uint32_t>(r.below(60)) << 23));  // subnormal .. 2^-68
      return SphereVec{r.coin() ? s : fMul(s, r.range(-1.0f, 1.0f)), fMul(s, r.range(-1.0f, 1.0f)), r.coin() ? s : r.sign(0.0f)};
    }
    case 6: {
      if (r.coin()) {  // squares that round to one subnormal unit each: n = 2a exactly, so t / n has components exactly +-0.5
        const float a = bitsFloat(0x1a1cc471u), c = r.coin() ? a : 3e-23f;  // (c: +-0.46 after normalisation, another face)
        const float v[3] = {r.sign(a), r.sign(a), r.sign(c)};
        const int rot = r.below(3);
        return SphereVec{v[rot], v[(rot + 1) % 3], v[(rot + 2) % 3]};
      }
      const float v[3] = {r.sign(0.5f), r.sign(0.5f), r.sign(r.coin() ? 0.70710677f : 0.70710683f)};
      const int rot = r.below(3);
      const float scale = bitsFloat(static_cast<uint32_t>(100 + r.below(56)) << 23);
      return SphereVec{fMul(v[rot], scale), fMul(v[(rot + 1) % 3], scale), fMul(v[(rot + 2) % 3], scale)};
    }
    case 7: {
      const float a = r.range(0.5f, 1.0f);
      SphereVec t{r.sign(a), r.sign(a), r.range(-a, a)};
      if (r.coin()) { const float x = t.x; t.x = t.z; t.z = x; }
      if (r.coin()) { const float y = t.y; t.y = t.z; t.z = y; }
      return t;
    }
    default: {
      float c[3] = {r.sign(0.0f), r.sign(0.0f), r.sign(0.0f)};
      c[r.below(3)] = r.sign(r.range(0.25f, 3.0f));
      return SphereVec{c[0], c[1], c[2]};
    }
  }
}

#ifndef __CUDA_ARCH__
// which cube-input face cubeInputHD picks (-1: none), whether |gx| or |gy| is exactly 1 there, whether a face it tries
// has its major component exactly at the +-0.5 threshold, and whether the face it picks does (host replica for the ledger)
int cubeFaceOf(float tx, float ty, float tz, bool* gOne, bool* half, bool* pickedHalf) {
  for (int f = 0; f < 6; ++f) {
    const float major = f < 2 ? tz : (f < 4 ? tx : ty), a = f < 4 && f >= 2 ? tz : tx, b = f < 4 ? ty : tz;
    *half = *half || major == ((f & 1) == 0 ? -0.5f : 0.5f);
    if ((f & 1) == 0 ? !(major <= -0.5f) : !(major >= 0.5f)) continue;
    const float gx = a / major, gy = b / major;
    if (gx >= -1.0f && gx <= 1.0f && gy >= -1.0f && gy <= 1.0f) {
      *gOne = std::fabs(gx) == 1.0f || std::fabs(gy) == 1.0f;
      *pickedHalf = std::fabs(major) == 0.5f;
      return f;
    }
  }
  return -1;
}
#endif

// a sphere geometry for the input lookup alone: equirect or cube input, mono / LR / TB input, input sizes odd and even
T360_HD SphereGeometry drawInputGeometry(Draw& r) {
  SphereGeometry g{};
  g.mapW = g.mapH = 16;
  g.kernelSize = 2;
  g.cubeInput = r.below(3) == 0;
  const int pack = r.below(3);
  g.packLR = pack == 1;
  g.packTB = pack == 2;
  g.inW = 1 + r.below(8192);
  g.inH = 1 + r.below(8192);
  g.inputExpand = r.coin() ? 1.0f : r.range(1.0f, 1.1f);
  g.inPixelWidth = fDiv(1.0f, static_cast<float>(g.inW));
  if (g.packLR) g.inPixelWidth = fMul(g.inPixelWidth, 2.0f);
  return g;
}

// a rig from the table (two-lens only, or any), copied so a probe can move a lens's coverage edge
T360_HD LensRigModel drawRig(const GateData& D, Draw& r, bool twoLens) { return D.rig[twoLens ? r.below(D.nRig2) : r.below(D.nRig)]; }
// a direction for a rig: a lens axis (rho == 0 on an axis-aligned rig), z == 0 (z1 == z0 on a back-to-back rig), or random
T360_HD SphereVec drawRigDirection(Draw& r, const LensRigModel& rig) {
  switch (r.below(4)) {
    case 0: {
      const LensModel& L = rig.lens[r.below(rig.numLenses)];
      return SphereVec{L.m[6], L.m[7], L.m[8]};
    }
    case 1: return SphereVec{r.range(-1.0f, 1.0f), r.range(-1.0f, 1.0f), r.sign(0.0f)};
    default: return drawVec(r, -1.0f, 1.0f);
  }
}

#define CHAIN_LAYOUTS "cube32 cube23 eac equirect barrel barrelSplit "
#define CHAIN_PLAIN_LAYOUTS "cube32 cube23 eac equirect - - "
#define CHAIN_NO_LAYOUTS "- - - - - - "
#define CHAIN_CLASSES "offCentreHorizontal offCentreFull splitLR splitTBvflip packLR packTB cubeInput oddMap oddInput K1 K2 K4 K8 -"

struct TwinGate {
  static constexpr uint64_t kSeed = 20261017ull;
  static constexpr int kOut = 4;
  enum Probe {
    kAtanf, kAsinf, kSqrt, kSincCos, kTrunc, kRound, kQuantize,                                  // A
    kAtan2, kPixelCentre, kToPixel, kRotate, kRayToSphere, kWarpOffCentre, kSphereInput, kLens,  // B
    kLensBlend0, kLensBlend1, kCameraRay,
    kFlat, kSphere, kSpherePlain, kLensChain, kLensChainPlain, kBlendChain, kBlendChainPlain,    // C
    kRectCtx, kRectCtxPinhole, kRectLens, kRectLensPinhole,
    kProbes
  };
  // the classes each probe's ledger names, in CLASS order, and the inputs per probe
  static constexpr ProbeInfo kInfo[kProbes] = {
      {"atanf", "", 1ull << 32, true},
      {"asinf", "", 1ull << 32, true},
      {"fSqrt", "", 1ull << 32, true},
      {"sincCos", "", 1ull << 32, true},
      {"truncToInt", "", 1ull << 32, true},
      {"roundHalfEven", "", 1ull << 32, true},
      {"quantizeAxis", "", 1ull << 32, true},
      {"libmAtan2f", "nan xIsOne zero inf ratioAbove2^60 negativeXRatioBelow2^-60 atanfTiny atanfBelow7/16 atanfBelow11/16 "
                     "atanfBelow19/16 atanfBelow39/16 atanfBelow2^24 atanfAbove2^24 atanfNearSplit", 1ull << 28},
      {"pixelCentre", "", 1ull << 28},
      {"toPixel", "", kToPixelFloats * kToPixelPlanes},
      {"rotateHD", "angles rawMatrix signedZeroQ", 1ull << 28},
      {"rayToSphereHD", "discNotPositive discBelowAlong ordinary", 1ull << 28},
      {"warpOffCentreHD", "horizontalWarped horizontalUnwarped fullWarped fullUnwarped", 1ull << 28},
      {"sphereInputHD", "cutPlusZero cutMinusZero pole barrelClampLow barrelClampHigh barrelNaN packLR0 packLR1 packTB0 packTB1 "
                        "face0 face1 face2 face3 face4 face5 gIsOne majorIsHalf noFace noFaceWithoutNaN pickedMajorIsHalf", 1ull << 28},
      {"lensPosition", "oneLens secondLens z1EqualsZ0 covered uncovered rhoZero thetaIsThetaMax thetaMaxPi", 1ull << 28},
      {"lensBlendPosition0", "bothCoveredW0 bothCoveredW256 ramp tie only0 only1 neither", 1ull << 27},
      {"lensBlendPosition1", "bothCoveredW0 bothCoveredW256 ramp tie only0 only1 neither", 1ull << 27},
      {"cameraRay", "equidistantRho0 equidistantRhoAbovePi/2 equidistantRhoAbovePi stereoBelow1 stereoAt1 stereoAbove1 panniniD0 "
                    "panniniD1 panniniKAbove1e7 equidistantZeroXY stereoZeroXY panniniZeroXY", 1ull << 28},
      {"flatSample", CHAIN_NO_LAYOUTS CHAIN_CLASSES " fold noFold", 1ull << 26},
      {"sphereSample<BARREL>", CHAIN_LAYOUTS CHAIN_CLASSES " deadZone", 1ull << 26},
      {"sphereSample<plain>", CHAIN_PLAIN_LAYOUTS CHAIN_CLASSES, 1ull << 26},
      {"lensSample<BARREL>", CHAIN_LAYOUTS CHAIN_CLASSES " covered uncovered", 1ull << 26},
      {"lensSample<plain>", CHAIN_PLAIN_LAYOUTS CHAIN_CLASSES " covered uncovered", 1ull << 26},
      {"lensBlendSample<BARREL>", CHAIN_LAYOUTS CHAIN_CLASSES " w0 w256 ramp", 1ull << 26},
      {"lensBlendSample<plain>", CHAIN_PLAIN_LAYOUTS CHAIN_CLASSES " w0 w256 ramp", 1ull << 26},
      {"rectilinearSample<ctx,any>", CHAIN_NO_LAYOUTS CHAIN_CLASSES " pinhole equidistant stereographic pannini", 1ull << 26},
      {"rectilinearSample<ctx,pinhole>", CHAIN_NO_LAYOUTS CHAIN_CLASSES " pinhole", 1ull << 26},
      {"rectilinearSample<lens,any>", CHAIN_NO_LAYOUTS CHAIN_CLASSES " pinhole equidistant stereographic pannini", 1ull << 26},
      {"rectilinearSample<lens,pinhole>", CHAIN_NO_LAYOUTS CHAIN_CLASSES " pinhole", 1ull << 26},
  };
  // bit 3 of word 1 of a sphereInputHD element in the second block
  static constexpr Flip kFlip = {kSphereInput, 3 * kBlock / 2 - 12345, 1, 3};

  using Data = GateData;
  struct HostData {
    std::vector<Rotation> rot;
    std::vector<LensRigModel> rig;
    std::vector<RectilinearCamera> cam;
    std::vector<GeoEntry> geo;
    std::vector<float> tab;
    int nRotReal = 0, nRig2 = 0, nCamPinhole = 0, nGeoPlain = 0;
  };
  template <int P>
  static T360_HD void probe(const Data& D, uint64_t i, Words<kOut>& w);
  static HostData makeData();
  static Data view(const HostData& H, int shift);
  static Data deviceData(const HostData& H, Data D, Uploads& up) {
    D.rot = up(H.rot); D.rig = up(H.rig); D.cam = up(H.cam); D.geo = up(H.geo); D.tab = up(H.tab);
    return D;
  }
};

// ---- the probes -------------------------------------------------------------------------------------------------------
template <int P>
T360_HD void TwinGate::probe(const GateData& D, uint64_t i, Words<kOut>& w) {
  Draw r(kSeed, P, i);
  if constexpr (P <= kQuantize) {
    const uint32_t b = patternA(D, i);
    const float x = bitsFloat(b);
    w.in[0] = b;
    if constexpr (P == kAtanf) w.out[0] = fw(libmAtanf(x));
    if constexpr (P == kAsinf) w.out[0] = fw(libmAsinf(x));
    if constexpr (P == kSqrt) w.out[0] = fw(fSqrt(x));
    if constexpr (P == kSincCos) {
      float s, c;
      sincCos(x, &s, &c);
      w.out[0] = fw(s);
      w.out[1] = fw(c);
    }
    if constexpr (P == kTrunc) w.out[0] = iw(truncToInt(x));
    if constexpr (P == kRound) w.out[0] = iw(roundHalfEven(x));
    if constexpr (P == kQuantize) {
      for (int k = 0; k < 4; ++k) {
        int first, frac;
        quantizeAxis(x, 1 << k, &first, &frac);
        w.out[k] = iw(first) << 5 | iw(frac);
      }
    }
  } else if constexpr (P == kAtan2) {
    uint32_t yb, xb;
    if (i < static_cast<uint64_t>(t360gate::kAtan2Specials * t360gate::kAtan2Specials))
      t360gate::atan2SpecialPair(static_cast<int>(i), &yb, &xb);
    else
      t360gate::atan2RandomPair(kSeed, i, &yb, &xb);
    w.in[0] = yb;
    w.in[1] = xb;
    w.out[0] = fw(libmAtan2f(bitsFloat(yb), bitsFloat(xb)));
#ifndef __CUDA_ARCH__
    const uint32_t ix = xb & 0x7fffffffu, iy = yb & 0x7fffffffu;
    const int32_t d = static_cast<int32_t>(iy) - static_cast<int32_t>(ix);
    const bool special = ix > 0x7f800000u || iy > 0x7f800000u || xb == 0x3f800000u || iy == 0 || ix == 0 || ix == 0x7f800000u ||
                         iy == 0x7f800000u;
    CLASS(0, ix > 0x7f800000u || iy > 0x7f800000u);
    CLASS(1, xb == 0x3f800000u && iy <= 0x7f800000u);
    CLASS(2, (iy == 0 || ix == 0) && ix <= 0x7f800000u && iy <= 0x7f800000u);
    CLASS(3, (ix == 0x7f800000u || iy == 0x7f800000u) && ix <= 0x7f800000u && iy <= 0x7f800000u);
    CLASS(4, !special && d > 0x1e7fffff);
    CLASS(5, !special && d <= 0x1e7fffff && static_cast<int32_t>(xb) < 0 && (d >> 23) < -60);
    if (!special && d <= 0x1e7fffff && !(static_cast<int32_t>(xb) < 0 && (d >> 23) < -60)) {
      const uint32_t z = floatBits(bitsFloat(yb) / bitsFloat(xb)) & 0x7fffffffu;  // atanf's argument
      CLASS(6, z <= 0x30ffffffu);
      CLASS(7, z > 0x30ffffffu && z <= 0x3edfffffu);
      CLASS(8, z > 0x3edfffffu && z <= 0x3f2fffffu);
      CLASS(9, z > 0x3f2fffffu && z <= 0x3f97ffffu);
      CLASS(10, z > 0x3f97ffffu && z <= 0x401bffffu);
      CLASS(11, z > 0x401bffffu && z <= 0x4bffffffu);
      CLASS(12, z > 0x4bffffffu);
      for (uint32_t t : {0x3edfffffu, 0x3f2fffffu, 0x3f97ffffu, 0x401bffffu, 0x4bffffffu})
        CLASS(13, z + 4 >= t && z <= t + 5);
    }
#endif
  } else if constexpr (P == kPixelCentre) {
    const int n = static_cast<int>(i >> 14) + 1, j = static_cast<int>(i & 16383);
    w.in[0] = iw(j);
    w.in[1] = iw(n);
    if (j < n) w.out[0] = fw(pixelCentre(j, n));
  } else if constexpr (P == kToPixel) {
    const uint64_t k = i % kToPixelFloats;
    const int n = toPixelWidth(static_cast<int>(i / kToPixelFloats));
    const uint32_t b = k <= 0x40000000ull ? static_cast<uint32_t>(k) : static_cast<uint32_t>(0x80000000ull + (k - 0x40000001ull));
    w.in[0] = b;
    w.in[1] = iw(n);
    w.out[0] = fw(toPixel(bitsFloat(b), n));
  } else if constexpr (P == kRotate) {
    const int k = r.below(D.nRot);
    const SphereVec q = drawQ(r), t = rotateHD(D.rot[k], q);
    w.in[0] = iw(k); w.in[1] = floatBits(q.x); w.in[2] = floatBits(q.y); w.in[3] = floatBits(q.z);
    w.out[0] = fw(t.x); w.out[1] = fw(t.y); w.out[2] = fw(t.z);
    CLASS(0, k < D.nRotReal);
    CLASS(1, k >= D.nRotReal);
    CLASS(2, (floatBits(q.x) | floatBits(q.y) | floatBits(q.z)) & 0x80000000u && (q.x == 0.0f || q.y == 0.0f || q.z == 0.0f));
  } else if constexpr (P == kRayToSphere) {
    SphereVec dv = r.coin() ? drawVec(r, -1.0f, 1.0f) : drawDirection(r, 8);
    const SphereVec o = drawOffset(r);
    const float t = rayToSphereHD(dv.x, dv.y, dv.z, o.x, o.y, o.z);
    w.in[0] = floatBits(dv.x); w.in[1] = floatBits(dv.y); w.in[2] = floatBits(dv.z); w.in[3] = floatBits(o.x);
    w.out[0] = fw(t);
#ifndef __CUDA_ARCH__
    const float along = dv.x * -o.x + dv.y * -o.y + dv.z * -o.z, off2 = o.x * o.x + o.y * o.y + o.z * o.z;
    const float disc = static_cast<float>(static_cast<double>(along * along - off2) + 1.0);
    CLASS(0, disc <= 0.0f);
    CLASS(1, disc > 0.0f && std::sqrt(disc) < along);
    CLASS(2, disc > 0.0f && !(std::sqrt(disc) < along));
#endif
  } else if constexpr (P == kWarpOffCentre) {
    SphereGeometry g{};
    g.offCentre = true;
    g.horizontalOffset = r.coin();
    const SphereVec o = drawOffset(r);
    g.ox = o.x; g.oy = o.y; g.oz = o.z;
    SphereVec q = drawQ(r);
    const SphereVec q0 = q;
    warpOffCentreHD(g, q);
    w.in[0] = floatBits(q0.x); w.in[1] = floatBits(q0.y); w.in[2] = floatBits(q0.z); w.in[3] = iw(g.horizontalOffset);
    w.out[0] = fw(q.x); w.out[1] = fw(q.y); w.out[2] = fw(q.z);
#ifndef __CUDA_ARCH__
    SphereVec n = q0;
    const float len = std::sqrt(n.x * n.x + n.y * n.y + n.z * n.z);
    n = {n.x / len, n.y / len, n.z / len};
    if (g.horizontalOffset) {
      const float h = std::sqrt(n.x * n.x + n.z * n.z);
      n = {n.x / h, n.y / h, n.z / h};
    }
    const float t = g.horizontalOffset ? rayToSphereHD(n.x, 0, n.z, g.ox, 0, g.oz) : rayToSphereHD(n.x, n.y, n.z, g.ox, g.oy, g.oz);
    CLASS(0, g.horizontalOffset && t > 0.0f);
    CLASS(1, g.horizontalOffset && !(t > 0.0f));
    CLASS(2, !g.horizontalOffset && t > 0.0f);
    CLASS(3, !g.horizontalOffset && !(t > 0.0f));
#endif
  } else if constexpr (P == kSphereInput) {
    const SphereGeometry g = drawInputGeometry(r);
    const bool barrel = r.coin(), eye = r.coin();
    const SphereVec t = drawDirection(r, r.below(9));
    float u, v;
    sphereInputHD(g, barrel, eye, t, &u, &v);
    w.in[0] = floatBits(t.x); w.in[1] = floatBits(t.y); w.in[2] = floatBits(t.z);
    w.in[3] = iw(g.cubeInput) | iw(g.packLR) << 1 | iw(g.packTB) << 2 | iw(barrel) << 3 | iw(eye) << 4 | iw(g.inW) << 5;
    w.out[0] = fw(u); w.out[1] = fw(v);
#ifndef __CUDA_ARCH__
    if (!g.cubeInput) {
      SphereGeometry plain = g;
      plain.packLR = plain.packTB = false;
      float u0, v0;
      sphereInputHD(plain, false, eye, t, &u0, &v0);
      const float lo = g.inPixelWidth * 0.5f, hi = 1.0f - lo;
      CLASS(0, t.x == 0.0f && !std::signbit(t.x) && t.z < 0.0f);
      CLASS(1, t.x == 0.0f && std::signbit(t.x) && t.z < 0.0f);
      CLASS(2, t.x == 0.0f && t.z == 0.0f && t.y != 0.0f);
      CLASS(3, barrel && u0 < lo);
      CLASS(4, barrel && u0 > hi);
      CLASS(5, barrel && u0 != u0);
      CLASS(6, g.packLR && !eye);
      CLASS(7, g.packLR && eye);
      CLASS(8, g.packTB && !eye);
      CLASS(9, g.packTB && eye);
    } else {
      const float n = std::sqrt(t.x * t.x + t.y * t.y + t.z * t.z);
      bool gOne = false, half = false, pickedHalf = false;
      const int f = cubeFaceOf(t.x / n, t.y / n, t.z / n, &gOne, &half, &pickedHalf);
      if (f >= 0) CLASS(10 + f, true);
      CLASS(16, f >= 0 && gOne);
      CLASS(17, half);
      CLASS(18, f < 0);
      CLASS(19, f < 0 && t.x == t.x && t.y == t.y && t.z == t.z);  // the fallback without a NaN component
      CLASS(20, f >= 0 && pickedHalf);
    }
#endif
  } else if constexpr (P == kLens) {
    LensRigModel rig = drawRig(D, r, false);
    const SphereVec d = drawRigDirection(r, rig);
    const bool tie = r.below(4) == 0;
    if (tie) {  // thetaMax exactly the theta of d for the lens lensPosition picks
      const float z0 = lensRow(rig.lens[0].m + 6, d), z1 = rig.numLenses > 1 ? lensRow(rig.lens[1].m + 6, d) : z0;
      LensModel& L = rig.lens[z1 > z0 ? 1 : 0];
      L.thetaMax = lensHit(L, d, z1 > z0 ? z1 : z0, 64, 64).theta;
    }
    const int inW = 1 + r.below(8192), inH = 1 + r.below(8192);
    float px, py;
    lensPosition(rig, d, inW, inH, &px, &py);
    w.in[0] = floatBits(d.x); w.in[1] = floatBits(d.y); w.in[2] = floatBits(d.z); w.in[3] = iw(tie);
    w.out[0] = fw(px); w.out[1] = fw(py);
#ifndef __CUDA_ARCH__
    const float z0 = lensRow(rig.lens[0].m + 6, d), z1 = rig.numLenses > 1 ? lensRow(rig.lens[1].m + 6, d) : z0;
    const LensModel& L = rig.lens[z1 > z0 ? 1 : 0];
    const LensHit h = lensHit(L, d, z1 > z0 ? z1 : z0, inW, inH);
    const float X = lensRow(L.m, d), Y = lensRow(L.m + 3, d);
    CLASS(0, rig.numLenses == 1);
    CLASS(1, rig.numLenses == 2 && z1 > z0);
    CLASS(2, rig.numLenses == 2 && z1 == z0);
    CLASS(3, h.covered);
    CLASS(4, !h.covered);
    CLASS(5, h.covered && X * X + Y * Y == 0.0f);
    CLASS(6, h.theta == L.thetaMax);
    CLASS(7, L.thetaMax >= 3.1415926f);
#endif
  } else if constexpr (P == kLensBlend0 || P == kLensBlend1) {
    const LensRigModel rig = drawRig(D, r, true);
    const SphereVec d = drawRigDirection(r, rig);
    float s;
    switch (r.below(4)) {
      case 0: s = 0.0f; break;
      case 1: {  // theta0 - theta1 scaled to 1/512: tw on a .5 tie
        const float t0 = lensHit(rig.lens[0], d, lensRow(rig.lens[0].m + 6, d), 64, 64).theta;
        const float t1 = lensHit(rig.lens[1], d, lensRow(rig.lens[1].m + 6, d), 64, 64).theta;
        s = fDiv(static_cast<float>(r.below(255) - 127) * 0.001953125f, fSub(t0, t1));
        break;
      }
      default: s = fDiv(1.0f, fMul(2.0f, r.range(0.0175f, 0.7f)));  // seams of 1 to 40 degrees
    }
    const int inW = 1 + r.below(8192), inH = 1 + r.below(8192);
    float p0[2], p1[2];
    const int wt = lensBlendPosition(rig, s, d, inW, inH, p0, p1);
    const float* p = P == kLensBlend0 ? p0 : p1;
    w.in[0] = floatBits(d.x); w.in[1] = floatBits(d.y); w.in[2] = floatBits(d.z); w.in[3] = floatBits(s);
    w.out[0] = iw(wt); w.out[1] = fw(p[0]); w.out[2] = fw(p[1]);
#ifndef __CUDA_ARCH__
    const LensHit h0 = lensHit(rig.lens[0], d, lensRow(rig.lens[0].m + 6, d), inW, inH);
    const LensHit h1 = lensHit(rig.lens[1], d, lensRow(rig.lens[1].m + 6, d), inW, inH);
    const float tw = (0.5f + (h0.theta - h1.theta) * s) * 256.0f;
    CLASS(0, h0.covered && h1.covered && wt == 0);
    CLASS(1, h0.covered && h1.covered && wt == 256);
    CLASS(2, wt > 0 && wt < 256);
    CLASS(3, h0.covered && h1.covered && tw > 0.0f && tw < 256.0f && tw - std::floor(tw) == 0.5f);
    CLASS(4, h0.covered && !h1.covered);
    CLASS(5, !h0.covered && h1.covered);
    CLASS(6, !h0.covered && !h1.covered);
#endif
  } else if constexpr (P == kCameraRay) {
    const int k = D.nCamPinhole + r.below(D.nCam - D.nCamPinhole);
    const RectilinearCamera& c = D.cam[k];
    float X, Y;
    switch (r.below(4)) {
      case 0: X = r.sign(0.0f); Y = r.range(-1.0f, 1.0f); break;
      case 1: X = r.range(-1.0f, 1.0f); Y = r.sign(0.0f); break;
      case 2: X = r.sign(r.coin() ? 1.0f : 0.0f); Y = r.sign(r.coin() ? 1.0f : 0.0f); break;
      default: X = r.range(-1.0f, 1.0f); Y = r.range(-1.0f, 1.0f);
    }
    const SphereVec q = cameraRay(c, X, Y);
    w.in[0] = iw(k); w.in[1] = floatBits(X); w.in[2] = floatBits(Y);
    w.out[0] = fw(q.x); w.out[1] = fw(q.y); w.out[2] = fw(q.z);
#ifndef __CUDA_ARCH__
    const float a = X * c.cx, b = Y * c.cy;
    const float rho = std::sqrt(a * a + b * b), ab = a * a + b * b;
    const float ue = X * c.cx * c.e;
    const bool zero = X == 0.0f || Y == 0.0f;
    CLASS(0, c.model == kCameraEquidistant && rho == 0.0f);
    CLASS(1, c.model == kCameraEquidistant && rho > 1.5707964f);
    CLASS(2, c.model == kCameraEquidistant && rho > 3.1415927f);
    CLASS(3, c.model == kCameraStereographic && ab < 1.0f);
    CLASS(4, c.model == kCameraStereographic && ab == 1.0f);
    CLASS(5, c.model == kCameraStereographic && ab > 1.0f);
    CLASS(6, c.model == kCameraPannini && c.d == 0.0f);
    CLASS(7, c.model == kCameraPannini && c.d == 1.0f);
    CLASS(8, c.model == kCameraPannini && ue * ue > 1e7f);
    CLASS(9, c.model == kCameraEquidistant && zero);
    CLASS(10, c.model == kCameraStereographic && zero);
    CLASS(11, c.model == kCameraPannini && zero);
#endif
  } else {  // tier C: whole chains
    constexpr bool kPlain = P == kSpherePlain || P == kLensChainPlain || P == kBlendChainPlain;
    const int gi = r.below(kPlain ? D.nGeoPlain : D.nGeo);
    const GeoEntry& e = D.geo[gi];
    const SphereGeometry& g = e.g;
    const float *colTab = D.tab + e.colTab, *rowTab = D.tab + e.rowTab;
    const int pi = r.below(g.mapH), pj = r.below(g.mapW);
    const Rotation& rot = D.rot[r.below(D.nRotReal)];
    w.in[0] = iw(gi); w.in[1] = iw(pi); w.in[2] = iw(pj);
    int32_t c0 = 0, rp = 0;
    if constexpr (P == kFlat) {
      FlatView v;
      v.yaw = r.below(8) == 0 ? r.sign(180.0f) : r.range(-400.0f, 400.0f);
      v.pitch = r.below(8) == 0 ? r.sign(90.0f) : r.range(-200.0f, 200.0f);
      v.hfov = r.range(1.0f, 360.0f);
      v.vfov = r.range(1.0f, 180.0f);
      flatSample(v, g, pi, pj, &c0, &rp);
      w.in[3] = floatBits(v.pitch);
#ifndef __CUDA_ARCH__
      bool fold;
      float y = pixelCentre(pi, g.mapH);
      if (g.splitTB) splitEye(y, g.vflip);
      flatLat(v, y, &fold);
      CLASS(20, fold);
      CLASS(21, !fold);
#endif
    } else if constexpr (P == kSphere || P == kSpherePlain) {
      sphereSample<P == kSphere>(g, rot, colTab, rowTab, pi, pj, &c0, &rp);
#ifndef __CUDA_ARCH__
      bool eye;
      SphereVec t;
      CLASS(20, !spherePoint<true>(g, rot, colTab, rowTab, pi, pj, &eye, &t));
#endif
    } else if constexpr (P == kLensChain || P == kLensChainPlain) {
      const int k = r.below(D.nRig);
      w.in[3] = iw(k);
      lensSample<P == kLensChain>(g, rot, D.rig[k], colTab, rowTab, pi, pj, &c0, &rp);
#ifndef __CUDA_ARCH__
      float px, py;
      lensPoint<true>(g, rot, D.rig[k], colTab, rowTab, pi, pj, &px, &py);
      CLASS(20, px == px);
      CLASS(21, px != px);
#endif
    } else if constexpr (P == kBlendChain || P == kBlendChainPlain) {
      const int k = r.below(D.nRig2);
      const float s = fDiv(1.0f, fMul(2.0f, r.range(0.0175f, 0.7f)));
      w.in[3] = iw(k);
      int32_t rec0[2], rec1[2];
      const int wt = lensBlendSample<P == kBlendChain>(g, rot, D.rig[k], s, colTab, rowTab, pi, pj, rec0, rec1);
      w.out[0] = iw(rec0[0]) * 512u + iw(wt);  // col0 fits 17 bits, w 9
      w.out[1] = iw(rec0[1]);
      w.out[2] = iw(rec1[0]);
      w.out[3] = iw(rec1[1]);
      CLASS(20, wt == 0);
      CLASS(21, wt == 256);
      CLASS(22, wt > 0 && wt < 256);
    } else {  // rectilinear views
      constexpr bool kLensIn = P == kRectLens || P == kRectLensPinhole;
      constexpr bool kAny = P == kRectCtx || P == kRectLens;
      const int k = kAny ? r.below(D.nCam) : r.below(D.nCamPinhole);
      const int rk = r.below(D.nRig);
      w.in[3] = iw(k);
      rectilinearSample<kLensIn, kAny>(g, D.cam[k], D.rig[rk], pi, pj, &c0, &rp);
      CLASS(20 + D.cam[k].model, true);
    }
    if constexpr (!(P == kBlendChain || P == kBlendChainPlain)) {
      w.out[0] = iw(c0);
      w.out[1] = iw(rp);
    }
#ifndef __CUDA_ARCH__
    // the geometry classes every chain is meant to reach
    const int layoutClass[] = {0, 1, -1, 3, 4, 5, 2};  // CUBEMAP_32, 23_OFFCENTER, EAC, EQUIRECT, BARREL, BARREL_SPLIT
    if (P != kFlat && P < kRectCtx) CLASS(layoutClass[g.outputLayout], true);
    CLASS(6, g.offCentre && g.horizontalOffset);
    CLASS(7, g.offCentre && !g.horizontalOffset);
    CLASS(8, g.splitLR);
    CLASS(9, g.splitTB && g.vflip);
    CLASS(10, g.packLR);
    CLASS(11, g.packTB);
    CLASS(12, g.cubeInput);
    CLASS(13, (g.mapW & 1) || (g.mapH & 1));
    CLASS(14, (g.inW & 1) || (g.inH & 1));
    CLASS(15, g.kernelSize == 1);
    CLASS(16, g.kernelSize == 2);
    CLASS(17, g.kernelSize == 4);
    CLASS(18, g.kernelSize == 8);
#endif
  }
}

TwinGate::HostData TwinGate::makeData() {
  HostData H;
  HostRng g{kSeed * 7919};
  const float angles[] = {0.0f, -0.0f, 90.0f, -90.0f, 180.0f, -180.0f, 45.0f, 270.0f, 1e6f};
  auto angle = [&] { return g.below(4) == 0 ? angles[g.below(9)] : static_cast<float>(g.uniform(-400, 400)); };
  for (int k = 0; k < 1536; ++k) H.rot.push_back(rotationFromAngles(angle(), angle(), angle()));
  H.nRotReal = static_cast<int>(H.rot.size());
  for (int k = 0; k < 512; ++k) {  // raw matrices: entries +-0, +-1, or arbitrary in [-1, 1]
    float m[9];
    for (float& v : m) {
      const int c = g.below(5);
      v = c == 0 ? 0.0f : c == 1 ? -0.0f : c == 2 ? 1.0f : c == 3 ? -1.0f : static_cast<float>(g.uniform(-1, 1));
    }
    H.rot.push_back(Rotation{m[0], m[1], m[2], m[3], m[4], m[5], m[6], m[7], m[8]});
  }

  // rigs: two-lens first (random, back-to-back axis-aligned), then one-lens (random, axis-aligned)
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
    for (float& k : L.k) k = static_cast<float>(g.uniform(-0.1, 0.1));
    const int t = g.below(4);
    L.thetaMax = t == 0 ? static_cast<float>(M_PI) : static_cast<float>(g.uniform(0.2, t == 1 ? M_PI_2 : M_PI));
    return L;
  };
  for (int k = 0; k < 384; ++k) {
    LensRigModel rig{};
    rig.numLenses = 2;
    const bool aligned = k % 3 == 0;
    rig.lens[0] = lens(aligned, false);
    rig.lens[1] = lens(aligned, true);
    H.rig.push_back(rig);
  }
  H.nRig2 = static_cast<int>(H.rig.size());
  for (int k = 0; k < 128; ++k) {
    LensRigModel rig{};
    rig.numLenses = 1;
    rig.lens[0] = lens(k % 4 == 0, false);
    H.rig.push_back(rig);
  }

  // cameras: pinholes first, then each other model over its range and at its edges
  auto pose = [&](int model, double hfov, double vfov, double d) {  // the library's own constants (cameraConstants)
    H.cam.push_back(cameraConstants(model, static_cast<float>(d), angle(), angle(), angle(), static_cast<float>(hfov), static_cast<float>(vfov)));
  };
  for (int k = 0; k < 256; ++k) pose(kCameraPinhole, g.uniform(1, 179), g.uniform(1, 179), 0);
  pose(kCameraPinhole, 179, 179, 0);
  H.nCamPinhole = static_cast<int>(H.cam.size());
  for (int k = 0; k < 256; ++k) pose(kCameraEquidistant, g.uniform(1, 360), g.uniform(1, 360), 0);
  for (double f : {180.0, 360.0, 250.0}) pose(kCameraEquidistant, f, f, 0);
  for (int k = 0; k < 256; ++k) pose(kCameraStereographic, g.uniform(1, 359), g.uniform(1, 359), 0);
  for (double f : {180.0, 359.0}) pose(kCameraStereographic, f, f, 0);  // cx == 1.0f: a^2 + b^2 == 1 at the edge
  for (int k = 0; k < 256; ++k) {
    const double d = g.uniform(0, 1), top = d < 1 ? 2.0 * std::acos(-d) * 180.0 / M_PI : 359.0;
    pose(kCameraPannini, g.uniform(1, std::min(359.0, top - 0.01)), g.uniform(1, 179), d);
  }
  for (double d : {0.0, 0.5, 0.9, 1.0})
    for (double delta : {1.0, 0.1, 0.01}) {  // hfov at the limit: cx up to ~1e4, k up to ~1e8
      const double top = d < 1 ? 2.0 * std::acos(-d) * 180.0 / M_PI : 359.0 + delta;
      pose(kCameraPannini, top - delta, g.uniform(1, 179), d);
    }

  // geometries: seeded contexts over every sphere output layout, input layout and stereo format, off-centre in both
  // modes, odd and even sizes, K = 1, 2, 4, 8; the barrel layouts last
  std::vector<std::pair<FrameTransformContext, std::array<int, 5>>> ctxs;
  const Layout layouts[] = {LAYOUT_CUBEMAP_32, LAYOUT_CUBEMAP_23_OFFCENTER, LAYOUT_EAC_32, LAYOUT_EQUIRECT, LAYOUT_BARREL, LAYOUT_BARREL_SPLIT};
  const StereoFormat stereo[] = {STEREO_FORMAT_MONO, STEREO_FORMAT_LR, STEREO_FORMAT_TB};
  for (int pass = 0; pass < 2; ++pass)
    for (int k = 0; k < 96; ++k) {
      const Layout layout = layouts[pass == 0 ? k % 4 : 4 + k % 2];
      FrameTransformContext c{};
      c.output_layout = layout;
      c.input_layout = g.below(3) == 0 ? LAYOUT_CUBEMAP_32 : LAYOUT_EQUIRECT;
      c.input_stereo_format = stereo[(k / 4) % 3];
      c.output_stereo_format = stereo[(k / 12) % 3];
      c.vflip = (k / 36) % 2;
      c.expand_coef = g.below(3) == 0 ? 1.0f : static_cast<float>(g.uniform(1.0, 1.1));
      c.input_expand_coef = g.below(2) == 0 ? 1.0f : static_cast<float>(g.uniform(1.0, 1.1));
      if (k % 3 == 1) {
        c.fixed_cube_offcenter_x = static_cast<float>(g.uniform(-0.7, 0.7));
        c.fixed_cube_offcenter_y = g.below(2) ? 0.0f : static_cast<float>(g.uniform(-0.7, 0.7));
        c.fixed_cube_offcenter_z = static_cast<float>(g.uniform(-0.7, 0.7));
        c.is_horizontal_offset = (k / 3) % 2;
      }
      const int K = 1 << (k % 4 == 0 ? 3 : (k / 2) % 4);
      ctxs.push_back({c, {8 + g.below(700), 8 + g.below(500), 16 + g.below(8000), 16 + g.below(4000), K}});
    }
  for (auto& [c, s] : ctxs) {
    GeoEntry e{};
    e.g = sphereGeometry(c, s[0], s[1], s[2], s[3], s[4]);
    const std::vector<float> t = buildSphereTables(e.g);
    e.colTab = static_cast<uint32_t>(H.tab.size());
    e.rowTab = e.colTab + static_cast<uint32_t>(t.empty() ? 0 : sphereTableRowOffset(e.g));
    H.tab.insert(H.tab.end(), t.begin(), t.end());
    H.geo.push_back(e);
    if (!barrelLayout(e.g.outputLayout)) H.nGeoPlain = static_cast<int>(H.geo.size());
  }
  H.tab.push_back(0.0f);
  return H;
}

GateData TwinGate::view(const HostData& H, int shift) {
  return GateData{H.rot.data(), static_cast<int>(H.rot.size()), H.nRotReal, H.rig.data(), static_cast<int>(H.rig.size()), H.nRig2,
                  H.cam.data(), static_cast<int>(H.cam.size()), H.nCamPinhole, H.geo.data(), static_cast<int>(H.geo.size()), H.nGeoPlain,
                  H.tab.data(), shift};
}

}  // namespace

int main(int argc, char** argv) { return runGate<TwinGate>(argc, argv); }
