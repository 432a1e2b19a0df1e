// Twin gate of the anti-aliased camera views: the device build of every float function the footprint adds
// (oriented_view.h: cameraXY, modelRay, rayDifferential, equirectJacobian, cubeInputFace, cubeJacobian, lensJacobian,
// mipLevelOf, mipScale, mipCameraPoint, mipCameraSample) against its host build, the one T360B200_cameraMipMaps runs.  The
// harness, its comparison rule and its modes are tests/twin_gate.cuh's.  Probes:
//   mipLevelOf         every 32-bit pattern of rho^2 (as a.a; b.b, the top level and the bias drawn): level and weight;
//   rayDifferential    each model's differential at drawn (X, Y) and half steps, cameras from cameraConstants;
//   equirectJacobian   drawn rays (near-pole, axis and arbitrary) and differentials, every input re-pack;
//   cubeJacobian       cubeInputFace of the normalised ray and the quotient rule on that face;
//   lensJacobian       drawn rig directions, rays on a lens axis (rho = 0, both signs of Z) included;
//   mipScale           drawn positions and level ratios;
//   mipCameraPoint / mipCameraSample, LENS = false and true: 2^24 (geometry, pixel) samples each over seeded contexts,
//   cameras of every model, rigs, maxLevel and lodBias.
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
  int nRig, nRigAxis;  // [0, nRigAxis): lenses along +-z (rho = 0 reachable)
  const ChainGeo* ctxGeo;
  int nCtxGeo;
  const ChainGeo* lensGeo;
  int nLensGeo;
};

struct MipGate {
  static constexpr uint64_t kSeed = 20261018ull;
  static constexpr int kOut = 6;
  enum Probe { kLod, kRayDiff, kEquirect, kCube, kLens, kScale, kPointCtx, kPointLens, kSampleCtx, kSampleLens, kProbes };
  static constexpr ProbeInfo kInfo[kProbes] = {
      {"mipLevelOf", "", 1ull << 32},       {"rayDifferential", "", 1ull << 26}, {"equirectJacobian", "", 1ull << 26},
      {"cubeJacobian", "", 1ull << 26},     {"lensJacobian", "", 1ull << 26},    {"mipScale", "", 1ull << 26},
      {"mipCameraPoint<ctx>", "", 1ull << 24},  {"mipCameraPoint<lens>", "", 1ull << 24}, {"mipCameraSample<ctx>", "", 1ull << 24},
      {"mipCameraSample<lens>", "", 1ull << 24},
  };
  // bit 5 of word 4 (the level) of a mipCameraSample<lens> element
  static constexpr Flip kFlip = {kSampleLens, kBlock / 2 + 4321, 4, 5};

  using Data = GateData;
  struct HostData {
    std::vector<RectilinearCamera> cam;
    std::vector<LensRigModel> rig;
    std::vector<ChainGeo> ctxGeo, lensGeo;
    int nRigAxis = 0;
  };
  template <int P>
  static T360_HD void probe(const Data& D, uint64_t i, Words<kOut>& w);
  static HostData makeData();
  static Data view(const HostData& H, int) {
    return GateData{H.cam.data(), static_cast<int>(H.cam.size()), H.rig.data(), static_cast<int>(H.rig.size()), H.nRigAxis,
                    H.ctxGeo.data(), static_cast<int>(H.ctxGeo.size()), H.lensGeo.data(), static_cast<int>(H.lensGeo.size())};
  }
  static Data deviceData(const HostData& H, Data D, Uploads& up) {
    D.cam = up(H.cam); D.rig = up(H.rig); D.ctxGeo = up(H.ctxGeo); D.lensGeo = up(H.lensGeo);
    return D;
  }
};

template <int P>
T360_HD void MipGate::probe(const GateData& D, uint64_t i, Words<kOut>& w) {
  Draw d(kSeed, P, i);
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

MipGate::HostData MipGate::makeData() {
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

}  // namespace

int main(int argc, char** argv) { return runGate<MipGate>(argc, argv); }
