// Twin gate of the rolling-shutter lens rigs: the device build of the rig motion's float steps (oriented_view.h:
// motionLens, the readout time and the fixed count of projections of lensMotionHit) and of the chains that call them
// (lensMotionPosition, lensMotionSample, cameraMotionSample) against their host build, the one T360B200_lensMotionMaps and
// T360B200_cameraMotionMaps run.  The harness, its comparison rule and its modes are tests/twin_gate.cuh's.  Probes:
//   motionLens          the interpolated M of drawn tables and readout times; the ledger's classes: t = 0, t = 1, and t on
//                       an inner segment boundary (t = k / (N - 1) with N - 1 a power of two, so s = t (N - 1) is exact);
//   lensMotionPosition  drawn rig directions, motions and readouts, hard (both = false and true) and feathered seams; the
//                       ledger's classes (lens 0's projections): a readout time clamped at 0 and at 1, the first
//                       projection covered and the last one not (the motion carried the point past the rim; the
//                       converse cannot happen: an uncovered projection keeps t, so every later one is the same), a
//                       projection at an inner segment boundary, and the hard seam, both lenses and the feathered seam;
//   lensMotionSample<BARREL> / <plain>: (geometry, pixel) samples over seeded contexts, rigs, photometries and motions;
//   cameraMotionSample<plain> / <MIP>: the same over seeded camera views.
#include "twin_gate.cuh"

using namespace t360;
using namespace t360gate;

namespace {

// ---- data the probes share (host-built, copied to the device) --------------------------------------------------------
struct SphereGeo {
  SphereGeometry g;  // a lens rig's output geometry (mono, equirect-like input fields)
  Rotation r;
  float seam;
  bool both, barrel;
  int colOffset, rowOffset;  // of its sphere tables in GateData::tables (-1: none)
};
struct CameraGeo {
  SphereGeometry g;  // a rig view's geometry
  MipGeometry m;
  int bias;
  float seam;
  bool both;
};
struct MotionRec {  // one motion: its table's offset in GateData::motionTables (2 lenses x n x 9), n and the readouts
  int offset, n;
  float readout[2][3];
};
struct GateData {
  const LensRigModel* rig;
  int nRig;
  const LensPhotoPlane* photo;
  int nPhoto;
  const MotionRec* motion;
  int nMotion;
  const float* motionTables;
  const SphereGeo* sphere;
  int nSphere;
  const float* tables;
  const CameraGeo* camGeo;
  int nCamGeo;
  const RectilinearCamera* cam;
  int nCam;
};

T360_HD SphereVec drawVec(Draw& d, float scale) { return SphereVec{d.component(scale), d.component(scale), d.component(scale)}; }
T360_HD RigMotion motionOf(const GateData& D, int k) {
  const MotionRec& m = D.motion[k];
  RigMotion mo;
  mo.table = D.motionTables + m.offset;
  mo.numSamples = m.n;
  for (int i = 0; i < 2; ++i)
    for (int c = 0; c < 3; ++c) mo.readout[i][c] = m.readout[i][c];
  return mo;
}
T360_HD uint32_t packLens(int level, int w, int gain) { return iw(level) | iw(w) << 8 | iw(gain) << 16; }

struct MotionGate {
  static constexpr uint64_t kSeed = 20261021ull;
  static constexpr int kOut = 11;
  enum Probe { kLens, kPosition, kSampleBarrel, kSamplePlain, kCameraPlain, kCameraMip, kProbes };
  static constexpr ProbeInfo kInfo[kProbes] = {
      {"motionLens", "t0 t1 boundary", 1ull << 26},
      {"lensMotionPosition", "clampedAt0 clampedAt1 coveredThenUncovered segmentBoundary hard feathered bothLenses", 1ull << 24},
      {"lensMotionSample<BARREL>", "", 1ull << 22},
      {"lensMotionSample<plain>", "", 1ull << 22},
      {"cameraMotionSample<plain>", "", 1ull << 22},
      {"cameraMotionSample<MIP>", "", 1ull << 22},
  };
  // bit 5 of word 4 (the gains) of a lensMotionSample<plain> element
  static constexpr Flip kFlip = {kSamplePlain, kBlock / 2 + 777, 4, 5};

  using Data = GateData;
  struct HostData {
    std::vector<LensRigModel> rig;
    std::vector<LensPhotoPlane> photo;
    std::vector<MotionRec> motion;
    std::vector<float> motionTables;
    std::vector<SphereGeo> sphere;
    std::vector<float> tables;
    std::vector<CameraGeo> camGeo;
    std::vector<RectilinearCamera> cam;
  };
  template <int P>
  static T360_HD void probe(const Data& D, uint64_t i, Words<kOut>& w);
  static HostData makeData();
  static Data view(const HostData& H, int) {
    return GateData{H.rig.data(), static_cast<int>(H.rig.size()), H.photo.data(), static_cast<int>(H.photo.size()), H.motion.data(),
                    static_cast<int>(H.motion.size()), H.motionTables.data(), H.sphere.data(), static_cast<int>(H.sphere.size()), H.tables.data(),
                    H.camGeo.data(), static_cast<int>(H.camGeo.size()), H.cam.data(), static_cast<int>(H.cam.size())};
  }
  static Data deviceData(const HostData& H, Data D, Uploads& up) {
    D.rig = up(H.rig); D.photo = up(H.photo); D.motion = up(H.motion); D.motionTables = up(H.motionTables);
    D.sphere = up(H.sphere); D.tables = up(H.tables); D.camGeo = up(H.camGeo); D.cam = up(H.cam);
    return D;
  }
};

template <int P>
T360_HD void MotionGate::probe(const GateData& D, uint64_t i, Words<kOut>& w) {
  Draw d(kSeed, P, i);
  for (int k = 0; k < kOut; ++k) w.out[k] = 0;
  const int mk = d.below(D.nMotion);
  const RigMotion mo = motionOf(D, mk);
  if constexpr (P == kLens) {
    const int lens = d.below(2), edge = d.below(4);
    const int n1 = mo.numSamples - 1;
    float t = d.range(0.0f, 1.0f);
    if (edge == 0) t = d.coin() ? 0.0f : 1.0f;
    if (edge == 1) t = fDiv(static_cast<float>(d.below(n1 + 1)), static_cast<float>(n1));
    const LensModel M = motionLens(D.rig[0].lens[0], mo, lens, t);
    w.in[0] = floatBits(t); w.in[1] = iw(mk); w.in[2] = iw(lens); w.in[3] = 0;
    for (int e = 0; e < 9; ++e) w.out[e] = fw(M.m[e]);
    const float s = fMul(t, static_cast<float>(n1));
    CLASS(0, t == 0.0f);
    CLASS(1, t == 1.0f);
    CLASS(2, s > 0.0f && s < static_cast<float>(n1) && s == static_cast<float>(truncToInt(s)));
  } else if constexpr (P == kPosition) {
    const LensRigModel& rig = D.rig[d.below(D.nRig)];
    const SphereVec t = drawVec(d, 1.0f);
    const LensPhotoPlane& c = D.photo[d.below(D.nPhoto)];
    const float s = rig.numLenses > 1 && d.coin() ? d.range(0.3f, 30.0f) : 0.0f;
    const bool both = d.coin();
    const int inW = 16 + d.below(8000), inH = 16 + d.below(8000);
    float p0[2], p1[2];
    int g0, g1;
    bool overlap;
    LensModel at[2];
    const int wt = lensMotionPosition(rig, mo, s, both, c, t, inW, inH, p0, p1, &g0, &g1, &overlap, at);
    w.in[0] = floatBits(t.x); w.in[1] = floatBits(t.y); w.in[2] = floatBits(t.z); w.in[3] = iw(mk);
    w.out[0] = fw(p0[0]); w.out[1] = fw(p0[1]); w.out[2] = fw(p1[0]); w.out[3] = fw(p1[1]);
    w.out[4] = iw(wt) | iw(overlap) << 9 | iw(both) << 10; w.out[5] = iw(g0) | iw(g1) << 16;
#ifndef __CUDA_ARCH__
    float times[kMotionProjections];
    LensModel a0;
    const LensHitR last = lensMotionHit(rig.lens[0], mo, 0, t, inW, inH, &a0, times);
    const LensModel first = motionLens(rig.lens[0], mo, 0, times[0]);
    const bool firstCovered = lensHit<true>(first, t, lensRow(first.m + 6, t), inW, inH).covered;
    bool at0 = false, at1 = false, boundary = false;
    for (int n = 1; n < kMotionProjections; ++n) {
      at0 |= times[n] == 0.0f;
      at1 |= times[n] == 1.0f;
      const float sn = fMul(times[n], static_cast<float>(mo.numSamples - 1));
      boundary |= sn > 0.0f && sn < static_cast<float>(mo.numSamples - 1) && sn == static_cast<float>(truncToInt(sn));
    }
    CLASS(0, at0);
    CLASS(1, at1);
    CLASS(2, firstCovered && !last.covered);
    CLASS(3, boundary);
    CLASS(4, s == 0.0f && !both);
    CLASS(5, s > 0.0f);
    CLASS(6, rig.numLenses > 1 && (both || s > 0.0f));
#endif
  } else if constexpr (P == kSampleBarrel || P == kSamplePlain) {
    int k = d.below(D.nSphere);
    while (D.sphere[k].barrel != (P == kSampleBarrel)) k = d.below(D.nSphere);  // (the kernels' instantiation for the layout)
    const SphereGeo& e = D.sphere[k];
    const LensRigModel& rig = D.rig[d.below(D.nRig)];
    const LensPhotoPlane& c = D.photo[d.below(D.nPhoto)];
    const float* colTab = e.colOffset < 0 ? nullptr : D.tables + e.colOffset;
    const float* rowTab = e.rowOffset < 0 ? nullptr : D.tables + e.rowOffset;
    const int row = d.below(e.g.mapH), col = d.below(e.g.mapW);
    const float s = rig.numLenses > 1 ? e.seam : 0.0f;
    int32_t r0[2], r1[2];
    int g0, g1;
    bool overlap;
    const int wt = P == kSampleBarrel
                       ? lensMotionSample<true>(e.g, e.r, rig, mo, s, e.both, c, colTab, rowTab, row, col, r0, r1, &g0, &g1, &overlap)
                       : lensMotionSample<false>(e.g, e.r, rig, mo, s, e.both, c, colTab, rowTab, row, col, r0, r1, &g0, &g1, &overlap);
    w.in[0] = iw(row); w.in[1] = iw(col); w.in[2] = iw(k); w.in[3] = iw(mk);
    w.out[0] = iw(r0[0]); w.out[1] = iw(r0[1]); w.out[2] = iw(r1[0]); w.out[3] = iw(r1[1]);
    w.out[4] = iw(g0) | iw(g1) << 16; w.out[5] = iw(wt) | iw(overlap) << 9;
  } else {
    const CameraGeo& e = D.camGeo[d.below(D.nCamGeo)];
    const RectilinearCamera& c = D.cam[d.below(D.nCam)];
    const LensRigModel& rig = D.rig[d.below(D.nRig)];
    const LensPhotoPlane& ph = D.photo[d.below(D.nPhoto)];
    const int row = d.below(e.g.mapH), col = d.below(e.g.mapW);
    const float s = rig.numLenses > 1 ? e.seam : 0.0f;
    CameraPhotoRecords lens[2] = {};
    bool overlap;
    const int wt = P == kCameraMip ? cameraMotionSample<true>(e.g, c, rig, mo, e.m, e.bias, s, e.both, ph, row, col, lens, &overlap)
                                   : cameraMotionSample<false>(e.g, c, rig, mo, e.m, e.bias, s, e.both, ph, row, col, lens, &overlap);
    w.in[0] = iw(row); w.in[1] = iw(col); w.in[2] = iw(c.model); w.in[3] = iw(mk);
    for (int l = 0; l < 2; ++l) {
      w.out[5 * l] = iw(lens[l].rec0[0]); w.out[5 * l + 1] = iw(lens[l].rec0[1]);
      w.out[5 * l + 2] = iw(lens[l].w ? lens[l].rec1[0] : 0); w.out[5 * l + 3] = iw(lens[l].w ? lens[l].rec1[1] : 0);
      w.out[5 * l + 4] = packLens(lens[l].level, lens[l].w, lens[l].gain);
    }
    w.out[10] = iw(wt) | iw(overlap) << 9 | iw(e.both) << 10;
  }
}

MotionGate::HostData MotionGate::makeData() {
  HostData H;
  HostRng g{kSeed * 7919};
  auto angle = [&] { return g.below(4) == 0 ? static_cast<float>(90 * g.below(4)) : static_cast<float>(g.uniform(-180, 180)); };
  auto matrix = [](const Rotation& r, float* m) {
    const float v[9] = {r.xx, r.xy, r.xz, r.yx, r.yy, r.yz, r.zx, r.zy, r.zz};
    std::memcpy(m, v, sizeof(v));
  };
  auto lens = [&](bool back) {
    LensModel L{};
    if (g.below(2)) {  // along +-z, its y row negated as lensRigModel stores it (-0 entries included)
      const float m[9] = {back ? -1.0f : 1.0f, 0.0f, back ? -0.0f : 0.0f, -0.0f, -1.0f, -0.0f, back ? -0.0f : 0.0f, 0.0f, back ? -1.0f : 1.0f};
      std::memcpy(L.m, m, sizeof(m));
    } else {
      matrix(rotationFromAngles(angle(), angle(), angle()), L.m);
    }
    L.ax = static_cast<float>(g.uniform(0.1, 0.5));
    L.bx = static_cast<float>(g.uniform(0.3, 0.7));
    L.ay = static_cast<float>(g.uniform(0.1, 0.5));
    L.by = static_cast<float>(g.uniform(0.3, 0.7));
    for (float& k : L.k) k = static_cast<float>(g.uniform(-0.05, 0.05));
    L.thetaMax = g.below(3) == 0 ? static_cast<float>(M_PI) : static_cast<float>(g.uniform(0.5, M_PI));
    return L;
  };
  for (int k = 0; k < 128; ++k) {
    LensRigModel rig{};
    rig.numLenses = 1 + k % 2;
    rig.lens[0] = lens(false);
    if (rig.numLenses == 2) rig.lens[1] = lens(true);
    H.rig.push_back(rig);
  }
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
  // motions: tables of 2 lenses x N samples, each a drawn base turned by small drawn angles (some samples equal to their
  // neighbours, some motions constant), readouts drawn from the header's examples, steep ones, constants on a segment
  // boundary (a = b = 0, c = k / (N - 1), N - 1 a power of two) and ones clamped at 0 or 1
  for (int k = 0; k < 256; ++k) {
    MotionRec m{};
    const int kind = k % 8;
    m.n = kind == 7 ? 1 + (1 << g.below(4)) : 2 + g.below(15);
    m.offset = static_cast<int>(H.motionTables.size());
    for (int l = 0; l < 2; ++l) {
      const float yaw = angle(), pitch = angle(), roll = angle();
      const bool still = g.below(4) == 0;
      float prev[9];
      for (int s = 0; s < m.n; ++s) {
        float e[9];
        if (still || (s > 0 && g.below(4) == 0)) {
          if (s == 0) matrix(rotationFromAngles(yaw, pitch, roll), e);
          else std::memcpy(e, prev, sizeof(e));
        } else {
          const double j = g.uniform(-3, 3);
          matrix(rotationFromAngles(yaw + static_cast<float>(j), pitch + static_cast<float>(g.uniform(-2, 2)), roll + static_cast<float>(j / 2)),
                 e);
        }
        if (still && s == 0 && g.below(2)) e[3] = e[5] = -0.0f;
        std::memcpy(prev, e, sizeof(e));
        H.motionTables.insert(H.motionTables.end(), e, e + 9);
      }
      float* r = m.readout[l];
      switch (kind) {
        case 0: r[0] = 0.0f; r[1] = 1.0f; r[2] = 0.0f; break;
        case 1: r[0] = 0.0f; r[1] = -1.0f; r[2] = 1.0f; break;
        case 2: r[0] = 2.0f; r[1] = 0.0f; r[2] = -1.0f; break;
        case 3: r[0] = r[1] = 0.0f; r[2] = g.below(2) ? static_cast<float>(g.uniform(-3, -0.01)) : static_cast<float>(g.uniform(1.01, 3)); break;
        case 7: r[0] = r[1] = 0.0f; r[2] = static_cast<float>(1 + g.below(m.n - 1 > 1 ? m.n - 2 : 1)) / static_cast<float>(m.n - 1); break;
        default:
          for (int c = 0; c < 3; ++c) r[c] = static_cast<float>(g.uniform(-4, 4));
      }
    }
    H.motion.push_back(m);
  }
  // sphere geometries: every sphere output layout, K = 1, 2, 4, 8, hard and feathered seams
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
    SphereGeo e{};
    e.g = sphereGeometry(c, 8 + g.below(1500), 8 + g.below(1500), 16 + g.below(8000), 16 + g.below(8000), 1 << (k / 6) % 4);
    e.r = rotationFromAngles(angle(), angle(), angle());
    e.seam = g.below(2) ? 0.0f : static_cast<float>(1.0 / (2.0 * g.uniform(0.01, 180) * M_PI / 180.0));
    e.both = g.below(2);
    e.barrel = barrelLayout(c.output_layout);
    const std::vector<float> t = buildSphereTables(e.g);
    e.colOffset = t.empty() ? -1 : static_cast<int>(H.tables.size());
    e.rowOffset = t.empty() ? -1 : e.colOffset + static_cast<int>(sphereTableRowOffset(e.g));
    H.tables.insert(H.tables.end(), t.begin(), t.end());
    H.sphere.push_back(e);
  }
  if (H.tables.empty()) H.tables.push_back(0.0f);
  // camera views: every model posed, mono geometries with maxLevel 0..8 and a bias
  for (int k = 0; k < 64; ++k) {
    auto pose = [&](int model, double hfov, double vfov, double dd) {
      H.cam.push_back(cameraConstants(model, static_cast<float>(dd), angle(), angle(), angle(), static_cast<float>(hfov), static_cast<float>(vfov)));
    };
    pose(kCameraPinhole, g.uniform(1, 179), g.uniform(1, 179), 0);
    pose(kCameraEquidistant, g.uniform(1, 360), g.uniform(1, 360), 0);
    pose(kCameraStereographic, g.uniform(1, 359), g.uniform(1, 359), 0);
    const double dd = g.uniform(0, 1), top = dd < 1 ? 2.0 * std::acos(-dd) * 180.0 / M_PI : 359.0;
    pose(kCameraPannini, g.uniform(1, std::min(359.0, top - 0.01)), g.uniform(1, 179), dd);
    pose(kCameraEquirect, g.uniform(1, 360), g.uniform(1, 180), 0);
  }
  for (int k = 0; k < 128; ++k) {
    FrameTransformContext c{};
    c.output_layout = LAYOUT_CUBEMAP_32;
    c.input_layout = LAYOUT_EQUIRECT;
    c.input_stereo_format = c.output_stereo_format = STEREO_FORMAT_MONO;
    c.expand_coef = c.input_expand_coef = 1.0f;
    c.width_scale_factor = c.height_scale_factor = 1.0f;
    CameraGeo e{};
    e.g = sphereGeometry(c, 7 + g.below(2000), 7 + g.below(2000), 8 + g.below(16000), 8 + g.below(8000), 1 << (k / 2) % 4);
    e.m = mipGeometry(e.g, k % 9);
    e.bias = g.below(2049) - 1024;
    e.seam = g.below(2) ? 0.0f : static_cast<float>(1.0 / (2.0 * g.uniform(0.01, 180) * M_PI / 180.0));
    e.both = g.below(2);
    H.camGeo.push_back(e);
  }
  return H;
}

}  // namespace

int main(int argc, char** argv) { return runGate<MotionGate>(argc, argv); }
