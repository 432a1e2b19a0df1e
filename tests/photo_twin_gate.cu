// Twin gate of the lens photometry: the device build of the float function it adds (oriented_view.h: lensGain, the
// falloff and the gain's quantisation) and of the chains that call it (lensPhotoPosition, lensPhotoPoint,
// lensPhotoSample) against their host build, the one T360B200_lensPhotoMaps runs.  The harness, its comparison rule and
// its modes are tests/twin_gate.cuh's.  Probes:
//   lensGain           lensHit<true> of drawn directions and lenses, then lensGain with drawn falloffs and gains; the
//                      ledger's classes: r = 0 (a ray on the lens axis), theta = thetaMax (the lens's bound set to the
//                      ray's own theta), V near the refusal bound (v1 = -(1 - e) / r^2, e down to 2^-20), Gq at its clamp
//                      (G >= 16), and rays the lens does not cover;
//   lensPhotoPosition  drawn rig directions, hard (both = false and true) and feathered seams;
//   lensPhotoSample<BARREL> / <plain>: 2^24 (geometry, pixel) samples each over seeded contexts, rigs and photometries.
#include "twin_gate.cuh"

using namespace t360;
using namespace t360gate;

namespace {

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

struct PhotoGate {
  static constexpr uint64_t kSeed = 20261019ull;
  static constexpr int kOut = 6;
  enum Probe { kGain, kPosition, kSampleBarrel, kSamplePlain, kProbes };
  static constexpr ProbeInfo kInfo[kProbes] = {
      {"lensGain", "r0 thetaMax nearBound clamp uncovered", 1ull << 28},
      {"lensPhotoPosition", "", 1ull << 26},
      {"lensPhotoSample<BARREL>", "", 1ull << 24},
      {"lensPhotoSample<plain>", "", 1ull << 24},
  };
  // bit 3 of word 5 (a gain) of a lensPhotoSample<plain> element
  static constexpr Flip kFlip = {kSamplePlain, kBlock / 2 + 4321, 5, 3};

  using Data = GateData;
  struct HostData {
    std::vector<LensRigModel> rig;
    std::vector<LensPhotoPlane> photo;
    std::vector<ChainGeo> geo;
    std::vector<float> tables;
    int nRigAxis = 0;
  };
  template <int P>
  static T360_HD void probe(const Data& D, uint64_t i, Words<kOut>& w);
  static HostData makeData();
  static Data view(const HostData& H, int) {
    return GateData{H.rig.data(), static_cast<int>(H.rig.size()), H.nRigAxis, H.photo.data(), static_cast<int>(H.photo.size()),
                    H.geo.data(), static_cast<int>(H.geo.size()), H.tables.data()};
  }
  static Data deviceData(const HostData& H, Data D, Uploads& up) {
    D.rig = up(H.rig); D.photo = up(H.photo); D.geo = up(H.geo); D.tables = up(H.tables);
    return D;
  }
};

template <int P>
T360_HD void PhotoGate::probe(const GateData& D, uint64_t i, Words<kOut>& w) {
  Draw d(kSeed, P, i);
  if constexpr (P == kGain) {
    const bool axis = d.below(8) == 0;
    LensModel L = D.rig[axis ? d.below(D.nRigAxis) : d.below(D.nRig)].lens[0];
    SphereVec t = axis ? SphereVec{d.sign(0.0f), d.sign(0.0f), d.range(0.1f, 2.0f)} : drawVec(d, 1.0f);
    const int edge = d.below(4);
    if (edge == 1) {  // the lens's bound exactly at this ray's theta
      const LensHitR h = lensHit<true>(L, t, lensRow(L.m + 6, t), 1000, 1000);
      if (h.theta == h.theta) L.thetaMax = h.theta;
    }
    const LensHitR h = lensHit<true>(L, t, lensRow(L.m + 6, t), 16 + d.below(8000), 16 + d.below(8000));
    float v[3] = {d.range(-0.3f, 0.1f), d.range(-0.05f, 0.05f), d.range(-0.005f, 0.005f)};
    float gain = d.coin() ? d.range(0.001f, 8.0f) : d.range(0.9f, 1.1f);
    if (edge == 2 && h.covered && h.r > 0.0f) {  // V near 0: v1 = -(1 - e) / r^2
      const float e = fDiv(1.0f, static_cast<float>(1u << d.below(21)));
      v[0] = fDiv(fSub(e, 1.0f), fMul(h.r, h.r));
      v[1] = v[2] = 0.0f;
    }
    if (edge == 3) {  // G >= 16 and around it
      gain = d.range(7.0f, 8.0f);
      v[0] = fDiv(d.range(-0.75f, -0.4f), fAdd(fMul(h.r == h.r ? h.r : 1.0f, h.r == h.r ? h.r : 1.0f), 1e-3f));
    }
    const int gq = lensGain(h, v, gain);
    w.in[0] = floatBits(t.x); w.in[1] = floatBits(t.y); w.in[2] = floatBits(v[0]); w.in[3] = floatBits(gain);
    w.out[0] = iw(gq); w.out[1] = fw(h.r); w.out[2] = fw(h.theta); w.out[3] = iw(h.covered);
    CLASS(0, h.covered && h.r == 0.0f);
    CLASS(1, h.covered && h.theta == L.thetaMax);
    CLASS(2, edge == 2 && h.covered && h.r > 0.0f && gq > 0);
    CLASS(3, gq == 65535);
    CLASS(4, !h.covered);
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

PhotoGate::HostData PhotoGate::makeData() {
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

}  // namespace

int main(int argc, char** argv) { return runGate<PhotoGate>(argc, argv); }
