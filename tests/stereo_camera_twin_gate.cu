// Twin gate of the camera views of a stereo rig and the equirect camera model: the device build of the functions the
// stereo call adds or reaches (oriented_view.h: cameraRay's equirect case, equirectRay, which the device compiles out of
// line; cameraPhotoPoint<MIP, true> and cameraPhotoSample<MIP, true>, with lensPhotoPosition<true> picking the lens by
// output eye) against their host build, the one T360B200_stereoCameraMaps runs.  The harness, its comparison rule and its
// modes are tests/twin_gate.cuh's.
// Probes:
//   cameraRay<equirect>      drawn (X, Y) through drawn equirect cameras (hfov up to 360, vfov up to 180, the exact 360 x
//                            180 window among them), X = +-1 and Y near +-1 included.  Ledger: lon = +-pi (hfov 360 at
//                            X = +-1), and lat within 0.1 degree of +-90;
//   cameraPhotoPoint<stereo> 2^24 (geometry, camera, rig, photometry, pixel) samples over seeded stereo rig views: mono, LR,
//                            TB and TB with vflip output splits at odd and even sizes, cameras of every model, maxLevel
//                            0..8, lodBias, statistics on and off.  Ledger: the columns either side of an LR eye boundary,
//                            the rows either side of a TB one, each lens's thetaMax (the lens's bound set to the pixel's
//                            own theta), the flipped eye of a TB vflip view, and the infinite footprint of mipLevelOf (the
//                            used lens's back axis, thetaMax = pi);
//   cameraPhotoSample<MIP,stereo> / <plain,stereo>: the same samples, quantised, in the kernel's two instantiations.
#include "twin_gate.cuh"

using namespace t360;
using namespace t360gate;

namespace {

// ---- data the probes share (host-built, copied to the device) --------------------------------------------------------
struct StereoGeo {
  SphereGeometry g;  // a stereo rig view's geometry: mono input fields, the output split set as the host sets it
  MipGeometry m;
  int bias;
  bool both;  // statistics on: the other lens is projected too
};
struct GateData {
  const RectilinearCamera* cam;
  int nCam, nCamAxis;  // [0, nCamAxis): unrotated pinholes (the centre pixel of an odd mono view looks down +z)
  const RectilinearCamera* eq;
  int nEq;  // equirect cameras (cameraRay<equirect>)
  const LensRigModel* rig;
  int nRig, nRigAxis;  // [0, nRigAxis): lenses along +-z (rho = 0 reachable), one of the two looking back
  const LensPhotoPlane* photo;
  int nPhoto;
  const StereoGeo* geo;
  int nGeo, nGeoMono;  // [0, nGeoMono): mono output splits with odd sides
};

T360_HD uint32_t packLens(int level, int w, int gain) { return iw(level) | iw(w) << 8 | iw(gain) << 16; }

struct StereoCameraGate {
  static constexpr uint64_t kSeed = 20261018ull;
  static constexpr int kOut = 11;
  enum Probe { kRay, kPoint, kSampleMip, kSamplePlain, kProbes };
  static constexpr ProbeInfo kInfo[kProbes] = {
      {"cameraRay<equirect>", "lonPi latPole", 1ull << 26},
      {"cameraPhotoPoint<stereo>", "eyeBoundaryCol eyeBoundaryRow thetaMax0 thetaMax1 tbVflip infiniteFootprint", 1ull << 24},
      {"cameraPhotoSample<MIP,stereo>", "", 1ull << 24},
      {"cameraPhotoSample<plain,stereo>", "", 1ull << 24},
  };
  // bit 5 of word 9 (lens 1's level, weight and gain) of a cameraPhotoSample<MIP,stereo> element
  static constexpr Flip kFlip = {kSampleMip, kBlock / 3 + 777, 9, 5};

  using Data = GateData;
  struct HostData {
    std::vector<RectilinearCamera> cam, eq;
    std::vector<LensRigModel> rig;
    std::vector<LensPhotoPlane> photo;
    std::vector<StereoGeo> geo;
    int nCamAxis = 0, nRigAxis = 0, nGeoMono = 0;
  };
  template <int P>
  static T360_HD void probe(const Data& D, uint64_t i, Words<kOut>& w);
  static HostData makeData();
  static Data view(const HostData& H, int) {
    return GateData{H.cam.data(), static_cast<int>(H.cam.size()), H.nCamAxis, H.eq.data(), static_cast<int>(H.eq.size()), H.rig.data(),
                    static_cast<int>(H.rig.size()), H.nRigAxis, H.photo.data(), static_cast<int>(H.photo.size()), H.geo.data(),
                    static_cast<int>(H.geo.size()), H.nGeoMono};
  }
  static Data deviceData(const HostData& H, Data D, Uploads& up) {
    D.cam = up(H.cam); D.eq = up(H.eq); D.rig = up(H.rig); D.photo = up(H.photo); D.geo = up(H.geo);
    return D;
  }
};

template <int P>
T360_HD void StereoCameraGate::probe(const GateData& D, uint64_t i, Words<kOut>& w) {
  Draw d(kSeed, P, i);
  if constexpr (P == kRay) {
    const RectilinearCamera& c = D.eq[d.below(D.nEq)];
    const float X = d.below(4) == 0 ? d.sign(1.0f) : d.range(-1.0f, 1.0f);
    const float Y = d.below(4) == 0 ? d.sign(d.range(0.998f, 1.0f)) : d.range(-1.0f, 1.0f);
    const SphereVec q = cameraRay(c, X, Y);
    w.in[0] = floatBits(X); w.in[1] = floatBits(Y); w.in[2] = floatBits(c.cx); w.in[3] = floatBits(c.cy);
    w.out[0] = fw(q.x); w.out[1] = fw(q.y); w.out[2] = fw(q.z);
    CLASS(0, (X == 1.0f || X == -1.0f) && c.cx == 3.14159274f);
    CLASS(1, fMul(Y, c.cy) > 1.56905f || fMul(Y, c.cy) < -1.56905f);  // within 0.1 degree of a pole
  } else {
    const bool axis = d.below(4) == 0;
    const StereoGeo& e = D.geo[axis ? d.below(D.nGeoMono) : d.below(D.nGeo)];
    const RectilinearCamera& c = D.cam[axis ? d.below(D.nCamAxis) : d.below(D.nCam)];
    LensRigModel rig = D.rig[axis ? d.below(D.nRigAxis) : d.below(D.nRig)];
    const LensPhotoPlane& ph = D.photo[d.below(D.nPhoto)];
    const bool centre = axis && d.coin();
    int row = centre ? e.g.mapH / 2 : d.below(e.g.mapH), col = centre ? e.g.mapW / 2 : d.below(e.g.mapW);
    if (!centre && d.below(8) == 0) {  // either side of the eye boundary
      if (e.g.splitLR) col = e.g.mapW / 2 - d.below(2);
      if (e.g.splitTB) row = e.g.mapH / 2 - d.below(2);
    }
    float X, Y;
    bool eye;
    cameraXY(e.g, row, col, &X, &Y, &eye);
    const SphereVec t = rotateHD(c.r, modelRay(c, X, Y));
    int edge = -1;
    if (d.below(8) == 0) {  // a lens's bound exactly at this pixel's theta
      edge = d.below(2);
      const LensModel& L = rig.lens[edge];
      const LensHit h = lensHit(L, t, lensRow(L.m + 6, t), e.g.inW, e.g.inH);
      if (h.theta == h.theta) rig.lens[edge].thetaMax = h.theta;
    }
    const int kind = e.g.splitLR ? 1 : (e.g.splitTB ? (e.g.vflip ? 3 : 2) : 0);
    w.in[0] = iw(row); w.in[1] = iw(col); w.in[2] = iw(c.model); w.in[3] = iw(kind);
    bool overlap;
    int wt;
    if constexpr (P == kPoint) {
      CameraPhotoLens lens[2];
      wt = cameraPhotoPoint<true, true>(e.g, c, rig, e.m, e.bias, 0.0f, e.both, ph, row, col, lens, &overlap);
      for (int l = 0; l < 2; ++l) {
        w.out[5 * l] = fw(lens[l].p0[0]); w.out[5 * l + 1] = fw(lens[l].p0[1]);
        w.out[5 * l + 2] = fw(lens[l].p1[0]); w.out[5 * l + 3] = fw(lens[l].p1[1]);
        w.out[5 * l + 4] = packLens(lens[l].level, lens[l].w, lens[l].gain);
      }
#ifndef __CUDA_ARCH__
      CLASS(0, e.g.splitLR && (col == e.g.mapW / 2 || col == e.g.mapW / 2 - 1));
      CLASS(1, e.g.splitTB && (row == e.g.mapH / 2 || row == e.g.mapH / 2 - 1));
      for (int l = 0; l < 2; ++l) {
        const LensModel& L = rig.lens[l];
        const bool used = lens[l].p0[0] == lens[l].p0[0];
        const float lx = lensRow(L.m, t), ly = lensRow(L.m + 3, t), Z = lensRow(L.m + 6, t);
        CLASS(2 + l, used && l == edge && libmAtan2f(fSqrt(fAdd(fMul(lx, lx), fMul(ly, ly))), Z) == L.thetaMax);
        CLASS(5, used && lx == 0.0f && ly == 0.0f && !(Z > 0.0f) && e.m.top > 0);
      }
      CLASS(4, e.g.splitTB && e.g.vflip && eye);
#endif
    } else {
      CameraPhotoRecords lens[2] = {};
      wt = P == kSampleMip ? cameraPhotoSample<true, true>(e.g, c, rig, e.m, e.bias, 0.0f, e.both, ph, row, col, lens, &overlap)
                           : cameraPhotoSample<false, true>(e.g, c, rig, e.m, e.bias, 0.0f, e.both, ph, row, col, lens, &overlap);
      for (int l = 0; l < 2; ++l) {
        w.out[5 * l] = iw(lens[l].rec0[0]); w.out[5 * l + 1] = iw(lens[l].rec0[1]);
        w.out[5 * l + 2] = iw(lens[l].w ? lens[l].rec1[0] : 0); w.out[5 * l + 3] = iw(lens[l].w ? lens[l].rec1[1] : 0);
        w.out[5 * l + 4] = packLens(lens[l].level, lens[l].w, lens[l].gain);
      }
    }
    w.out[10] = iw(wt) | iw(overlap) << 9 | iw(e.both) << 10 | iw(eye) << 11;
  }
}

StereoCameraGate::HostData StereoCameraGate::makeData() {
  HostData H;
  HostRng g{kSeed * 7919};
  auto angle = [&] { return g.below(4) == 0 ? static_cast<float>(90 * g.below(4)) : static_cast<float>(g.uniform(-180, 180)); };
  auto small = [&] { return static_cast<float>(g.uniform(-25, 25)); };
  // cameras: unrotated pinholes first (the centre pixel of an odd mono view looks down +z exactly), then every model posed
  // about the rig's forward axis
  for (int k = 0; k < 16; ++k) H.cam.push_back(cameraConstants(kCameraPinhole, 0.0f, 0.0f, 0.0f, 0.0f, static_cast<float>(g.uniform(1, 179)),
                                                               static_cast<float>(g.uniform(1, 179))));
  H.nCamAxis = static_cast<int>(H.cam.size());
  auto pose = [&](int model, double hfov, double vfov, double d) {
    const bool wild = g.below(4) == 0;
    H.cam.push_back(cameraConstants(model, static_cast<float>(d), wild ? angle() : small(), wild ? angle() : small(), wild ? angle() : small(),
                                    static_cast<float>(hfov), static_cast<float>(vfov)));
  };
  for (int k = 0; k < 128; ++k) {
    pose(kCameraPinhole, g.uniform(1, 179), g.uniform(1, 179), 0);
    pose(kCameraEquidistant, g.uniform(1, 360), g.uniform(1, 360), 0);
    pose(kCameraStereographic, g.uniform(1, 359), g.uniform(1, 359), 0);
    const double d = g.uniform(0, 1), top = d < 1 ? 2.0 * std::acos(-d) * 180.0 / M_PI : 359.0;
    pose(kCameraPannini, g.uniform(1, std::min(359.0, top - 0.01)), g.uniform(1, 179), d);
    if (k % 4 == 0) pose(kCameraEquirect, 180.0, 180.0, 0);
    else pose(kCameraEquirect, g.uniform(1, 360), g.uniform(1, 180), 0);
  }
  // equirect cameras of the ray probe: the exact 360 x 180 and 180 x 180 windows, then drawn fields
  for (int k = 0; k < 64; ++k) {
    const double h = k % 4 == 0 ? 360.0 : (k % 4 == 1 ? 180.0 : g.uniform(1, 360)), v = k % 4 < 2 ? 180.0 : g.uniform(1, 180);
    H.eq.push_back(cameraConstants(kCameraEquirect, 0.0f, angle(), angle(), angle(), static_cast<float>(h), static_cast<float>(v)));
  }
  // rigs: lenses along +-z first (one forward, one back, either way round: a used lens's back axis is reachable in either
  // eye), then stereo pairs: two forward lenses with small rotations, their circles on either half
  auto lens = [&](int axisAligned /* 0: rotated, 1: +z, -1: -z */, bool forward) {
    LensModel L{};
    if (axisAligned) {
      const float s = static_cast<float>(axisAligned);
      const float m[9] = {s, 0, 0, 0, -1.0f, 0, 0, 0, s};
      std::memcpy(L.m, m, sizeof(m));
    } else {
      const Rotation r = forward ? rotationFromAngles(small() / 8, small() / 8, small() / 8) : rotationFromAngles(angle(), angle(), angle());
      const float m[9] = {r.xx, r.xy, r.xz, r.yx, r.yy, r.yz, r.zx, r.zy, r.zz};
      std::memcpy(L.m, m, sizeof(m));
    }
    L.ax = static_cast<float>(g.uniform(0.1, 0.3));
    L.bx = static_cast<float>(g.uniform(0.2, 0.8));
    L.ay = static_cast<float>(g.uniform(0.2, 0.5));
    L.by = static_cast<float>(g.uniform(0.3, 0.7));
    for (float& k : L.k) k = static_cast<float>(g.uniform(-0.05, 0.05));
    L.thetaMax = g.below(3) == 0 ? static_cast<float>(M_PI) : static_cast<float>(g.uniform(0.5, M_PI));
    return L;
  };
  for (int k = 0; k < 64; ++k) {
    LensRigModel rig{};
    rig.numLenses = 2;
    rig.lens[0] = lens(k % 2 ? -1 : 1, true);
    rig.lens[1] = lens(k % 2 ? 1 : -1, true);
    H.rig.push_back(rig);
  }
  H.nRigAxis = static_cast<int>(H.rig.size());
  for (int k = 0; k < 64; ++k) {
    LensRigModel rig{};
    rig.numLenses = 2;
    rig.lens[0] = lens(0, k % 4 != 0);
    rig.lens[1] = lens(0, k % 4 != 0);
    H.rig.push_back(rig);
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
  // geometries: mono views with odd sides first (their centre pixel), then mono, LR, TB and TB with vflip at odd and even
  // sizes, K = 1, 2, 4, 8, maxLevel 0..8 and a bias, statistics on and off
  auto geo = [&](int k, int split, bool oddSides) {
    FrameTransformContext c{};
    c.output_layout = LAYOUT_CUBEMAP_32;
    c.input_layout = LAYOUT_EQUIRECT;
    c.input_stereo_format = c.output_stereo_format = STEREO_FORMAT_MONO;
    c.expand_coef = c.input_expand_coef = 1.0f;
    c.width_scale_factor = c.height_scale_factor = 1.0f;
    c.vflip = split == 3;
    int mapW = 8 + g.below(2000), mapH = 8 + g.below(2000);
    if (oddSides) mapW |= 1, mapH |= 1;
    StereoGeo e{};
    e.g = sphereGeometry(c, mapW, mapH, 8 + g.below(16000), 8 + g.below(8000), 1 << (k / 2) % 4);
    e.g.splitLR = split == 1;  // (as viewGeometry sets them: the output split alone, no input re-pack)
    e.g.splitTB = split >= 2;
    e.m = mipGeometry(e.g, k % 9);
    e.bias = g.below(2049) - 1024;
    e.both = g.below(2);
    H.geo.push_back(e);
  };
  for (int k = 0; k < 64; ++k) geo(k, 0, true);
  H.nGeoMono = static_cast<int>(H.geo.size());
  for (int k = 0; k < 256; ++k) geo(k, k % 4, g.below(2));
  return H;
}

}  // namespace

int main(int argc, char** argv) { return runGate<StereoCameraGate>(argc, argv); }
