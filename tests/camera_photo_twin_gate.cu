// Twin gate of the camera views of a lens rig with photometry: the device build of the functions the call adds or splits
// (oriented_view.h: lensJacobian with the lens as an argument, cameraPhotoPoint, cameraPhotoSample) against their host
// build, the one T360B200_cameraPhotoMaps runs.  The harness, its comparison rule and its modes are tests/twin_gate.cuh's.
// Probes:
//   lensJacobian<lens>     drawn rig directions through a drawn lens of the rig (the farther one included), rays on that
//                          lens's axis (rho = 0, both signs of Z) included;
//   cameraPhotoPoint       2^24 (geometry, camera, rig, photometry, pixel) samples over seeded rig views, cameras of every
//                          model, maxLevel 0..8, lodBias, hard (both = false and true) and feathered seams.  The ledger's
//                          classes: a used lens's ray on its axis (the centre pixel of an odd-sized view looking down it),
//                          theta = thetaMax (the lens's bound set to the pixel's own theta), belt pixels (0 < w < 256), and
//                          the infinite footprint of mipLevelOf (a used lens's back axis, thetaMax = pi);
//   cameraPhotoSample<MIP> / <plain>: the same samples, quantised, in the kernel's two instantiations.
#include "twin_gate.cuh"

using namespace t360;
using namespace t360gate;

namespace {

// ---- data the probes share (host-built, copied to the device) --------------------------------------------------------
struct ChainGeo {
  SphereGeometry g;  // a rig view's geometry (mono, equirect-like input fields)
  MipGeometry m;
  int bias;
  float seam;  // seamScale (0: the hard seam)
  bool both;
};
struct GateData {
  const RectilinearCamera* cam;
  int nCam, nCamAxis;  // [0, nCamAxis): unrotated pinholes (the centre pixel of an odd view looks down +z)
  const LensRigModel* rig;
  int nRig, nRigAxis;  // [0, nRigAxis): lenses along +-z (rho = 0 reachable)
  const LensPhotoPlane* photo;
  int nPhoto;
  const ChainGeo* geo;
  int nGeo;
};

T360_HD uint32_t packLens(int level, int w, int gain) { return iw(level) | iw(w) << 8 | iw(gain) << 16; }

struct CameraPhotoGate {
  static constexpr uint64_t kSeed = 20261020ull;
  static constexpr int kOut = 11;
  enum Probe { kJacobian, kPoint, kSampleMip, kSamplePlain, kProbes };
  static constexpr ProbeInfo kInfo[kProbes] = {
      {"lensJacobian<lens>", "", 1ull << 26},
      {"cameraPhotoPoint", "lensAxis thetaMax belt infiniteFootprint", 1ull << 24},
      {"cameraPhotoSample<MIP>", "", 1ull << 24},
      {"cameraPhotoSample<plain>", "", 1ull << 24},
  };
  // bit 7 of word 4 (lens 0's level, weight and gain) of a cameraPhotoSample<MIP> element
  static constexpr Flip kFlip = {kSampleMip, kBlock / 2 + 1234, 4, 7};

  using Data = GateData;
  struct HostData {
    std::vector<RectilinearCamera> cam;
    std::vector<LensRigModel> rig;
    std::vector<LensPhotoPlane> photo;
    std::vector<ChainGeo> geo;
    int nCamAxis = 0, nRigAxis = 0;
  };
  template <int P>
  static T360_HD void probe(const Data& D, uint64_t i, Words<kOut>& w);
  static HostData makeData();
  static Data view(const HostData& H, int) {
    return GateData{H.cam.data(), static_cast<int>(H.cam.size()), H.nCamAxis, H.rig.data(), static_cast<int>(H.rig.size()), H.nRigAxis,
                    H.photo.data(), static_cast<int>(H.photo.size()), H.geo.data(), static_cast<int>(H.geo.size())};
  }
  static Data deviceData(const HostData& H, Data D, Uploads& up) {
    D.cam = up(H.cam); D.rig = up(H.rig); D.photo = up(H.photo); D.geo = up(H.geo);
    return D;
  }
};

template <int P>
T360_HD void CameraPhotoGate::probe(const GateData& D, uint64_t i, Words<kOut>& w) {
  Draw d(kSeed, P, i);
  if constexpr (P == kJacobian) {
    const bool axis = d.below(4) == 0;
    const LensRigModel& rig = D.rig[axis ? d.below(D.nRigAxis) : d.below(D.nRig)];
    const int l = rig.numLenses > 1 ? d.below(2) : 0;
    SphereVec t = drawVec(d, 1.0f);
    if (axis) t = SphereVec{d.sign(0.0f), d.sign(0.0f), d.sign(d.range(0.1f, 2.0f))};  // rho = 0 on either lens's axis
    const SphereVec rx = drawVec(d, 0.01f), ry = drawVec(d, 0.01f);
    const int inW = 16 + d.below(8000), inH = 16 + d.below(8000);
    float a[2], b[2];
    lensJacobian(rig.lens[l], lensRow(rig.lens[l].m + 6, t), t, rx, ry, inW, inH, a, b);
    w.in[0] = floatBits(t.x); w.in[1] = floatBits(t.y); w.in[2] = floatBits(t.z); w.in[3] = iw(l);
    w.out[0] = fw(a[0]); w.out[1] = fw(a[1]); w.out[2] = fw(b[0]); w.out[3] = fw(b[1]);
  } else {
    const ChainGeo& e = D.geo[d.below(D.nGeo)];
    const bool axis = d.below(4) == 0;
    const RectilinearCamera& c = D.cam[axis ? d.below(D.nCamAxis) : d.below(D.nCam)];
    LensRigModel rig = D.rig[axis ? d.below(D.nRigAxis) : d.below(D.nRig)];
    const LensPhotoPlane& ph = D.photo[d.below(D.nPhoto)];
    const bool centre = axis && d.coin() && (e.g.mapW & 1) && (e.g.mapH & 1);
    const int row = centre ? e.g.mapH / 2 : d.below(e.g.mapH), col = centre ? e.g.mapW / 2 : d.below(e.g.mapW);
    float X, Y;
    bool eye;
    cameraXY(e.g, row, col, &X, &Y, &eye);
    const SphereVec t = rotateHD(c.r, modelRay(c, X, Y));
    int edge = -1;
    if (d.below(8) == 0) {  // a lens's bound exactly at this pixel's theta
      edge = rig.numLenses > 1 ? d.below(2) : 0;
      const LensModel& L = rig.lens[edge];
      const LensHit h = lensHit(L, t, lensRow(L.m + 6, t), e.g.inW, e.g.inH);
      if (h.theta == h.theta) rig.lens[edge].thetaMax = h.theta;
    }
    const float s = rig.numLenses > 1 ? e.seam : 0.0f;
    w.in[0] = iw(row); w.in[1] = iw(col); w.in[2] = iw(c.model); w.in[3] = floatBits(s);
    bool overlap;
    int wt;
    if constexpr (P == kPoint) {
      CameraPhotoLens lens[2];
      wt = cameraPhotoPoint<true>(e.g, c, rig, e.m, e.bias, s, e.both, ph, row, col, lens, &overlap);
      for (int l = 0; l < 2; ++l) {
        w.out[5 * l] = fw(lens[l].p0[0]); w.out[5 * l + 1] = fw(lens[l].p0[1]);
        w.out[5 * l + 2] = fw(lens[l].p1[0]); w.out[5 * l + 3] = fw(lens[l].p1[1]);
        w.out[5 * l + 4] = packLens(lens[l].level, lens[l].w, lens[l].gain);
      }
#ifndef __CUDA_ARCH__
      for (int l = 0; l < rig.numLenses; ++l) {
        const LensModel& L = rig.lens[l];
        const bool used = lens[l].p0[0] == lens[l].p0[0];
        const bool onAxis = lensRow(L.m, t) == 0.0f && lensRow(L.m + 3, t) == 0.0f;
        const float Z = lensRow(L.m + 6, t);
        CLASS(0, used && onAxis);
        CLASS(1, used && l == edge && libmAtan2f(fSqrt(fAdd(fMul(lensRow(L.m, t), lensRow(L.m, t)), fMul(lensRow(L.m + 3, t), lensRow(L.m + 3, t)))), Z) ==
                                          L.thetaMax);
        CLASS(3, used && onAxis && !(Z > 0.0f) && e.m.top > 0);
      }
      CLASS(2, wt > 0 && wt < 256);
#endif
    } else {
      CameraPhotoRecords lens[2] = {};
      wt = P == kSampleMip ? cameraPhotoSample<true>(e.g, c, rig, e.m, e.bias, s, e.both, ph, row, col, lens, &overlap)
                           : cameraPhotoSample<false>(e.g, c, rig, e.m, e.bias, s, e.both, ph, row, col, lens, &overlap);
      for (int l = 0; l < 2; ++l) {
        w.out[5 * l] = iw(lens[l].rec0[0]); w.out[5 * l + 1] = iw(lens[l].rec0[1]);
        w.out[5 * l + 2] = iw(lens[l].w ? lens[l].rec1[0] : 0); w.out[5 * l + 3] = iw(lens[l].w ? lens[l].rec1[1] : 0);
        w.out[5 * l + 4] = packLens(lens[l].level, lens[l].w, lens[l].gain);
      }
    }
    w.out[10] = iw(wt) | iw(overlap) << 9 | iw(e.both) << 10;
  }
}

CameraPhotoGate::HostData CameraPhotoGate::makeData() {
  HostData H;
  HostRng g{kSeed * 7919};
  auto angle = [&] { return g.below(4) == 0 ? static_cast<float>(90 * g.below(4)) : static_cast<float>(g.uniform(-180, 180)); };
  // cameras: unrotated pinholes first (the centre pixel of an odd view looks down +z exactly), then every model posed
  for (int k = 0; k < 16; ++k) H.cam.push_back(cameraConstants(kCameraPinhole, 0.0f, 0.0f, 0.0f, 0.0f, static_cast<float>(g.uniform(1, 179)),
                                                               static_cast<float>(g.uniform(1, 179))));
  H.nCamAxis = static_cast<int>(H.cam.size());
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
  // rigs: lenses along +-z first (their axes reach rho = 0 exactly; lens 1 looks down -z), then rotated ones
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
  // geometries: a rig view's (mono), odd and even sizes, K = 1, 2, 4, 8, maxLevel 0..8 and a bias, hard and feathered seams
  for (int k = 0; k < 256; ++k) {
    FrameTransformContext c{};
    c.output_layout = LAYOUT_CUBEMAP_32;
    c.input_layout = LAYOUT_EQUIRECT;
    c.input_stereo_format = c.output_stereo_format = STEREO_FORMAT_MONO;
    c.expand_coef = c.input_expand_coef = 1.0f;
    c.width_scale_factor = c.height_scale_factor = 1.0f;
    ChainGeo e{};
    e.g = sphereGeometry(c, 7 + g.below(2000), 7 + g.below(2000), 8 + g.below(16000), 8 + g.below(8000), 1 << (k / 2) % 4);
    e.m = mipGeometry(e.g, k % 9);
    e.bias = g.below(2049) - 1024;
    e.seam = g.below(2) ? 0.0f : static_cast<float>(1.0 / (2.0 * g.uniform(0.01, 180) * M_PI / 180.0));
    e.both = g.below(2);
    H.geo.push_back(e);
  }
  return H;
}

}  // namespace

int main(int argc, char** argv) { return runGate<CameraPhotoGate>(argc, argv); }
