// Host geometry planner: output pixel -> source coordinate, for every layout pair of the hot path.
//
// Behavioural spec: reference VideoFrameTransform.cpp:893-1316 (transformPos), :863-891
// (transformInputPos), :796-861 (transformCubeFacePos), :53-75 (intersectSphereOffset), :101-123
// (normalize_equirectangular) and the map loop :534-556.  Parity with the reference is a float32
// rounding-reproduction problem (SURVEY.md 7 hard part 1): every expression below is typed so that it
// rounds where the reference's expression rounds -- float where the reference is float, double where
// the reference mixes in M_PI or a double literal -- and this file must be compiled WITHOUT fused
// multiply-add contraction (-ffp-contract=off, no -march=native).  tests/test_host_plan.py checks the
// result bit-for-bit against the compiled reference for every layout.
//
// Organisation (differs from the reference's single switch-heavy function): a Projector is built once
// per plane from the context; it precomputes the stream constants (rotation coefficients, off-centre
// vector, stereo modes) and exposes the pipeline as small stages:
//   eye split -> surface point on the unit cube / sphere -> off-centre warp -> rotation -> input lookup
//   -> eye re-pack.
#include <cmath>
#include <cstdio>
#include <algorithm>
#include <thread>
#include <vector>

#include "flat_view.h"
#include "host_plan.h"
#include "oriented_view.h"

namespace t360 {
namespace {

constexpr double kTiny = 1e-9;  // reference kEpsilon (cpp:33)

struct Vec3 {
  float x, y, z;
};

// Corner + edge directions of each cube face, in the 3x2 arrangement (cpp:38-49, 1153-1184) and in
// the 2x3 off-centre arrangement (cpp:1119-1151).  Components are exactly 0 or +-1 / +-0.5.
struct FaceFrame {
  Vec3 origin, du, dv;
};
constexpr Vec3 C000{-0.5f, -0.5f, -0.5f}, C100{0.5f, -0.5f, -0.5f}, C110{0.5f, 0.5f, -0.5f}, C001{-0.5f, -0.5f, 0.5f},
    C101{0.5f, -0.5f, 0.5f}, C011{-0.5f, 0.5f, 0.5f};
constexpr Vec3 XP{1, 0, 0}, YP{0, 1, 0}, ZP{0, 0, 1}, XN{-1, 0, 0}, ZN{0, 0, -1};
constexpr FaceFrame kFrames32[6] = {
    {C101, ZN, YP},  // RIGHT
    {C000, ZP, YP},  // LEFT
    {C011, XP, ZN},  // TOP
    {C000, XP, ZP},  // BOTTOM
    {C001, XP, YP},  // FRONT
    {C100, XN, YP},  // BACK
};
constexpr FaceFrame kFrames23[6] = {
    {C001, YP, ZN}, {C110, XN, ZP}, {C101, YP, XN}, {C100, XN, YP}, {C100, YP, ZP}, {C101, XN, ZN},
};

class Projector {
 public:
  Projector(const FrameTransformContext& c, float inputPixelWidth) : c_(c), inPixW_(inputPixelWidth) {
    // Euler angles -> rotation coefficients (cpp:1233-1244; oriented_view.h, shared with the per-frame orientation path)
    const Rotation r = rotationFromAngles(c.fixed_yaw, c.fixed_pitch, c.fixed_roll);
    rxx_ = r.xx; rxy_ = r.xy; rxz_ = r.xz;
    ryx_ = r.yx; ryy_ = r.yy; ryz_ = r.yz;
    rzx_ = r.zx; rzy_ = r.zy; rzz_ = r.zz;
    offCentre_ = std::abs(c.fixed_cube_offcenter_x) > kTiny || std::abs(c.fixed_cube_offcenter_y) > kTiny ||
                 std::abs(c.fixed_cube_offcenter_z) > kTiny;
    barrel_ = c.output_layout == LAYOUT_BARREL || c.output_layout == LAYOUT_BARREL_SPLIT;
  }

  bool valid() const {
    switch (c_.output_layout) {
      case LAYOUT_CUBEMAP_32: case LAYOUT_CUBEMAP_23_OFFCENTER: case LAYOUT_FLAT_FIXED: case LAYOUT_EQUIRECT:
      case LAYOUT_BARREL: case LAYOUT_BARREL_SPLIT: case LAYOUT_EAC_32: return true;
      default: return false;
    }
  }

  // (x, y) in [0,1)^2 of the output plane -> (u, v) in [0,1]^2 of the input plane; (-1, 0) = unmapped.
  void project(float x, float y, float* u, float* v) const {
    const bool secondEye = splitOutputEyes(x, y);
    bool mapped = true;
    if (c_.output_layout == LAYOUT_FLAT_FIXED) {
      flatWindow(x, y, u, v);
    } else {
      y = 1.0f - y;  // image rows grow downwards, the cube's v axis upwards (cpp:936-938)
      Vec3 q;
      mapped = surfacePoint(x, y, q);
      if (mapped) {
        if (offCentre_) warpOffCentre(q);
        Vec3 t;
        t.x = q.x * rxx_ - q.y * rxy_ + q.z * rxz_;
        t.y = q.x * ryx_ - q.y * ryy_ + q.z * ryz_;
        t.z = q.x * rzx_ - q.y * rzy_ + q.z * rzz_;
        t.y = -t.y;
        lookupInput(t, u, v);
      }
    }
    if (!mapped) {
      *u = -1;
      *v = 0;
      return;
    }
    // second eye lives in the other half of a stacked / side-by-side input (cpp:1278-1300)
    if (c_.input_stereo_format == STEREO_FORMAT_TB) *v = packEye(*v, secondEye);
    else if (c_.input_stereo_format == STEREO_FORMAT_LR) *u = packEye(*u, secondEye);
  }

 private:
  // cpp:903-931: a stereo OUTPUT holds two complete projections; fold to one and remember which.
  bool splitOutputEyes(float& x, float& y) const {
    if (c_.input_stereo_format == STEREO_FORMAT_MONO) return false;
    if (c_.output_stereo_format == STEREO_FORMAT_LR) return splitEye(x, false);
    if (c_.output_stereo_format == STEREO_FORMAT_TB) return splitEye(y, c_.vflip != 0);
    return false;
  }

  // cpp:1265-1271, folded over a pole / wrapped around the seam (cpp:101-123): flat_view.h, shared with the per-view kernel
  void flatWindow(float x, float y, float* u, float* v) const {
    const FlatView view{c_.fixed_yaw, c_.fixed_pitch, c_.fixed_hfov, c_.fixed_vfov};
    bool fold;
    *v = flatLat(view, y, &fold);
    *u = flatLon(view, x, fold);
  }

  static Vec3 onSphere(float yaw, float pitch) {  // cpp:1095-1101 (float trig)
    const float sy = std::sin(yaw), sp = std::sin(pitch), cy = std::cos(yaw), cp = std::cos(pitch);
    return Vec3{sy * cp, sp, cy * cp};
  }

  Vec3 onCube(const FaceFrame* frames, int face, float fx, float fy) const {
    fx = (fx - 0.5f) * c_.expand_coef + 0.5f;  // cpp:1115-1116
    fy = (fy - 0.5f) * c_.expand_coef + 0.5f;
    const FaceFrame& f = frames[face];
    return Vec3{f.origin.x + f.du.x * fx + f.dv.x * fy, f.origin.y + f.du.y * fx + f.dv.y * fy,
                f.origin.z + f.du.z * fx + f.dv.z * fy};  // cpp:1187-1189
  }

  // Where the output pixel sits on the unit cube (or unit sphere); false = barrel dead zone.
  bool surfacePoint(float x, float y, Vec3& q) const {
    const float e = c_.expand_coef;
    switch (c_.output_layout) {
      case LAYOUT_CUBEMAP_32:
      case LAYOUT_EAC_32: {  // cpp:943-950, 1069-1078
        // (x == 1 happens: the centre column of a side-by-side stereo output of odd width folds to exactly 1.  The
        // reference then switches on a face number past BACK and uses an uninitialised face basis; here, as in
        // oracle/t360_oracle.c, such a pixel takes the last face's basis -- DESIGN.md 7.)
        const int row = static_cast<int>(y * 2), col = static_cast<int>(x * 3);
        float fx = x * 3.0f - col, fy = y * 2.0f - row;
        if (c_.output_layout == LAYOUT_EAC_32) { fx = equiAngular(fx); fy = equiAngular(fy); }  // (tan in double: oriented_view.h)
        q = onCube(kFrames32, std::min(std::max(col + (1 - row) * 3, 0), 5), fx, fy);
        return true;
      }
      case LAYOUT_CUBEMAP_23_OFFCENTER: {  // cpp:951-958
        const int row = static_cast<int>(y * 3), col = static_cast<int>(x * 2);
        q = onCube(kFrames23, std::min(std::max(col + (2 - row) * 2, 0), 5), x * 2.0f - col, y * 3.0f - row);  // see above
        return true;
      }
      case LAYOUT_EQUIRECT:  // cpp:965-969
        q = onSphere(equirectYaw(x), equirectPitch(y));
        return true;
      case LAYOUT_BARREL: {  // cpp:970-982
        if (x <= 0.8f) {  // (angles: oriented_view.h, shared with the per-frame pose path)
          q = onSphere(barrelYaw(x, e), barrelPitch(y, e));
          return true;
        }
        const int half = static_cast<int>(y * 2);
        return capDisc(half == 1 ? TOP : BOTTOM, x * 5.0f - 4.0f, y * 2.0f - half, q);
      }
      case LAYOUT_BARREL_SPLIT: {  // cpp:983-1068
        if (3.0f * x <= 2.0f) {
          const int half = static_cast<int>(y * 2);
          q = onSphere(barrelSplitYaw(x, half, e), barrelSplitPitch(y, half, e));
          return true;
        }
        const int quarter = static_cast<int>(y * 4);
        float fx = x * 3.0f - 2.0f, fy = y;
        switch (quarter) {
          case 0: fy = fy * 2.0f; fx = 1.0f - fx; fy = (0.5f - fy) * e; break;
          case 1: fy = fy * 2.0f; fx = 1.0f - fx; fy = 1.0f - e * (fy - 0.5f); break;
          case 2: fy = fy * 2.0f - 0.5f; fy = 1.0f - e * (1.0f - fy); break;
          case 3: fy = fy * 2.0f - 1.5f; fy = fy * e; break;
          default: break;
        }
        return capDisc((quarter == 1 || quarter == 3) ? TOP : BOTTOM, fx, fy, q);
      }
      default:
        return false;
    }
  }

  // barrel end caps are discs inscribed in a cube face (cpp:1106-1113)
  bool capDisc(int face, float fx, float fy, Vec3& q) const {
    const float r2 = (fx - 0.5f) * (fx - 0.5f) + (fy - 0.5f) * (fy - 0.5f);
    if (r2 > 0.25f * c_.expand_coef * c_.expand_coef) return false;
    q = onCube(kFrames32, face, fx, fy);
    return true;
  }

  // distance along unit ray d from the displaced eye to the unit sphere (cpp:53-75)
  static float rayToSphere(float dx, float dy, float dz, float ox, float oy, float oz) {
    const float along = dx * -ox + dy * -oy + dz * -oz;
    const float off2 = ox * ox + oy * oy + oz * oz;
    float disc = static_cast<float>(along * along - off2 + 1.0);
    if (disc <= 0.0f) return 0.0f;
    disc = std::sqrt(disc);
    if (disc < along) return 0.0f;
    return disc - along;
  }

  void warpOffCentre(Vec3& q) const {  // cpp:1192-1230
    const float ox = c_.fixed_cube_offcenter_x, oy = c_.fixed_cube_offcenter_y, oz = c_.fixed_cube_offcenter_z;
    float n = std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z);
    q.x = q.x / n; q.y = q.y / n; q.z = q.z / n;
    if (c_.is_horizontal_offset) {
      n = std::sqrt(q.x * q.x + q.z * q.z);
      q.x = q.x / n; q.y = q.y / n; q.z = q.z / n;
      const float t = rayToSphere(q.x, 0, q.z, ox, 0, oz);
      if (t > 0.0f) { q.x = q.x * t - ox; q.z = q.z * t - oz; }
    } else {
      const float t = rayToSphere(q.x, q.y, q.z, ox, oy, oz);
      if (t > 0.0f) { q.x = q.x * t - ox; q.y = q.y * t - oy; q.z = q.z * t - oz; }
    }
  }

  void lookupInput(const Vec3& t, float* u, float* v) const {  // cpp:863-891
    const float n = std::sqrt(t.x * t.x + t.y * t.y + t.z * t.z);
    if (c_.input_layout == LAYOUT_CUBEMAP_32) {
      cubeInput(t.x / n, t.y / n, t.z / n, u, v);
      return;
    }
    const float lon = -atan2f(-t.x / n, t.z / n);
    float uu = static_cast<float>(lon / (M_PI * 2.0f) + 0.5f);
    if (barrel_) {  // keep clear of ffmpeg's right-edge padding (cpp:881-886)
      uu = std::min(uu, 1.0f - inPixW_ * 0.5f);
      uu = std::max(uu, inPixW_ * 0.5f);
    }
    *u = uu;
    *v = static_cast<float>(asinf(-t.y / n) / M_PI + 0.5f);
  }

  // unit direction -> 3x2 cubemap INPUT (cpp:796-861).  Faces are tried in the reference's order:
  // -z, +z, -x, +x, -y, +y; the first whose gnomonic coordinates fall inside [-1,1]^2 wins.
  void cubeInput(float tx, float ty, float tz, float* u, float* v) const {
    struct Probe { float major, a, b; bool neg; int col; int row; int su, sv; };
    const float e = c_.input_expand_coef;
    // (column centre, row centre) of each input face in sixths / quarters, and the sign of each axis
    const Probe probes[6] = {
        {tz, tx, ty, true, 5, 3, +1, +1},  {tz, tx, ty, false, 3, 3, +1, -1}, {tx, tz, ty, true, 3, 1, -1, +1},
        {tx, tz, ty, false, 1, 1, -1, -1}, {ty, tx, tz, true, 1, 3, -1, +1},  {ty, tx, tz, false, 5, 1, +1, +1},
    };
    for (const Probe& p : probes) {
      if (p.neg ? !(p.major <= -0.5f) : !(p.major >= 0.5f)) continue;
      const float gx = p.a / p.major, gy = p.b / p.major;
      if (gx >= -1.0 && gx <= 1.0 && gy >= -1.0 && gy <= 1.0) {
        const float sx = gx / e, sy = gy / e;
        *u = (p.su > 0 ? static_cast<float>(p.col) + sx : static_cast<float>(p.col) - sx) / 6.0f;
        *v = (p.sv > 0 ? static_cast<float>(p.row) + sy : static_cast<float>(p.row) - sy) / 4.0f;
        return;
      }
    }
    *u = -1.0f;
    *v = 0.0f;
  }

  FrameTransformContext c_;
  float inPixW_;
  float rxx_, rxy_, rxz_, ryx_, ryy_, ryz_, rzx_, rzy_, rzz_;
  bool offCentre_ = false, barrel_ = false;
};

}  // namespace

bool projectPoint(const FrameTransformContext& ctx, float x, float y, float inputPixelWidth, float* outX, float* outY) {
  Projector p(ctx, inputPixelWidth);
  if (!p.valid()) return false;
  p.project(x, y, outX, outY);
  return true;
}

bool buildWarpMap(HostPlan& plan) {
  float inPixW = 1.0f / plan.inW;  // cpp:528-531
  if (plan.ctx.input_stereo_format == STEREO_FORMAT_LR) inPixW *= 2;
  const Projector proj(plan.ctx, inPixW);
  if (!proj.valid()) {
    std::printf("Invalid layout type %d.\n", static_cast<int>(plan.ctx.output_layout));
    return false;
  }
  const int W = plan.mapW, H = plan.mapH, inW = plan.inW, inH = plan.inH;
  plan.map.resize(static_cast<size_t>(W) * H * 2);
  float* out = plan.map.data();
  auto rows = [&](int r0, int r1) {
    for (int i = r0; i < r1; ++i) {
      const float y = pixelCentre(i, H);  // cpp:537
      float* row = out + static_cast<size_t>(i) * W * 2;
      for (int j = 0; j < W; ++j) {
        const float x = pixelCentre(j, W);  // cpp:538
        float u, v;
        proj.project(x, y, &u, &v);
        row[2 * j] = toPixel(u, inW);  // pixel centres sit at integers for the sampler (cpp:544-545)
        row[2 * j + 1] = toPixel(v, inH);
      }
    }
  };
  unsigned nt = std::thread::hardware_concurrency();
  if (nt == 0) nt = 1;
  if (nt > 32) nt = 32;
  if (static_cast<size_t>(W) * H < (1u << 16)) nt = 1;
  std::vector<std::thread> pool;
  const int chunk = (H + static_cast<int>(nt) - 1) / static_cast<int>(nt);
  for (unsigned t = 1; t < nt; ++t) {
    const int r0 = static_cast<int>(t) * chunk, r1 = std::min(H, r0 + chunk);
    if (r0 < r1) pool.emplace_back(rows, r0, r1);
  }
  rows(0, std::min(H, chunk));
  for (auto& th : pool) th.join();
  return true;
}

}  // namespace t360
