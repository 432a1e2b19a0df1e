// Sphere-output position chain with the orientation as a parameter: one definition for the host and the per-frame
// orientation gather kernel (oriented_gather.cu).
//
// For output pixel (i, j) of a CUBEMAP_32, CUBEMAP_23_OFFCENTER, EAC_32 or EQUIRECT map, the planner (geometry.cpp,
// Projector::project) computes: pixel centre -> output eye split -> point on the unit cube / sphere -> off-centre warp ->
// rotation by yaw / pitch / roll -> input lookup (EQUIRECT: atan2f, asinf; CUBEMAP_32: gnomonic face coordinates) -> input
// eye re-pack -> u * inW - 0.5f, v * inH - 0.5f -> cv::remap's 1/32-pixel quantisation.  Only the rotation depends on
// the orientation.  What remains of libm is reproduced or tabulated so the device gets the planner's bits:
//   - the EAC warp (double tan) depends on the column only for x and on the row only for y, and EQUIRECT's sin / cos of
//     yaw / pitch (float sinf / cosf, FMA ifuncs on the host) on the column / the row: per-plan host tables
//     (buildSphereTables, from the planner's own expressions: equiAngular, equirectYaw, equirectPitch below);
//   - the rotation coefficients (double sin / cos of the angles, stored as float): computed on the host per frame by
//     rotationFromAngles, which Projector's constructor calls too;
//   - sqrtf, atan2f, asinf: __fsqrt_rn and the libm ports (libm_ports.h); the double steps of rayToSphere and of the
//     equirectangular lookup: explicit __d*_rn and __double2float_rn.
// As in flat_view.h, every float operation on the device is an explicit _rn intrinsic and the host code is compiled with
// -ffp-contract=off.
#pragma once

#include <cmath>
#include <cstdint>
#include <vector>

#include "Transform360/VideoFrameTransformHelper.h"
#include "flat_view.h"
#include "libm_ports.h"

namespace t360 {

struct Orientation {
  float yaw, pitch, roll;  // degrees, as FrameTransformContext::fixed_*
};

// q' = (q.x * xx - q.y * xy + q.z * xz, ...): the planner's rotation (reference cpp:1233-1244)
struct Rotation {
  float xx, xy, xz, yx, yy, yz, zx, zy, zz;
};

// Euler angles converted in double and stored as float, the coefficient groups parenthesised as the reference has them
// (cpp:1233-1244).  Host only: the device receives the result.
inline Rotation rotationFromAngles(float yaw, float pitch, float roll) {
  const float s1 = static_cast<float>(std::sin(yaw * M_PI / 180.0f));
  const float s2 = static_cast<float>(std::sin(pitch * M_PI / 180.0f));
  const float s3 = static_cast<float>(std::sin(roll * M_PI / 180.0f));
  const float c1 = static_cast<float>(std::cos(yaw * M_PI / 180.0f));
  const float c2 = static_cast<float>(std::cos(pitch * M_PI / 180.0f));
  const float c3 = static_cast<float>(std::cos(roll * M_PI / 180.0f));
  Rotation r;
  r.xx = c1 * c3 + s1 * s2 * s3;  r.xy = c3 * s1 * s2 - c1 * s3;  r.xz = c2 * s1;
  r.yx = c2 * s3;                 r.yy = c2 * c3;                 r.yz = -s2;
  r.zx = c1 * s2 * s3 - c3 * s1;  r.zy = c1 * c3 * s2 + s1 * s3;  r.zz = c1 * c2;
  return r;
}

// The view-independent libm steps of the planner (host only)
inline float equiAngular(float t) { return static_cast<float>(std::tan((t - 0.5f) * M_PI * 0.5f) * 0.5f + 0.5f); }  // cpp:1074-1075
inline float equirectYaw(float x) { return static_cast<float>((2.0f * x - 1.0f) * M_PI); }                            // cpp:965-969
inline float equirectPitch(float y) { return static_cast<float>((y - 0.5f) * M_PI); }

// Everything the chain needs besides the orientation and the tables.
struct SphereGeometry {
  int mapW, mapH, inW, inH;
  int kernelSize;            // 1 (nearest), 2, 4, 8
  int outputLayout;          // LAYOUT_CUBEMAP_32, LAYOUT_CUBEMAP_23_OFFCENTER, LAYOUT_EAC_32, LAYOUT_EQUIRECT
  bool cubeInput;            // input_layout CUBEMAP_32 (else EQUIRECT)
  bool splitLR, splitTB;     // the output holds two eyes side by side / stacked (only when the input is stereo)
  bool vflip;
  bool packLR, packTB;       // the input holds two eyes side by side / stacked
  bool offCentre, horizontalOffset;
  float expand, inputExpand;  // expand_coef, input_expand_coef
  float ox, oy, oz;           // fixed_cube_offcenter_*
};

// Per-plan tables (buildSphereTables), [mapW] or [2 mapW] column entries followed by [mapH] or [2 mapH] row entries:
// EAC_32: the warped face coordinate of the column / the row; EQUIRECT: sin, cos of the column's yaw / the row's pitch.
// Other layouts need none.
inline size_t sphereTableRowOffset(const SphereGeometry& g) {
  return g.outputLayout == LAYOUT_EQUIRECT ? 2 * static_cast<size_t>(g.mapW) : g.outputLayout == LAYOUT_EAC_32 ? g.mapW : 0;
}

// The coordinate of column j / row i after the output eye split; the row already flipped upwards (cpp:936-938).
T360_HD float sphereColumnX(const SphereGeometry& g, int j) {
  float x = pixelCentre(j, g.mapW);
  if (g.splitLR) splitEye(x, false);
  return x;
}
T360_HD float sphereRowY(const SphereGeometry& g, int i) {
  float y = pixelCentre(i, g.mapH);
  if (g.splitTB) splitEye(y, g.vflip);
  return fSub(1.0f, y);
}

inline std::vector<float> buildSphereTables(const SphereGeometry& g) {
  std::vector<float> t;
  if (g.outputLayout == LAYOUT_EAC_32) {
    t.resize(static_cast<size_t>(g.mapW) + g.mapH);
    for (int j = 0; j < g.mapW; ++j) {
      const float x = sphereColumnX(g, j);
      t[j] = equiAngular(x * 3.0f - static_cast<int>(x * 3));
    }
    for (int i = 0; i < g.mapH; ++i) {
      const float y = sphereRowY(g, i);
      t[g.mapW + i] = equiAngular(y * 2.0f - static_cast<int>(y * 2));
    }
  } else if (g.outputLayout == LAYOUT_EQUIRECT) {
    t.resize(2 * (static_cast<size_t>(g.mapW) + g.mapH));
    for (int j = 0; j < g.mapW; ++j) {
      const float a = equirectYaw(sphereColumnX(g, j));
      t[2 * j] = std::sin(a);
      t[2 * j + 1] = std::cos(a);
    }
    for (int i = 0; i < g.mapH; ++i) {
      const float a = equirectPitch(sphereRowY(g, i));
      t[2 * g.mapW + 2 * i] = std::sin(a);
      t[2 * g.mapW + 2 * i + 1] = std::cos(a);
    }
  }
  return t;
}

struct SphereVec {
  float x, y, z;
};

// Corner + edge directions of cube face `face` (geometry.cpp kFrames32 / kFrames23): components are exactly 0, +-1, +-0.5.
T360_HD void cubeFaceFrame(bool offCentreLayout, int face, SphereVec& o, SphereVec& du, SphereVec& dv) {
  const float h = 0.5f;
  if (!offCentreLayout) {
    switch (face) {
      case 0: o = {h, -h, h}; du = {0, 0, -1}; dv = {0, 1, 0}; return;     // RIGHT
      case 1: o = {-h, -h, -h}; du = {0, 0, 1}; dv = {0, 1, 0}; return;    // LEFT
      case 2: o = {-h, h, h}; du = {1, 0, 0}; dv = {0, 0, -1}; return;     // TOP
      case 3: o = {-h, -h, -h}; du = {1, 0, 0}; dv = {0, 0, 1}; return;    // BOTTOM
      case 4: o = {-h, -h, h}; du = {1, 0, 0}; dv = {0, 1, 0}; return;     // FRONT
      default: o = {h, -h, -h}; du = {-1, 0, 0}; dv = {0, 1, 0}; return;  // BACK
    }
  }
  switch (face) {
    case 0: o = {-h, -h, h}; du = {0, 1, 0}; dv = {0, 0, -1}; return;
    case 1: o = {h, h, -h}; du = {-1, 0, 0}; dv = {0, 0, 1}; return;
    case 2: o = {h, -h, h}; du = {0, 1, 0}; dv = {-1, 0, 0}; return;
    case 3: o = {h, -h, -h}; du = {-1, 0, 0}; dv = {0, 1, 0}; return;
    case 4: o = {h, -h, -h}; du = {0, 1, 0}; dv = {0, 0, 1}; return;
    default: o = {h, -h, h}; du = {-1, 0, 0}; dv = {0, 0, -1}; return;
  }
}

T360_HD SphereVec onCubeFace(const SphereGeometry& g, bool offCentreLayout, int face, float fx, float fy) {  // cpp:1115-1116, 1187-1189
  fx = fAdd(fMul(fSub(fx, 0.5f), g.expand), 0.5f);
  fy = fAdd(fMul(fSub(fy, 0.5f), g.expand), 0.5f);
  SphereVec o, du, dv;
  cubeFaceFrame(offCentreLayout, face, o, du, dv);
  return SphereVec{fAdd(fAdd(o.x, fMul(du.x, fx)), fMul(dv.x, fy)), fAdd(fAdd(o.y, fMul(du.y, fx)), fMul(dv.y, fy)),
                   fAdd(fAdd(o.z, fMul(du.z, fx)), fMul(dv.z, fy))};
}

T360_HD int clampFace(int f) { return f < 0 ? 0 : (f > 5 ? 5 : f); }

// distance along unit ray d from the displaced eye to the unit sphere (cpp:53-75)
T360_HD float rayToSphereHD(float dx, float dy, float dz, float ox, float oy, float oz) {
  const float along = fAdd(fAdd(fMul(dx, -ox), fMul(dy, -oy)), fMul(dz, -oz));
  const float off2 = fAdd(fAdd(fMul(ox, ox), fMul(oy, oy)), fMul(oz, oz));
  const float d = fSub(fMul(along, along), off2);
#ifdef __CUDA_ARCH__
  float disc = __double2float_rn(__dadd_rn(static_cast<double>(d), 1.0));
#else
  float disc = static_cast<float>(d + 1.0);
#endif
  if (disc <= 0.0f) return 0.0f;
  disc = fSqrt(disc);
  if (disc < along) return 0.0f;
  return fSub(disc, along);
}

T360_HD void warpOffCentreHD(const SphereGeometry& g, SphereVec& q) {  // cpp:1192-1230
  float n = fSqrt(fAdd(fAdd(fMul(q.x, q.x), fMul(q.y, q.y)), fMul(q.z, q.z)));
  q.x = fDiv(q.x, n); q.y = fDiv(q.y, n); q.z = fDiv(q.z, n);
  if (g.horizontalOffset) {
    n = fSqrt(fAdd(fMul(q.x, q.x), fMul(q.z, q.z)));
    q.x = fDiv(q.x, n); q.y = fDiv(q.y, n); q.z = fDiv(q.z, n);
    const float t = rayToSphereHD(q.x, 0, q.z, g.ox, 0, g.oz);
    if (t > 0.0f) { q.x = fSub(fMul(q.x, t), g.ox); q.z = fSub(fMul(q.z, t), g.oz); }
  } else {
    const float t = rayToSphereHD(q.x, q.y, q.z, g.ox, g.oy, g.oz);
    if (t > 0.0f) { q.x = fSub(fMul(q.x, t), g.ox); q.y = fSub(fMul(q.y, t), g.oy); q.z = fSub(fMul(q.z, t), g.oz); }
  }
}

// unit direction -> 3x2 cubemap input (cpp:796-861): faces tried as -z, +z, -x, +x, -y, +y; the first whose gnomonic
// coordinates fall inside [-1, 1]^2 wins
T360_HD void cubeInputHD(const SphereGeometry& g, float tx, float ty, float tz, float* u, float* v) {
#pragma unroll 1
  for (int f = 0; f < 6; ++f) {
    float major, a, b;
    bool neg = (f & 1) == 0;
    int col, row, su, sv;
    switch (f) {
      case 0: major = tz; a = tx; b = ty; col = 5; row = 3; su = 1; sv = 1; break;
      case 1: major = tz; a = tx; b = ty; col = 3; row = 3; su = 1; sv = -1; break;
      case 2: major = tx; a = tz; b = ty; col = 3; row = 1; su = -1; sv = 1; break;
      case 3: major = tx; a = tz; b = ty; col = 1; row = 1; su = -1; sv = -1; break;
      case 4: major = ty; a = tx; b = tz; col = 1; row = 3; su = -1; sv = 1; break;
      default: major = ty; a = tx; b = tz; col = 5; row = 1; su = 1; sv = 1; break;
    }
    if (neg ? !(major <= -0.5f) : !(major >= 0.5f)) continue;
    const float gx = fDiv(a, major), gy = fDiv(b, major);
    if (gx >= -1.0f && gx <= 1.0f && gy >= -1.0f && gy <= 1.0f) {
      const float sx = fDiv(gx, g.inputExpand), sy = fDiv(gy, g.inputExpand);
      *u = fDiv(su > 0 ? fAdd(static_cast<float>(col), sx) : fSub(static_cast<float>(col), sx), 6.0f);
      *v = fDiv(sv > 0 ? fAdd(static_cast<float>(row), sy) : fSub(static_cast<float>(row), sy), 4.0f);
      return;
    }
  }
  *u = -1.0f;
  *v = 0.0f;
}

// The sampling record {col0, rowPhase} of output pixel (i, j), as HostPlan::samples holds it.  colTab / rowTab: the plan's
// tables (buildSphereTables) at column and row offset.
T360_HD void sphereSample(const SphereGeometry& g, const Rotation& r, const float* colTab, const float* rowTab, int i, int j,
                          int32_t* col0, int32_t* rowPhase) {
  float x = pixelCentre(j, g.mapW), y = pixelCentre(i, g.mapH);
  bool eye = false;
  if (g.splitLR) eye = splitEye(x, false);
  else if (g.splitTB) eye = splitEye(y, g.vflip);
  y = fSub(1.0f, y);
  SphereVec q;
  if (g.outputLayout == LAYOUT_EQUIRECT) {  // cpp:1095-1101: (sin yaw cos pitch, sin pitch, cos yaw cos pitch)
    const float sy = colTab[2 * j], cy = colTab[2 * j + 1], sp = rowTab[2 * i], cp = rowTab[2 * i + 1];
    q = SphereVec{fMul(sy, cp), sp, fMul(cy, cp)};
  } else if (g.outputLayout == LAYOUT_CUBEMAP_23_OFFCENTER) {  // cpp:951-958
    const int row = truncToInt(fMul(y, 3.0f)), col = truncToInt(fMul(x, 2.0f));
    q = onCubeFace(g, true, clampFace(col + (2 - row) * 2), fSub(fMul(x, 2.0f), static_cast<float>(col)),
                   fSub(fMul(y, 3.0f), static_cast<float>(row)));
  } else {  // CUBEMAP_32, EAC_32 (cpp:943-950, 1069-1078)
    const int row = truncToInt(fMul(y, 2.0f)), col = truncToInt(fMul(x, 3.0f));
    float fx, fy;
    if (g.outputLayout == LAYOUT_EAC_32) {
      fx = colTab[j];
      fy = rowTab[i];
    } else {
      fx = fSub(fMul(x, 3.0f), static_cast<float>(col));
      fy = fSub(fMul(y, 2.0f), static_cast<float>(row));
    }
    q = onCubeFace(g, false, clampFace(col + (1 - row) * 3), fx, fy);
  }
  if (g.offCentre) warpOffCentreHD(g, q);
  const float tx = fAdd(fSub(fMul(q.x, r.xx), fMul(q.y, r.xy)), fMul(q.z, r.xz));
  const float ty = -fAdd(fSub(fMul(q.x, r.yx), fMul(q.y, r.yy)), fMul(q.z, r.yz));
  const float tz = fAdd(fSub(fMul(q.x, r.zx), fMul(q.y, r.zy)), fMul(q.z, r.zz));
  const float n = fSqrt(fAdd(fAdd(fMul(tx, tx), fMul(ty, ty)), fMul(tz, tz)));  // cpp:863-891
  float u, v;
  if (g.cubeInput) {
    cubeInputHD(g, fDiv(tx, n), fDiv(ty, n), fDiv(tz, n), &u, &v);
  } else {
    const float lon = -libmAtan2f(fDiv(-tx, n), fDiv(tz, n));
    const float lat = libmAsinf(fDiv(-ty, n));
#ifdef __CUDA_ARCH__
    u = __double2float_rn(__dadd_rn(__ddiv_rn(static_cast<double>(lon), M_PI * 2.0f), 0.5));
    v = __double2float_rn(__dadd_rn(__ddiv_rn(static_cast<double>(lat), M_PI), 0.5));
#else
    u = static_cast<float>(lon / (M_PI * 2.0f) + 0.5f);
    v = static_cast<float>(lat / M_PI + 0.5f);
#endif
  }
  if (g.packTB) v = packEye(v, eye);  // cpp:1278-1300
  else if (g.packLR) u = packEye(u, eye);
  int c0, fracX, r0, fracY;
  quantizeAxis(toPixel(u, g.inW), g.kernelSize, &c0, &fracX);
  quantizeAxis(toPixel(v, g.inH), g.kernelSize, &r0, &fracY);
  *col0 = c0;
  *rowPhase = r0 * 1024 + fracY * 32 + fracX;
}

// The geometry of a plan for `ctx` (mapW x mapH map of an inW x inH input)
inline SphereGeometry sphereGeometry(const FrameTransformContext& ctx, int mapW, int mapH, int inW, int inH, int kernelSize) {
  const bool stereoIn = ctx.input_stereo_format != STEREO_FORMAT_MONO;
  constexpr double kTiny = 1e-9;  // reference kEpsilon (cpp:33), as geometry.cpp decides whether to warp
  SphereGeometry g{};
  g.mapW = mapW; g.mapH = mapH; g.inW = inW; g.inH = inH;
  g.kernelSize = kernelSize;
  g.outputLayout = ctx.output_layout;
  g.cubeInput = ctx.input_layout == LAYOUT_CUBEMAP_32;
  g.splitLR = stereoIn && ctx.output_stereo_format == STEREO_FORMAT_LR;
  g.splitTB = stereoIn && ctx.output_stereo_format == STEREO_FORMAT_TB;
  g.vflip = ctx.vflip != 0;
  g.packLR = ctx.input_stereo_format == STEREO_FORMAT_LR;
  g.packTB = ctx.input_stereo_format == STEREO_FORMAT_TB;
  g.offCentre = std::abs(ctx.fixed_cube_offcenter_x) > kTiny || std::abs(ctx.fixed_cube_offcenter_y) > kTiny ||
                std::abs(ctx.fixed_cube_offcenter_z) > kTiny;
  g.horizontalOffset = ctx.is_horizontal_offset != 0;
  g.expand = ctx.expand_coef;
  g.inputExpand = ctx.input_expand_coef;
  g.ox = ctx.fixed_cube_offcenter_x; g.oy = ctx.fixed_cube_offcenter_y; g.oz = ctx.fixed_cube_offcenter_z;
  return g;
}

// Whether the per-frame orientation chain covers the layouts of `ctx`
inline bool orientedLayouts(const FrameTransformContext& ctx) {
  const int o = ctx.output_layout, in = ctx.input_layout;
  return (o == LAYOUT_CUBEMAP_32 || o == LAYOUT_CUBEMAP_23_OFFCENTER || o == LAYOUT_EAC_32 || o == LAYOUT_EQUIRECT) &&
         (in == LAYOUT_EQUIRECT || in == LAYOUT_CUBEMAP_32);
}

}  // namespace t360
