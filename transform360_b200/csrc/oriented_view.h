// Sphere-output position chain with the orientation as a parameter: one definition for the host and the per-frame
// orientation gather kernel (view_gather.cu).
//
// For output pixel (i, j) of a CUBEMAP_32, CUBEMAP_23_OFFCENTER, EAC_32, EQUIRECT, BARREL or BARREL_SPLIT map, the planner
// (geometry.cpp, Projector::project) computes: pixel centre -> output eye split -> point on the unit cube / sphere (or the
// barrel dead zone) -> off-centre warp -> rotation by yaw / pitch / roll -> input lookup (EQUIRECT: atan2f, asinf, and for
// barrel outputs a clamp clear of the right edge; CUBEMAP_32: gnomonic face coordinates) -> input eye re-pack ->
// u * inW - 0.5f, v * inH - 0.5f -> cv::remap's 1/32-pixel quantisation.  Only the rotation depends on the orientation.
// What remains of libm is reproduced or tabulated so the device gets the planner's bits:
//   - the EAC warp (double tan) depends on the column only for x and on the row only for y, and the sin / cos of yaw /
//     pitch of EQUIRECT and of the barrel bands (float sinf / cosf, FMA ifuncs on the host) on the column (BARREL_SPLIT:
//     and the row half) / the row: per-plan host tables (buildSphereTables, from the planner's own expressions:
//     equiAngular, equirectYaw, equirectPitch, barrelYaw, barrelPitch, barrelSplitYaw, barrelSplitPitch below);
//   - the barrel end caps are float + - * only (the face, BARREL_SPLIT's quarter turns, the disc test): on the device;
//   - the rotation coefficients (double sin / cos of the angles, stored as float): computed on the host per frame by
//     rotationFromAngles, which Projector's constructor calls too;
//   - sqrtf, atan2f, asinf: __fsqrt_rn and the libm ports (libm_ports.h); the double steps of rayToSphere and of the
//     equirectangular lookup: explicit __d*_rn and __double2float_rn.
// As in flat_view.h, every float operation on the device is an explicit _rn intrinsic and the host code is compiled with
// -ffp-contract=off.
#pragma once

#include <cmath>
#include <cstdint>
#include <type_traits>
#include <vector>

#include "Transform360/VideoFrameTransformHelper.h"
#include "flat_view.h"
#include "libm_ports.h"

namespace t360 {

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
inline float barrelYaw(float x, float e) { return static_cast<float>((2.5f * x - 1.0f) * e * M_PI); }      // cpp:970-982
inline float barrelPitch(float y, float e) { return static_cast<float>((y * 0.5f - 0.25f) * e * M_PI); }
inline float barrelSplitYaw(float x, int half, float e) {                                                  // cpp:983-1000
  return static_cast<float>(((3.0f / 2.0f * x - 0.5f) * e - half + 1.0f) * M_PI);
}
inline float barrelSplitPitch(float y, int half, float e) { return static_cast<float>((y - 0.25f - 0.5f * half) * e * M_PI); }

T360_HD bool barrelLayout(int layout) { return layout == LAYOUT_BARREL || layout == LAYOUT_BARREL_SPLIT; }

// Per-plan tables (buildSphereTables), column entries followed by row entries:
//   EAC_32: [mapW] / [mapH], the warped face coordinate of the column / the row;
//   EQUIRECT, BARREL: [mapW][2] / [mapH][2], sin and cos of the column's yaw / the row's pitch;
//   BARREL_SPLIT: [2][mapW][2] / [mapH][2], sin and cos of the yaw of the column in row half 0 and 1 / of the row's pitch.
// (BARREL columns past the band, and BARREL_SPLIT columns past it, have entries nobody reads.)  Other layouts need none.
inline size_t sphereTableRowOffset(const SphereGeometry& g) {
  const size_t w = static_cast<size_t>(g.mapW);
  switch (g.outputLayout) {
    case LAYOUT_EQUIRECT: case LAYOUT_BARREL: return 2 * w;
    case LAYOUT_BARREL_SPLIT: return 4 * w;
    case LAYOUT_EAC_32: return w;
    default: return 0;
  }
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
  } else if (g.outputLayout == LAYOUT_EQUIRECT || barrelLayout(g.outputLayout)) {
    const size_t rows = sphereTableRowOffset(g);
    t.resize(rows + 2 * static_cast<size_t>(g.mapH));
    auto sinCos = [&t](size_t at, float a) {
      t[at] = std::sin(a);
      t[at + 1] = std::cos(a);
    };
    const float e = g.expand;
    for (int j = 0; j < g.mapW; ++j) {
      const float x = sphereColumnX(g, j);
      if (g.outputLayout == LAYOUT_EQUIRECT) sinCos(2 * j, equirectYaw(x));
      else if (g.outputLayout == LAYOUT_BARREL) sinCos(2 * j, barrelYaw(x, e));
      else
        for (int half = 0; half < 2; ++half) sinCos(2 * (static_cast<size_t>(half) * g.mapW + j), barrelSplitYaw(x, half, e));
    }
    for (int i = 0; i < g.mapH; ++i) {
      const float y = sphereRowY(g, i);
      const float a = g.outputLayout == LAYOUT_EQUIRECT ? equirectPitch(y)
                      : g.outputLayout == LAYOUT_BARREL ? barrelPitch(y, e)
                                                        : barrelSplitPitch(y, static_cast<int>(y * 2), e);
      sinCos(rows + 2 * static_cast<size_t>(i), a);
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

// (sin yaw cos pitch, sin pitch, cos yaw cos pitch) from a column and a row entry of the tables (cpp:1095-1101)
T360_HD SphereVec onSphereHD(const float* yawSinCos, const float* pitchSinCos) {
  const float sy = yawSinCos[0], cy = yawSinCos[1], sp = pitchSinCos[0], cp = pitchSinCos[1];
  return SphereVec{fMul(sy, cp), sp, fMul(cy, cp)};
}

// Where a BARREL / BARREL_SPLIT output pixel sits (cpp:970-1068, 1106-1113): the band on the unit sphere from the tables,
// an end cap on the TOP / BOTTOM cube face.  false: outside the cap's disc (the dead zone).
T360_HD bool barrelPoint(const SphereGeometry& g, const float* colTab, const float* rowTab, int i, int j, float x, float y, SphereVec& q) {
  const float e = g.expand;
  float fx, fy;
  int face;
  if (g.outputLayout == LAYOUT_BARREL) {
    if (x <= 0.8f) {
      q = onSphereHD(colTab + 2 * j, rowTab + 2 * i);
      return true;
    }
    const int half = truncToInt(fMul(y, 2.0f));
    face = half == 1 ? TOP : BOTTOM;
    fx = fSub(fMul(x, 5.0f), 4.0f);
    fy = fSub(fMul(y, 2.0f), static_cast<float>(half));
  } else {
    if (fMul(3.0f, x) <= 2.0f) {
      const int half = truncToInt(fMul(y, 2.0f));  // (0 or 1: y = 1 - the row's centre after the eye split, in [0, 1))
      q = onSphereHD(colTab + 2 * (static_cast<size_t>(half) * g.mapW + j), rowTab + 2 * i);
      return true;
    }
    const int quarter = truncToInt(fMul(y, 4.0f));
    fx = fSub(fMul(x, 3.0f), 2.0f);
    fy = y;
    switch (quarter) {  // the caps' four quarters, the first two turned by 180 degrees
      case 0: fy = fMul(fy, 2.0f); fx = fSub(1.0f, fx); fy = fMul(fSub(0.5f, fy), e); break;
      case 1: fy = fMul(fy, 2.0f); fx = fSub(1.0f, fx); fy = fSub(1.0f, fMul(e, fSub(fy, 0.5f))); break;
      case 2: fy = fSub(fMul(fy, 2.0f), 0.5f); fy = fSub(1.0f, fMul(e, fSub(1.0f, fy))); break;
      case 3: fy = fSub(fMul(fy, 2.0f), 1.5f); fy = fMul(fy, e); break;
      default: break;
    }
    face = (quarter == 1 || quarter == 3) ? TOP : BOTTOM;
  }
  const float dx = fSub(fx, 0.5f), dy = fSub(fy, 0.5f);
  if (fAdd(fMul(dx, dx), fMul(dy, dy)) > fMul(fMul(0.25f, e), e)) return false;
  q = onCubeFace(g, false, face, fx, fy);
  return true;
}

// q rotated by r: the planner's rotation, its y row negated (cpp:1233-1244)
T360_HD SphereVec rotateHD(const Rotation& r, const SphereVec& q) {
  return SphereVec{fAdd(fSub(fMul(q.x, r.xx), fMul(q.y, r.xy)), fMul(q.z, r.xz)),
                   -fAdd(fSub(fMul(q.x, r.yx), fMul(q.y, r.yy)), fMul(q.z, r.yz)),
                   fAdd(fSub(fMul(q.x, r.zx), fMul(q.y, r.zy)), fMul(q.z, r.zz))};
}

// The output half of the chain for output pixel (i, j): pixel centre -> output eye split -> point on the cube / sphere ->
// off-centre warp -> rotation by r.  *eye: the output eye; *t: the rotated direction (not normalised), the vector the input
// lookup maps.  Returns false for a barrel dead zone (*t is then not set).  colTab / rowTab: the plan's tables
// (buildSphereTables) at column and row offset.  BARREL = false leaves the barrel layouts out of the code.
template <bool BARREL = true>
T360_HD bool spherePoint(const SphereGeometry& g, const Rotation& r, const float* colTab, const float* rowTab, int i, int j, bool* eye,
                         SphereVec* t) {
  float x = pixelCentre(j, g.mapW), y = pixelCentre(i, g.mapH);
  *eye = false;
  if (g.splitLR) *eye = splitEye(x, false);
  else if (g.splitTB) *eye = splitEye(y, g.vflip);
  y = fSub(1.0f, y);
  const bool barrel = BARREL && barrelLayout(g.outputLayout);
  SphereVec q;
  bool mapped = true;
  if (barrel) {
    mapped = barrelPoint(g, colTab, rowTab, i, j, x, y, q);
  } else if (g.outputLayout == LAYOUT_EQUIRECT) {
    q = onSphereHD(colTab + 2 * j, rowTab + 2 * i);
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
  if (mapped) {
    if (g.offCentre) warpOffCentreHD(g, q);
    *t = rotateHD(r, q);
  }
  return mapped;
}

// The input lookup of rotated direction t (not normalised) in output eye `eye`: (*u, *v) in the input, re-packed for a
// stereo input (cpp:863-891, 1278-1300).  EQUIRECT (any input but CUBEMAP_32): atan2f / asinf, and with `barrel` u kept
// half an input pixel clear of 0 and 1; CUBEMAP_32: gnomonic face coordinates.  Shared by the sphere outputs (sphereSample)
// and the rectilinear views (rectilinearPosition).
T360_HD void sphereInputHD(const SphereGeometry& g, bool barrel, bool eye, const SphereVec& t, float* u, float* v) {
  const float tx = t.x, ty = t.y, tz = t.z;
  const float n = fSqrt(fAdd(fAdd(fMul(tx, tx), fMul(ty, ty)), fMul(tz, tz)));  // cpp:863-891
  if (g.cubeInput) {
    cubeInputHD(g, fDiv(tx, n), fDiv(ty, n), fDiv(tz, n), u, v);
  } else {
    const float lon = -libmAtan2f(fDiv(-tx, n), fDiv(tz, n));
    const float lat = libmAsinf(fDiv(-ty, n));
#ifdef __CUDA_ARCH__
    *u = __double2float_rn(__dadd_rn(__ddiv_rn(static_cast<double>(lon), M_PI * 2.0f), 0.5));
    *v = __double2float_rn(__dadd_rn(__ddiv_rn(static_cast<double>(lat), M_PI), 0.5));
#else
    *u = static_cast<float>(lon / (M_PI * 2.0f) + 0.5f);
    *v = static_cast<float>(lat / M_PI + 0.5f);
#endif
    if (barrel) {  // std::min, then std::max, as the ternaries they are: a NaN u stays NaN (cpp:881-886)
      const float lo = fMul(g.inPixelWidth, 0.5f), hi = fSub(1.0f, lo);
      *u = hi < *u ? hi : *u;
      *u = *u < lo ? lo : *u;
    }
  }
  if (g.packTB) *v = packEye(*v, eye);  // cpp:1278-1300
  else if (g.packLR) *u = packEye(*u, eye);
}

// The sampling record {col0, rowPhase} of output pixel (i, j), as HostPlan::samples holds it: spherePoint, then the input
// lookup.  BARREL = false leaves the barrel layouts out of the code (the orientation kernel's instantiations for the other
// layouts).
template <bool BARREL = true>
T360_HD void sphereSample(const SphereGeometry& g, const Rotation& r, const float* colTab, const float* rowTab, int i, int j,
                          int32_t* col0, int32_t* rowPhase) {
  const bool barrel = BARREL && barrelLayout(g.outputLayout);
  bool eye;
  SphereVec t;
  const bool mapped = spherePoint<BARREL>(g, r, colTab, rowTab, i, j, &eye, &t);
  float u = -1.0f, v = 0.0f;  // the dead zone's position, not re-packed (cpp:1304-1306)
  if (mapped) sphereInputHD(g, barrel, eye, t, &u, &v);
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
  g.inPixelWidth = 1.0f / inW;  // cpp:528-531, as buildWarpMap
  if (g.packLR) g.inPixelWidth *= 2;
  return g;
}

// ---- fisheye lens input ---------------------------------------------------------------------------------------------
// A rig of one or two fisheye lenses with OpenCV's fisheye (Kannala-Brandt) calibration replaces the input lookup: the
// rotated direction d = (tx, ty, tz) of spherePoint (the rig frame: x right, y up, z forward, the frame an equirect input
// shows at u = atan2(x, z) / 2pi + 0.5) goes to the lens whose axis it is closest to (the larger Z; ties to lens 0), then
//   (X, Y, Z) = M d               (M: the lens's R^T with its y row negated: OpenCV camera coordinates, y down)
//   rho = sqrt(X^2 + Y^2), theta = atan2(rho, Z)         (theta > thetaMax: not covered, NaN)
//   theta_d = theta (1 + t (k1 + t (k2 + t (k3 + t k4)))), t = theta^2      (Horner)
//   (x', y') = theta_d / rho (X, Y), (0, 0) at rho = 0
//   position = ((fx x' + cx + 0.5) / calibWidth) inW - 0.5 = (ax x' + bx) inW - 0.5, and likewise for y
// Only + - * /, sqrt and atan2 (libmAtan2f), so host and device give the same bits; the constants are computed on the
// host in double and stored as float (lensRigModel, video_frame_transform.cpp).
struct LensModel {
  float m[9];              // rig direction -> camera coordinates, row major
  float ax, bx, ay, by;    // fx / calibWidth, (cx + 0.5) / calibWidth, fy / calibHeight, (cy + 0.5) / calibHeight
  float k[4];              // k1 .. k4
  float thetaMax;          // maxAngle in radians
};
struct LensRigModel {
  int numLenses;  // 1 or 2
  LensModel lens[2];
};

T360_HD float lensRow(const float* m, const SphereVec& d) { return fAdd(fAdd(fMul(m[0], d.x), fMul(m[1], d.y)), fMul(m[2], d.z)); }

// What one lens makes of rig direction d: theta, whether it covers d (theta <= thetaMax), and where it does, the source
// position (px, py) in an inW x inH plane (NaN for both where it does not).  Z = lensRow(L.m + 6, d), which the callers
// have already computed.  The one place the lens projection is written: the hard seam (lensPosition) and the feathered
// seam (lensBlendPosition) both call it.  R = true also keeps r = theta_d, the distorted angle (so the image radius is
// f theta_d), for the photometric falloff (lensGain), in a LensHitR; the callers that do not need it compile exactly as
// they did before it was kept.
struct LensHit {
  float theta, px, py;
  bool covered;
};
struct LensHitR : LensHit {
  float r;  // theta_d where covered
};
template <bool R = false>
T360_HD std::conditional_t<R, LensHitR, LensHit> lensHit(const LensModel& L, const SphereVec& d, float Z, int inW, int inH) {
  const float X = lensRow(L.m, d), Y = lensRow(L.m + 3, d);
  const float rho = fSqrt(fAdd(fMul(X, X), fMul(Y, Y)));
  std::conditional_t<R, LensHitR, LensHit> h;
  h.theta = libmAtan2f(rho, Z);
  h.covered = h.theta <= L.thetaMax;
  if (!h.covered) {
    h.px = h.py = bitsFloat(0x7fc00000u);
    if constexpr (R) h.r = h.px;
    return h;
  }
  const float t = fMul(h.theta, h.theta);
  const float poly = fAdd(1.0f, fMul(t, fAdd(L.k[0], fMul(t, fAdd(L.k[1], fMul(t, fAdd(L.k[2], fMul(t, L.k[3]))))))));
  const float s = rho > 0.0f ? fDiv(fMul(h.theta, poly), rho) : 0.0f;
  if constexpr (R) h.r = fMul(h.theta, poly);
  h.px = toPixel(fAdd(fMul(L.ax, fMul(s, X)), L.bx), inW);
  h.py = toPixel(fAdd(fMul(L.ay, fMul(s, Y)), L.by), inH);
  return h;
}

// The source position (*px, *py) of rig direction d in an inW x inH plane; NaN for both where no lens covers d.
T360_HD void lensPosition(const LensRigModel& rig, const SphereVec& d, int inW, int inH, float* px, float* py) {
  const float z0 = lensRow(rig.lens[0].m + 6, d);
  const float z1 = rig.numLenses > 1 ? lensRow(rig.lens[1].m + 6, d) : z0;
  const bool second = z1 > z0;
  const LensHit h = lensHit(second ? rig.lens[1] : rig.lens[0], d, second ? z1 : z0, inW, inH);
  *px = h.px;
  *py = h.py;
}

// The feathered seam's weight (0..256) of lens 1 where both lenses cover a direction: a linear ramp in theta0 - theta1,
// t = 0.5 + (theta0 - theta1) s rounded to 1/256 (half to even) and clamped
T360_HD int seamWeight(float theta0, float theta1, float s) {
  const float tw = fMul(fAdd(0.5f, fMul(fSub(theta0, theta1), s)), 256.0f);
  return tw <= 0.0f ? 0 : (tw >= 256.0f ? 256 : roundHalfEven(tw));
}

// The feathered seam of a two-lens rig (T360B200_transformFrameLensBlendAsync): both lenses' view of d and the weight w
// (0..256) of lens 1.  Where both cover d, w is a linear ramp in theta0 - theta1, t = 0.5 + (theta0 - theta1) s rounded to
// 1/256 and clamped (s = 1 / (2 seamWidth), seamWidth in radians, computed on the host in double: lensSeamScale); where
// one covers d, that lens alone (w = 0 or 256).  p0 / p1: lens 0's / lens 1's source position, NaN where that lens does
// not contribute (it does not cover d, or w gives it no weight).  Returns w; 0 where neither lens covers d.
T360_HD int lensBlendPosition(const LensRigModel& rig, float s, const SphereVec& d, int inW, int inH, float* p0, float* p1) {
  const LensHit h0 = lensHit(rig.lens[0], d, lensRow(rig.lens[0].m + 6, d), inW, inH);
  const LensHit h1 = lensHit(rig.lens[1], d, lensRow(rig.lens[1].m + 6, d), inW, inH);
  int w = h1.covered ? 256 : 0;
  if (h0.covered && h1.covered) w = seamWeight(h0.theta, h1.theta, s);
  const float nan = bitsFloat(0x7fc00000u);
  p0[0] = w < 256 ? h0.px : nan;
  p0[1] = w < 256 ? h0.py : nan;
  p1[0] = w > 0 ? h1.px : nan;
  p1[1] = w > 0 ? h1.py : nan;
  return w;
}

// The map entry of output pixel (i, j) of a lens rig: spherePoint, then lensPosition; NaN in a barrel dead zone.  The
// geometry's input fields other than inW / inH play no part.
template <bool BARREL = true>
T360_HD void lensPoint(const SphereGeometry& g, const Rotation& r, const LensRigModel& rig, const float* colTab, const float* rowTab, int i,
                       int j, float* px, float* py) {
  bool eye;
  SphereVec d;
  if (!spherePoint<BARREL>(g, r, colTab, rowTab, i, j, &eye, &d)) {
    *px = *py = bitsFloat(0x7fc00000u);
    return;
  }
  lensPosition(rig, d, g.inW, g.inH, px, py);
}

// The sampling record of output pixel (i, j) of a lens rig: its map entry, quantised as quantizeWarpMap quantises a
// caller's map, so T360B200_lensMap -> T360B200_generateMapFromWarp plans the records the lens kernel computes.
template <bool BARREL = true>
T360_HD void lensSample(const SphereGeometry& g, const Rotation& r, const LensRigModel& rig, const float* colTab, const float* rowTab, int i,
                        int j, int32_t* col0, int32_t* rowPhase) {
  float px, py;
  lensPoint<BARREL>(g, r, rig, colTab, rowTab, i, j, &px, &py);
  int r0, fracX, fracY;
  quantizeAxis(px, g.kernelSize, col0, &fracX);
  quantizeAxis(py, g.kernelSize, &r0, &fracY);
  *rowPhase = r0 * 1024 + fracY * 32 + fracX;
}

// The two map entries and the weight of output pixel (i, j) of a two-lens rig with a feathered seam: spherePoint, then
// lensBlendPosition; both entries NaN and w = 0 in a barrel dead zone.  (T360B200_lensBlendMaps)
template <bool BARREL = true>
T360_HD int lensBlendPoint(const SphereGeometry& g, const Rotation& r, const LensRigModel& rig, float s, const float* colTab,
                           const float* rowTab, int i, int j, float* p0, float* p1) {
  bool eye;
  SphereVec d;
  if (!spherePoint<BARREL>(g, r, colTab, rowTab, i, j, &eye, &d)) {
    p0[0] = p0[1] = p1[0] = p1[1] = bitsFloat(0x7fc00000u);
    return 0;
  }
  return lensBlendPosition(rig, s, d, g.inW, g.inH, p0, p1);
}

// The sampling records of output pixel (i, j) of a two-lens rig with a feathered seam, lens 0's in rec0 and lens 1's in
// rec1 ({col0, rowPhase}, quantised as lensSample quantises its entry), and the weight w of lens 1 (the return value).
template <bool BARREL = true>
T360_HD int lensBlendSample(const SphereGeometry& g, const Rotation& r, const LensRigModel& rig, float s, const float* colTab,
                            const float* rowTab, int i, int j, int32_t* rec0, int32_t* rec1) {
  float p[2][2];
  const int w = lensBlendPoint<BARREL>(g, r, rig, s, colTab, rowTab, i, j, p[0], p[1]);
  int32_t* rec[2] = {rec0, rec1};
  for (int l = 0; l < 2; ++l) {
    int r0, fracX, fracY;
    quantizeAxis(p[l][0], g.kernelSize, &rec[l][0], &fracX);
    quantizeAxis(p[l][1], g.kernelSize, &r0, &fracY);
    rec[l][1] = r0 * 1024 + fracY * 32 + fracX;
  }
  return w;
}

// ---- photometric correction of a lens rig (T360B200_transformFrameLensPhotoAsync, T360B200_lensPhotoMaps) -------------
// Each lens's sample s of plane p is corrected before the seam combines the two:
//   V = 1 + t (v1 + t (v2 + t v3)), t = r^2, r = theta_d (lensHit<true>)  the lens's radial falloff
//   Gq = min(round_half_even(gain_p / V * 4096), 65535)                     (lensGain)
//   s' = clamp(P + (((s - P) Gq + Oq 256 + 2048) >> 12), 0, 255)          (photoCorrect; Oq = round(16 offset_p))
// with the pivot P = lumaPivot for luma, 128 for chroma.  The constants of one plane, per lens, are computed on the host
// (lensPhotoPlane, video_frame_transform.cpp).
struct LensPhotoPlane {
  float v[2][3];  // v1..v3 of each lens
  float gain[2];  // gain_p of each lens
  int offset[2];  // Oq of each lens: the offset in 1/16 code value
  int pivot;
};

// Gq of lens hit h: the one place the falloff is written (the kernel and the host twin both call it).  0 where the lens
// does not cover the direction; 0 also for a V that is not positive or a NaN (the host refuses falloffs that reach 0).
T360_HD int lensGain(const LensHitR& h, const float* v, float gain) {
  if (!h.covered) return 0;
  const float t = fMul(h.r, h.r);
  const float V = fAdd(1.0f, fMul(t, fAdd(v[0], fMul(t, fAdd(v[1], fMul(t, v[2]))))));
  const float q = fMul(fDiv(gain, V), 4096.0f);
  return q >= 65535.0f ? 65535 : (q > 0.0f ? roundHalfEven(q) : 0);
}

// s' of sample s (0..255), gain Gq, offset Oq and pivot P, in integers
T360_HD int photoCorrect(int s, int gq, int oq, int pivot) {
  const int c = pivot + (((s - pivot) * gq + oq * 256 + 2048) >> 12);
  return c < 0 ? 0 : (c > 255 ? 255 : c);
}

// Both lenses' view of rig direction d for the photometric calls, and the weight w (0..256) of lens 1.  s = 0: the hard
// seam, w = 256 where lens 1 is the closer lens (lensPosition's choice), else 0; s > 0: the feathered seam's w
// (lensBlendPosition).  p0 / p1: lens 0's / lens 1's source position wherever that lens covers d (NaN elsewhere), g0 / g1
// its Gq (lensGain; 0 where it does not cover d); *overlap: both lenses cover d.  both = false with the hard seam computes
// the closer lens only (the other's position NaN, its gain 0, no overlap): all the frame needs when no statistics are taken.
// STEREO (a stereo rig, s = 0): output eye `eye` picks the lens instead of the closer axis; lens e is eye e's.
template <bool STEREO = false>
T360_HD int lensPhotoPosition(const LensRigModel& rig, float s, bool both, const LensPhotoPlane& c, const SphereVec& d, int inW, int inH,
                              float* p0, float* p1, int* g0, int* g1, bool* overlap, bool eye = false) {
  const float nan = bitsFloat(0x7fc00000u);
  const float z0 = lensRow(rig.lens[0].m + 6, d);
  const float z1 = rig.numLenses > 1 ? lensRow(rig.lens[1].m + 6, d) : z0;
  const bool second = STEREO ? eye : z1 > z0;
  if (s == 0.0f && !both) {  // the closer lens alone, as lensPosition projects it
    const int l = second ? 1 : 0;
    const LensHitR h = lensHit<true>(rig.lens[l], d, second ? z1 : z0, inW, inH);
    float* p = second ? p1 : p0;
    float* q = second ? p0 : p1;
    p[0] = h.px; p[1] = h.py;
    q[0] = q[1] = nan;
    *(second ? g1 : g0) = lensGain(h, c.v[l], c.gain[l]);
    *(second ? g0 : g1) = 0;
    *overlap = false;
    return second ? 256 : 0;
  }
  LensHitR h0 = lensHit<true>(rig.lens[0], d, z0, inW, inH), h1;
  h1.covered = false;
  h1.px = h1.py = h1.r = nan;
  if (rig.numLenses > 1) h1 = lensHit<true>(rig.lens[1], d, z1, inW, inH);
  int w = second ? 256 : 0;
  if (s > 0.0f) {
    w = h1.covered ? 256 : 0;
    if (h0.covered && h1.covered) w = seamWeight(h0.theta, h1.theta, s);
  }
  p0[0] = h0.px; p0[1] = h0.py;
  p1[0] = h1.px; p1[1] = h1.py;
  *g0 = lensGain(h0, c.v[0], c.gain[0]);
  *g1 = lensGain(h1, c.v[1], c.gain[1]);
  *overlap = h0.covered && h1.covered;
  return w;
}

// The two map entries, the weight and the two gains of output pixel (i, j) of a lens rig with photometry: spherePoint,
// then lensPhotoPosition; both entries NaN, w = 0, both gains 0 and no overlap in a barrel dead zone.
// (T360B200_lensPhotoMaps)
template <bool BARREL = true>
T360_HD int lensPhotoPoint(const SphereGeometry& g, const Rotation& r, const LensRigModel& rig, float s, bool both, const LensPhotoPlane& c,
                           const float* colTab, const float* rowTab, int i, int j, float* p0, float* p1, int* g0, int* g1, bool* overlap) {
  bool eye;
  SphereVec d;
  if (!spherePoint<BARREL>(g, r, colTab, rowTab, i, j, &eye, &d)) {
    p0[0] = p0[1] = p1[0] = p1[1] = bitsFloat(0x7fc00000u);
    *g0 = *g1 = 0;
    *overlap = false;
    return 0;
  }
  return lensPhotoPosition(rig, s, both, c, d, g.inW, g.inH, p0, p1, g0, g1, overlap);
}

// The sampling records of output pixel (i, j) of a lens rig with photometry, lens 0's in rec0 and lens 1's in rec1
// (quantised as lensSample quantises its entry), the gains, the overlap and the weight w of lens 1 (the return value).
template <bool BARREL = true>
T360_HD int lensPhotoSample(const SphereGeometry& g, const Rotation& r, const LensRigModel& rig, float s, bool both, const LensPhotoPlane& c,
                            const float* colTab, const float* rowTab, int i, int j, int32_t* rec0, int32_t* rec1, int* g0, int* g1,
                            bool* overlap) {
  float p[2][2];
  const int w = lensPhotoPoint<BARREL>(g, r, rig, s, both, c, colTab, rowTab, i, j, p[0], p[1], g0, g1, overlap);
  int32_t* rec[2] = {rec0, rec1};
  for (int l = 0; l < 2; ++l) {
    int r0, fracX, fracY;
    quantizeAxis(p[l][0], g.kernelSize, &rec[l][0], &fracX);
    quantizeAxis(p[l][1], g.kernelSize, &r0, &fracY);
    rec[l][1] = r0 * 1024 + fracY * 32 + fracX;
  }
  return w;
}

// ---- camera views (rectilinear and the other camera models) ---------------------------------------------------------
// A virtual camera in place of the cube / sphere output: output pixel (i, j) of a mapW x mapH plane, x and y its centre
// after the output eye split (as spherePoint), y' = 1 - y, X = 2x - 1, Y = 2y' - 1 (+-1 at the plane's outer pixel edges),
// looks along the model's ray q, rotated by the pose as spherePoint rotates its point:
//   kCameraPinhole        q = (X cx, Y cy, 1), cx = tan(hfov / 2), cy = tan(vfov / 2).  So with hfov = vfov = 90 an N x N
//                         view is the FRONT face of a 3N x 2N CUBEMAP_32 output of the same orientation;
//   kCameraEquidistant    a = X cx, b = Y cy (cx = hfov pi / 360, cy = vfov pi / 360: the angle to the axis), rho the
//                         length of (a, b), q = (a S, b S, C) with S = sin rho / rho, C = cos rho (sincCos);
//   kCameraStereographic  a = X cx, b = Y cy (cx = tan(hfov / 4), cy = tan(vfov / 4)), q = (2a, 2b, 1 - a^2 - b^2);
//   kCameraPannini        u = X cx, w = Y cy (cx = (d + 1) sin h / (d + cos h), h = hfov / 2, cy = tan(vfov / 2)),
//                         k = (u e)^2, c = (-k d + sqrt(1 + k dd)) / (k + 1) (e = 1 / (d + 1), dd = 1 - d^2: Sharpless et
//                         al.'s inverse with its discriminant k^2 d^2 - (k + 1)(k d^2 - 1) expanded, so it cannot cancel),
//                         q = (u (d + c) e, w (d + c) e, c), proportional to (sin lon, tan lat, cos lon), c = cos lon;
//   kCameraEquirect       lon = X cx, lat = Y cy (cx = hfov pi / 360, cy = vfov pi / 360), q = (cos lat sin lon, sin lat,
//                         cos lat cos lon), sin a = a S(a) and cos a = C(a) from sincCos (even in a; |lon| <= pi lies in its
//                         range).  4 is not a model: the model numbers are public, and 4 stays refused.
// The per-pose constants are computed on the host in double and stored as float (cameraConstants in
// video_frame_transform.cpp).  The input is the context's (sphereInputHD, BORDER_WRAP) or a lens rig (lensPosition,
// BORDER_TRANSPARENT).  Only + - * / and sqrt on the output half, so host and device agree bit for bit.
enum CameraModel { kCameraPinhole = 0, kCameraEquidistant = 1, kCameraStereographic = 2, kCameraPannini = 3, kCameraEquirect = 5 };
struct RectilinearCamera {
  Rotation r;
  float cx, cy;  // the model's per-axis constants above
  int model;     // CameraModel (the same for every pixel of a launch: a warp-uniform branch)
  float d, e, dd;  // kCameraPannini: d, 1 / (d + 1), 1 - d^2
};

// The per-frame constants of a pose (degrees) and a camera model: the rotation, and the model's constants in double,
// stored as float.  Host only: the device receives the result (T360B200_cameraMap and the camera kernels).
inline RectilinearCamera cameraConstants(int model, float pannini, float yaw, float pitch, float roll, float hfov, float vfov) {
  RectilinearCamera c{};
  c.r = rotationFromAngles(yaw, pitch, roll);
  c.model = model;
  const double h = static_cast<double>(hfov) * M_PI / 360.0, v = static_cast<double>(vfov) * M_PI / 360.0;  // half angles
  switch (model) {
    case kCameraEquidistant:
    case kCameraEquirect:
      c.cx = static_cast<float>(h);
      c.cy = static_cast<float>(v);
      break;
    case kCameraStereographic:
      c.cx = static_cast<float>(std::tan(h / 2.0));
      c.cy = static_cast<float>(std::tan(v / 2.0));
      break;
    case kCameraPannini: {
      const double d = pannini;
      c.cx = static_cast<float>((d + 1.0) * std::sin(h) / (d + std::cos(h)));
      c.cy = static_cast<float>(std::tan(v));
      c.d = pannini;
      c.e = static_cast<float>(1.0 / (d + 1.0));
      c.dd = static_cast<float>(1.0 - d * d);
      break;
    }
    default:
      c.cx = static_cast<float>(std::tan(h));
      c.cy = static_cast<float>(std::tan(v));
  }
  return c;
}

// sin(rho) / rho (1 at rho = 0) and cos(rho) for rho in [0, pi sqrt 2] from + - * / only: h = rho / 4, the Taylor
// polynomials of sin(h) / h and cos(h) in h^2 (|h| <= 1.12: the first dropped terms are below 1e-9), then two angle
// doublings: sin 2h / 2h = (sin h / h) cos h, cos 2h = 1 - 2 sin^2 h.  tests/test_camera_models.py compares it with
// double over every float of the range.
T360_HD void sincCos(float rho, float* sinc, float* cosine) {
  const float h = fMul(rho, 0.25f), t = fMul(h, h);
  float s = fAdd(fMul(t, -1.0f / 6227020800.0f), 1.0f / 39916800.0f);  // sin(h) / h = sum (-t)^n / (2n + 1)!
  s = fSub(fMul(t, s), 1.0f / 362880.0f);
  s = fAdd(fMul(t, s), 1.0f / 5040.0f);
  s = fSub(fMul(t, s), 1.0f / 120.0f);
  s = fAdd(fMul(t, s), 1.0f / 6.0f);
  s = fSub(1.0f, fMul(t, s));
  float c = fAdd(fMul(t, -1.0f / 87178291200.0f), 1.0f / 479001600.0f);  // cos(h) = sum (-t)^n / (2n)!
  c = fSub(fMul(t, c), 1.0f / 3628800.0f);
  c = fAdd(fMul(t, c), 1.0f / 40320.0f);
  c = fSub(fMul(t, c), 1.0f / 720.0f);
  c = fAdd(fMul(t, c), 1.0f / 24.0f);
  c = fSub(fMul(t, c), 0.5f);
  c = fAdd(fMul(t, c), 1.0f);
  float a = h;
  for (int k = 0; k < 2; ++k) {  // (s, c) of angle a -> of angle 2a
    const float sn = fMul(a, s);
    s = fMul(s, c);
    c = fSub(1.0f, fMul(2.0f, fMul(sn, sn)));
    a = fMul(a, 2.0f);
  }
  *sinc = s;
  *cosine = c;
}

// The equirect model's ray at longitude lon and latitude lat.  Out of line on the device, and tested inside cameraRay's
// last case rather than as a case of its own, so the other models' branches compile as they did before the model existed.
#ifdef __CUDA_ARCH__
__device__ __noinline__
#else
inline
#endif
SphereVec equirectRay(float lon, float lat) {
  float sl, cl, sp, cp;
  sincCos(lon, &sl, &cl);
  sincCos(lat, &sp, &cp);
  return SphereVec{fMul(cp, fMul(lon, sl)), fMul(lat, sp), fMul(cp, cl)};
}

// The ray q (not rotated, not normalised) of the pixel at (X, Y) for the models other than the pinhole
T360_HD SphereVec cameraRay(const RectilinearCamera& c, float X, float Y) {
  switch (c.model) {
    case kCameraEquidistant: {
      const float a = fMul(X, c.cx), b = fMul(Y, c.cy);
      float s, co;
      sincCos(fSqrt(fAdd(fMul(a, a), fMul(b, b))), &s, &co);
      return SphereVec{fMul(a, s), fMul(b, s), co};
    }
    case kCameraStereographic: {
      const float a = fMul(X, c.cx), b = fMul(Y, c.cy);
      return SphereVec{fMul(2.0f, a), fMul(2.0f, b), fSub(fSub(1.0f, fMul(a, a)), fMul(b, b))};
    }
    default: {  // kCameraPannini, kCameraEquirect
      if (c.model == kCameraEquirect) return equirectRay(fMul(X, c.cx), fMul(Y, c.cy));
      const float u = fMul(X, c.cx), w = fMul(Y, c.cy);
      const float ue = fMul(u, c.e), k = fMul(ue, ue);
      const float cl = fDiv(fAdd(-fMul(k, c.d), fSqrt(fAdd(1.0f, fMul(k, c.dd)))), fAdd(k, 1.0f));
      const float f = fMul(fAdd(c.d, cl), c.e);
      return SphereVec{fMul(u, f), fMul(w, f), cl};
    }
  }
}

// Steps 1-5 of the contract for output pixel (i, j): the rotated ray (not normalised) and the output eye.  The geometry's
// mapW, mapH, splitLR, splitTB and vflip play a part.  ANY_MODEL = false: c is a pinhole (the kernel's own loop for
// pinhole launches, which so keeps the rectilinear view's code).  (These are cameraXY's steps and modelRay's pinhole ray,
// written out: built on them, the rectilinear kernels compile to different SASS.)
template <bool ANY_MODEL = true>
T360_HD SphereVec rectilinearPoint(const SphereGeometry& g, const RectilinearCamera& c, int i, int j, bool* eye) {
  float x = pixelCentre(j, g.mapW), y = pixelCentre(i, g.mapH);
  *eye = false;
  if (g.splitLR) *eye = splitEye(x, false);
  else if (g.splitTB) *eye = splitEye(y, g.vflip);
  y = fSub(1.0f, y);
  const float X = fSub(fMul(2.0f, x), 1.0f), Y = fSub(fMul(2.0f, y), 1.0f);
  if (!ANY_MODEL || c.model == kCameraPinhole) return rotateHD(c.r, SphereVec{fMul(X, c.cx), fMul(Y, c.cy), 1.0f});
  return rotateHD(c.r, cameraRay(c, X, Y));
}

// The CV_32FC2 map entry (*px, *py) of output pixel (i, j) of a rectilinear view: LENS = false the context's input
// (sphereInputHD, no barrel clamp), LENS = true the rig's hard seam (NaN where no lens covers the ray).
template <bool LENS, bool ANY_MODEL = true>
T360_HD void rectilinearPosition(const SphereGeometry& g, const RectilinearCamera& c, const LensRigModel& rig, int i, int j, float* px,
                                 float* py) {
  bool eye;
  const SphereVec d = rectilinearPoint<ANY_MODEL>(g, c, i, j, &eye);
  if constexpr (LENS) {
    lensPosition(rig, d, g.inW, g.inH, px, py);
  } else {
    float u, v;
    sphereInputHD(g, false, eye, d, &u, &v);
    *px = toPixel(u, g.inW);
    *py = toPixel(v, g.inH);
  }
}

// The sampling record of output pixel (i, j) of a rectilinear view: its map entry quantised as quantizeWarpMap quantises a
// caller's map, so T360B200_rectilinearMap -> T360B200_generateMapFromWarp plans the records the kernel computes.
template <bool LENS, bool ANY_MODEL = true>
T360_HD void rectilinearSample(const SphereGeometry& g, const RectilinearCamera& c, const LensRigModel& rig, int i, int j, int32_t* col0,
                               int32_t* rowPhase) {
  float px, py;
  rectilinearPosition<LENS, ANY_MODEL>(g, c, rig, i, j, &px, &py);
  int r0, fracX, fracY;
  quantizeAxis(px, g.kernelSize, col0, &fracX);
  quantizeAxis(py, g.kernelSize, &r0, &fracY);
  *rowPhase = r0 * 1024 + fracY * 32 + fracX;
}

// ---- anti-aliased camera views (T360B200_cameraMipMaps, T360B200_transformFrameCameraMipAsync) -----------------------
// A camera view sampled from an input pyramid (level l + 1 = INTER_AREA of level l to half its size, rounded up), each
// pixel at the level its footprint asks for (Williams 1983), the footprint from ray differentials (Igehy 1999):
//   rx = R (q(X + dX/2, Y) - q(X - dX/2, Y)), ry = R (q(X, Y + dY/2) - q(X, Y - dY/2)) (q: the model's ray, R: the pose),
//   a = J rx, b = J ry with J the Jacobian, at the pixel's rotated ray t, of the input lookup the pixel takes, in level-0
//   pixels of the plane; rho^2 = max(a.a, b.b); lambda = 1/2 log2 rho^2 in 1/256 level from the float's bits.
// The Jacobians are written out analytically with + - * / and sqrt (the lookup's atan2 / asin are not differentiated
// through libm; a lens's theta, which its projection needs anyway, is libmAtan2f), so host and device agree bit for bit.
constexpr int kMipMaxLevels = 8;
struct MipGeometry {
  float halfX, halfY;             // dX / 2, dY / 2: one column / row of one eye in X and Y (host, double -> float)
  int top;                        // the plane's top level T (0: no pyramid)
  float sx[kMipMaxLevels + 1];    // W_l / W_0, H_l / H_0 (host, double -> float; [0] unused)
  float sy[kMipMaxLevels + 1];
};

// The pyramid of a w x h plane for maxLevel: its top level T, the largest l <= maxLevel whose sides ceil(w / 2^l),
// ceil(h / 2^l) are both >= 8 (0 if there is none), and the sides of levels 0..T.  The one place the level sizes are
// walked: the host twin's constants (mipGeometry), the frame call's scratch and launches, and the kernel's level table all
// take them from here.
struct MipSizes {
  int top;
  int w[kMipMaxLevels + 1], h[kMipMaxLevels + 1];
};
T360_HD MipSizes mipSizes(int w, int h, int maxLevel) {
  MipSizes m{};
  m.w[0] = w;
  m.h[0] = h;
  while (m.top < maxLevel && (m.w[m.top] + 1) / 2 >= 8 && (m.h[m.top] + 1) / 2 >= 8) {
    m.w[m.top + 1] = (m.w[m.top] + 1) / 2;
    m.h[m.top + 1] = (m.h[m.top] + 1) / 2;
    ++m.top;
  }
  return m;
}

// The footprint constants of one plane of a camera view (g: the camera view's geometry) for maxLevel: dX / 2 and dY / 2
// (one column / row of one eye), the top level, and the levels' size ratios, in double and stored as float.  Host only:
// the device receives the result (T360B200_cameraMipMaps and the frame call).
inline MipGeometry mipGeometry(const SphereGeometry& g, int maxLevel) {
  const MipSizes z = mipSizes(g.inW, g.inH, maxLevel);
  MipGeometry m{};
  m.halfX = static_cast<float>((g.splitLR ? 2.0 : 1.0) / g.mapW);
  m.halfY = static_cast<float>((g.splitTB ? 2.0 : 1.0) / g.mapH);
  m.top = z.top;
  for (int l = 0; l <= z.top; ++l) {
    m.sx[l] = static_cast<float>(static_cast<double>(z.w[l]) / g.inW);
    m.sy[l] = static_cast<float>(static_cast<double>(z.h[l]) / g.inH);
  }
  return m;
}

// The pixel's X, Y (steps 1-3 of the camera contract, +-1 at the plane's outer pixel edges) and its output eye
T360_HD void cameraXY(const SphereGeometry& g, int i, int j, float* X, float* Y, bool* eye) {
  float x = pixelCentre(j, g.mapW), y = pixelCentre(i, g.mapH);
  *eye = false;
  if (g.splitLR) *eye = splitEye(x, false);
  else if (g.splitTB) *eye = splitEye(y, g.vflip);
  y = fSub(1.0f, y);
  *X = fSub(fMul(2.0f, x), 1.0f);
  *Y = fSub(fMul(2.0f, y), 1.0f);
}

// The ray q (not rotated, not normalised) of any model, the pinhole's as rectilinearPoint writes it
T360_HD SphereVec modelRay(const RectilinearCamera& c, float X, float Y) {
  if (c.model == kCameraPinhole) return SphereVec{fMul(X, c.cx), fMul(Y, c.cy), 1.0f};
  return cameraRay(c, X, Y);
}

// R (q(X1, Y1) - q(X0, Y0)): the rotated ray differential between two points of the image plane
T360_HD SphereVec rayDifferential(const RectilinearCamera& c, float X0, float Y0, float X1, float Y1) {
  const SphereVec a = modelRay(c, X1, Y1), b = modelRay(c, X0, Y0);
  return rotateHD(c.r, SphereVec{fSub(a.x, b.x), fSub(a.y, b.y), fSub(a.z, b.z)});
}

// The chart Jacobian of the equirect lookup u = atan2(x, z) / 2pi + 1/2, v = 1/2 - asin(y / |t|) / pi at t, applied to
// ray differential d, in level-0 pixels (the input eye re-pack's halving included):
//   du = su (z dx - x dz) / (x^2 + z^2),                         su = inW / 2pi
//   dv = sv (dy (x^2 + z^2) - y (x dx + z dz)) / (|t|^2 sqrt(x^2 + z^2)),  sv = inH / pi  (the sign is dropped)
// At a pole (x = z = 0) the quotients are infinite or NaN.
T360_HD void equirectJacobian(const SphereGeometry& g, const SphereVec& t, const SphereVec& d, float* du, float* dv) {
  const float su = fMul(static_cast<float>(g.inW), g.packLR ? 0.0795774715f : 0.159154943f);
  const float sv = fMul(static_cast<float>(g.inH), g.packTB ? 0.159154943f : 0.318309886f);
  const float h2 = fAdd(fMul(t.x, t.x), fMul(t.z, t.z));
  const float r2 = fAdd(h2, fMul(t.y, t.y));
  *du = fDiv(fMul(su, fSub(fMul(t.z, d.x), fMul(t.x, d.z))), h2);
  const float num = fSub(fMul(d.y, h2), fMul(t.y, fAdd(fMul(t.x, d.x), fMul(t.z, d.z))));
  *dv = fDiv(fMul(sv, num), fMul(r2, fSqrt(h2)));
}

// The face cubeInputHD picks for the normalised direction (tx, ty, tz), its tests written as there: 0..5, -1 for none
T360_HD int cubeInputFace(float tx, float ty, float tz) {
#pragma unroll 1
  for (int f = 0; f < 6; ++f) {
    const float major = f < 2 ? tz : (f < 4 ? tx : ty);
    const float a = f < 4 ? (f < 2 ? tx : tz) : tx, b = f < 4 ? ty : tz;
    if ((f & 1) == 0 ? !(major <= -0.5f) : !(major >= 0.5f)) continue;
    const float gx = fDiv(a, major), gy = fDiv(b, major);
    if (gx >= -1.0f && gx <= 1.0f && gy >= -1.0f && gy <= 1.0f) return f;
  }
  return -1;
}

// The chart Jacobian of the CUBEMAP_32 lookup on face f (the gnomonic quotient rule: d(a / m) = (da m - a dm) / m^2, with
// u = (col +- gx / e) / 6, v = (row +- gy / e) / 4), applied to d, in level-0 pixels
T360_HD void cubeJacobian(const SphereGeometry& g, int f, const SphereVec& t, const SphereVec& d, float* du, float* dv) {
  const float m = f < 2 ? t.z : (f < 4 ? t.x : t.y), dm = f < 2 ? d.z : (f < 4 ? d.x : d.y);
  const float a = f < 4 ? (f < 2 ? t.x : t.z) : t.x, da = f < 4 ? (f < 2 ? d.x : d.z) : d.x;
  const float b = f < 4 ? t.y : t.z, db = f < 4 ? d.y : d.z;
  const float m2 = fMul(m, m);
  const float su = fDiv(static_cast<float>(g.inW), fMul(g.packLR ? 12.0f : 6.0f, g.inputExpand));
  const float sv = fDiv(static_cast<float>(g.inH), fMul(g.packTB ? 8.0f : 4.0f, g.inputExpand));
  *du = fDiv(fMul(su, fSub(fMul(da, m), fMul(a, dm))), m2);
  *dv = fDiv(fMul(sv, fSub(fMul(db, m), fMul(b, dm))), m2);
}

// The Kannala-Brandt projection's Jacobian for lens L, applied to rx and ry, in level-0 pixels; Z = lensRow(L.m + 6, t),
// which the callers have already computed.  With rho = |(X, Y)|, theta = atan2(rho, Z), s = theta_d / rho (lensHit),
// theta_d'(theta) = 1 + 3 k1 t + 5 k2 t^2 + 7 k3 t^3 + 9 k4 t^4 (t = theta^2):
//   drho = (X dX + Y dY) / rho,  dtheta = (Z drho - rho dZ) / (rho^2 + Z^2),  ds = (theta_d' dtheta - s drho) / rho,
//   dx' = s dX + X ds,  dy' = s dY + Y ds,  a = (ax inW dx', ay inH dy').
// At rho = 0 (theta = 0 for Z > 0) the limit is dx' = dX / Z, dy' = dY / Z; on the back axis (Z <= 0) it is infinite.
T360_HD void lensJacobian(const LensModel& L, float Z, const SphereVec& t, const SphereVec& rx, const SphereVec& ry, int inW, int inH,
                          float* a, float* b) {
  const float X = lensRow(L.m, t), Y = lensRow(L.m + 3, t);
  const float cx = fMul(L.ax, static_cast<float>(inW)), cy = fMul(L.ay, static_cast<float>(inH));
  const float rho = fSqrt(fAdd(fMul(X, X), fMul(Y, Y)));
  const SphereVec* d[2] = {&rx, &ry};
  float* out[2] = {a, b};
  if (!(rho > 0.0f)) {
    const float inv = Z > 0.0f ? fDiv(1.0f, Z) : bitsFloat(0x7f800000u);
    for (int k = 0; k < 2; ++k) {
      out[k][0] = fMul(cx, fMul(lensRow(L.m, *d[k]), inv));
      out[k][1] = fMul(cy, fMul(lensRow(L.m + 3, *d[k]), inv));
    }
    return;
  }
  const float theta = libmAtan2f(rho, Z), tt = fMul(theta, theta);
  const float poly = fAdd(1.0f, fMul(tt, fAdd(L.k[0], fMul(tt, fAdd(L.k[1], fMul(tt, fAdd(L.k[2], fMul(tt, L.k[3]))))))));
  const float dpoly = fAdd(1.0f, fMul(tt, fAdd(fMul(3.0f, L.k[0]), fMul(tt, fAdd(fMul(5.0f, L.k[1]), fMul(tt, fAdd(fMul(7.0f, L.k[2]),
                                                                                                           fMul(tt, fMul(9.0f, L.k[3])))))))));
  const float s = fDiv(fMul(theta, poly), rho);
  const float q2 = fAdd(fMul(rho, rho), fMul(Z, Z));
  for (int k = 0; k < 2; ++k) {
    const float dX = lensRow(L.m, *d[k]), dY = lensRow(L.m + 3, *d[k]), dZ = lensRow(L.m + 6, *d[k]);
    const float drho = fDiv(fAdd(fMul(X, dX), fMul(Y, dY)), rho);
    const float dtheta = fDiv(fSub(fMul(Z, drho), fMul(rho, dZ)), q2);
    const float ds = fDiv(fSub(fMul(dpoly, dtheta), fMul(s, drho)), rho);
    out[k][0] = fMul(cx, fAdd(fMul(s, dX), fMul(X, ds)));
    out[k][1] = fMul(cy, fAdd(fMul(s, dY), fMul(Y, ds)));
  }
}

// ... for the lens lensPosition picks (the closer lens; ties to lens 0)
T360_HD void lensJacobian(const LensRigModel& rig, const SphereVec& t, const SphereVec& rx, const SphereVec& ry, int inW, int inH,
                          float* a, float* b) {
  const float z0 = lensRow(rig.lens[0].m + 6, t);
  const float z1 = rig.numLenses > 1 ? lensRow(rig.lens[1].m + 6, t) : z0;
  lensJacobian(z1 > z0 ? rig.lens[1] : rig.lens[0], z1 > z0 ? z1 : z0, t, rx, ry, inW, inH, a, b);
}

// lambda256 = ((int32) bits(rho^2) - 0x3f800000) >> 16 + bias256 (1/2 log2 rho^2 in 1/256 level, piecewise linear between
// powers of two), 256 T where rho^2 = max(aa, bb) is not below +inf; then the level clamp(lambda256 >> 8, 0, T) and the
// weight of the next level, lambda256 & 255 where 0 <= lambda256 < 256 T and 0 elsewhere.  Returns the level.
T360_HD int mipLevelOf(float aa, float bb, int top, int bias256, int* w) {
  const float inf = bitsFloat(0x7f800000u);
  int lam = 256 * top;
  if (aa < inf && bb < inf) lam = ((static_cast<int32_t>(floatBits(aa > bb ? aa : bb)) - 0x3f800000) >> 16) + bias256;
  *w = lam >= 0 && lam < 256 * top ? (lam & 255) : 0;
  const int level = lam >> 8;
  return level < 0 ? 0 : (level > top ? top : level);
}

// A level-0 position in level l's pixels, l >= 1: ((p + 0.5) s_l) - 0.5, each step rounded to float
T360_HD float mipScale(float p, float s) { return fSub(fMul(fAdd(p, 0.5f), s), 0.5f); }

// The footprint, level and map entries of output pixel (i, j) of an anti-aliased camera view: p0 = the camera view's entry
// (rectilinearPosition's bits) in level `level`'s pixels, p1 = the entry in level + 1's pixels (NaN where *w = 0).
// Returns the level.
template <bool LENS>
T360_HD int mipCameraPoint(const SphereGeometry& g, const RectilinearCamera& c, const LensRigModel& rig, const MipGeometry& m, int bias256,
                           int i, int j, float* p0, float* p1, int* w) {
  float X, Y;
  bool eye;
  cameraXY(g, i, j, &X, &Y, &eye);
  const SphereVec t = rotateHD(c.r, modelRay(c, X, Y));
  float px, py;
  if constexpr (LENS) {
    lensPosition(rig, t, g.inW, g.inH, &px, &py);
  } else {
    float u, v;
    sphereInputHD(g, false, eye, t, &u, &v);
    px = toPixel(u, g.inW);
    py = toPixel(v, g.inH);
  }
  int level = 0;
  *w = 0;
  if (m.top > 0) {
    const SphereVec rx = rayDifferential(c, fSub(X, m.halfX), Y, fAdd(X, m.halfX), Y);
    const SphereVec ry = rayDifferential(c, X, fSub(Y, m.halfY), X, fAdd(Y, m.halfY));
    float a[2], b[2];
    if constexpr (LENS) {
      lensJacobian(rig, t, rx, ry, g.inW, g.inH, a, b);
    } else if (g.cubeInput) {
      const float n = fSqrt(fAdd(fAdd(fMul(t.x, t.x), fMul(t.y, t.y)), fMul(t.z, t.z)));
      const int f = cubeInputFace(fDiv(t.x, n), fDiv(t.y, n), fDiv(t.z, n));
      const float nan = bitsFloat(0x7fc00000u);
      a[0] = a[1] = b[0] = b[1] = nan;
      if (f >= 0) {
        cubeJacobian(g, f, t, rx, &a[0], &a[1]);
        cubeJacobian(g, f, t, ry, &b[0], &b[1]);
      }
    } else {
      equirectJacobian(g, t, rx, &a[0], &a[1]);
      equirectJacobian(g, t, ry, &b[0], &b[1]);
    }
    level = mipLevelOf(fAdd(fMul(a[0], a[0]), fMul(a[1], a[1])), fAdd(fMul(b[0], b[0]), fMul(b[1], b[1])), m.top, bias256, w);
  }
  p0[0] = level ? mipScale(px, m.sx[level]) : px;
  p0[1] = level ? mipScale(py, m.sy[level]) : py;
  const float nan = bitsFloat(0x7fc00000u);
  p1[0] = *w ? mipScale(px, m.sx[level + 1]) : nan;
  p1[1] = *w ? mipScale(py, m.sy[level + 1]) : nan;
  return level;
}

// The sampling records of output pixel (i, j) of an anti-aliased camera view: mipCameraPoint's entries quantised as
// rectilinearSample quantises its entry (rec1 only where *w > 0).  Returns the level.
template <bool LENS>
T360_HD int mipCameraSample(const SphereGeometry& g, const RectilinearCamera& c, const LensRigModel& rig, const MipGeometry& m, int bias256,
                            int i, int j, int32_t* rec0, int32_t* rec1, int* w) {
  float p0[2], p1[2];
  const int level = mipCameraPoint<LENS>(g, c, rig, m, bias256, i, j, p0, p1, w);
  int r0, fracX, fracY;
  quantizeAxis(p0[0], g.kernelSize, &rec0[0], &fracX);
  quantizeAxis(p0[1], g.kernelSize, &r0, &fracY);
  rec0[1] = r0 * 1024 + fracY * 32 + fracX;
  if (*w) {
    quantizeAxis(p1[0], g.kernelSize, &rec1[0], &fracX);
    quantizeAxis(p1[1], g.kernelSize, &r0, &fracY);
    rec1[1] = r0 * 1024 + fracY * 32 + fracX;
  }
  return level;
}

// ---- anisotropic camera views (T360B200_cameraAnisoMaps, T360B200_transformFrameCameraAnisoAsync) --------------------
// The anti-aliased view's footprint a, b, read by N = 2^e probes spread along its longer screen axis (the column axis
// where a.a >= b.b, else the row axis), each probe at the level of max(long / N, short): the probes along the major axis
// of hardware anisotropic filtering (McCormack et al. 1999), with the longer screen-axis derivative in place of the
// ellipse's true major axis.  With N = 1 the probe is the centre ray, and the records are mipCameraSample's.
// (These are written beside mipCameraPoint rather than through it: built on a shared footprint step, the anti-aliased
// views' kernels compile to different SASS.)

// lambda256 of the longer and the shorter axis, L(x) = ((int32) bits(x) - 0x3f800000) >> 16 as mipLevelOf takes it;
// e = min(ceil((L(max) - L(min)) / 256), maxLog2), lambda256 = max(L(max) - 256 e, L(min)) + bias256, and the level and
// next-level weight from lambda256 as mipLevelOf takes them.  Where aa or bb is not below +inf (an exact pole, NaN),
// mipLevelOf itself with e = 0.  A zero or denormal axis gives e = maxLog2.  Returns the level.
T360_HD int anisoLevelOf(float aa, float bb, int top, int bias256, int maxLog2, int* w, int* e) {
  const float inf = bitsFloat(0x7f800000u);
  *e = 0;
  if (!(aa < inf && bb < inf)) return mipLevelOf(aa, bb, top, bias256, w);
  const int hi = (static_cast<int32_t>(floatBits(aa > bb ? aa : bb)) - 0x3f800000) >> 16;
  const int lo = (static_cast<int32_t>(floatBits(aa > bb ? bb : aa)) - 0x3f800000) >> 16;
  const int steps = (hi - lo + 255) >> 8;
  *e = steps < maxLog2 ? steps : maxLog2;
  const int shortened = hi - 256 * *e;
  const int lam = (shortened > lo ? shortened : lo) + bias256;
  *w = lam >= 0 && lam < 256 * top ? (lam & 255) : 0;
  const int level = lam >> 8;
  return level < 0 ? 0 : (level > top ? top : level);
}

// The centre of output pixel (i, j) of an anisotropic camera view and what its probes share: the footprint is taken
// wherever there is a pyramid or more than one probe (maxLog2 > 0), as mipCameraPoint takes it, else level 0, weight 0, e 0.
struct AnisoFootprint {
  float X, Y;       // the pixel's centre (cameraXY)
  SphereVec t;      // its rotated ray
  bool eye;         // its output eye
  bool rows;        // the probes lie along the row axis (Y), not the column axis (X)
  int level, w, e;  // the probes' level, the next level's weight (0..255), log2 of the probe count
};
template <bool LENS>
T360_HD AnisoFootprint anisoFootprint(const SphereGeometry& g, const RectilinearCamera& c, const LensRigModel& rig, const MipGeometry& m,
                                      int bias256, int maxLog2, int i, int j) {
  AnisoFootprint f{};
  cameraXY(g, i, j, &f.X, &f.Y, &f.eye);
  f.t = rotateHD(c.r, modelRay(c, f.X, f.Y));
  if (m.top > 0 || maxLog2 > 0) {
    const SphereVec& t = f.t;
    const SphereVec rx = rayDifferential(c, fSub(f.X, m.halfX), f.Y, fAdd(f.X, m.halfX), f.Y);
    const SphereVec ry = rayDifferential(c, f.X, fSub(f.Y, m.halfY), f.X, fAdd(f.Y, m.halfY));
    float a[2], b[2];
    if constexpr (LENS) {
      lensJacobian(rig, t, rx, ry, g.inW, g.inH, a, b);
    } else if (g.cubeInput) {
      const float n = fSqrt(fAdd(fAdd(fMul(t.x, t.x), fMul(t.y, t.y)), fMul(t.z, t.z)));
      const int face = cubeInputFace(fDiv(t.x, n), fDiv(t.y, n), fDiv(t.z, n));
      const float nan = bitsFloat(0x7fc00000u);
      a[0] = a[1] = b[0] = b[1] = nan;
      if (face >= 0) {
        cubeJacobian(g, face, t, rx, &a[0], &a[1]);
        cubeJacobian(g, face, t, ry, &b[0], &b[1]);
      }
    } else {
      equirectJacobian(g, t, rx, &a[0], &a[1]);
      equirectJacobian(g, t, ry, &b[0], &b[1]);
    }
    const float aa = fAdd(fMul(a[0], a[0]), fMul(a[1], a[1])), bb = fAdd(fMul(b[0], b[0]), fMul(b[1], b[1]));
    f.level = anisoLevelOf(aa, bb, m.top, bias256, maxLog2, &f.w, &f.e);
    f.rows = !(aa >= bb);
  }
  return f;
}

// The map entries of probe k (0..2^f.e - 1) of footprint f: p0 in level f.level's pixels, p1 in level + 1's (NaN where
// f.w = 0).  The probe's centre is X + o_k dX / 2 (or Y + o_k dY / 2 on the row axis), o_k = (2k + 1 - N) / N (exact for
// N a power of two), each step rounded to float; with N = 1 it is the pixel's centre ray as it is.  Each probe takes the
// camera view's whole lookup, so on cube-map input it picks its own face and on a rig its own closer lens.
template <bool LENS>
T360_HD void anisoCameraPoint(const SphereGeometry& g, const RectilinearCamera& c, const LensRigModel& rig, const MipGeometry& m,
                              const AnisoFootprint& f, int k, float* p0, float* p1) {
  SphereVec t = f.t;
  if (f.e > 0) {
    const int n = 1 << f.e;
    const float o = fDiv(static_cast<float>(2 * k + 1 - n), static_cast<float>(n));
    t = f.rows ? rotateHD(c.r, modelRay(c, f.X, fAdd(f.Y, fMul(o, m.halfY))))
               : rotateHD(c.r, modelRay(c, fAdd(f.X, fMul(o, m.halfX)), f.Y));
  }
  float px, py;
  if constexpr (LENS) {
    lensPosition(rig, t, g.inW, g.inH, &px, &py);
  } else {
    float u, v;
    sphereInputHD(g, false, f.eye, t, &u, &v);
    px = toPixel(u, g.inW);
    py = toPixel(v, g.inH);
  }
  p0[0] = f.level ? mipScale(px, m.sx[f.level]) : px;
  p0[1] = f.level ? mipScale(py, m.sy[f.level]) : py;
  const float nan = bitsFloat(0x7fc00000u);
  p1[0] = f.w ? mipScale(px, m.sx[f.level + 1]) : nan;
  p1[1] = f.w ? mipScale(py, m.sy[f.level + 1]) : nan;
}

// The sampling records of probe k: anisoCameraPoint's entries quantised as mipCameraSample quantises its entries (rec1
// only where f.w > 0)
template <bool LENS>
T360_HD void anisoCameraSample(const SphereGeometry& g, const RectilinearCamera& c, const LensRigModel& rig, const MipGeometry& m,
                               const AnisoFootprint& f, int k, int32_t* rec0, int32_t* rec1) {
  float p0[2], p1[2];
  anisoCameraPoint<LENS>(g, c, rig, m, f, k, p0, p1);
  int r0, fracX, fracY;
  quantizeAxis(p0[0], g.kernelSize, &rec0[0], &fracX);
  quantizeAxis(p0[1], g.kernelSize, &r0, &fracY);
  rec0[1] = r0 * 1024 + fracY * 32 + fracX;
  if (f.w) {
    quantizeAxis(p1[0], g.kernelSize, &rec1[0], &fracX);
    quantizeAxis(p1[1], g.kernelSize, &r0, &fracY);
    rec1[1] = r0 * 1024 + fracY * 32 + fracX;
  }
}

// ---- camera views of a lens rig with photometry (T360B200_cameraPhotoMaps, T360B200_transformFrameCameraPhotoAsync) ---
// The camera view's ray (cameraXY, modelRay, rotateHD: the rig is mono), then lensPhotoPosition as the photometric lens
// call applies it; with a pyramid each lens that covers the ray takes its own footprint from its own Kannala-Brandt
// Jacobian (lensJacobian of that lens), level (mipLevelOf) and entries (mipScale), as mipCameraPoint takes them for the
// closer lens.  So a belt pixel may gather up to four windows: two lenses x two levels.
// One lens's part of a pixel (cameraPhotoPoint): cameraMipMaps's four values for that lens and its gain
struct CameraPhotoLens {
  float p0[2], p1[2];  // the entry in level `level`'s pixels and in level + 1's (NaN where w = 0 or the lens is not used)
  int level, w;        // its level and the weight of the next (0, 0 where the lens is not used)
  int gain;            // Gq (lensGain; 0 where the lens does not cover the ray)
};
// ... quantised (cameraPhotoSample): {col0, rowPhase} at `level` and, where w > 0, at level + 1
struct CameraPhotoRecords {
  int32_t rec0[2], rec1[2];
  int level, w, gain;
};

// Both lenses' part of output pixel (i, j) of a camera view of a rig with photometry and the seam weight w (0..256) of
// lens 1 (the return value; lensPhotoPosition's s, both and c).  A lens is used where lensPhotoPosition gives it an entry
// (it covers the ray; with the hard seam and both = false the closer lens only).  MIP = false, or m.top = 0: no pyramid,
// every used lens at level 0 with weight 0.  With the identity photometry and s = 0 the closer lens's entries are
// cameraMipMaps' (cameraMap's without a pyramid) and its gain 4096.
// STEREO (a stereo rig, T360B200_transformFrameStereoCameraAsync; s = 0): the pixel's output eye e picks lens e, so w =
// 256 e; the other lens is projected only with both (the statistics).
template <bool MIP, bool STEREO = false>
T360_HD int cameraPhotoPoint(const SphereGeometry& g, const RectilinearCamera& c, const LensRigModel& rig, const MipGeometry& m, int bias256,
                             float s, bool both, const LensPhotoPlane& ph, int i, int j, CameraPhotoLens* lens, bool* overlap) {
  float X, Y;
  bool eye;
  cameraXY(g, i, j, &X, &Y, &eye);
  const SphereVec t = rotateHD(c.r, modelRay(c, X, Y));
  float p[2][2];
  const int w = lensPhotoPosition<STEREO>(rig, s, both, ph, t, g.inW, g.inH, p[0], p[1], &lens[0].gain, &lens[1].gain, overlap, eye);
  const bool used[2] = {p[0][0] == p[0][0], p[1][0] == p[1][0]};
  const bool footprint = MIP && m.top > 0 && (used[0] || used[1]);
  SphereVec rx{}, ry{};
  if (footprint) {
    rx = rayDifferential(c, fSub(X, m.halfX), Y, fAdd(X, m.halfX), Y);
    ry = rayDifferential(c, X, fSub(Y, m.halfY), X, fAdd(Y, m.halfY));
  }
  const float nan = bitsFloat(0x7fc00000u);
  for (int l = 0; l < 2; ++l) {
    CameraPhotoLens& e = lens[l];
    e.level = e.w = 0;
    if (footprint && used[l]) {
      float a[2], b[2];
      lensJacobian(rig.lens[l], lensRow(rig.lens[l].m + 6, t), t, rx, ry, g.inW, g.inH, a, b);
      e.level = mipLevelOf(fAdd(fMul(a[0], a[0]), fMul(a[1], a[1])), fAdd(fMul(b[0], b[0]), fMul(b[1], b[1])), m.top, bias256, &e.w);
    }
    e.p0[0] = e.level ? mipScale(p[l][0], m.sx[e.level]) : p[l][0];
    e.p0[1] = e.level ? mipScale(p[l][1], m.sy[e.level]) : p[l][1];
    e.p1[0] = e.w ? mipScale(p[l][0], m.sx[e.level + 1]) : nan;
    e.p1[1] = e.w ? mipScale(p[l][1], m.sy[e.level + 1]) : nan;
  }
  return w;
}

// The sampling records of output pixel (i, j): cameraPhotoPoint's entries quantised as mipCameraSample quantises its
// entries (rec1 only where w > 0).  Returns the seam weight w of lens 1.
template <bool MIP, bool STEREO = false>
T360_HD int cameraPhotoSample(const SphereGeometry& g, const RectilinearCamera& c, const LensRigModel& rig, const MipGeometry& m, int bias256,
                              float s, bool both, const LensPhotoPlane& ph, int i, int j, CameraPhotoRecords* lens, bool* overlap) {
  CameraPhotoLens e[2];
  const int w = cameraPhotoPoint<MIP, STEREO>(g, c, rig, m, bias256, s, both, ph, i, j, e, overlap);
  for (int l = 0; l < 2; ++l) {
    int r0, fracX, fracY;
    quantizeAxis(e[l].p0[0], g.kernelSize, &lens[l].rec0[0], &fracX);
    quantizeAxis(e[l].p0[1], g.kernelSize, &r0, &fracY);
    lens[l].rec0[1] = r0 * 1024 + fracY * 32 + fracX;
    if (e[l].w) {
      quantizeAxis(e[l].p1[0], g.kernelSize, &lens[l].rec1[0], &fracX);
      quantizeAxis(e[l].p1[1], g.kernelSize, &r0, &fracY);
      lens[l].rec1[1] = r0 * 1024 + fracY * 32 + fracX;
    }
    lens[l].level = e[l].level;
    lens[l].w = e[l].w;
    lens[l].gain = e[l].gain;
  }
  return w;
}

// ---- rolling-shutter lens rigs (T360B200_lensMotionMaps, T360B200_cameraMotionMaps and their frame calls) ---------------
// Each lens's M depends on the readout time t of the point it projects: M(t) = M_k + f (M_k+1 - M_k) between the sample
// matrices of the rig motion (the table: [numLenses][numSamples][9], computed on the host in double and stored as float,
// rigMotionTable in video_frame_transform.cpp), and t = clamp((a u + b v) + c, 0, 1) of the lens point's normalised
// calibration coordinates.  lensMotionHit solves t = readout(project(M(t) d)) by a fixed count of refinements from t =
// 0.5; everything else (the projection, the gain, the seam weight, the footprint) is the photometric calls' code with
// the lens's M replaced.  With all-zero deltas every table entry is the lens's own M and the interpolation returns it as
// it is, so the records are the photometric calls' bit for bit.
constexpr int kMotionMaxSamples = 16;
constexpr int kMotionProjections = 3;  // the fixed point refined twice
struct RigMotion {
  const float* table;      // [numLenses][numSamples][9]: M_ik (device memory in a launch, host memory in the twins)
  int numSamples;          // N, 2..16
  float readout[2][3];     // (a, b, c) of each lens
};

// A table entry: read-only global loads on the device (the table is at most 1152 bytes and stays in L1)
T360_HD float motionEntry(const float* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}

// Lens L with the M of readout time t (0..1) of lens `lens`: s = t (N - 1), k = min(floor(s), N - 2), f = s - k, each
// entry M_k + f (M_k+1 - M_k), or M_k itself where both neighbours hold the same value
T360_HD LensModel motionLens(const LensModel& L, const RigMotion& mo, int lens, float t) {
  const float s = fMul(t, static_cast<float>(mo.numSamples - 1));
  int k = truncToInt(s);
  k = k > mo.numSamples - 2 ? mo.numSamples - 2 : k;
  const float f = fSub(s, static_cast<float>(k));
  const float* a = mo.table + (lens * mo.numSamples + k) * 9;
  LensModel M = L;
#pragma unroll
  for (int e = 0; e < 9; ++e) {
    const float lo = motionEntry(a + e), hi = motionEntry(a + 9 + e);
    M.m[e] = lo == hi ? lo : fAdd(lo, fMul(f, fSub(hi, lo)));
  }
  return M;
}

// Z of rig direction d under lens `lens`'s M at t = 0.5: the hard seam's lens choice
T360_HD float motionZ(const LensModel& L, const RigMotion& mo, int lens, const SphereVec& d) {
  return lensRow(motionLens(L, mo, lens, 0.5f).m + 6, d);
}

// The readout time of where lens M projects d (h covers d): t = clamp((a u + b v) + c, 0, 1), with u, v the normalised
// calibration coordinates lensHit forms before toPixel (its s = theta_d / rho, recomputed from the hit's r = theta_d)
T360_HD float readoutTime(const LensModel& M, const LensHitR& h, const SphereVec& d, const float* r) {
  const float X = lensRow(M.m, d), Y = lensRow(M.m + 3, d);
  const float rho = fSqrt(fAdd(fMul(X, X), fMul(Y, Y)));
  const float s = rho > 0.0f ? fDiv(h.r, rho) : 0.0f;
  const float u = fAdd(fMul(M.ax, fMul(s, X)), M.bx), v = fAdd(fMul(M.ay, fMul(s, Y)), M.by);
  const float t = fAdd(fAdd(fMul(r[0], u), fMul(r[1], v)), r[2]);
  return t > 0.0f ? (t < 1.0f ? t : 1.0f) : 0.0f;
}

// Lens `lens` of the rig with the motion, for rig direction d: kMotionProjections projections, each with the M of the
// current readout time, which a covered hit moves to its own readout time.  Returns the last hit; *at: the lens with that
// hit's M (the footprint's lens).  *times (optional): the readout times the projections used.
T360_HD LensHitR lensMotionHit(const LensModel& L, const RigMotion& mo, int lens, const SphereVec& d, int inW, int inH, LensModel* at,
                               float* times = nullptr) {
  float t = 0.5f;
  LensHitR h;
#pragma unroll 1
  for (int n = 0; n < kMotionProjections; ++n) {
    if (times) times[n] = t;
    *at = motionLens(L, mo, lens, t);
    h = lensHit<true>(*at, d, lensRow(at->m + 6, d), inW, inH);
    if (h.covered) t = readoutTime(*at, h, d, mo.readout[lens]);
  }
  return h;
}

// lensPhotoPosition (not STEREO) with the motion: the hard seam picks the lens by Z under each lens's M at t = 0.5, and
// each projected lens is lensMotionHit's.  at[l]: lens l with its last M where it was projected (the footprint's lens).
T360_HD int lensMotionPosition(const LensRigModel& rig, const RigMotion& mo, float s, bool both, const LensPhotoPlane& c, const SphereVec& d,
                               int inW, int inH, float* p0, float* p1, int* g0, int* g1, bool* overlap, LensModel* at) {
  const float nan = bitsFloat(0x7fc00000u);
  const float z0 = motionZ(rig.lens[0], mo, 0, d);
  const float z1 = rig.numLenses > 1 ? motionZ(rig.lens[1], mo, 1, d) : z0;
  const bool second = z1 > z0;
  if (s == 0.0f && !both) {  // the closer lens alone
    const int l = second ? 1 : 0;
    const LensHitR h = lensMotionHit(rig.lens[l], mo, l, d, inW, inH, &at[l]);
    float* p = second ? p1 : p0;
    float* q = second ? p0 : p1;
    p[0] = h.px; p[1] = h.py;
    q[0] = q[1] = nan;
    *(second ? g1 : g0) = lensGain(h, c.v[l], c.gain[l]);
    *(second ? g0 : g1) = 0;
    *overlap = false;
    return second ? 256 : 0;
  }
  LensHitR h0 = lensMotionHit(rig.lens[0], mo, 0, d, inW, inH, &at[0]), h1;
  h1.covered = false;
  h1.px = h1.py = h1.r = nan;
  if (rig.numLenses > 1) h1 = lensMotionHit(rig.lens[1], mo, 1, d, inW, inH, &at[1]);
  int w = second ? 256 : 0;
  if (s > 0.0f) {
    w = h1.covered ? 256 : 0;
    if (h0.covered && h1.covered) w = seamWeight(h0.theta, h1.theta, s);
  }
  p0[0] = h0.px; p0[1] = h0.py;
  p1[0] = h1.px; p1[1] = h1.py;
  *g0 = lensGain(h0, c.v[0], c.gain[0]);
  *g1 = lensGain(h1, c.v[1], c.gain[1]);
  *overlap = h0.covered && h1.covered;
  return w;
}

// lensPhotoPoint with the motion (T360B200_lensMotionMaps)
template <bool BARREL = true>
T360_HD int lensMotionPoint(const SphereGeometry& g, const Rotation& r, const LensRigModel& rig, const RigMotion& mo, float s, bool both,
                            const LensPhotoPlane& c, const float* colTab, const float* rowTab, int i, int j, float* p0, float* p1, int* g0,
                            int* g1, bool* overlap) {
  bool eye;
  SphereVec d;
  if (!spherePoint<BARREL>(g, r, colTab, rowTab, i, j, &eye, &d)) {
    p0[0] = p0[1] = p1[0] = p1[1] = bitsFloat(0x7fc00000u);
    *g0 = *g1 = 0;
    *overlap = false;
    return 0;
  }
  LensModel at[2];
  return lensMotionPosition(rig, mo, s, both, c, d, g.inW, g.inH, p0, p1, g0, g1, overlap, at);
}

// lensPhotoSample with the motion (the kLensMotion kernels)
template <bool BARREL = true>
T360_HD int lensMotionSample(const SphereGeometry& g, const Rotation& r, const LensRigModel& rig, const RigMotion& mo, float s, bool both,
                             const LensPhotoPlane& c, const float* colTab, const float* rowTab, int i, int j, int32_t* rec0, int32_t* rec1,
                             int* g0, int* g1, bool* overlap) {
  float p[2][2];
  const int w = lensMotionPoint<BARREL>(g, r, rig, mo, s, both, c, colTab, rowTab, i, j, p[0], p[1], g0, g1, overlap);
  int32_t* rec[2] = {rec0, rec1};
  for (int l = 0; l < 2; ++l) {
    int r0, fracX, fracY;
    quantizeAxis(p[l][0], g.kernelSize, &rec[l][0], &fracX);
    quantizeAxis(p[l][1], g.kernelSize, &r0, &fracY);
    rec[l][1] = r0 * 1024 + fracY * 32 + fracX;
  }
  return w;
}

// cameraPhotoPoint (not STEREO) with the motion: the lenses from lensMotionPosition, and each used lens's footprint from
// lensJacobian of that lens with its last M (the motion's own stretch of the footprint is left out)
template <bool MIP>
T360_HD int cameraMotionPoint(const SphereGeometry& g, const RectilinearCamera& c, const LensRigModel& rig, const RigMotion& mo,
                              const MipGeometry& m, int bias256, float s, bool both, const LensPhotoPlane& ph, int i, int j, CameraPhotoLens* lens,
                              bool* overlap) {
  float X, Y;
  bool eye;
  cameraXY(g, i, j, &X, &Y, &eye);
  const SphereVec t = rotateHD(c.r, modelRay(c, X, Y));
  float p[2][2];
  LensModel at[2];
  const int w = lensMotionPosition(rig, mo, s, both, ph, t, g.inW, g.inH, p[0], p[1], &lens[0].gain, &lens[1].gain, overlap, at);
  const bool used[2] = {p[0][0] == p[0][0], p[1][0] == p[1][0]};
  const bool footprint = MIP && m.top > 0 && (used[0] || used[1]);
  SphereVec rx{}, ry{};
  if (footprint) {
    rx = rayDifferential(c, fSub(X, m.halfX), Y, fAdd(X, m.halfX), Y);
    ry = rayDifferential(c, X, fSub(Y, m.halfY), X, fAdd(Y, m.halfY));
  }
  const float nan = bitsFloat(0x7fc00000u);
  for (int l = 0; l < 2; ++l) {
    CameraPhotoLens& e = lens[l];
    e.level = e.w = 0;
    if (footprint && used[l]) {
      float a[2], b[2];
      lensJacobian(at[l], lensRow(at[l].m + 6, t), t, rx, ry, g.inW, g.inH, a, b);
      e.level = mipLevelOf(fAdd(fMul(a[0], a[0]), fMul(a[1], a[1])), fAdd(fMul(b[0], b[0]), fMul(b[1], b[1])), m.top, bias256, &e.w);
    }
    e.p0[0] = e.level ? mipScale(p[l][0], m.sx[e.level]) : p[l][0];
    e.p0[1] = e.level ? mipScale(p[l][1], m.sy[e.level]) : p[l][1];
    e.p1[0] = e.w ? mipScale(p[l][0], m.sx[e.level + 1]) : nan;
    e.p1[1] = e.w ? mipScale(p[l][1], m.sy[e.level + 1]) : nan;
  }
  return w;
}

// cameraPhotoSample with the motion (the kCameraMotion kernels)
template <bool MIP>
T360_HD int cameraMotionSample(const SphereGeometry& g, const RectilinearCamera& c, const LensRigModel& rig, const RigMotion& mo,
                               const MipGeometry& m, int bias256, float s, bool both, const LensPhotoPlane& ph, int i, int j,
                               CameraPhotoRecords* lens, bool* overlap) {
  CameraPhotoLens e[2];
  const int w = cameraMotionPoint<MIP>(g, c, rig, mo, m, bias256, s, both, ph, i, j, e, overlap);
  for (int l = 0; l < 2; ++l) {
    int r0, fracX, fracY;
    quantizeAxis(e[l].p0[0], g.kernelSize, &lens[l].rec0[0], &fracX);
    quantizeAxis(e[l].p0[1], g.kernelSize, &r0, &fracY);
    lens[l].rec0[1] = r0 * 1024 + fracY * 32 + fracX;
    if (e[l].w) {
      quantizeAxis(e[l].p1[0], g.kernelSize, &lens[l].rec1[0], &fracX);
      quantizeAxis(e[l].p1[1], g.kernelSize, &r0, &fracY);
      lens[l].rec1[1] = r0 * 1024 + fracY * 32 + fracX;
    }
    lens[l].level = e[l].level;
    lens[l].w = e[l].w;
    lens[l].gain = e[l].gain;
  }
  return w;
}

// Whether the per-frame orientation chain covers the layouts of `ctx`
inline bool orientedLayouts(const FrameTransformContext& ctx) {
  const int o = ctx.output_layout, in = ctx.input_layout;
  return (o == LAYOUT_CUBEMAP_32 || o == LAYOUT_CUBEMAP_23_OFFCENTER || o == LAYOUT_EAC_32 || o == LAYOUT_EQUIRECT) &&
         (in == LAYOUT_EQUIRECT || in == LAYOUT_CUBEMAP_32);
}

}  // namespace t360
