// FLAT_FIXED output position, one definition for the host planner and the per-view gather kernel.
//
// For output pixel (i, j) of an mapW x mapH FLAT_FIXED map, the planner computes (reference cpp:537-545, 903-931,
// 1265-1300, and cv::remap's quantisation, SURVEY.md Appendix A):
//   x = (j + 0.5f) / W, y = (i + 0.5f) / H  ->  output eye split  ->  flat window (lon, lat), folded once over a pole and
//   wrapped around the seam  ->  input eye re-pack  ->  u * inW - 0.5f, v * inH - 0.5f  ->  1/32-pixel quantisation.
// Every step is an IEEE-rounded float + - * / and no libm call, so the device can reproduce the planner bit for bit if
// nothing is contracted into an FMA: on the device each operation below is an explicit __f*_rn intrinsic (nvcc contracts
// by default and the library is compiled in one command), on the host a plain operator (host code is compiled with
// -ffp-contract=off).  geometry.cpp (Projector::flatWindow, the eye split and re-pack, the map loop) and sampling.cpp
// (quantizeWarpMap) call these functions, so the planner and the kernel cannot drift apart.
//
// The chain separates by axis: the source column and its phase depend on the output column, the eye and whether the pixel
// lies beyond a pole (fold); the source row and its phase on the output row and the eye.  flatColumn / flatRow are those
// two halves; flatSample puts them together for one pixel.
#pragma once

#include <cmath>
#include <cstdint>

#ifdef __CUDACC__
#define T360_HD __host__ __device__ __forceinline__
#else
#define T360_HD inline
#endif

namespace t360 {

struct FlatView {
  float yaw, pitch, hfov, vfov;  // degrees, as FrameTransformContext::fixed_*
};

// Everything a position chain needs besides its per-frame constants (oriented_view.h: sphereGeometry).  The FLAT_FIXED
// chain reads the map (scaled output) size, the input plane size, the kernel size and the stereo fields.
struct SphereGeometry {
  int mapW, mapH, inW, inH;
  int kernelSize;            // 1 (nearest), 2, 4, 8
  bool splitLR, splitTB;     // the output holds two eyes side by side / stacked (only when the input is stereo)
  bool vflip;
  bool packLR, packTB;       // the input holds two eyes side by side / stacked
  bool cubeInput;            // input_layout CUBEMAP_32 (else treated as EQUIRECT, as the planner does)
  bool offCentre, horizontalOffset;
  int outputLayout;
  float expand, inputExpand;  // expand_coef, input_expand_coef
  float ox, oy, oz;           // fixed_cube_offcenter_*
  float inPixelWidth;         // 1.0f / inW, doubled for a side-by-side input: barrel outputs keep u half of it clear of 0 and 1
};

T360_HD float fAdd(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
T360_HD float fSub(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
T360_HD float fMul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
T360_HD float fDiv(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}

// static_cast<int>(float) as x86 does it (cvttss2si): truncation, INT_MIN ("integer indefinite") for NaN and values outside
// the int range.  The device's conversion saturates instead, so the range is checked explicitly there.
T360_HD int truncToInt(float v) {
#ifdef __CUDA_ARCH__
  if (!(v > -2147483904.0f && v < 2147483648.0f)) return INT32_MIN;
  return __float2int_rz(v);
#else
  return static_cast<int>(v);
#endif
}

// cvRound(float) as OpenCV computes it on x86 (cvtss2si, also in its SIMD paths): round half to even in the default FP
// environment, and INT_MIN ("integer indefinite") for NaN and for values outside the int range.  It matters: an
// off-centre projection with is_horizontal_offset divides by zero at the poles (reference cpp:1203-1206), the map holds
// NaN there, and cv::remap samples column / row sat16(INT_MIN >> 5) = -32768 under BORDER_WRAP; a huge FLAT_FIXED pitch
// or vfov leaves lat outside [0, 1] after the single fold, with the same effect.  (__float2int_rn saturates.)
T360_HD int roundHalfEven(float v) {
  if (!(v >= -2147483648.0f && v < 2147483648.0f)) return INT32_MIN;
#ifdef __CUDA_ARCH__
  return __float2int_rn(v);
#else
  return static_cast<int>(std::lrintf(v));
#endif
}
T360_HD int clampToShort(int v) { return v < -32768 ? -32768 : (v > 32767 ? 32767 : v); }

// x = (j + 0.5f) / W (reference cpp:537-538)
T360_HD float pixelCentre(int j, int n) { return fDiv(fAdd(static_cast<float>(j), 0.5f), static_cast<float>(n)); }

// Output eye split (reference cpp:903-931), one axis: a stereo output holds two complete projections; fold the coordinate
// to one and return the eye.  (Only one axis is split: LR folds x, TB folds y with the optional flip.)
T360_HD bool splitEye(float& t, bool flip) {
  if (t > 0.5f) {
    t = fDiv(fSub(t, 0.5f), 0.5f);
    if (flip) t = fSub(1.0f, t);
    return true;
  }
  t = fDiv(t, 0.5f);
  return false;
}

// The flat window (reference cpp:1265-1271) with normalize_equirectangular (cpp:101-123), split into its two halves.
// lat: returns the latitude after the single fold over a pole, and whether it folded.
T360_HD float flatLat(const FlatView& v, float y, bool* fold) {
  float lat = fAdd(fDiv(fSub(fMul(fSub(y, 0.5f), v.vfov), v.pitch), 180.0f), 0.5f);
  *fold = true;
  if (lat >= 1.0f) return fSub(2.0f, lat);
  if (lat < 0.0f) return -lat;
  *fold = false;
  return lat;
}
// lon: half a turn more when the latitude folded, then wrapped once into [0, 1)
T360_HD float flatLon(const FlatView& v, float x, bool fold) {
  float lon = fAdd(fDiv(fAdd(fMul(fSub(x, 0.5f), v.hfov), v.yaw), 360.0f), 0.5f);
  if (fold) lon = fAdd(lon, 0.5f);
  if (lon >= 1.0f) lon = fSub(lon, static_cast<float>(truncToInt(lon)));
  else if (lon < 0.0f) lon = fAdd(lon, static_cast<float>(truncToInt(-lon) + 1));
  return lon;
}

// Input eye re-pack (reference cpp:1278-1300), one axis: the second eye lives in the other half of the input.
T360_HD float packEye(float t, bool secondEye) { return secondEye ? fAdd(fMul(t, 0.5f), 0.5f) : fMul(t, 0.5f); }

// u * inW - 0.5f: pixel centres sit at integers for the sampler (reference cpp:544-545)
T360_HD float toPixel(float u, int n) { return fSub(fMul(u, static_cast<float>(n)), 0.5f); }

// cv::remap's quantisation of one coordinate of a CV_32FC2 map (sampling.cpp: quantizeWarpMap): *first = the first tap
// (column or row) before wrapping, *frac = its 1/32 phase (0 for nearest).
T360_HD void quantizeAxis(float f, int k, int* first, int* frac) {
  if (k == 1) {
    *first = clampToShort(roundHalfEven(f));
    *frac = 0;
    return;
  }
  const int q = roundHalfEven(fMul(f, 32.0f));
  *first = clampToShort(q >> 5) - (k / 2 - 1);
  *frac = q & 31;
}

// The column half of output pixel column j: source column and phase for the given fold and eye.  Returns the eye the
// column itself selects (a side-by-side output); *colEye is meaningless otherwise.
struct FlatColumn {
  int col0, fracX;
};
T360_HD FlatColumn flatColumn(const FlatView& v, const SphereGeometry& g, int j, bool fold, bool eye) {
  float x = pixelCentre(j, g.mapW);
  if (g.splitLR) eye = splitEye(x, false);
  float u = flatLon(v, x, fold);
  if (g.packLR) u = packEye(u, eye);
  FlatColumn c;
  quantizeAxis(toPixel(u, g.inW), g.kernelSize, &c.col0, &c.fracX);
  return c;
}
T360_HD bool flatColumnEye(const SphereGeometry& g, int j) {
  float x = pixelCentre(j, g.mapW);
  return g.splitLR && splitEye(x, false);
}

// The row half of output row i: rowPart = first tap row << 10 | fracY << 5 (add fracX for the record's rowPhase), whether
// the row lies beyond a pole, and the eye the row itself selects (a stacked output).
struct FlatRow {
  int rowPart;
  bool fold, eye;
};
T360_HD FlatRow flatRow(const FlatView& v, const SphereGeometry& g, int i, bool columnEye) {
  float y = pixelCentre(i, g.mapH);
  FlatRow r;
  r.eye = g.splitTB ? splitEye(y, g.vflip) : columnEye;
  float lat = flatLat(v, y, &r.fold);
  if (g.packTB) lat = packEye(lat, r.eye);
  int row0, fracY;
  quantizeAxis(toPixel(lat, g.inH), g.kernelSize, &row0, &fracY);
  r.rowPart = row0 * 1024 + (fracY << 5);
  return r;
}

// The sampling record {col0, rowPhase} of output pixel (i, j), as HostPlan::samples holds it.
T360_HD void flatSample(const FlatView& v, const SphereGeometry& g, int i, int j, int32_t* col0, int32_t* rowPhase) {
  const bool colEye = flatColumnEye(g, j);
  const FlatRow r = flatRow(v, g, i, colEye);
  const FlatColumn c = flatColumn(v, g, j, r.fold, r.eye);
  *col0 = c.col0;
  *rowPhase = r.rowPart + c.fracX;
}

}  // namespace t360
