// Host-side planning for the projection-remap hot path.  Pure C++17, no CUDA, no OpenCV.
//
// Everything the reference computes once per stream in VideoFrameTransform::generateMapForPlane
// (reference VideoFrameTransform.cpp:504-576) is produced here: the per-pixel source coordinates,
// their fixed-point form as cv::remap consumes them, the segmented low-pass tile table with its
// Gaussian taps, and the fixed-point interpolation weight tables.  All float arithmetic follows the
// reference's rounding sequence (compile with -ffp-contract=off; see geometry.cpp).
#pragma once

#include <cstdint>
#include <vector>

#include "Transform360/VideoFrameTransformHelper.h"

namespace t360 {

// One rectangle of the input plane with its own separable Gaussian
// (reference SegmentFilteringConfig, VideoFrameTransform.h:25-38, plus filterKernelsX_/Y_).
struct LowPassSegment {
  int left, top, width, height;
  int kxOffset, kxCount;  // into HostPlan::taps
  int kyOffset, kyCount;
};

// Sampling record per output pixel, 8 bytes.  col0 = first tap column before wrapping
// (= sat16(X >> 5) - (k/2 - 1), or the rounded column for nearest); rowPhase = (row0 << 10) | phase.
struct SamplePoint {
  int32_t col0;
  int32_t rowPhase;
};

// cv::resize(INTER_AREA) from the render size (mapW x mapH) down to the requested output size, used when
// width/height_scale_factor != 1 (reference cpp:755-777).  Integer ratios average whole cells; other ratios weight
// partially covered source pixels with the tables OpenCV's computeResizeAreaTab produces.
struct AreaTap {
  int src;      // source column / row
  float alpha;  // its share of the destination cell
};
struct AreaAxis {
  std::vector<AreaTap> taps;   // grouped by destination index, in OpenCV's order
  std::vector<int> first;      // [dst + 1]: taps of destination i are taps[first[i] .. first[i+1])
};
// One axis of cv::resize(INTER_AREA) when at least one axis ENLARGES (a scale factor below 1): OpenCV runs its 8-bit
// fixed-point bilinear kernel with "area mode" coefficients on both axes.  Destination d reads source ofs[d] and
// ofs[d] + 1 with the 11-bit weights coef[2d], coef[2d + 1]; from d == dmax on only source ofs[d] (weight 2048).
struct AreaLinearAxis {
  std::vector<int> ofs;
  std::vector<int16_t> coef;
  int dmax = 0;
};
struct AreaResizePlan {
  bool needed = false;
  bool enlarge = false;      // the bilinear variant (lx, ly) instead of the area tables
  int srcW = 0, srcH = 0, dstW = 0, dstH = 0;
  int cellW = 0, cellH = 0;  // > 0: both ratios are integers (fast path), else use the axes below
  AreaAxis x, y;
  AreaLinearAxis lx, ly;
};

struct HostPlan {
  FrameTransformContext ctx{};
  int inW = 0, inH = 0;
  int outW = 0, outH = 0;   // as requested by the caller
  int mapW = 0, mapH = 0;   // scaled output size (== outW x outH unless *_scale_factor != 1)
  int kernelSize = 0;       // 1, 2, 4, 8 taps per axis
  bool transparentBorder = false;  // barrel layouts (reference cpp:716-719), or a caller's warp map with BORDER_TRANSPARENT
  bool warp = false;               // map is a caller's warp map (buildWarpHostPlan): ctx contributes its interpolation only
  std::vector<float> map;          // [mapH][mapW][2]
  std::vector<SamplePoint> samples;  // [mapH][mapW]
  std::vector<LowPassSegment> segments;
  std::vector<float> taps;
  AreaResizePlan resize;
};

// Geometry: fills plan.map (reference cpp:534-556).  Multi-threaded over rows.  false if the layout is invalid.
bool buildWarpMap(HostPlan& plan);
// Single point, exposed for tests (reference transformPos, cpp:893-1316).
bool projectPoint(const FrameTransformContext& ctx, float x, float y, float inputPixelWidth, float* outX, float* outY);

// Fixed-point conversion of plan.map exactly as cv::remap does it for a CV_32FC2 map (SURVEY.md Appendix A).
void quantizeWarpMap(HostPlan& plan);

// Low-pass plan: fills plan.segments / plan.taps (reference calcualteFilteringConfig, cpp:367-501).
bool buildLowPassPlan(HostPlan& plan);

// OpenCV's INTER_* fixed-point tables: int16 [1024][k][k], built once per process.  Returns k.
int remapTable(int interpolationAlg, const int16_t** table);
inline int kernelSizeOf(int interpolationAlg) {
  switch (interpolationAlg) {
    case NEAREST: return 1;
    case LINEAR: return 2;
    case CUBIC: return 4;
    case LANCZOS4: return 8;
    default: return 0;
  }
}

// cv::resize(INTER_AREA) from srcW x srcH to dstW x dstH (reference cpp:770-776).
void buildAreaResize(int srcW, int srcH, int dstW, int dstH, AreaResizePlan& r);
// Fills plan.resize for (mapW x mapH) -> (outW x outH).
void buildAreaResizePlan(HostPlan& plan);

// Whole plan for one plane; returns false (message on stdout) on invalid parameters.
bool buildHostPlan(const FrameTransformContext& ctx, int inW, int inH, int outW, int outH, HostPlan& plan);

// cv::remap's border modes a caller's warp map may use (OpenCV's values)
constexpr int kBorderWrap = 3, kBorderTransparent = 5;
// The largest warp map per axis: pole-cap records hold 16-bit output positions.
constexpr int kMaxWarpMapSide = 65536;
// Whole plan for one plane from a caller's CV_32FC2 map [mapH][mapW][2] (host memory) instead of the context's geometry:
// the map is sampled from an inW x inH plane with ctx's interpolation and `border`, rendered at mapW x mapH (outW x outH
// = the map's size), without low-pass.  Returns false (message on stdout) for a null map, non-positive sizes, a map side
// above kMaxWarpMapSide, a border other than kBorderWrap / kBorderTransparent, an unknown interpolation_alg and low-pass
// on (the reference derives its segments from the output layout, which a caller's map does not have).
bool buildWarpHostPlan(const FrameTransformContext& ctx, const float* map, int mapW, int mapH, int inW, int inH, int border,
                       HostPlan& plan);

}  // namespace t360
