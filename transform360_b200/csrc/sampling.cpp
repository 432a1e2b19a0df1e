// Fixed-point sampling plan: turns the float warp map into what the gather kernels consume, and builds
// the interpolation weight tables.  The arithmetic to be reproduced is OpenCV's cv::remap for an 8-bit
// source with a CV_32FC2 map (the call at reference VideoFrameTransform.cpp:748-754); OpenCV is an
// external, un-pinned dependency of the reference (CMakeLists.txt:11), its published algorithm is
// restated in SURVEY.md Appendix A and pinned against cv2 4.13.0 in tests/test_oracle_pin.py:
//   * coordinates are quantised to 1/32 pixel with round-half-even, integer parts saturate to int16;
//   * a k x k window (k = 2, 4, 8) is weighted with 15-bit fixed-point products of two 1-D kernels,
//     each 2-D entry rounded separately and the window patched so that it sums to exactly 32768;
//   * the result is (sum + 16384) >> 15, saturated to 8 bits.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#include "flat_view.h"
#include "host_plan.h"

namespace t360 {
namespace {

constexpr int kFracBits = 5, kPhases1D = 1 << kFracBits, kPhases2D = kPhases1D * kPhases1D;
constexpr int kWeightOne = 1 << 15;
// (roundHalfEven, cvRound as OpenCV computes it on x86, and clampToShort: flat_view.h)

// 1-D interpolation kernels at offset t in [0,1): taps for positions -(k/2-1) .. k/2
void taps1D(int k, float t, float* w) {
  if (k == 2) {
    w[0] = 1.f - t;
    w[1] = t;
  } else if (k == 4) {  // Keys cubic, a = -0.75
    const float a = -0.75f;
    w[0] = ((a * (t + 1) - 5 * a) * (t + 1) + 8 * a) * (t + 1) - 4 * a;
    w[1] = ((a + 2) * t - (a + 3)) * t * t + 1;
    w[2] = ((a + 2) * (1 - t) - (a + 3)) * (1 - t) * (1 - t) + 1;
    w[3] = 1.f - w[0] - w[1] - w[2];
  } else {  // Lanczos a = 4, evaluated through the angle-addition form OpenCV uses
    if (t < FLT_EPSILON) {
      for (int i = 0; i < 8; ++i) w[i] = 0;
      w[3] = 1;
      return;
    }
    const double r = 0.70710678118654752440084436210485;
    const double rot[8][2] = {{1, 0}, {-r, -r}, {0, 1}, {r, -r}, {-1, 0}, {r, r}, {0, -1}, {-r, r}};
    const double phi0 = -(t + 3) * M_PI * 0.25, s0 = std::sin(phi0), c0 = std::cos(phi0);
    float total = 0;
    for (int i = 0; i < 8; ++i) {
      const double phi = -(t + 3 - i) * M_PI * 0.25;
      w[i] = static_cast<float>((rot[i][0] * s0 + rot[i][1] * c0) / (phi * phi));
      total += w[i];
    }
    total = 1.f / total;
    for (int i = 0; i < 8; ++i) w[i] *= total;
  }
}

std::unique_ptr<int16_t[]> buildTable(int k) {
  std::unique_ptr<int16_t[]> tab(new int16_t[static_cast<size_t>(kPhases2D) * k * k]());
  float oneD[kPhases1D * 8];
  const float step = 1.f / kPhases1D;
  for (int p = 0; p < kPhases1D; ++p) taps1D(k, p * step, oneD + p * k);
  for (int py = 0; py < kPhases1D; ++py)
    for (int px = 0; px < kPhases1D; ++px) {
      int16_t* cell = tab.get() + static_cast<size_t>(py * kPhases1D + px) * k * k;
      int total = 0;
      for (int r = 0; r < k; ++r) {
        const float wy = oneD[py * k + r];
        for (int c = 0; c < k; ++c) {
          const float w = wy * oneD[px * k + c];
          total += cell[r * k + c] = static_cast<int16_t>(clampToShort(roundHalfEven(w * kWeightOne)));
        }
      }
      if (total == kWeightOne) continue;
      const int excess = total - kWeightOne;
      if (k == 2) {
        // only the (0,0) phase: weight 1.0 saturates to 32767 and OpenCV's patch lands on entry (1,1)
        cell[3] = static_cast<int16_t>(cell[3] - excess);
        continue;
      }
      // patch the largest (deficit) or smallest (excess) entry of the 2x2 block at [k/2, k/2+2)^2
      const int h = k / 2;
      int hiR = h, hiC = h, loR = h, loC = h;
      for (int r = h; r < h + 2; ++r)
        for (int c = h; c < h + 2; ++c) {
          if (cell[r * k + c] < cell[loR * k + loC]) { loR = r; loC = c; }
          else if (cell[r * k + c] > cell[hiR * k + hiC]) { hiR = r; hiC = c; }
        }
      if (excess < 0) cell[hiR * k + hiC] = static_cast<int16_t>(cell[hiR * k + hiC] - excess);
      else cell[loR * k + loC] = static_cast<int16_t>(cell[loR * k + loC] - excess);
    }
  return tab;
}

}  // namespace

int remapTable(int interpolationAlg, const int16_t** table) {
  static std::mutex mu;
  static std::unique_ptr<int16_t[]> cache[9];
  const int k = kernelSizeOf(interpolationAlg);
  if (k < 2) {
    if (table) *table = nullptr;
    return k;
  }
  std::lock_guard<std::mutex> lock(mu);
  if (!cache[k]) cache[k] = buildTable(k);
  if (table) *table = cache[k].get();
  return k;
}

void quantizeWarpMap(HostPlan& plan) {
  const int k = plan.kernelSize;
  const size_t n = static_cast<size_t>(plan.mapW) * plan.mapH;
  plan.samples.resize(n);
  const float* m = plan.map.data();
  // independent per pixel: rows are split over up to 32 host threads like the warp map itself
  unsigned nt = std::thread::hardware_concurrency();
  if (nt == 0) nt = 1;
  if (nt > 32) nt = 32;
  if (n < (1u << 16)) nt = 1;
  const size_t chunk = (n + nt - 1) / nt;
  auto range = [&plan, m, k](size_t begin, size_t end) {
  for (size_t i = begin; i < end; ++i) {
    // per axis (flat_view.h, shared with the per-view kernel): sat16(round(f * 32) >> 5) - (k/2 - 1) and the 1/32 phase
    int col0, fracX, row0, fracY;
    quantizeAxis(m[2 * i], k, &col0, &fracX);
    quantizeAxis(m[2 * i + 1], k, &row0, &fracY);
    plan.samples[i] = SamplePoint{col0, row0 * 1024 + fracY * kPhases1D + fracX};
  }
  };
  std::vector<std::thread> pool;
  for (unsigned t = 1; t < nt; ++t)
    if (t * chunk < n) pool.emplace_back(range, t * chunk, std::min(n, (t + 1) * chunk));
  range(0, std::min(n, chunk));
  for (auto& th : pool) th.join();
}

namespace {
// OpenCV 4.x imgproc/resize.cpp computeResizeAreaTab, one axis
AreaAxis areaAxis(int ssize, int dsize, double scale) {
  AreaAxis a;
  a.first.reserve(static_cast<size_t>(dsize) + 1);
  for (int d = 0; d < dsize; ++d) {
    a.first.push_back(static_cast<int>(a.taps.size()));
    const double f1 = d * scale, f2 = f1 + scale;
    const double cell = std::min(scale, ssize - f1);
    int s1 = static_cast<int>(std::ceil(f1)), s2 = static_cast<int>(std::floor(f2));
    s2 = std::min(s2, ssize - 1);
    s1 = std::min(s1, s2);
    if (s1 - f1 > 1e-3) a.taps.push_back(AreaTap{s1 - 1, static_cast<float>((s1 - f1) / cell)});
    for (int sx = s1; sx < s2; ++sx) a.taps.push_back(AreaTap{sx, static_cast<float>(1.0 / cell)});
    if (f2 - s2 > 1e-3) a.taps.push_back(AreaTap{s2, static_cast<float>(std::min(std::min(f2 - s2, 1.), cell) / cell)});
  }
  a.first.push_back(static_cast<int>(a.taps.size()));
  return a;
}
}  // namespace

namespace {
// OpenCV 4.x imgproc/resize.cpp, the INTER_LINEAR set-up with its "area mode" coefficients (interpolation ==
// INTER_AREA, scale < 1 on some axis): sx = floor(dx * scale); fx = (dx + 1) - (sx + 1) * inv_scale, 0 if not positive,
// else its fractional part; clamped at the last source sample; weights = cvRound({1 - fx, fx} * 2048).  Pinned
// bit-exact against cv2 4.13 through the oracle (tests/test_oracle_pin.py).
AreaLinearAxis areaLinearAxis(int dn, int sn, double scale, double inv) {
  AreaLinearAxis a;
  a.ofs.resize(static_cast<size_t>(dn));
  a.coef.resize(static_cast<size_t>(dn) * 2);
  a.dmax = dn;
  for (int d = 0; d < dn; ++d) {
    int s = static_cast<int>(std::floor(d * scale));
    float f = static_cast<float>((d + 1) - (s + 1) * inv);
    f = f <= 0 ? 0.f : f - static_cast<float>(std::floor(f));
    if (s < 0) { f = 0; s = 0; }
    if (s + 1 >= sn) {
      a.dmax = std::min(a.dmax, d);
      if (s >= sn - 1) { f = 0; s = sn - 1; }
    }
    a.ofs[d] = s;
    const long c0 = std::lrintf((1.f - f) * 2048.f), c1 = std::lrintf(f * 2048.f);
    a.coef[2 * d] = static_cast<int16_t>(std::min(c0, 32767l));
    a.coef[2 * d + 1] = static_cast<int16_t>(std::min(c1, 32767l));
  }
  return a;
}
}  // namespace

void buildAreaResize(int srcW, int srcH, int dstW, int dstH, AreaResizePlan& r) {
  r = AreaResizePlan{};
  r.srcW = srcW; r.srcH = srcH; r.dstW = dstW; r.dstH = dstH;
  r.needed = r.srcW != r.dstW || r.srcH != r.dstH;  // reference cpp:735-737
  if (!r.needed) return;
  // cv::resize: scale = 1. / ((double)dsize / ssize); INTER_AREA takes the area paths only when shrinking both ways
  const double invX = static_cast<double>(r.dstW) / r.srcW, invY = static_cast<double>(r.dstH) / r.srcH;
  const double sx = 1.0 / invX, sy = 1.0 / invY;
  if (sx < 1.0 || sy < 1.0) {
    r.enlarge = true;
    r.lx = areaLinearAxis(r.dstW, r.srcW, sx, invX);
    r.ly = areaLinearAxis(r.dstH, r.srcH, sy, invY);
    return;
  }
  const int ix = static_cast<int>(std::lrint(sx)), iy = static_cast<int>(std::lrint(sy));
  if (std::abs(sx - ix) < DBL_EPSILON && std::abs(sy - iy) < DBL_EPSILON) {
    r.cellW = ix; r.cellH = iy;
    return;
  }
  r.x = areaAxis(r.srcW, r.dstW, sx);
  r.y = areaAxis(r.srcH, r.dstH, sy);
}

void buildAreaResizePlan(HostPlan& plan) { buildAreaResize(plan.mapW, plan.mapH, plan.outW, plan.outH, plan.resize); }

namespace {
// What every plan does with its float map: the fixed-point records (when there is an interpolator) and the area resize.
void samplePlan(HostPlan& plan) {
  if (plan.kernelSize > 0) quantizeWarpMap(plan);
  buildAreaResizePlan(plan);
}
}  // namespace

bool buildWarpHostPlan(const FrameTransformContext& ctx, const float* map, int mapW, int mapH, int inW, int inH, int border,
                       HostPlan& plan) {
  plan = HostPlan{};
  plan.ctx = ctx;
  const char* why = nullptr;
  if (!map) why = "the map is NULL";
  else if (mapW <= 0 || mapH <= 0 || inW <= 0 || inH <= 0) why = "non-positive map or input size";
  else if (mapW > kMaxWarpMapSide || mapH > kMaxWarpMapSide) why = "the map is larger than 65536 in a dimension";
  else if (border != kBorderWrap && border != kBorderTransparent) why = "border must be 3 (BORDER_WRAP) or 5 (BORDER_TRANSPARENT)";
  else if (kernelSizeOf(ctx.interpolation_alg) == 0) why = "unknown interpolation_alg";
  else if (ctx.enable_low_pass_filter) why = "the low-pass filter needs an output layout (set enable_low_pass_filter = 0)";
  if (why) {
    std::printf("Could not generate map from a warp map: %s (map %dx%d, input %dx%d, border %d).\n", why, mapW, mapH, inW, inH, border);
    return false;
  }
  plan.inW = inW; plan.inH = inH;
  plan.outW = plan.mapW = mapW;
  plan.outH = plan.mapH = mapH;
  plan.kernelSize = kernelSizeOf(ctx.interpolation_alg);
  plan.transparentBorder = border == kBorderTransparent;
  plan.warp = true;
  plan.map.assign(map, map + static_cast<size_t>(mapW) * mapH * 2);
  samplePlan(plan);
  return true;
}

bool buildHostPlan(const FrameTransformContext& ctx, int inW, int inH, int outW, int outH, HostPlan& plan) {
  plan = HostPlan{};
  plan.ctx = ctx;
  if (inW <= 0 || inH <= 0 || outW <= 0 || outH <= 0) {
    std::printf("Could not generate map: non-positive plane size %dx%d -> %dx%d.\n", inW, inH, outW, outH);
    return false;
  }
  plan.inW = inW; plan.inH = inH; plan.outW = outW; plan.outH = outH;
  // render size before the optional area down-scale (reference cpp:524-526)
  plan.mapW = static_cast<int>(ctx.width_scale_factor * outW + 0.5);
  plan.mapH = static_cast<int>(ctx.height_scale_factor * outH + 0.5);
  if (plan.mapW <= 0 || plan.mapH <= 0) {
    std::printf("Could not generate map: scale factors give an empty plane.\n");
    return false;
  }
  plan.kernelSize = kernelSizeOf(ctx.interpolation_alg);
  plan.transparentBorder = ctx.output_layout == LAYOUT_BARREL || ctx.output_layout == LAYOUT_BARREL_SPLIT;
  if (!buildWarpMap(plan)) return false;
  samplePlan(plan);
  if (ctx.enable_low_pass_filter) {
    // (num_horizontal_segments <= 0 is not an error in the reference: with adjust_kernel its tile loop simply does not
    // run, cpp:235, so every band is left without tiles and the "blurred" plane stays zero; without adjust_kernel the
    // value is ignored, cpp:224-225.  num_vertical_segments <= 0 divides by zero there; refused here.)
    if (ctx.num_vertical_segments < 1) {
      std::printf("Could not generate map: num_vertical_segments must be positive.\n");
      return false;
    }
    if (!buildLowPassPlan(plan)) return false;
  }
  return true;
}

}  // namespace t360
