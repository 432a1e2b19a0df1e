// oracle/ref_driver.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// Links against the reference's own, unmodified VideoFrameTransform.cpp and
// VideoFrameTransformHandler.cpp (compiled from the reference checkout where they
// lie, see oracle/Makefile) and exposes, in addition to the reference C-ABI
// those files export, read-only accessors for the plan the reference computed:
//   warpMats_                 (reference VideoFrameTransform.h:150)
//   filterKernelsX_/Y_        (reference VideoFrameTransform.h:155)
//   segmentFilteringConfigs_  (reference VideoFrameTransform.h:159)
// plus the setter for the OpenCV hooks declared in shim/opencv2/opencv.hpp.
// The output .so lives in oracle/_ref/ (git-ignored, a build product).

#include <map>
#include <string>
#include <thread>
#include <vector>

#include <opencv2/opencv.hpp>

#define private public
#include "VideoFrameTransform.h"
#undef private

extern "C" {

t360ref_remap_hook g_t360ref_remap = nullptr;
t360ref_sep_hook g_t360ref_sep = nullptr;
t360ref_resize_hook g_t360ref_resize = nullptr;

void t360ref_set_hooks(t360ref_remap_hook r, t360ref_sep_hook s, t360ref_resize_hook z) {
  g_t360ref_remap = r;
  g_t360ref_sep = s;
  g_t360ref_resize = z;
}

// Map for a plan index: returns pointer to float32[rows][cols][2] (x, y), or NULL.
const float* t360ref_map(VideoFrameTransform* t, int idx, int* rows, int* cols, size_t* stepBytes) {
  auto it = t->warpMats_.find(idx);
  if (it == t->warpMats_.end() || it->second.empty()) return nullptr;
  *rows = it->second.rows;
  *cols = it->second.cols;
  *stepBytes = it->second.step;
  return reinterpret_cast<const float*>(it->second.data);
}

int t360ref_num_segments(VideoFrameTransform* t, int idx) {
  auto it = t->segmentFilteringConfigs_.find(idx);
  return it == t->segmentFilteringConfigs_.end() ? 0 : static_cast<int>(it->second.size());
}

// Segment i of plan idx: rect[4] = left, top, width, height; kernel lengths in nk[2] = {nx, ny}.
int t360ref_segment(VideoFrameTransform* t, int idx, int i, int* rect, int* nk) {
  auto it = t->segmentFilteringConfigs_.find(idx);
  if (it == t->segmentFilteringConfigs_.end() || i < 0 || i >= static_cast<int>(it->second.size())) return 0;
  const SegmentFilteringConfig& c = it->second[i];
  rect[0] = c.left; rect[1] = c.top; rect[2] = c.width; rect[3] = c.height;
  const cv::Mat& kx = t->filterKernelsX_[idx][i];
  const cv::Mat& ky = t->filterKernelsY_[idx][i];
  nk[0] = kx.rows * kx.cols;
  nk[1] = ky.rows * ky.cols;
  return 1;
}

// Copies the taps of segment i (axis 0 = X kernel, 1 = Y kernel) into out[n].
int t360ref_kernel(VideoFrameTransform* t, int idx, int i, int axis, float* out, int n) {
  auto& vec = axis == 0 ? t->filterKernelsX_[idx] : t->filterKernelsY_[idx];
  if (i < 0 || i >= static_cast<int>(vec.size())) return 0;
  const cv::Mat& k = vec[i];
  int len = k.rows * k.cols;
  if (len != n) return 0;
  for (int j = 0; j < len; ++j) out[j] = k.at<float>(0, j);
  return 1;
}

int t360ref_sizeof_context() { return static_cast<int>(sizeof(FrameTransformContext)); }

}  // extern "C"
