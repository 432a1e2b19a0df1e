// The job lists of the segmented low-pass: how a plan's segments are cut into jobs for the strip, tile and direct kernels,
// how the lists of a frame's planes are merged into one, and the byte image the device holds them in.  Pure host code
// (no CUDA call), so that the CPU test-suite can check it without a GPU (T360B200_hostPlanBlurLists).  Job formats:
// kernels.cuh.
#pragma once

#include <cstddef>
#include <cstdint>
#include <vector>

#include "host_plan.h"
#include "kernels.cuh"

namespace t360 {

// The low-pass jobs of one plane size (or, merged, of a frame's planes) on the host.
struct BlurLists {
  std::vector<StripJob> strips[kStripMaxHy];  // by vertical half-size 1..3, heaviest first
  std::vector<BlurJob> tiles, direct;
  std::vector<float> taps;
  // per entry of taps: 1 + the index of the plan's tap it copies, 0 for a padding zero; in a merged list plus the plane
  // << kTapPlaneShift (the per-view low-pass refills the taps from it without cutting the jobs again)
  std::vector<int> tapSource;
  int tileSmem = 0;
};
constexpr int kTapPlaneShift = 28;

// Tiles of the plan, applied once (mono) or to both halves of a stereo frame (reference cpp:630-691), cut into jobs for
// planes of planeW x planeH.  Segments that do not fit the plane are dropped, like the reference's caught cv::Exception.
// *needsClear (if asked for): whether some pixel of the plane lies under no segment -- it depends on the plane size and
// the segment rectangles only, not on the taps.
void buildBlurLists(const std::vector<LowPassSegment>& segments, const std::vector<float>& planTaps, int planeW, int planeH,
                    int stereoFormat, BlurLists& out, bool* needsClear);

// The strip jobs of a frame's planes as one list: plane p's taps follow the previous planes' at a 16-byte aligned offset,
// its jobs' tap offsets are rebased onto them and carry p in `edge` (kStripPlaneShift).  Tile and direct jobs are not
// merged (a frame whose planes have any runs per plane).
BlurLists mergeBlurLists(const BlurLists* const* planes, int numPlanes);

// Where the arrays of a BlurLists lie in its device image (byte offsets) and how many entries each has.
struct BlurLayout {
  int numStrips[kStripMaxHy] = {}, numTiles = 0, numDirect = 0, numTaps = 0, tileSmem = 0;
  size_t stripAt[kStripMaxHy] = {}, tileAt = 0, directAt = 0, tapAt = 0;
};

// Appends the job arrays of `l` to `jobs` and its taps to `taps` (the same vector for one image), every array at a 16-byte
// aligned offset (the strip kernel reads the horizontal taps as float4).
BlurLayout packBlurLists(const BlurLists& l, std::vector<uint8_t>& jobs, std::vector<uint8_t>& taps);

}  // namespace t360
