// Pyramid gate: one level of the anti-aliased camera views' input pyramid (pyramidLevelKernel, csrc/kernels.cu) for 1-3
// planes in one launchPyramidLevel call, on buffers the caller owns.  tests/test_pyramid.py builds it as a shared object
// with the library's nvcc flags (transform360_b200/build.py), compiling csrc/kernels.cu and the host planner
// (sampling.cpp, with the geometry.cpp and lowpass_plan.cpp its plan step calls) into it, and drives it through ctypes
// with torch device buffers, so the test chooses every base address, pitch and size.
//
// The tap tables are what VideoFrameTransform::buildPyramids hands the kernel: buildAreaResize of the level's sizes;
// exact 2 x 2 cells (cellW == cellH == 2) pass no tables (xTaps == nullptr); otherwise both axes' taps packed as
// int2 {src, float bits} and the first[] arrays as int, each array at an 8-byte aligned offset of one byte buffer.
//
//   int pyramidGateTaps(srcW, srcH, dstW, dstH, bytes, capacity, offsets[4], counts[4])
//       the packed tables of one level: 1 exact cells (no tables), 0 tables (offsets of xTaps, xFirst, yTaps, yFirst in
//       bytes, counts their elements; bytes may be null to ask for the size in offsets[0]), -1 a size the pyramid never
//       has (an integer ratio other than 2 x 2, or an enlarging axis), -2 bytes too small.  No CUDA call.
//   int pyramidGateLevel(numPlanes, planes)
//       uploads the planes' tables, runs launchPyramidLevel on the legacy default stream and waits for it: the CUDA
//       error code (0 on success), or -1 for a plane the pyramid never has.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>
#include <vector>

#include "host_plan.h"
#include "kernels.cuh"

namespace {

struct Packed {
  size_t at[4] = {SIZE_MAX, 0, 0, 0};  // xTaps, xFirst, yTaps, yFirst (xTaps SIZE_MAX: exact 2 x 2 cells)
  int count[4] = {0, 0, 0, 0};
};

// buildPyramids' packing of one level into b: returns false for sizes that are neither exact 2 x 2 cells nor area taps
bool pack(int srcW, int srcH, int dstW, int dstH, std::vector<uint8_t>& b, Packed& out) {
  t360::AreaResizePlan r;
  t360::buildAreaResize(srcW, srcH, dstW, dstH, r);
  out = Packed{};
  if (!r.needed || r.enlarge) return false;
  if (r.cellW != 0) return r.cellW == 2 && r.cellH == 2;
  auto append = [&b](const void* data, size_t bytes) {
    b.resize((b.size() + 7) & ~size_t{7});
    const size_t at = b.size();
    b.insert(b.end(), static_cast<const uint8_t*>(data), static_cast<const uint8_t*>(data) + bytes);
    return at;
  };
  auto packed = [](const t360::AreaAxis& a) {
    std::vector<int2> v(a.taps.size());
    for (size_t i = 0; i < v.size(); ++i) {
      int bits;
      std::memcpy(&bits, &a.taps[i].alpha, sizeof(bits));
      v[i] = int2{a.taps[i].src, bits};
    }
    return v;
  };
  const std::vector<int2> xt = packed(r.x), yt = packed(r.y);
  out.at[0] = append(xt.data(), xt.size() * sizeof(int2));
  out.at[1] = append(r.x.first.data(), r.x.first.size() * sizeof(int));
  out.at[2] = append(yt.data(), yt.size() * sizeof(int2));
  out.at[3] = append(r.y.first.data(), r.y.first.size() * sizeof(int));
  out.count[0] = static_cast<int>(xt.size());
  out.count[1] = static_cast<int>(r.x.first.size());
  out.count[2] = static_cast<int>(yt.size());
  out.count[3] = static_cast<int>(r.y.first.size());
  return true;
}

}  // namespace

// One plane of a launch as the test passes it: device addresses and sizes.
struct GatePlane {
  unsigned long long src, dst;
  int srcW, srcH, srcPitch, dstW, dstH, dstPitch;
};

extern "C" __attribute__((visibility("default"))) int pyramidGateTaps(int srcW, int srcH, int dstW, int dstH, uint8_t* bytes,
                                                                      size_t capacity, unsigned long long* offsets, int* counts) {
  std::vector<uint8_t> b;
  Packed p;
  if (!pack(srcW, srcH, dstW, dstH, b, p)) return -1;
  for (int k = 0; k < 4; ++k) {
    offsets[k] = p.at[k];
    counts[k] = p.count[k];
  }
  if (p.at[0] == SIZE_MAX) return 1;
  if (!bytes) {
    offsets[0] = b.size();
    return 0;
  }
  if (capacity < b.size()) return -2;
  std::memcpy(bytes, b.data(), b.size());
  return 0;
}

extern "C" __attribute__((visibility("default"))) int pyramidGateLevel(int numPlanes, const GatePlane* planes) {
  if (numPlanes < 1 || numPlanes > t360::kMaxFramePlanes) return -1;
  std::vector<uint8_t> b;  // every plane's tables in one buffer, as buildPyramids stages them
  Packed at[t360::kMaxFramePlanes];
  for (int p = 0; p < numPlanes; ++p) {
    const GatePlane& g = planes[p];
    if (!pack(g.srcW, g.srcH, g.dstW, g.dstH, b, at[p])) return -1;
  }
  uint8_t* taps = nullptr;
  cudaError_t err = cudaSuccess;
  if (!b.empty()) {
    err = cudaMalloc(&taps, b.size());
    if (err == cudaSuccess) err = cudaMemcpy(taps, b.data(), b.size(), cudaMemcpyHostToDevice);
  }
  if (err == cudaSuccess) {
    t360::PyramidParams pp{};
    pp.numPlanes = numPlanes;
    for (int p = 0; p < numPlanes; ++p) {
      const GatePlane& g = planes[p];
      t360::PyramidPlane& v = pp.plane[p];
      v.src = reinterpret_cast<const uint8_t*>(g.src);
      v.dst = reinterpret_cast<uint8_t*>(g.dst);
      v.srcW = g.srcW; v.srcH = g.srcH; v.srcPitch = g.srcPitch;
      v.dstW = g.dstW; v.dstH = g.dstH; v.dstPitch = g.dstPitch;
      if (at[p].at[0] != SIZE_MAX) {
        v.xTaps = reinterpret_cast<const int2*>(taps + at[p].at[0]);
        v.xFirst = reinterpret_cast<const int*>(taps + at[p].at[1]);
        v.yTaps = reinterpret_cast<const int2*>(taps + at[p].at[2]);
        v.yFirst = reinterpret_cast<const int*>(taps + at[p].at[3]);
      }
    }
    err = t360::launchPyramidLevel(pp, 0);
    if (err == cudaSuccess) err = cudaStreamSynchronize(0);
  }
  if (taps) {
    const cudaError_t freed = cudaFree(taps);
    if (err == cudaSuccess) err = freed;
  }
  return static_cast<int>(err);
}
