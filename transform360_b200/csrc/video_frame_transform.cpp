// class VideoFrameTransform + the extern "C" boundary.
//
// Mirrors the reference's public surface (VideoFrameTransform.h:40-75, VideoFrameTransformHandler.cpp:18-64):
// same class name behind the opaque handle, same four C entry points, same bool/int results, messages on
// stdout.  Everything behind it is new: the host planner (geometry.cpp, lowpass_plan.cpp, sampling.cpp)
// produces the plan, it is uploaded once, and each frame plane is two kernel launches at most
// (segmented low-pass, gather).  There is no CPU pixel path: if CUDA is unavailable the calls fail.
#include <cuda.h>  // CUtensorMap types; the encoder is looked up at run time, libcuda is not linked
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <climits>
#include <cmath>
#include <condition_variable>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <shared_mutex>
#include <stdexcept>
#include <string>
#include <string_view>
#include <thread>
#include <vector>

#include "host_plan.h"
#include "gather_plan.h"
#include "kernels.cuh"
#include "lowpass_jobs.h"
#include "transform360_b200.h"

#define T360_API extern "C" __attribute__((visibility("default")))

namespace {

using t360::BlurJob;
using t360::GatherJob;
using t360::HostPlan;
using t360::StripJob;

struct CudaFail {
  cudaError_t err;
  const char* what;
};

#define CU(call)                                       \
  do {                                                 \
    cudaError_t e__ = (call);                          \
    if (e__ != cudaSuccess) throw CudaFail{e__, #call}; \
  } while (0)

// body()'s result, or false with a message prefixed by `what` when it throws.  A CUDA error is cleared, so that the
// caller's next runtime call does not report it again.
template <class Body>
bool guarded(std::string_view what, Body&& body) {
  const int n = static_cast<int>(what.size());
  try {
    return body();
  } catch (const CudaFail& f) {
    std::printf("%.*s. Error: CUDA %s (%s) in %s\n", n, what.data(), cudaGetErrorName(f.err), cudaGetErrorString(f.err), f.what);
    cudaGetLastError();
  } catch (const std::exception& ex) {
    std::printf("%.*s. Error: %s\n", n, what.data(), ex.what());
  }
  return false;
}

template <typename T>
struct DeviceBuffer {
  T* ptr = nullptr;
  size_t count = 0;
  DeviceBuffer() = default;
  DeviceBuffer(const DeviceBuffer&) = delete;
  DeviceBuffer& operator=(const DeviceBuffer&) = delete;
  DeviceBuffer(DeviceBuffer&& o) noexcept : ptr(o.ptr), count(o.count) { o.ptr = nullptr; o.count = 0; }
  DeviceBuffer& operator=(DeviceBuffer&& o) noexcept {
    if (this != &o) { release(); ptr = o.ptr; count = o.count; o.ptr = nullptr; o.count = 0; }
    return *this;
  }
  ~DeviceBuffer() { release(); }
  void release() {
    if (ptr) cudaFree(ptr);
    ptr = nullptr;
    count = 0;
  }
  void reserve(size_t n) {  // grow-only
    if (n <= count) return;
    release();
    CU(cudaMalloc(reinterpret_cast<void**>(&ptr), n * sizeof(T)));
    count = n;
  }
  size_t bytes() const { return count * sizeof(T); }
};

// Device-resident plan of one plan index (what the reference keeps in warpMats_, filterKernelsX_/Y_,
// segmentFilteringConfigs_; VideoFrameTransform.h:150-159).
struct DevicePlan {
  int inW = 0, inH = 0, outW = 0, outH = 0, mapW = 0, mapH = 0;
  int kernelSize = 0;
  bool transparent = false, lowPass = false;
  bool warp = false;  // made from a caller's warp map (generateMapFromWarp): no geometry to re-plan or to compute per frame
  int stereoFormat = STEREO_FORMAT_MONO;  // input_stereo_format of the context the plan was made with (low-pass passes)
  DeviceBuffer<int2> samples;      // full records: tile-major, lane-ordered, 8 bytes per pixel (whole-plane general kernels)
  DeviceBuffer<uint32_t> records;  // compact records of the frame kernel's jobs (kernels.cuh): 2.5 - 4 bytes per pixel (pole caps: 8)
  int tilesPerRow = 0;
  // gather jobs: share blocks and tiles whose source windows fit a TMA staging box, pole-cap and border jobs
  DeviceBuffer<GatherJob> gatherJobs;  // every job of the plane, in launch order (gather_plan.h: jobLaunchRank)
  std::vector<GatherJob> hostJobs;     // the same list on the host: merged per frame by gatherFrame()
  std::vector<int> jobNeedRows;        // per host job: the source rows [0, n) it reads (streaming host planes in)
  std::vector<t360::JobRect> jobRects; // per host job: the output rectangle it writes into (streaming host planes out)
  int numJobs = 0, numStaged = 0, numBorder = 0;  // staged: jobs with a TMA box; border: jobs reading through L1
  // low-pass: the job lists of one plane size, on the host (the whole-frame entry point merges the planes' lists) and
  // packed into one device image
  struct BlurSet {
    t360::BlurLists lists;
    t360::BlurLayout layout;
    DeviceBuffer<uint8_t> image;
    bool needsClear = false;
  };
  BlurSet blur;  // for the plane size the plan was generated for
  // (a caller may pass planes of another size: the reference then filters the segments that still fit, cpp:173-204)
  std::vector<t360::LowPassSegment> segments;
  std::vector<float> planTaps;
  mutable std::map<std::pair<int, int>, BlurSet> otherBlurs;
  // cv::resize(INTER_AREA) after the gather whenever the requested output size differs from the map's (reference
  // cpp:735-737: decided per call): tables per output size, made on first use
  struct Resize {
    int cellW = 0, cellH = 0, xMax = 0;  // cellW > 0: integer ratios; < 0: the enlarging (bilinear) variant; 0: area tables
    DeviceBuffer<int2> xTaps, yTaps, xLinear, yLinear;
    DeviceBuffer<int> xFirst, yFirst;
  };
  bool resizeNeeded = false;  // for the size the map was generated for
  mutable std::map<std::pair<int, int>, Resize> resizes;
  // the per-frame orientation path's view-independent tables (oriented_view.h: buildSphereTables): EAC_32, EQUIRECT, BARREL,
  // BARREL_SPLIT
  DeviceBuffer<float> sphereTables;
  size_t deviceBytes() const {
    return samples.bytes() + records.bytes() + gatherJobs.bytes() + blur.image.bytes();
  }
};

// Whether the low-pass of a frame's planes, every one of which has low-pass, runs as one strip launch per vertical
// half-size for all of them: every plane has the size it was planned for, the plan is not transparent, its segments cover
// the plane (!clear[p]) and its lists (lists[p]) hold strip jobs only.
bool mergeable(const DevicePlan* const* plans, const t360::BlurLists* const* lists, const bool* clear, int numPlanes, const int* inW,
               const int* inH) {
  if (numPlanes < 2) return false;
  for (int p = 0; p < numPlanes; ++p) {
    const DevicePlan& d = *plans[p];
    if (d.transparent || inW[p] != d.inW || inH[p] != d.inH || clear[p] || !lists[p]->tiles.empty() || !lists[p]->direct.empty())
      return false;
  }
  return true;
}

// The host-side half of a plan index (no CUDA call): the planner's result and, for interpolating plans, the gather plan.
struct HostIndexPlan {
  HostPlan host;
  t360::GatherPlan gather;
};
// The gather plan of a host plan: staged (the persistent frame kernel's jobs) for k >= 2 under BORDER_WRAP.
void gatherOnHost(HostIndexPlan& p) {
  if (p.host.kernelSize > 0) t360::buildGatherPlan(p.host, p.host.kernelSize >= 2 && !p.host.transparentBorder, p.gather);
}
bool planOnHost(const FrameTransformContext& ctx, int inW, int inH, int outW, int outH, HostIndexPlan& p) {
  if (!t360::buildHostPlan(ctx, inW, inH, outW, outH, p.host)) return false;
  gatherOnHost(p);
  return true;
}
// ... from a caller's warp map instead of the context's geometry (T360B200_generateMapFromWarp)
bool planWarpOnHost(const FrameTransformContext& ctx, const float* map, int mapW, int mapH, int inW, int inH, int border, HostIndexPlan& p) {
  if (!t360::buildWarpHostPlan(ctx, map, mapW, mapH, inW, inH, border, p.host)) return false;
  gatherOnHost(p);
  return true;
}

// A driver API function through the runtime's entry point table (nullptr if the driver has none): libcuda is never linked.
void* driverEntry(const char* name) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q{};
  if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
    cudaGetLastError();
    p = nullptr;
  }
  return p;
}

// How long the background planner waits after a reconfigureAsync before it plans that context: a camera path or a slider
// sends a command every frame, and restarting a re-plan of about a second for each of them would keep the host's cores
// busy for the whole move while the frames are served on the per-frame kernels anyway.
constexpr std::chrono::milliseconds kSettleInterval{250};

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled through the runtime's driver entry point table: the library must still dlopen()
// on a machine without libcuda.so (CPU-only planning, tests), so libcuda is never linked.
EncodeTiledFn tensorMapEncoder() {
  static const EncodeTiledFn fn = reinterpret_cast<EncodeTiledFn>(driverEntry("cuTensorMapEncodeTiled"));
  return fn;
}

// Describes a pitch-linear 8-bit plane to the TMA unit with box shape `index` of kernel size k (kernels.cuh: boxMapIndex).
bool encodePlaneMap(CUtensorMap* map, const uint8_t* base, int w, int h, int pitch, int k, int index) {
  EncodeTiledFn enc = tensorMapEncoder();
  if (!enc) return false;
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (pitch & 15)) return false;
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(w), static_cast<cuuint64_t>(h)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(pitch)};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(t360::boxMapW(k, index)), static_cast<cuuint32_t>(t360::boxMapRows(k, index))};
  const cuuint32_t elem[2] = {1, 1};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t*>(base), dims, strides, box, elem,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,  // (none / 64 / 256 B: no difference)
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Everything one image plane needs to be in flight independently of the others: the frame entry point runs the
// luma plane on the caller's stream and the two chroma planes on their own lanes.
constexpr int kPlaneLanes = 3;
static_assert(kPlaneLanes == t360::kMaxFramePlanes, "the frame kernel takes one PlaneView per lane");
// The tensor maps of one source plane (every box shape of its kernel size): encoding one takes the driver about a
// microsecond, a frame needs up to 48, and callers come back with the same few planes (a decoder's surface pool, the
// library's own low-pass plane), so every lane remembers the last few.
struct PlaneMaps {
  const uint8_t* base = nullptr;
  int w = 0, h = 0, pitch = 0, k = 0;
  CUtensorMap maps[t360::kMaxBoxMaps];
};
struct PlaneLane {
  static constexpr int kMapCache = 32;  // (a decoder's surface pool holds 10 - 20 frames)
  PlaneMaps mapCache[kMapCache];
  int mapCacheNext = 0;
  cudaStream_t main = nullptr;                       // chroma lanes only (lane 0 runs on the caller's stream)
  cudaEvent_t done = nullptr;                        // recorded when this lane's plane has been enqueued completely
  DeviceBuffer<uint8_t> blurred;                     // low-pass output of this plane
  DeviceBuffer<uint8_t> scaled;                      // render target at map size when an area resize follows
  DeviceBuffer<uint8_t> pyramid;                     // levels 1..T of this plane's input pyramid (anti-aliased camera views)
  DeviceBuffer<int> claimCounter;                    // dynamic tile scheduler of this lane's gather launch
};

// Where the gather of one plane writes (dst, at the map's size) and where its result must end up (out, the caller's
// plane): the same plane, or a lane's plane and the INTER_AREA tables from it to the caller's (see
// VideoFrameTransform::renderTarget).
struct PlaneTarget {
  uint8_t* dst = nullptr;
  int dstPitch = 0, dstW = 0, dstH = 0;
  uint8_t* out = nullptr;
  int outPitch = 0, outW = 0, outH = 0;
  const DevicePlan::Resize* resize = nullptr;
};

// What the gather stage of one image plane needs once its source is ready (see VideoFrameTransform::prepareGather).
struct GatherWork {
  const DevicePlan* plan = nullptr;
  t360::PlaneView view{};
  bool staged = false;                       // TMA-describable: may run in the persistent (per-plane / per-frame) kernel
  CUtensorMap maps[t360::kMaxBoxMaps];
  PlaneTarget target;
};

// The merged lists of a frame of 2 or 3 planes, built once per plan generation: the gather jobs of every plane in one
// list (jobLaunchRank order, the plane in outY) and the planes' low-pass strip jobs in one image (mergeBlurLists).
struct FrameLists {
  unsigned long long generation = ~0ull;
  DeviceBuffer<GatherJob> gatherJobs;
  int numGatherJobs = 0;
  DeviceBuffer<uint8_t> blurImage;
  t360::BlurLayout blurLayout;
};
// ... as one frame launches them (copied out under the lock)
struct FrameListRefs {
  const GatherJob* gatherJobs;
  int numGatherJobs;
  const uint8_t* blurImage;
  t360::BlurLayout blurLayout;
};

// How the synchronous host-pointer call streams a large plane through the GPU (t360::scheduleWaves): the input arrives in
// `chunks` row bands; wave c = the gather jobs that only read rows delivered by chunks 0..c; rects[c] = the output
// rectangles that are complete after wave c (copied back while later chunks are still on their way: PCIe carries both
// directions at once).
struct WavePlan {
  int chunks = 0;
  const void* plan = nullptr;  // the DevicePlan it was made for
  unsigned long long generation = ~0ull;
  t360::WaveSchedule schedule;
  DeviceBuffer<GatherJob> jobs;  // wave-major
};

// The streamed host-plane call is ~100 runtime calls (chunk copies, events, wave launches, rectangle copies); issued one by
// one the host thread becomes the bottleneck (measured: no faster than the plain path).  For page-locked caller planes the
// whole sequence is captured once per (plan, buffers) into a CUDA graph and replayed with one launch.
struct PlaneGraph {
  const void* plan; unsigned long long generation; const void* in; const void* out; int inPitch, outPitch;
  const void* stagingIn; const void* stagingOut;  // (the staging planes grow on demand: a graph made for old ones is stale)
  int inW, inH, outW, outH;
  int kernels;
  cudaGraphExec_t exec; unsigned long long lastUse;
};

// The per-view low-pass lists of a stream slot's previous frame and what they were made from.  The jobs (rectangles, tap
// counts and offsets) depend on the view only through the segments' tap counts and on which neighbouring segments carry
// identical taps; when those agree with the previous frame's, the jobs are reused and only the taps are refilled.
struct ViewBlurCache {
  std::vector<long long> key;
  bool merged = false;
  std::vector<uint8_t> jobs;
  std::vector<int> tapCodes;  // per float of the tap image: plane << kTapPlaneShift | (1 + plan tap), 0 for a zero
  t360::BlurLayout layout[2];  // merged: [0]; else per plan index
  bool clear[2] = {false, false};  // per plan index: some pixel lies under no segment
};

// Page-locked staging of lists that change from frame to frame (the per-view low-pass jobs and taps): a few entries, each
// a page-locked host buffer and a device buffer, reused round robin.  An entry is refilled only after the frame that last
// read it has finished on the device (its event), and a frame whose lists equal the previous frame's reuses that entry
// without any copy.  Device memory stays bounded: kEntries buffers of the largest list seen.
struct UploadRing {
  static constexpr int kEntries = 3;
  struct Entry {
    uint8_t* host = nullptr;    // page-locked
    uint8_t* device = nullptr;  // stream-ordered allocation on the slot's stream
    size_t capacity = 0;
    cudaEvent_t released = nullptr;  // recorded after the last frame that reads `device`
    bool inFlight = false;
  };
  Entry entries[kEntries];
  int last = -1;                    // the entry that holds lastContent
  std::vector<uint8_t> lastContent;
};

// Everything asynchronous work on ONE caller stream shares: the lanes (scratch planes, side streams, job schedulers) and
// the scheduler of the whole-frame launch.  Work on the same stream is ordered, so one set per stream is enough; callers
// that enqueue on several streams at once get a set per stream instead of racing for one.
struct StreamSlot {
  PlaneLane lanes[kPlaneLanes];
  DeviceBuffer<int> frameClaim;
  cudaEvent_t fork = nullptr;
  UploadRing viewJobs, viewTaps;  // the per-frame calls' low-pass lists (VideoFrameTransform::viewLowPass)
  ViewBlurCache viewBlur;
  // the per-frame orientation kernel's tables while a reconfigureAsync is pending (the plans' tables are for the old context),
  // and the context and plan generation they were built for
  // (also the lens kernel's tables, which have no plan to come from), and the context and map sizes they were built for
  UploadRing sphereTables;
  std::vector<uint8_t> sphereBytes;
  size_t sphereAt[kPlaneLanes] = {SIZE_MAX, SIZE_MAX, SIZE_MAX};  // per plane: where its tables start in sphereBytes
  FrameTransformContext sphereCtx{};
  std::vector<int> sphereSizes;  // mapW, mapH per plane
  // the INTER_AREA tap tables of the anti-aliased camera views' pyramid levels that are not exact 2 x 2 cells, and the
  // plane sizes and top levels they were built for (VideoFrameTransform::buildPyramids)
  UploadRing mipTaps;
  std::vector<uint8_t> mipTapBytes;
  struct MipTapsAt {
    size_t xTaps = SIZE_MAX, xFirst, yTaps, yFirst;  // byte offsets in mipTapBytes (SIZE_MAX: exact 2 x 2 cells)
  } mipTapAt[kPlaneLanes][t360::kMipMaxLevels];      // per plane and level l (at l - 1)
  std::vector<int> mipSizes;                         // inW, inH, top per plane
  // the rig motion's sample table of the motion calls (they change every frame)
  UploadRing motionTables;
  std::vector<uint8_t> motionBytes;
};

// A w x h scratch plane in buf (a lane's or the staging planes), grown on demand: its pitch, 256-byte aligned
int scratchPlane(DeviceBuffer<uint8_t>& buf, int w, int h) {
  constexpr int kPitchAlign = 256;
  const int pitch = (w + kPitchAlign - 1) / kPitchAlign * kPitchAlign;
  buf.reserve(static_cast<size_t>(pitch) * h + 64);
  return pitch;
}

// The device planes of a whole-frame call: plane p is read from in[p] (inW x inH, inPitch bytes per row) and written to
// out[p].
struct FramePlanes {
  int numPlanes = 0;
  const uint8_t* in[kPlaneLanes];
  uint8_t* out[kPlaneLanes];
  int inW[kPlaneLanes], inH[kPlaneLanes], inPitch[kPlaneLanes], outW[kPlaneLanes], outH[kPlaneLanes], outPitch[kPlaneLanes];
};

// The frame of a whole-frame call's arrays, checked on the host: false, with a message prefixed by `what`, for a NULL
// array, a plane count outside 1..kPlaneLanes, or a plane that is NULL, has no pixels or a pitch short of its width.
bool describeFrame(const char* what, int numPlanes, const uint8_t* const* dIn, uint8_t* const* dOut, const int* inW, const int* inH,
                   const int* inPitch, const int* outW, const int* outH, const int* outPitch, FramePlanes& f) {
  if (!dIn || !dOut || !inW || !inH || !inPitch || !outW || !outH || !outPitch) {
    std::printf("%s. Error: a NULL argument\n", what);
    return false;
  }
  if (numPlanes < 1 || numPlanes > kPlaneLanes) {
    std::printf("%s. Error: %d planes (1..%d supported)\n", what, numPlanes, kPlaneLanes);
    return false;
  }
  f.numPlanes = numPlanes;
  for (int p = 0; p < numPlanes; ++p) {
    if (!dIn[p] || !dOut[p] || inW[p] <= 0 || inH[p] <= 0 || outW[p] <= 0 || outH[p] <= 0 || inPitch[p] < inW[p] || outPitch[p] < outW[p]) {
      std::printf("%s. Error: invalid description of plane %d\n", what, p);
      return false;
    }
    f.in[p] = dIn[p]; f.out[p] = dOut[p];
    f.inW[p] = inW[p]; f.inH[p] = inH[p]; f.inPitch[p] = inPitch[p];
    f.outW[p] = outW[p]; f.outH[p] = outH[p]; f.outPitch[p] = outPitch[p];
  }
  return true;
}

// ---- per-frame views, orientations and poses: their checks against a context and the context they render with ---------
// The context with the five view fields replaced
void setPose(FrameTransformContext& ctx, const T360Pose& pose) {
  ctx.fixed_yaw = pose.yaw;
  ctx.fixed_pitch = pose.pitch;
  ctx.fixed_roll = pose.roll;
  ctx.fixed_hfov = pose.hfov;
  ctx.fixed_vfov = pose.vfov;
}

std::string formatted(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
std::string formatted(const char* fmt, ...) {
  char buf[320];
  va_list args;
  va_start(args, fmt);
  std::vsnprintf(buf, sizeof(buf), fmt, args);
  va_end(args);
  return buf;
}

// Each puts its fields into ctx and returns "", or returns why ctx cannot take them.  A view is a pose with the context's
// roll (which the FLAT_FIXED chain does not use), an orientation one with the context's fields of view.
std::string withFields(FrameTransformContext& ctx, const T360Pose& pose) {
  if (!std::isfinite(pose.yaw) || !std::isfinite(pose.pitch) || !std::isfinite(pose.roll) || !std::isfinite(pose.hfov) ||
      !std::isfinite(pose.vfov))
    return formatted("the pose (yaw %g, pitch %g, roll %g, hfov %g, vfov %g) is not finite", pose.yaw, pose.pitch, pose.roll, pose.hfov,
                     pose.vfov);
  if (ctx.output_layout < 0 || ctx.output_layout >= LAYOUT_N) return formatted("output_layout %d is not a layout", static_cast<int>(ctx.output_layout));
  setPose(ctx, pose);
  return {};
}
std::string withFields(FrameTransformContext& ctx, const T360View& view) {
  if (!std::isfinite(view.yaw) || !std::isfinite(view.pitch) || !std::isfinite(view.hfov) || !std::isfinite(view.vfov))
    return formatted("the view (yaw %g, pitch %g, hfov %g, vfov %g) is not finite", view.yaw, view.pitch, view.hfov, view.vfov);
  if (ctx.output_layout != LAYOUT_FLAT_FIXED)
    return formatted("per-frame views need output_layout FLAT_FIXED (%d), the transform has %d", static_cast<int>(LAYOUT_FLAT_FIXED),
                     static_cast<int>(ctx.output_layout));
  setPose(ctx, T360Pose{view.yaw, view.pitch, ctx.fixed_roll, view.hfov, view.vfov});
  return {};
}
std::string withFields(FrameTransformContext& ctx, const T360Orientation& o) {
  if (!std::isfinite(o.yaw) || !std::isfinite(o.pitch) || !std::isfinite(o.roll))
    return formatted("the orientation (yaw %g, pitch %g, roll %g) is not finite", o.yaw, o.pitch, o.roll);
  if (!t360::orientedLayouts(ctx))
    return formatted("per-frame orientations need output_layout CUBEMAP_32, CUBEMAP_23_OFFCENTER, EAC_32 or EQUIRECT and input_layout "
                     "EQUIRECT or CUBEMAP_32, the transform has %d -> %d%s", static_cast<int>(ctx.input_layout),
                     static_cast<int>(ctx.output_layout),
                     ctx.output_layout == LAYOUT_FLAT_FIXED ? " (FLAT_FIXED views: T360B200_transformFrameViewAsync)" : "");
  setPose(ctx, T360Pose{o.yaw, o.pitch, o.roll, ctx.fixed_hfov, ctx.fixed_vfov});
  return {};
}

// The upload ring entry may be refilled once the work enqueued on s so far has finished (nullptr: nothing to release)
void releaseAfter(UploadRing::Entry* e, cudaStream_t s) {
  if (!e) return;
  CU(cudaEventRecord(e->released, s));
  e->inFlight = true;
}

// ---- warp maps (T360B200_remapFrameAsync) ------------------------------------------------------------------------------
// true, with the reason in *why, when the caller's device maps (mapPitch in bytes) cannot remap frame f with this border
bool mapRefused(const FrameTransformContext& ctx, const float* const* maps, const int* mapPitch, int border, const FramePlanes& f,
                std::string* why) {
  if (border != t360::kBorderWrap && border != t360::kBorderTransparent) {
    *why = formatted("border %d (3: BORDER_WRAP, 5: BORDER_TRANSPARENT)", border);
    return true;
  }
  for (int p = 0; p < f.numPlanes; ++p) {
    if (!maps[p]) {
      *why = formatted("invalid description of plane %d", p);
      return true;
    }
    if (mapPitch[p] % 8 != 0 || mapPitch[p] / 8 < f.outW[p] || (reinterpret_cast<uintptr_t>(maps[p]) & 7)) {
      *why = formatted("the map of plane %d (pitch %d bytes) must be 8-byte aligned with a pitch that is a multiple of 8 and at least 8 x the "
                       "output width %d", p, mapPitch[p], f.outW[p]);
      return true;
    }
  }
  if (t360::kernelSizeOf(ctx.interpolation_alg) == 0) {
    *why = formatted("no interpolation algorithm %d", static_cast<int>(ctx.interpolation_alg));
    return true;
  }
  if (ctx.enable_low_pass_filter) {
    *why = "the low-pass filter needs an output layout (set enable_low_pass_filter = 0)";
    return true;
  }
  return false;
}

// ---- fisheye lens rigs (T360B200_lensMap, T360B200_transformFrameLensAsync; oriented_view.h: lensSample) ----------------
// true, with the reason in *why, when the rig's lenses cannot be used (the rig itself, whatever the output)
bool rigRefused(const T360LensRig* rig, std::string* why) {
  char buf[256];
  auto refuse = [&](const char* fmt, auto... args) {
    std::snprintf(buf, sizeof(buf), fmt, args...);
    *why = buf;
    return true;
  };
  if (rig->numLenses != 1 && rig->numLenses != 2) return refuse("numLenses %d (1 or 2 supported)", rig->numLenses);
  if (rig->calibWidth <= 0 || rig->calibHeight <= 0) return refuse("calibration size %dx%d is not positive", rig->calibWidth, rig->calibHeight);
  for (int i = 0; i < rig->numLenses; ++i) {
    const T360Lens& L = rig->lens[i];
    for (float v : {L.fx, L.fy, L.cx, L.cy, L.k[0], L.k[1], L.k[2], L.k[3], L.yaw, L.pitch, L.roll, L.maxAngle})
      if (!std::isfinite(v)) return refuse("lens %d has a field that is not finite", i);
    if (!(L.fx > 0.0f) || !(L.fy > 0.0f)) return refuse("lens %d: fx %g and fy %g must be positive", i, L.fx, L.fy);
    if (!(L.maxAngle > 0.0f && L.maxAngle <= 180.0f)) return refuse("lens %d: maxAngle %g is outside (0, 180]", i, L.maxAngle);
    // theta_d(theta) must be strictly increasing on [0, maxAngle], or the lens would fold the image over: its derivative
    // 1 + 3 k1 t^2 + 5 k2 t^4 + 7 k3 t^6 + 9 k4 t^8 > 0 on a fine grid
    constexpr int kSteps = 4096;
    const double tMax = L.maxAngle * M_PI / 180.0;
    for (int s = 0; s <= kSteps; ++s) {
      const double t = tMax * s / kSteps, t2 = t * t;
      const double d = 1.0 + t2 * (3.0 * L.k[0] + t2 * (5.0 * L.k[1] + t2 * (7.0 * L.k[2] + t2 * 9.0 * L.k[3])));
      if (!(d > 0.0))
        return refuse("lens %d: theta_d(theta) of k = (%g, %g, %g, %g) stops increasing at %.3f degrees, inside maxAngle %g (it would mirror "
                      "the image)", i, L.k[0], L.k[1], L.k[2], L.k[3], t * 180.0 / M_PI, L.maxAngle);
    }
  }
  return false;
}

// true, with the reason in *why, when the lens path cannot serve ctx with this rig and orientation
bool lensRefused(const FrameTransformContext& ctx, const T360LensRig* rig, const T360Orientation* o, std::string* why) {
  if (!rig || !o) {
    *why = "a NULL rig or orientation";
    return true;
  }
  if (!std::isfinite(o->yaw) || !std::isfinite(o->pitch) || !std::isfinite(o->roll)) {
    *why = formatted("the orientation (yaw %g, pitch %g, roll %g) is not finite", o->yaw, o->pitch, o->roll);
    return true;
  }
  if (rigRefused(rig, why)) return true;
  const int layout = ctx.output_layout;
  if (layout == LAYOUT_FLAT_FIXED || layout < 0 || layout >= LAYOUT_N) {
    *why = formatted("output_layout %d (a lens rig needs CUBEMAP_32, CUBEMAP_23_OFFCENTER, EAC_32, EQUIRECT, BARREL or BARREL_SPLIT)", layout);
    return true;
  }
  if (ctx.enable_low_pass_filter) {
    *why = "the low-pass filter is not available for a lens rig (set enable_low_pass_filter = 0)";
    return true;
  }
  if (t360::kernelSizeOf(ctx.interpolation_alg) == 0) {
    *why = formatted("no interpolation algorithm %d", static_cast<int>(ctx.interpolation_alg));
    return true;
  }
  return false;
}

// What the feathered seam needs of a rig that is otherwise usable: two lenses, and a belt width in [0.01, 180] degrees (the
// lower bound keeps lensSeamScale finite)
bool featherRefused(const T360LensRig& rig, float seamWidth, std::string* why) {
  if (rig.numLenses != 2) {
    *why = formatted("numLenses %d: a feathered seam needs two lenses (one lens: T360B200_transformFrameLensAsync)", rig.numLenses);
    return true;
  }
  if (!(seamWidth >= 0.01f && seamWidth <= 180.0f)) {
    *why = formatted("seamWidth %g degrees is outside [0.01, 180]", seamWidth);
    return true;
  }
  return false;
}
// lensRefused, plus featherRefused
bool lensBlendRefused(const FrameTransformContext& ctx, const T360LensRig* rig, float seamWidth, const T360Orientation* o, std::string* why) {
  return lensRefused(ctx, rig, o, why) || featherRefused(*rig, seamWidth, why);
}

// s = 1 / (2 seamWidth), seamWidth in radians: lens 1's weight rises from 0 to 1 while theta0 - theta1 goes from
// -seamWidth to +seamWidth, so a back-to-back pair blends across a belt seamWidth degrees wide (oriented_view.h:
// lensBlendPosition)
float lensSeamScale(float seamWidth) { return static_cast<float>(1.0 / (2.0 * static_cast<double>(seamWidth) * M_PI / 180.0)); }

// Ry(yaw) Rx(-pitch) Rz(roll) of angles in degrees, in double: the lens extrinsics' rotation (and the rig motion's)
void extrinsicRotation(float yaw, float pitch, float roll, double r[3][3]) {
  const double a = yaw * M_PI / 180.0, b = -pitch * M_PI / 180.0, g = roll * M_PI / 180.0;
  const double ry[3][3] = {{std::cos(a), 0, std::sin(a)}, {0, 1, 0}, {-std::sin(a), 0, std::cos(a)}};
  const double rx[3][3] = {{1, 0, 0}, {0, std::cos(b), -std::sin(b)}, {0, std::sin(b), std::cos(b)}};
  const double rz[3][3] = {{std::cos(g), -std::sin(g), 0}, {std::sin(g), std::cos(g), 0}, {0, 0, 1}};
  double ryx[3][3];
  for (int u = 0; u < 3; ++u)
    for (int v = 0; v < 3; ++v) ryx[u][v] = ry[u][0] * rx[0][v] + ry[u][1] * rx[1][v] + ry[u][2] * rx[2][v];
  for (int u = 0; u < 3; ++u)
    for (int v = 0; v < 3; ++v) r[u][v] = ryx[u][0] * rz[0][v] + ryx[u][1] * rz[1][v] + ryx[u][2] * rz[2][v];
}

// A lens's M from its rotation r: R^T, the y row negated (OpenCV's camera coordinates), stored as float
void lensMatrix(const double r[3][3], float* m) {
  for (int u = 0; u < 3; ++u)
    for (int v = 0; v < 3; ++v) m[3 * u + v] = static_cast<float>(u == 1 ? -r[v][u] : r[v][u]);
}

// The per-frame constants of a rig (oriented_view.h: LensModel), in double and stored as float
t360::LensRigModel lensRigModel(const T360LensRig& rig) {
  t360::LensRigModel m{};
  m.numLenses = rig.numLenses;
  for (int i = 0; i < rig.numLenses; ++i) {
    const T360Lens& L = rig.lens[i];
    double r[3][3];
    extrinsicRotation(L.yaw, L.pitch, L.roll, r);
    t360::LensModel& l = m.lens[i];
    lensMatrix(r, l.m);
    l.ax = static_cast<float>(static_cast<double>(L.fx) / rig.calibWidth);
    l.bx = static_cast<float>((static_cast<double>(L.cx) + 0.5) / rig.calibWidth);
    l.ay = static_cast<float>(static_cast<double>(L.fy) / rig.calibHeight);
    l.by = static_cast<float>((static_cast<double>(L.cy) + 0.5) / rig.calibHeight);
    for (int j = 0; j < 4; ++j) l.k[j] = L.k[j];
    l.thetaMax = static_cast<float>(L.maxAngle * M_PI / 180.0);
  }
  return m;
}

// ---- rolling-shutter lens rigs (T360B200_lensMotionMaps, T360B200_cameraMotionMaps and their frame calls) ---------------
// true, with the reason in *why, when a rig motion cannot be used with a usable rig: NULL, a sample count outside [2, 16],
// a delta angle that is not finite or lies outside [-30, 30] degrees, a readout field of a lens that is read that is not
// finite
bool motionRefused(const T360LensRig& rig, const T360RigMotion* mo, std::string* why) {
  if (!mo) {
    *why = "a NULL motion";
    return true;
  }
  if (mo->numSamples < 2 || mo->numSamples > t360::kMotionMaxSamples) {
    *why = formatted("numSamples %d is outside [2, %d]", mo->numSamples, t360::kMotionMaxSamples);
    return true;
  }
  for (int k = 0; k < mo->numSamples; ++k) {
    const T360Orientation& d = mo->delta[k];
    for (float a : {d.yaw, d.pitch, d.roll})
      if (!std::isfinite(a) || !(a >= -30.0f && a <= 30.0f)) {
        *why = formatted("delta[%d] (yaw %g, pitch %g, roll %g) must be finite and lie in [-30, 30] degrees", k, d.yaw, d.pitch, d.roll);
        return true;
      }
  }
  for (int i = 0; i < rig.numLenses; ++i) {
    const T360LensReadout& r = mo->readout[i];
    if (!std::isfinite(r.a) || !std::isfinite(r.b) || !std::isfinite(r.c)) {
      *why = formatted("the readout of lens %d has a field that is not finite", i);
      return true;
    }
  }
  return false;
}

// The motion's sample matrices M_ik, [numLenses][numSamples][9] floats: lens i's rotation R_i turned by delta[k], R_ik =
// Rot(delta[k]) R_i in double, then lensMatrix; a zero delta gives lensRigModel's M itself
std::vector<float> rigMotionTable(const T360LensRig& rig, const T360RigMotion& mo, const t360::LensRigModel& model) {
  std::vector<float> t(static_cast<size_t>(rig.numLenses) * mo.numSamples * 9);
  for (int i = 0; i < rig.numLenses; ++i) {
    const T360Lens& L = rig.lens[i];
    double ri[3][3];
    extrinsicRotation(L.yaw, L.pitch, L.roll, ri);
    for (int k = 0; k < mo.numSamples; ++k) {
      float* m = t.data() + (static_cast<size_t>(i) * mo.numSamples + k) * 9;
      const T360Orientation& d = mo.delta[k];
      if (d.yaw == 0.0f && d.pitch == 0.0f && d.roll == 0.0f) {
        std::memcpy(m, model.lens[i].m, sizeof(model.lens[i].m));
        continue;
      }
      double q[3][3], r[3][3];
      extrinsicRotation(d.yaw, d.pitch, d.roll, q);
      for (int u = 0; u < 3; ++u)
        for (int v = 0; v < 3; ++v) r[u][v] = q[u][0] * ri[0][v] + q[u][1] * ri[1][v] + q[u][2] * ri[2][v];
      lensMatrix(r, m);
    }
  }
  return t;
}

// The per-frame constants of a motion (oriented_view.h: RigMotion) with its table at `table`
t360::RigMotion rigMotion(const T360RigMotion& mo, const float* table) {
  t360::RigMotion m{};
  m.table = table;
  m.numSamples = mo.numSamples;
  for (int i = 0; i < 2; ++i) {
    m.readout[i][0] = mo.readout[i].a;
    m.readout[i][1] = mo.readout[i].b;
    m.readout[i][2] = mo.readout[i].c;
  }
  return m;
}

// true, with the reason in *why, when seamWidth is neither 0 (the hard seam) nor a feathered seam's width (the photometric
// calls' seam; featherRefused checks the rest of a feathered seam against the rig)
bool seamWidthRefused(float seamWidth, std::string* why) {
  if (!std::isfinite(seamWidth) || seamWidth < 0.0f || (seamWidth > 0.0f && seamWidth < 0.01f)) {
    *why = formatted("seamWidth %g degrees is neither 0 (the hard seam) nor in [0.01, 180]", seamWidth);
    return true;
  }
  return false;
}

// true, with the reason in *why, when a photometry cannot correct the lenses of a usable rig: NULL, out of range, or a
// falloff that reaches 0 inside a lens's coverage
bool photometryRefused(const T360LensRig& rig, const T360RigPhotometry* ph, std::string* why) {
  if (!ph) {
    *why = "a NULL photometry";
    return true;
  }
  if (ph->lumaPivot < 0 || ph->lumaPivot > 255) {
    *why = formatted("lumaPivot %d is outside 0..255", ph->lumaPivot);
    return true;
  }
  for (int i = 0; i < rig.numLenses; ++i) {
    const T360LensPhotometry& L = ph->lens[i];
    for (int k = 0; k < 3; ++k)
      if (!std::isfinite(L.vignetting[k]) || !std::isfinite(L.gain[k]) || !std::isfinite(L.offset[k])) {
        *why = formatted("the photometry of lens %d has a field that is not finite", i);
        return true;
      }
    for (int k = 0; k < 3; ++k) {
      if (!(L.gain[k] > 0.0f && L.gain[k] <= 8.0f)) {
        *why = formatted("lens %d: gain[%d] %g is outside (0, 8]", i, k, L.gain[k]);
        return true;
      }
      if (!(L.offset[k] >= -64.0f && L.offset[k] <= 64.0f)) {
        *why = formatted("lens %d: offset[%d] %g is outside [-64, 64]", i, k, L.offset[k]);
        return true;
      }
    }
    // V(r) = 1 + v1 r^2 + v2 r^4 + v3 r^6 must stay positive for every r = theta_d the lens reaches: [0, theta_d(maxAngle)]
    // (theta_d increases on [0, maxAngle]: rigRefused), on a fine grid
    const T360Lens& lens = rig.lens[i];
    const double tMax = lens.maxAngle * M_PI / 180.0, t2 = tMax * tMax;
    const double rMax = tMax * (1.0 + t2 * (lens.k[0] + t2 * (lens.k[1] + t2 * (lens.k[2] + t2 * lens.k[3]))));
    constexpr int kSteps = 4096;
    for (int s = 0; s <= kSteps; ++s) {
      const double r = rMax * s / kSteps, q = r * r;
      const double v = 1.0 + q * (L.vignetting[0] + q * (L.vignetting[1] + q * L.vignetting[2]));
      if (!(v > 0.0)) {
        *why = formatted("lens %d: the falloff V(r) of vignetting (%g, %g, %g) reaches %g at r = %.4f, inside the lens's theta_d(maxAngle) %.4f",
                         i, L.vignetting[0], L.vignetting[1], L.vignetting[2], v, r, rMax);
        return true;
      }
    }
  }
  return false;
}

// true, with the reason in *why, when the photometric lens call cannot serve ctx with this rig, photometry, seam and
// orientation: the lens call's refusals (seamWidth = 0, the hard seam) or the blend call's (seamWidth > 0), and
// photometryRefused's
bool lensPhotoRefused(const FrameTransformContext& ctx, const T360LensRig* rig, const T360RigPhotometry* ph, float seamWidth,
                      const T360Orientation* o, std::string* why) {
  if (seamWidthRefused(seamWidth, why)) return true;
  if (seamWidth > 0.0f ? lensBlendRefused(ctx, rig, seamWidth, o, why) : lensRefused(ctx, rig, o, why)) return true;
  return photometryRefused(*rig, ph, why);
}

// The per-frame constants of plane `plane` (0 luma, 1 and 2 chroma) of a rig's photometry (oriented_view.h: LensPhotoPlane);
// lens 1's stay zero for a one-lens rig
t360::LensPhotoPlane lensPhotoPlane(const T360RigPhotometry& ph, int numLenses, int plane) {
  t360::LensPhotoPlane c{};
  c.pivot = plane == 0 ? ph.lumaPivot : 128;
  for (int i = 0; i < numLenses; ++i) {
    const T360LensPhotometry& L = ph.lens[i];
    for (int k = 0; k < 3; ++k) c.v[i][k] = L.vignetting[k];
    c.gain[i] = L.gain[plane];
    c.offset[i] = static_cast<int>(std::lround(16.0 * static_cast<double>(L.offset[plane])));  // (half away from zero)
  }
  return c;
}

// The context the lens path renders with: the output fields of ctx, a mono equirect-like input (the fields the rig
// replaces, which play no part in the output half of the chain), no scaling
FrameTransformContext lensContext(const FrameTransformContext& ctx) {
  FrameTransformContext c = ctx;
  c.input_layout = LAYOUT_EQUIRECT;
  c.input_stereo_format = STEREO_FORMAT_MONO;
  c.output_stereo_format = STEREO_FORMAT_MONO;
  c.input_expand_coef = 1.0f;
  c.width_scale_factor = c.height_scale_factor = 1.0f;
  return c;
}

// The host twin of the lens kernels for one outW x outH plane of an inW x inH input: point(g, r, colTab, rowTab, i, j,
// i * outW + j) for every output pixel, with the geometry, tables and rotation those kernels get for ctx and o
template <class Point>
void forLensPixels(const FrameTransformContext& ctx, const T360Orientation& o, int inW, int inH, int outW, int outH, Point&& point) {
  const t360::SphereGeometry g = t360::sphereGeometry(lensContext(ctx), outW, outH, inW, inH, t360::kernelSizeOf(ctx.interpolation_alg));
  const std::vector<float> tables = t360::buildSphereTables(g);
  const float* colTab = tables.data();
  const float* rowTab = tables.empty() ? nullptr : tables.data() + t360::sphereTableRowOffset(g);
  const t360::Rotation r = t360::rotationFromAngles(o.yaw, o.pitch, o.roll);
  for (int i = 0; i < outH; ++i)
    for (int j = 0; j < outW; ++j) point(g, r, colTab, rowTab, i, j, static_cast<size_t>(i) * outW + j);
}

// ---- camera views: the rectilinear, camera, anti-aliased (mip), photometric and stereo calls (T360B200_cameraMap and
// T360B200_transformFrameCameraAsync, the rectilinear pair, which is the pinhole camera, T360B200_cameraMipMaps, ...CameraMip...,
// ...CameraPhoto... and ...StereoCamera...; oriented_view.h: rectilinearSample, mipCameraSample, cameraPhotoSample) --------
static_assert(T360_CAMERA_PINHOLE == t360::kCameraPinhole && T360_CAMERA_EQUIDISTANT == t360::kCameraEquidistant &&
              T360_CAMERA_STEREOGRAPHIC == t360::kCameraStereographic && T360_CAMERA_PANNINI == t360::kCameraPannini &&
              T360_CAMERA_EQUIRECT == t360::kCameraEquirect);
constexpr T360Camera kPinhole{T360_CAMERA_PINHOLE, 0.0f};

// What a camera call was given; the arguments a call does not take stay NULL / 0.  rig == nullptr: a view of the
// context's input.  photometric: the call corrects the rig's lenses, so it needs a rig and a photometry (the photometric
// and stereo calls); stereo: each eye takes its own lens (no seam).  minify == nullptr: no pyramid.  motion: a rig motion
// over the readout (the camera-motion calls: a photometric view).  aniso: the anisotropic calls, maxProbes probes per
// pixel along its footprint's longer axis (a plain view with a minify).
struct CameraView {
  const T360LensRig* rig = nullptr;
  const T360RigPhotometry* photometry = nullptr;
  float seamWidth = 0.0f;
  const T360Pose* pose = nullptr;
  const T360Camera* camera = nullptr;
  const T360Minify* minify = nullptr;
  unsigned long long* stats = nullptr;
  bool photometric = false;
  bool stereo = false;
  const T360RigMotion* motion = nullptr;
  bool moving = false;  // (the camera-motion calls: motion is checked, NULL included)
  int maxProbes = 1;
  bool aniso = false;   // (the anisotropic calls: maxProbes is checked, and so is a NULL minify)
};
// A view of ctx's input (rig == nullptr) or of a rig's lenses as they are: the rectilinear, camera and camera-mip calls
CameraView plainView(const T360LensRig* rig, const T360Pose* pose, const T360Camera* camera, const T360Minify* minify = nullptr) {
  return {rig, nullptr, 0.0f, pose, camera, minify};
}
// A view of a rig's lenses with photometry: the photometric call, and the stereo call (seamWidth 0)
CameraView photoView(const T360LensRig* rig, const T360RigPhotometry* photometry, float seamWidth, const T360Pose* pose, const T360Camera* camera,
                     const T360Minify* minify, unsigned long long* stats, bool stereo) {
  return {rig, photometry, seamWidth, pose, camera, minify, stats, true, stereo};
}
// A view of a rig's lenses with photometry and a rig motion: the camera-motion calls
CameraView motionView(const T360LensRig* rig, const T360RigPhotometry* photometry, float seamWidth, const T360Pose* pose, const T360Camera* camera,
                      const T360Minify* minify, const T360RigMotion* motion, unsigned long long* stats) {
  CameraView v = photoView(rig, photometry, seamWidth, pose, camera, minify, stats, false);
  v.motion = motion;
  v.moving = true;
  return v;
}

// A view of ctx's input or of a rig's lenses with up to maxProbes probes per pixel: the anisotropic calls
CameraView anisoView(const T360LensRig* rig, const T360Pose* pose, const T360Camera* camera, const T360Minify* minify, int maxProbes) {
  CameraView v = plainView(rig, pose, camera, minify);
  v.maxProbes = maxProbes;
  v.aniso = true;
  return v;
}

// true, with the reason in *why, when maxProbes is not a power of two in 1..16
bool maxProbesRefused(int maxProbes, std::string* why) {
  if (maxProbes == 1 || maxProbes == 2 || maxProbes == 4 || maxProbes == 8 || maxProbes == 16) return false;
  *why = formatted("maxProbes %d is not 1, 2, 4, 8 or 16", maxProbes);
  return true;
}

// log2 maxProbes, the form the footprint and the kernels take it in
int probesLog2(int maxProbes) {
  int e = 0;
  while ((2 << e) <= maxProbes) ++e;
  return e;
}

// true, with the reason in *why, when `minify` is NULL or out of range
bool minifyRefused(const T360Minify* minify, std::string* why) {
  if (!minify) {
    *why = "a NULL minify";
    return true;
  }
  if (minify->maxLevel < 0 || minify->maxLevel > t360::kMipMaxLevels) {
    *why = formatted("maxLevel %d is outside [0, %d]", minify->maxLevel, t360::kMipMaxLevels);
    return true;
  }
  if (!std::isfinite(minify->lodBias) || !(minify->lodBias >= -4.0f && minify->lodBias <= 4.0f)) {
    *why = formatted("lodBias %g must be finite and lie in [-4, 4]", minify->lodBias);
    return true;
  }
  return false;
}

// true, with the reason in *why, when view v of ctx's input or of its rig cannot be rendered, in this order: a photometric
// view's NULL rig; a stereo rig without two lenses or an output_stereo_format other than TB, LR or MONO; the pose, the
// camera and its fields of view, the rig (rigRefused), the low-pass filter and the interpolation; a photometric view's
// seam (seamWidthRefused, featherRefused) and photometry (photometryRefused); the minify where there is one (an
// anisotropic view's NULL minify included); a moving view's motion (motionRefused); an anisotropic view's maxProbes
// (maxProbesRefused).  The output layout plays no part: the pose replaces it.
bool viewRefused(const FrameTransformContext& ctx, const CameraView& v, std::string* why) {
  if (v.photometric && !v.rig) {
    *why = v.stereo ? "a NULL rig (a stereo rig's lenses are its eyes)" : "a NULL rig (the photometry corrects a rig's lenses)";
    return true;
  }
  if (v.stereo) {
    if (v.rig->numLenses != 2) {
      *why = formatted("numLenses %d: a stereo rig has two lenses, lens 0 the left eye's and lens 1 the right eye's", v.rig->numLenses);
      return true;
    }
    const int sf = ctx.output_stereo_format;
    if (sf != STEREO_FORMAT_TB && sf != STEREO_FORMAT_LR && sf != STEREO_FORMAT_MONO) {
      *why = formatted("output_stereo_format %d (a stereo rig's views are LR, TB or MONO: eye 0 alone)", sf);
      return true;
    }
  }
  const T360Pose* pose = v.pose;
  if (!pose) {
    *why = "a NULL pose";
    return true;
  }
  if (!std::isfinite(pose->yaw) || !std::isfinite(pose->pitch) || !std::isfinite(pose->roll) || !std::isfinite(pose->hfov) ||
      !std::isfinite(pose->vfov)) {
    *why = formatted("the pose (yaw %g, pitch %g, roll %g, hfov %g, vfov %g) is not finite", pose->yaw, pose->pitch, pose->roll, pose->hfov,
                     pose->vfov);
    return true;
  }
  if (!v.camera) {
    *why = "a NULL camera";
    return true;
  }
  const float h = pose->hfov, vf = pose->vfov;
  switch (v.camera->model) {
    case T360_CAMERA_PINHOLE:
      if (!(h > 0.0f && h <= 179.0f) || !(vf > 0.0f && vf <= 179.0f)) *why = formatted("hfov %g and vfov %g must lie in (0, 179] degrees", h, vf);
      break;
    case T360_CAMERA_EQUIDISTANT:
      if (!(h > 0.0f && h <= 360.0f) || !(vf > 0.0f && vf <= 360.0f))
        *why = formatted("hfov %g and vfov %g must lie in (0, 360] degrees for an equidistant camera", h, vf);
      break;
    case T360_CAMERA_STEREOGRAPHIC:
      if (!(h > 0.0f && h <= 359.0f) || !(vf > 0.0f && vf <= 359.0f))
        *why = formatted("hfov %g and vfov %g must lie in (0, 359] degrees for a stereographic camera", h, vf);
      break;
    case T360_CAMERA_PANNINI: {
      const float d = v.camera->pannini;
      if (!(d >= 0.0f && d <= 1.0f)) *why = formatted("the Pannini distance %g must lie in [0, 1]", d);
      else if (!(h > 0.0f && h <= 359.0f) || !(vf > 0.0f && vf <= 179.0f))
        *why = formatted("hfov %g must lie in (0, 359] and vfov %g in (0, 179] degrees for a Pannini camera", h, vf);
      else if (!(d + std::cos(static_cast<double>(h) * M_PI / 360.0) > 0.0))
        *why = formatted("a Pannini camera with distance %g sees at most 2 acos(-%g) degrees across, not hfov %g", d, d, h);
      break;
    }
    case T360_CAMERA_EQUIRECT:
      if (!(h > 0.0f && h <= 360.0f) || !(vf > 0.0f && vf <= 180.0f))
        *why = formatted("hfov %g must lie in (0, 360] and vfov %g in (0, 180] degrees for an equirect camera", h, vf);
      break;
    default:
      *why = formatted("no camera model %d", v.camera->model);
  }
  if (!why->empty()) return true;
  if (v.rig && rigRefused(v.rig, why)) return true;
  if (ctx.enable_low_pass_filter) {
    *why = "the low-pass filter is not available for a camera view (set enable_low_pass_filter = 0)";
    return true;
  }
  if (t360::kernelSizeOf(ctx.interpolation_alg) == 0) {
    *why = formatted("no interpolation algorithm %d", static_cast<int>(ctx.interpolation_alg));
    return true;
  }
  if (v.photometric) {
    if (seamWidthRefused(v.seamWidth, why) || (v.seamWidth > 0.0f && featherRefused(*v.rig, v.seamWidth, why))) return true;
    if (photometryRefused(*v.rig, v.photometry, why)) return true;
  }
  if ((v.minify || v.aniso) && minifyRefused(v.minify, why)) return true;
  if (v.moving && motionRefused(*v.rig, v.motion, why)) return true;
  return v.aniso && maxProbesRefused(v.maxProbes, why);
}

// The per-frame constants of v's pose and camera (oriented_view.h: cameraConstants)
t360::RectilinearCamera cameraConstants(const CameraView& v) {
  return t360::cameraConstants(v.camera->model, v.camera->pannini, v.pose->yaw, v.pose->pitch, v.pose->roll, v.pose->hfov, v.pose->vfov);
}

// round(256 lodBias), half away from zero: the bias in 1/256 of a level
int mipBias(const T360Minify& m) { return static_cast<int>(std::lround(256.0 * static_cast<double>(m.lodBias))); }

// The geometry of one outW x outH plane of an inW x inH input in view v: ctx's (its stereo formats and input layout,
// cube-map input_expand_coef), or with a rig lensContext's (mono); a stereo rig's takes the output eye split of ctx's
// output_stereo_format (whatever input_stereo_format says).  No tables.
t360::SphereGeometry viewGeometry(const FrameTransformContext& ctx, const CameraView& v, int inW, int inH, int outW, int outH) {
  t360::SphereGeometry g = t360::sphereGeometry(v.rig ? lensContext(ctx) : ctx, outW, outH, inW, inH, t360::kernelSizeOf(ctx.interpolation_alg));
  if (v.stereo) {
    g.splitLR = ctx.output_stereo_format == STEREO_FORMAT_LR;
    g.splitTB = ctx.output_stereo_format == STEREO_FORMAT_TB;
  }
  return g;
}

// The host twin of the camera kernels for one outW x outH plane of an inW x inH input: point(g, c, model, m, bias, i, j,
// i * outW + j) for every output pixel, with the geometry, camera constants (oriented_view.h: cameraConstants), rig model
// (empty without a rig), footprint constants (maxLevel 0 without a minify) and bias those kernels get for ctx and v.  The
// arguments are not refused.
template <class Point>
void forCameraPixels(const FrameTransformContext& ctx, const CameraView& v, int inW, int inH, int outW, int outH, Point&& point) {
  const t360::SphereGeometry g = viewGeometry(ctx, v, inW, inH, outW, outH);
  const t360::RectilinearCamera c = cameraConstants(v);
  const t360::LensRigModel model = v.rig ? lensRigModel(*v.rig) : t360::LensRigModel{};
  const t360::MipGeometry m = t360::mipGeometry(g, v.minify ? v.minify->maxLevel : 0);
  const int bias = v.minify ? mipBias(*v.minify) : 0;
  for (int i = 0; i < outH; ++i)
    for (int j = 0; j < outW; ++j) point(g, c, model, m, bias, i, j, static_cast<size_t>(i) * outW + j);
}

// ---- the entry points' guards --------------------------------------------------------------------------------------------
// true, with the reason in *why, when `name` (a lens or plane index) is outside 0..hi
bool indexRefused(const char* name, int value, int hi, std::string* why) {
  if (value >= 0 && value <= hi) return false;
  *why = formatted("%s %d is outside 0..%d", name, value, hi);
  return true;
}

// true, with `message` in *why, when an output array is NULL or a plane size is not positive
bool outputsRefused(std::initializer_list<const void*> arrays, int inW, int inH, int outW, int outH, const char* message, std::string* why) {
  if (std::find(arrays.begin(), arrays.end(), nullptr) == arrays.end() && inW > 0 && inH > 0 && outW > 0 && outH > 0) return false;
  *why = message;
  return true;
}

// A host twin: a NULL context, then refused(*ctx, &why) (the call's refusals, then its own array, size and index checks),
// then body(*ctx).  0 and "<what>. Error: <why>" on stdout when refused, else 1.
template <class Refused, class Body>
int twinCall(const char* what, const FrameTransformContext* ctx, Refused&& refused, Body&& body) {
  std::string why;
  if (!ctx) why = "a NULL context";
  else refused(*ctx, &why);
  if (!why.empty()) {
    std::printf("%s. Error: %s\n", what, why.c_str());
    return 0;
  }
  body(*ctx);
  return 1;
}

}  // namespace

class VideoFrameTransform {
 public:
  explicit VideoFrameTransform(FrameTransformContext* ctx) {
    std::memcpy(&ctx_, ctx, sizeof(ctx_));
    const char* e = std::getenv("T360B200_PIN_HOST_PLANES");
    pinHostPlanes_ = e && *e && *e != '0';
    if (const char* m = std::getenv("T360B200_PIPELINE_MIN_BYTES")) pipelineMinBytes_ = std::atoll(m);  // tests: 0 = always
    const char* strict = std::getenv("T360B200_PIPELINE_STRICT");
    pipelineStrict_ = strict && *strict && *strict != '0';
  }
  void setPinHostPlanes(bool on) { pinHostPlanes_ = on; }

  ~VideoFrameTransform() {
    {  // the background planner finishes the plan it is making, if any, and installs nothing more
      std::lock_guard<std::mutex> async(asyncMu_);
      asyncStop_ = true;
    }
    asyncCv_.notify_all();
    if (worker_.joinable()) worker_.join();
    if (deviceReady_) {
      cudaSetDevice(device_);
      plans_.clear();
      for (auto& w : weights_) w.release();
      for (auto& w : weightImages_) w.release();
      stagingIn_.release(); stagingOut_.release();
      for (HostRange& r : hostRanges_)
        if (r.pinned) cudaHostUnregister(reinterpret_cast<void*>(r.base));
      for (auto& kv : slots_) {
        for (PlaneLane& l : kv.second->lanes) {
          l.blurred.release();
          l.scaled.release();
          l.claimCounter.release();
          if (l.main) cudaStreamDestroy(l.main);
          if (l.done) cudaEventDestroy(l.done);
        }
        kv.second->frameClaim.release();
        if (kv.second->fork) cudaEventDestroy(kv.second->fork);
        for (UploadRing* ring : {&kv.second->viewJobs, &kv.second->viewTaps, &kv.second->sphereTables, &kv.second->motionTables})
          for (UploadRing::Entry& e : ring->entries) {
            if (e.released) cudaEventSynchronize(e.released);
            if (e.device) cudaFree(e.device);
            if (e.host) cudaFreeHost(e.host);
            if (e.released) cudaEventDestroy(e.released);
          }
      }
      for (FrameLists& f : frameLists_) {
        f.gatherJobs.release();
        f.blurImage.release();
      }
      trace_.release();
      for (cudaEvent_t e : chunkIn_) cudaEventDestroy(e);
      for (cudaEvent_t e : waveDone_) cudaEventDestroy(e);
      for (cudaEvent_t e : copiedOut_) cudaEventDestroy(e);
      for (WavePlan& w : wavePlans_) w.jobs.release();
      for (PlaneGraph& g : planeGraphs_) cudaGraphExecDestroy(g.exec);
      for (cudaEvent_t e : {graphFork_, graphJoinIn_, graphJoinOut_}) if (e) cudaEventDestroy(e);
      if (copyIn_) cudaStreamDestroy(copyIn_);
      if (copyOut_) cudaStreamDestroy(copyOut_);
      if (stream_) cudaStreamDestroy(stream_);
    }
  }

  // reference generateMapForPlane (cpp:504-576): plan on the host, upload once.
  bool generateMapForPlane(int inW, int inH, int outW, int outH, int planIndex) {
    return installPlan(planIndex, [&](const FrameTransformContext& ctx, HostIndexPlan& host) {
      return planOnHost(ctx, inW, inH, outW, outH, host);
    });
  }

  // T360B200_generateMapFromWarp: as generateMapForPlane, from the caller's map (buildWarpHostPlan refuses before any CUDA
  // call)
  bool generateMapFromWarp(const float* map, int mapW, int mapH, int inW, int inH, int border, int planIndex) {
    return installPlan(planIndex, [&](const FrameTransformContext& c, HostIndexPlan& host) {
      return planWarpOnHost(c, map, mapW, mapH, inW, inH, border, host);
    });
  }

  // Plans index planIndex on the host with the current context (plan(ctx, host), false: refused with a message), uploads it
  // and installs it in place of the index's previous plan.
  template <class Plan>
  bool installPlan(int planIndex, Plan&& plan) {
    return guarded("Could not generate map for plane " + std::to_string(planIndex), [&] {
      reconfigureWait(true);  // a pending reconfigureAsync re-plans the other indices: it is finished first
      std::lock_guard<std::mutex> planLock(planMu_);
      FrameTransformContext ctx;
      {
        std::shared_lock<std::shared_mutex> config(configMu_);
        ctx = ctx_;
      }
      HostIndexPlan host;
      if (!plan(ctx, host)) return false;
      const DeviceRestore restoreDevice = ensureDevice();
      DevicePlan d = upload(host, ctx);
      std::lock_guard<std::mutex> lock(mu_);
      plans_[planIndex] = std::move(d);
      ++planGeneration_;
      return true;
    });
  }

  // Replaces the context of a running transform: every plan index is re-planned for `next` with the sizes it was
  // generated with.  Host planning (all indices at once) and the upload run while other threads keep enqueuing frames with
  // the old plans; the entry points are held off only while the plans are swapped (install), and the old plans are
  // released once the device has finished the work enqueued before the swap (retire).  A pending reconfigureAsync is
  // discarded.  On any failure the old configuration stays in effect.
  bool reconfigure(const FrameTransformContext& next) {
    return guarded("Could not reconfigure the transform", [&] {
      std::lock_guard<std::mutex> planLock(planMu_);  // (one re-plan at a time, also against generateMapForPlane)
      if (refuseWarpPlans("Could not reconfigure the transform")) return false;
      unsigned long long seq;
      {
        std::lock_guard<std::mutex> async(asyncMu_);
        seq = asyncSeq_;
      }
      const std::vector<PlanSizes> sizes = plannedSizes();
      if (sizes.empty()) {  // nothing planned yet: the next generateMapForPlane uses the new context (no CUDA call here)
        std::unique_lock<std::shared_mutex> config(configMu_);
        std::memcpy(&ctx_, &next, sizeof(ctx_));
        return true;
      }
      std::vector<HostIndexPlan> host;
      if (!planAll(next, sizes, host, "Could not reconfigure the transform")) return false;
      const DeviceRestore restoreDevice = ensureDevice();
      PlanSet set = makePlanSet(next, sizes, host);
      install(set, next, seq, true);
      retire(set);
      return true;
    });
  }

  // T360B200_reconfigureAsync: `next` is in effect for every frame enqueued after the call returns; until its plans are in,
  // whole frames take the per-frame kernels (perFrameLocked) and the per-plane entry points wait for the plans.  The plans are
  // made by the background planner (planInBackground).  Host checks only: every refusal comes before any CUDA call, and so
  // does the return.
  bool reconfigureAsync(const FrameTransformContext& next) {
    if (refuseWarpPlans("Could not reconfigure the transform asynchronously")) return false;
    const std::vector<PlanSizes> sizes = plannedSizes();
    if (const char* why = asyncRefusal(next, sizes)) {
      std::printf("Could not reconfigure the transform asynchronously. Error: %s\n", why);
      return false;
    }
    {
      std::unique_lock<std::shared_mutex> config(configMu_);  // no call of an entry point is in progress from here on
      if (ctx_.input_layout != next.input_layout || ctx_.output_layout != next.output_layout ||
          ctx_.input_stereo_format != next.input_stereo_format || ctx_.output_stereo_format != next.output_stereo_format ||
          ctx_.width_scale_factor != next.width_scale_factor || ctx_.height_scale_factor != next.height_scale_factor) {
        std::printf("Could not reconfigure the transform asynchronously. Error: the layouts, stereo formats and scale factors size "
                    "the planes and maps and cannot change here (T360B200_reconfigure can change them)\n");
        return false;
      }
      std::memcpy(&ctx_, &next, sizeof(ctx_));
      if (sizes.empty()) return true;  // nothing planned yet: the next generateMapForPlane uses the new context
      perFrameOnly_ = true;
      std::lock_guard<std::mutex> async(asyncMu_);
      ++asyncSeq_;
      asyncCtx_ = next;
      asyncLast_ = std::chrono::steady_clock::now();
      if (!worker_.joinable()) worker_ = std::thread(&VideoFrameTransform::planInBackground, this);
    }
    asyncCv_.notify_all();
    return true;
  }

  // T360B200_reconfigureWait: 1 when the plans of the current context are in effect, -1 when the background planner failed
  // on it, else 0 (block = false) or, with block, the result once the planner has finished -- without the settle interval,
  // and only after the plans the swap replaced have been released (asyncRetiring_), so device memory is back when it returns.
  int reconfigureWait(bool block) {
    std::unique_lock<std::mutex> async(asyncMu_);
    if (block) {
      if (asyncSettled_ != asyncSeq_) {
        asyncHurry_ = true;
        asyncCv_.notify_all();
      }
      asyncCv_.wait(async, [this] { return (asyncSettled_ == asyncSeq_ && !asyncRetiring_) || asyncStop_; });
    }
    if (asyncSettled_ != asyncSeq_) return 0;
    return asyncFailed_ ? -1 : 1;
  }

  // reference transformFramePlane (cpp:1319-1351): host or device planes, synchronous.
  bool transformFramePlane(uint8_t* in, uint8_t* out, int inW, int inH, int inPitch, int outW, int outH, int outPitch,
                           int planIndex, int imagePlaneIndex) {
    const std::string what = "Could not transform the plane " + std::to_string(imagePlaneIndex);
    return guarded(what, [&] {
      if (!in || !out || inW <= 0 || inH <= 0 || outW <= 0 || outH <= 0 || inPitch < inW || outPitch < outW) {
        std::printf("%s. Error: invalid plane description\n", what.c_str());
        return false;
      }
      std::shared_lock<std::shared_mutex> config = lockPlanned("Could not transform the plane");
      if (!config.owns_lock()) return false;
      const DeviceRestore restoreDevice = ensureDevice();
      const DevicePlan* plan = findPlan(planIndex, imagePlaneIndex);
      if (!plan) return false;
      {  // the same plan and caller buffers as in an earlier streamed call: replay its graph (no driver query, no set-up)
        std::lock_guard<std::mutex> hostLock(hostCallMu_);
        if (PlaneGraph* g = findPlaneGraph(*plan, in, out, inW, inH, inPitch, outW, outH, outPitch)) return replayPlaneGraph(*g);
      }
      const bool inOnDevice = isDevicePointer(in), outOnDevice = isDevicePointer(out);
      if (plan->kernelSize == 0) {  // reference cpp:780-784: message, output untouched, true
        std::printf("Could not find interpolation algorithm for plane %d", imagePlaneIndex);
        return true;
      }
      // (the reference object may be called from several threads on different planes; here such calls take turns)
      std::lock_guard<std::mutex> hostLock(hostCallMu_);
      if (!inOnDevice && !outOnDevice && pipelineEligible(*plan, inW, inH, outW, outH))
        return transformHostPlanePipelined(*plan, in, out, inW, inH, inPitch, outW, outH, outPitch, planIndex, imagePlaneIndex);
      const uint8_t* dIn = in;
      uint8_t* dOut = out;
      int dInPitch = inPitch, dOutPitch = outPitch;
      // (both planes before any copy: pinning one may re-register a range the other one is copied from)
      if (!inOnDevice) pinIfRecurring(in, static_cast<size_t>(inPitch) * (inH - 1) + inW);
      if (!outOnDevice) pinIfRecurring(out, static_cast<size_t>(outPitch) * (outH - 1) + outW);
      if (!inOnDevice) {
        dInPitch = scratchPlane(stagingIn_, inW, inH);
        CU(cudaMemcpy2DAsync(stagingIn_.ptr, dInPitch, in, inPitch, inW, inH, cudaMemcpyHostToDevice, stream_));
        dIn = stagingIn_.ptr;
      }
      if (!outOnDevice) {
        dOutPitch = scratchPlane(stagingOut_, outW, outH);
        dOut = stagingOut_.ptr;
        // a transparent luma plane keeps the caller's bytes (renderTarget): they go into the staging plane first
        if (plan->transparent && !planIndex)
          CU(cudaMemcpy2DAsync(dOut, dOutPitch, out, outPitch, outW, outH, cudaMemcpyHostToDevice, stream_));
      }
      if (!enqueue(*plan, planIndex != 0, dIn, dOut, inW, inH, dInPitch, outW, outH, dOutPitch, stream_, imagePlaneIndex,
                   slotFor(stream_).lanes[0]))
        return false;
      if (!outOnDevice)
        CU(cudaMemcpy2DAsync(out, outPitch, dOut, dOutPitch, outW, outH, cudaMemcpyDeviceToHost, stream_));
      CU(cudaStreamSynchronize(stream_));
      return true;
    });
  }

  // ---- streaming a large host plane through the device -------------------------------------------------------
  bool pipelineEligible(const DevicePlan& plan, int inW, int inH, int outW, int outH) const {
    return plan.numJobs > 0 && !plan.transparent && !plan.lowPass && inW == plan.inW && inH == plan.inH &&
           outW == plan.mapW && outH == plan.mapH && static_cast<long long>(inW) * inH >= pipelineMinBytes_ && inH >= 64;
  }

  WavePlan& wavePlanFor(const DevicePlan& plan, int planIndex, int chunks) {
    WavePlan& w = wavePlans_[planIndex ? 1 : 0];
    if (w.plan == &plan && w.chunks == chunks && w.generation == planGeneration_) return w;
    w.chunks = chunks;
    w.plan = &plan;
    w.generation = planGeneration_;
    w.schedule = t360::scheduleWaves(plan.jobNeedRows, plan.jobRects, plan.inH, plan.mapW, plan.mapH, chunks);
    std::vector<GatherJob> all;
    all.reserve(w.schedule.order.size());
    for (int i : w.schedule.order) all.push_back(plan.hostJobs[i]);
    w.jobs.reserve(all.size());
    CU(cudaMemcpy(w.jobs.ptr, all.data(), all.size() * sizeof(GatherJob), cudaMemcpyHostToDevice));
    return w;
  }

  // The graph of an earlier streamed call with this plan, these caller planes and the current staging planes, or nullptr.
  // Graphs made for replaced plans or staging planes are forgotten first.
  PlaneGraph* findPlaneGraph(const DevicePlan& plan, const uint8_t* in, const uint8_t* out, int inW, int inH, int inPitch, int outW, int outH,
                             int outPitch) {
    PlaneGraph* g = nullptr;
    for (size_t i = 0; i < planeGraphs_.size();) {
      PlaneGraph& c = planeGraphs_[i];
      if (c.stagingIn != stagingIn_.ptr || c.stagingOut != stagingOut_.ptr || c.generation != planGeneration_) {
        cudaGraphExecDestroy(c.exec);
        planeGraphs_.erase(planeGraphs_.begin() + static_cast<long>(i));
        continue;
      }
      if (c.plan == &plan && c.in == in && c.out == out && c.inPitch == inPitch && c.outPitch == outPitch && c.inW == inW && c.inH == inH &&
          c.outW == outW && c.outH == outH)
        g = &c;
      ++i;
    }
    return g;
  }

  bool replayPlaneGraph(PlaneGraph& g) {
    g.lastUse = ++graphClock_;
    CU(cudaGraphLaunch(g.exec, stream_));
    t360::countKernelLaunches(g.kernels);
    CU(cudaStreamSynchronize(stream_));
    return true;
  }

  // reference transformFramePlane for large host planes (same result as the plain path): chunked H2D || gather || D2H
  bool transformHostPlanePipelined(const DevicePlan& plan, uint8_t* in, uint8_t* out, int inW, int inH, int inPitch, int outW, int outH,
                                   int outPitch, int planIndex, int imagePlaneIndex) {
    const int chunks = t360::pipelineChunks(inW, inH);
    WavePlan& w = wavePlanFor(plan, planIndex, chunks);
    const t360::WaveSchedule& ws = w.schedule;
    if (!copyIn_) {
      CU(cudaStreamCreateWithFlags(&copyIn_, cudaStreamNonBlocking));
      CU(cudaStreamCreateWithFlags(&copyOut_, cudaStreamNonBlocking));
      for (cudaEvent_t* e : {&graphFork_, &graphJoinIn_, &graphJoinOut_}) CU(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    }
    while (static_cast<int>(chunkIn_.size()) < chunks) {
      for (std::vector<cudaEvent_t>* v : {&chunkIn_, &waveDone_, &copiedOut_}) {
        cudaEvent_t e = nullptr;
        CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        v->push_back(e);
      }
    }
    pinIfRecurring(in, static_cast<size_t>(inPitch) * (inH - 1) + inW);
    pinIfRecurring(out, static_cast<size_t>(outPitch) * (outH - 1) + outW);
    const int dInPitch = scratchPlane(stagingIn_, inW, inH), dOutPitch = scratchPlane(stagingOut_, outW, outH);
    PlaneLane& hostLane = slotFor(stream_).lanes[0];
    GatherWork work;
    if (!prepareGather(plan, planIndex != 0, stagingIn_.ptr, stagingOut_.ptr, inW, inH, dInPitch, outW, outH, dOutPitch, stream_,
                       imagePlaneIndex, hostLane, work))
      return false;
    if (!work.staged) {  // the plane cannot be described to the TMA unit after all: plain path
      CU(cudaMemcpy2DAsync(stagingIn_.ptr, dInPitch, in, inPitch, inW, inH, cudaMemcpyHostToDevice, stream_));
      gatherPlane(work, hostLane, stream_);
      CU(cudaMemcpy2DAsync(out, outPitch, stagingOut_.ptr, dOutPitch, outW, outH, cudaMemcpyDeviceToHost, stream_));
      CU(cudaStreamSynchronize(stream_));
      return true;
    }
    armScheduler(hostLane.claimCounter, stream_);
    CU(t360::prepareGatherFrame(plan.kernelSize));
    // pipelineStrict_ (T360B200_PIPELINE_STRICT): the staging planes start out poisoned, chunk c + 1 is uploaded only after
    // wave c, and wave c + 1 runs only after wave c's rectangles are back on the host.  A legal order of the same work in
    // which a job that reads rows not yet delivered, or a band copied back before its last writer, gives wrong bytes on
    // every call instead of only when a copy loses its race against a kernel.
    auto issue = [&](bool forkJoin) {
      if (pipelineStrict_) {
        CU(cudaMemsetAsync(stagingIn_.ptr, kStrictPoison, static_cast<size_t>(dInPitch) * inH, stream_));
        CU(cudaMemsetAsync(stagingOut_.ptr, kStrictPoison, static_cast<size_t>(dOutPitch) * outH, stream_));
      }
      if (forkJoin || pipelineStrict_) {  // (capture: the side streams become branches of the graph)
        CU(cudaEventRecord(graphFork_, stream_));
        CU(cudaStreamWaitEvent(copyIn_, graphFork_, 0));
        CU(cudaStreamWaitEvent(copyOut_, graphFork_, 0));
      }
      t360::FrameGatherParams fp{};
      fp.plane[0] = work.view;
      fp.weightImage = reinterpret_cast<const uint4*>(weightImages_[plan.kernelSize].ptr);
      fp.kernelSize = plan.kernelSize;
      fp.numPlanes = 1;
      for (int c = 0; c < chunks; ++c) {
        const int r0 = c ? ws.chunkRowEnd[c - 1] : 0, r1 = ws.chunkRowEnd[c];
        if (r1 > r0)
          CU(cudaMemcpy2DAsync(stagingIn_.ptr + static_cast<size_t>(r0) * dInPitch, dInPitch, in + static_cast<size_t>(r0) * inPitch, inPitch, inW,
                               r1 - r0, cudaMemcpyHostToDevice, copyIn_));
        CU(cudaEventRecord(chunkIn_[c], copyIn_));
        CU(cudaStreamWaitEvent(stream_, chunkIn_[c], 0));
        if (pipelineStrict_ && c) CU(cudaStreamWaitEvent(stream_, copiedOut_[c - 1], 0));
        const int n = ws.waveStart[c + 1] - ws.waveStart[c];
        if (n > 0) {
          t360::StagedParams jobs{w.jobs.ptr + ws.waveStart[c], n, hostLane.claimCounter.ptr, nullptr};
          CU(t360::launchGatherFrame(fp, jobs, work.maps, numSMs_, stream_, /*programmatic=*/false));
        }
        if (!ws.rects[c].empty() || (pipelineStrict_ && c + 1 < chunks)) CU(cudaEventRecord(waveDone_[c], stream_));
        if (!ws.rects[c].empty()) {
          CU(cudaStreamWaitEvent(copyOut_, waveDone_[c], 0));
          for (const t360::JobRect& r : ws.rects[c])
            CU(cudaMemcpy2DAsync(out + static_cast<size_t>(r.y0) * outPitch + r.x0, outPitch,
                                 stagingOut_.ptr + static_cast<size_t>(r.y0) * dOutPitch + r.x0, dOutPitch, r.x1 - r.x0, r.y1 - r.y0,
                                 cudaMemcpyDeviceToHost, copyOut_));
        }
        if (pipelineStrict_ && c + 1 < chunks) {
          CU(cudaStreamWaitEvent(copyIn_, waveDone_[c], 0));
          CU(cudaEventRecord(copiedOut_[c], copyOut_));
        }
      }
      if (forkJoin) {
        CU(cudaEventRecord(graphJoinIn_, copyIn_));
        CU(cudaEventRecord(graphJoinOut_, copyOut_));
        CU(cudaStreamWaitEvent(stream_, graphJoinIn_, 0));
        CU(cudaStreamWaitEvent(stream_, graphJoinOut_, 0));
      }
    };
    if (memoryTypeOf(in) == cudaMemoryTypeHost && memoryTypeOf(out) == cudaMemoryTypeHost) {
      PlaneGraph* g = findPlaneGraph(plan, in, out, inW, inH, inPitch, outW, outH, outPitch);
      if (!g) {
        if (planeGraphs_.size() >= 24) {  // (a frame pool recycles a handful of buffers; forget the least recently used)
          auto oldest = std::min_element(planeGraphs_.begin(), planeGraphs_.end(), [](const PlaneGraph& a, const PlaneGraph& b) { return a.lastUse < b.lastUse; });
          cudaGraphExecDestroy(oldest->exec);
          planeGraphs_.erase(oldest);
        }
        CU(cudaStreamSynchronize(stream_));
        cudaGraph_t graph = nullptr;
        CU(cudaStreamBeginCapture(stream_, cudaStreamCaptureModeThreadLocal));
        try {
          issue(true);
        } catch (...) {
          cudaStreamEndCapture(stream_, &graph);
          if (graph) cudaGraphDestroy(graph);
          throw;
        }
        CU(cudaStreamEndCapture(stream_, &graph));
        cudaGraphExec_t exec = nullptr;
        const cudaError_t e = cudaGraphInstantiate(&exec, graph, 0);
        cudaGraphDestroy(graph);
        if (e != cudaSuccess) throw CudaFail{e, "cudaGraphInstantiate"};
        int kernels = 0;
        for (int c = 0; c < chunks; ++c) kernels += ws.waveStart[c + 1] > ws.waveStart[c];
        planeGraphs_.push_back(PlaneGraph{&plan, planGeneration_, in, out, inPitch, outPitch, stagingIn_.ptr, stagingOut_.ptr, inW, inH, outW, outH,
                                          kernels, exec, 0});
        g = &planeGraphs_.back();
        t360::countKernelLaunches(-kernels);  // (counted once while capturing; every replay counts)
      }
      return replayPlaneGraph(*g);
    }
    issue(false);
    CU(cudaStreamSynchronize(stream_));
    CU(cudaStreamSynchronize(copyOut_));
    return true;
  }

  // device to device, asynchronous
  bool transformDevice(const uint8_t* dIn, uint8_t* dOut, int inW, int inH, int inPitch, int outW, int outH,
                       int outPitch, int planIndex, cudaStream_t stream) {
    return guarded("Could not transform the plane " + std::to_string(planIndex), [&] {
      std::shared_lock<std::shared_mutex> config = lockPlanned("Could not transform the plane");
      if (!config.owns_lock()) return false;
      const DeviceRestore restoreDevice = ensureDevice();
      const DevicePlan* plan = findPlan(planIndex, planIndex);
      if (!plan) return false;
      cudaStream_t s = stream ? stream : stream_;
      return enqueue(*plan, planIndex != 0, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, s, planIndex, slotFor(s).lanes[0]);
    });
  }

  // Whole frame, device to device, asynchronous: plane 0 with plan 0 on the caller's stream, planes 1.. with plan 1
  // on their own lanes (the planes are independent: reference vf_transform360.c:368-397 loops over them).
  bool transformFrameDevice(const FramePlanes& f, cudaStream_t stream) {
    const int numPlanes = f.numPlanes;
    return guarded("Could not transform the frame", [&] {
      std::shared_lock<std::shared_mutex> config(configMu_);
      while (perFrameOnly_) {  // a reconfigureAsync is pending: the per-frame kernels serve planes of the planned sizes
        if (planesOfPlannedSize(f))
          return perFrameLocked("Could not transform the frame while its plan is pending", ctx_, f, stream);
        config.unlock();
        if (reconfigureWait(true) < 0) {
          std::printf("Could not transform the frame. Error: the background planner failed on the current context\n");
          return false;
        }
        config.lock();
      }
      const DeviceRestore restoreDevice = ensureDevice();
      cudaStream_t s = stream ? stream : stream_;
      StreamSlot& slot = slotFor(s);
      PlaneLane* lanes_ = slot.lanes;
      cudaEvent_t frameFork_ = slot.fork;
      const DevicePlan* plans[kPlaneLanes];
      bool sideWork = false;  // does any chroma plane have work before its gather (low-pass, pre-fill)?
      for (int p = 0; p < numPlanes; ++p) {
        if (!(plans[p] = findPlan(p ? 1 : 0, p))) return false;
        if (p) sideWork = sideWork || plans[p]->lowPass || plans[p]->transparent;
      }
      // Low-pass of all planes in one launch per vertical kernel size when every plane takes the strip kernel only
      const t360::BlurLists* lists[kPlaneLanes];
      bool clear[kPlaneLanes], lowPass = true;
      for (int p = 0; p < numPlanes; ++p) {
        lists[p] = &plans[p]->blur.lists;
        clear[p] = plans[p]->blur.needsClear;
        lowPass = lowPass && plans[p]->lowPass;
      }
      const bool mergedBlur = lowPass && mergeable(plans, lists, clear, numPlanes, f.inW, f.inH);
      if (mergedBlur) {
        blurFrame(plans, f, lanes_, s);
        sideWork = false;
      }
      // Stage 1, planes side by side (chroma on its own lanes): everything before the gather.
      const bool fork = numPlanes > 1 && sideWork;
      if (fork) CU(cudaEventRecord(frameFork_, s));
      GatherWork work[kPlaneLanes];
      bool allStaged = true;
      for (int p = numPlanes - 1; p >= 0; --p) {
        cudaStream_t ps = (p && fork) ? lanes_[p].main : s;
        if (p && fork) CU(cudaStreamWaitEvent(ps, frameFork_, 0));
        if (!prepareGather(*plans[p], p > 0, f.in[p], f.out[p], f.inW[p], f.inH[p], f.inPitch[p], f.outW[p], f.outH[p], f.outPitch[p], ps, p,
                           lanes_[p], work[p], mergedBlur))
          return false;
        allStaged = allStaged && work[p].staged;
      }
      if (allStaged && numPlanes > 1) {
        // Stage 2: ONE persistent launch gathers every plane (reference vf_transform360.c:368-397 loops over them).
        if (fork)
          for (int p = 1; p < numPlanes; ++p) {
            CU(cudaEventRecord(lanes_[p].done, lanes_[p].main));
            CU(cudaStreamWaitEvent(s, lanes_[p].done, 0));
          }
        gatherFrame(work, numPlanes, s, slot);
        for (int p = 0; p < numPlanes; ++p) finishTarget(work[p].target, s);
        return true;
      }
      // some plane needs the general kernel (barrel layouts, nearest, unaligned planes): per-plane launches
      if (numPlanes > 1 && !fork) CU(cudaEventRecord(frameFork_, s));
      for (int p = numPlanes - 1; p >= 0; --p) {
        cudaStream_t ps = p ? lanes_[p].main : s;
        if (p && !fork) CU(cudaStreamWaitEvent(ps, frameFork_, 0));
        if (work[p].plan->kernelSize) {
          gatherPlane(work[p], lanes_[p], ps);
          finishTarget(work[p].target, ps);
        }
        if (p) CU(cudaEventRecord(lanes_[p].done, ps));
      }
      for (int p = 1; p < numPlanes; ++p) CU(cudaStreamWaitEvent(s, lanes_[p].done, 0));
      return true;
    });
  }

  bool lowPassDevice(const uint8_t* dIn, uint8_t* dOut, int w, int h, int inPitch, int outPitch, int planIndex,
                     cudaStream_t stream) {
    return guarded("Could not filter plane " + std::to_string(planIndex), [&] {
      std::shared_lock<std::shared_mutex> config = lockPlanned("Could not filter the plane");
      if (!config.owns_lock()) return false;
      const DeviceRestore restoreDevice = ensureDevice();
      const DevicePlan* plan = findPlan(planIndex, planIndex);
      if (!plan) return false;
      if (!plan->lowPass) {
        std::printf("Could not filter plane %d. Error: plan has no low-pass stage\n", planIndex);
        return false;
      }
      runLowPass(*plan, dIn, dOut, w, h, inPitch, outPitch, stream ? stream : stream_);
      return true;
    });
  }

  // Whole frame with per-frame view fields (T360B200_transformFrameViewAsync, ...OrientedAsync, ...PoseAsync): the frame a
  // fresh transform would give for the context with the fields of `fields` (a T360View, T360Orientation or T360Pose, checked
  // by withFields) substituted, with no re-plan (perFrameLocked).  `what` names the call in the messages.
  template <class Fields>
  bool transformFrameWith(const char* what, const Fields& fields, const FramePlanes& f, cudaStream_t stream) {
    std::shared_lock<std::shared_mutex> config(configMu_);
    if (refuseWarpPlans(what)) return false;
    FrameTransformContext ctx = ctx_;
    const std::string why = withFields(ctx, fields);
    if (!why.empty()) {
      std::printf("%s. Error: %s\n", what, why.c_str());
      return false;
    }
    return perFrameLocked(what, ctx, f, stream);
  }

  // Whole frame through the caller's per-plane device maps (T360B200_remapFrameAsync): one gather launch for all planes,
  // every record computed from its map entry as quantizeWarpMap does, so a map gives what generateMapFromWarp plans for it.
  // Needs no plan; the interpolation comes from the current context.  Every refusal comes before the first CUDA call, and
  // nothing here synchronises the device.
  bool remapFrame(const float* const* maps, const int* mapPitch, int border, const FramePlanes& f, cudaStream_t stream) {
    auto refused = [&](const FrameTransformContext& ctx, std::string* why) { return mapRefused(ctx, maps, mapPitch, border, f, why); };
    return unplannedFrame("Could not remap the frame", stream, refused, [&](const FrameTransformContext& ctx, int, cudaStream_t s) {
      t360::PerFrameGatherParams gp{};
      for (int p = 0; p < f.numPlanes; ++p) {
        gp.plane[p].geometry = t360::SphereGeometry{f.outW[p], f.outH[p], f.inW[p], f.inH[p]};
        gp.plane[p].map = reinterpret_cast<const float2*>(maps[p]);
        gp.plane[p].mapPitch = mapPitch[p] / 8;
      }
      gp.transparent = border == t360::kBorderTransparent;
      perFrameGather(t360::PerFrameSource::kMap, gp, ctx, f, f.in, f.inPitch, nullptr, gp.transparent, nullptr, nullptr, nullptr, s);
      return true;
    });
  }

  // Whole frame of a fisheye lens rig (T360B200_transformFrameLensAsync): one gather launch for all planes, every record
  // computed by lensSample (oriented_view.h), so a rig gives what lensMap -> generateMapFromWarp plans for it.  Needs no
  // plan and leaves the plans alone; the output layout's tables come through the slot's upload ring.  Every refusal comes
  // before the first CUDA call, and nothing here synchronises the device.
  // seamWidth: nullptr for the hard seam; else the belt in degrees across which two lenses are blended
  // (T360B200_transformFrameLensBlendAsync: lensBlendSample), the same steps with the blend source.
  // photo: a photometry (T360B200_transformFrameLensPhotoAsync: lensPhotoSample), with *seamWidth 0 for the hard seam; each
  // lens's sample is corrected before the seam, and with stats set (device, [numPlanes][6]) the overlap's sums are zeroed
  // with a memset and accumulated by the same gather.
  // moving: a photometric frame with a rig motion (T360B200_transformFrameLensMotionAsync: lensMotionSample), motion checked
  // after the photometric refusals; its sample table comes through the slot's upload ring.
  bool transformFrameLens(const char* what, const T360LensRig* rig, const float* seamWidth, const T360Orientation* o, const FramePlanes& f,
                          cudaStream_t stream, const T360RigPhotometry* photo = nullptr, unsigned long long* stats = nullptr,
                          bool moving = false, const T360RigMotion* motion = nullptr) {
    auto refused = [&](const FrameTransformContext& ctx, std::string* why) {
      if (photo) return lensPhotoRefused(ctx, rig, photo, *seamWidth, o, why) || (moving && motionRefused(*rig, motion, why));
      return seamWidth ? lensBlendRefused(ctx, rig, *seamWidth, o, why) : lensRefused(ctx, rig, o, why);
    };
    return unplannedFrame(what, stream, refused, [&](const FrameTransformContext& ctx, int k, cudaStream_t s) {
      const FrameTransformContext lens = lensContext(ctx);
      const float* tables[kPlaneLanes];
      UploadRing::Entry* staged = nullptr;
      sphereTablesFor(lens, f.numPlanes, f.outW, f.outH, slotFor(s), s, tables, &staged);
      t360::PerFrameGatherParams gp{};
      for (int p = 0; p < f.numPlanes; ++p) gp.plane[p].geometry = t360::sphereGeometry(lens, f.outW[p], f.outH[p], f.inW[p], f.inH[p], k);
      gp.rotation = t360::rotationFromAngles(o->yaw, o->pitch, o->roll);
      gp.rig = lensRigModel(*rig);
      const bool feathered = seamWidth && *seamWidth > 0.0f;
      if (feathered) gp.seamScale = lensSeamScale(*seamWidth);
      t360::PerFrameSource source = feathered ? t360::PerFrameSource::kLensBlend : t360::PerFrameSource::kLens;
      UploadRing::Entry* motionStaged = nullptr;
      if (photo) {
        source = moving ? t360::PerFrameSource::kLensMotion : t360::PerFrameSource::kLensPhoto;
        for (int p = 0; p < f.numPlanes; ++p) gp.photo.plane[p] = lensPhotoPlane(*photo, rig->numLenses, p);
        gp.photo.stats = stats;
        if (moving) gp.motion = stageMotion(*rig, *motion, gp.rig, slotFor(s), s, &motionStaged);
        if (stats) CU(cudaMemsetAsync(stats, 0, sizeof(unsigned long long) * t360::kPhotoStats * f.numPlanes, s));
      }
      perFrameGather(source, gp, ctx, f, f.in, f.inPitch, nullptr, /*transparent=*/true, tables, staged, nullptr, s);
      releaseAfter(motionStaged, s);
      return true;
    });
  }

  // Whole frame of camera view v (the rectilinear, camera, camera-mip, camera-photo and stereo calls): one gather launch
  // for all planes, every record computed by the chain of its source (oriented_view.h), so the view gives what its host
  // twin describes.  The source follows from v:
  //   - kRectilinear (rectilinearSample) without a photometry where no plane has a level above 0 (no minify, maxLevel 0,
  //     or planes too small for a level): cameraMap -> generateMapFromWarp's frame;
  //   - kCameraMip (mipCameraSample) without a photometry, after the planes' pyramids (buildPyramids);
  //   - kCameraPhoto / kStereoCamera (cameraPhotoSample<MIP, stereo>) with one, after the pyramids when a plane has a
  //     level, and with v.stats (device, [numPlanes][6]) the overlap's sums zeroed with a memset first and accumulated by
  //     the same gather;
  //   - kCameraMotion (cameraMotionSample<MIP>) for a moving view: kCameraPhoto's steps, and the motion's sample table
  //     through the slot's upload ring;
  //   - kCameraAniso (anisoFootprint, anisoCameraSample) for an anisotropic view with maxProbes > 1, after the pyramids
  //     when a plane has a level (without one, the probes supersample level 0).  With maxProbes = 1 its records are
  //     kCameraMip's (kRectilinear's without a level), so it takes that source.
  // rig == nullptr: the context's input under BORDER_WRAP; else the rig's lenses under BORDER_TRANSPARENT, with the lens
  // call's pre-fill.  Needs no plan and leaves the plans alone; no tables.
  bool transformFrameView(const char* what, const CameraView& v, const FramePlanes& f, cudaStream_t stream) {
    auto refused = [&](const FrameTransformContext& ctx, std::string* why) {
      if (viewRefused(ctx, v, why)) return true;
      for (int p = 0; v.photometric && v.minify && v.minify->maxLevel > 0 && p < f.numPlanes; ++p)
        if (f.inW[p] > 2 * 65535 || f.inH[p] > 2 * 65535) {  // (documented by the photometric and stereo calls)
          *why = formatted("input plane %d is %dx%d: a pyramid needs sides of at most 131070", p, f.inW[p], f.inH[p]);
          return true;
        }
      return false;
    };
    return unplannedFrame(what, stream, refused, [&](const FrameTransformContext& ctx, int, cudaStream_t s) {
      t360::PerFrameGatherParams gp{};
      int topMax = 0;
      for (int p = 0; p < f.numPlanes; ++p) {
        gp.plane[p].geometry = viewGeometry(ctx, v, f.inW[p], f.inH[p], f.outW[p], f.outH[p]);
        gp.mip[p].geometry = t360::mipGeometry(gp.plane[p].geometry, v.minify ? v.minify->maxLevel : 0);
        topMax = std::max(topMax, gp.mip[p].geometry.top);
      }
      gp.lens = v.rig != nullptr;
      gp.camera = cameraConstants(v);
      if (v.rig) gp.rig = lensRigModel(*v.rig);
      if (v.seamWidth > 0.0f) gp.seamScale = lensSeamScale(v.seamWidth);
      if (v.minify) gp.mipBias = mipBias(*v.minify);
      t360::PerFrameSource source = topMax > 0 ? t360::PerFrameSource::kCameraMip : t360::PerFrameSource::kRectilinear;
      if (v.aniso && v.maxProbes > 1) {
        source = t360::PerFrameSource::kCameraAniso;
        gp.cameraAniso = static_cast<uint8_t>(probesLog2(v.maxProbes));
      }
      UploadRing::Entry* motionStaged = nullptr;
      if (v.moving) gp.motion = stageMotion(*v.rig, *v.motion, gp.rig, slotFor(s), s, &motionStaged);
      if (v.photometric) {
        source = v.stereo ? t360::PerFrameSource::kStereoCamera
                          : (v.moving ? t360::PerFrameSource::kCameraMotion : t360::PerFrameSource::kCameraPhoto);
        for (int p = 0; p < f.numPlanes; ++p) gp.photo.plane[p] = lensPhotoPlane(*v.photometry, v.rig->numLenses, p);
        gp.photo.stats = v.stats;
        if (v.stats) CU(cudaMemsetAsync(v.stats, 0, sizeof(unsigned long long) * t360::kPhotoStats * f.numPlanes, s));
      }
      UploadRing::Entry* staged = nullptr;
      if (topMax > 0) buildPyramids(f, gp, slotFor(s), s, &staged);
      perFrameGather(source, gp, ctx, f, f.in, f.inPitch, nullptr, gp.lens, nullptr, nullptr, nullptr, s);
      releaseAfter(staged, s);
      releaseAfter(motionStaged, s);
      return true;
    });
  }

  // Levels 1..top of every plane's pyramid (gp.mip[p].geometry.top) into the slot's scratch, on s: level l of all planes
  // that have it in one launch (launchPyramidLevel), so T_max launches.  Fills gp.mip[p].level.  The tap tables of the
  // levels that are not exact 2 x 2 cells are built on the host when a plane size or top level changes and staged through
  // the slot's upload ring (*staged: the entry to release after the gather).
  void buildPyramids(const FramePlanes& f, t360::PerFrameGatherParams& gp, StreamSlot& slot, cudaStream_t s, UploadRing::Entry** staged) {
    constexpr int kPitchAlign = 256;
    // levels 1..top of plane p in its lane's scratch, one after the other, each at a 256-byte pitch
    std::vector<int> key;
    int topMax = 0;
    for (int p = 0; p < f.numPlanes; ++p) {
      const t360::MipSizes z = t360::mipSizes(f.inW[p], f.inH[p], gp.mip[p].geometry.top);
      size_t at = 0;
      for (int l = 1; l <= z.top; ++l) {
        gp.mip[p].level[l - 1] = {nullptr, z.w[l], z.h[l], (z.w[l] + kPitchAlign - 1) / kPitchAlign * kPitchAlign};
        at += static_cast<size_t>(gp.mip[p].level[l - 1].pitch) * z.h[l];
      }
      if (at) slot.lanes[p].pyramid.reserve(at + 64);
      at = 0;
      for (int l = 1; l <= z.top; ++l) {
        t360::PerFrameGatherParams::MipLevel& L = gp.mip[p].level[l - 1];
        L.bytes = slot.lanes[p].pyramid.ptr + at;
        at += static_cast<size_t>(L.pitch) * L.h;
      }
      key.insert(key.end(), {f.inW[p], f.inH[p], z.top});
      topMax = std::max(topMax, z.top);
    }
    // the tap tables of the levels that are not exact 2 x 2 cells, rebuilt when a plane size or top level changes
    if (slot.mipSizes != key) {
      std::vector<uint8_t>& b = slot.mipTapBytes;
      b.clear();
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
      for (int p = 0; p < f.numPlanes; ++p) {
        for (int l = 1; l <= gp.mip[p].geometry.top; ++l) {
          const int w = l == 1 ? f.inW[p] : gp.mip[p].level[l - 2].w, h = l == 1 ? f.inH[p] : gp.mip[p].level[l - 2].h;
          t360::AreaResizePlan r;
          t360::buildAreaResize(w, h, gp.mip[p].level[l - 1].w, gp.mip[p].level[l - 1].h, r);
          StreamSlot::MipTapsAt& at = slot.mipTapAt[p][l - 1];
          at = {};
          if (r.cellW == 0) {  // (else cellW == cellH == 2: the kernel's exact cells)
            const std::vector<int2> xt = packed(r.x), yt = packed(r.y);
            at.xTaps = append(xt.data(), xt.size() * sizeof(int2));
            at.xFirst = append(r.x.first.data(), r.x.first.size() * sizeof(int));
            at.yTaps = append(yt.data(), yt.size() * sizeof(int2));
            at.yFirst = append(r.y.first.data(), r.y.first.size() * sizeof(int));
          }
        }
      }
      slot.mipSizes = key;
    }
    const uint8_t* taps = slot.mipTapBytes.empty() ? nullptr : stageUpload(slot.mipTaps, slot.mipTapBytes, s, staged);
    for (int l = 1; l <= topMax; ++l) {
      t360::PyramidParams pp{};
      for (int p = 0; p < f.numPlanes; ++p) {
        if (gp.mip[p].geometry.top < l) continue;
        const t360::PerFrameGatherParams::MipLevel& dst = gp.mip[p].level[l - 1];
        t360::PyramidPlane& v = pp.plane[pp.numPlanes++];
        if (l == 1) {
          v.src = f.in[p]; v.srcW = f.inW[p]; v.srcH = f.inH[p]; v.srcPitch = f.inPitch[p];
        } else {
          const t360::PerFrameGatherParams::MipLevel& below = gp.mip[p].level[l - 2];
          v.src = below.bytes; v.srcW = below.w; v.srcH = below.h; v.srcPitch = below.pitch;
        }
        v.dst = dst.bytes; v.dstW = dst.w; v.dstH = dst.h; v.dstPitch = dst.pitch;
        const StreamSlot::MipTapsAt& at = slot.mipTapAt[p][l - 1];
        if (at.xTaps != SIZE_MAX) {
          v.xTaps = reinterpret_cast<const int2*>(taps + at.xTaps);
          v.xFirst = reinterpret_cast<const int*>(taps + at.xFirst);
          v.yTaps = reinterpret_cast<const int2*>(taps + at.yTaps);
          v.yFirst = reinterpret_cast<const int*>(taps + at.yFirst);
        }
      }
      CU(t360::launchPyramidLevel(pp, s));
    }
  }

  // The steps of the per-frame calls that need no plan (lens rigs, rectilinear views): under the reader lock, so frame-exact
  // against reconfigure and reconfigureAsync, refused(ctx, &why) is asked before any CUDA call (0 and a message prefixed by
  // `what`); then enqueue(ctx, k, s) sets up the planes and launches the gather on the caller's stream (nullptr: the
  // transform's).  Nothing here synchronises the device.
  template <class Refused, class Enqueue>
  bool unplannedFrame(const char* what, cudaStream_t stream, Refused&& refused, Enqueue&& enqueue) {
    return guarded(what, [&] {
      std::shared_lock<std::shared_mutex> config(configMu_);
      const FrameTransformContext ctx = ctx_;
      std::string why;
      if (refused(ctx, &why)) {
        std::printf("%s. Error: %s\n", what, why.c_str());
        return false;
      }
      const int k = t360::kernelSizeOf(ctx.interpolation_alg);
      const DeviceRestore restoreDevice = ensureDevice();
      return enqueue(ctx, k, stream ? stream : stream_);
    });
  }

  // The frame a fresh transform made with `ctx` would give, on the per-frame kernels, with the reader lock held: the
  // per-frame calls' frames, and every whole frame while a reconfigureAsync is pending.  The gather computes its sampling
  // records itself (view_gather.cu): for FLAT_FIXED from the view (flat_view.h), for every other layout from the rotation
  // and per-plan tables (oriented_view.h).  Everything that ctx may change against the plans comes from ctx: the kernel size
  // and weights, low-pass on or off and its segments (re-planned on the host, viewLowPass), and while a reconfigureAsync is
  // pending the tables (built on the host and uploaded in stream order, sphereTablesFor); only the plane and map sizes, which
  // ctx cannot change, come from the plans.  Scale factors render at the map's size, then resize with INTER_AREA.  Every
  // refusal comes before the first CUDA call, with a message prefixed by `what`.  Nothing here synchronises the device, and
  // the plans' sampling data is not read.
  bool perFrameLocked(const char* what, const FrameTransformContext& ctx, const FramePlanes& f, cudaStream_t stream) {
    return guarded(what, [&] {
      const int numPlanes = f.numPlanes;
      const int k = t360::kernelSizeOf(ctx.interpolation_alg);
      const DevicePlan* plans[kPlaneLanes];
      for (int p = 0; p < numPlanes; ++p) {
        if (!(plans[p] = findPlan(p ? 1 : 0, p))) return false;
        if (f.inW[p] != plans[p]->inW || f.inH[p] != plans[p]->inH) {
          std::printf("%s. Error: input plane %d is %dx%d, its map was generated for %dx%d\n", what, p, f.inW[p], f.inH[p], plans[p]->inW,
                      plans[p]->inH);
          return false;
        }
        if (k == 0) {
          std::printf("%s. Error: no interpolation algorithm %d\n", what, ctx.interpolation_alg);
          return false;
        }
      }
      const DeviceRestore restoreDevice = ensureDevice();
      cudaStream_t s = stream ? stream : stream_;
      StreamSlot& slot = slotFor(s);
      const uint8_t* src[kPlaneLanes];
      int srcPitch[kPlaneLanes];
      for (int p = 0; p < numPlanes; ++p) { src[p] = f.in[p]; srcPitch[p] = f.inPitch[p]; }
      if (ctx.enable_low_pass_filter && !viewLowPass(what, ctx, plans, f, slot, s, src, srcPitch)) return false;

      const bool flat = ctx.output_layout == LAYOUT_FLAT_FIXED;
      const float* tables[kPlaneLanes] = {};
      UploadRing::Entry* staged = nullptr;  // (pending: the tables come through the slot's ring)
      if (!flat) {
        for (int p = 0; p < numPlanes; ++p) tables[p] = plans[p]->sphereTables.ptr;
        if (perFrameOnly_) {
          int mapW[kPlaneLanes], mapH[kPlaneLanes];
          for (int p = 0; p < numPlanes; ++p) { mapW[p] = plans[p]->mapW; mapH[p] = plans[p]->mapH; }
          sphereTablesFor(ctx, numPlanes, mapW, mapH, slot, s, tables, &staged);
        }
      }
      t360::PerFrameGatherParams gp{};
      for (int p = 0; p < numPlanes; ++p)
        gp.plane[p].geometry = t360::sphereGeometry(ctx, plans[p]->mapW, plans[p]->mapH, plans[p]->inW, plans[p]->inH, k);
      if (flat) gp.view = t360::FlatView{ctx.fixed_yaw, ctx.fixed_pitch, ctx.fixed_hfov, ctx.fixed_vfov};
      else gp.rotation = t360::rotationFromAngles(ctx.fixed_yaw, ctx.fixed_pitch, ctx.fixed_roll);
      perFrameGather(flat ? t360::PerFrameSource::kView : t360::PerFrameSource::kSphere, gp, ctx, f, src, srcPitch, plans, false, tables,
                     staged, &slot, s);
      return true;
    });
  }

  // The one gather launch of a per-frame call (launchPerFrameGather) for the planes of f, on s: gp holds the per-frame
  // constants and each plane's geometry (and map); src / srcPitch are the planes' inputs.  With plans (the whole-frame
  // calls) a plane renders at its plan's map size with the plan's border, and a scale factor resizes it into f's plane with
  // INTER_AREA through the slot's scratch plane; without (remap, lens rigs, rectilinear views) it renders into f's plane
  // with BORDER_TRANSPARENT where `transparent`.  tables: the planes' sphere tables (nullptr: none); `staged` the upload
  // ring entry they came through, released after the launch.
  void perFrameGather(t360::PerFrameSource source, t360::PerFrameGatherParams& gp, const FrameTransformContext& ctx, const FramePlanes& f,
                      const uint8_t* const* src, const int* srcPitch, const DevicePlan* const* plans, bool transparent,
                      const float* const* tables, UploadRing::Entry* staged, StreamSlot* slot, cudaStream_t s) {
    PlaneTarget dst[kPlaneLanes];
    for (int p = 0; p < f.numPlanes; ++p) {
      const DevicePlan* plan = plans ? plans[p] : nullptr;
      dst[p] = renderTarget(plan, p > 0, plan ? plan->transparent : transparent, f.out[p], f.outPitch[p], f.outW[p], f.outH[p],
                            plan ? &slot->lanes[p].scaled : nullptr, s);
      t360::PerFramePlane& v = gp.plane[p];
      v.src = src[p];
      v.srcPitch = srcPitch[p];
      v.dst = dst[p].dst;
      v.dstPitch = dst[p].dstPitch;
      v.colTable = tables ? tables[p] : nullptr;
      v.rowTable = v.colTable ? v.colTable + t360::sphereTableRowOffset(v.geometry) : nullptr;
    }
    gp.numPlanes = f.numPlanes;
    gp.kernelSize = t360::kernelSizeOf(ctx.interpolation_alg);
    gp.weights = deviceWeights(ctx.interpolation_alg);
    CU(t360::launchPerFrameGather(gp, source, numSMs_, s));
    releaseAfter(staged, s);
    for (int p = 0; p < f.numPlanes; ++p) finishTarget(dst[p], s);
  }

  // tuning aid: a timeline of the consumer groups of the last frame gather (see StagedParams::trace)
  void enableTrace(bool on) { traceEnabled_ = on; }
  size_t readTrace(unsigned long long* out, size_t maxWords) {
    if (!trace_.ptr) return 0;
    if (!out) return trace_.count;  // the caller asks how large a buffer the trace needs
    const size_t n = std::min(maxWords, trace_.count);
    if (cudaMemcpy(out, trace_.ptr, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost) != cudaSuccess) return 0;
    return n;
  }

  bool synchronize() {
    if (!deviceReady_) return true;
    return cudaStreamSynchronize(stream_) == cudaSuccess;
  }
  cudaStream_t stream() {
    try { const DeviceRestore restoreDevice = ensureDevice(); } catch (...) { return nullptr; }
    return stream_;
  }
  bool tileCounts(int planIndex, int counts[4]) {
    std::lock_guard<std::mutex> lock(mu_);
    auto it = plans_.find(planIndex);
    if (it == plans_.end()) return false;
    counts[0] = it->second.numStaged; counts[1] = it->second.numBorder;
    const t360::BlurLayout& b = it->second.blur.layout;
    counts[2] = b.numStrips[0] + b.numStrips[1] + b.numStrips[2];
    counts[3] = b.numTiles + b.numDirect;
    return true;
  }
  size_t planBytes(int planIndex) {
    std::lock_guard<std::mutex> lock(mu_);
    auto it = plans_.find(planIndex);
    return it == plans_.end() ? 0 : it->second.deviceBytes();
  }

 private:
  StreamSlot& slotFor(cudaStream_t s) {
    std::lock_guard<std::mutex> lock(slotMu_);
    std::unique_ptr<StreamSlot>& slot = slots_[s];
    if (!slot) {
      slot.reset(new StreamSlot);
      for (int i = 0; i < kPlaneLanes; ++i) {
        PlaneLane& l = slot->lanes[i];
        if (i > 0) CU(cudaStreamCreateWithFlags(&l.main, cudaStreamNonBlocking));
        CU(cudaEventCreateWithFlags(&l.done, cudaEventDisableTiming));
      }
      CU(cudaEventCreateWithFlags(&slot->fork, cudaEventDisableTiming));
    }
    return *slot;
  }

  // The transform lives on the device that was current when it first touched CUDA.  Calls from a thread whose current
  // device is another one switch to it for their duration and switch back (the guard), like a library should.
  struct DeviceRestore {
    int previous = -1;
    DeviceRestore() = default;
    DeviceRestore(const DeviceRestore&) = delete;
    DeviceRestore& operator=(const DeviceRestore&) = delete;
    DeviceRestore(DeviceRestore&& o) noexcept : previous(o.previous) { o.previous = -1; }
    ~DeviceRestore() { if (previous >= 0) cudaSetDevice(previous); }
  };
  DeviceRestore ensureDevice() {
    DeviceRestore guard;
    if (deviceReady_) {
      int current = device_;
      CU(cudaGetDevice(&current));
      if (current != device_) {
        CU(cudaSetDevice(device_));
        guard.previous = current;
      }
      return guard;
    }
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) throw CudaFail{e != cudaSuccess ? e : cudaErrorNoDevice, "cudaGetDeviceCount (no CUDA device: this library has no CPU fallback)"};
    CU(cudaGetDevice(&device_));  // honour the caller's current device (one process per GPU sets it before)
    cudaDeviceProp prop{};
    CU(cudaGetDeviceProperties(&prop, device_));
    numSMs_ = prop.multiProcessorCount;
    CU(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
    if (auto getCurrent = reinterpret_cast<CUresult (*)(CUcontext*)>(driverEntry("cuCtxGetCurrent"))) getCurrent(&cuContext_);
    deviceReady_ = true;
    return guard;
  }

  // Pageable host planes are copied through the driver's bounce buffers at a fraction of PCIe speed.  When enabled
  // (T360B200_setPinHostPlanes or T360B200_PIN_HOST_PLANES=1), a plane address seen for the second time is page-locked
  // in place with cudaHostRegister so that later frames in the same buffer are DMA'd directly.  Opt-in because the
  // caller must not free such a buffer while the transform is alive (it is unregistered in the destructor).
  // A registration covers whole pages, so it can take in the first or last page of another caller plane.  The runtime
  // takes a plane whose first byte is registered for page-locked memory throughout and refuses a copy that runs past
  // the registration (cudaErrorInvalidValue), so a plane that overlaps one of these registrations without lying inside
  // it is merged into it (one registration of the union), or, if that fails, the registration is dropped.  Called for
  // both planes of a call before its first copy, with nothing in flight.
  void pinIfRecurring(const void* ptr, size_t bytes) {
    if (!pinHostPlanes_ || !ptr || !bytes) return;
    const uintptr_t page = 4096, lo = reinterpret_cast<uintptr_t>(ptr) & ~(page - 1);
    const size_t len = ((reinterpret_cast<uintptr_t>(ptr) + bytes + page - 1) & ~(page - 1)) - lo;
    for (HostRange& r : hostRanges_) {
      if (!r.pinned || lo + len <= r.base || lo >= r.base + r.bytes) continue;
      if (lo >= r.base && lo + len <= r.base + r.bytes) return;  // inside a registration: page-locked already
      for (PlaneGraph& g : planeGraphs_) cudaGraphExecDestroy(g.exec);  // (their copies assumed the old registration)
      planeGraphs_.clear();
      cudaHostUnregister(reinterpret_cast<void*>(r.base));
      const uintptr_t ulo = std::min(lo, r.base), uhi = std::max(lo + len, r.base + r.bytes);
      if (cudaHostRegister(reinterpret_cast<void*>(ulo), uhi - ulo, cudaHostRegisterDefault) == cudaSuccess) {
        r.base = ulo;
        r.bytes = uhi - ulo;
        return;
      }
      cudaGetLastError();
      r.pinned = false;
      r.seen = -1000000;  // its planes go through the bounce buffers from now on
    }
    if (memoryTypeOf(ptr) != cudaMemoryTypeUnregistered) return;
    for (HostRange& r : hostRanges_) {
      if (r.base != lo || r.bytes != len) continue;
      if (!r.pinned && ++r.seen >= 2) {
        if (cudaHostRegister(reinterpret_cast<void*>(lo), len, cudaHostRegisterDefault) == cudaSuccess) r.pinned = true;
        else { cudaGetLastError(); r.seen = -1000000; }  // do not retry this range
      }
      return;
    }
    if (hostRanges_.size() < 64) hostRanges_.push_back(HostRange{lo, len, 1, false});
  }

  // The kind of memory p points into, or -1 (the error cleared) when the runtime cannot tell
  static int memoryTypeOf(const void* p) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
      cudaGetLastError();
      return -1;
    }
    return a.type;
  }

  static bool isDevicePointer(const void* p) {
    const int t = memoryTypeOf(p);
    return t == cudaMemoryTypeDevice || t == cudaMemoryTypeManaged;
  }

  const DevicePlan* findPlan(int planIndex, int imagePlaneIndex) {
    std::lock_guard<std::mutex> lock(mu_);
    auto it = plans_.find(planIndex);
    if (it == plans_.end()) {
      std::printf("Could not transform the plane %d. Error: no map was generated for index %d\n", imagePlaneIndex, planIndex);
      return nullptr;
    }
    return &it->second;
  }

  const int16_t* deviceWeights(int interpolationAlg) {
    const int16_t* host = nullptr;
    const int k = t360::remapTable(interpolationAlg, &host);
    if (k < 2) return nullptr;
    std::lock_guard<std::mutex> lock(lazyMu_);  // (a frame served for a pending context may be the first of its kernel size)
    auto& buf = weights_[k];
    if (!buf.ptr) {
      buf.reserve(static_cast<size_t>(1024) * k * k);
      CU(cudaMemcpy(buf.ptr, host, buf.bytes(), cudaMemcpyHostToDevice));
      // the frame kernel's shared-memory image of the same table (slot-permuted; two copies for the cubic table)
      const std::vector<uint8_t> image = t360::buildWeightImage(k, host);
      weightImages_[k].reserve(image.size());
      CU(cudaMemcpy(weightImages_[k].ptr, image.data(), image.size(), cudaMemcpyHostToDevice));
    }
    return buf.ptr;
  }

  // The device half of a plan index, for the context `ctx` it was planned with (moves the gather plan's job lists out).
  DevicePlan upload(HostIndexPlan& p, const FrameTransformContext& ctx) {
    const HostPlan& h = p.host;
    DevicePlan d;
    d.inW = h.inW; d.inH = h.inH; d.outW = h.outW; d.outH = h.outH; d.mapW = h.mapW; d.mapH = h.mapH;
    d.kernelSize = h.kernelSize;
    d.transparent = h.transparentBorder;
    d.warp = h.warp;
    d.stereoFormat = ctx.input_stereo_format;
    if (d.kernelSize > 0) {
      deviceWeights(ctx.interpolation_alg);
      t360::GatherPlan& g = p.gather;
      d.tilesPerRow = g.tilesPerRow;
      d.samples.reserve(g.records.size());
      CU(cudaMemcpy(d.samples.ptr, g.records.data(), g.records.size() * sizeof(int2), cudaMemcpyHostToDevice));
      d.numStaged = g.totalStaged();
      d.numBorder = g.numBorder;
      d.numJobs = static_cast<int>(g.launchJobs.size());
      d.hostJobs = t360::deviceJobs(g);
      if (!d.hostJobs.empty()) {
        d.gatherJobs.reserve(d.hostJobs.size());
        CU(cudaMemcpy(d.gatherJobs.ptr, d.hostJobs.data(), d.hostJobs.size() * sizeof(GatherJob), cudaMemcpyHostToDevice));
      }
      if (!g.compact.empty() || !g.capRecords.empty()) {  // one buffer: the tiles' records, then the pole caps'
        const std::vector<uint32_t> records = t360::deviceRecords(g, d.kernelSize);
        d.records.reserve(records.size());
        CU(cudaMemcpy(d.records.ptr, records.data(), records.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
      }
      d.jobNeedRows = std::move(g.launchNeedRows);
      d.jobRects = std::move(g.launchRects);
    }
    d.lowPass = ctx.enable_low_pass_filter != 0;
    if (d.lowPass) {
      d.segments = h.segments;
      d.planTaps = h.taps;
      buildBlurSet(d.segments, d.planTaps, h.inW, h.inH, d.stereoFormat, d.blur);
    }
    d.resizeNeeded = h.resize.needed;
    if (d.resizeNeeded) resizeFor(d, d.outW, d.outH);
    if (d.kernelSize > 0 && !d.warp && ctx.output_layout != LAYOUT_FLAT_FIXED) {  // (a warp map has no layout)
      const std::vector<float> t = t360::buildSphereTables(t360::sphereGeometry(ctx, h.mapW, h.mapH, h.inW, h.inH, h.kernelSize));
      if (!t.empty()) {
        d.sphereTables.reserve(t.size());
        CU(cudaMemcpy(d.sphereTables.ptr, t.data(), t.size() * sizeof(float), cudaMemcpyHostToDevice));
      }
    }
    return d;
  }

  // the INTER_AREA tables from the plan's map size to outW x outH, on the device
  const DevicePlan::Resize& resizeFor(const DevicePlan& plan, int outW, int outH) {
    std::lock_guard<std::mutex> lock(lazyMu_);
    auto it = plan.resizes.find({outW, outH});
    if (it != plan.resizes.end()) return it->second;
    t360::AreaResizePlan r;
    t360::buildAreaResize(plan.mapW, plan.mapH, outW, outH, r);
    DevicePlan::Resize& d = plan.resizes[{outW, outH}];
    auto upload2 = [](const std::vector<int2>& v, DeviceBuffer<int2>& buf) {
      buf.reserve(std::max<size_t>(v.size(), 1));
      if (!v.empty()) CU(cudaMemcpy(buf.ptr, v.data(), v.size() * sizeof(int2), cudaMemcpyHostToDevice));
    };
    if (r.enlarge) {
      d.cellW = d.cellH = -1;
      d.xMax = r.lx.dmax;
      auto pack = [](const t360::AreaLinearAxis& a) {
        std::vector<int2> v(a.ofs.size());
        for (size_t i = 0; i < a.ofs.size(); ++i)
          v[i] = int2{a.ofs[i], static_cast<int>(static_cast<uint16_t>(a.coef[2 * i]) | (static_cast<uint32_t>(static_cast<uint16_t>(a.coef[2 * i + 1])) << 16))};
        return v;
      };
      upload2(pack(r.lx), d.xLinear);
      upload2(pack(r.ly), d.yLinear);
    } else if (r.cellW > 0) {
      d.cellW = r.cellW; d.cellH = r.cellH;
    } else {
      auto uploadAxis = [&](const t360::AreaAxis& a, DeviceBuffer<int2>& taps, DeviceBuffer<int>& first) {
        std::vector<int2> packed(a.taps.size());
        for (size_t i = 0; i < a.taps.size(); ++i) {
          int bits;
          std::memcpy(&bits, &a.taps[i].alpha, sizeof(bits));
          packed[i] = int2{a.taps[i].src, bits};
        }
        upload2(packed, taps);
        first.reserve(a.first.size());
        CU(cudaMemcpy(first.ptr, a.first.data(), a.first.size() * sizeof(int), cudaMemcpyHostToDevice));
      };
      uploadAxis(r.x, d.xTaps, d.xFirst);
      uploadAxis(r.y, d.yTaps, d.yFirst);
    }
    return d;
  }

  // The low-pass lists of one plane size: cut on the host, packed into one image, uploaded once (plan generation, or the
  // first use of a size)
  void buildBlurSet(const std::vector<t360::LowPassSegment>& segments, const std::vector<float>& planTaps, int planeW, int planeH,
                    int stereoFormat, DevicePlan::BlurSet& d) {
    t360::buildBlurLists(segments, planTaps, planeW, planeH, stereoFormat, d.lists, &d.needsClear);
    std::vector<uint8_t> image;
    d.layout = t360::packBlurLists(d.lists, image, image);
    if (image.empty()) return;
    d.image.reserve(image.size());
    CU(cudaMemcpy(d.image.ptr, image.data(), image.size(), cudaMemcpyHostToDevice));
  }

  // the low-pass jobs of a plan for planes of w x h (the planned size, or whatever the caller passes)
  const DevicePlan::BlurSet& blurFor(const DevicePlan& plan, int w, int h) {
    if (w == plan.inW && h == plan.inH) return plan.blur;
    std::lock_guard<std::mutex> lock(lazyMu_);
    auto it = plan.otherBlurs.find({w, h});
    if (it != plan.otherBlurs.end()) return it->second;
    DevicePlan::BlurSet& set = plan.otherBlurs[{w, h}];
    buildBlurSet(plan.segments, plan.planTaps, w, h, plan.stereoFormat, set);
    return set;
  }

  // The low-pass of planes fp.plane[0 .. numPlanes) from one packed list (its arrays at `jobs` / `taps` + the layout's
  // offsets): the strip jobs of every plane in one launch per vertical half-size (a job's plane is in its `edge`), then
  // the tile and direct jobs, which only a single plane's list has.  clear: zero the planes first (reference cpp:625:
  // Mat::zeros under dropped segments).
  void launchLowPass(const t360::BlurLayout& l, bool clear, const uint8_t* jobs, const uint8_t* taps, t360::FrameStripParams fp, int numPlanes,
                     cudaStream_t s) {
    const t360::FrameStripParams::Plane& a = fp.plane[0];
    if (clear)
      for (int p = 0; p < numPlanes; ++p) CU(cudaMemset2DAsync(fp.plane[p].dst, fp.plane[p].dstPitch, 0, fp.plane[p].width, fp.plane[p].height, s));
    fp.numPlanes = numPlanes;
    fp.taps = reinterpret_cast<const float*>(taps + l.tapAt);
    for (int c = 0; c < t360::kStripMaxHy; ++c) {
      if (!l.numStrips[c]) continue;
      fp.jobs = reinterpret_cast<const StripJob*>(jobs + l.stripAt[c]);
      fp.numJobs = l.numStrips[c];
      CU(t360::launchBlurFrameStrips(fp, c + 1, s));
    }
    t360::BlurParams bp{a.src, a.dst, a.width, a.height, a.srcPitch, a.dstPitch, reinterpret_cast<const BlurJob*>(jobs + l.tileAt), l.numTiles,
                        fp.taps, l.tileSmem};
    if (bp.numJobs) CU(t360::launchBlur(bp, s));
    if (l.numDirect) {
      bp.jobs = reinterpret_cast<const BlurJob*>(jobs + l.directAt);
      bp.numJobs = l.numDirect;
      CU(t360::launchBlurDirect(bp, s));
    }
  }

  void runLowPass(const DevicePlan& plan, const uint8_t* dIn, uint8_t* dOut, int w, int h, int inPitch, int outPitch,
                  cudaStream_t s) {
    const DevicePlan::BlurSet& b = blurFor(plan, w, h);
    t360::FrameStripParams fp{};
    fp.plane[0] = {dIn, dOut, w, h, inPitch, outPitch};
    launchLowPass(b.layout, b.needsClear, b.image.ptr, b.image.ptr, fp, 1, s);
  }

  // the tensor maps of a source plane, from the lane's cache or freshly encoded (false: not TMA-describable)
  static bool planeMaps(PlaneLane& lane, const uint8_t* src, int w, int h, int pitch, int k,
                        CUtensorMap (&out)[t360::kMaxBoxMaps]) {
    for (const PlaneMaps& e : lane.mapCache)
      if (e.base == src && e.w == w && e.h == h && e.pitch == pitch && e.k == k) {
        std::memcpy(out, e.maps, sizeof(e.maps));
        return true;
      }
    PlaneMaps fresh;
    for (int m = 0; m < t360::boxMaps(k); ++m)
      if (!encodePlaneMap(&fresh.maps[m], src, w, h, pitch, k, m)) return false;
    fresh.base = src; fresh.w = w; fresh.h = h; fresh.pitch = pitch; fresh.k = k;
    lane.mapCache[lane.mapCacheNext] = fresh;
    lane.mapCacheNext = (lane.mapCacheNext + 1) % PlaneLane::kMapCache;
    std::memcpy(out, fresh.maps, sizeof(fresh.maps));
    return true;
  }

  // reference transformPlane (cpp:707-794): [low-pass] -> gather [-> area resize].  Device pointers, asynchronous.
  bool enqueue(const DevicePlan& plan, bool chroma, const uint8_t* dIn, uint8_t* dOut, int inW, int inH, int inPitch, int outW,
               int outH, int outPitch, cudaStream_t s, int imagePlaneIndex, PlaneLane& lane) {
    GatherWork w;
    if (!prepareGather(plan, chroma, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, s, imagePlaneIndex, lane, w)) return false;
    if (plan.kernelSize == 0) return true;
    gatherPlane(w, lane, s);
    finishTarget(w.target, s);
    return true;
  }

  // Everything before the gather of one plane: argument checks, the render target, the low-pass stage.  chroma: the plane
  // is a chroma plane (plan index != 0).
  bool prepareGather(const DevicePlan& plan, bool chroma, const uint8_t* dIn, uint8_t* dOut, int inW, int inH, int inPitch, int outW,
                     int outH, int outPitch, cudaStream_t s, int imagePlaneIndex, PlaneLane& lane, GatherWork& w, bool blurDone = false) {
    w.plan = &plan;
    if (plan.kernelSize == 0) {
      std::printf("Could not find interpolation algorithm for plane %d", imagePlaneIndex);  // reference cpp:780-784
      return true;
    }
    const PlaneTarget& t = w.target = renderTarget(&plan, chroma, plan.transparent, dOut, outPitch, outW, outH, &lane.scaled, s);
    const uint8_t* src = dIn;
    int srcPitch = inPitch;
    if (plan.lowPass) {
      const int bp = scratchPlane(lane.blurred, inW, inH);
      if (!blurDone) runLowPass(plan, dIn, lane.blurred.ptr, inW, inH, inPitch, bp, s);
      src = lane.blurred.ptr;
      srcPitch = bp;
    }
    w.view = t360::PlaneView{src, t.dst, reinterpret_cast<const uint4*>(plan.records.ptr), inW, inH, srcPitch, t.dstW, t.dstH, t.dstPitch};
    // staged tiles need the plane the plan was made for (their windows were proven in-bounds for it) and a
    // TMA-describable layout (16-byte aligned base and pitch); otherwise every tile takes the general kernel
    w.staged = plan.numJobs > 0 && !plan.transparent && inW == plan.inW && inH == plan.inH;
    if (w.staged) w.staged = planeMaps(lane, src, inW, inH, srcPitch, plan.kernelSize, w.maps);
    return true;
  }

  static void armScheduler(DeviceBuffer<int>& counter, cudaStream_t s) {
    if (counter.ptr) return;  // zeroed once; every launch leaves it zeroed again
    counter.reserve(2);
    CU(cudaMemsetAsync(counter.ptr, 0, 2 * sizeof(int), s));
  }

  // The gather of one plane as its own launch.
  void gatherPlane(const GatherWork& w, PlaneLane& lane, cudaStream_t s) {
    const DevicePlan& plan = *w.plan;
    if (w.staged) {
      armScheduler(lane.claimCounter, s);
      t360::FrameGatherParams fp{};
      fp.plane[0] = w.view;
      fp.weightImage = reinterpret_cast<const uint4*>(weightImages_[plan.kernelSize].ptr);
      fp.kernelSize = plan.kernelSize;
      fp.numPlanes = 1;
      t360::StagedParams jobs{plan.gatherJobs.ptr, plan.numJobs, lane.claimCounter.ptr, nullptr};
      CU(t360::launchGatherFrame(fp, jobs, w.maps, numSMs_, s));
    } else {
      const t360::PlaneView& v = w.view;
      t360::GatherParams gp{v.src, v.srcW, v.srcH, v.srcPitch, v.dst, v.dstW, v.dstH, v.dstPitch, plan.samples.ptr, plan.tilesPerRow,
                            weights_[plan.kernelSize].ptr, plan.kernelSize, plan.transparent ? 1 : 0};
      CU(t360::launchGather(gp, numSMs_, s));
    }
  }

  // The low-pass of all planes of a frame (mergeable): one launch per vertical kernel half-size.
  void blurFrame(const DevicePlan* const* plans, const FramePlanes& f, PlaneLane* lanes, cudaStream_t s) {
    const FrameListRefs l = frameLists(plans, f.numPlanes);
    t360::FrameStripParams fp{};
    for (int p = 0; p < f.numPlanes; ++p) {
      const int bp = scratchPlane(lanes[p].blurred, f.inW[p], f.inH[p]);
      fp.plane[p] = {f.in[p], lanes[p].blurred.ptr, f.inW[p], f.inH[p], f.inPitch[p], bp};
    }
    launchLowPass(l.blurLayout, false, l.blurImage, l.blurImage, fp, f.numPlanes, s);
  }

  // The low-pass of a per-frame call's frame (perFrameLocked): the segments and taps of every plan index for the context,
  // the job lists cut from them, uploaded through the slot's rings, and the launches -- one per vertical kernel size for all
  // planes when every plane takes the strip kernel only (as blurFrame), else per plane (as runLowPass).  src / srcPitch
  // receive the blurred planes.
  bool viewLowPass(const char* what, const FrameTransformContext& ctx, const DevicePlan* const* plans, const FramePlanes& f, StreamSlot& slot,
                   cudaStream_t s, const uint8_t** src, int* srcPitch) {
    const int numPlanes = f.numPlanes;
    const int indices = numPlanes > 1 ? 2 : 1;
    HostPlan h[2];
    // what the job lists depend on: the plans (generation), the planes, and per segment its rectangle, tap counts and
    // offsets and whether its taps equal its left neighbour's (buildBlurLists merges such segments)
    std::vector<long long> key{static_cast<long long>(planGeneration_), numPlanes};
    for (int idx = 0; idx < indices; ++idx) {
      const DevicePlan& plan = *plans[idx];
      h[idx].ctx = ctx;
      h[idx].inW = plan.inW; h[idx].inH = plan.inH; h[idx].outW = plan.outW; h[idx].outH = plan.outH; h[idx].mapW = plan.mapW; h[idx].mapH = plan.mapH;
      if (!t360::buildLowPassPlan(h[idx])) {
        std::printf("%s. Error: no low-pass plan for index %d\n", what, idx);
        return false;
      }
      key.push_back(reinterpret_cast<intptr_t>(&plan));
      key.push_back(static_cast<long long>(h[idx].taps.size()));
      const std::vector<float>& taps = h[idx].taps;
      const t360::LowPassSegment* prev = nullptr;
      for (const t360::LowPassSegment& g : h[idx].segments) {
        const bool same = prev && g.kxCount == prev->kxCount && g.kyCount == prev->kyCount &&
                          std::memcmp(&taps[g.kxOffset], &taps[prev->kxOffset], sizeof(float) * g.kxCount) == 0 &&
                          std::memcmp(&taps[g.kyOffset], &taps[prev->kyOffset], sizeof(float) * g.kyCount) == 0;
        for (long long v : {g.left, g.top, g.width, g.height, g.kxOffset, g.kxCount, g.kyOffset, g.kyCount}) key.push_back(v);
        key.push_back(same);
        prev = &g;
      }
    }
    ViewBlurCache& c = slot.viewBlur;
    std::vector<uint8_t> taps;
    if (c.key == key) {  // same jobs as the slot's previous frame: refill the taps only
      taps.resize(c.tapCodes.size() * sizeof(float));
      float* t = reinterpret_cast<float*>(taps.data());
      for (size_t i = 0; i < c.tapCodes.size(); ++i) {
        const int code = c.tapCodes[i];
        t[i] = code ? h[(code >> t360::kTapPlaneShift) ? 1 : 0].taps[(code & ((1 << t360::kTapPlaneShift) - 1)) - 1] : 0.f;
      }
    } else {
      c = ViewBlurCache{};
      t360::BlurLists lists[2];
      // coverage: the plan's, computed once per plan, unless a reconfigureAsync is pending (its segment counts may differ)
      for (int idx = 0; idx < indices; ++idx) {
        c.clear[idx] = plans[idx]->blur.needsClear;
        t360::buildBlurLists(h[idx].segments, h[idx].taps, plans[idx]->inW, plans[idx]->inH, plans[idx]->stereoFormat, lists[idx],
                             perFrameOnly_ ? &c.clear[idx] : nullptr);
      }
      const t360::BlurLists* perPlane[kPlaneLanes];
      bool clear[kPlaneLanes];
      for (int p = 0; p < numPlanes; ++p) {
        perPlane[p] = &lists[p ? 1 : 0];
        clear[p] = c.clear[p ? 1 : 0];
      }
      c.merged = mergeable(plans, perPlane, clear, numPlanes, f.inW, f.inH);
      // one byte image of the jobs and one of the taps, with the provenance of every tap (tapSource; in a merged list it
      // carries the plane already)
      auto appendCodes = [&](const t360::BlurLists& l, const t360::BlurLayout& at, int plane) {
        c.tapCodes.resize(taps.size() / sizeof(float), 0);
        for (size_t i = 0; i < l.tapSource.size(); ++i)
          c.tapCodes[at.tapAt / sizeof(float) + i] = l.tapSource[i] ? (plane << t360::kTapPlaneShift) | l.tapSource[i] : 0;
      };
      if (c.merged) {
        const t360::BlurLists all = t360::mergeBlurLists(perPlane, numPlanes);
        c.layout[0] = t360::packBlurLists(all, c.jobs, taps);
        appendCodes(all, c.layout[0], 0);
      } else {
        for (int idx = 0; idx < indices; ++idx) {
          c.layout[idx] = t360::packBlurLists(lists[idx], c.jobs, taps);
          appendCodes(lists[idx], c.layout[idx], idx);
        }
      }
      c.key = std::move(key);
    }
    UploadRing::Entry* used[2];
    const uint8_t* dJobs = stageUpload(slot.viewJobs, c.jobs, s, &used[0]);
    const uint8_t* dTaps = stageUpload(slot.viewTaps, taps, s, &used[1]);
    t360::FrameStripParams fp{};
    for (int p = 0; p < numPlanes; ++p) {
      const int bp = scratchPlane(slot.lanes[p].blurred, f.inW[p], f.inH[p]);
      src[p] = slot.lanes[p].blurred.ptr;
      srcPitch[p] = bp;
      fp.plane[p] = {f.in[p], slot.lanes[p].blurred.ptr, f.inW[p], f.inH[p], f.inPitch[p], bp};
    }
    if (c.merged) {
      launchLowPass(c.layout[0], false, dJobs, dTaps, fp, numPlanes, s);
    } else {
      for (int p = 0; p < numPlanes; ++p) {
        t360::FrameStripParams one{};
        one.plane[0] = fp.plane[p];
        launchLowPass(c.layout[p ? 1 : 0], c.clear[p ? 1 : 0], dJobs, dTaps, one, 1, s);
      }
    }
    for (UploadRing::Entry* e : used) releaseAfter(e, s);
    return true;
  }

  // `bytes` on the device for work enqueued next on `s`: the ring entry that already holds them, or the next entry, refilled
  // (page-locked copy, cudaMemcpyAsync on `s`) once the frame that last read it has finished.
  static const uint8_t* stageUpload(UploadRing& ring, const std::vector<uint8_t>& bytes, cudaStream_t s, UploadRing::Entry** used) {
    if (ring.last >= 0 && ring.lastContent == bytes) {
      *used = &ring.entries[ring.last];
      return ring.entries[ring.last].device;
    }
    const int i = (ring.last + 1) % UploadRing::kEntries;
    UploadRing::Entry& e = ring.entries[i];
    ring.last = -1;  // (until the entry holds the new bytes)
    if (!e.released) CU(cudaEventCreateWithFlags(&e.released, cudaEventDisableTiming));
    if (e.inFlight) CU(cudaEventSynchronize(e.released));
    e.inFlight = false;
    if (bytes.size() > e.capacity) {  // grows to the largest list seen (rarely: the list sizes depend on the tap counts)
      const size_t cap = std::max<size_t>(bytes.size() + bytes.size() / 4, 4096);
      if (e.host) CU(cudaFreeHost(e.host));
      e.host = nullptr;
      if (e.device) CU(cudaFreeAsync(e.device, s));
      e.device = nullptr;
      e.capacity = 0;
      CU(cudaHostAlloc(reinterpret_cast<void**>(&e.host), cap, cudaHostAllocDefault));
      CU(cudaMallocAsync(reinterpret_cast<void**>(&e.device), cap, s));
      e.capacity = cap;
    }
    if (!bytes.empty()) {
      std::memcpy(e.host, bytes.data(), bytes.size());
      CU(cudaMemcpyAsync(e.device, e.host, bytes.size(), cudaMemcpyHostToDevice, s));
    }
    ring.last = i;
    ring.lastContent = bytes;
    *used = &e;
    return e.device;
  }

  // The merged lists of a frame of numPlanes (2 or 3) planes, built on first use in a plan generation.  A rebuild waits for
  // the device: frames of the previous generation may still read the entry's buffers.
  FrameListRefs frameLists(const DevicePlan* const* plans, int numPlanes) {
    std::lock_guard<std::mutex> lock(frameListsMu_);
    FrameLists& f = frameLists_[numPlanes - 2];
    if (f.generation != planGeneration_) {
      if (f.generation != ~0ull) CU(cudaDeviceSynchronize());
      buildFrameLists(plans, numPlanes, f);
      f.generation = planGeneration_;
    }
    return FrameListRefs{f.gatherJobs.ptr, f.numGatherJobs, f.blurImage.ptr, f.blurLayout};
  }

  // Fills `f` with the merged lists of frames of numPlanes planes (f's buffers are not read by any work in flight).
  void buildFrameLists(const DevicePlan* const* plans, int numPlanes, FrameLists& f) {
    std::vector<GatherJob> jobs;
    const t360::BlurLists* lists[kPlaneLanes];
    for (int p = 0; p < numPlanes; ++p) {
      for (GatherJob t : plans[p]->hostJobs) {
        t.outY |= p << t360::kJobPlaneShift;
        jobs.push_back(t);
      }
      lists[p] = &plans[p]->blur.lists;
    }
    std::stable_sort(jobs.begin(), jobs.end(), [](const GatherJob& a, const GatherJob& b) { return t360::jobLaunchRank(a) < t360::jobLaunchRank(b); });
    std::vector<uint8_t> image;
    const t360::BlurLayout layout = t360::packBlurLists(t360::mergeBlurLists(lists, numPlanes), image, image);
    f.gatherJobs.reserve(jobs.size());
    if (!jobs.empty()) CU(cudaMemcpy(f.gatherJobs.ptr, jobs.data(), jobs.size() * sizeof(GatherJob), cudaMemcpyHostToDevice));
    f.blurImage.reserve(image.size());
    if (!image.empty()) CU(cudaMemcpy(f.blurImage.ptr, image.data(), image.size(), cudaMemcpyHostToDevice));
    f.numGatherJobs = static_cast<int>(jobs.size());
    f.blurLayout = layout;
  }

  // The gathers of all planes of a frame as ONE launch (every plane staged).
  void gatherFrame(const GatherWork* work, int numPlanes, cudaStream_t s, StreamSlot& slot) {
    const DevicePlan* plans[kPlaneLanes];
    for (int p = 0; p < numPlanes; ++p) plans[p] = work[p].plan;
    const FrameListRefs f = frameLists(plans, numPlanes);
    armScheduler(slot.frameClaim, s);
    t360::FrameGatherParams fp{};
    CUtensorMap maps[kPlaneLanes][t360::kMaxBoxMaps];
    for (int p = 0; p < numPlanes; ++p) {
      fp.plane[p] = work[p].view;
      std::memcpy(maps[p], work[p].maps, sizeof(work[p].maps));
    }
    fp.weightImage = reinterpret_cast<const uint4*>(weightImages_[work[0].plan->kernelSize].ptr);
    fp.kernelSize = work[0].plan->kernelSize;
    fp.numPlanes = numPlanes;
    if (traceEnabled_) {
      trace_.reserve(static_cast<size_t>(numSMs_) * t360::gatherGroups(work[0].plan->kernelSize) * t360::kTraceJobsPerGroup * 4);
      CU(cudaMemsetAsync(trace_.ptr, 0, trace_.bytes(), s));
    }
    t360::StagedParams jobs{f.gatherJobs, f.numGatherJobs, slot.frameClaim.ptr, traceEnabled_ ? trace_.ptr : nullptr};
    CU(t360::launchGatherFrame(fp, jobs, maps, numSMs_, s));
  }

  // The render target of one plane's gather into the caller's plane `out`, pre-filled on s (reference transformPlane,
  // cpp:735-777).  When the caller's size is the map's, the gather writes into `out`; else (scale factors, or a caller that
  // asks for another size than it planned) into the scratch plane at the map's size, and finishTarget resizes it into `out`
  // with INTER_AREA.  BORDER_TRANSPARENT (`transparent`) leaves a pixel whose anchor tap lies outside the source as it
  // finds it, so the target is filled first: `out` with 128 for a chroma plane, nothing for luma (it keeps the caller's
  // bytes); the scratch plane with 0 (luma) or 128 (chroma).  plan: nullptr for the calls without one, which render at
  // the output's size (remap, lens rigs, rectilinear views).
  PlaneTarget renderTarget(const DevicePlan* plan, bool chroma, bool transparent, uint8_t* out, int outPitch, int outW, int outH,
                           DeviceBuffer<uint8_t>* scratch, cudaStream_t s) {
    PlaneTarget t{out, outPitch, outW, outH, out, outPitch, outW, outH, nullptr};
    if (plan && (outW != plan->mapW || outH != plan->mapH)) {
      t.resize = &resizeFor(*plan, outW, outH);
      t.dstPitch = scratchPlane(*scratch, plan->mapW, plan->mapH);
      t.dst = scratch->ptr;
      t.dstW = plan->mapW;
      t.dstH = plan->mapH;
      if (transparent) CU(cudaMemset2DAsync(t.dst, t.dstPitch, chroma ? 128 : 0, t.dstW, t.dstH, s));
    } else if (transparent && chroma) {
      CU(cudaMemset2DAsync(out, outPitch, 128, outW, outH, s));
    }
    return t;
  }

  // What follows the gather: the INTER_AREA resize when the plane was rendered at the map's size into a scratch plane.
  void finishTarget(const PlaneTarget& t, cudaStream_t s) {
    if (!t.resize) return;
    const DevicePlan::Resize& r = *t.resize;
    t360::AreaParams ap{t.dst, t.out, t.dstW, t.dstH, t.dstPitch, t.outW, t.outH, t.outPitch,
                        r.cellW, r.cellH, r.xTaps.ptr, r.xFirst.ptr, r.yTaps.ptr, r.yFirst.ptr, r.xLinear.ptr, r.yLinear.ptr, r.xMax};
    CU(t360::launchAreaResize(ap, s));
  }

  // ---- re-planning: reconfigure and the background planner of reconfigureAsync --------------------------------------
  struct PlanSizes { int index, inW, inH, outW, outH; };
  std::vector<PlanSizes> plannedSizes() {
    std::lock_guard<std::mutex> lock(mu_);
    std::vector<PlanSizes> sizes;
    for (const auto& kv : plans_) sizes.push_back({kv.first, kv.second.inW, kv.second.inH, kv.second.outW, kv.second.outH});
    return sizes;
  }

  // Whether frame planes of these sizes can take the per-frame kernels (the planned input sizes; a missing plan index is
  // reported by the path that follows).
  bool planesOfPlannedSize(const FramePlanes& f) {
    std::lock_guard<std::mutex> lock(mu_);
    for (int p = 0; p < f.numPlanes; ++p) {
      auto it = plans_.find(p ? 1 : 0);
      if (it != plans_.end() && (f.inW[p] != it->second.inW || f.inH[p] != it->second.inH)) return false;
    }
    return true;
  }

  // Whether some plan index holds a plan made from a caller's warp map; if so the calls that derive positions from the
  // context (re-plans, per-frame views, orientations and poses) are refused with a message prefixed by `what`.
  bool refuseWarpPlans(const char* what) {
    std::lock_guard<std::mutex> lock(mu_);
    for (const auto& kv : plans_)
      if (kv.second.warp) {
        std::printf("%s. Error: plan index %d was generated from a warp map, which has no geometry to re-plan or to move "
                    "(generateMapForPlane on the index replaces it)\n", what, kv.first);
        return true;
      }
    return false;
  }

  // The reader lock for an entry point that needs the plans of the current context: while a reconfigureAsync is pending it
  // first waits for them (without the settle interval).  Not owning the lock: the background planner failed (message).
  std::shared_lock<std::shared_mutex> lockPlanned(const char* what) {
    for (;;) {
      std::shared_lock<std::shared_mutex> config(configMu_);
      if (!perFrameOnly_) return config;
      config.unlock();
      if (reconfigureWait(true) < 0) {
        std::printf("%s. Error: the background planner failed on the current context\n", what);
        return {};
      }
    }
  }

  // Why reconfigureAsync refuses `next` (nullptr: accepted).  A refused context would leave frames on the per-frame kernels
  // with no plan ever to follow, so everything the planner can refuse is refused here, on the host.  With the layouts, stereo
  // formats and scale factors unchanged (checked under the writer lock) every plane and map size is the planned one, and what
  // buildHostPlan (sampling.cpp) refuses comes down to:
  //   - a non-positive plane or map size, and an invalid output layout (buildWarpMap): planned already, cannot occur;
  //   - with low-pass on, num_vertical_segments < 1, and whatever buildLowPassPlan (lowpass_plan.cpp) refuses: the same
  //     count, an invalid layout, a band of no rows.  It is run here for every planned index, so a refusal it may add later
  //     is caught too.
  // Refused besides: an interpolation_alg that is not NEAREST, LINEAR, CUBIC or LANCZOS4 (buildHostPlan makes a plan without
  // gather for it; the per-frame kernels need a kernel size), and a float field that is not finite.
  static const char* asyncRefusal(const FrameTransformContext& next, const std::vector<PlanSizes>& sizes) {
    if (t360::kernelSizeOf(next.interpolation_alg) == 0) return "unknown interpolation_alg";
    for (float v : {next.input_expand_coef, next.expand_coef, next.width_scale_factor, next.height_scale_factor, next.fixed_yaw,
                    next.fixed_pitch, next.fixed_roll, next.fixed_hfov, next.fixed_vfov, next.fixed_cube_offcenter_x,
                    next.fixed_cube_offcenter_y, next.fixed_cube_offcenter_z, next.kernel_height_scale_factor, next.min_kernel_half_height,
                    next.max_kernel_half_height, next.kernel_adjust_factor})
      if (!std::isfinite(v)) return "a float field is not finite";
    if (!next.enable_low_pass_filter) return nullptr;
    if (next.num_vertical_segments < 1) return "num_vertical_segments must be positive";
    for (const PlanSizes& z : sizes) {
      HostPlan h;
      h.ctx = next;
      h.inW = z.inW; h.inH = z.inH; h.outW = z.outW; h.outH = z.outH;
      h.mapW = static_cast<int>(next.width_scale_factor * z.outW + 0.5);
      h.mapH = static_cast<int>(next.height_scale_factor * z.outH + 0.5);
      if (!t360::buildLowPassPlan(h)) return "the low-pass planner refuses the context";
    }
    return nullptr;
  }

  // Host planning of every index in `sizes` for `next`, side by side (false: message, prefixed with `what`).
  static bool planAll(const FrameTransformContext& next, const std::vector<PlanSizes>& sizes, std::vector<HostIndexPlan>& host,
                      const char* what) {
    host.assign(sizes.size(), HostIndexPlan{});
    std::vector<int> planned(sizes.size(), 0);
    std::vector<std::string> errors(sizes.size());
    auto planOne = [&](size_t i) {
      try {
        planned[i] = planOnHost(next, sizes[i].inW, sizes[i].inH, sizes[i].outW, sizes[i].outH, host[i]);
      } catch (const std::exception& ex) {
        errors[i] = ex.what();
      }
    };
    std::vector<std::thread> pool;  // luma and chroma side by side (each planner is multi-threaded over rows as well)
    for (size_t i = 1; i < sizes.size(); ++i) pool.emplace_back(planOne, i);
    planOne(0);
    for (std::thread& t : pool) t.join();
    for (size_t i = 0; i < sizes.size(); ++i)
      if (!planned[i]) {
        std::printf("%s. Error: no plan for index %d%s%s\n", what, sizes[i].index, errors[i].empty() ? "" : ": ", errors[i].c_str());
        return false;
      }
    return true;
  }

  // Everything a context's plans are on the device, made off the enqueue path into fresh buffers: the plans of every index
  // and the merged lists of 2- and 3-plane frames (so the first frame after the swap does not rebuild them in frameLists,
  // which waits for the device).  After install() it holds what was swapped out.
  struct PlanSet {
    std::map<int, DevicePlan> plans;
    FrameLists lists[kPlaneLanes - 1];
    std::vector<PlaneGraph> graphs;
  };
  PlanSet makePlanSet(const FrameTransformContext& next, const std::vector<PlanSizes>& sizes, std::vector<HostIndexPlan>& host) {
    PlanSet set;
    for (size_t i = 0; i < sizes.size(); ++i) set.plans.emplace(sizes[i].index, upload(host[i], next));
    auto luma = set.plans.find(0), chroma = set.plans.find(1);
    if (luma != set.plans.end() && chroma != set.plans.end()) {
      const DevicePlan* planes[kPlaneLanes] = {&luma->second, &chroma->second, &chroma->second};
      for (int n = 2; n <= kPlaneLanes; ++n) {
        buildFrameLists(planes, n, set.lists[n - 2]);
        set.lists[n - 2].generation = planGeneration_ + 1;  // (the generation install() starts: planMu_ is held until then)
      }
    }
    return set;
  }

  // Swaps `set` in under the writer lock, with no device wait: from here on every entry point uses its plans.  `next`, the
  // context they were made for, becomes the current one unless a reconfigureAsync newer than `seq` has arrived since; then
  // the current context stays the newer one and whole frames stay on the per-frame kernels.  With `evenIfSuperseded`
  // false such a set is not swapped in (false returned).  Either way `set` then holds what retire() must release.
  bool install(PlanSet& set, const FrameTransformContext& next, unsigned long long seq, bool evenIfSuperseded) {
    std::unique_lock<std::shared_mutex> config(configMu_);  // no call of an entry point is in progress from here on
    std::lock_guard<std::mutex> async(asyncMu_);
    const bool current = asyncSeq_ == seq;
    if (!current && !evenIfSuperseded) return false;
    {
      std::lock_guard<std::mutex> lock(mu_);
      std::lock_guard<std::mutex> listsLock(frameListsMu_);
      plans_.swap(set.plans);
      for (int i = 0; i < kPlaneLanes - 1; ++i) std::swap(frameLists_[i], set.lists[i]);
      set.graphs.swap(planeGraphs_);  // (they launch the old plans' jobs)
      ++planGeneration_;  // the wave plans and the per-view low-pass caches are rebuilt on first use
    }
    if (current) {
      std::memcpy(&ctx_, &next, sizeof(ctx_));
      perFrameOnly_ = false;
      asyncSettled_ = seq;
      asyncFailed_ = false;
      asyncCv_.notify_all();
    }
    return true;
  }

  // Releases what install() swapped out (or a set that was never swapped in) once the device has finished everything
  // enqueued so far: frames enqueued before the swap may still read the old plans and lists.
  void retire(PlanSet& old) {
    CU(cudaDeviceSynchronize());
    for (PlaneGraph& g : old.graphs) cudaGraphExecDestroy(g.exec);
    old.graphs.clear();
    old.plans.clear();
    for (FrameLists& f : old.lists) f = FrameLists{};
  }

  // The background planner (one thread per transform, started by the first reconfigureAsync after a plan): plans the
  // latest pending context once no newer one has arrived for kSettleInterval (at once when someone waits for it), and
  // installs it unless it has been superseded meanwhile.
  void planInBackground() {
    std::unique_lock<std::mutex> async(asyncMu_);
    bool contextSet = false;
    while (!asyncStop_) {
      if (asyncSettled_ == asyncSeq_) {
        asyncCv_.wait(async);
        continue;
      }
      const auto due = asyncLast_ + kSettleInterval;
      if (!asyncHurry_ && std::chrono::steady_clock::now() < due) {
        asyncCv_.wait_until(async, due);
        continue;
      }
      asyncHurry_ = false;
      const unsigned long long seq = asyncSeq_;
      const FrameTransformContext next = asyncCtx_;
      async.unlock();
      if (!contextSet && cuContext_) {  // the context the transform's frames live in (a caller may have made its own)
        if (auto setCurrent = reinterpret_cast<CUresult (*)(CUcontext)>(driverEntry("cuCtxSetCurrent"))) setCurrent(cuContext_);
        contextSet = true;
      }
      const bool failed = !planPending(next, seq);
      async.lock();
      if (failed && asyncSeq_ == seq && asyncSettled_ != seq) {
        asyncSettled_ = seq;
        asyncFailed_ = true;
        asyncCv_.notify_all();
      }
    }
  }

  // One background plan of `next` (reconfigureAsync number `seq`): false when planning or the upload failed (message).
  bool planPending(const FrameTransformContext& next, unsigned long long seq) {
    const char* what = "Could not reconfigure the transform in the background";
    auto superseded = [&] {
      std::lock_guard<std::mutex> async(asyncMu_);
      return asyncSeq_ != seq || asyncSettled_ == seq || asyncStop_;  // (settled: T360B200_reconfigure took over)
    };
    return guarded(what, [&] {
      std::lock_guard<std::mutex> planLock(planMu_);
      if (superseded()) return true;
      const std::vector<PlanSizes> sizes = plannedSizes();
      std::vector<HostIndexPlan> host;
      if (!planAll(next, sizes, host, what)) return false;
      if (superseded()) return true;
      const DeviceRestore restoreDevice = ensureDevice();
      PlanSet set = makePlanSet(next, sizes, host);
      // a blocking reconfigureWait that the swap wakes returns only once the old plans are released as well
      struct Retiring {
        VideoFrameTransform* t;
        explicit Retiring(VideoFrameTransform* self) : t(self) {
          std::lock_guard<std::mutex> async(t->asyncMu_);
          t->asyncRetiring_ = true;
        }
        ~Retiring() {
          std::lock_guard<std::mutex> async(t->asyncMu_);
          t->asyncRetiring_ = false;
          t->asyncCv_.notify_all();
        }
      } retiring(this);
      install(set, next, seq, false);
      retire(set);
      return true;
    });
  }

  // The per-frame kernels' sphere tables of the planes when no plan holds them (a pending reconfigureAsync, whose context
  // the plans were not made with, and lens frames): planes of mapW[p] x mapH[p], built on the host when the context or a size
  // changes (planes of the same size share them), staged through the slot's upload ring on `s`.  tables[p] receive the
  // device tables (nullptr for layouts without any); *used the ring entry to release after the launch.
  void sphereTablesFor(const FrameTransformContext& ctx, int numPlanes, const int* mapW, const int* mapH, StreamSlot& slot, cudaStream_t s,
                       const float** tables, UploadRing::Entry** used) {
    FrameTransformContext key = ctx;  // (the orientation plays no part in the tables)
    key.fixed_yaw = key.fixed_pitch = key.fixed_roll = key.fixed_hfov = key.fixed_vfov = 0;
    std::vector<int> sizes;
    for (int p = 0; p < numPlanes; ++p) sizes.insert(sizes.end(), {mapW[p], mapH[p]});
    if (slot.sphereSizes != sizes || std::memcmp(&slot.sphereCtx, &key, sizeof(key)) != 0) {
      slot.sphereBytes.clear();
      for (int p = 0; p < numPlanes; ++p) {
        int same = 0;
        while (same < p && (mapW[same] != mapW[p] || mapH[same] != mapH[p])) ++same;
        if (same < p) {
          slot.sphereAt[p] = slot.sphereAt[same];
          continue;
        }
        // (the tables depend on the map, not on the input)
        const std::vector<float> t =
            t360::buildSphereTables(t360::sphereGeometry(ctx, mapW[p], mapH[p], 1, 1, t360::kernelSizeOf(ctx.interpolation_alg)));
        slot.sphereAt[p] = t.empty() ? SIZE_MAX : slot.sphereBytes.size();
        const uint8_t* bytes = reinterpret_cast<const uint8_t*>(t.data());
        slot.sphereBytes.insert(slot.sphereBytes.end(), bytes, bytes + t.size() * sizeof(float));
      }
      slot.sphereCtx = key;
      slot.sphereSizes = sizes;
    }
    for (int p = 0; p < numPlanes; ++p) tables[p] = nullptr;
    if (slot.sphereBytes.empty()) return;
    const uint8_t* d = stageUpload(slot.sphereTables, slot.sphereBytes, s, used);
    for (int p = 0; p < numPlanes; ++p) {
      const size_t at = slot.sphereAt[p];
      if (at != SIZE_MAX) tables[p] = reinterpret_cast<const float*>(d + at);
    }
  }

  // The motion's sample table (rigMotionTable) on the device for work enqueued next on s, through the slot's upload ring
  // (*used: the entry to release after the launch), and the motion's per-frame constants pointing at it
  t360::RigMotion stageMotion(const T360LensRig& rig, const T360RigMotion& motion, const t360::LensRigModel& model, StreamSlot& slot,
                              cudaStream_t s, UploadRing::Entry** used) {
    const std::vector<float> table = rigMotionTable(rig, motion, model);
    const uint8_t* bytes = reinterpret_cast<const uint8_t*>(table.data());
    slot.motionBytes.assign(bytes, bytes + table.size() * sizeof(float));
    return rigMotion(motion, reinterpret_cast<const float*>(stageUpload(slot.motionTables, slot.motionBytes, s, used)));
  }

  FrameTransformContext ctx_;
  // Every entry point that enqueues work holds configMu_ shared for as long as it uses a plan or ctx_; install() swaps the
  // plans and reconfigureAsync replaces ctx_ under it exclusively.  planMu_ serialises planning (generateMapForPlane,
  // reconfigure, the background planner).  Lock order: planMu_, configMu_, asyncMu_, hostCallMu_, then the others.
  // Nothing waits for the background planner while holding configMu_ or planMu_.
  std::shared_mutex configMu_;
  std::mutex planMu_;
  std::mutex mu_;
  std::mutex lazyMu_;  // tables made on first use (resizeFor, blurFor, deviceWeights)
  std::map<int, DevicePlan> plans_;
  DeviceBuffer<int16_t> weights_[9];       // OpenCV's tables [1024][k][k] (general kernels), by kernel size
  DeviceBuffer<uint8_t> weightImages_[9];  // their shared-memory images for the frame kernel
  DeviceBuffer<uint8_t> stagingIn_, stagingOut_;
  std::mutex hostCallMu_;  // the synchronous host-pointer path shares the staging planes and the streams: one call at a time
  cudaStream_t copyIn_ = nullptr, copyOut_ = nullptr;
  std::vector<cudaEvent_t> chunkIn_, waveDone_, copiedOut_;  // per chunk
  WavePlan wavePlans_[2];  // plan index 0 / 1
  long long pipelineMinBytes_ = 6ll << 20;
  bool pipelineStrict_ = false;  // T360B200_PIPELINE_STRICT (tests): see transformHostPlanPipelined
  static constexpr uint8_t kStrictPoison = 0xA5;
  std::vector<PlaneGraph> planeGraphs_;  // (see PlaneGraph)
  unsigned long long graphClock_ = 0;
  cudaEvent_t graphFork_ = nullptr, graphJoinIn_ = nullptr, graphJoinOut_ = nullptr;
  // opt-in page-locking of recurring pageable caller planes (ffmpeg recycles its frame pool): see pinIfRecurring()
  struct HostRange { uintptr_t base; size_t bytes; int seen; bool pinned; };
  std::vector<HostRange> hostRanges_;
  bool pinHostPlanes_ = false;
  std::mutex slotMu_;
  std::map<cudaStream_t, std::unique_ptr<StreamSlot>> slots_;
  FrameLists frameLists_[kPlaneLanes - 1];  // frames of 2 and 3 planes
  std::mutex frameListsMu_;
  DeviceBuffer<unsigned long long> trace_;
  bool traceEnabled_ = false;
  unsigned long long planGeneration_ = 0;
  cudaStream_t stream_ = nullptr;
  int device_ = 0, numSMs_ = 0;
  bool deviceReady_ = false;
  CUcontext cuContext_ = nullptr;  // the context current when the transform first touched CUDA (the background planner's)
  // reconfigureAsync: ctx_ is not the context the plans were made with, so whole frames take the per-frame kernels (configMu_)
  bool perFrameOnly_ = false;
  // the background planner (planInBackground), under asyncMu_: reconfigureAsync calls accepted after a plan existed, and the
  // number of the last one settled (installed, taken over by reconfigure, or failed: asyncFailed_)
  std::mutex asyncMu_;
  std::condition_variable asyncCv_;
  std::thread worker_;
  unsigned long long asyncSeq_ = 0, asyncSettled_ = 0;
  bool asyncFailed_ = false, asyncHurry_ = false, asyncStop_ = false;
  bool asyncRetiring_ = false;  // the background planner has swapped in a set and is releasing the one it replaced
  FrameTransformContext asyncCtx_{};
  std::chrono::steady_clock::time_point asyncLast_{};
};

// ---- the reference C-ABI (VideoFrameTransformHandler.h:22-47) ------------------------------------------
T360_API VideoFrameTransform* VideoFrameTransform_new(FrameTransformContext* ctx) {
  if (!ctx) return nullptr;
  return new (std::nothrow) VideoFrameTransform(ctx);
}

T360_API void VideoFrameTransform_delete(VideoFrameTransform* transform) { delete transform; }

T360_API int VideoFrameTransform_generateMapForPlane(VideoFrameTransform* transform, int inputWidth, int inputHeight,
                                                     int outputWidth, int outputHeight, int transformMatPlaneIndex) {
  if (!transform) return 0;
  return transform->generateMapForPlane(inputWidth, inputHeight, outputWidth, outputHeight, transformMatPlaneIndex);
}

T360_API int T360B200_generateMapFromWarp(VideoFrameTransform* t, const float* map, int mapW, int mapH, int inW, int inH, int border,
                                          int planIndex) {
  if (!t) return 0;
  return t->generateMapFromWarp(map, mapW, mapH, inW, inH, border, planIndex);
}

T360_API int VideoFrameTransform_transformFramePlane(VideoFrameTransform* transform, uint8_t* inputData,
                                                     uint8_t* outputData, int inputWidth, int inputHeight,
                                                     int inputWidthWithPadding, int outputWidth, int outputHeight,
                                                     int outputWidthWithPadding, int transformMatPlaneIndex,
                                                     int imagePlaneIndex) {
  if (!transform) return 0;
  return transform->transformFramePlane(inputData, outputData, inputWidth, inputHeight, inputWidthWithPadding,
                                        outputWidth, outputHeight, outputWidthWithPadding, transformMatPlaneIndex,
                                        imagePlaneIndex);
}

// ---- extensions (transform360_b200.h) --------------------------------------------------------------------
struct T360HostPlan {
  HostPlan plan;
  t360::GatherPlan gather;  // built on first use by T360B200_hostPlanGather
  bool gatherBuilt = false;
  std::vector<GatherJob> deviceJobs;      // built on first use by T360B200_hostPlanDeviceLists
  std::vector<uint32_t> deviceRecords;
  std::vector<uint8_t> blurImage;  // the last T360B200_hostPlanBlurLists image made with this plan first
  t360::WaveSchedule waves;        // the last T360B200_hostPlanWaves schedule
  std::vector<int32_t> waveRects;  // its rectangles, {wave, x0, y0, x1, y1} each
};

T360_API T360HostPlan* T360B200_hostPlanCreate(const FrameTransformContext* ctx, int inW, int inH, int outW, int outH) {
  if (!ctx) return nullptr;
  std::unique_ptr<T360HostPlan> p(new (std::nothrow) T360HostPlan);
  if (!p) return nullptr;
  try {
    if (!t360::buildHostPlan(*ctx, inW, inH, outW, outH, p->plan)) return nullptr;
  } catch (const std::exception& ex) {
    std::printf("Could not build the host plan. Error: %s\n", ex.what());
    return nullptr;
  }
  return p.release();
}
T360_API T360HostPlan* T360B200_hostPlanCreateFromWarp(const FrameTransformContext* ctx, const float* map, int mapW, int mapH, int inW,
                                                       int inH, int border) {
  if (!ctx) return nullptr;
  std::unique_ptr<T360HostPlan> p(new (std::nothrow) T360HostPlan);
  if (!p) return nullptr;
  try {
    if (!t360::buildWarpHostPlan(*ctx, map, mapW, mapH, inW, inH, border, p->plan)) return nullptr;
  } catch (const std::exception& ex) {
    std::printf("Could not build the host plan. Error: %s\n", ex.what());
    return nullptr;
  }
  return p.release();
}
T360_API void T360B200_hostPlanDestroy(T360HostPlan* plan) { delete plan; }
T360_API int T360B200_hostPlanInfo(const T360HostPlan* plan, int info[6]) {
  if (!plan || !info) return 0;
  info[0] = plan->plan.mapW; info[1] = plan->plan.mapH;
  info[2] = static_cast<int>(plan->plan.segments.size());
  info[3] = static_cast<int>(plan->plan.taps.size());
  info[4] = plan->plan.kernelSize;
  info[5] = 0;
  return 1;
}
T360_API const float* T360B200_hostPlanMap(const T360HostPlan* plan) { return plan ? plan->plan.map.data() : nullptr; }
T360_API const int32_t* T360B200_hostPlanSamples(const T360HostPlan* plan) {
  return plan && !plan->plan.samples.empty() ? reinterpret_cast<const int32_t*>(plan->plan.samples.data()) : nullptr;
}
T360_API int T360B200_hostPlanGather(T360HostPlan* plan, int info[10], const int32_t** jobs, const int32_t** records,
                                     const uint32_t** compact) {
  if (!plan || !info || plan->plan.kernelSize <= 0) return 0;
  try {
    if (!plan->gatherBuilt) {
      t360::buildGatherPlan(plan->plan, plan->plan.kernelSize >= 2 && !plan->plan.transparentBorder, plan->gather);
      plan->gatherBuilt = true;
    }
  } catch (const std::exception& ex) {
    std::printf("Could not build the gather plan. Error: %s\n", ex.what());
    return 0;
  }
  const t360::GatherPlan& g = plan->gather;
  info[0] = g.tilesPerRow; info[1] = g.tileRows; info[2] = g.tileH; info[3] = static_cast<int>(g.jobs.size());
  info[4] = g.numStaged[0]; info[5] = g.numStaged[1]; info[6] = g.numSeam; info[7] = g.numGeneral;
  info[8] = g.numShare; info[9] = static_cast<int>(g.compact.size());
  if (jobs) *jobs = g.jobs.empty() ? nullptr : reinterpret_cast<const int32_t*>(g.jobs.data());
  if (records) *records = reinterpret_cast<const int32_t*>(g.records.data());
  if (compact) *compact = g.compact.empty() ? nullptr : g.compact.data();
  return 1;
}
T360_API int T360B200_hostPlanPoleCaps(T360HostPlan* plan, int info[4], const int32_t** capJobs, const uint32_t** capRecords,
                                       const int32_t** launchJobs) {
  int gatherInfo[10];
  if (!plan || !info || !T360B200_hostPlanGather(plan, gatherInfo, nullptr, nullptr, nullptr)) return 0;
  const t360::GatherPlan& g = plan->gather;
  info[0] = g.numCap; info[1] = g.numBorder; info[2] = static_cast<int>(g.capRecords.size());
  info[3] = static_cast<int>(g.launchJobs.size());
  if (capJobs) *capJobs = g.capJobs.empty() ? nullptr : reinterpret_cast<const int32_t*>(g.capJobs.data());
  if (capRecords) *capRecords = g.capRecords.empty() ? nullptr : g.capRecords.data();
  if (launchJobs) *launchJobs = g.launchJobs.empty() ? nullptr : reinterpret_cast<const int32_t*>(g.launchJobs.data());
  return 1;
}
T360_API int T360B200_hostPlanLaunchExtents(T360HostPlan* plan, int* numJobs, const int32_t** needRows, const int32_t** rects) {
  int gatherInfo[10];
  if (!plan || !numJobs || !T360B200_hostPlanGather(plan, gatherInfo, nullptr, nullptr, nullptr)) return 0;
  const t360::GatherPlan& g = plan->gather;
  *numJobs = static_cast<int>(g.launchJobs.size());
  if (needRows) *needRows = g.launchNeedRows.empty() ? nullptr : g.launchNeedRows.data();
  if (rects) *rects = g.launchRects.empty() ? nullptr : reinterpret_cast<const int32_t*>(g.launchRects.data());
  return 1;
}
T360_API int T360B200_hostPlanWaves(T360HostPlan* plan, int chunks, const int32_t* needRows, int info[3], const int32_t** chunkRowEnd,
                                    const int32_t** waveStart, const int32_t** order, const int32_t** rects) {
  int gatherInfo[10];
  if (!plan || !info || chunks < 0 || chunks > 64 || !T360B200_hostPlanGather(plan, gatherInfo, nullptr, nullptr, nullptr)) return 0;
  const t360::GatherPlan& g = plan->gather;
  const HostPlan& h = plan->plan;
  if (!chunks) chunks = t360::pipelineChunks(h.inW, h.inH);
  const std::vector<int> rows = needRows ? std::vector<int>(needRows, needRows + g.launchNeedRows.size()) : g.launchNeedRows;
  plan->waves = t360::scheduleWaves(rows, g.launchRects, h.inH, h.mapW, h.mapH, chunks);
  plan->waveRects.clear();
  for (int c = 0; c < chunks; ++c)
    for (const t360::JobRect& r : plan->waves.rects[c]) plan->waveRects.insert(plan->waveRects.end(), {c, r.x0, r.y0, r.x1, r.y1});
  info[0] = chunks;
  info[1] = static_cast<int>(plan->waves.order.size());
  info[2] = static_cast<int>(plan->waveRects.size() / 5);
  if (chunkRowEnd) *chunkRowEnd = plan->waves.chunkRowEnd.data();
  if (waveStart) *waveStart = plan->waves.waveStart.data();
  if (order) *order = plan->waves.order.empty() ? nullptr : plan->waves.order.data();
  if (rects) *rects = plan->waveRects.empty() ? nullptr : plan->waveRects.data();
  return 1;
}
T360_API int T360B200_hostPlanDeviceLists(T360HostPlan* plan, int info[2], const int32_t** jobs, const uint32_t** records) {
  int gatherInfo[10];
  if (!plan || !info || !jobs || !records || !T360B200_hostPlanGather(plan, gatherInfo, nullptr, nullptr, nullptr)) return 0;
  const t360::GatherPlan& g = plan->gather;
  if (plan->deviceJobs.size() != g.launchJobs.size()) {
    plan->deviceJobs = t360::deviceJobs(g);
    plan->deviceRecords = t360::deviceRecords(g, plan->plan.kernelSize);
  }
  info[0] = static_cast<int>(plan->deviceJobs.size());
  info[1] = static_cast<int>(plan->deviceRecords.size());
  *jobs = plan->deviceJobs.empty() ? nullptr : reinterpret_cast<const int32_t*>(plan->deviceJobs.data());
  *records = plan->deviceRecords.empty() ? nullptr : plan->deviceRecords.data();
  return 1;
}
T360_API int T360B200_hostPlanBlurLists(T360HostPlan* const* plans, int numPlans, int width, int height, int layout[15],
                                        const uint8_t** image) {
  if (!plans || numPlans < 1 || numPlans > t360::kMaxFramePlanes || !layout || !image) return 0;
  for (int p = 0; p < numPlans; ++p)
    if (!plans[p]) return 0;
  try {
    t360::BlurLists lists[t360::kMaxFramePlanes];
    const t360::BlurLists* planes[t360::kMaxFramePlanes];
    bool clear = false;
    for (int p = 0; p < numPlans; ++p) {
      const HostPlan& h = plans[p]->plan;
      bool c = false;
      t360::buildBlurLists(h.segments, h.taps, width > 0 ? width : h.inW, height > 0 ? height : h.inH, h.ctx.input_stereo_format, lists[p], &c);
      clear = clear || c;
      planes[p] = &lists[p];
    }
    std::vector<uint8_t>& img = plans[0]->blurImage;
    img.clear();
    const t360::BlurLayout l = t360::packBlurLists(numPlans > 1 ? t360::mergeBlurLists(planes, numPlans) : lists[0], img, img);
    const long long v[15] = {l.numStrips[0], l.numStrips[1], l.numStrips[2], l.numTiles, l.numDirect, l.numTaps, l.tileSmem, clear,
                             static_cast<long long>(l.stripAt[0]), static_cast<long long>(l.stripAt[1]), static_cast<long long>(l.stripAt[2]),
                             static_cast<long long>(l.tileAt), static_cast<long long>(l.directAt), static_cast<long long>(l.tapAt),
                             static_cast<long long>(img.size())};
    for (int i = 0; i < 15; ++i) layout[i] = static_cast<int>(v[i]);
    *image = img.data();
    return 1;
  } catch (const std::exception& ex) {
    std::printf("Could not build the low-pass lists. Error: %s\n", ex.what());
    return 0;
  }
}
T360_API int T360B200_hostPlanSegment(const T360HostPlan* plan, int i, int rect[4], int numTaps[2], const float** kx,
                                      const float** ky) {
  if (!plan || i < 0 || i >= static_cast<int>(plan->plan.segments.size())) return 0;
  const t360::LowPassSegment& s = plan->plan.segments[i];
  rect[0] = s.left; rect[1] = s.top; rect[2] = s.width; rect[3] = s.height;
  numTaps[0] = s.kxCount; numTaps[1] = s.kyCount;
  if (kx) *kx = plan->plan.taps.data() + s.kxOffset;
  if (ky) *ky = plan->plan.taps.data() + s.kyOffset;
  return 1;
}
T360_API int T360B200_remapTable(int interpolationAlg, const int16_t** table) { return t360::remapTable(interpolationAlg, table); }
T360_API int T360B200_dealLanes(int interpolationAlg, int n, const int32_t* phases, int32_t* laneOf, int32_t* copyOf) {
  const int16_t* table = nullptr;
  const int k = t360::remapTable(interpolationAlg, &table);
  if (k < 2 || n < 0 || n > 32 || !phases || !laneOf || !copyOf) return -1;
  int slot[32], lane[32], copy[32];
  for (int i = 0; i < n; ++i) slot[i] = t360::weightSlotOf(k, phases[i] & 1023);
  const int wavefronts = t360::dealLanes(k, t360::weightCopies(k), n, slot, lane, copy);
  for (int i = 0; i < n; ++i) { laneOf[i] = lane[i]; copyOf[i] = copy[i]; }
  return wavefronts;
}

T360_API int T360B200_weightImage(int interpolationAlg, const uint8_t** image) {
  static std::mutex mu;
  static std::map<int, std::vector<uint8_t>> images;
  const int16_t* table = nullptr;
  const int k = t360::remapTable(interpolationAlg, &table);
  if (k < 2 || !image) return 0;
  std::lock_guard<std::mutex> lock(mu);
  auto it = images.find(k);
  if (it == images.end()) it = images.emplace(k, t360::buildWeightImage(k, table)).first;
  *image = it->second.data();
  return static_cast<int>(it->second.size());
}

T360_API int T360B200_transformFramePlaneAsync(VideoFrameTransform* t, const uint8_t* dIn, uint8_t* dOut, int inW, int inH,
                                               int inPitch, int outW, int outH, int outPitch, int planIndex, void* stream) {
  if (!t || !dIn || !dOut) return 0;
  return t->transformDevice(dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, planIndex, static_cast<cudaStream_t>(stream));
}
T360_API int T360B200_transformFrameAsync(VideoFrameTransform* t, int numPlanes, const uint8_t* const* dIn, uint8_t* const* dOut,
                                          const int* inW, const int* inH, const int* inPitch, const int* outW, const int* outH,
                                          const int* outPitch, void* stream) {
  FramePlanes f;
  if (!t || !describeFrame("Could not transform the frame", numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, f)) return 0;
  return t->transformFrameDevice(f, static_cast<cudaStream_t>(stream));
}
T360_API int T360B200_lowPassPlaneAsync(VideoFrameTransform* t, const uint8_t* dIn, uint8_t* dOut, int w, int h, int inPitch,
                                        int outPitch, int planIndex, void* stream) {
  if (!t || !dIn || !dOut) return 0;
  return t->lowPassDevice(dIn, dOut, w, h, inPitch, outPitch, planIndex, static_cast<cudaStream_t>(stream));
}
T360_API int T360B200_reconfigure(VideoFrameTransform* t, const FrameTransformContext* ctx) {
  if (!t || !ctx) return 0;
  return t->reconfigure(*ctx);
}
T360_API int T360B200_reconfigureAsync(VideoFrameTransform* t, const FrameTransformContext* ctx) {
  if (!t || !ctx) return 0;
  return t->reconfigureAsync(*ctx);
}
T360_API int T360B200_reconfigureWait(VideoFrameTransform* t, int block) {
  if (!t) return -1;
  return t->reconfigureWait(block != 0);
}
T360_API int T360B200_transformFrameViewAsync(VideoFrameTransform* t, const T360View* view, int numPlanes, const uint8_t* const* dIn,
                                              uint8_t* const* dOut, const int* inW, const int* inH, const int* inPitch, const int* outW,
                                              const int* outH, const int* outPitch, void* stream) {
  const char* what = "Could not transform the frame with a view";
  FramePlanes f;
  if (!t || !view || !describeFrame(what, numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, f)) return 0;
  return t->transformFrameWith(what, *view, f, static_cast<cudaStream_t>(stream));
}
// The sampling records of one plane of `ctx` with the frame's view fields `fields` (withFields) as the per-frame kernels
// compute them: FLAT_FIXED by flat_view.h, every other layout by oriented_view.h.  `what` names the call in the messages.
template <class Fields>
static int perFrameSamples(const char* what, const FrameTransformContext* context, const Fields* fields, int inW, int inH, int outW, int outH,
                           int32_t* samples) {
  if (!context || !fields || !samples) return 0;
  FrameTransformContext ctx = *context;
  const std::string why = withFields(ctx, *fields);
  if (!why.empty()) {
    std::printf("Could not compute the %s's samples. Error: %s\n", what, why.c_str());
    return 0;
  }
  const int k = t360::kernelSizeOf(ctx.interpolation_alg);
  const int mapW = static_cast<int>(ctx.width_scale_factor * outW + 0.5), mapH = static_cast<int>(ctx.height_scale_factor * outH + 0.5);
  if (k == 0 || inW <= 0 || inH <= 0 || outW <= 0 || outH <= 0 || mapW <= 0 || mapH <= 0) {
    std::printf("Could not compute the %s's samples. Error: invalid interpolation or plane sizes\n", what);
    return 0;
  }
  const t360::SphereGeometry g = t360::sphereGeometry(ctx, mapW, mapH, inW, inH, k);
  if (ctx.output_layout == LAYOUT_FLAT_FIXED) {
    const t360::FlatView v{ctx.fixed_yaw, ctx.fixed_pitch, ctx.fixed_hfov, ctx.fixed_vfov};
    for (int i = 0; i < mapH; ++i)
      for (int j = 0; j < mapW; ++j) {
        int32_t* out = samples + 2 * (static_cast<size_t>(i) * mapW + j);
        t360::flatSample(v, g, i, j, out, out + 1);
      }
    return 1;
  }
  const std::vector<float> tables = t360::buildSphereTables(g);
  const float* colTab = tables.data();
  const float* rowTab = tables.empty() ? nullptr : tables.data() + t360::sphereTableRowOffset(g);
  const t360::Rotation r = t360::rotationFromAngles(ctx.fixed_yaw, ctx.fixed_pitch, ctx.fixed_roll);
  for (int i = 0; i < mapH; ++i)
    for (int j = 0; j < mapW; ++j) {
      int32_t* out = samples + 2 * (static_cast<size_t>(i) * mapW + j);
      t360::sphereSample(g, r, colTab, rowTab, i, j, out, out + 1);
    }
  return 1;
}

T360_API int T360B200_viewSamples(const FrameTransformContext* ctx, const T360View* view, int inW, int inH, int outW, int outH, int32_t* samples) {
  return perFrameSamples("view", ctx, view, inW, inH, outW, outH, samples);
}
T360_API int T360B200_transformFrameOrientedAsync(VideoFrameTransform* t, const T360Orientation* orientation, int numPlanes,
                                                  const uint8_t* const* dIn, uint8_t* const* dOut, const int* inW, const int* inH,
                                                  const int* inPitch, const int* outW, const int* outH, const int* outPitch, void* stream) {
  const char* what = "Could not transform the frame with an orientation";
  FramePlanes f;
  if (!t || !orientation || !describeFrame(what, numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, f)) return 0;
  return t->transformFrameWith(what, *orientation, f, static_cast<cudaStream_t>(stream));
}
T360_API int T360B200_orientedSamples(const FrameTransformContext* ctx, const T360Orientation* orientation, int inW, int inH, int outW,
                                      int outH, int32_t* samples) {
  return perFrameSamples("orientation", ctx, orientation, inW, inH, outW, outH, samples);
}
T360_API int T360B200_transformFramePoseAsync(VideoFrameTransform* t, const T360Pose* pose, int numPlanes, const uint8_t* const* dIn,
                                              uint8_t* const* dOut, const int* inW, const int* inH, const int* inPitch, const int* outW,
                                              const int* outH, const int* outPitch, void* stream) {
  const char* what = "Could not transform the frame with a pose";
  FramePlanes f;
  if (!t || !pose || !describeFrame(what, numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, f)) return 0;
  return t->transformFrameWith(what, *pose, f, static_cast<cudaStream_t>(stream));
}
T360_API int T360B200_poseSamples(const FrameTransformContext* ctx, const T360Pose* pose, int inW, int inH, int outW, int outH, int32_t* samples) {
  return perFrameSamples("pose", ctx, pose, inW, inH, outW, outH, samples);
}
T360_API int T360B200_remapFrameAsync(VideoFrameTransform* t, int numPlanes, const float* const* maps, const int* mapPitches, int border,
                                      const uint8_t* const* dIn, uint8_t* const* dOut, const int* inW, const int* inH, const int* inPitch,
                                      const int* outW, const int* outH, const int* outPitch, void* stream) {
  const char* what = "Could not remap the frame";
  if (!t || !maps || !mapPitches) {
    std::printf("%s. Error: a NULL argument\n", what);
    return 0;
  }
  FramePlanes f;
  if (!describeFrame(what, numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, f)) return 0;
  return t->remapFrame(maps, mapPitches, border, f, static_cast<cudaStream_t>(stream));
}
namespace {
// A rig or camera frame call: a NULL transform, then the frame's arrays (describeFrame), then run(*t, f, stream).
template <class Run>
int frameCall(const char* what, VideoFrameTransform* t, int numPlanes, const uint8_t* const* dIn, uint8_t* const* dOut, const int* inW,
              const int* inH, const int* inPitch, const int* outW, const int* outH, const int* outPitch, void* stream, Run&& run) {
  if (!t) {
    std::printf("%s. Error: a NULL argument\n", what);
    return 0;
  }
  FramePlanes f;
  if (!describeFrame(what, numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, f)) return 0;
  return run(*t, f, static_cast<cudaStream_t>(stream));
}
}  // namespace
T360_API int T360B200_lensMap(const FrameTransformContext* ctx, const T360LensRig* rig, const T360Orientation* orientation, int inW, int inH,
                              int outW, int outH, float* map) {
  auto refused = [&](const FrameTransformContext& c, std::string* why) {
    return lensRefused(c, rig, orientation, why) ||
           outputsRefused({map}, inW, inH, outW, outH, "a NULL map or a plane size that is not positive", why);
  };
  return twinCall("Could not compute the lens map", ctx, refused, [&](const FrameTransformContext& c) {
    const t360::LensRigModel model = lensRigModel(*rig);
    forLensPixels(c, *orientation, inW, inH, outW, outH, [&](const t360::SphereGeometry& g, const t360::Rotation& r, const float* colTab,
                                                             const float* rowTab, int i, int j, size_t at) {
      t360::lensPoint(g, r, model, colTab, rowTab, i, j, map + 2 * at, map + 2 * at + 1);
    });
  });
}
T360_API int T360B200_lensBlendMaps(const FrameTransformContext* ctx, const T360LensRig* rig, float seamWidth, const T360Orientation* orientation,
                                    int inW, int inH, int outW, int outH, float* map0, float* map1, uint16_t* weight) {
  auto refused = [&](const FrameTransformContext& c, std::string* why) {
    return lensBlendRefused(c, rig, seamWidth, orientation, why) ||
           outputsRefused({map0, map1, weight}, inW, inH, outW, outH, "a NULL map or weight array or a plane size that is not positive", why);
  };
  return twinCall("Could not compute the lens blend maps", ctx, refused, [&](const FrameTransformContext& c) {
    const t360::LensRigModel model = lensRigModel(*rig);
    const float s = lensSeamScale(seamWidth);
    forLensPixels(c, *orientation, inW, inH, outW, outH, [&](const t360::SphereGeometry& g, const t360::Rotation& r, const float* colTab,
                                                             const float* rowTab, int i, int j, size_t at) {
      weight[at] = static_cast<uint16_t>(t360::lensBlendPoint(g, r, model, s, colTab, rowTab, i, j, map0 + 2 * at, map1 + 2 * at));
    });
  });
}
T360_API int T360B200_transformFrameLensAsync(VideoFrameTransform* t, const T360LensRig* rig, const T360Orientation* orientation, int numPlanes,
                                              const uint8_t* const* dIn, uint8_t* const* dOut, const int* inW, const int* inH, const int* inPitch,
                                              const int* outW, const int* outH, const int* outPitch, void* stream) {
  const char* what = "Could not transform the frame with a lens rig";
  return frameCall(what, t, numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, stream,
                   [&](VideoFrameTransform& vft, const FramePlanes& f, cudaStream_t s) { return vft.transformFrameLens(what, rig, nullptr, orientation, f, s); });
}
T360_API int T360B200_transformFrameLensBlendAsync(VideoFrameTransform* t, const T360LensRig* rig, float seamWidth, const T360Orientation* orientation,
                                                   int numPlanes, const uint8_t* const* dIn, uint8_t* const* dOut, const int* inW, const int* inH,
                                                   const int* inPitch, const int* outW, const int* outH, const int* outPitch, void* stream) {
  const char* what = "Could not blend the frame of a lens rig";
  return frameCall(what, t, numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, stream,
                   [&](VideoFrameTransform& vft, const FramePlanes& f, cudaStream_t s) { return vft.transformFrameLens(what, rig, &seamWidth, orientation, f, s); });
}
T360_API int T360B200_lensPhotoMaps(const FrameTransformContext* ctx, const T360LensRig* rig, const T360RigPhotometry* photometry, float seamWidth,
                                    const T360Orientation* orientation, int plane, int inW, int inH, int outW, int outH, float* map0, float* map1,
                                    uint16_t* weight, uint16_t* gain0, uint16_t* gain1) {
  auto refused = [&](const FrameTransformContext& c, std::string* why) {
    return lensPhotoRefused(c, rig, photometry, seamWidth, orientation, why) || indexRefused("plane", plane, 2, why) ||
           outputsRefused({map0, map1, weight, gain0, gain1}, inW, inH, outW, outH,
                          "a NULL map, weight or gain array or a plane size that is not positive", why);
  };
  return twinCall("Could not compute the lens photometry maps", ctx, refused, [&](const FrameTransformContext& c) {
    const t360::LensRigModel model = lensRigModel(*rig);
    const t360::LensPhotoPlane ph = lensPhotoPlane(*photometry, rig->numLenses, plane);
    const float s = seamWidth > 0.0f ? lensSeamScale(seamWidth) : 0.0f;
    forLensPixels(c, *orientation, inW, inH, outW, outH, [&](const t360::SphereGeometry& g, const t360::Rotation& r, const float* colTab,
                                                             const float* rowTab, int i, int j, size_t at) {
      int g0, g1;
      bool overlap;
      weight[at] = static_cast<uint16_t>(
          t360::lensPhotoPoint(g, r, model, s, /*both=*/true, ph, colTab, rowTab, i, j, map0 + 2 * at, map1 + 2 * at, &g0, &g1, &overlap));
      gain0[at] = static_cast<uint16_t>(g0);
      gain1[at] = static_cast<uint16_t>(g1);
    });
  });
}
T360_API int T360B200_transformFrameLensPhotoAsync(VideoFrameTransform* t, const T360LensRig* rig, const T360RigPhotometry* photometry,
                                                   float seamWidth, const T360Orientation* orientation, unsigned long long* deviceStats,
                                                   int numPlanes, const uint8_t* const* dIn, uint8_t* const* dOut, const int* inW, const int* inH,
                                                   const int* inPitch, const int* outW, const int* outH, const int* outPitch, void* stream) {
  const char* what = "Could not transform the frame of a lens rig with photometry";
  if (t && !photometry) {  // (before the frame's checks: without a photometry transformFrameLens is the plain lens call)
    std::printf("%s. Error: a NULL photometry\n", what);
    return 0;
  }
  return frameCall(what, t, numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, stream,
                   [&](VideoFrameTransform& vft, const FramePlanes& f, cudaStream_t s) {
                     return vft.transformFrameLens(what, rig, &seamWidth, orientation, f, s, photometry, deviceStats);
                   });
}
T360_API int T360B200_lensMotionMaps(const FrameTransformContext* ctx, const T360LensRig* rig, const T360RigPhotometry* photometry, float seamWidth,
                                     const T360Orientation* orientation, const T360RigMotion* motion, int plane, int inW, int inH, int outW,
                                     int outH, float* map0, float* map1, uint16_t* weight, uint16_t* gain0, uint16_t* gain1) {
  auto refused = [&](const FrameTransformContext& c, std::string* why) {
    return lensPhotoRefused(c, rig, photometry, seamWidth, orientation, why) || motionRefused(*rig, motion, why) ||
           indexRefused("plane", plane, 2, why) ||
           outputsRefused({map0, map1, weight, gain0, gain1}, inW, inH, outW, outH,
                          "a NULL map, weight or gain array or a plane size that is not positive", why);
  };
  return twinCall("Could not compute the lens motion maps", ctx, refused, [&](const FrameTransformContext& c) {
    const t360::LensRigModel model = lensRigModel(*rig);
    const std::vector<float> table = rigMotionTable(*rig, *motion, model);
    const t360::RigMotion mo = rigMotion(*motion, table.data());
    const t360::LensPhotoPlane ph = lensPhotoPlane(*photometry, rig->numLenses, plane);
    const float s = seamWidth > 0.0f ? lensSeamScale(seamWidth) : 0.0f;
    forLensPixels(c, *orientation, inW, inH, outW, outH, [&](const t360::SphereGeometry& g, const t360::Rotation& r, const float* colTab,
                                                             const float* rowTab, int i, int j, size_t at) {
      int g0, g1;
      bool overlap;
      weight[at] = static_cast<uint16_t>(t360::lensMotionPoint(g, r, model, mo, s, /*both=*/true, ph, colTab, rowTab, i, j, map0 + 2 * at,
                                                               map1 + 2 * at, &g0, &g1, &overlap));
      gain0[at] = static_cast<uint16_t>(g0);
      gain1[at] = static_cast<uint16_t>(g1);
    });
  });
}
T360_API int T360B200_transformFrameLensMotionAsync(VideoFrameTransform* t, const T360LensRig* rig, const T360RigPhotometry* photometry,
                                                    float seamWidth, const T360Orientation* orientation, const T360RigMotion* motion,
                                                    unsigned long long* deviceStats, int numPlanes, const uint8_t* const* dIn, uint8_t* const* dOut,
                                                    const int* inW, const int* inH, const int* inPitch, const int* outW, const int* outH,
                                                    const int* outPitch, void* stream) {
  const char* what = "Could not transform the frame of a lens rig with a rig motion";
  if (t && !photometry) {  // (as the photometric call: without a photometry transformFrameLens is the plain lens call)
    std::printf("%s. Error: a NULL photometry\n", what);
    return 0;
  }
  return frameCall(what, t, numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, stream,
                   [&](VideoFrameTransform& vft, const FramePlanes& f, cudaStream_t s) {
                     return vft.transformFrameLens(what, rig, &seamWidth, orientation, f, s, photometry, deviceStats, true, motion);
                   });
}
namespace {
int cameraMap(const char* what, const FrameTransformContext* ctx, const CameraView& v, int inW, int inH, int outW, int outH, float* map) {
  auto refused = [&](const FrameTransformContext& c, std::string* why) {
    return viewRefused(c, v, why) || outputsRefused({map}, inW, inH, outW, outH, "a NULL map or a plane size that is not positive", why);
  };
  return twinCall(what, ctx, refused, [&](const FrameTransformContext& c) {
    forCameraPixels(c, v, inW, inH, outW, outH, [&](const t360::SphereGeometry& g, const t360::RectilinearCamera& cam, const t360::LensRigModel& model,
                                                    const t360::MipGeometry&, int, int i, int j, size_t at) {
      if (v.rig) t360::rectilinearPosition<true>(g, cam, model, i, j, map + 2 * at, map + 2 * at + 1);
      else t360::rectilinearPosition<false>(g, cam, model, i, j, map + 2 * at, map + 2 * at + 1);
    });
  });
}
// The twin of one lens and plane of a photometric (cameraPhotoMaps), stereo (stereoCameraMaps) or moving
// (cameraMotionMaps) view: cameraPhotoPoint<true, stereo> or cameraMotionPoint<true> of every pixel with both lenses
// projected; lensWeight the seam weight or the eye weight 256 e
int cameraPhotoMaps(const char* what, const FrameTransformContext* ctx, const CameraView& v, int lens, int plane, int inW, int inH, int outW,
                    int outH, float* map0, float* map1, uint8_t* level, uint16_t* weight, uint16_t* gain, uint16_t* lensWeight) {
  auto refused = [&](const FrameTransformContext& c, std::string* why) {
    return viewRefused(c, v, why) || indexRefused("lens", lens, 1, why) || indexRefused("plane", plane, 2, why) ||
           outputsRefused({map0, map1, level, weight, gain, lensWeight}, inW, inH, outW, outH,
                          "a NULL map, level, weight or gain array or a plane size that is not positive", why);
  };
  return twinCall(what, ctx, refused, [&](const FrameTransformContext& c) {
    const t360::LensPhotoPlane ph = lensPhotoPlane(*v.photometry, v.rig->numLenses, plane);
    const float s = v.seamWidth > 0.0f ? lensSeamScale(v.seamWidth) : 0.0f;
    const std::vector<float> table = v.moving ? rigMotionTable(*v.rig, *v.motion, lensRigModel(*v.rig)) : std::vector<float>{};
    const t360::RigMotion mo = v.moving ? rigMotion(*v.motion, table.data()) : t360::RigMotion{};
    forCameraPixels(c, v, inW, inH, outW, outH, [&](const t360::SphereGeometry& g, const t360::RectilinearCamera& cam, const t360::LensRigModel& model,
                                                    const t360::MipGeometry& m, int bias, int i, int j, size_t at) {
      t360::CameraPhotoLens e[2];
      bool overlap;
      lensWeight[at] = static_cast<uint16_t>(v.moving ? t360::cameraMotionPoint<true>(g, cam, model, mo, m, bias, s, /*both=*/true, ph, i, j, e, &overlap)
                                             : v.stereo ? t360::cameraPhotoPoint<true, true>(g, cam, model, m, bias, s, /*both=*/true, ph, i, j, e, &overlap)
                                                        : t360::cameraPhotoPoint<true>(g, cam, model, m, bias, s, /*both=*/true, ph, i, j, e, &overlap));
      map0[2 * at] = e[lens].p0[0];
      map0[2 * at + 1] = e[lens].p0[1];
      map1[2 * at] = e[lens].p1[0];
      map1[2 * at + 1] = e[lens].p1[1];
      level[at] = static_cast<uint8_t>(e[lens].level);
      weight[at] = static_cast<uint16_t>(e[lens].w);
      gain[at] = static_cast<uint16_t>(e[lens].gain);
    });
  });
}
int transformFrameView(const char* what, VideoFrameTransform* t, const CameraView& v, int numPlanes, const uint8_t* const* dIn, uint8_t* const* dOut,
                       const int* inW, const int* inH, const int* inPitch, const int* outW, const int* outH, const int* outPitch, void* stream) {
  return frameCall(what, t, numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, stream,
                   [&](VideoFrameTransform& vft, const FramePlanes& f, cudaStream_t s) { return vft.transformFrameView(what, v, f, s); });
}
}  // namespace
T360_API int T360B200_cameraMap(const FrameTransformContext* ctx, const T360LensRig* rig, const T360Pose* pose, const T360Camera* camera, int inW,
                                int inH, int outW, int outH, float* map) {
  return cameraMap("Could not compute the camera map", ctx, plainView(rig, pose, camera), inW, inH, outW, outH, map);
}
T360_API int T360B200_transformFrameCameraAsync(VideoFrameTransform* t, const T360LensRig* rig, const T360Pose* pose, const T360Camera* camera,
                                                int numPlanes, const uint8_t* const* dIn, uint8_t* const* dOut, const int* inW, const int* inH,
                                                const int* inPitch, const int* outW, const int* outH, const int* outPitch, void* stream) {
  return transformFrameView("Could not transform the frame with a camera view", t, plainView(rig, pose, camera), numPlanes, dIn,
                            dOut, inW, inH, inPitch, outW, outH, outPitch, stream);
}
T360_API int T360B200_rectilinearMap(const FrameTransformContext* ctx, const T360LensRig* rig, const T360Pose* pose, int inW, int inH, int outW,
                                     int outH, float* map) {
  return cameraMap("Could not compute the rectilinear map", ctx, plainView(rig, pose, &kPinhole), inW, inH, outW, outH, map);
}
T360_API int T360B200_transformFrameRectilinearAsync(VideoFrameTransform* t, const T360LensRig* rig, const T360Pose* pose, int numPlanes,
                                                     const uint8_t* const* dIn, uint8_t* const* dOut, const int* inW, const int* inH,
                                                     const int* inPitch, const int* outW, const int* outH, const int* outPitch, void* stream) {
  return transformFrameView("Could not transform the frame with a rectilinear view", t, plainView(rig, pose, &kPinhole), numPlanes,
                            dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, stream);
}
T360_API int T360B200_cameraMipMaps(const FrameTransformContext* ctx, const T360LensRig* rig, const T360Pose* pose, const T360Camera* camera,
                                    const T360Minify* minify, int inW, int inH, int outW, int outH, float* map0, float* map1, uint8_t* level,
                                    uint16_t* weight) {
  const CameraView v = plainView(rig, pose, camera, minify);
  auto refused = [&](const FrameTransformContext& c, std::string* why) {
    return viewRefused(c, v, why) || (!minify && minifyRefused(minify, why)) ||
           outputsRefused({map0, map1, level, weight}, inW, inH, outW, outH, "a NULL map, level or weight array or a plane size that is not positive",
                          why);
  };
  return twinCall("Could not compute the camera mip maps", ctx, refused, [&](const FrameTransformContext& c) {
    forCameraPixels(c, v, inW, inH, outW, outH, [&](const t360::SphereGeometry& g, const t360::RectilinearCamera& cam, const t360::LensRigModel& model,
                                                    const t360::MipGeometry& m, int bias, int i, int j, size_t at) {
      int w;
      level[at] = static_cast<uint8_t>(rig ? t360::mipCameraPoint<true>(g, cam, model, m, bias, i, j, map0 + 2 * at, map1 + 2 * at, &w)
                                           : t360::mipCameraPoint<false>(g, cam, model, m, bias, i, j, map0 + 2 * at, map1 + 2 * at, &w));
      weight[at] = static_cast<uint16_t>(w);
    });
  });
}
T360_API int T360B200_transformFrameCameraMipAsync(VideoFrameTransform* t, const T360LensRig* rig, const T360Pose* pose, const T360Camera* camera,
                                                   const T360Minify* minify, int numPlanes, const uint8_t* const* dIn, uint8_t* const* dOut,
                                                   const int* inW, const int* inH, const int* inPitch, const int* outW, const int* outH,
                                                   const int* outPitch, void* stream) {
  const char* what = "Could not transform the frame with an anti-aliased camera view";
  return frameCall(what, t, numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, stream,
                   [&](VideoFrameTransform& vft, const FramePlanes& f, cudaStream_t s) {
                     std::string why;
                     if (minifyRefused(minify, &why)) {  // (this call checks its minify before the pose and camera)
                       std::printf("%s. Error: %s\n", what, why.c_str());
                       return false;
                     }
                     return vft.transformFrameView(what, plainView(rig, pose, camera, minify), f, s);
                   });
}
T360_API int T360B200_cameraAnisoMaps(const FrameTransformContext* ctx, const T360LensRig* rig, const T360Pose* pose, const T360Camera* camera,
                                      const T360Minify* minify, int maxProbes, int inW, int inH, int outW, int outH, float* map0, float* map1,
                                      uint8_t* level, uint16_t* weight, uint8_t* probes) {
  const CameraView v = anisoView(rig, pose, camera, minify, maxProbes);
  auto refused = [&](const FrameTransformContext& c, std::string* why) {
    return viewRefused(c, v, why) || outputsRefused({map0, map1, level, weight, probes}, inW, inH, outW, outH,
                                                    "a NULL map, level, weight or probes array or a plane size that is not positive", why);
  };
  return twinCall("Could not compute the camera aniso maps", ctx, refused, [&](const FrameTransformContext& c) {
    const int maxLog2 = probesLog2(maxProbes);
    const size_t plane = static_cast<size_t>(outW) * outH;
    forCameraPixels(c, v, inW, inH, outW, outH, [&](const t360::SphereGeometry& g, const t360::RectilinearCamera& cam, const t360::LensRigModel& model,
                                                    const t360::MipGeometry& m, int bias, int i, int j, size_t at) {
      const t360::AnisoFootprint f = rig ? t360::anisoFootprint<true>(g, cam, model, m, bias, maxLog2, i, j)
                                         : t360::anisoFootprint<false>(g, cam, model, m, bias, maxLog2, i, j);
      for (int k = 0; k < maxProbes; ++k) {
        float* p0 = map0 + 2 * (k * plane + at);
        float* p1 = map1 + 2 * (k * plane + at);
        if (k >= (1 << f.e)) {
          p0[0] = p0[1] = p1[0] = p1[1] = t360::bitsFloat(0x7fc00000u);
        } else if (rig) {
          t360::anisoCameraPoint<true>(g, cam, model, m, f, k, p0, p1);
        } else {
          t360::anisoCameraPoint<false>(g, cam, model, m, f, k, p0, p1);
        }
      }
      level[at] = static_cast<uint8_t>(f.level);
      weight[at] = static_cast<uint16_t>(f.w);
      probes[at] = static_cast<uint8_t>(1 << f.e);
    });
  });
}
T360_API int T360B200_transformFrameCameraAnisoAsync(VideoFrameTransform* t, const T360LensRig* rig, const T360Pose* pose, const T360Camera* camera,
                                                     const T360Minify* minify, int maxProbes, int numPlanes, const uint8_t* const* dIn,
                                                     uint8_t* const* dOut, const int* inW, const int* inH, const int* inPitch, const int* outW,
                                                     const int* outH, const int* outPitch, void* stream) {
  const char* what = "Could not transform the frame with an anisotropic camera view";
  return frameCall(what, t, numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, stream,
                   [&](VideoFrameTransform& vft, const FramePlanes& f, cudaStream_t s) {
                     std::string why;
                     if (minifyRefused(minify, &why)) {  // (as the camera-mip call: the minify before the pose and camera)
                       std::printf("%s. Error: %s\n", what, why.c_str());
                       return false;
                     }
                     return vft.transformFrameView(what, anisoView(rig, pose, camera, minify, maxProbes), f, s);
                   });
}
T360_API int T360B200_cameraPhotoMaps(const FrameTransformContext* ctx, const T360LensRig* rig, const T360RigPhotometry* photometry, float seamWidth,
                                      const T360Pose* pose, const T360Camera* camera, const T360Minify* minify, int lens, int plane, int inW,
                                      int inH, int outW, int outH, float* map0, float* map1, uint8_t* level, uint16_t* weight, uint16_t* gain,
                                      uint16_t* seamWeight) {
  return cameraPhotoMaps("Could not compute the camera photometry maps", ctx,
                         photoView(rig, photometry, seamWidth, pose, camera, minify, nullptr, false),
                         lens, plane, inW, inH, outW, outH, map0, map1, level, weight, gain, seamWeight);
}
T360_API int T360B200_transformFrameCameraPhotoAsync(VideoFrameTransform* t, const T360LensRig* rig, const T360RigPhotometry* photometry,
                                                     float seamWidth, const T360Pose* pose, const T360Camera* camera, const T360Minify* minify,
                                                     unsigned long long* deviceStats, int numPlanes, const uint8_t* const* dIn,
                                                     uint8_t* const* dOut, const int* inW, const int* inH, const int* inPitch, const int* outW,
                                                     const int* outH, const int* outPitch, void* stream) {
  return transformFrameView("Could not transform the frame with a camera view of a lens rig with photometry", t,
                            photoView(rig, photometry, seamWidth, pose, camera, minify, deviceStats, false),
                            numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, stream);
}
T360_API int T360B200_cameraMotionMaps(const FrameTransformContext* ctx, const T360LensRig* rig, const T360RigPhotometry* photometry, float seamWidth,
                                       const T360Pose* pose, const T360Camera* camera, const T360Minify* minify, const T360RigMotion* motion, int lens,
                                       int plane, int inW, int inH, int outW, int outH, float* map0, float* map1, uint8_t* level, uint16_t* weight,
                                       uint16_t* gain, uint16_t* seamWeight) {
  return cameraPhotoMaps("Could not compute the camera motion maps", ctx, motionView(rig, photometry, seamWidth, pose, camera, minify, motion, nullptr),
                         lens, plane, inW, inH, outW, outH, map0, map1, level, weight, gain, seamWeight);
}
T360_API int T360B200_transformFrameCameraMotionAsync(VideoFrameTransform* t, const T360LensRig* rig, const T360RigPhotometry* photometry,
                                                      float seamWidth, const T360Pose* pose, const T360Camera* camera, const T360Minify* minify,
                                                      const T360RigMotion* motion, unsigned long long* deviceStats, int numPlanes,
                                                      const uint8_t* const* dIn, uint8_t* const* dOut, const int* inW, const int* inH,
                                                      const int* inPitch, const int* outW, const int* outH, const int* outPitch, void* stream) {
  return transformFrameView("Could not transform the frame with a camera view of a lens rig with a rig motion", t,
                            motionView(rig, photometry, seamWidth, pose, camera, minify, motion, deviceStats),
                            numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, stream);
}
T360_API int T360B200_stereoCameraMaps(const FrameTransformContext* ctx, const T360LensRig* rig, const T360RigPhotometry* photometry, const T360Pose* pose,
                                       const T360Camera* camera, const T360Minify* minify, int lens, int plane, int inW, int inH, int outW, int outH,
                                       float* map0, float* map1, uint8_t* level, uint16_t* weight, uint16_t* gain, uint16_t* eyeWeight) {
  return cameraPhotoMaps("Could not compute the stereo camera maps", ctx,
                         photoView(rig, photometry, 0.0f, pose, camera, minify, nullptr, true),
                         lens, plane, inW, inH, outW, outH, map0, map1, level, weight, gain, eyeWeight);
}
T360_API int T360B200_transformFrameStereoCameraAsync(VideoFrameTransform* t, const T360LensRig* rig, const T360RigPhotometry* photometry,
                                                      const T360Pose* pose, const T360Camera* camera, const T360Minify* minify,
                                                      unsigned long long* deviceStats, int numPlanes, const uint8_t* const* dIn,
                                                      uint8_t* const* dOut, const int* inW, const int* inH, const int* inPitch, const int* outW,
                                                      const int* outH, const int* outPitch, void* stream) {
  return transformFrameView("Could not transform the frame with a camera view of a stereo rig", t,
                            photoView(rig, photometry, 0.0f, pose, camera, minify, deviceStats, true),
                            numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, stream);
}
T360_API void T360B200_setPinHostPlanes(VideoFrameTransform* t, int enable) { if (t) t->setPinHostPlanes(enable != 0); }
T360_API void T360B200_debugTrace(VideoFrameTransform* t, int enable) { if (t) t->enableTrace(enable != 0); }
T360_API unsigned long long T360B200_debugTraceRead(VideoFrameTransform* t, unsigned long long* out, unsigned long long maxWords) {
  return t ? t->readTrace(out, maxWords) : 0;
}
T360_API int T360B200_synchronize(VideoFrameTransform* t) { return t ? t->synchronize() : 0; }
T360_API void* T360B200_stream(VideoFrameTransform* t) { return t ? t->stream() : nullptr; }
T360_API unsigned long long T360B200_kernelLaunchCount(void) { return t360::kernelLaunchCount(); }
T360_API unsigned long long T360B200_planDeviceBytes(VideoFrameTransform* t, int planIndex) { return t ? t->planBytes(planIndex) : 0; }
T360_API int T360B200_planTileCounts(VideoFrameTransform* t, int planIndex, int counts[4]) {
  return t && counts ? t->tileCounts(planIndex, counts) : 0;
}
T360_API int T360B200_deviceCount(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}
T360_API const char* T360B200_version(void) { return "transform360-b200 0.1 (sm_90a)"; }
