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
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <stdexcept>
#include <vector>

#include "host_plan.h"
#include "gather_plan.h"
#include "kernels.cuh"
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
  DeviceBuffer<int2> samples;      // full records: tile-major, lane-ordered, 8 bytes per pixel (general kernels / jobs)
  DeviceBuffer<uint32_t> records;  // compact records of the staged jobs (kernels.cuh): 2.5 - 4 bytes per pixel
  int tilesPerRow = 0;
  // gather jobs: share blocks and tiles whose source windows fit a TMA staging box, and the rest
  DeviceBuffer<GatherJob> gatherJobs;  // every job of the plane, sorted by kind (general, seam, class 1, share, class 0)
  std::vector<GatherJob> hostJobs;     // the same list on the host: merged per frame by gatherFrame()
  std::vector<int> jobNeedRows;        // per host job: the source rows [0, n) it reads (streaming host planes in)
  int numJobs = 0, numStaged[2] = {}, numSeam = 0, numShare = 0, numFallback = 0;
  int totalStaged() const { return numSeam + numShare + numStaged[0] + numStaged[1]; }
  // low-pass: register-resident strip jobs grouped by vertical half-size 1..3, and the rest (large vertical kernels),
  // for one plane size
  struct BlurSet {
    DeviceBuffer<StripJob> stripJobs[t360::kStripMaxHy];
    int numStripJobs[t360::kStripMaxHy] = {};
    DeviceBuffer<BlurJob> tileJobs, directJobs;
    int numTileJobs = 0, numDirectJobs = 0, tileSmem = 0;
    DeviceBuffer<float> taps;
    bool needsClear = false;
    std::vector<StripJob> hostStrips[t360::kStripMaxHy];  // (the whole-frame entry point merges the planes' strip jobs)
    std::vector<float> hostTaps;
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
  size_t deviceBytes() const {
    return samples.bytes() + records.bytes() + gatherJobs.bytes() + blur.stripJobs[0].bytes() + blur.stripJobs[1].bytes() + blur.stripJobs[2].bytes() +
           blur.tileJobs.bytes() + blur.directJobs.bytes() + blur.taps.bytes();
  }
};

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled through the runtime's driver entry point table: the library must still dlopen()
// on a machine without libcuda.so (CPU-only planning, tests), so libcuda is never linked.
EncodeTiledFn tensorMapEncoder() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q{};
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
      cudaGetLastError();
      p = nullptr;
    }
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

// Describes a pitch-linear 8-bit plane to the TMA unit with variant `variant` of the staging box of class `cls` of kernel
// size k (kernels.cuh: boxVariantRows).
bool encodePlaneMap(CUtensorMap* map, const uint8_t* base, int w, int h, int pitch, int k, int cls, int variant) {
  EncodeTiledFn enc = tensorMapEncoder();
  if (!enc) return false;
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (pitch & 15)) return false;
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(w), static_cast<cuuint64_t>(h)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(pitch)};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(t360::stageBoxW(k, cls)), static_cast<cuuint32_t>(t360::boxVariantRows(k, cls, variant))};
  const cuuint32_t elem[2] = {1, 1};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t*>(base), dims, strides, box, elem,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,  // (none / 64 / 256 B: no difference)
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Everything one image plane needs to be in flight independently of the others: the frame entry point runs the
// luma plane on the caller's stream and the two chroma planes on their own lanes.
constexpr int kPlaneLanes = 3;
static_assert(kPlaneLanes == t360::kMaxFramePlanes, "the frame kernel takes one PlaneView per lane");
// The tensor maps of one source plane (every box class and variant): encoding one takes the driver about a
// microsecond, a frame needs 21, and callers come back with the same few planes (a decoder's surface pool, the
// library's own low-pass plane), so every lane remembers the last few.
struct PlaneMaps {
  const uint8_t* base = nullptr;
  int w = 0, h = 0, pitch = 0, k = 0;
  CUtensorMap maps[t360::kNumBoxClasses][t360::kBoxVariants];
};
struct PlaneLane {
  static constexpr int kMapCache = 32;  // (a decoder's surface pool holds 10 - 20 frames)
  PlaneMaps mapCache[kMapCache];
  int mapCacheNext = 0;
  cudaStream_t main = nullptr;                       // chroma lanes only (lane 0 runs on the caller's stream)
  cudaEvent_t done = nullptr;                        // recorded when this lane's plane has been enqueued completely
  DeviceBuffer<uint8_t> blurred;                     // low-pass output of this plane
  DeviceBuffer<uint8_t> scaled;                      // render target at map size when an area resize follows
  DeviceBuffer<int> claimCounter;                    // dynamic tile scheduler of this lane's gather launch
};

// What the gather stage of one image plane needs once its source is ready (see VideoFrameTransform::prepareGather).
struct GatherWork {
  const DevicePlan* plan = nullptr;
  t360::PlaneView view{};
  bool staged = false;                       // TMA-describable: may run in the persistent (per-plane / per-frame) kernel
  CUtensorMap maps[t360::kNumBoxClasses][t360::kBoxVariants];
  uint8_t* finalOut = nullptr;               // where the area resize (if any) delivers
  int finalPitch = 0, finalW = 0, finalH = 0, imagePlane = 0;
  const void* resizeTables = nullptr;
};

// The tiles of all planes of a frame in one list (general, class 1, class 0; luma first inside each kind), rebuilt
// when a map is regenerated.
struct FrameJobList {
  DeviceBuffer<GatherJob> tiles;
  int numTiles = 0, numPlanes = 0;
  unsigned long long generation = ~0ull;
  DeviceBuffer<int> claimCounter;
};

// How the synchronous host-pointer call streams a large plane through the GPU: the input arrives in `chunks` row bands;
// wave c = the gather jobs that only read rows delivered by chunks 0..c; rects[c] = the output rectangles that are
// complete after wave c (copied back while later chunks are still on their way: PCIe carries both directions at once).
struct WavePlan {
  struct Rect { int x, y, w, h; };
  int chunks = 0;
  const void* plan = nullptr;  // the DevicePlan it was made for
  unsigned long long generation = ~0ull;
  std::vector<int> chunkRowEnd, waveStart;
  DeviceBuffer<GatherJob> jobs;  // wave-major
  std::vector<std::vector<Rect>> rects;
};

// Everything asynchronous work on ONE caller stream shares: the lanes (scratch planes, side streams, job schedulers) and
// the scheduler of the whole-frame launch.  Work on the same stream is ordered, so one set per stream is enough; callers
// that enqueue on several streams at once get a set per stream instead of racing for one.
struct StreamSlot {
  PlaneLane lanes[kPlaneLanes];
  DeviceBuffer<int> frameClaim;
  cudaEvent_t fork = nullptr;
};

// The strip jobs of all planes of a frame, by vertical half-size, with one merged tap buffer (rebuilt when a map is).
struct FrameBlurList {
  DeviceBuffer<StripJob> jobs[t360::kStripMaxHy];
  int numJobs[t360::kStripMaxHy] = {};
  DeviceBuffer<float> taps;
  int numPlanes = 0;
  unsigned long long generation = ~0ull;
};

constexpr int kPitchAlign = 256;
inline int alignedPitch(int w) { return (w + kPitchAlign - 1) / kPitchAlign * kPitchAlign; }

}  // namespace

class VideoFrameTransform {
 public:
  explicit VideoFrameTransform(FrameTransformContext* ctx) {
    std::memcpy(&ctx_, ctx, sizeof(ctx_));
    const char* e = std::getenv("T360B200_PIN_HOST_PLANES");
    pinHostPlanes_ = e && *e && *e != '0';
    if (const char* m = std::getenv("T360B200_PIPELINE_MIN_BYTES")) pipelineMinBytes_ = std::atoll(m);  // tests: 0 = always
    if (const char* m = std::getenv("T360B200_PIPELINE_CHUNKS")) pipelineChunks_ = std::atoi(m);       // tuning
    if (const char* m = std::getenv("T360B200_PIPELINE_BLOCKS")) pipelineBlocks_ = std::atoi(m);
    if (const char* m = std::getenv("T360B200_PIPELINE_IN_STREAMS")) pipelineInStreams_ = std::atoi(m);
  }
  void setPinHostPlanes(bool on) { pinHostPlanes_ = on; }

  ~VideoFrameTransform() {
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
      }
      frameJobs_.tiles.release();
      for (auto& b : frameBlur_.jobs) b.release();
      frameBlur_.taps.release();
      trace_.release();
      frameJobs_.claimCounter.release();
      for (cudaEvent_t e : chunkIn_) cudaEventDestroy(e);
      for (cudaEvent_t e : waveDone_) cudaEventDestroy(e);
      for (WavePlan& w : wavePlans_) w.jobs.release();
      for (PlaneGraph& g : planeGraphs_) cudaGraphExecDestroy(g.exec);
      for (cudaEvent_t e : {graphFork_, graphJoinIn_, graphJoinOut_}) if (e) cudaEventDestroy(e);
      if (copyIn_) cudaStreamDestroy(copyIn_);
      if (copyIn2_) cudaStreamDestroy(copyIn2_);
      if (copyOut_) cudaStreamDestroy(copyOut_);
      if (stream_) cudaStreamDestroy(stream_);
    }
  }

  // reference generateMapForPlane (cpp:504-576): plan on the host, upload once.
  bool generateMapForPlane(int inW, int inH, int outW, int outH, int planIndex) {
    try {
      HostPlan host;
      if (!t360::buildHostPlan(ctx_, inW, inH, outW, outH, host)) return false;
      const DeviceRestore restoreDevice = ensureDevice();
      std::lock_guard<std::mutex> lock(mu_);
      plans_[planIndex] = upload(host);
      ++planGeneration_;
      return true;
    } catch (const CudaFail& f) {
      std::printf("Could not generate map for plane %d. Error: CUDA %s (%s) in %s\n", planIndex,
                  cudaGetErrorName(f.err), cudaGetErrorString(f.err), f.what);
    } catch (const std::exception& ex) {
      std::printf("Could not generate map for plane %d. Error: %s\n", planIndex, ex.what());
    }
    return false;
  }

  // reference transformFramePlane (cpp:1319-1351): host or device planes, synchronous.
  bool transformFramePlane(uint8_t* in, uint8_t* out, int inW, int inH, int inPitch, int outW, int outH, int outPitch,
                           int planIndex, int imagePlaneIndex) {
    try {
      if (!in || !out || inW <= 0 || inH <= 0 || outW <= 0 || outH <= 0 || inPitch < inW || outPitch < outW) {
        std::printf("Could not transform the plane %d. Error: invalid plane description\n", imagePlaneIndex);
        return false;
      }
      const DeviceRestore restoreDevice = ensureDevice();
      const DevicePlan* plan = findPlan(planIndex, imagePlaneIndex);
      if (!plan) return false;
      {  // the same plan and caller buffers as in an earlier streamed call: replay its graph (no driver query, no set-up)
        std::lock_guard<std::mutex> hostLock(hostCallMu_);
        if (replayPlaneGraph(*plan, in, out, inW, inH, inPitch, outW, outH, outPitch)) return true;
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
      if (!inOnDevice) {
        pinIfRecurring(in, static_cast<size_t>(inPitch) * (inH - 1) + inW);
        dInPitch = alignedPitch(inW);
        stagingIn_.reserve(static_cast<size_t>(dInPitch) * inH + 64);
        CU(cudaMemcpy2DAsync(stagingIn_.ptr, dInPitch, in, inPitch, inW, inH, cudaMemcpyHostToDevice, stream_));
        dIn = stagingIn_.ptr;
      }
      if (!outOnDevice) {
        pinIfRecurring(out, static_cast<size_t>(outPitch) * (outH - 1) + outW);
        dOutPitch = alignedPitch(outW);
        stagingOut_.reserve(static_cast<size_t>(dOutPitch) * outH + 64);
        dOut = stagingOut_.ptr;
        if (plan->transparent) {
          // barrel layouts leave unmapped pixels untouched: chroma planes start at 128 (reference cpp:743-747),
          // the luma plane keeps whatever the caller's buffer holds
          if (planIndex) CU(cudaMemset2DAsync(dOut, dOutPitch, 128, outW, outH, stream_));
          else CU(cudaMemcpy2DAsync(dOut, dOutPitch, out, outPitch, outW, outH, cudaMemcpyHostToDevice, stream_));
        }
      } else if (plan->transparent && planIndex) {
        CU(cudaMemset2DAsync(dOut, dOutPitch, 128, outW, outH, stream_));
      }
      if (!enqueue(*plan, dIn, dOut, inW, inH, dInPitch, outW, outH, dOutPitch, stream_, imagePlaneIndex, slotFor(stream_).lanes[0])) return false;
      if (!outOnDevice)
        CU(cudaMemcpy2DAsync(out, outPitch, dOut, dOutPitch, outW, outH, cudaMemcpyDeviceToHost, stream_));
      CU(cudaStreamSynchronize(stream_));
      return true;
    } catch (const CudaFail& f) {
      std::printf("Could not transform the plane %d. Error: CUDA %s (%s) in %s\n", imagePlaneIndex,
                  cudaGetErrorName(f.err), cudaGetErrorString(f.err), f.what);
      cudaGetLastError();
    } catch (const std::exception& ex) {
      std::printf("Could not transform the plane %d. Error: %s\n", imagePlaneIndex, ex.what());
    }
    return false;
  }

  // ---- streaming a large host plane through the device -------------------------------------------------------
  bool pipelineEligible(const DevicePlan& plan, int inW, int inH, int outW, int outH) const {
    return plan.totalStaged() > 0 && !plan.transparent && !plan.lowPass && inW == plan.inW && inH == plan.inH &&
           outW == plan.mapW && outH == plan.mapH && static_cast<long long>(inW) * inH >= pipelineMinBytes_ && inH >= 64;
  }

  WavePlan& wavePlanFor(const DevicePlan& plan, int planIndex, int chunks) {
    WavePlan& w = wavePlans_[planIndex ? 1 : 0];
    if (w.plan == &plan && w.chunks == chunks && w.generation == planGeneration_) return w;
    w.chunks = chunks;
    w.plan = &plan;
    w.generation = planGeneration_;
    const int rowsPer = ((plan.inH + chunks - 1) / chunks + 7) & ~7;
    w.chunkRowEnd.assign(chunks, plan.inH);
    for (int c = 0; c < chunks; ++c) w.chunkRowEnd[c] = std::min(plan.inH, (c + 1) * rowsPer);
    auto waveOf = [&](int needRows) {
      int c = 0;
      while (c + 1 < chunks && w.chunkRowEnd[c] < needRows) ++c;
      return c;
    };
    std::vector<std::vector<GatherJob>> byWave(chunks);
    // Which output rectangles are complete after which wave: 32-row bands of the full width by default (contiguous
    // copies: a band split into the three faces of a cube-map row finishes earlier per face, but strided rectangle
    // copies are much slower than whole contiguous bands; T360B200_PIPELINE_BLOCKS > 1 splits anyway).
    int blocks = 1;
    for (int nb : {4, 3, 2})
      if (plan.mapW % (nb * t360::kShareW) == 0 && nb <= pipelineBlocks_) { blocks = nb; break; }
    const int blockW = plan.mapW / blocks, bands = (plan.mapH + 31) / 32;
    std::vector<int> complete(static_cast<size_t>(bands) * blocks, 0);
    for (size_t i = 0; i < plan.hostJobs.size(); ++i) {
      const int c = waveOf(plan.jobNeedRows[i]);
      byWave[c].push_back(plan.hostJobs[i]);
      int rect[4];
      t360::jobOutputRect(plan.hostJobs[i], plan.kernelSize, rect);
      for (int band = rect[1] / 32; band <= (std::min(rect[3], plan.mapH) - 1) / 32; ++band) {
        int& slot = complete[static_cast<size_t>(band) * blocks + rect[0] / blockW];
        slot = std::max(slot, c);
      }
    }
    std::vector<GatherJob> all;
    w.waveStart.assign(chunks + 1, 0);
    for (int c = 0; c < chunks; ++c) {
      t360::spreadGeneralJobs(byWave[c]);
      w.waveStart[c] = static_cast<int>(all.size());
      all.insert(all.end(), byWave[c].begin(), byWave[c].end());
    }
    w.waveStart[chunks] = static_cast<int>(all.size());
    w.jobs.reserve(all.size());
    CU(cudaMemcpy(w.jobs.ptr, all.data(), all.size() * sizeof(GatherJob), cudaMemcpyHostToDevice));
    w.rects.assign(chunks, {});
    for (int b = 0; b < blocks; ++b)
      for (int band = 0; band < bands;) {  // vertically adjacent bands of a block that complete together: one copy
        const int c = complete[static_cast<size_t>(band) * blocks + b];
        int end = band + 1;
        while (end < bands && complete[static_cast<size_t>(end) * blocks + b] == c) ++end;
        w.rects[c].push_back(WavePlan::Rect{b * blockW, band * 32, blockW, std::min(plan.mapH, end * 32) - band * 32});
        band = end;
      }
    return w;
  }

  static bool isPinnedHost(const void* p) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
      cudaGetLastError();
      return false;
    }
    return a.type == cudaMemoryTypeHost;
  }

  bool replayPlaneGraph(const DevicePlan& plan, const uint8_t* in, const uint8_t* out, int inW, int inH, int inPitch, int outW, int outH,
                        int outPitch) {
    for (PlaneGraph& c : planeGraphs_) {
      if (c.plan != &plan || c.in != in || c.out != out || c.inPitch != inPitch || c.outPitch != outPitch || c.generation != planGeneration_ ||
          c.stagingIn != stagingIn_.ptr || c.stagingOut != stagingOut_.ptr || c.inW != inW || c.inH != inH || c.outW != outW || c.outH != outH)
        continue;
      c.lastUse = ++graphClock_;
      CU(cudaGraphLaunch(c.exec, stream_));
      t360::countKernelLaunches(c.kernels);
      CU(cudaStreamSynchronize(stream_));
      return true;
    }
    return false;
  }

  // reference transformFramePlane for large host planes (same result as the plain path): chunked H2D || gather || D2H
  bool transformHostPlanePipelined(const DevicePlan& plan, uint8_t* in, uint8_t* out, int inW, int inH, int inPitch, int outW, int outH,
                                   int outPitch, int planIndex, int imagePlaneIndex) {
    const long long bytes = static_cast<long long>(inW) * inH;
    const int chunks = pipelineChunks_ > 1 ? std::min(pipelineChunks_, 32)
                                           : static_cast<int>(std::min<long long>(8, std::max<long long>(2, bytes / (3ll << 20))));
    WavePlan& w = wavePlanFor(plan, planIndex, chunks);
    if (!copyIn_) {
      CU(cudaStreamCreateWithFlags(&copyIn_, cudaStreamNonBlocking));
      CU(cudaStreamCreateWithFlags(&copyIn2_, cudaStreamNonBlocking));
      CU(cudaStreamCreateWithFlags(&copyOut_, cudaStreamNonBlocking));
      for (cudaEvent_t* e : {&graphFork_, &graphJoinIn_, &graphJoinOut_}) CU(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    }
    while (static_cast<int>(chunkIn_.size()) < chunks) {
      cudaEvent_t a = nullptr, b = nullptr;
      CU(cudaEventCreateWithFlags(&a, cudaEventDisableTiming));
      chunkIn_.push_back(a);
      CU(cudaEventCreateWithFlags(&b, cudaEventDisableTiming));
      waveDone_.push_back(b);
    }
    pinIfRecurring(in, static_cast<size_t>(inPitch) * (inH - 1) + inW);
    pinIfRecurring(out, static_cast<size_t>(outPitch) * (outH - 1) + outW);
    const int dInPitch = alignedPitch(inW), dOutPitch = alignedPitch(outW);
    stagingIn_.reserve(static_cast<size_t>(dInPitch) * inH + 64);
    stagingOut_.reserve(static_cast<size_t>(dOutPitch) * outH + 64);
    PlaneLane& hostLane = slotFor(stream_).lanes[0];
    GatherWork work;
    if (!prepareGather(plan, stagingIn_.ptr, stagingOut_.ptr, inW, inH, dInPitch, outW, outH, dOutPitch, stream_, imagePlaneIndex, hostLane, work))
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
    auto issue = [&](bool forkJoin) {
      if (forkJoin) {  // (capture: the side streams become branches of the graph)
        CU(cudaEventRecord(graphFork_, stream_));
        CU(cudaStreamWaitEvent(copyIn_, graphFork_, 0));
        if (pipelineInStreams_ > 1) CU(cudaStreamWaitEvent(copyIn2_, graphFork_, 0));
        CU(cudaStreamWaitEvent(copyOut_, graphFork_, 0));
      }
      t360::FrameGatherParams fp{};
      fp.plane[0] = work.view;
      fp.weightImage = reinterpret_cast<const uint4*>(weightImages_[plan.kernelSize].ptr);
      fp.kernelSize = plan.kernelSize;
      fp.numPlanes = 1;
      for (int c = 0; c < chunks; ++c) {
        const int r0 = c ? w.chunkRowEnd[c - 1] : 0, r1 = w.chunkRowEnd[c];
        // (with two inbound streams the set-up of band c + 1 hides under the transfer of band c)
        cudaStream_t inStream = (pipelineInStreams_ > 1 && (c & 1)) ? copyIn2_ : copyIn_;
        if (r1 > r0)
          CU(cudaMemcpy2DAsync(stagingIn_.ptr + static_cast<size_t>(r0) * dInPitch, dInPitch, in + static_cast<size_t>(r0) * inPitch, inPitch, inW,
                               r1 - r0, cudaMemcpyHostToDevice, inStream));
        CU(cudaEventRecord(chunkIn_[c], inStream));
        CU(cudaStreamWaitEvent(stream_, chunkIn_[c], 0));
        const int n = w.waveStart[c + 1] - w.waveStart[c];
        if (n > 0) {
          t360::StagedParams jobs{w.jobs.ptr + w.waveStart[c], n, hostLane.claimCounter.ptr, nullptr};
          CU(t360::launchGatherFrame(fp, jobs, work.maps, numSMs_, stream_, /*programmatic=*/false));
        }
        if (!w.rects[c].empty()) {
          CU(cudaEventRecord(waveDone_[c], stream_));
          CU(cudaStreamWaitEvent(copyOut_, waveDone_[c], 0));
          for (const WavePlan::Rect& r : w.rects[c])
            CU(cudaMemcpy2DAsync(out + static_cast<size_t>(r.y) * outPitch + r.x, outPitch,
                                 stagingOut_.ptr + static_cast<size_t>(r.y) * dOutPitch + r.x, dOutPitch, r.w, r.h, cudaMemcpyDeviceToHost, copyOut_));
        }
      }
      if (forkJoin) {
        if (pipelineInStreams_ > 1) {  // (the second inbound stream joins through the first)
          CU(cudaEventRecord(graphJoinIn_, copyIn2_));
          CU(cudaStreamWaitEvent(copyIn_, graphJoinIn_, 0));
        }
        CU(cudaEventRecord(graphJoinIn_, copyIn_));
        CU(cudaEventRecord(graphJoinOut_, copyOut_));
        CU(cudaStreamWaitEvent(stream_, graphJoinIn_, 0));
        CU(cudaStreamWaitEvent(stream_, graphJoinOut_, 0));
      }
    };
    if (std::getenv("T360B200_PIPELINE_TIMING")) {  // tuning aid: the timeline of one streamed call on stdout
      std::vector<cudaEvent_t> ev(3 * chunks + 1);
      for (cudaEvent_t& e : ev) CU(cudaEventCreate(&e));
      CU(cudaStreamSynchronize(stream_));
      CU(cudaEventRecord(ev[3 * chunks], stream_));
      CU(cudaStreamWaitEvent(copyIn_, ev[3 * chunks], 0));
      CU(cudaStreamWaitEvent(copyOut_, ev[3 * chunks], 0));
      t360::FrameGatherParams fp{};
      fp.plane[0] = work.view;
      fp.weightImage = reinterpret_cast<const uint4*>(weightImages_[plan.kernelSize].ptr);
      fp.kernelSize = plan.kernelSize;
      fp.numPlanes = 1;
      for (int c = 0; c < chunks; ++c) {
        const int r0 = c ? w.chunkRowEnd[c - 1] : 0, r1 = w.chunkRowEnd[c];
        CU(cudaMemcpy2DAsync(stagingIn_.ptr + static_cast<size_t>(r0) * dInPitch, dInPitch, in + static_cast<size_t>(r0) * inPitch, inPitch, inW,
                             r1 - r0, cudaMemcpyHostToDevice, copyIn_));
        CU(cudaEventRecord(ev[3 * c], copyIn_));
        CU(cudaStreamWaitEvent(stream_, ev[3 * c], 0));
        const int n = w.waveStart[c + 1] - w.waveStart[c];
        if (n > 0) {
          t360::StagedParams jobs{w.jobs.ptr + w.waveStart[c], n, hostLane.claimCounter.ptr, nullptr};
          CU(t360::launchGatherFrame(fp, jobs, work.maps, numSMs_, stream_, false));
        }
        CU(cudaEventRecord(ev[3 * c + 1], stream_));
        CU(cudaStreamWaitEvent(copyOut_, ev[3 * c + 1], 0));
        for (const WavePlan::Rect& r : w.rects[c])
          CU(cudaMemcpy2DAsync(out + static_cast<size_t>(r.y) * outPitch + r.x, outPitch, stagingOut_.ptr + static_cast<size_t>(r.y) * dOutPitch + r.x,
                               dOutPitch, r.w, r.h, cudaMemcpyDeviceToHost, copyOut_));
        CU(cudaEventRecord(ev[3 * c + 2], copyOut_));
      }
      CU(cudaStreamSynchronize(stream_));
      CU(cudaStreamSynchronize(copyOut_));
      std::printf("streamed plane %d (%dx%d -> %dx%d, %d chunks): chunk | H2D done | wave done (jobs) | D2H done (rects, bytes) [us]\n", imagePlaneIndex, inW,
                  inH, outW, outH, chunks);
      for (int c = 0; c < chunks; ++c) {
        float a = 0, b = 0, d = 0;
        cudaEventElapsedTime(&a, ev[3 * chunks], ev[3 * c]);
        cudaEventElapsedTime(&b, ev[3 * chunks], ev[3 * c + 1]);
        cudaEventElapsedTime(&d, ev[3 * chunks], ev[3 * c + 2]);
        long long bytes = 0;
        for (const WavePlan::Rect& r : w.rects[c]) bytes += static_cast<long long>(r.w) * r.h;
        std::printf("  %2d | %7.1f | %7.1f (%5d) | %7.1f (%2zu, %lld)\n", c, a * 1e3, b * 1e3, w.waveStart[c + 1] - w.waveStart[c], d * 1e3,
                    w.rects[c].size(), bytes);
      }
      for (cudaEvent_t e : ev) cudaEventDestroy(e);
      return true;
    }
    if (isPinnedHost(in) && isPinnedHost(out)) {
      PlaneGraph* g = nullptr;
      for (size_t i = 0; i < planeGraphs_.size();) {
        PlaneGraph& c = planeGraphs_[i];
        if (c.stagingIn != stagingIn_.ptr || c.stagingOut != stagingOut_.ptr || c.generation != planGeneration_) {
          cudaGraphExecDestroy(c.exec);
          planeGraphs_.erase(planeGraphs_.begin() + static_cast<long>(i));
          continue;
        }
        if (c.plan == &plan && c.in == in && c.out == out && c.inPitch == inPitch && c.outPitch == outPitch) g = &c;
        ++i;
      }
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
        for (int c = 0; c < chunks; ++c) kernels += w.waveStart[c + 1] > w.waveStart[c];
        planeGraphs_.push_back(PlaneGraph{&plan, planGeneration_, in, out, inPitch, outPitch, stagingIn_.ptr, stagingOut_.ptr, inW, inH, outW, outH,
                                          kernels, exec, 0});
        g = &planeGraphs_.back();
        t360::countKernelLaunches(-kernels);  // (counted once while capturing; every replay counts below)
      }
      g->lastUse = ++graphClock_;
      CU(cudaGraphLaunch(g->exec, stream_));
      t360::countKernelLaunches(g->kernels);
      CU(cudaStreamSynchronize(stream_));
      return true;
    }
    issue(false);
    CU(cudaStreamSynchronize(stream_));
    CU(cudaStreamSynchronize(copyOut_));
    if (pipelineInStreams_ > 1) CU(cudaStreamSynchronize(copyIn2_));
    return true;
  }

  // device to device, asynchronous
  bool transformDevice(const uint8_t* dIn, uint8_t* dOut, int inW, int inH, int inPitch, int outW, int outH,
                       int outPitch, int planIndex, cudaStream_t stream) {
    try {
      const DeviceRestore restoreDevice = ensureDevice();
      const DevicePlan* plan = findPlan(planIndex, planIndex);
      if (!plan) return false;
      cudaStream_t s = stream ? stream : stream_;
      if (plan->transparent && planIndex) CU(cudaMemset2DAsync(dOut, outPitch, 128, outW, outH, s));
      return enqueue(*plan, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, s, planIndex, slotFor(s).lanes[0]);
    } catch (const CudaFail& f) {
      std::printf("Could not transform the plane %d. Error: CUDA %s (%s) in %s\n", planIndex, cudaGetErrorName(f.err),
                  cudaGetErrorString(f.err), f.what);
      cudaGetLastError();
    } catch (const std::exception& ex) {
      std::printf("Could not transform the plane %d. Error: %s\n", planIndex, ex.what());
    }
    return false;
  }

  // Whole frame, device to device, asynchronous: plane 0 with plan 0 on the caller's stream, planes 1.. with plan 1
  // on their own lanes (the planes are independent: reference vf_transform360.c:368-397 loops over them).
  bool transformFrameDevice(int numPlanes, const uint8_t* const* dIn, uint8_t* const* dOut, const int* inW, const int* inH,
                            const int* inPitch, const int* outW, const int* outH, const int* outPitch, cudaStream_t stream) {
    try {
      if (numPlanes < 1 || numPlanes > kPlaneLanes) {
        std::printf("Could not transform the frame. Error: %d planes (1..%d supported)\n", numPlanes, kPlaneLanes);
        return false;
      }
      const DeviceRestore restoreDevice = ensureDevice();
      cudaStream_t s = stream ? stream : stream_;
      StreamSlot& slot = slotFor(s);
      PlaneLane* lanes_ = slot.lanes;
      cudaEvent_t frameFork_ = slot.fork;
      const DevicePlan* plans[kPlaneLanes];
      bool sideWork = false;  // does any chroma plane have work before its gather (low-pass, pre-fill)?
      bool anyTransparent = false;
      for (int p = 0; p < numPlanes; ++p) {
        if (!(plans[p] = findPlan(p ? 1 : 0, p))) return false;
        if (p) sideWork = sideWork || plans[p]->lowPass || plans[p]->transparent;
        anyTransparent = anyTransparent || plans[p]->transparent;
      }
      // Low-pass of all planes in one launch per vertical kernel size when every plane takes the strip kernel only
      const bool mergedBlur = !anyTransparent && blurFrame(plans, numPlanes, dIn, inW, inH, inPitch, lanes_, s);
      if (mergedBlur) sideWork = false;
      // Stage 1, planes side by side (chroma on its own lanes): everything before the gather.
      const bool fork = numPlanes > 1 && sideWork;
      if (fork) CU(cudaEventRecord(frameFork_, s));
      GatherWork work[kPlaneLanes];
      bool allStaged = true;
      for (int p = numPlanes - 1; p >= 0; --p) {
        cudaStream_t ps = (p && fork) ? lanes_[p].main : s;
        if (p && fork) CU(cudaStreamWaitEvent(ps, frameFork_, 0));
        if (plans[p]->transparent && p) CU(cudaMemset2DAsync(dOut[p], outPitch[p], 128, outW[p], outH[p], ps));
        if (!prepareGather(*plans[p], dIn[p], dOut[p], inW[p], inH[p], inPitch[p], outW[p], outH[p], outPitch[p], ps, p, lanes_[p], work[p], mergedBlur))
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
        for (int p = 0; p < numPlanes; ++p) finishGather(work[p], s);
        return true;
      }
      // some plane needs the general kernel (barrel layouts, nearest, unaligned planes): per-plane launches
      if (numPlanes > 1 && !fork) CU(cudaEventRecord(frameFork_, s));
      for (int p = numPlanes - 1; p >= 0; --p) {
        cudaStream_t ps = p ? lanes_[p].main : s;
        if (p && !fork) CU(cudaStreamWaitEvent(ps, frameFork_, 0));
        if (work[p].plan->kernelSize) {
          gatherPlane(work[p], lanes_[p], ps);
          finishGather(work[p], ps);
        }
        if (p) CU(cudaEventRecord(lanes_[p].done, ps));
      }
      for (int p = 1; p < numPlanes; ++p) CU(cudaStreamWaitEvent(s, lanes_[p].done, 0));
      return true;
    } catch (const CudaFail& f) {
      std::printf("Could not transform the frame. Error: CUDA %s (%s) in %s\n", cudaGetErrorName(f.err), cudaGetErrorString(f.err), f.what);
      cudaGetLastError();
    } catch (const std::exception& ex) {
      std::printf("Could not transform the frame. Error: %s\n", ex.what());
    }
    return false;
  }

  bool lowPassDevice(const uint8_t* dIn, uint8_t* dOut, int w, int h, int inPitch, int outPitch, int planIndex,
                     cudaStream_t stream) {
    try {
      const DeviceRestore restoreDevice = ensureDevice();
      const DevicePlan* plan = findPlan(planIndex, planIndex);
      if (!plan) return false;
      if (!plan->lowPass) {
        std::printf("Could not filter plane %d. Error: plan has no low-pass stage\n", planIndex);
        return false;
      }
      runLowPass(*plan, dIn, dOut, w, h, inPitch, outPitch, stream ? stream : stream_);
      return true;
    } catch (const CudaFail& f) {
      std::printf("Could not filter plane %d. Error: CUDA %s (%s) in %s\n", planIndex, cudaGetErrorName(f.err),
                  cudaGetErrorString(f.err), f.what);
      cudaGetLastError();
    }
    return false;
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
    counts[0] = it->second.totalStaged(); counts[1] = it->second.numFallback;
    counts[2] = it->second.blur.numStripJobs[0] + it->second.blur.numStripJobs[1] + it->second.blur.numStripJobs[2];
    counts[3] = it->second.blur.numTileJobs + it->second.blur.numDirectJobs;
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
    deviceReady_ = true;
    return guard;
  }

  // Pageable host planes are copied through the driver's bounce buffers at a fraction of PCIe speed.  When enabled
  // (T360B200_setPinHostPlanes or T360B200_PIN_HOST_PLANES=1), a plane address seen for the second time is page-locked
  // in place with cudaHostRegister so that later frames in the same buffer are DMA'd directly.  Opt-in because the
  // caller must not free such a buffer while the transform is alive (it is unregistered in the destructor).
  void pinIfRecurring(const void* ptr, size_t bytes) {
    if (!pinHostPlanes_ || !ptr || !bytes) return;
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) { cudaGetLastError(); return; }
    if (a.type != cudaMemoryTypeUnregistered) return;
    const uintptr_t page = 4096, lo = reinterpret_cast<uintptr_t>(ptr) & ~(page - 1);
    const size_t len = ((reinterpret_cast<uintptr_t>(ptr) + bytes + page - 1) & ~(page - 1)) - lo;
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

  static bool isDevicePointer(const void* p) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
      cudaGetLastError();
      return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
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

  DevicePlan upload(const HostPlan& h) {
    DevicePlan d;
    d.inW = h.inW; d.inH = h.inH; d.outW = h.outW; d.outH = h.outH; d.mapW = h.mapW; d.mapH = h.mapH;
    d.kernelSize = h.kernelSize;
    d.transparent = h.transparentBorder;
    if (d.kernelSize > 0) {
      deviceWeights(ctx_.interpolation_alg);
      t360::GatherPlan g;
      t360::buildGatherPlan(h, d.kernelSize >= 2 && !d.transparent, g);
      d.tilesPerRow = g.tilesPerRow;
      d.samples.reserve(g.records.size());
      CU(cudaMemcpy(d.samples.ptr, g.records.data(), g.records.size() * sizeof(int2), cudaMemcpyHostToDevice));
      d.numFallback = g.numGeneral;
      d.numSeam = g.numSeam;
      d.numShare = g.numShare;
      for (int c = 0; c < 2; ++c) d.numStaged[c] = g.numStaged[c];
      d.numJobs = static_cast<int>(g.jobs.size());
      if (!g.jobs.empty()) {
        std::vector<GatherJob> launchOrder = g.jobs;  // (hostJobs stay sorted by kind: gatherFrame() merges the planes)
        t360::spreadGeneralJobs(launchOrder);
        d.gatherJobs.reserve(launchOrder.size());
        CU(cudaMemcpy(d.gatherJobs.ptr, launchOrder.data(), launchOrder.size() * sizeof(GatherJob), cudaMemcpyHostToDevice));
      }
      if (!g.compact.empty()) {
        d.records.reserve(g.compact.size());
        CU(cudaMemcpy(d.records.ptr, g.compact.data(), g.compact.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
      }
      d.hostJobs = std::move(g.jobs);
      d.jobNeedRows = std::move(g.jobNeedRows);
    }
    d.lowPass = ctx_.enable_low_pass_filter != 0;
    if (d.lowPass) {
      d.segments = h.segments;
      d.planTaps = h.taps;
      buildBlurJobs(d.segments, d.planTaps, h.inW, h.inH, d.blur);
    }
    d.resizeNeeded = h.resize.needed;
    if (d.resizeNeeded) resizeFor(d, d.outW, d.outH);
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

  // Tiles of the plan, applied once (mono) or to both halves of a stereo frame (reference cpp:630-691), cut
  // into CTA-sized jobs.  Segments that do not fit the plane are dropped, like the reference's caught cv::Exception.
  void buildBlurJobs(const std::vector<t360::LowPassSegment>& segments, const std::vector<float>& planTaps, int planeW, int planeH,
                     DevicePlan::BlurSet& d) {
    struct { const std::vector<t360::LowPassSegment>& segments; const std::vector<float>& taps; int inW, inH; } h{segments, planTaps, planeW, planeH};
    std::vector<BlurJob> tiles, direct;
    std::vector<StripJob> strips[t360::kStripMaxHy];
    std::vector<float> taps = h.taps;  // original taps first (offsets of the plan stay valid), padded copies appended
    int offX[2] = {0, 0}, offY[2] = {0, 0}, passes = 1;
    if (ctx_.input_stereo_format == STEREO_FORMAT_LR) { passes = 2; offX[1] = static_cast<int>(0.5 * h.inW); }
    else if (ctx_.input_stereo_format == STEREO_FORMAT_TB) { passes = 2; offY[1] = static_cast<int>(0.5 * h.inH); }
    std::vector<uint8_t> covered(static_cast<size_t>(h.inW) * h.inH, 0);
    int tileSmem = 0;
    // a warp-job covers 256 columns x `rows` rows; keep the grid at several thousand warps even for small planes
    const long long stripsPerRow = (h.inW + t360::kStripW - 1) / t360::kStripW;
    // (each job recomputes 2*hy rows of horizontal sums at its top and bottom, so never fewer than 8 rows)
    const long long wanted = static_cast<long long>(h.inH) * stripsPerRow / 5000;
    const int rowsBudget = wanted >= 32 ? 32 : (wanted >= 16 ? 16 : 8);

    auto sameTaps = [&](int offA, int nA, int offB, int nB) {
      return nA == nB && (offA == offB || std::memcmp(&h.taps[offA], &h.taps[offB], sizeof(float) * nA) == 0);
    };
    // horizontal taps zero-padded to whole chunks of 4 at a 16-byte aligned offset (fma(0, p, s) == s exactly)
    std::map<std::pair<int, int>, std::pair<int, int>> paddedKx;
    auto padKx = [&](int off, int n) {
      auto it = paddedKx.find({off, n});
      if (it != paddedKx.end()) return it->second;
      while (taps.size() % 4) taps.push_back(0.f);
      const int at = static_cast<int>(taps.size()), chunks = (n + 3) / 4;
      for (int i = 0; i < chunks * 4; ++i) taps.push_back(i < n ? h.taps[off + i] : 0.f);
      return paddedKx[{off, n}] = std::make_pair(at, chunks);
    };
    std::map<int, int> paddedKy1;  // a single vertical tap k becomes {0, k, 0}
    auto padKy = [&](int off, int n) {
      if (n != 1) return off;
      auto it = paddedKy1.find(off);
      if (it != paddedKy1.end()) return it->second;
      const int at = static_cast<int>(taps.size());
      taps.push_back(0.f); taps.push_back(h.taps[off]); taps.push_back(0.f);
      return paddedKy1[off] = at;
    };

    for (int pass = 0; pass < passes; ++pass) {
      // segments of one band that are horizontally adjacent and carry bit-identical kernels (always the case when
      // the view-dependent scale is 1, e.g. no off-centre projection) are merged into one wide segment
      // a segment that does not fit the plane is dropped, like the reference's caught cv::Exception (cpp:183-203) -- each
      // one on its own, before any merging
      auto fits = [&](const t360::LowPassSegment& g) {
        const int l = g.left + offX[pass], t = g.top + offY[pass];
        return l >= 0 && t >= 0 && g.width > 0 && g.height > 0 && l + g.width <= h.inW && t + g.height <= h.inH;
      };
      size_t i = 0;
      while (i < h.segments.size()) {
        t360::LowPassSegment s = h.segments[i];
        size_t j = i + 1;
        if (!fits(s)) { i = j; continue; }
        while (j < h.segments.size()) {
          const t360::LowPassSegment& n = h.segments[j];
          if (n.top != s.top || n.height != s.height || n.left != s.left + s.width || !fits(n) ||
              !sameTaps(n.kxOffset, n.kxCount, s.kxOffset, s.kxCount) || !sameTaps(n.kyOffset, n.kyCount, s.kyOffset, s.kyCount))
            break;
          s.width += n.width;
          ++j;
        }
        i = j;
        const int left = s.left + offX[pass], top = s.top + offY[pass];
        for (int y = 0; y < s.height; ++y) std::memset(&covered[static_cast<size_t>(top + y) * h.inW + left], 1, s.width);
        const int hy = s.kyCount / 2;
        if (hy <= t360::kStripMaxHy && (s.kyCount & 1) && (s.kxCount & 1)) {
          const auto kx = padKx(s.kxOffset, s.kxCount);
          const int kyOff = padKy(s.kyOffset, s.kyCount), hx = s.kxCount / 2;
          const int rows = std::min(rowsBudget, kx.second <= 3 ? 32 : (kx.second <= 8 ? 16 : 8));
          for (int ty = 0; ty < s.height; ty += rows)
            for (int tx = 0; tx < s.width; tx += t360::kStripW) {
              StripJob j{left + tx, top + ty, std::min(t360::kStripW, s.width - tx), std::min(rows, s.height - ty),
                         kx.first, kx.second, s.kxCount, kyOff, 0};
              // interior strips read whole aligned words: first byte - 3 and the last prefetched group must stay in the row
              const int firstByte = j.x0 - hx, lastByte = j.x0 + t360::kStripW - t360::kStripLanePx - hx + 4 * (kx.second + 3) + 7;
              j.edge = (firstByte - 4 < 0 || lastByte >= h.inW) ? 1 : 0;
              strips[std::max(hy, 1) - 1].push_back(j);
            }
        } else {
          for (int ty = 0; ty < s.height; ty += t360::kBlurTileH)
            for (int tx = 0; tx < s.width; tx += t360::kBlurTileW) {
              BlurJob j{left + tx, top + ty, std::min(t360::kBlurTileW, s.width - tx), std::min(t360::kBlurTileH, s.height - ty),
                        s.kxOffset, s.kxCount, s.kyOffset, s.kyCount};
              const long long need = static_cast<long long>(t360::blurTileSmem(j.w, j.h, j.kxCount, j.kyCount));
              if (need <= t360::kBlurMaxSmem) {
                tiles.push_back(j);
                tileSmem = std::max(tileSmem, static_cast<int>(need));
              } else {
                direct.push_back(j);
              }
            }
        }
      }
    }
    d.needsClear = std::find(covered.begin(), covered.end(), 0) != covered.end();
    for (int c = 0; c < t360::kStripMaxHy; ++c) {
      // heaviest jobs first: the hardware block scheduler then balances the tail
      std::stable_sort(strips[c].begin(), strips[c].end(), [](const StripJob& a, const StripJob& b) {
        return static_cast<long long>(a.kxChunks + 2) * a.h * (1 + 3 * a.edge) > static_cast<long long>(b.kxChunks + 2) * b.h * (1 + 3 * b.edge);
      });
      d.numStripJobs[c] = static_cast<int>(strips[c].size());
      d.hostStrips[c] = strips[c];
      if (strips[c].empty()) continue;
      d.stripJobs[c].reserve(strips[c].size());
      CU(cudaMemcpy(d.stripJobs[c].ptr, strips[c].data(), strips[c].size() * sizeof(StripJob), cudaMemcpyHostToDevice));
    }
    d.numTileJobs = static_cast<int>(tiles.size());
    d.numDirectJobs = static_cast<int>(direct.size());
    d.tileSmem = tileSmem;
    if (!tiles.empty()) {
      d.tileJobs.reserve(tiles.size());
      CU(cudaMemcpy(d.tileJobs.ptr, tiles.data(), tiles.size() * sizeof(BlurJob), cudaMemcpyHostToDevice));
    }
    if (!direct.empty()) {
      d.directJobs.reserve(direct.size());
      CU(cudaMemcpy(d.directJobs.ptr, direct.data(), direct.size() * sizeof(BlurJob), cudaMemcpyHostToDevice));
    }
    d.hostTaps = taps;
    if (!taps.empty()) {
      d.taps.reserve(taps.size());
      CU(cudaMemcpy(d.taps.ptr, taps.data(), taps.size() * sizeof(float), cudaMemcpyHostToDevice));
    }
  }

  // the low-pass jobs of a plan for planes of w x h (the planned size, or whatever the caller passes)
  const DevicePlan::BlurSet& blurFor(const DevicePlan& plan, int w, int h) {
    if (w == plan.inW && h == plan.inH) return plan.blur;
    std::lock_guard<std::mutex> lock(lazyMu_);
    auto it = plan.otherBlurs.find({w, h});
    if (it != plan.otherBlurs.end()) return it->second;
    DevicePlan::BlurSet& set = plan.otherBlurs[{w, h}];
    buildBlurJobs(plan.segments, plan.planTaps, w, h, set);
    return set;
  }

  void runLowPass(const DevicePlan& plan, const uint8_t* dIn, uint8_t* dOut, int w, int h, int inPitch, int outPitch,
                  cudaStream_t s) {
    const DevicePlan::BlurSet& b = blurFor(plan, w, h);
    if (b.needsClear) CU(cudaMemset2DAsync(dOut, outPitch, 0, w, h, s));  // reference cpp:625: Mat::zeros under dropped segments
    for (int c = 0; c < t360::kStripMaxHy; ++c) {
      if (!b.numStripJobs[c]) continue;
      t360::StripParams sp{dIn, dOut, w, h, inPitch, outPitch, b.stripJobs[c].ptr, b.numStripJobs[c], b.taps.ptr};
      CU(t360::launchBlurStrips(sp, c + 1, s));
    }
    t360::BlurParams bp{dIn, dOut, w, h, inPitch, outPitch, b.tileJobs.ptr, b.numTileJobs, b.taps.ptr, b.tileSmem};
    if (b.numTileJobs) CU(t360::launchBlur(bp, s));
    if (b.numDirectJobs) {
      bp.jobs = b.directJobs.ptr;
      bp.numJobs = b.numDirectJobs;
      CU(t360::launchBlurDirect(bp, s));
    }
  }

  // the tensor maps of a source plane, from the lane's cache or freshly encoded (false: not TMA-describable)
  static bool planeMaps(PlaneLane& lane, const uint8_t* src, int w, int h, int pitch, int k,
                        CUtensorMap (&out)[t360::kNumBoxClasses][t360::kBoxVariants]) {
    for (const PlaneMaps& e : lane.mapCache)
      if (e.base == src && e.w == w && e.h == h && e.pitch == pitch && e.k == k) {
        std::memcpy(out, e.maps, sizeof(e.maps));
        return true;
      }
    PlaneMaps fresh;
    for (int c = 0; c < t360::kNumBoxClasses; ++c)
      for (int v = 0; v < t360::kBoxVariants; ++v) {
        if (v > 0 && t360::boxVariantRows(k, c, v) == t360::boxVariantRows(k, c, 0)) {
          fresh.maps[c][v] = fresh.maps[c][0];  // (class 1 has one height)
          continue;
        }
        if (!encodePlaneMap(&fresh.maps[c][v], src, w, h, pitch, k, c, v)) return false;
      }
    fresh.base = src; fresh.w = w; fresh.h = h; fresh.pitch = pitch; fresh.k = k;
    lane.mapCache[lane.mapCacheNext] = fresh;
    lane.mapCacheNext = (lane.mapCacheNext + 1) % PlaneLane::kMapCache;
    std::memcpy(out, fresh.maps, sizeof(fresh.maps));
    return true;
  }

  // reference transformPlane (cpp:707-794): [low-pass] -> gather [-> area resize].  Device pointers, asynchronous.
  bool enqueue(const DevicePlan& plan, const uint8_t* dIn, uint8_t* dOut, int inW, int inH, int inPitch, int outW,
               int outH, int outPitch, cudaStream_t s, int imagePlaneIndex, PlaneLane& lane) {
    GatherWork w;
    if (!prepareGather(plan, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, s, imagePlaneIndex, lane, w)) return false;
    if (plan.kernelSize == 0) return true;
    gatherPlane(w, lane, s);
    finishGather(w, s);
    return true;
  }

  // Everything before the gather of one plane: argument checks, the render target, the low-pass stage.
  bool prepareGather(const DevicePlan& plan, const uint8_t* dIn, uint8_t* dOut, int inW, int inH, int inPitch, int outW,
                     int outH, int outPitch, cudaStream_t s, int imagePlaneIndex, PlaneLane& lane, GatherWork& w, bool blurDone = false) {
    w.plan = &plan;
    w.imagePlane = imagePlaneIndex;
    if (plan.kernelSize == 0) {
      std::printf("Could not find interpolation algorithm for plane %d", imagePlaneIndex);  // reference cpp:780-784
      return true;
    }
    // reference cpp:735-737, 755-777: whenever the requested output size is not the map's (scale factors, or a caller
    // that asks for another size than it planned), render at the map's size into a plane pre-filled with 0 (plan index
    // 0) / 128 (others), then cv::resize(INTER_AREA) to the requested size
    w.finalOut = dOut;
    w.finalPitch = outPitch;
    w.finalW = outW;
    w.finalH = outH;
    w.resizeTables = nullptr;
    if (outW != plan.mapW || outH != plan.mapH) {
      w.resizeTables = &resizeFor(plan, outW, outH);
      const int sp = alignedPitch(plan.mapW);
      lane.scaled.reserve(static_cast<size_t>(sp) * plan.mapH + 64);
      if (plan.transparent) CU(cudaMemset2DAsync(lane.scaled.ptr, sp, planIndexOf(plan) ? 128 : 0, plan.mapW, plan.mapH, s));
      dOut = lane.scaled.ptr;
      outPitch = sp;
      outW = plan.mapW;
      outH = plan.mapH;
    }
    const uint8_t* src = dIn;
    int srcPitch = inPitch;
    if (plan.lowPass) {
      const int bp = alignedPitch(inW);
      lane.blurred.reserve(static_cast<size_t>(bp) * inH + 64);
      if (!blurDone) runLowPass(plan, dIn, lane.blurred.ptr, inW, inH, inPitch, bp, s);
      src = lane.blurred.ptr;
      srcPitch = bp;
    }
    w.view = t360::PlaneView{src, dOut, plan.samples.ptr, reinterpret_cast<const uint4*>(plan.records.ptr), inW, inH, srcPitch,
                             outW, outH, outPitch, plan.tilesPerRow, 0};
    // staged tiles need the plane the plan was made for (their windows were proven in-bounds for it) and a
    // TMA-describable layout (16-byte aligned base and pitch); otherwise every tile takes the general kernel
    w.staged = plan.totalStaged() > 0 && !plan.transparent && inW == plan.inW && inH == plan.inH;
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
      t360::GatherParams gp{v.src, v.srcW, v.srcH, v.srcPitch, v.dst, v.dstW, v.dstH, v.dstPitch, v.samples, v.tilesPerRow,
                            weights_[plan.kernelSize].ptr, plan.kernelSize, plan.transparent ? 1 : 0};
      CU(t360::launchGather(gp, numSMs_, s));
    }
  }

  // The low-pass of all planes of a frame: one launch per vertical kernel half-size.  false: not applicable (a plane
  // without low-pass, of another size than planned, or with segments the strip kernel cannot take) -- per-plane launches.
  bool blurFrame(const DevicePlan* const* plans, int numPlanes, const uint8_t* const* dIn, const int* inW, const int* inH, const int* inPitch,
                 PlaneLane* lanes, cudaStream_t s) {
    if (numPlanes < 2) return false;
    for (int p = 0; p < numPlanes; ++p) {
      const DevicePlan& plan = *plans[p];
      if (!plan.lowPass || inW[p] != plan.inW || inH[p] != plan.inH || plan.blur.numTileJobs || plan.blur.numDirectJobs || plan.blur.needsClear)
        return false;
    }
    FrameBlurList& f = frameBlur_;
    {
      std::lock_guard<std::mutex> lock(frameJobsMu_);
      if (f.generation != planGeneration_ || f.numPlanes != numPlanes) {
        std::vector<StripJob> merged[t360::kStripMaxHy];
        std::vector<float> taps;
        for (int p = 0; p < numPlanes; ++p) {
          const DevicePlan::BlurSet& b = plans[p]->blur;
          while (taps.size() % 4) taps.push_back(0.f);  // (the padded horizontal taps stay 16-byte aligned)
          const int base = static_cast<int>(taps.size());
          taps.insert(taps.end(), b.hostTaps.begin(), b.hostTaps.end());
          for (int c = 0; c < t360::kStripMaxHy; ++c)
            for (StripJob j : b.hostStrips[c]) {
              j.kxOffset += base;
              j.kyOffset += base;
              j.edge |= p << t360::kStripPlaneShift;
              merged[c].push_back(j);
            }
        }
        CU(cudaDeviceSynchronize());  // a previous frame may still be reading the old lists
        for (int c = 0; c < t360::kStripMaxHy; ++c) {
          // heaviest jobs first: the hardware block scheduler then balances the tail
          std::stable_sort(merged[c].begin(), merged[c].end(), [](const StripJob& a, const StripJob& b) {
            return static_cast<long long>(a.kxChunks + 2) * a.h * (1 + 3 * (a.edge & 1)) > static_cast<long long>(b.kxChunks + 2) * b.h * (1 + 3 * (b.edge & 1));
          });
          f.numJobs[c] = static_cast<int>(merged[c].size());
          if (merged[c].empty()) continue;
          f.jobs[c].reserve(merged[c].size());
          CU(cudaMemcpy(f.jobs[c].ptr, merged[c].data(), merged[c].size() * sizeof(StripJob), cudaMemcpyHostToDevice));
        }
        f.taps.reserve(std::max<size_t>(taps.size(), 4));
        CU(cudaMemcpy(f.taps.ptr, taps.data(), taps.size() * sizeof(float), cudaMemcpyHostToDevice));
        f.numPlanes = numPlanes;
        f.generation = planGeneration_;
      }
    }
    t360::FrameStripParams fp{};
    for (int p = 0; p < numPlanes; ++p) {
      const int bp = alignedPitch(inW[p]);
      lanes[p].blurred.reserve(static_cast<size_t>(bp) * inH[p] + 64);
      fp.plane[p] = {dIn[p], lanes[p].blurred.ptr, inW[p], inH[p], inPitch[p], bp};
    }
    fp.taps = f.taps.ptr;
    for (int c = 0; c < t360::kStripMaxHy; ++c) {
      if (!f.numJobs[c]) continue;
      fp.jobs = f.jobs[c].ptr;
      fp.numJobs = f.numJobs[c];
      CU(t360::launchBlurFrameStrips(fp, c + 1, s));
    }
    return true;
  }

  // The gathers of all planes of a frame as ONE launch (every plane staged).
  void gatherFrame(const GatherWork* work, int numPlanes, cudaStream_t s, StreamSlot& slot) {
    FrameJobList& f = frameJobs_;
    std::unique_lock<std::mutex> listLock(frameJobsMu_);
    if (f.generation != planGeneration_ || f.numPlanes != numPlanes) {
      std::vector<GatherJob> merged;
      const int order[7] = {t360::kJobGeneral, t360::kJobSeam, t360::kJobClass1, t360::kJobShareStay, t360::kJobShare, t360::kJobClass0, t360::kJobClass0};
      for (int step = 0; step < 7; ++step)  // (quadrant jobs last, like in the per-plane lists)
        for (int p = 0; p < numPlanes; ++p)
          for (GatherJob t : work[p].plan->hostJobs) {
            const int kind = order[step];
            if (((t.outY >> t360::kJobKindShift) & t360::kJobKindMask) != kind) continue;
            if (kind == t360::kJobClass0 && ((t.outX & t360::kJobQuadMask) != 0) != (step == 6)) continue;
            t.outY |= p << t360::kJobPlaneShift;
            merged.push_back(t);
          }
      t360::spreadGeneralJobs(merged);
      CU(cudaDeviceSynchronize());  // a previous frame (on any stream) may still be reading the old list
      f.tiles.reserve(merged.size());
      CU(cudaMemcpy(f.tiles.ptr, merged.data(), merged.size() * sizeof(GatherJob), cudaMemcpyHostToDevice));
      f.numTiles = static_cast<int>(merged.size());
      f.numPlanes = numPlanes;
      f.generation = planGeneration_;
    }
    listLock.unlock();
    armScheduler(slot.frameClaim, s);
    t360::FrameGatherParams fp{};
    CUtensorMap maps[kPlaneLanes][t360::kNumBoxClasses][t360::kBoxVariants];
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
    t360::StagedParams jobs{f.tiles.ptr, f.numTiles, slot.frameClaim.ptr, traceEnabled_ ? trace_.ptr : nullptr};
    CU(t360::launchGatherFrame(fp, jobs, maps, numSMs_, s));
  }

  // What follows the gather: the INTER_AREA down-scale when the map was rendered at a scaled size.
  void finishGather(const GatherWork& w, cudaStream_t s) {
    const DevicePlan& plan = *w.plan;
    if (!w.resizeTables) return;
    const DevicePlan::Resize& r = *static_cast<const DevicePlan::Resize*>(w.resizeTables);
    t360::AreaParams ap{w.view.dst, w.finalOut, plan.mapW, plan.mapH, w.view.dstPitch, w.finalW, w.finalH, w.finalPitch,
                        r.cellW, r.cellH, r.xTaps.ptr, r.xFirst.ptr, r.yTaps.ptr, r.yFirst.ptr, r.xLinear.ptr, r.yLinear.ptr, r.xMax};
    CU(t360::launchAreaResize(ap, s));
  }

  int planIndexOf(const DevicePlan& plan) {  // the transformMatPlaneIndex a plan was generated for
    std::lock_guard<std::mutex> lock(mu_);
    for (auto& kv : plans_)
      if (&kv.second == &plan) return kv.first;
    return 0;
  }

  FrameTransformContext ctx_;
  std::mutex mu_;
  std::mutex lazyMu_;  // per-size tables made on first use (resizeFor, blurFor)
  std::map<int, DevicePlan> plans_;
  DeviceBuffer<int16_t> weights_[9];       // OpenCV's tables [1024][k][k] (general kernels), by kernel size
  DeviceBuffer<uint8_t> weightImages_[9];  // their shared-memory images for the frame kernel
  DeviceBuffer<uint8_t> stagingIn_, stagingOut_;
  std::mutex hostCallMu_;  // the synchronous host-pointer path shares the staging planes and the streams: one call at a time
  cudaStream_t copyIn_ = nullptr, copyIn2_ = nullptr, copyOut_ = nullptr;
  std::vector<cudaEvent_t> chunkIn_, waveDone_;
  WavePlan wavePlans_[2];  // plan index 0 / 1
  long long pipelineMinBytes_ = 6ll << 20;
  int pipelineChunks_ = 0, pipelineBlocks_ = 0;  // 0: automatic
  int pipelineInStreams_ = 1;
  // The streamed call is ~100 runtime calls (chunk copies, events, wave launches, rectangle copies); issued one by one
  // the host thread becomes the bottleneck (measured: no faster than the plain path).  For page-locked caller planes the
  // whole sequence is captured once per (plan, buffers) into a CUDA graph and replayed with one launch.
  struct PlaneGraph {
    const void* plan; unsigned long long generation; const void* in; const void* out; int inPitch, outPitch;
    const void* stagingIn; const void* stagingOut;  // (the staging planes grow on demand: a graph made for old ones is stale)
    int inW, inH, outW, outH;
    int kernels;
    cudaGraphExec_t exec; unsigned long long lastUse;
  };
  std::vector<PlaneGraph> planeGraphs_;
  unsigned long long graphClock_ = 0;
  cudaEvent_t graphFork_ = nullptr, graphJoinIn_ = nullptr, graphJoinOut_ = nullptr;
  // opt-in page-locking of recurring pageable caller planes (ffmpeg recycles its frame pool): see pinIfRecurring()
  struct HostRange { uintptr_t base; size_t bytes; int seen; bool pinned; };
  std::vector<HostRange> hostRanges_;
  bool pinHostPlanes_ = false;
  std::mutex slotMu_;
  std::map<cudaStream_t, std::unique_ptr<StreamSlot>> slots_;
  FrameJobList frameJobs_;
  FrameBlurList frameBlur_;
  std::mutex frameJobsMu_;
  DeviceBuffer<unsigned long long> trace_;
  bool traceEnabled_ = false;
  unsigned long long planGeneration_ = 0;
  cudaStream_t stream_ = nullptr;
  int device_ = 0, numSMs_ = 0;
  bool deviceReady_ = false;
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
  if (!t || !dIn || !dOut || !inW || !inH || !inPitch || !outW || !outH || !outPitch) return 0;
  return t->transformFrameDevice(numPlanes, dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, static_cast<cudaStream_t>(stream));
}
T360_API int T360B200_lowPassPlaneAsync(VideoFrameTransform* t, const uint8_t* dIn, uint8_t* dOut, int w, int h, int inPitch,
                                        int outPitch, int planIndex, void* stream) {
  if (!t || !dIn || !dOut) return 0;
  try {
    return t->lowPassDevice(dIn, dOut, w, h, inPitch, outPitch, planIndex, static_cast<cudaStream_t>(stream));
  } catch (const std::exception& ex) {
    std::printf("Could not filter plane %d. Error: %s\n", planIndex, ex.what());
    return 0;
  }
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
