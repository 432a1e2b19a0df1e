/* transform360-b200: extensions beyond the reference's four-function C-ABI.
 *
 * Nothing here is needed by a drop-in caller (see Transform360/VideoFrameTransformHandler.h).
 * These entry points exist for (1) zero-copy / asynchronous callers that already hold frames in
 * device memory (e.g. an AV_PIX_FMT_CUDA filter, bench.py's device-resident leg), and (2) tests that
 * inspect the host-side plan without a GPU.  Plain C, plain pointers and sizes, no torch types.
 */
#ifndef TRANSFORM360_B200_EXT_H
#define TRANSFORM360_B200_EXT_H

#include "Transform360/VideoFrameTransformHandler.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- host-only plan inspection (never touches CUDA) ------------------------------------------ */
typedef struct T360HostPlan T360HostPlan;

/* Runs the host planner (the re-implementation of the reference's generateMapForPlane, cpp:504-576)
 * for one plane and keeps the result in host memory. */
T360HostPlan* T360B200_hostPlanCreate(const FrameTransformContext* ctx, int inputWidth, int inputHeight,
                                      int outputWidth, int outputHeight);
void T360B200_hostPlanDestroy(T360HostPlan* plan);
/* info[0..5] = mapWidth, mapHeight, numSegments, numTaps, kernelSizeOfInterpolation, numTileJobs */
int T360B200_hostPlanInfo(const T360HostPlan* plan, int info[6]);
/* float32 [mapHeight][mapWidth][2]: the reference's warp map values (cpp:544-545) */
const float* T360B200_hostPlanMap(const T360HostPlan* plan);
/* int32 [mapHeight][mapWidth][2]: what the kernels consume.  word0 = first tap column (before wrapping),
 * word1 = (first tap row << 10) | phase, phase = (fracY32 << 5) | fracX32 (0 for nearest). */
const int32_t* T360B200_hostPlanSamples(const T360HostPlan* plan);
/* The gather plan of the host plan (no GPU needed): how the output plane is cut into jobs for the persistent gather
 * kernel and how the sampling records are laid out for it (formats: csrc/kernels.cuh).  info = {tilesPerRow, tileRows,
 * tileH of the full records, numJobs, class-0 jobs, class-1 jobs, seam jobs, general jobs, share jobs, words of compact
 * records}; *jobs: numJobs x 4 ints {outX, outY | kind << 24, boxX | boxY << 16 | box variant, recordOffset (16-byte units)} in launch
 * order (NULL when the plan is not staged: nearest neighbour, barrel layouts); *records: the full records,
 * tilesPerRow * tileRows * tileH * 32 pairs {col0 | column << 27, row0 << 10 | phase}, tile-major; *compact: the compact
 * records of the staged jobs (32-bit words).  Returns 1 on success.  The pointers stay valid until
 * T360B200_hostPlanDestroy. */
int T360B200_hostPlanGather(T360HostPlan* plan, int info[10], const int32_t** jobs, const int32_t** records,
                            const uint32_t** compact);
/* How the host deals the n <= 32 pixels of one warp step to lanes and copies of the weight table (csrc/gather_plan.h:
 * dealLanes): phases[i] = (fracY32 << 5) | fracX32 of pixel i; laneOf[i] / copyOf[i] receive its lane and table copy.
 * Returns the modelled shared-memory wavefronts of one 128-bit weight load of the warp (0 when n < 32: identity deal). */
int T360B200_dealLanes(int interpolationAlg, int n, const int32_t* phases, int32_t* laneOf, int32_t* copyOf);
/* The frame kernel's shared-memory image of the interpolation table (csrc/kernels.cuh: "Weight tables in shared
 * memory"); returns its size in bytes (0 if unsupported). */
int T360B200_weightImage(int interpolationAlg, const uint8_t** image);
/* low-pass segment i in the reference's order: rect = left, top, width, height; taps = kx then ky */
int T360B200_hostPlanSegment(const T360HostPlan* plan, int i, int rect[4], int numTaps[2], const float** kx,
                             const float** ky);
/* OpenCV-compatible fixed-point interpolation table: int16 [1024][k][k]; returns k (0 if unsupported) */
int T360B200_remapTable(int interpolationAlg, const int16_t** table);

/* ---- device-resident / asynchronous entry points ----------------------------------------------- */
/* Same contract as VideoFrameTransform_transformFramePlane, but both planes are CUDA device pointers,
 * the work is enqueued on `cudaStream` (a cudaStream_t; NULL = the transform's own stream) and the call
 * returns without synchronising.  Returns 1 if everything was enqueued.  Scratch planes and job schedulers are kept
 * per stream: work on one stream is ordered, different streams (also from different host threads) do not interfere. */
int T360B200_transformFramePlaneAsync(VideoFrameTransform* transform, const uint8_t* deviceInput,
                                      uint8_t* deviceOutput, int inputWidth, int inputHeight, int inputPitch,
                                      int outputWidth, int outputHeight, int outputPitch,
                                      int transformMatPlaneIndex, void* cudaStream);
/* All planes of one frame in one call, device to device, asynchronous on `cudaStream`: plane 0 uses plan index 0,
 * planes 1 and 2 plan index 1 (the reference filter's convention, vf_transform360.c:372).  The low-pass stages of the
 * planes run side by side (chroma on internal streams); one gather launch then takes the tiles of every plane;
 * `cudaStream` observes the completion of all of it.  Arrays have numPlanes (1..3) entries: device pointers, per-plane
 * widths / heights / pitches in bytes.  Scratch planes and schedulers are per stream (see above); generateMapForPlane
 * must not run concurrently with frames in flight. */
int T360B200_transformFrameAsync(VideoFrameTransform* transform, int numPlanes, const uint8_t* const* deviceInputs,
                                 uint8_t* const* deviceOutputs, const int* inputWidths, const int* inputHeights,
                                 const int* inputPitches, const int* outputWidths, const int* outputHeights,
                                 const int* outputPitches, void* cudaStream);
/* Runs only the segmented low-pass stage (reference filterPlane, cpp:621-704) device to device. */
int T360B200_lowPassPlaneAsync(VideoFrameTransform* transform, const uint8_t* deviceInput, uint8_t* deviceOutput,
                               int width, int height, int inputPitch, int outputPitch,
                               int transformMatPlaneIndex, void* cudaStream);
/* Opt-in (also: environment T360B200_PIN_HOST_PLANES=1): page-lock pageable caller planes in place the second time
 * the same buffer is seen (cudaHostRegister), so that recycled frame-pool buffers are DMA'd at full PCIe speed.  The
 * caller must keep such buffers alive until VideoFrameTransform_delete. */
void T360B200_setPinHostPlanes(VideoFrameTransform* transform, int enable);
/* Tuning aid: when enabled, every whole-frame gather launch records a timeline of its consumer groups (per group and job:
 * wait start, data ready, done in ns of %globaltimer, job kind; 64 jobs per group, groups = SMs x groups per CTA);
 * T360B200_debugTraceRead copies it out after the stream has been synchronised and returns the number of 64-bit words;
 * with out == NULL it copies nothing and returns the size of the trace buffer in 64-bit words (the largest trace any
 * frame of this transform has needed so far; a smaller frame leaves the rows of its unused groups zero). */
void T360B200_debugTrace(VideoFrameTransform* transform, int enable);
unsigned long long T360B200_debugTraceRead(VideoFrameTransform* transform, unsigned long long* out, unsigned long long maxWords);
/* Blocks until everything enqueued on the transform's own stream has finished; 1 = ok. */
int T360B200_synchronize(VideoFrameTransform* transform);
/* The transform's own stream (cudaStream_t) */
void* T360B200_stream(VideoFrameTransform* transform);

/* ---- bookkeeping ---------------------------------------------------------------------------------- */
/* Number of this library's kernels launched by the calling process so far. */
unsigned long long T360B200_kernelLaunchCount(void);
/* Bytes of device memory held by the plan of one index (sampling plan + low-pass tables). */
unsigned long long T360B200_planDeviceBytes(VideoFrameTransform* transform, int transformMatPlaneIndex);
/* counts[0] = gather tiles staged through TMA into shared memory, counts[1] = tiles on the general (L1) path,
 * counts[2] = low-pass warp-jobs on the register-resident strip kernel, counts[3] = low-pass jobs on the general
 * (large vertical kernel) paths. */
int T360B200_planTileCounts(VideoFrameTransform* transform, int transformMatPlaneIndex, int counts[4]);
/* CUDA devices visible (0 when there is none or the driver is absent). */
int T360B200_deviceCount(void);
const char* T360B200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* TRANSFORM360_B200_EXT_H */
