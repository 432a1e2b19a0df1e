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
/* cv::remap's border modes for a caller's warp map (OpenCV's values) */
#define T360_BORDER_WRAP 3
#define T360_BORDER_TRANSPARENT 5
/* The host twin of T360B200_generateMapFromWarp: the plan of one plane from the caller's map, in host memory, for the
 * inspectors above and below (map = the caller's map, mapWidth x mapHeight, no low-pass segments).  NULL, with a message on
 * stdout, for whatever T360B200_generateMapFromWarp refuses. */
T360HostPlan* T360B200_hostPlanCreateFromWarp(const FrameTransformContext* ctx, const float* map, int mapWidth, int mapHeight,
                                              int inputWidth, int inputHeight, int border);
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
/* What the frame kernel runs for the general jobs of T360B200_hostPlanGather (the pole caps, whose windows fit no box as
 * a 32 x 32 tile), and the whole launch list.  info = {pole-cap jobs, border jobs, words of *capRecords, launch jobs};
 * *capJobs: (pole-cap + border jobs) x 4 ints in the job format, record offsets counting on after the compact records
 * (the device buffer holds compact records, then *capRecords); *launchJobs: the job list the kernel claims from, in
 * launch order (every job of T360B200_hostPlanGather but the general ones, and *capJobs).  Formats: csrc/kernels.cuh.
 * Returns 1 on success; the pointers stay valid until T360B200_hostPlanDestroy. */
int T360B200_hostPlanPoleCaps(T360HostPlan* plan, int info[4], const int32_t** capJobs, const uint32_t** capRecords,
                              const int32_t** launchJobs);
/* Per job of the launch list of T360B200_hostPlanPoleCaps, what the planner records for streaming a host plane through the
 * device: *needRows = the source rows [0, n) the job reads (the whole plane if a window wraps vertically), *rects = the
 * bounding rectangle {x0, y0, x1, y1} (exclusive ends) of the output pixels it writes.  *numJobs = launch jobs.  Returns 1
 * on success; the pointers stay valid until T360B200_hostPlanDestroy. */
int T360B200_hostPlanLaunchExtents(T360HostPlan* plan, int* numJobs, const int32_t** needRows, const int32_t** rects);
/* The schedule the synchronous host-pointer call streams a large plane with (csrc/gather_plan.h: scheduleWaves), for
 * `chunks` input row bands (0: as many as the call takes for the plan's input size).  needRows: per launch job, in place of
 * the planner's (NULL: the planner's).  info = {chunks, launch jobs, rectangles}; *chunkRowEnd: per chunk the end of the
 * rows delivered with it; *waveStart: chunks + 1 entries, wave c = (*order)[waveStart[c] .. waveStart[c + 1]); *order: the
 * launch-job indices wave by wave; *rects: per output rectangle {wave it is copied back after, x0, y0, x1, y1}.  Returns 1
 * on success; the pointers stay valid until the next call with this plan or its T360B200_hostPlanDestroy. */
int T360B200_hostPlanWaves(T360HostPlan* plan, int chunks, const int32_t* needRows, int info[3], const int32_t** chunkRowEnd,
                           const int32_t** waveStart, const int32_t** order, const int32_t** rects);
/* The job list and record buffer the frame kernel reads (csrc/gather_plan.h: deviceJobs, deviceRecords): the launch list
 * of T360B200_hostPlanPoleCaps with the width of each class-0 source box (csrc/kernels.cuh: class0BoxW) in bits 28-31
 * of recordOffset, and the compact records followed by the pole-cap records, the window offsets of a job with a narrow
 * box at that box's pitch.  info = {jobs, words of records}.  Returns 1 on success; the pointers stay valid until
 * T360B200_hostPlanDestroy. */
int T360B200_hostPlanDeviceLists(T360HostPlan* plan, int info[2], const int32_t** jobs, const uint32_t** records);
/* How the host deals the n <= 32 pixels of one warp step to lanes and copies of the weight table (csrc/gather_plan.h:
 * dealLanes): phases[i] = (fracY32 << 5) | fracX32 of pixel i; laneOf[i] / copyOf[i] receive its lane and table copy.
 * Returns the modelled shared-memory wavefronts of one 128-bit weight load of the warp (0 when n < 32: identity deal). */
int T360B200_dealLanes(int interpolationAlg, int n, const int32_t* phases, int32_t* laneOf, int32_t* copyOf);
/* The frame kernel's shared-memory image of the interpolation table (csrc/kernels.cuh: "Weight tables in shared
 * memory"); returns its size in bytes (0 if unsupported). */
int T360B200_weightImage(int interpolationAlg, const uint8_t** image);
/* The low-pass job lists of plans[0 .. numPlans) (no GPU needed) for planes of width x height (0: each plan's input size),
 * as the device holds them: one plan's lists, or for 2-3 plans (the planes of a frame) their strip jobs merged into one
 * list (the plane in each job's edge field).  *image: the packed lists (formats: csrc/kernels.cuh, csrc/lowpass_jobs.h),
 * valid until the next call with the same plans[0] or its T360B200_hostPlanDestroy.  layout = {strip jobs by vertical
 * half-size 1..3 (3 counts), tile jobs, direct jobs, taps, tile shared-memory bytes, needsClear (some pixel lies under no
 * segment), byte offsets of the three strip arrays, of the tiles, the direct jobs and the taps, image bytes}.  Returns 1
 * on success. */
int T360B200_hostPlanBlurLists(T360HostPlan* const* plans, int numPlans, int width, int height, int layout[15],
                               const uint8_t** image);
/* low-pass segment i in the reference's order: rect = left, top, width, height; taps = kx then ky */
int T360B200_hostPlanSegment(const T360HostPlan* plan, int i, int rect[4], int numTaps[2], const float** kx,
                             const float** ky);
/* OpenCV-compatible fixed-point interpolation table: int16 [1024][k][k]; returns k (0 if unsupported) */
int T360B200_remapTable(int interpolationAlg, const int16_t** table);

/* ---- warp maps: remap through the caller's own map ------------------------------------------------ */
/* Installs the plan of plan index transformMatPlaneIndex, as VideoFrameTransform_generateMapForPlane does, from the caller's
 * map instead of the context's geometry: `map` (host memory, float32 [mapHeight][mapWidth][2], cv::remap's CV_32FC2 map: the
 * source x, y of every output pixel) is sampled from planes of inputWidth x inputHeight with the context's interpolation_alg
 * and `border` (T360_BORDER_WRAP or T360_BORDER_TRANSPARENT), bit for bit as cv::remap does (NaN, infinities and coordinates
 * beyond the int16 range included).  Every frame entry point then serves the index unchanged (transformFramePlane with host
 * or device planes, T360B200_transformFramePlaneAsync, T360B200_transformFrameAsync); an output size other than the map's
 * takes the INTER_AREA resize, and under BORDER_TRANSPARENT chroma outputs (plan index 1) are pre-filled with 128 while luma
 * outputs keep the caller's bytes where no source pixel lands.  Returns 1 on success; 0 with a message on stdout, before any
 * CUDA call, for a NULL map, non-positive sizes, a map larger than 65536 in a dimension, another border, an unknown
 * interpolation_alg or enable_low_pass_filter != 0.  While an index holds such a plan, T360B200_reconfigure,
 * T360B200_reconfigureAsync and the view, orientation and pose calls are refused (0, a message, no CUDA call);
 * VideoFrameTransform_generateMapForPlane on the index replaces the warp plan. */
int T360B200_generateMapFromWarp(VideoFrameTransform* transform, const float* map, int mapWidth, int mapHeight, int inputWidth,
                                 int inputHeight, int border, int transformMatPlaneIndex);
/* One frame through per-plane maps in device memory, a map per plane of its output plane's size (float32 pairs, row r at
 * deviceMaps[p] + r * mapPitches[p] bytes; the base 8-byte aligned, the pitch a multiple of 8 of at least 8 x the output
 * width): the frame T360B200_generateMapFromWarp with the same maps would give, with the context's interpolation_alg and
 * `border`, BORDER_TRANSPARENT's chroma pre-fill included, and no plan: one kernel launch gathers every plane, each pixel's
 * sampling record computed from its map entry.  The asynchronous contract of T360B200_transformFrameAsync: the call never
 * synchronises the device, so the maps may change every frame (keep them alive until the frame is done).  Returns 1 if
 * everything was enqueued; 0 with a message on stdout, before any CUDA call, for 0 or more than 3 planes, NULL maps or
 * planes, a map pitch or alignment as above violated, another border, an unknown interpolation_alg or low-pass on. */
int T360B200_remapFrameAsync(VideoFrameTransform* transform, int numPlanes, const float* const* deviceMaps, const int* mapPitches,
                             int border, const uint8_t* const* deviceInputs, uint8_t* const* deviceOutputs, const int* inputWidths,
                             const int* inputHeights, const int* inputPitches, const int* outputWidths, const int* outputHeights,
                             const int* outputPitches, void* cudaStream);

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
 * must not run concurrently with frames in flight (T360B200_reconfigure and T360B200_reconfigureAsync may). */
int T360B200_transformFrameAsync(VideoFrameTransform* transform, int numPlanes, const uint8_t* const* deviceInputs,
                                 uint8_t* const* deviceOutputs, const int* inputWidths, const int* inputHeights,
                                 const int* inputPitches, const int* outputWidths, const int* outputHeights,
                                 const int* outputPitches, void* cudaStream);
/* Runs only the segmented low-pass stage (reference filterPlane, cpp:621-704) device to device. */
int T360B200_lowPassPlaneAsync(VideoFrameTransform* transform, const uint8_t* deviceInput, uint8_t* deviceOutput,
                               int width, int height, int inputPitch, int outputPitch,
                               int transformMatPlaneIndex, void* cudaStream);
/* Replaces the transform's FrameTransformContext. Every plan index generated so far is re-planned for the new
 * context with the sizes it was generated with. Returns 1 on success. 0: message on stdout, old configuration
 * still fully in effect.
 * Frame-exact: work enqueued before the call (any entry point, any stream) completes with the old configuration, work
 * enqueued after it returns uses the new one.  The call may overlap frames in flight and calls on other threads: host
 * planning and the upload run while they continue; the call then swaps the plans, waits for the device's work enqueued so
 * far and releases the old ones.  Any field may change as long as the caller keeps the plane sizes it generated the maps for
 * (layouts, stereo formats and scale factors included).  Before any generateMapForPlane only the context is replaced
 * and no CUDA call is made. */
int T360B200_reconfigure(VideoFrameTransform* transform, const FrameTransformContext* ctx);
/* Replaces the transform's FrameTransformContext without waiting for a re-plan.  Returns 1 after checks on the host only
 * (no device wait, no planning): every frame enqueued after the call, through any entry point and on any stream, equals bit
 * for bit what a fresh transform made with *ctx gives; work enqueued before it uses the old context.  Until the new plans
 * are in, whole frames (T360B200_transformFrameAsync, and the view, orientation and pose calls) are served by the per-frame
 * kernels, which compute every sampling position from the context; the per-plane entry points (transformFramePlane,
 * T360B200_transformFramePlaneAsync, T360B200_lowPassPlaneAsync) and whole frames of another plane size than planned
 * wait for the plans.  A background thread plans the latest context once no newer call has arrived for a settle
 * interval (0.25 s), uploads the plans into fresh buffers, swaps them in without stalling the threads that enqueue frames
 * and releases the old ones after a device wait of its own; from then on frames take the planned frame kernel again.  A
 * plan superseded while it was being made is discarded.  Any field may change except the ones that size the planes and
 * maps (input / output layout, both stereo formats, both scale factors: use T360B200_reconfigure).  Refused, before any
 * CUDA call, with 0 and a message on stdout and the old context left in effect: a change of one of those fields, an
 * unknown interpolation_alg, a float field that is not finite, and a context the low-pass planner refuses for one of the
 * generated plan indices.  Before any generateMapForPlane only the context is replaced and no CUDA call is made.
 * T360B200_reconfigure and generateMapForPlane discard / finish a pending plan first; VideoFrameTransform_delete waits
 * for at most the plan being made. */
int T360B200_reconfigureAsync(VideoFrameTransform* transform, const FrameTransformContext* ctx);
/* Whether the plans of the current context are in effect: 1 yes; 0 not yet (block == 0); -1 the background planner failed on
 * it (message on stdout; frames keep being served by the per-frame kernels).  With block != 0 it plans at once, without the
 * settle interval, and returns 1 or -1 when done, after the device memory of the plans it replaced has been released. */
int T360B200_reconfigureWait(VideoFrameTransform* transform, int block);
/* A FLAT_FIXED view, in degrees, as the context's fixed_yaw, fixed_pitch, fixed_hfov and fixed_vfov. */
typedef struct T360View {
  float yaw, pitch, hfov, vfov;
} T360View;
/* One frame of a FLAT_FIXED transform with its own view, without re-planning: the arguments and the asynchronous contract
 * of T360B200_transformFrameAsync, plus `view`.  The frame equals, bit for bit, what a fresh transform would give for the
 * transform's current context with fixed_yaw, fixed_pitch, fixed_hfov and fixed_vfov replaced by *view (low-pass and the
 * INTER_AREA resize for scale factors != 1 included); the transform's context is not changed.  The gather computes the
 * sampling positions from the view in one launch for all planes; a view-dependent low-pass is re-planned on the host and
 * its lists are uploaded in stream order from page-locked memory (skipped when they equal the previous frame's on that
 * stream).  The call never synchronises the device, so views may change every frame.  Like every entry point it is
 * frame-exact against T360B200_reconfigure.  Returns 1 if everything was enqueued; 0 with a message on stdout for an
 * output_layout other than FLAT_FIXED, a non-finite view, a plan index that was never generated, or an input plane of
 * another size than its map was generated for. */
int T360B200_transformFrameViewAsync(VideoFrameTransform* transform, const T360View* view, int numPlanes,
                                     const uint8_t* const* deviceInputs, uint8_t* const* deviceOutputs, const int* inputWidths,
                                     const int* inputHeights, const int* inputPitches, const int* outputWidths,
                                     const int* outputHeights, const int* outputPitches, void* cudaStream);
/* Host only, no CUDA: the sampling records the per-view kernel computes for one plane of a FLAT_FIXED context with the view
 * substituted, int32 [mapHeight][mapWidth][2] (map = scaled output size) in the format of T360B200_hostPlanSamples.
 * Returns 1 on success; 0 (message on stdout) for another layout, a non-finite view or invalid sizes. */
int T360B200_viewSamples(const FrameTransformContext* ctx, const T360View* view, int inputWidth, int inputHeight,
                         int outputWidth, int outputHeight, int32_t* samples);
/* An orientation, in degrees, as the context's fixed_yaw, fixed_pitch and fixed_roll. */
typedef struct T360Orientation {
  float yaw, pitch, roll;
} T360Orientation;
/* One frame of a CUBEMAP_32, CUBEMAP_23_OFFCENTER, EAC_32 or EQUIRECT transform (input EQUIRECT or CUBEMAP_32) with its own
 * orientation, without re-planning: the arguments and the asynchronous contract of T360B200_transformFrameAsync, plus
 * `orientation`.  The frame equals, bit for bit, what a fresh transform would give for the transform's current context
 * with fixed_yaw, fixed_pitch and fixed_roll replaced by *orientation (low-pass and the INTER_AREA resize for scale factors
 * != 1 included); the transform's context is not changed.  The gather computes every pixel's sampling position from the
 * orientation in one launch for all planes; a low-pass is re-planned on the host for the orientation's yaw and pitch and
 * its lists are uploaded in stream order from page-locked memory, as in T360B200_transformFrameViewAsync.  The call never
 * synchronises the device, so the orientation may change every frame, and it is frame-exact against
 * T360B200_reconfigure.  Returns 1 if everything was enqueued; 0 with a message on stdout for FLAT_FIXED (use
 * T360B200_transformFrameViewAsync), BARREL or BARREL_SPLIT output, a non-finite orientation, a plan index that was never
 * generated, or an input plane of another size than its map was generated for. */
int T360B200_transformFrameOrientedAsync(VideoFrameTransform* transform, const T360Orientation* orientation, int numPlanes,
                                         const uint8_t* const* deviceInputs, uint8_t* const* deviceOutputs,
                                         const int* inputWidths, const int* inputHeights, const int* inputPitches,
                                         const int* outputWidths, const int* outputHeights, const int* outputPitches,
                                         void* cudaStream);
/* Host only, no CUDA: the sampling records the per-frame orientation kernel computes for one plane of `ctx` with the
 * orientation substituted, int32 [mapHeight][mapWidth][2] (map = scaled output size) in the format of
 * T360B200_hostPlanSamples.  Returns 1 on success; 0 (message on stdout) for layouts without per-frame orientation, a
 * non-finite orientation or invalid sizes. */
int T360B200_orientedSamples(const FrameTransformContext* ctx, const T360Orientation* orientation, int inputWidth,
                             int inputHeight, int outputWidth, int outputHeight, int32_t* samples);
/* A camera pose, in degrees, as the context's fixed_yaw, fixed_pitch, fixed_roll, fixed_hfov and fixed_vfov. */
typedef struct T360Pose {
  float yaw, pitch, roll, hfov, vfov;
} T360Pose;
/* One frame of any transform with its own pose, without re-planning: the arguments and the asynchronous contract of
 * T360B200_transformFrameAsync, plus `pose`.  The frame equals, bit for bit, what a fresh transform would give for the
 * transform's current context with its five view fields replaced by *pose (low-pass, the INTER_AREA resize for scale
 * factors != 1 and the barrel layouts' transparent border included: chroma planes are pre-filled with 128, luma keeps the
 * caller's bytes where no source pixel lands); the transform's context is not changed.  Every output layout is served, and
 * for layouts other than FLAT_FIXED every input layout (any input but CUBEMAP_32 is read as equirect, as the planner
 * does): FLAT_FIXED through the per-view kernel (roll plays no part in it), the others through the per-frame orientation
 * kernel, so a caller can pass the current camera every frame without knowing which serves its layout.  Without low-pass
 * a frame is one kernel launch.  The call never synchronises the device, and it is frame-exact against
 * T360B200_reconfigure.  Returns 1 if everything was enqueued; 0 with a message on stdout, before any CUDA call, for a
 * non-finite pose field, a transform without interpolation algorithm, a plan index that was never generated, an input
 * plane of another size than its map was generated for, or 0 or more than 3 planes. */
int T360B200_transformFramePoseAsync(VideoFrameTransform* transform, const T360Pose* pose, int numPlanes,
                                     const uint8_t* const* deviceInputs, uint8_t* const* deviceOutputs, const int* inputWidths,
                                     const int* inputHeights, const int* inputPitches, const int* outputWidths,
                                     const int* outputHeights, const int* outputPitches, void* cudaStream);
/* Host only, no CUDA: the sampling records the per-frame kernels compute for one plane of `ctx` with the pose substituted,
 * int32 [mapHeight][mapWidth][2] (map = scaled output size) in the format of T360B200_hostPlanSamples.  Returns 1 on
 * success; 0 (message on stdout) for an unknown output layout, a non-finite pose or invalid sizes. */
int T360B200_poseSamples(const FrameTransformContext* ctx, const T360Pose* pose, int inputWidth, int inputHeight,
                         int outputWidth, int outputHeight, int32_t* samples);
/* ---- fisheye camera input -------------------------------------------------------------------------
 * One or two fisheye lenses with OpenCV's fisheye (Kannala-Brandt) calibration, the K and D of cv2.fisheye.calibrate, as
 * the input of a sphere output.
 *
 * Rig frame: the frame of the direction the output chain hands to the input lookup (after the off-centre warp and the
 * rotation by the orientation, which turn the output exactly as for an equirect input): x right, y up, z forward; an
 * equirect input would show direction d at u = atan2(x, z) / 2pi + 0.5, v = 0.5 - asin(y / |d|) / pi.
 *
 * Lens i: R = Ry(yaw) Rx(-pitch) Rz(roll) (Ry(a) = [[c,0,s],[0,1,0],[-s,0,c]], Rx(b) = [[1,0,0],[0,c,-s],[0,s,c]],
 * Rz(g) = [[c,-s,0],[s,c,0],[0,0,1]]), so its optical axis is (cos pitch sin yaw, sin pitch, cos pitch cos yaw) and a back
 * lens has yaw 180.  (X, Y', Z) = R^T d, and (X, Y, Z) = (X, -Y', Z) are OpenCV's camera coordinates (y down).
 * rho = sqrt(X^2 + Y^2), theta = atan2(rho, Z), theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 + k4 theta^8),
 * (x', y') = theta_d / rho (X, Y) ((0, 0) at rho = 0).  In a plane of inW x inH the source position is
 * ((fx x' + cx + 0.5) / calibWidth) inW - 0.5, and likewise for y: at the calibration size fx x' + cx, which is
 * cv2.fisheye.projectPoints (skew 0) for Z > 0; chroma planes scale the calibration as the planned layouts do.
 * A direction goes to the lens with the larger Z / |d| (ties: lens 0), with a hard seam (feathered: the blend calls
 * below); theta > maxAngle, and a barrel
 * dead zone, are uncovered.  Sampling is BORDER_TRANSPARENT: uncovered pixels and pixels whose anchor tap lies outside the
 * source keep what the output holds (luma the caller's bytes, chroma 128, pre-filled).
 *
 * The context supplies the output: output_layout (CUBEMAP_32, CUBEMAP_23_OFFCENTER, EAC_32, EQUIRECT, BARREL or
 * BARREL_SPLIT) and its geometry fields (expand_coef, fixed_cube_offcenter_*, is_horizontal_offset), vflip and
 * interpolation_alg; the orientation comes with each call.  Not read: input_layout, input_expand_coef, both stereo formats
 * and both scale factors (the rig is mono, and output planes are rendered at their own size).
 *
 * Refused, with 0 and a message on stdout before any CUDA call: a NULL rig or orientation, numLenses other than 1 or 2,
 * non-positive calibration sizes, a non-finite field (of the orientation or of a used lens), fx or fy <= 0, maxAngle outside
 * (0, 180], a distortion whose theta_d(theta) is not strictly increasing on [0, maxAngle] (it would mirror the image),
 * FLAT_FIXED or an unknown output layout, enable_low_pass_filter != 0 and an unknown interpolation_alg. */
typedef struct T360Lens {
  float fx, fy, cx, cy; /* intrinsics in pixels of a calibWidth x calibHeight frame */
  float k[4];           /* k1 .. k4 */
  float yaw, pitch, roll; /* extrinsics, degrees */
  float maxAngle;       /* half field of view covered, degrees */
} T360Lens;
typedef struct T360LensRig {
  int numLenses, calibWidth, calibHeight;
  T360Lens lens[2];
} T360LensRig;
/* Host only, no CUDA: the CV_32FC2 map (float32 [outputHeight][outputWidth][2], NaN where uncovered) of one plane of
 * inputWidth x inputHeight.  T360B200_generateMapFromWarp(map, ..., T360_BORDER_TRANSPARENT, index) plans it for a fixed
 * pose: every frame entry point, the streamed host path and the INTER_AREA resize then serve it, and frames equal, bit for
 * bit, those of T360B200_transformFrameLensAsync for the same rig and orientation.  Returns 1; 0 (message) for the refusals
 * above, a NULL map or non-positive sizes. */
int T360B200_lensMap(const FrameTransformContext* ctx, const T360LensRig* rig, const T360Orientation* orientation, int inputWidth,
                     int inputHeight, int outputWidth, int outputHeight, float* map);
/* One frame of a lens rig, every plane in one gather launch: the arguments and the asynchronous contract of
 * T360B200_transformFrameAsync, plus `rig` and `orientation`, both of which may change every frame.  Needs no plan: it works
 * on a transform that was never planned as on one holding context or warp plans, and does not touch them.  The output
 * layout's tables are built on the host and uploaded in stream order when the context or an output size changes.  Takes the
 * reader lock, so it is frame-exact against T360B200_reconfigure and T360B200_reconfigureAsync, and never synchronises the
 * device.  Returns 1 if everything was enqueued; 0 with a message on stdout, before any CUDA call, for the refusals above,
 * 0 or more than 3 planes, or an invalid plane description. */
int T360B200_transformFrameLensAsync(VideoFrameTransform* transform, const T360LensRig* rig, const T360Orientation* orientation,
                                     int numPlanes, const uint8_t* const* deviceInputs, uint8_t* const* deviceOutputs,
                                     const int* inputWidths, const int* inputHeights, const int* inputPitches,
                                     const int* outputWidths, const int* outputHeights, const int* outputPitches, void* cudaStream);
/* ---- fisheye lens rigs with a feathered seam --------------------------------------------------------
 * A two-lens rig whose lenses are blended across a belt of seamWidth degrees instead of meeting at a hard seam.  Rig,
 * orientation and context mean what they mean above.  For the rig direction d of an output pixel, each lens i gives
 * theta_i = atan2(rho, Z) of its camera coordinates, covers d when theta_i <= its maxAngle, and then has the source
 * position above.  The weight w (0..256) of lens 1:
 *   - both lenses cover d: t = 0.5 + (theta0 - theta1) s, with s = 1 / (2 seamWidth pi / 180) (computed in double, used
 *     as float; every float step rounded to nearest), tw = 256 t, w = 0 for tw <= 0, 256 for tw >= 256, else tw rounded
 *     half to even.  For back-to-back lenses of half-angle A this is a linear ramp across a belt seamWidth degrees wide,
 *     centred on the seam; it lies inside both lenses' coverage when seamWidth <= 2 (A - 90): 10 for 190-degree lenses;
 *   - only lens i covers d: w = 0 for lens 0, 256 for lens 1 (this also fills directions the hard seam leaves
 *     uncovered when the closer lens does not reach them);
 *   - neither covers d, or d is in a barrel dead zone: uncovered, the pixel keeps what the output holds.
 * a = lens 0's sample where w < 256, b = lens 1's where w > 0, each interpolated with BORDER_TRANSPARENT as above.  Where
 * both exist the pixel is (a (256 - w) + b w + 128) >> 8; where BORDER_TRANSPARENT skips one (its anchor tap lies outside
 * the source), the other alone; where it skips both, the pixel keeps what the output holds.  Pre-fill as above: chroma
 * 128, luma the caller's bytes.
 *
 * Refused, with 0 and a message on stdout before any CUDA call: the refusals of the lens calls above, numLenses other than
 * 2 (a single lens has no seam: T360B200_transformFrameLensAsync), and a seamWidth that is not finite or lies outside
 * [0.01, 180]. */
/* Host only, no CUDA: the host twin of T360B200_transformFrameLensBlendAsync for one plane of inputWidth x inputHeight.
 * map0, map1: CV_32FC2 maps (float32 [outputHeight][outputWidth][2]) of lens 0 and lens 1, NaN where that lens does not
 * contribute (it does not cover the pixel's direction, or w gives it no weight); weight: w (uint16 [outputHeight]
 * [outputWidth], 0 where neither lens covers the pixel).  cv::remap of each map with BORDER_TRANSPARENT, combined as above,
 * gives the frame call's plane bit for bit.  Returns 1; 0 (message) for the refusals above, a NULL array or non-positive
 * sizes. */
int T360B200_lensBlendMaps(const FrameTransformContext* ctx, const T360LensRig* rig, float seamWidth, const T360Orientation* orientation,
                           int inputWidth, int inputHeight, int outputWidth, int outputHeight, float* map0, float* map1, uint16_t* weight);
/* One frame of a two-lens rig with a feathered seam, every plane in one gather launch: the arguments and the asynchronous
 * contract of T360B200_transformFrameLensAsync, plus seamWidth, which may change every frame like the rig and the
 * orientation.  Needs no plan and does not touch the plans; takes the reader lock; never synchronises the device.  Returns 1
 * if everything was enqueued; 0 with a message on stdout, before any CUDA call, for the refusals above, 0 or more than 3
 * planes, or an invalid plane description. */
int T360B200_transformFrameLensBlendAsync(VideoFrameTransform* transform, const T360LensRig* rig, float seamWidth,
                                          const T360Orientation* orientation, int numPlanes, const uint8_t* const* deviceInputs,
                                          uint8_t* const* deviceOutputs, const int* inputWidths, const int* inputHeights,
                                          const int* inputPitches, const int* outputWidths, const int* outputHeights,
                                          const int* outputPitches, void* cudaStream);
/* ---- lens photometry ---------------------------------------------------------------------------------
 * The lens calls above move pixels only: each lens loses light towards its rim, where the seam lies, and the two sensors
 * of a dual-fisheye camera run their own exposure and white balance, so a seam (hard or feathered) shows a brightness
 * step.  These calls correct each lens's sample before the seam combines them, and measure the mismatch that is left.
 * The model is in code values, as the frame holds them: no transfer function is applied.  V is the falloff measured in code
 * values (for example fitted to a flat-field frame); scaling every plane about its pivot by one factor models a scale of
 * R'G'B', and the per-plane gains and offsets model the exposure and a colour cast between the lenses.
 *
 * For each lens sample s the frame uses (plane p, lens i), every float step rounded to nearest, + - * / only, in this
 * order on the host and on the device:
 *   r = theta_d = theta (1 + k1 theta^2 + ...) of the lens calls (so the image radius of the pixel is f r: a falloff
 *     measured against the pixel radius R at the calibration size is a polynomial in R / f);
 *   t = r r, V = 1 + t (v1 + t (v2 + t v3)), G = gain_p / V;
 *   Gq = G 4096 rounded half to even, at most 65535 (G >= 16);
 *   Oq = round(16 offset_p), computed on the host, half away from zero;
 *   P = lumaPivot for plane 0, 128 for planes 1 and 2;
 *   s' = clamp(P + ((((s - P) Gq) + Oq 256 + 2048) >> 12), 0, 255), >> an arithmetic shift.
 * vignetting = 0, gain = 1 and offset = 0 give Gq = 4096 and s' = s: the frames of the lens calls above, bit for bit.
 *
 * Seams: seamWidth == 0 is the hard seam of T360B200_transformFrameLensAsync (1 or 2 lenses, the closer lens carries the
 * pixel); seamWidth in [0.01, 180] the feathered seam of T360B200_transformFrameLensBlendAsync (2 lenses, its w).  Each
 * lens's sample is corrected before the combination: the feathered seam gives (a' (256 - w) + b' w + 128) >> 8.  Samples
 * that BORDER_TRANSPARENT skips stay skipped, and the pre-fill is the lens calls' (chroma 128, luma the caller's bytes).
 *
 * Statistics: deviceStats (device memory, NULL: none) receives [numPlanes][6] sums per frame, n, sum a', sum b', sum a'^2,
 * sum b'^2, sum a' b', over the output pixels where both lenses cover the pixel's direction and neither sample is skipped;
 * a' and b' are lens 0's and lens 1's corrected samples.  With the hard seam too: there the overlap's pixels gather the
 * other lens for the statistics only, and the frame is the same as without them.  The call zeroes the buffer in stream
 * order before the gather; the sums are integers, exact whatever the order of accumulation.  A one-lens rig gives zeros.
 * Every output pixel weighs the same, whatever solid angle it covers: an equirect output, for example, over-weights the
 * poles.
 *
 * Refused, with 0 and a message on stdout before any CUDA call: every refusal of T360B200_transformFrameLensAsync, and with
 * seamWidth > 0 every refusal of T360B200_transformFrameLensBlendAsync; a seamWidth that is negative, not finite or in
 * (0, 0.01); a NULL photometry; lumaPivot outside 0..255; a field of a lens that is read (lens[1] with two lenses) that
 * is not finite, a gain outside (0, 8] or an offset outside [-64, 64]; a falloff with V(r) <= 0 somewhere on [0,
 * theta_d(maxAngle)] (checked in double on a 4096-step grid). */
typedef struct T360LensPhotometry {
  float vignetting[3]; /* v1..v3 of the falloff V(r) = 1 + v1 r^2 + v2 r^4 + v3 r^6, r = theta_d (radians) */
  float gain[3];       /* per plane: 0 = luma, 1 and 2 = chroma; finite, in (0, 8] */
  float offset[3];     /* per plane, in code values; finite, in [-64, 64] */
} T360LensPhotometry;
typedef struct T360RigPhotometry {
  int lumaPivot;              /* 0..255: the level luma scales about (16 limited range, 0 full range); chroma scales about 128 */
  T360LensPhotometry lens[2]; /* lens[1] is read only with numLenses == 2 */
} T360RigPhotometry;
/* Host only, no CUDA: the host twin of T360B200_transformFrameLensPhotoAsync for plane `plane` (0..2) of inputWidth x
 * inputHeight.  map0, map1: CV_32FC2 maps (float32 [outputHeight][outputWidth][2]) of lens 0 and lens 1, the lens's entry
 * wherever it covers the pixel's direction, NaN elsewhere; weight: w (uint16 [outputHeight][outputWidth]), 0 or 256 from
 * the lens choice of the hard seam, the blend weight of the feathered one; gain0, gain1: each lens's Gq for the plane
 * (uint16), 0 where it does not cover the pixel.  The frame's plane is cv::remap of each map with BORDER_TRANSPARENT, then
 * s', then: w = 0 lens 0's alone, w = 256 lens 1's alone, else the combination above (the other alone where one is
 * skipped); the statistics are the sums over the pixels where both maps are finite and neither sample is skipped.
 * Returns 1; 0 (message) for the refusals above, a plane outside 0..2, a NULL array or non-positive sizes. */
int T360B200_lensPhotoMaps(const FrameTransformContext* ctx, const T360LensRig* rig, const T360RigPhotometry* photometry, float seamWidth,
                           const T360Orientation* orientation, int plane, int inputWidth, int inputHeight, int outputWidth,
                           int outputHeight, float* map0, float* map1, uint16_t* weight, uint16_t* gain0, uint16_t* gain1);
/* One frame of a lens rig with photometry, every plane in one gather launch: the arguments and the asynchronous contract
 * of T360B200_transformFrameLensAsync, plus photometry, seamWidth and deviceStats, which may change every frame like the
 * rig and the orientation.  Needs no plan and does not touch the plans; takes the reader lock; never synchronises the
 * device.  Zeroing deviceStats is a memset.  There is no planned path: a plan carries one record per pixel.  Returns 1 if
 * everything was enqueued; 0 with a message on stdout, before any CUDA call, for the refusals above, 0 or more than 3
 * planes, or an invalid plane description. */
int T360B200_transformFrameLensPhotoAsync(VideoFrameTransform* transform, const T360LensRig* rig, const T360RigPhotometry* photometry,
                                          float seamWidth, const T360Orientation* orientation, unsigned long long* deviceStats,
                                          int numPlanes, const uint8_t* const* deviceInputs, uint8_t* const* deviceOutputs,
                                          const int* inputWidths, const int* inputHeights, const int* inputPitches,
                                          const int* outputWidths, const int* outputHeights, const int* outputPitches, void* cudaStream);
/* ---- rectilinear views -------------------------------------------------------------------------------
 * A perspective (pinhole) virtual camera looking into 360-degree or fisheye footage: reframing with pan, tilt, roll and
 * zoom, or undistortion of a fisheye lens.  The camera is a T360Pose (degrees).  For output pixel (i, j) of a plane of
 * mapW x mapH (the output plane's own size):
 *   1. x = (j + 0.5) / mapW, y = (i + 0.5) / mapH (float);
 *   2. the output eye split of the sphere outputs: a stereo input with output_stereo_format LR or TB gives two views of
 *      the same pose, side by side (x folded) or stacked (y folded, flipped with vflip); with a mono output, eye 0;
 *   3. y' = 1 - y;
 *   4. the ray q = ((2x - 1) tx, (2y' - 1) ty, 1), tx = tan(hfov / 2), ty = tan(vfov / 2), computed in double and stored
 *      as float.  So hfov and vfov are the full angles between the plane's outer pixel edges, and pixels are square when
 *      tan(vfov / 2) / tan(hfov / 2) = mapH / mapW;
 *   5. q rotated by yaw, pitch and roll exactly as the sphere outputs rotate their points: with hfov = vfov = 90 the view
 *      of an N x N plane is the FRONT face (bottom row, middle) of a 3N x 2N CUBEMAP_32 output of the same orientation;
 *   6. the input:
 *      - without a rig, the context's input: CUBEMAP_32 (gnomonic, with input_expand_coef) or, for any other
 *        input_layout, equirect (u = atan2(x, z) / 2pi + 0.5 of the rotated ray, as the sphere outputs); the input eye
 *        re-pack of a stereo input, then u inW - 0.5, v inH - 0.5.  Sampled with BORDER_WRAP;
 *      - with a rig (the rig frame above), the lens with the larger Z and its projection, a hard seam, NaN where no lens
 *        covers the ray.  Sampled with BORDER_TRANSPARENT: chroma planes are pre-filled with 128, luma keeps the caller's
 *        bytes where no source pixel lands.
 * Not read: output_layout, expand_coef, fixed_yaw .. fixed_vfov (the pose replaces them), fixed_cube_offcenter_*,
 * is_horizontal_offset and both scale factors (each plane renders at its own output size: no INTER_AREA resize); with a rig
 * also input_layout, input_expand_coef and both stereo formats (the rig is mono).
 *
 * Refused, with 0 and a message on stdout before any CUDA call: a NULL pose, a pose field that is not finite, hfov or vfov
 * outside (0, 179], enable_low_pass_filter != 0, an unknown interpolation_alg, and with a rig every refusal of the lens
 * calls about the rig itself (numLenses, calibration size, lens fields, distortion). */
/* Host only, no CUDA: the CV_32FC2 map (float32 [outputHeight][outputWidth][2]; with a rig NaN where uncovered) of one plane
 * of inputWidth x inputHeight, rig = NULL for the context's input.  T360B200_generateMapFromWarp(map, ..., T360_BORDER_WRAP,
 * or T360_BORDER_TRANSPARENT with a rig, index) plans it for a fixed pose: every frame entry point, the streamed host path
 * included, then gives the frames of T360B200_transformFrameRectilinearAsync bit for bit.  Returns 1; 0 (message) for the
 * refusals above, a NULL context or map, or non-positive sizes. */
int T360B200_rectilinearMap(const FrameTransformContext* ctx, const T360LensRig* rig, const T360Pose* pose, int inputWidth, int inputHeight,
                            int outputWidth, int outputHeight, float* map);
/* One frame of a rectilinear view, every plane in one gather launch: the arguments and the asynchronous contract of
 * T360B200_transformFrameAsync, plus `rig` (NULL: the context's input) and `pose`, both of which may change every frame.
 * Needs no plan: it works on a transform that was never planned as on one holding context or warp plans, and does not touch
 * them.  Takes the reader lock, so it is frame-exact against T360B200_reconfigure and T360B200_reconfigureAsync, and never
 * synchronises the device.  Returns 1 if everything was enqueued; 0 with a message on stdout, before any CUDA call, for the
 * refusals above, 0 or more than 3 planes, or an invalid plane description. */
int T360B200_transformFrameRectilinearAsync(VideoFrameTransform* transform, const T360LensRig* rig, const T360Pose* pose, int numPlanes,
                                            const uint8_t* const* deviceInputs, uint8_t* const* deviceOutputs, const int* inputWidths,
                                            const int* inputHeights, const int* inputPitches, const int* outputWidths,
                                            const int* outputHeights, const int* outputPitches, void* cudaStream);
/* ---- camera models ---------------------------------------------------------------------------------
 * The views above with another camera than the pinhole: a fisheye (equidistant) lens for dome masters and virtual
 * fisheye footage, a stereographic one for "little planet" shots, and Pannini for wide reframing that keeps vertical and
 * radial lines straight.  Everything is as for the rectilinear views (the pose, the rig, the input lookup and its border,
 * the pre-fill, the fields not read) except step 4, the ray q before the rotation.  With X = 2x - 1 and Y = 2y' - 1 (+-1
 * at the plane's outer pixel edges), the per-pose constants computed in double and stored as float, and every per-pixel
 * step in float rounded to nearest:
 *   PINHOLE        tx = tan(hfov / 2), ty = tan(vfov / 2); q = (X tx, Y ty, 1): the rectilinear view, bit for bit.
 *                  hfov, vfov in (0, 179];
 *   EQUIDISTANT    ax = hfov pi / 360, ay = vfov pi / 360; a = X ax, b = Y ay, rho = sqrt(a^2 + b^2),
 *                  q = (a S, b S, C) with S = sin rho / rho (1 at rho = 0) and C = cos rho: a pixel's angle to the axis is
 *                  proportional to its distance from the centre.  With hfov = vfov = 180 on a square plane the inscribed
 *                  circle is the front hemisphere (a dome master); the plane is full frame, no circular mask.  hfov, vfov
 *                  in (0, 360];
 *   STEREOGRAPHIC  sx = tan(hfov / 4), sy = tan(vfov / 4); a = X sx, b = Y sy, q = (2a, 2b, 1 - a^2 - b^2): the angle to
 *                  the axis is 2 atan(sqrt(a^2 + b^2)).  Looking at the nadir (pitch -90) with 200-300 degrees, a little
 *                  planet.  hfov, vfov in (0, 359];
 *   PANNINI        d = pannini in [0, 1], h = hfov / 2; xe = (d + 1) sin h / (d + cos h), ye = tan(vfov / 2); u = X xe,
 *                  w = Y ye, k = u^2 / (d + 1)^2, c = (-k d + sqrt(k^2 d^2 - (k + 1)(k d^2 - 1))) / (k + 1),
 *                  q = (u (d + c) / (d + 1), w (d + c) / (d + 1), c), proportional to (sin lon, tan lat, cos lon) with
 *                  c = cos lon (Sharpless et al.'s inverse; computed as k = (u / (d + 1))^2, c = (-k d + sqrt(1 + k (1 -
 *                  d^2))) / (k + 1)).  Vertical lines stay vertical and radial lines through the centre straight; d = 0
 *                  is the pinhole up to rounding, vfov is the field of the centre column.  hfov in (0, 359] with
 *                  d + cos(hfov / 2) > 0, vfov in (0, 179];
 *   EQUIRECT       ax = hfov pi / 360, ay = vfov pi / 360; lon = X ax, lat = Y ay, q = (cos lat sin lon, sin lat,
 *                  cos lat cos lon), with sin a = a S(a) and cos a = C(a) of the EQUIDISTANT row (S and C are even, and
 *                  |lon| <= pi): a latitude / longitude window.  With hfov = vfov = 180 it is a VR180 eye's half-equirect;
 *                  with hfov = 360, vfov = 180 and a zero pose the full equirect.  hfov in (0, 360], vfov in (0, 180].
 * Model 4 is not assigned and is refused (EQUIRECT was added after it had been pinned as refused).
 * Every model gives every pixel a ray, so a view of the context's input has no NaN in its map.
 *
 * Refused, with 0 and a message on stdout before any CUDA call: the refusals of the rectilinear views with the field
 * ranges above instead of (0, 179], a NULL camera, an unknown model, and for PANNINI a pannini that is not finite or lies
 * outside [0, 1], and d + cos(hfov / 2) <= 0. */
#define T360_CAMERA_PINHOLE 0
#define T360_CAMERA_EQUIDISTANT 1
#define T360_CAMERA_STEREOGRAPHIC 2
#define T360_CAMERA_PANNINI 3
#define T360_CAMERA_EQUIRECT 5
typedef struct T360Camera {
  int model;     /* T360_CAMERA_* */
  float pannini; /* d, read by T360_CAMERA_PANNINI only */
} T360Camera;
/* Host only, no CUDA: T360B200_rectilinearMap with `camera` (float32 [outputHeight][outputWidth][2]; with a rig NaN where
 * uncovered).  T360B200_generateMapFromWarp(map, ..., T360_BORDER_WRAP, or T360_BORDER_TRANSPARENT with a rig, index)
 * plans it for a fixed pose and camera, and then gives the frames of T360B200_transformFrameCameraAsync bit for bit.
 * Returns 1; 0 (message) for the refusals above, a NULL context or map, or non-positive sizes. */
int T360B200_cameraMap(const FrameTransformContext* ctx, const T360LensRig* rig, const T360Pose* pose, const T360Camera* camera,
                       int inputWidth, int inputHeight, int outputWidth, int outputHeight, float* map);
/* One frame of a camera view, every plane in one gather launch: T360B200_transformFrameRectilinearAsync with `camera`,
 * which may change every frame like the rig and the pose.  Needs no plan and does not touch the plans; takes the reader
 * lock; never synchronises the device.  Returns 1 if everything was enqueued; 0 with a message on stdout, before any CUDA
 * call, for the refusals above, 0 or more than 3 planes, or an invalid plane description. */
int T360B200_transformFrameCameraAsync(VideoFrameTransform* transform, const T360LensRig* rig, const T360Pose* pose, const T360Camera* camera,
                                       int numPlanes, const uint8_t* const* deviceInputs, uint8_t* const* deviceOutputs,
                                       const int* inputWidths, const int* inputHeights, const int* inputPitches, const int* outputWidths,
                                       const int* outputHeights, const int* outputPitches, void* cudaStream);
/* ---- anti-aliased camera views ----------------------------------------------------------------------
 * The camera views above sample the input at one point per output pixel, as cv::remap does, so a view much smaller than
 * the part of the input it covers (a dome master or a little planet of an 8K input, a thumbnail) aliases.  These calls
 * sample an input pyramid instead, each pixel at the level its footprint asks for (Williams 1983), the footprint from ray
 * differentials (Igehy 1999).  For each plane of inW x inH rendered at mapW x mapH:
 *   1. pyramid: level 0 is the input plane; level l + 1 is cv::resize(level l, (ceil(W_l / 2), ceil(H_l / 2)),
 *      INTER_AREA) (exact 2 x 2 cells as (sum + 2) >> 2, other sizes with OpenCV's area taps).  The plane's top level T is
 *      the largest l <= maxLevel whose sides are both >= 8 (0 if none), so a small chroma plane may stop before its luma
 *      plane.  Each plane has its own pyramid;
 *   2. footprint: X, Y as in steps 1-3 of the camera views; dX = 2 / mapW (4 / mapW with an LR output split) and dY =
 *      2 / mapH (4 / mapH with a TB split) are one column / row of one eye, computed on the host in double and stored as
 *      float (as dX / 2 and dY / 2).  rx = R (q(X + dX/2, Y) - q(X - dX/2, Y)) and ry = R (q(X, Y + dY/2) - q(X, Y - dY/2)),
 *      q the model's ray of step 4 and R the rotation of step 5.  With t the pixel's rotated ray, a = J rx and b = J ry,
 *      J the Jacobian at t of the input lookup the pixel takes, in level-0 pixels of the plane (the input eye re-pack's
 *      halving included):
 *        equirect    du = inW / 2pi (z dx - x dz) / (x^2 + z^2),
 *                    dv = inH / pi (dy (x^2 + z^2) - y (x dx + z dz)) / ((x^2 + y^2 + z^2) sqrt(x^2 + z^2));
 *        CUBEMAP_32  on the face the lookup picks, major component m and face coordinates a, b: du = inW / (6 e)
 *                    (da m - a dm) / m^2, dv = inH / (4 e) (db m - b dm) / m^2, e = input_expand_coef;
 *        a rig       on the lens the lookup picks, (X, Y, Z) its camera coordinates, rho = |(X, Y)|, theta = atan2(rho,
 *                    Z), s = theta_d / rho, theta_d' = 1 + 3 k1 theta^2 + 5 k2 theta^4 + 7 k3 theta^6 + 9 k4 theta^8:
 *                    drho = (X dX + Y dY) / rho, dtheta = (Z drho - rho dZ) / (rho^2 + Z^2), ds = (theta_d' dtheta -
 *                    s drho) / rho, dx' = s dX + X ds, dy' = s dY + Y ds, a = (fx / calibWidth inW dx', fy / calibHeight
 *                    inH dy'); at rho = 0 dx' = dX / Z, dy' = dY / Z (infinite for Z <= 0).
 *      Every step in float with + - * / and sqrt only (no libm function is differentiated), as the chains above;
 *   3. level and weight: rho^2 = max(a.a, b.b) (NaN-propagating); lambda = ((int32) bits(rho^2) - 0x3f800000) >> 16
 *      (arithmetic shift) + round(256 lodBias) (half away from zero, on the host): 1/2 log2 rho^2 in 1/256 of a level, with a
 *      log2 that is exact at powers of two and linear between them (at most 0.043 level off); lambda = 256 T where rho^2
 *      is not below +inf (an equirect's exact pole).  level = clamp(lambda >> 8, 0, T); the weight of the next level
 *      w = lambda & 255 where 0 <= lambda < 256 T, else 0;
 *   4. records: (px, py) the pixel's T360B200_cameraMap entry; at level l >= 1 px_l = ((px + 0.5) sx_l) - 0.5 and likewise
 *      py_l, sx_l = W_l / W_0 and sy_l = H_l / H_0 computed in double and stored as float, each step rounded to float (at
 *      level 0 the entry as it is).  Each entry is quantised as cv::remap quantises a CV_32FC2 map;
 *   5. pixel: a = the gather of level `level`, b = the gather of level + 1 where w > 0; the pixel is
 *      (a (256 - w) + b w + 128) >> 8.  Without a rig every level is sampled with BORDER_WRAP at its own size; with a rig
 *      BORDER_TRANSPARENT, and where one of the two samples is skipped the other stands alone, where both are the output
 *      keeps its bytes (the pre-fill of the camera views).
 * maxLevel = 0 is T360B200_transformFrameCameraAsync exactly (one launch, no pyramid); a frame whose planes all have T = 0
 * is too.  Else a frame takes T_max + 1 launches: one per pyramid level over every plane that has it, then the gather.
 * There is no planned path for a fixed pose: a plan carries one record per pixel.
 *
 * Refused, with 0 and a message on stdout before any CUDA call: every refusal of the camera views, a NULL minify, maxLevel
 * outside [0, 8], and a lodBias that is not finite or lies outside [-4, 4]. */
typedef struct T360Minify {
  int maxLevel;  /* 0..8: pyramid levels above the input; 0 = T360B200_transformFrameCameraAsync exactly */
  float lodBias; /* levels added to every pixel's level of detail, finite, in [-4, 4] (> 0 blurs, < 0 sharpens) */
} T360Minify;
/* Host only, no CUDA: the twin of one plane of inputWidth x inputHeight.  map0 / map1: float32 [outputHeight][outputWidth]
 * [2], the entry of each pixel in its level's pixels / in level + 1's pixels (NaN where the weight is 0); level: uint8
 * [outputHeight][outputWidth]; weight: uint16, w of step 3.  cv::remap of each level's entries over the pyramid
 * (cv::resize with INTER_AREA, repeated), combined as in step 5, gives the plane of T360B200_transformFrameCameraMipAsync
 * bit for bit.  maxLevel = 0 gives T360B200_cameraMap's map, level 0 and weight 0.  Returns 1; 0 (message) for the refusals
 * above, a NULL context or array, or non-positive sizes. */
int T360B200_cameraMipMaps(const FrameTransformContext* ctx, const T360LensRig* rig, const T360Pose* pose, const T360Camera* camera,
                           const T360Minify* minify, int inputWidth, int inputHeight, int outputWidth, int outputHeight, float* map0,
                           float* map1, uint8_t* level, uint16_t* weight);
/* One frame of an anti-aliased camera view: T360B200_transformFrameCameraAsync's arguments and asynchronous contract, plus
 * `minify`, which may change every frame like the rig, pose and camera.  Needs no plan and does not touch the plans; takes
 * the reader lock; never synchronises the device.  The pyramids live in per-stream scratch of about a third of the input
 * planes, grown on demand.  Returns 1 if everything was enqueued; 0 with a message on stdout, before any CUDA call, for
 * the refusals above, 0 or more than 3 planes, or an invalid plane description. */
int T360B200_transformFrameCameraMipAsync(VideoFrameTransform* transform, const T360LensRig* rig, const T360Pose* pose,
                                          const T360Camera* camera, const T360Minify* minify, int numPlanes,
                                          const uint8_t* const* deviceInputs, uint8_t* const* deviceOutputs, const int* inputWidths,
                                          const int* inputHeights, const int* inputPitches, const int* outputWidths,
                                          const int* outputHeights, const int* outputPitches, void* cudaStream);
/* ---- anisotropic camera views ------------------------------------------------------------------------------------
 * The anti-aliased views above pick one level per pixel from the longer footprint axis, so where the footprint is a long
 * thin ellipse (a little planet's outer ring, the rim of a wide dome, an equirect camera near its poles, any oblique
 * view) the short axis is blurred as much as the long one.  These calls read the pyramid with N probes per pixel spread
 * along its longer axis, each at the level of max(long / N, short): the probes along the major axis of hardware
 * anisotropic filtering (McCormack et al., Feline, 1999), with the longer screen-axis derivative in place of the
 * ellipse's true major axis.  Steps 1-2 of the anti-aliased views (the pyramid; the footprint a, b of the centre ray)
 * are unchanged; aa = a.a and bb = b.b as there.  Each step below is computed bit for bit alike on host and device:
 *   1. probe count and level: where aa or bb is not below +inf (an exact pole, NaN), step 3 of the anti-aliased views
 *      with N = 1.  Otherwise, with L(x) = ((int32) bits(x) - 0x3f800000) >> 16: lmaj = L(max(aa, bb)), lmin =
 *      L(min(aa, bb)), e = min((lmaj - lmin + 255) >> 8, log2 maxProbes), N = 1 << e, lambda = max(lmaj - 256 e, lmin) +
 *      round(256 lodBias); level and next-level weight follow from lambda as in step 3 (clamped to [0, T], w = lambda &
 *      255 inside).  A zero aa or bb gives the largest N.  The footprint is taken wherever T > 0 or maxProbes > 1, so
 *      maxLevel = 0 with maxProbes > 1 supersamples level 0 along the long axis;
 *   2. probe rays: the axis is the column axis where aa >= bb, the row axis otherwise.  Probe k (0..N-1) sits at o_k =
 *      (2k + 1 - N) / N (exact in float): Xk = X + o_k dX / 2 on the column axis, Yk = Y + o_k dY / 2 on the row axis,
 *      each operation rounded to float (with N = 1 the centre ray itself, no offset added).  Each probe takes the camera
 *      view's whole chain (the model's ray, the pose, then the context's input lookup with the pixel's eye or the rig's
 *      closer lens), so on cube-map input each probe picks its own face and on a rig its own lens.  Its entries at level
 *      and level + 1 are step 4's; all probes share the pixel's level and weight;
 *   3. pixel: v_k is step 5 of the anti-aliased views on probe k's entries.  BORDER_WRAP (the context's input): (sum v_k +
 *      N / 2) >> e.  BORDER_TRANSPARENT (a rig): a probe whose two samples are both skipped drops out, and with n probes
 *      left the pixel is (sum v_k + n / 2) / n (integer division); n = 0 keeps the output's bytes (the pre-fill).
 * maxProbes = 1 gives T360B200_transformFrameCameraMipAsync byte for byte (records, levels, weights, frames), and with
 * maxLevel = 0 T360B200_transformFrameCameraAsync.  A frame takes the camera-mip call's launches: T_max + 1 (one per
 * pyramid level, then the gather), or one without a pyramid.  The probe loop multiplies a pixel's chain and gathers by
 * its N.  There is no planned path: a plan carries one record per pixel.
 *
 * Refused, with 0 and a message on stdout before any CUDA call: every refusal of T360B200_transformFrameCameraMipAsync,
 * then a maxProbes other than 1, 2, 4, 8 or 16. */
/* Host only, no CUDA: the twin of one plane of inputWidth x inputHeight.  map0 / map1: float32 [maxProbes][outputHeight]
 * [outputWidth][2], probe k's entry in its level's pixels / in level + 1's pixels (map1 NaN where the weight is 0; both
 * NaN for k >= N); level: uint8 [outputHeight][outputWidth]; weight: uint16, the next level's weight; probes: uint8, N.
 * cv::remap of each probe's entries over the pyramid, each probe's levels blended as in step 5 of the anti-aliased views,
 * then the probes averaged as in step 3, gives the plane of T360B200_transformFrameCameraAnisoAsync bit for bit.  With
 * maxProbes = 1, probe 0 is T360B200_cameraMipMaps' arrays.  Returns 1; 0 (message) for the refusals above, a NULL context
 * or array, or non-positive sizes. */
int T360B200_cameraAnisoMaps(const FrameTransformContext* ctx, const T360LensRig* rig, const T360Pose* pose, const T360Camera* camera,
                             const T360Minify* minify, int maxProbes, int inputWidth, int inputHeight, int outputWidth, int outputHeight,
                             float* map0, float* map1, uint8_t* level, uint16_t* weight, uint8_t* probes);
/* One frame of an anisotropic camera view: T360B200_transformFrameCameraMipAsync's arguments and asynchronous contract,
 * plus maxProbes, which may change every frame like the rig, pose, camera and minify.  Needs no plan and does not touch
 * the plans; takes the reader lock; never synchronises the device; the pyramids use the camera-mip call's scratch.
 * Returns 1 if everything was enqueued; 0 with a message on stdout, before any CUDA call, for the refusals above, 0 or
 * more than 3 planes, or an invalid plane description. */
int T360B200_transformFrameCameraAnisoAsync(VideoFrameTransform* transform, const T360LensRig* rig, const T360Pose* pose,
                                            const T360Camera* camera, const T360Minify* minify, int maxProbes, int numPlanes,
                                            const uint8_t* const* deviceInputs, uint8_t* const* deviceOutputs, const int* inputWidths,
                                            const int* inputHeights, const int* inputPitches, const int* outputWidths,
                                            const int* outputHeights, const int* outputPitches, void* cudaStream);
/* ---- camera views of a lens rig with photometry ----------------------------------------------------------
 * The camera views above take a rig's hard, uncorrected seam, so a view panned across the seam of a dual-fisheye clip
 * shows the step the lens photometry removes from sphere outputs.  This call gives the rectilinear view (the pinhole
 * camera, bit for bit), the other camera models and the anti-aliased views of a rig the photometry and the seam of
 * T360B200_transformFrameLensPhotoAsync.  Per output pixel of each plane:
 *   1. ray: steps 1-5 of the camera views (X, Y, the model's ray q, the pose's rotation); the rig is mono, so there is no
 *      eye split;
 *   2. lenses: the lens photometry's per-lens step on that ray: each lens's entry (the lens calls' projection, NaN where
 *      the lens does not cover the ray), its Gq, and the seam weight w of lens 1 (0 or 256 from the closer lens with
 *      seamWidth = 0; the feathered seam's w otherwise);
 *   3. pyramid (minify not NULL and the plane's top level T > 0; the pyramid of the anti-aliased views, step 1): each lens
 *      whose entry is finite takes its own footprint, steps 2-3 of the anti-aliased views with the Jacobian of that lens
 *      (not the closer lens's), so its own level and next-level weight, and its entries at those levels (step 4).  A lens
 *      that does not cover the ray has level 0 and weight 0.  A pixel in the seam's belt may so gather four windows, two
 *      lenses at two levels each;
 *   4. combining: each lens's sample S_i is the blend of its two levels (step 5 of the anti-aliased views; its level-0
 *      sample alone without a pyramid), then S_i' = s' of the lens photometry with that lens's Gq and Oq, then the seam
 *      combines S_0' and S_1' exactly as T360B200_transformFrameLensPhotoAsync does.  Samples that BORDER_TRANSPARENT skips
 *      stay skipped; the pre-fill and the output bytes that are kept are the lens calls' (chroma 128, luma the caller's);
 *   5. statistics: deviceStats (device memory, NULL: none) receives the lens photometry's [numPlanes][6] sums over S_0'
 *      and S_1', where both lenses cover the ray and neither sample is skipped, zeroed with a memset in stream order.
 *      Every output pixel weighs the same.
 * With the identity photometry (vignetting 0, gain 1, offset 0) and seamWidth = 0 the frame is
 * T360B200_transformFrameCameraAsync's with the rig byte for byte without a pyramid (minify NULL or maxLevel 0), and
 * T360B200_transformFrameCameraMipAsync's with the rig with one.  Taking statistics never changes the frame.  The limits of
 * the lens photometry (no transfer function, one falloff for every plane, centred; gains chosen by the caller) and of the
 * anti-aliased views (an isotropic footprint; a lens's dark surround reaches its rim texels at coarse levels) carry over.
 * A frame takes one launch, or T_max + 1 with a pyramid (one per level, then the gather), plus the memset with statistics.
 *
 * Refused, with 0 and a message on stdout before any CUDA call: a NULL rig (the photometry is per lens); every refusal of
 * T360B200_transformFrameCameraAsync with a rig; a seamWidth that is negative, not finite or in (0, 0.01), and with
 * seamWidth > 0 a rig of one lens or a seamWidth above 180; every refusal of the photometry of
 * T360B200_transformFrameLensPhotoAsync; and where minify is not NULL every refusal of T360B200_transformFrameCameraMipAsync
 * about it, and (frame call only) with maxLevel > 0 an input plane side above 131070. */
/* Host only, no CUDA: the twin of plane `plane` (0..2) of inputWidth x inputHeight, one lens (0 or 1) per call.  map0,
 * map1, level, weight: T360B200_cameraMipMaps' four arrays for that lens (the entry in its level's pixels, in level + 1's
 * pixels, the level, the next level's weight); NaN entries, level 0 and weight 0 where the lens does not cover the ray.
 * gain: that lens's Gq (uint16, 0 where it does not cover the ray); seamWeight: w of step 2 (uint16).  Both lenses'
 * entries are given wherever they cover the ray, with either seam.  cv::remap of each level's entries over the pyramid,
 * blended as in step 4 per lens, then s', then the seam (the other alone where one is skipped) gives the frame's plane bit
 * for bit; the statistics are the sums over the pixels where both lenses' map0 entries are finite and neither sample is
 * skipped.  With the identity photometry and seamWidth = 0 the closer lens's arrays are T360B200_cameraMipMaps' with the rig
 * where it covers the ray (T360B200_cameraMap's entries without a pyramid) and its gain 4096.  Returns 1; 0 (message) for
 * the refusals above, a lens outside 0..1, a plane outside 0..2, a NULL context or array, or non-positive sizes. */
int T360B200_cameraPhotoMaps(const FrameTransformContext* ctx, const T360LensRig* rig, const T360RigPhotometry* photometry, float seamWidth,
                             const T360Pose* pose, const T360Camera* camera, const T360Minify* minify /* NULL: no pyramid */, int lens,
                             int plane, int inputWidth, int inputHeight, int outputWidth, int outputHeight, float* map0, float* map1,
                             uint8_t* level, uint16_t* weight, uint16_t* gain, uint16_t* seamWeight);
/* One frame of a camera view of a lens rig with photometry, every plane in one gather launch after the pyramid's: the
 * arguments and asynchronous contract of T360B200_transformFrameCameraMipAsync with a rig, plus photometry, seamWidth and
 * deviceStats; every argument may change every frame.  Needs no plan and does not touch the plans; takes the reader lock;
 * never synchronises the device.  There is no planned path: a plan carries one record per pixel.  Returns 1 if everything
 * was enqueued; 0 with a message on stdout, before any CUDA call, for the refusals above, 0 or more than 3 planes, or an
 * invalid plane description. */
int T360B200_transformFrameCameraPhotoAsync(VideoFrameTransform* transform, const T360LensRig* rig, const T360RigPhotometry* photometry,
                                            float seamWidth, const T360Pose* pose, const T360Camera* camera,
                                            const T360Minify* minify /* NULL: no pyramid */, unsigned long long* deviceStats /* NULL: none */,
                                            int numPlanes, const uint8_t* const* deviceInputs, uint8_t* const* deviceOutputs,
                                            const int* inputWidths, const int* inputHeights, const int* inputPitches,
                                            const int* outputWidths, const int* outputHeights, const int* outputPitches, void* cudaStream);
/* ---- camera views of a stereo rig ---------------------------------------------------------------------------------
 * A stereo fisheye rig (a VR180 camera, a dual-fisheye cinema lens, a pair of action cameras) has two lenses that both
 * look forward, lens 0 the left eye and lens 1 the right eye, their circles anywhere in the frame (cx, cy: some cameras put
 * the left eye's circle on the right).  This call renders one view per eye with the camera views' pose and models and the
 * photometry and pyramid of T360B200_transformFrameCameraPhotoAsync.  With the EQUIRECT model at 180 x 180 and an LR
 * output, each eye is a VR180 half-equirect.  Per output pixel of each plane:
 *   1. eye split: the context's output_stereo_format, whatever input_stereo_format says: LR side by side (x folded), TB
 *      stacked (y folded, the lower eye's y flipped with vflip), MONO eye 0 alone.  The footprint's dX and dY are one column and
 *      row of one eye, as in the anti-aliased views;
 *   2. ray: steps 1-5 of the camera views; the same pose for both eyes (each lens's own extrinsics carry the stereo
 *      rectification);
 *   3. lens: eye e takes lens e and only lens e.  Where lens e does not cover the ray, or its samples are skipped
 *      (BORDER_TRANSPARENT), the pixel keeps its bytes (the pre-fill: chroma 128, luma the caller's); it never falls back to
 *      the other eye's lens, which would show the wrong parallax;
 *   4. pyramid, photometry, statistics: steps 3-5 of T360B200_transformFrameCameraPhotoAsync with lens e's footprint, its
 *      two levels and its Gq and Oq; s' of lens e is the pixel.  With deviceStats each pixel also gathers the other lens
 *      for the statistics only, so the sums run over the output pixels of both eyes whose ray both lenses cover where
 *      neither sample is skipped: they measure the exposure and colour mismatch between the eyes over their common field
 *      (near objects add parallax noise to them: a scene point closer than a few metres lies at other pixels in the two
 *      eyes).
 * With MONO output and no statistics the frame is T360B200_transformFrameCameraPhotoAsync's with the one-lens rig {lens
 * 0} and seamWidth 0, byte for byte, with and without a pyramid.  With the identity photometry and no pyramid, the twin's
 * two map0 arrays combined by eye (lens 1's where eyeWeight is 256) and planned with T360B200_generateMapFromWarp(...,
 * T360_BORDER_TRANSPARENT) give the frame through T360B200_transformFrameAsync for a fixed pose.  A frame takes one launch,
 * or T_max + 1 with a pyramid, plus the memset with statistics.
 *
 * Refused, with 0 and a message on stdout before any CUDA call: a NULL rig or numLenses other than 2; an
 * output_stereo_format other than TB, LR or MONO; every refusal of T360B200_transformFrameCameraPhotoAsync except the seam's;
 * and (frame call only) with maxLevel > 0 an input plane side above 131070. */
/* Host only, no CUDA: the twin of plane `plane` (0..2) of inputWidth x inputHeight, one lens (0 or 1) per call.  map0,
 * map1, level, weight, gain: T360B200_cameraPhotoMaps' arrays for that lens (NaN entries, level 0, weight 0 and gain 0
 * where it does not cover the ray), given wherever it covers the ray, in both eyes.  eyeWeight (uint16): 0 on eye-0
 * pixels, 256 on eye-1 pixels.  So the oracle composite of T360B200_cameraPhotoMaps, with eyeWeight as the seam weight,
 * gives the frame bit for bit, and its statistics the frame's.  Returns 1; 0 (message) for the refusals above, a lens
 * outside 0..1, a plane outside 0..2, a NULL context or array, or non-positive sizes. */
int T360B200_stereoCameraMaps(const FrameTransformContext* ctx, const T360LensRig* rig, const T360RigPhotometry* photometry, const T360Pose* pose,
                              const T360Camera* camera, const T360Minify* minify /* NULL: no pyramid */, int lens, int plane, int inputWidth,
                              int inputHeight, int outputWidth, int outputHeight, float* map0, float* map1, uint8_t* level, uint16_t* weight,
                              uint16_t* gain, uint16_t* eyeWeight);
/* One frame of a camera view of a stereo rig, every plane in one gather launch after the pyramid's: the arguments and
 * asynchronous contract of T360B200_transformFrameCameraPhotoAsync without seamWidth; every argument may change every
 * frame.  Needs no plan and does not touch the plans; takes the reader lock; never synchronises the device.  Returns 1 if
 * everything was enqueued; 0 with a message on stdout, before any CUDA call, for the refusals above, 0 or more than 3
 * planes, or an invalid plane description. */
int T360B200_transformFrameStereoCameraAsync(VideoFrameTransform* transform, const T360LensRig* rig, const T360RigPhotometry* photometry,
                                             const T360Pose* pose, const T360Camera* camera, const T360Minify* minify /* NULL: no pyramid */,
                                             unsigned long long* deviceStats /* NULL: none */, int numPlanes, const uint8_t* const* deviceInputs,
                                             uint8_t* const* deviceOutputs, const int* inputWidths, const int* inputHeights,
                                             const int* inputPitches, const int* outputWidths, const int* outputHeights,
                                             const int* outputPitches, void* cudaStream);
/* ---- rolling-shutter lens rigs ------------------------------------------------------------------------------------
 * A CMOS sensor reads its rows over milliseconds, not at one instant, so a camera that turns during the readout records
 * each row from another orientation: the per-frame orientation removes the shake between frames and leaves the shear and
 * wobble within the frame.  These calls give the photometric lens and camera calls a rig motion over the readout.
 *
 * Readout time: lens i's point at normalised calibration coordinates u = (fx x' + cx + 0.5) / calibWidth, v = (fy y' + cy
 * + 0.5) / calibHeight (the lens projection above, before the plane's size is applied; the same for every plane) is read
 * at t = (a u + b v) + c, each step in float rounded to nearest, clamped to [0, 1] (a NaN gives 0), with (a, b, c) =
 * readout[i].  (0, 1, 0): top to bottom over the whole frame; (0, -1, 1): bottom to top; (2, 0, -1): left to right over
 * the right half of a side-by-side frame (a sensor mounted at 90 degrees).
 * Sample matrices: the rig at t_k = k / (N - 1), k = 0..N-1 (N = numSamples), is turned by delta[k] from where the frame's
 * orientation (sphere outputs) or pose (camera views) puts it: lens i's extrinsic rotation becomes R_ik = Rot(delta[k]) R_i,
 * Rot(yaw, pitch, roll) = Ry(yaw) Rx(-pitch) Rz(roll) as for the lens extrinsics, computed in double; M_ik is R_ik^T with
 * its y row negated (the lens projection's M), stored as float.  A zero delta gives the lens's own M bit for bit.
 * Per pixel and lens, for the direction d the camera or sphere chain hands to the lens:
 *   1. t = 0.5;
 *   2. three projections, each: s = t (N - 1), k = min(floor(s), N - 2), f = s - k; M = M_ik + f (M_i,k+1 - M_ik) per
 *      entry, each step rounded (an entry equal in both neighbours is taken as it is, so a -0 entry stays -0); the lens
 *      projection with M; where it covers d, t becomes the readout time of its (u, v), where it does not t stays;
 *   3. the third projection is the lens's entry, theta, coverage and theta_d (for Gq).
 * So the fixed point t = readout(project(M(t) d)) is refined twice, a fixed count, and host and device agree bit for bit.
 * The hard seam picks the lens with the larger Z under each lens's M at t = 0.5; the feathered seam's weight takes each
 * lens's third-projection theta; the statistics' overlap is where both third projections cover d.  With a pyramid, a lens's
 * footprint is its Jacobian (the anti-aliased views' step 2) with its third-projection M: the motion's own stretch of the
 * footprint is left out.  Matrix interpolation is part of the contract, not an approximation of a slerp (it differs from
 * one at third order in the angle between neighbouring samples).
 * All-zero deltas give the records, frames and statistics of the photometric calls bit for bit, for any readout and N.
 *
 * Refused, with 0 and a message on stdout before any CUDA call, after every refusal of the call extended (and, for the
 * host twins, before their index, array and size checks): a NULL motion, numSamples outside [2, 16], a delta angle that is
 * not finite or lies outside [-30, 30] degrees, and a readout field of a lens that is read (readout[1] with two lenses)
 * that is not finite.  The stereo camera call takes no motion. */
typedef struct T360LensReadout {
  float a, b, c; /* readout time of a lens point: t = a u + b v + c, clamped to [0, 1] */
} T360LensReadout;
typedef struct T360RigMotion {
  int numSamples;             /* 2..16 */
  T360Orientation delta[16];  /* the rig at readout time t_k = k / (numSamples - 1), turned from where it was for the
                                 frame's orientation / pose; degrees, each in [-30, 30] */
  T360LensReadout readout[2]; /* readout[1] is read only with two lenses */
} T360RigMotion;
/* Host only, no CUDA: the host twin of T360B200_transformFrameLensMotionAsync: T360B200_lensPhotoMaps' arguments and arrays
 * with `motion`.  The oracle composite of T360B200_lensPhotoMaps' arrays (cv::remap of each map, s', the seam) gives the
 * frame's plane and statistics bit for bit.  Returns 1; 0 (message) for the refusals above, a plane outside 0..2, a NULL
 * array or non-positive sizes. */
int T360B200_lensMotionMaps(const FrameTransformContext* ctx, const T360LensRig* rig, const T360RigPhotometry* photometry, float seamWidth,
                            const T360Orientation* orientation, const T360RigMotion* motion, int plane, int inputWidth, int inputHeight,
                            int outputWidth, int outputHeight, float* map0, float* map1, uint16_t* weight, uint16_t* gain0, uint16_t* gain1);
/* One frame of a lens rig with photometry and a rig motion over the readout, every plane in one gather launch:
 * T360B200_transformFrameLensPhotoAsync's arguments and asynchronous contract plus `motion`, which may change every frame.
 * With the identity photometry it is the motion version of the lens (seamWidth 0) and blend calls.  The sample table
 * (numLenses x numSamples x 9 floats) is uploaded in stream order from page-locked memory.  Returns 1 if everything was
 * enqueued; 0 with a message on stdout, before any CUDA call, for the refusals above, 0 or more than 3 planes, or an
 * invalid plane description. */
int T360B200_transformFrameLensMotionAsync(VideoFrameTransform* transform, const T360LensRig* rig, const T360RigPhotometry* photometry,
                                           float seamWidth, const T360Orientation* orientation, const T360RigMotion* motion,
                                           unsigned long long* deviceStats, int numPlanes, const uint8_t* const* deviceInputs,
                                           uint8_t* const* deviceOutputs, const int* inputWidths, const int* inputHeights,
                                           const int* inputPitches, const int* outputWidths, const int* outputHeights,
                                           const int* outputPitches, void* cudaStream);
/* Host only, no CUDA: the host twin of T360B200_transformFrameCameraMotionAsync: T360B200_cameraPhotoMaps' arguments and
 * arrays with `motion` after minify.  Returns 1; 0 (message) for the refusals above, a lens outside 0..1, a plane outside
 * 0..2, a NULL array or non-positive sizes. */
int T360B200_cameraMotionMaps(const FrameTransformContext* ctx, const T360LensRig* rig, const T360RigPhotometry* photometry, float seamWidth,
                              const T360Pose* pose, const T360Camera* camera, const T360Minify* minify /* NULL: no pyramid */,
                              const T360RigMotion* motion, int lens, int plane, int inputWidth, int inputHeight, int outputWidth,
                              int outputHeight, float* map0, float* map1, uint8_t* level, uint16_t* weight, uint16_t* gain,
                              uint16_t* seamWeight);
/* One frame of a camera view of a lens rig with photometry and a rig motion over the readout (rectilinear views, every
 * camera model, the pyramid, the seam and the statistics): T360B200_transformFrameCameraPhotoAsync's arguments and
 * asynchronous contract plus `motion` after minify.  With one lens, this undistorts, stabilises and corrects the readout
 * of an action camera in one pass.  Returns 1 if everything was enqueued; 0 with a message on stdout, before any CUDA
 * call, for the refusals above, 0 or more than 3 planes, or an invalid plane description. */
int T360B200_transformFrameCameraMotionAsync(VideoFrameTransform* transform, const T360LensRig* rig, const T360RigPhotometry* photometry,
                                             float seamWidth, const T360Pose* pose, const T360Camera* camera,
                                             const T360Minify* minify /* NULL: no pyramid */, const T360RigMotion* motion,
                                             unsigned long long* deviceStats /* NULL: none */, int numPlanes,
                                             const uint8_t* const* deviceInputs, uint8_t* const* deviceOutputs, const int* inputWidths,
                                             const int* inputHeights, const int* inputPitches, const int* outputWidths,
                                             const int* outputHeights, const int* outputPitches, void* cudaStream);
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
/* counts[0] = gather jobs staged through TMA into shared memory, counts[1] = gather jobs reading through L1 (border jobs),
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
