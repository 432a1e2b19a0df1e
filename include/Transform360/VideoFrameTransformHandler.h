/* transform360-b200: the drop-in C-ABI.
 *
 * These four entry points are exactly what the reference's ffmpeg filter binds
 * (reference Transform360/Library/VideoFrameTransformHandler.h:22-47, implemented in
 * VideoFrameTransformHandler.cpp:18-64; called from vf_transform360.c:141, 157-158, 334, 383-394).
 * Same names, same argument order and meaning, same 1 = ok / 0 = failure convention, no exception
 * ever crosses the boundary, error text goes to stdout like the reference's printf.
 *
 * What differs is behind them: planning runs on the host, every per-frame pixel is produced by
 * hand-written sm_90a CUDA kernels (no OpenCV, no CPU fallback: without a usable CUDA device
 * generateMapForPlane / transformFramePlane print the CUDA error and return 0).
 */
#ifndef TRANSFORM360_B200_VIDEOFRAMETRANSFORMHANDLER_H
#define TRANSFORM360_B200_VIDEOFRAMETRANSFORMHANDLER_H

#include "VideoFrameTransformHelper.h"

#ifdef __cplusplus
extern "C" {
#endif

#ifdef __cplusplus
typedef class VideoFrameTransform VideoFrameTransform;
#else
typedef struct VideoFrameTransform VideoFrameTransform;
#endif

/* Replaces handler.cpp:18-20.  Copies *ctx; the caller keeps ownership of ctx.  Never touches the GPU. */
VideoFrameTransform* VideoFrameTransform_new(FrameTransformContext* ctx);

/* Replaces handler.cpp:22-24.  NULL-safe.  Releases the device plan, staging buffers and stream. */
void VideoFrameTransform_delete(VideoFrameTransform* transform);

/* Replaces handler.cpp:26-40 -> VideoFrameTransform::generateMapForPlane (cpp:504-576).
 * Builds and uploads the plan for one plan index (0 = luma-sized planes, 1 = chroma-sized planes):
 * the per-pixel sampling plan equivalent to the reference's CV_32FC2 warp map, and, when
 * enable_low_pass_filter is set, the tile table and Gaussian taps of the segmented low-pass.
 * Calling it again for the same index replaces the plan (the reference appends duplicate tiles). */
int VideoFrameTransform_generateMapForPlane(VideoFrameTransform* transform, int inputWidth, int inputHeight,
                                            int outputWidth, int outputHeight, int transformMatPlaneIndex);

/* Replaces handler.cpp:42-64 -> VideoFrameTransform::transformFramePlane (cpp:1319-1351).
 * inputData / outputData: 8-bit planes, row pitch = *WidthWithPadding bytes, only `width` bytes per row
 * are read / written.  Host pointers (what ffmpeg passes) are staged through the GPU inside the call;
 * CUDA device pointers are detected and used in place.  Synchronous: the output is complete on return. */
int VideoFrameTransform_transformFramePlane(VideoFrameTransform* transform, uint8_t* inputData, uint8_t* outputData,
                                            int inputWidth, int inputHeight, int inputWidthWithPadding,
                                            int outputWidth, int outputHeight, int outputWidthWithPadding,
                                            int transformMatPlaneIndex, int imagePlaneIndex);

#ifdef __cplusplus
}
#endif

#endif /* TRANSFORM360_B200_VIDEOFRAMETRANSFORMHANDLER_H */
