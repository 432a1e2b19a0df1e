/* vf_transform360_cuda.c -- libavfilter glue for CUDA frames on top of transform360-b200.
 *
 * The reference ships Transform360/vf_transform360.c: a software-frame filter that calls
 * VideoFrameTransform_transformFramePlane once per plane with host pointers (vf:338-402).  That file links against this
 * library unchanged (tests/test_filter_surface.py).  This file is the variant for pipelines whose frames already live
 * on the GPU (NVDEC -> ... -> NVENC): frames of AV_PIX_FMT_CUDA with sw_format yuv420p or gray8 go through
 * T360B200_transformFrameAsync -- every plane of the frame in one call, device to device, on the device context's
 * stream -- so no pixel crosses PCIe.
 *
 *   ffmpeg -hwaccel cuda -hwaccel_output_format cuda -i in.mp4 \
 *          -vf "scale_cuda=format=yuv420p,transform360_cuda=cube_edge_length=1280:interpolation_alg=cubic" -c:v h264_nvenc out.mp4
 *
 * Options carry the names, defaults and ranges of the reference filter's table (vf:407-987) and the output size follows
 * its config_output (vf:167-304); they write straight into the FrameTransformContext handed to VideoFrameTransform_new.
 * Differences, on purpose: "size=WxH" is honoured (the reference accepts and then ignores it, vf:306-326); "sync=0" lets
 * the frame travel downstream without a stream synchronisation (consumers on the same stream need none).  The view and
 * quality options are also runtime commands (sendcmd, zmq; see t360_process_command).
 * To build inside an ffmpeg tree: copy to libavfilter/, add `extern const AVFilter ff_vf_transform360_cuda;` to
 * allfilters.c and `OBJS-$(CONFIG_TRANSFORM360_CUDA_FILTER) += vf_transform360_cuda.o` to the Makefile, link
 * -lTransform360 (INTEGRATION.md).
 */
#include <stdio.h>
#include <string.h>

#include "avfilter.h"
#include "internal.h"
#include "libavutil/hwcontext.h"
#include "libavutil/hwcontext_cuda_internal.h"
#include "libavutil/opt.h"
#include "libavutil/pixdesc.h"
#include "video.h"

#include "Transform360/VideoFrameTransformHandler.h"
#include "Transform360/VideoFrameTransformHelper.h"
#include "transform360_b200.h"

typedef struct T360CudaContext {
  const AVClass* av_class;
  FrameTransformContext params; /* the option table writes here */
  char* out_w;
  char* out_h;
  char* out_size;
  int cube_edge_length, max_cube_edge_length;
  int max_output_w, max_output_h; /* accepted for compatibility; the reference never reads them either */
  int sync;

  VideoFrameTransform* transform;
  int maps_ready;
  int sw_format, num_planes;
  AVBufferRef* out_frames;
  AVCUDADeviceContext* cuda;
} T360CudaContext;

static int plane_extent(int full, int plane, int log2_sub) { return plane ? -((-full) >> log2_sub) : full; }

static int parse_extent(const char* text, int* value) {
  char* end = NULL;
  double v = text ? strtod(text, &end) : 0;
  if (!text || end == text || v < 1 || v > 32768) return AVERROR(EINVAL);
  *value = (int)v;
  return 0;
}

static av_cold int t360_init(AVFilterContext* ctx) {
  T360CudaContext* s = ctx->priv;
  if (s->out_size && (s->out_w || s->out_h)) {
    av_log(ctx, AV_LOG_ERROR, "give either size or w/h, not both\n");
    return AVERROR(EINVAL);
  }
  if (!s->out_w != !s->out_h) {
    av_log(ctx, AV_LOG_ERROR, "w and h go together\n");
    return AVERROR(EINVAL);
  }
  return 0;
}

static av_cold void t360_uninit(AVFilterContext* ctx) {
  T360CudaContext* s = ctx->priv;
  if (s->transform) VideoFrameTransform_delete(s->transform);
  s->transform = NULL;
  s->maps_ready = 0;
  av_buffer_unref(&s->out_frames);
}

static int t360_query_formats(AVFilterContext* ctx) {
  static const enum AVPixelFormat only_cuda[] = {AV_PIX_FMT_CUDA, AV_PIX_FMT_NONE};
  return ff_set_common_formats(ctx, ff_make_format_list((const int*)only_cuda));
}

/* stereo guesses, cube edge, output extent: the rules of vf:182-301 */
static int decide_output_size(AVFilterContext* ctx, int in_w, int in_h, int* out_w, int* out_h) {
  T360CudaContext* s = ctx->priv;
  FrameTransformContext* p = &s->params;
  if (p->input_stereo_format == STEREO_FORMAT_GUESS) {
    const int aspect = in_w / in_h;
    p->input_stereo_format = aspect == 1 ? STEREO_FORMAT_TB : aspect == 4 ? STEREO_FORMAT_LR : STEREO_FORMAT_MONO;
  }
  if (p->output_stereo_format == STEREO_FORMAT_GUESS) {
    if (p->input_stereo_format == STEREO_FORMAT_MONO) p->output_stereo_format = STEREO_FORMAT_MONO;
    else p->output_stereo_format = p->output_layout == LAYOUT_CUBEMAP_23_OFFCENTER ? STEREO_FORMAT_LR : STEREO_FORMAT_TB;
  }
  int edge = s->cube_edge_length;
  if (s->max_cube_edge_length > 0) {
    edge = in_w / (p->input_stereo_format == STEREO_FORMAT_LR ? 8 : 4);
    if (edge > s->max_cube_edge_length) edge = s->max_cube_edge_length;
  }
  edge &= ~15; /* macroblocks must not straddle cube faces */
  s->cube_edge_length = edge;
  int w = *out_w, h = *out_h; /* the link's own size when nothing below decides */
  if (edge > 0 && p->output_layout == LAYOUT_CUBEMAP_32) {
    w = 3 * edge;
    h = 2 * edge;
  } else if (edge > 0 && p->output_layout == LAYOUT_CUBEMAP_23_OFFCENTER) {
    w = 2 * edge;
    h = 3 * edge;
  } else if (edge <= 0) {
    int rc = 0;
    if (s->out_size) {
      if (sscanf(s->out_size, "%dx%d", &w, &h) != 2 || w < 1 || h < 1) rc = AVERROR(EINVAL);
    } else {
      rc = parse_extent(s->out_w, &w);
      if (!rc) rc = parse_extent(s->out_h, &h);
    }
    if (rc) {
      av_log(ctx, AV_LOG_ERROR, "no usable output size: set cube_edge_length, size or w and h\n");
      return rc;
    }
  }
  if (p->output_stereo_format == STEREO_FORMAT_TB) h *= 2;
  else if (p->output_stereo_format == STEREO_FORMAT_LR) w *= 2;
  *out_w = w;
  *out_h = h;
  return 0;
}

static int t360_config_output(AVFilterLink* outlink) {
  AVFilterContext* ctx = outlink->src;
  AVFilterLink* inlink = ctx->inputs[0];
  T360CudaContext* s = ctx->priv;
  int w = outlink->w, h = outlink->h;
  int rc = decide_output_size(ctx, inlink->w, inlink->h, &w, &h);
  if (rc) return rc;
  outlink->w = w;
  outlink->h = h;

  if (!inlink->hw_frames_ctx) {
    av_log(ctx, AV_LOG_ERROR, "transform360_cuda needs CUDA frames on its input (hw_frames_ctx is missing)\n");
    return AVERROR(EINVAL);
  }
  AVHWFramesContext* in_frames = (AVHWFramesContext*)inlink->hw_frames_ctx->data;
  if (in_frames->sw_format != AV_PIX_FMT_YUV420P && in_frames->sw_format != AV_PIX_FMT_GRAY8) {
    av_log(ctx, AV_LOG_ERROR, "planar 8-bit frames only (yuv420p, gray8); put scale_cuda=format=yuv420p in front\n");
    return AVERROR(ENOSYS);
  }
  s->sw_format = in_frames->sw_format;
  s->num_planes = av_pix_fmt_count_planes(s->sw_format);
  s->cuda = in_frames->device_ctx->hwctx;

  av_buffer_unref(&s->out_frames);
  s->out_frames = av_hwframe_ctx_alloc(in_frames->device_ref);
  if (!s->out_frames) return AVERROR(ENOMEM);
  AVHWFramesContext* out_frames = (AVHWFramesContext*)s->out_frames->data;
  out_frames->format = AV_PIX_FMT_CUDA;
  out_frames->sw_format = s->sw_format;
  out_frames->width = FFALIGN(w, 32);
  out_frames->height = FFALIGN(h, 32);
  if ((rc = av_hwframe_ctx_init(s->out_frames)) < 0) return rc;
  av_buffer_unref(&outlink->hw_frames_ctx);
  outlink->hw_frames_ctx = av_buffer_ref(s->out_frames);
  return outlink->hw_frames_ctx ? 0 : AVERROR(ENOMEM);
}

/* both sampling plans (luma-sized, chroma-sized), once the link sizes are known; like vf:100-165 this waits for the
 * first frame, so that a graph can be configured on a machine without the device */
static int make_maps(AVFilterContext* ctx) {
  T360CudaContext* s = ctx->priv;
  const AVFilterLink* in = ctx->inputs[0];
  const AVFilterLink* out = ctx->outputs[0];
  const AVPixFmtDescriptor* d = av_pix_fmt_desc_get(s->sw_format);
  if (!s->transform && !(s->transform = VideoFrameTransform_new(&s->params))) return AVERROR(ENOMEM);
  for (int idx = 0; idx < 2; idx++) {
    if (!VideoFrameTransform_generateMapForPlane(s->transform, plane_extent(in->w, idx, d->log2_chroma_w),
                                                 plane_extent(in->h, idx, d->log2_chroma_h),
                                                 plane_extent(out->w, idx, d->log2_chroma_w),
                                                 plane_extent(out->h, idx, d->log2_chroma_h), idx)) {
      av_log(ctx, AV_LOG_ERROR, "no sampling plan for plane index %d\n", idx);
      return AVERROR(EINVAL);
    }
  }
  s->maps_ready = 1;
  return 0;
}

static int t360_filter_frame(AVFilterLink* inlink, AVFrame* in) {
  AVFilterContext* ctx = inlink->dst;
  AVFilterLink* outlink = ctx->outputs[0];
  T360CudaContext* s = ctx->priv;
  CudaFunctions* cu = s->cuda->internal->cuda_dl;
  AVFrame* out = NULL;
  CUcontext popped;
  int rc = AVERROR(EINVAL);

  if (in->format != AV_PIX_FMT_CUDA || !in->hw_frames_ctx) {
    av_log(ctx, AV_LOG_ERROR, "got a frame that is not in device memory\n");
    goto done;
  }
  if (cu->cuCtxPushCurrent(s->cuda->cuda_ctx)) {
    rc = AVERROR_EXTERNAL;
    goto done;
  }
  if (!s->maps_ready && (rc = make_maps(ctx)) < 0) goto pop;
  if (!(out = av_frame_alloc())) {
    rc = AVERROR(ENOMEM);
    goto pop;
  }
  if ((rc = av_hwframe_get_buffer(outlink->hw_frames_ctx, out, 0)) < 0) goto pop;
  out->width = outlink->w;
  out->height = outlink->h;
  if ((rc = av_frame_copy_props(out, in)) < 0) goto pop;

  {
    const AVPixFmtDescriptor* d = av_pix_fmt_desc_get(s->sw_format);
    const uint8_t* src[3];
    uint8_t* dst[3];
    int in_w[3], in_h[3], in_pitch[3], out_w[3], out_h[3], out_pitch[3];
    for (int p = 0; p < s->num_planes; p++) {
      src[p] = in->data[p];
      dst[p] = out->data[p];
      in_w[p] = plane_extent(inlink->w, p, d->log2_chroma_w);
      in_h[p] = plane_extent(inlink->h, p, d->log2_chroma_h);
      out_w[p] = plane_extent(outlink->w, p, d->log2_chroma_w);
      out_h[p] = plane_extent(outlink->h, p, d->log2_chroma_h);
      in_pitch[p] = in->linesize[p];
      out_pitch[p] = out->linesize[p];
    }
    rc = T360B200_transformFrameAsync(s->transform, s->num_planes, src, dst, in_w, in_h, in_pitch, out_w, out_h, out_pitch,
                                      s->cuda->stream)
             ? 0
             : AVERROR_EXTERNAL;
    /* `in` is released below: its buffer goes back to the decoder's pool, which may hand it out again while the
     * gather still reads it unless the stream is drained first */
    if (!rc && s->sync && cu->cuStreamSynchronize(s->cuda->stream)) rc = AVERROR_EXTERNAL;
  }
pop:
  cu->cuCtxPopCurrent(&popped);
done:
  av_frame_free(&in);
  if (rc < 0) {
    av_frame_free(&out);
    return rc;
  }
  return ff_filter_frame(outlink, out);
}

/* Runtime commands (sendcmd, zmq): the view and quality options below are marked AV_OPT_FLAG_RUNTIME_PARAM.  Before the
 * first frame a command only updates the parameters.  After it, every accepted command hands the updated parameters to
 * T360B200_reconfigureAsync, which returns in microseconds without re-planning: frames filtered before the command keep
 * the old parameters, every later frame has the new ones.  The transform serves those frames on its per-frame kernels
 * while it plans the new parameters in the background, once commands have paused for a quarter of a second, and then
 * returns to the planned frame kernel by itself; the frames are the same either way.  So the camera can move every frame
 * (head tracking, a camera path, stabilisation) and a quality change does not stall the pipeline for a re-plan.
 * Options that could change the output link's size or format (size, cube edge, layouts, stereo formats, scale factors)
 * are refused with ENOSYS, invalid values (including parameters the transform refuses) with EINVAL; a refused command
 * leaves every parameter as it was.
 * This needs AV_OPT_FLAG_RUNTIME_PARAM and ff_filter_process_command (FFmpeg 4.2 and later).  A libavfilter without
 * runtime options builds the filter without commands: the options are then fixed at init, as in the reference filter. */
#ifdef AV_OPT_FLAG_RUNTIME_PARAM
#define T360_COMMANDS 1
#define VFR (AV_OPT_FLAG_VIDEO_PARAM | AV_OPT_FLAG_FILTERING_PARAM | AV_OPT_FLAG_RUNTIME_PARAM)
#else
#define T360_COMMANDS 0
#define VFR (AV_OPT_FLAG_VIDEO_PARAM | AV_OPT_FLAG_FILTERING_PARAM)
#endif

#if T360_COMMANDS
static int t360_process_command(AVFilterContext* ctx, const char* cmd, const char* arg, char* res, int res_len, int flags) {
  T360CudaContext* s = ctx->priv;
  const FrameTransformContext before = s->params;
  int rc = ff_filter_process_command(ctx, cmd, arg, res, res_len, flags);
  if (rc == AVERROR(ENOSYS)) return rc;
  if (rc < 0) {
    s->params = before;
    av_log(ctx, AV_LOG_ERROR, "invalid value '%s' for %s\n", arg, cmd);
    return AVERROR(EINVAL);
  }
  if (!s->maps_ready) return 0;
  rc = T360B200_reconfigureAsync(s->transform, &s->params) ? 0 : AVERROR(EINVAL); /* (host checks only: no CUDA call) */
  if (rc) {
    s->params = before;
    av_log(ctx, AV_LOG_ERROR, "the transform refused %s=%s; the previous configuration stays in effect\n", cmd, arg);
  }
  return rc;
}
#endif

#define FIELD(f) offsetof(T360CudaContext, f)
#define PARAM(f) offsetof(T360CudaContext, params.f)
#define VF (AV_OPT_FLAG_VIDEO_PARAM | AV_OPT_FLAG_FILTERING_PARAM)
#define TEXT(name, help, off) {name, help, off, AV_OPT_TYPE_STRING, {.str = NULL}, 0, 0, VF, NULL}
#define INT(name, help, off, def, lo, hi, unit) {name, help, off, AV_OPT_TYPE_INT, {.i64 = def}, lo, hi, VF, unit}
#define REAL(name, help, off, def, lo, hi) {name, help, off, AV_OPT_TYPE_FLOAT, {.dbl = def}, lo, hi, VF, NULL}
#define RUNTIME_INT(name, help, off, def, lo, hi, unit) {name, help, off, AV_OPT_TYPE_INT, {.i64 = def}, lo, hi, VFR, unit}
#define RUNTIME_REAL(name, help, off, def, lo, hi) {name, help, off, AV_OPT_TYPE_FLOAT, {.dbl = def}, lo, hi, VFR, NULL}
#define NAMED(name, value, unit) {name, NULL, 0, AV_OPT_TYPE_CONST, {.i64 = value}, 0, 0, VF, unit}
#define NAMED2(upper, lower, value, unit) NAMED(upper, value, unit), NAMED(lower, value, unit)

static const AVOption transform360_cuda_options[] = {
    /* output size (vf:408-447) */
    TEXT("w", "output width", FIELD(out_w)), TEXT("width", "output width", FIELD(out_w)),
    TEXT("h", "output height", FIELD(out_h)), TEXT("height", "output height", FIELD(out_h)),
    TEXT("size", "output size, WxH", FIELD(out_size)), TEXT("s", "output size, WxH", FIELD(out_size)),
    INT("cube_edge_length", "edge of one cube face in pixels (rounded down to a multiple of 16)", FIELD(cube_edge_length), 0, 0, 16384, NULL),
    INT("max_cube_edge_length", "derive the edge from the input width, at most this", FIELD(max_cube_edge_length), 0, 0, 16384, NULL),
    INT("max_output_h", "accepted, unused", FIELD(max_output_h), 0, 0, 16384, NULL),
    INT("max_output_w", "accepted, unused", FIELD(max_output_w), 0, 0, 16384, NULL),
    /* projection (vf:448-720) */
    INT("input_stereo_format", "stereo packing of the input", PARAM(input_stereo_format), STEREO_FORMAT_GUESS, 0, STEREO_FORMAT_N - 1, "stereo"),
    INT("output_stereo_format", "stereo packing of the output", PARAM(output_stereo_format), STEREO_FORMAT_GUESS, 0, STEREO_FORMAT_N - 1, "stereo"),
    NAMED2("TB", "tb", STEREO_FORMAT_TB, "stereo"), NAMED2("LR", "lr", STEREO_FORMAT_LR, "stereo"),
    NAMED2("MONO", "mono", STEREO_FORMAT_MONO, "stereo"), NAMED2("GUESS", "guess", STEREO_FORMAT_GUESS, "stereo"),
    INT("input_layout", "projection of the input", PARAM(input_layout), LAYOUT_EQUIRECT, 0, LAYOUT_N - 1, "layout"),
    INT("output_layout", "projection of the output", PARAM(output_layout), LAYOUT_CUBEMAP_32, 0, LAYOUT_N - 1, "layout"),
    NAMED2("CUBEMAP_32", "cubemap_32", LAYOUT_CUBEMAP_32, "layout"),
    NAMED2("CUBEMAP_23_OFFCENTER", "cubemap_23_offcenter", LAYOUT_CUBEMAP_23_OFFCENTER, "layout"),
    NAMED2("EQUIRECT", "equirect", LAYOUT_EQUIRECT, "layout"), NAMED2("FLAT_FIXED", "flat_fixed", LAYOUT_FLAT_FIXED, "layout"),
    NAMED2("BARREL", "barrel", LAYOUT_BARREL, "layout"), NAMED2("BARREL_SPLIT", "barrel_split", LAYOUT_BARREL_SPLIT, "layout"),
    NAMED2("EAC_32", "eac_32", LAYOUT_EAC_32, "layout"),
    /* the view: runtime commands too */
    RUNTIME_INT("vflip", "flip the second eye of a TB output", PARAM(vflip), 0, 0, 1, "flag"), NAMED("false", 0, "flag"), NAMED("true", 1, "flag"),
    RUNTIME_INT("is_horizontal_offset", "off-centre shift along the view axis only", PARAM(is_horizontal_offset), 0, 0, 1, NULL),
    RUNTIME_REAL("input_expand_coef", "face expansion of a cubemap input", PARAM(input_expand_coef), 1.01f, 0, 10),
    RUNTIME_REAL("expand_coef", "face expansion of the output", PARAM(expand_coef), 1.01f, 0, 10),
    RUNTIME_REAL("yaw", "degrees", PARAM(fixed_yaw), 0, -360, 360), RUNTIME_REAL("pitch", "degrees", PARAM(fixed_pitch), 0, -180, 180),
    RUNTIME_REAL("roll", "degrees", PARAM(fixed_roll), 0, -180, 180),
    RUNTIME_REAL("hfov", "flat_fixed: horizontal field of view, degrees", PARAM(fixed_hfov), 120, -360, 360),
    RUNTIME_REAL("vfov", "flat_fixed: vertical field of view, degrees", PARAM(fixed_vfov), 110, -180, 180),
    RUNTIME_REAL("cube_offcenter_x", "off-centre projection", PARAM(fixed_cube_offcenter_x), 0, -1, 1),
    RUNTIME_REAL("cube_offcenter_y", "off-centre projection", PARAM(fixed_cube_offcenter_y), 0, -1, 1),
    RUNTIME_REAL("cube_offcenter_z", "off-centre projection", PARAM(fixed_cube_offcenter_z), 0, -1, 1),
    /* sampling and the segmented low-pass (vf:721-986); runtime commands except the scale factors (they size the render) */
    RUNTIME_INT("interpolation_alg", "nearest, linear, cubic or lanczos4", PARAM(interpolation_alg), CUBIC, 0, 4, "interp"),
    NAMED2("NEAREST", "nearest", NEAREST, "interp"), NAMED2("LINEAR", "linear", LINEAR, "interp"),
    NAMED2("CUBIC", "cubic", CUBIC, "interp"), NAMED2("LANCZOS4", "lanczos4", LANCZOS4, "interp"),
    REAL("width_scale_factor", "render at this multiple of the width, then area-resize", PARAM(width_scale_factor), 1, 0, 10),
    REAL("height_scale_factor", "render at this multiple of the height, then area-resize", PARAM(height_scale_factor), 1, 0, 10),
    RUNTIME_INT("enable_low_pass_filter", "anti-alias the input per segment", PARAM(enable_low_pass_filter), 1, 0, 1, NULL),
    INT("enable_multi_threading", "accepted; the GPU takes all segments at once", PARAM(enable_multi_threading), 1, 0, 1, NULL),
    RUNTIME_INT("num_vertical_segments", "low-pass bands top to bottom", PARAM(num_vertical_segments), 5, 2, 500, NULL),
    RUNTIME_INT("num_horizontal_segments", "low-pass bands left to right", PARAM(num_horizontal_segments), 1, 1, 500, NULL),
    RUNTIME_REAL("kernel_height_scale_factor", "vertical kernel size factor", PARAM(kernel_height_scale_factor), 1, 0.1, 100),
    RUNTIME_REAL("min_kernel_half_height", "lower clamp of the vertical kernel", PARAM(min_kernel_half_height), 1, 0.5, 200),
    RUNTIME_REAL("max_kernel_half_height", "upper clamp of the vertical kernel", PARAM(max_kernel_half_height), 10000, 0.5, 100000),
    RUNTIME_INT("adjust_kernel", "scale the kernel with the off-centre magnification", PARAM(adjust_kernel), 1, 0, 1, NULL),
    RUNTIME_REAL("kernel_adjust_factor", "factor of that adjustment", PARAM(kernel_adjust_factor), 1, 0.1, 100),
    /* this filter only */
    INT("sync", "drain the stream before the frame travels on", FIELD(sync), 1, 0, 1, NULL),
    {NULL}};

static const AVClass transform360_cuda_class = {
    .class_name = "transform360_cuda",
    .item_name = av_default_item_name,
    .option = transform360_cuda_options,
    .version = LIBAVUTIL_VERSION_INT,
    .category = AV_CLASS_CATEGORY_FILTER,
};

static const AVFilterPad t360_cuda_inputs[] = {{.name = "default", .type = AVMEDIA_TYPE_VIDEO, .filter_frame = t360_filter_frame}, {NULL}};
static const AVFilterPad t360_cuda_outputs[] = {{.name = "default", .type = AVMEDIA_TYPE_VIDEO, .config_props = t360_config_output}, {NULL}};

AVFilter ff_vf_transform360_cuda = {
    .name = "transform360_cuda",
    .description = NULL_IF_CONFIG_SMALL("360-degree projection transform of CUDA frames (transform360-b200)"),
    .init = t360_init,
    .uninit = t360_uninit,
    .query_formats = t360_query_formats,
    .priv_size = sizeof(T360CudaContext),
    .priv_class = &transform360_cuda_class,
    .inputs = t360_cuda_inputs,
    .outputs = t360_cuda_outputs,
#if T360_COMMANDS
    .process_command = t360_process_command,
#endif
    .flags_internal = FF_FILTER_FLAG_HWFRAME_AWARE,
};
