/* oracle/t360_oracle.h -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C CPU restatement of the Transform360 projection-remap hot path:
 *   - the reference's geometry and low-pass plan (VideoFrameTransform.cpp), and
 *   - the OpenCV 4.x arithmetic the reference delegates pixels to (cv::remap with a
 *     CV_32FC2 map / cv::sepFilter2D u8->u8 with float kernels), which is a third-party
 *     dependency ABSENT from the reference (CMakeLists.txt:11 find_package(OpenCV),
 *     un-pinned; the build in this image is opencv-python-headless 4.13.0.92).
 *
 * PARITY PIN: the reference ships no tests, golden vectors or fixtures (SURVEY.md 4), so
 * this oracle is pinned against OUTPUTS OF THE REFERENCE ITSELF RUN HERE: oracle/_ref
 * (the unmodified reference sources compiled against oracle/shim, driving cv2 4.13.0) --
 * see tests/test_oracle_pin.py and the committed fixtures in tests/golden/.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / reference legs may
 * use this library.  The product (transform360_b200/) never links or loads it.
 */
#ifndef T360_ORACLE_H
#define T360_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Same 28 x 4-byte layout as the reference's FrameTransformContext (VideoFrameTransformHelper.h:56-90). */
typedef struct T360OContext {
  int input_layout, output_layout, input_stereo_format, output_stereo_format, vflip;
  float input_expand_coef, expand_coef;
  int interpolation_alg;
  float width_scale_factor, height_scale_factor;
  float fixed_yaw, fixed_pitch, fixed_roll, fixed_hfov, fixed_vfov;
  float fixed_cube_offcenter_x, fixed_cube_offcenter_y, fixed_cube_offcenter_z;
  int is_horizontal_offset, enable_low_pass_filter;
  float kernel_height_scale_factor, min_kernel_half_height, max_kernel_half_height;
  int enable_multi_threading, num_vertical_segments, num_horizontal_segments, adjust_kernel;
  float kernel_adjust_factor;
} T360OContext;

enum { T360O_CUBEMAP_32 = 0, T360O_CUBEMAP_23_OFFCENTER = 1, T360O_FLAT_FIXED = 2, T360O_EQUIRECT = 3,
       T360O_BARREL = 4, T360O_BARREL_SPLIT = 5, T360O_EAC_32 = 6, T360O_LAYOUT_N = 7 };
enum { T360O_TB = 0, T360O_LR = 1, T360O_MONO = 2, T360O_GUESS = 3, T360O_STEREO_N = 4 };
enum { T360O_NEAREST = 0, T360O_LINEAR = 1, T360O_CUBIC = 2, T360O_LANCZOS4 = 4 };
enum { T360O_BORDER_CONSTANT = 0, T360O_BORDER_REPLICATE = 1, T360O_BORDER_WRAP = 3, T360O_BORDER_TRANSPARENT = 5 };

typedef struct T360OSegment {
  int left, top, width, height; /* reference SegmentFilteringConfig, VideoFrameTransform.h:25-38 */
  int nkx, nky;                 /* tap counts */
  int kx_off, ky_off;           /* offsets into the taps array */
} T360OSegment;

/* ---- geometry (reference cpp:504-576, 893-1316, 863-891, 796-861, 53-75) ---- */
int t360o_scaled_dims(const T360OContext* c, int outW, int outH, int* sW, int* sH);
int t360o_transform_pos(const T360OContext* c, float x, float y, float inputPixelWidth, float* outX, float* outY);
/* map: float32[sH][sW][2]; returns 1 on success */
int t360o_generate_map(const T360OContext* c, int inW, int inH, int outW, int outH, float* map);

/* ---- low-pass plan (reference cpp:78-94, 126-170, 210-501) ---- */
/* returns number of segments, or -1 if the buffers are too small; *ntaps = floats used */
int t360o_filter_plan(const T360OContext* c, int inW, int inH, int scaledOutW, int scaledOutH,
                      T360OSegment* segs, int maxSegs, float* taps, int maxTaps, int* ntaps);

/* ---- OpenCV arithmetic (SURVEY.md Appendix A / B) ---- */
int t360o_remap_ksize(int interp);
void t360o_build_itab(int interp, int16_t* itab /* [1024][k][k] */);
void t360o_remap_u8(const uint8_t* src, int sw, int sh, size_t spitch, uint8_t* dst, int dw, int dh,
                    size_t dpitch, const float* mapxy /* [dh][dw][2] */, int interp, int border);
void t360o_sepfilter_roi_u8(const uint8_t* parent, int pw, int ph, size_t ppitch, int rx, int ry, int rw,
                            int rh, uint8_t* dstParent, size_t dpitch, const float* kx, int nkx,
                            const float* ky, int nky);
/* reference filterPlane (cpp:621-704): applies the plan once (MONO) or twice (LR/TB) */
void t360o_filter_plane(const T360OContext* c, const uint8_t* src, int w, int h, size_t spitch,
                        uint8_t* dst, size_t dpitch, const T360OSegment* segs, int nsegs, const float* taps);
/* cv::resize(INTER_AREA) for 8-bit single-channel SHRINKING (OpenCV 4.x resize.cpp: resizeAreaFast_ for integer
 * ratios -- (sum+2)>>2 for 2x2, cvRound(sum * (1.f/area)) otherwise -- and resizeArea_ with computeResizeAreaTab
 * for the rest).  Returns 0 (nothing written) when either axis would be enlarged. */
int t360o_resize_area_u8(const uint8_t* src, int sw, int sh, size_t spitch, uint8_t* dst, int dw, int dh, size_t dpitch);
/* reference transformPlane (cpp:707-794): [low-pass] -> remap [-> area resize when the map was planned at a scaled
 * size, cpp:755-777].  map/segs/taps as produced above; returns 1 on success, 0 if the resize would enlarge. */
int t360o_transform_plane(const T360OContext* c, const uint8_t* src, int inW, int inH, size_t spitch,
                          uint8_t* dst, int outW, int outH, size_t dpitch, const float* map, int mapW,
                          int mapH, int mapIndex, const T360OSegment* segs, int nsegs, const float* taps);

/* ---- synthetic input + hashes (SURVEY.md 8d / Appendix D) ---- */
void t360o_noise_plane(uint8_t* dst, int w, int h, size_t pitch, uint32_t plane, uint32_t frame);
uint64_t t360o_fnv1a64(const void* p, size_t n);

#ifdef __cplusplus
}
#endif
#endif
