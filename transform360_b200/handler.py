"""Python mirror of the reference's C handler (VideoFrameTransformHandler.h:22-47) over libTransform360.so.

This is a thin ctypes binding of the drop-in C-ABI -- the same four entry points the reference's ffmpeg
filter calls (vf_transform360.c:141, 157, 334, 383) -- plus the extension entry points of
``include/transform360_b200.h``.  It exists so that tests, ``bench.py`` and the multi-GPU stream driver
can call the product exactly the way a C caller would.  There is no Python or CPU pixel path here: if the
shared library is missing, ``load()`` raises; if no CUDA device is usable the C calls return 0.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import numpy as np

PKG = Path(__file__).resolve().parent
LIB_PATH = PKG / "lib" / "libTransform360.so"

# enums of Transform360/VideoFrameTransformHelper.h
LAYOUT_CUBEMAP_32, LAYOUT_CUBEMAP_23_OFFCENTER, LAYOUT_FLAT_FIXED, LAYOUT_EQUIRECT = 0, 1, 2, 3
LAYOUT_BARREL, LAYOUT_BARREL_SPLIT, LAYOUT_EAC_32, LAYOUT_N = 4, 5, 6, 7
STEREO_FORMAT_TB, STEREO_FORMAT_LR, STEREO_FORMAT_MONO, STEREO_FORMAT_GUESS, STEREO_FORMAT_N = 0, 1, 2, 3, 4
NEAREST, LINEAR, CUBIC, LANCZOS4 = 0, 1, 2, 4
BORDER_WRAP, BORDER_TRANSPARENT = 3, 5  # cv::remap's border modes for a caller's warp map (include/transform360_b200.h)


def _warp_map(map) -> np.ndarray:
    """A caller's CV_32FC2 warp map as a C-contiguous float32 [h][w][2] array."""
    m = np.ascontiguousarray(map, np.float32)
    if m.ndim != 3 or m.shape[2] != 2:
        raise ValueError(f"a warp map is float32 [h][w][2] (x, y per output pixel), got shape {m.shape}")
    return m


def _frame_args(in_planes, out_planes, dims):
    """The arguments of a whole-frame call after the transform: (number of planes, input and output plane arrays, the six
    size and pitch arrays), and the ctypes arrays they point into, which must outlive the call."""
    n = len(in_planes)
    VP, IA = C.c_void_p * n, C.c_int * n
    d_in = VP(*[p[0] for p in in_planes])
    d_out = VP(*[p[0] for p in out_planes])
    arrs = [IA(*[d[0] for d in dims]), IA(*[d[1] for d in dims]), IA(*[p[1] for p in in_planes]),
            IA(*[d[2] for d in dims]), IA(*[d[3] for d in dims]), IA(*[p[1] for p in out_planes])]
    ptrs = [C.cast(a, C.c_void_p) for a in arrs]
    return n, C.cast(d_in, C.c_void_p), C.cast(d_out, C.c_void_p), ptrs, (d_in, d_out, arrs)


def _samples(fn, ctx, fields, in_w, in_h, out_w, out_h) -> np.ndarray:
    """int32 [map_h][map_w][2] sampling records from fn(ctx, fields, in_w, in_h, out_w, out_h, out), a T360B200_*Samples
    call; ValueError when it refuses the arguments."""
    scaled = lambda f, n: int(float(np.float32(f) * np.float32(n)) + 0.5)  # (float product, double sum: buildHostPlan)
    map_w, map_h = scaled(ctx.width_scale_factor, out_w), scaled(ctx.height_scale_factor, out_h)
    out = np.zeros((max(map_h, 0), max(map_w, 0), 2), np.int32)
    if not fn(C.byref(ctx), C.byref(fields), in_w, in_h, out_w, out_h, out.ctypes.data):
        raise ValueError(f"{fn.__name__} refused the arguments (message on stdout)")
    return out


class FrameTransformContext(C.Structure):
    """28 x 4 bytes, field for field the reference's struct (VideoFrameTransformHelper.h:56-90)."""
    _fields_ = [
        ("input_layout", C.c_int), ("output_layout", C.c_int),
        ("input_stereo_format", C.c_int), ("output_stereo_format", C.c_int),
        ("vflip", C.c_int), ("input_expand_coef", C.c_float), ("expand_coef", C.c_float),
        ("interpolation_alg", C.c_int), ("width_scale_factor", C.c_float),
        ("height_scale_factor", C.c_float), ("fixed_yaw", C.c_float), ("fixed_pitch", C.c_float),
        ("fixed_roll", C.c_float), ("fixed_hfov", C.c_float), ("fixed_vfov", C.c_float),
        ("fixed_cube_offcenter_x", C.c_float), ("fixed_cube_offcenter_y", C.c_float),
        ("fixed_cube_offcenter_z", C.c_float), ("is_horizontal_offset", C.c_int),
        ("enable_low_pass_filter", C.c_int), ("kernel_height_scale_factor", C.c_float),
        ("min_kernel_half_height", C.c_float), ("max_kernel_half_height", C.c_float),
        ("enable_multi_threading", C.c_int), ("num_vertical_segments", C.c_int),
        ("num_horizontal_segments", C.c_int), ("adjust_kernel", C.c_int),
        ("kernel_adjust_factor", C.c_float),
    ]


FILTER_DEFAULTS = dict(  # the reference's AVOption defaults (vf_transform360.c:407-987)
    input_layout=LAYOUT_EQUIRECT, output_layout=LAYOUT_CUBEMAP_32, input_stereo_format=STEREO_FORMAT_MONO,
    output_stereo_format=STEREO_FORMAT_MONO, vflip=0, input_expand_coef=1.01, expand_coef=1.01,
    interpolation_alg=CUBIC, width_scale_factor=1.0, height_scale_factor=1.0, fixed_yaw=0.0, fixed_pitch=0.0,
    fixed_roll=0.0, fixed_hfov=120.0, fixed_vfov=110.0, fixed_cube_offcenter_x=0.0, fixed_cube_offcenter_y=0.0,
    fixed_cube_offcenter_z=0.0, is_horizontal_offset=0, enable_low_pass_filter=1, kernel_height_scale_factor=1.0,
    min_kernel_half_height=1.0, max_kernel_half_height=10000.0, enable_multi_threading=1, num_vertical_segments=5,
    num_horizontal_segments=1, adjust_kernel=1, kernel_adjust_factor=1.0)


class T360View(C.Structure):
    """A FLAT_FIXED view in degrees (include/transform360_b200.h), as the context's fixed_yaw / pitch / hfov / vfov."""
    _fields_ = [("yaw", C.c_float), ("pitch", C.c_float), ("hfov", C.c_float), ("vfov", C.c_float)]


def as_view(view) -> T360View:
    """A T360View from a T360View or a (yaw, pitch, hfov, vfov) sequence."""
    return view if isinstance(view, T360View) else T360View(*[float(v) for v in view])


class T360Orientation(C.Structure):
    """An orientation in degrees (include/transform360_b200.h), as the context's fixed_yaw / pitch / roll."""
    _fields_ = [("yaw", C.c_float), ("pitch", C.c_float), ("roll", C.c_float)]


def as_orientation(orientation) -> T360Orientation:
    """A T360Orientation from a T360Orientation or a (yaw, pitch, roll) sequence."""
    if isinstance(orientation, T360Orientation):
        return orientation
    return T360Orientation(*[float(v) for v in orientation])


class T360Pose(C.Structure):
    """A camera pose in degrees (include/transform360_b200.h), as the context's fixed_yaw / pitch / roll / hfov / vfov."""
    _fields_ = [("yaw", C.c_float), ("pitch", C.c_float), ("roll", C.c_float), ("hfov", C.c_float), ("vfov", C.c_float)]


def as_pose(pose) -> T360Pose:
    """A T360Pose from a T360Pose or a (yaw, pitch, roll, hfov, vfov) sequence."""
    return pose if isinstance(pose, T360Pose) else T360Pose(*[float(v) for v in pose])


T360_CAMERA_PINHOLE, T360_CAMERA_EQUIDISTANT, T360_CAMERA_STEREOGRAPHIC, T360_CAMERA_PANNINI = 0, 1, 2, 3
T360_CAMERA_EQUIRECT = 5  # (4 is not a model)


class T360Camera(C.Structure):
    """The camera model of a view (include/transform360_b200.h): T360_CAMERA_*, and Pannini's d (read by T360_CAMERA_PANNINI
    only)."""
    _fields_ = [("model", C.c_int), ("pannini", C.c_float)]


def as_camera(camera) -> T360Camera:
    """A T360Camera from a T360Camera, a model, or a (model, pannini) sequence."""
    if isinstance(camera, T360Camera):
        return camera
    if isinstance(camera, (tuple, list)):
        return T360Camera(int(camera[0]), float(camera[1]))
    return T360Camera(int(camera), 0.0)


class T360Minify(C.Structure):
    """The pyramid of an anti-aliased camera view (include/transform360_b200.h): maxLevel in 0..8 levels above the input (0:
    the plain camera view), lodBias in [-4, 4] levels added to every pixel's level of detail."""
    _fields_ = [("maxLevel", C.c_int), ("lodBias", C.c_float)]


def as_minify(minify) -> T360Minify:
    """A T360Minify from a T360Minify, a max level, or a (max_level, lod_bias) sequence."""
    if isinstance(minify, T360Minify):
        return minify
    if isinstance(minify, (tuple, list)):
        return T360Minify(int(minify[0]), float(minify[1]))
    return T360Minify(int(minify), 0.0)


def mip_level_sizes(w: int, h: int, max_level: int) -> list[tuple[int, int]]:
    """The (width, height) of levels 0..T of a w x h plane's pyramid for max_level: each level half the one below, rounded
    up, and T the largest level <= max_level whose sides are both >= 8."""
    sizes = [(w, h)]
    while len(sizes) <= max_level and (sizes[-1][0] + 1) // 2 >= 8 and (sizes[-1][1] + 1) // 2 >= 8:
        sizes.append(((sizes[-1][0] + 1) // 2, (sizes[-1][1] + 1) // 2))
    return sizes


class T360Lens(C.Structure):
    """One fisheye lens (include/transform360_b200.h): OpenCV fisheye intrinsics fx, fy, cx, cy in pixels of the rig's
    calibration frame, distortion k1..k4, extrinsics yaw / pitch / roll in degrees, and the half field of view it covers."""
    _fields_ = [("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("k", C.c_float * 4),
                ("yaw", C.c_float), ("pitch", C.c_float), ("roll", C.c_float), ("maxAngle", C.c_float)]


class T360LensRig(C.Structure):
    """One or two fisheye lenses calibrated on a calibWidth x calibHeight frame (include/transform360_b200.h)."""
    _fields_ = [("numLenses", C.c_int), ("calibWidth", C.c_int), ("calibHeight", C.c_int), ("lens", T360Lens * 2)]


class T360LensPhotometry(C.Structure):
    """The photometry of one lens (include/transform360_b200.h): vignetting v1..v3 of the falloff V(r) = 1 + v1 r^2 +
    v2 r^4 + v3 r^6 (r = theta_d in radians), and per plane (0 luma, 1 and 2 chroma) a gain in (0, 8] and an offset in
    [-64, 64] code values."""
    _fields_ = [("vignetting", C.c_float * 3), ("gain", C.c_float * 3), ("offset", C.c_float * 3)]


class T360RigPhotometry(C.Structure):
    """The photometry of a rig (include/transform360_b200.h): lumaPivot (0..255, the level luma scales about; chroma scales
    about 128) and one T360LensPhotometry per lens."""
    _fields_ = [("lumaPivot", C.c_int), ("lens", T360LensPhotometry * 2)]


class T360LensReadout(C.Structure):
    """When a lens reads a point (include/transform360_b200.h): t = a u + b v + c, clamped to [0, 1], of the point's
    normalised calibration coordinates u = (fx x' + cx + 0.5) / calibWidth, v = (fy y' + cy + 0.5) / calibHeight."""
    _fields_ = [("a", C.c_float), ("b", C.c_float), ("c", C.c_float)]


class T360RigMotion(C.Structure):
    """A rig's motion over the readout (include/transform360_b200.h): numSamples (2..16) orientations delta[k] of the rig
    at readout time k / (numSamples - 1), turned from the frame's orientation or pose (degrees, each in [-30, 30]), and
    each lens's readout (readout[1] is read only with two lenses)."""
    _fields_ = [("numSamples", C.c_int), ("delta", T360Orientation * 16), ("readout", T360LensReadout * 2)]


def rig_motion(deltas, readouts=((0.0, 1.0, 0.0), (0.0, 1.0, 0.0))) -> T360RigMotion:
    """A T360RigMotion from a sequence of (yaw, pitch, roll) deltas (numSamples = len(deltas)) and one or two (a, b, c)
    readouts."""
    m = T360RigMotion(len(deltas))
    for k, d in enumerate(deltas):
        m.delta[k] = as_orientation(d)
    for i, r in enumerate(readouts):
        m.readout[i] = T360LensReadout(*[float(x) for x in r])
    return m


def make_context(**overrides) -> FrameTransformContext:
    vals = dict(FILTER_DEFAULTS)
    for k in overrides:
        if k not in vals:
            raise AttributeError(f"FrameTransformContext has no field {k!r}")
    vals.update(overrides)
    return FrameTransformContext(**vals)


_lib = None


def load(path: os.PathLike | None = None):
    """dlopen()s the product library.  Raises if it has not been built: there is no fallback."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = Path(path) if path else Path(os.environ.get("T360B200_LIB") or LIB_PATH)  # T360B200_LIB: experiment builds
    if not p.exists():
        raise FileNotFoundError(f"{p} not found: build it with `python -m transform360_b200.build` (needs nvcc); "
                                "transform360_b200 has no CPU fallback")
    L = C.CDLL(str(p), mode=os.RTLD_LOCAL)
    vp, ci = C.c_void_p, C.c_int
    # the tail of every frame entry point: dIn, dOut, inW, inH, inPitch, outW, outH, outPitch, stream
    planes = [vp, vp] + [vp] * 6 + [vp]
    L.VideoFrameTransform_new.restype = vp
    L.VideoFrameTransform_new.argtypes = [C.POINTER(FrameTransformContext)]
    L.VideoFrameTransform_delete.restype = None
    L.VideoFrameTransform_delete.argtypes = [vp]
    L.VideoFrameTransform_generateMapForPlane.restype = ci
    L.VideoFrameTransform_generateMapForPlane.argtypes = [vp] + [ci] * 5
    L.VideoFrameTransform_transformFramePlane.restype = ci
    L.VideoFrameTransform_transformFramePlane.argtypes = [vp, vp, vp] + [ci] * 8
    L.T360B200_hostPlanCreate.restype = vp
    L.T360B200_hostPlanCreate.argtypes = [C.POINTER(FrameTransformContext)] + [ci] * 4
    L.T360B200_hostPlanCreateFromWarp.restype = vp
    L.T360B200_hostPlanCreateFromWarp.argtypes = [C.POINTER(FrameTransformContext), vp] + [ci] * 5
    L.T360B200_generateMapFromWarp.restype = ci
    L.T360B200_generateMapFromWarp.argtypes = [vp, vp] + [ci] * 6
    L.T360B200_remapFrameAsync.restype = ci
    L.T360B200_remapFrameAsync.argtypes = [vp, ci, vp, vp, ci] + planes
    L.T360B200_hostPlanDestroy.restype = None
    L.T360B200_hostPlanDestroy.argtypes = [vp]
    L.T360B200_hostPlanInfo.restype = ci
    L.T360B200_hostPlanInfo.argtypes = [vp, C.POINTER(ci)]
    L.T360B200_hostPlanMap.restype = vp
    L.T360B200_hostPlanMap.argtypes = [vp]
    L.T360B200_hostPlanSamples.restype = vp
    L.T360B200_hostPlanSamples.argtypes = [vp]
    L.T360B200_hostPlanSegment.restype = ci
    L.T360B200_hostPlanSegment.argtypes = [vp, ci, C.POINTER(ci), C.POINTER(ci), C.POINTER(vp), C.POINTER(vp)]
    L.T360B200_hostPlanGather.restype = ci
    L.T360B200_hostPlanGather.argtypes = [vp, C.POINTER(ci), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
    L.T360B200_hostPlanPoleCaps.restype = ci
    L.T360B200_hostPlanBlurLists.restype = ci
    L.T360B200_hostPlanBlurLists.argtypes = [vp, ci, ci, ci, C.POINTER(ci), C.POINTER(vp)]
    L.T360B200_hostPlanPoleCaps.argtypes = [vp, C.POINTER(ci), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
    L.T360B200_hostPlanLaunchExtents.restype = ci
    L.T360B200_hostPlanLaunchExtents.argtypes = [vp, C.POINTER(ci), C.POINTER(vp), C.POINTER(vp)]
    L.T360B200_hostPlanWaves.restype = ci
    L.T360B200_hostPlanWaves.argtypes = [vp, ci, vp, C.POINTER(ci)] + [C.POINTER(vp)] * 4
    L.T360B200_hostPlanDeviceLists.restype = ci
    L.T360B200_hostPlanDeviceLists.argtypes = [vp, C.POINTER(ci), C.POINTER(vp), C.POINTER(vp)]
    L.T360B200_weightImage.restype = ci
    L.T360B200_weightImage.argtypes = [ci, C.POINTER(vp)]
    L.T360B200_remapTable.restype = ci
    L.T360B200_remapTable.argtypes = [ci, C.POINTER(vp)]
    L.T360B200_transformFramePlaneAsync.restype = ci
    L.T360B200_transformFramePlaneAsync.argtypes = [vp, vp, vp] + [ci] * 7 + [vp]
    L.T360B200_transformFrameAsync.restype = ci
    L.T360B200_transformFrameAsync.argtypes = [vp, ci] + planes
    L.T360B200_lowPassPlaneAsync.restype = ci
    L.T360B200_lowPassPlaneAsync.argtypes = [vp, vp, vp] + [ci] * 5 + [vp]
    L.T360B200_reconfigure.restype = ci
    L.T360B200_reconfigure.argtypes = [vp, C.POINTER(FrameTransformContext)]
    L.T360B200_reconfigureAsync.restype = ci
    L.T360B200_reconfigureAsync.argtypes = [vp, C.POINTER(FrameTransformContext)]
    L.T360B200_reconfigureWait.restype = ci
    L.T360B200_reconfigureWait.argtypes = [vp, ci]
    L.T360B200_transformFrameViewAsync.restype = ci
    L.T360B200_transformFrameViewAsync.argtypes = [vp, C.POINTER(T360View), ci] + planes
    L.T360B200_viewSamples.restype = ci
    L.T360B200_viewSamples.argtypes = [C.POINTER(FrameTransformContext), C.POINTER(T360View)] + [ci] * 4 + [vp]
    L.T360B200_transformFrameOrientedAsync.restype = ci
    L.T360B200_transformFrameOrientedAsync.argtypes = [vp, C.POINTER(T360Orientation), ci] + planes
    L.T360B200_orientedSamples.restype = ci
    L.T360B200_orientedSamples.argtypes = [C.POINTER(FrameTransformContext), C.POINTER(T360Orientation)] + [ci] * 4 + [vp]
    L.T360B200_transformFramePoseAsync.restype = ci
    L.T360B200_transformFramePoseAsync.argtypes = [vp, C.POINTER(T360Pose), ci] + planes
    L.T360B200_poseSamples.restype = ci
    L.T360B200_poseSamples.argtypes = [C.POINTER(FrameTransformContext), C.POINTER(T360Pose)] + [ci] * 4 + [vp]
    L.T360B200_lensMap.restype = ci
    L.T360B200_lensMap.argtypes = [C.POINTER(FrameTransformContext), C.POINTER(T360LensRig), C.POINTER(T360Orientation)] + [ci] * 4 + [vp]
    L.T360B200_transformFrameLensAsync.restype = ci
    L.T360B200_transformFrameLensAsync.argtypes = [vp, C.POINTER(T360LensRig), C.POINTER(T360Orientation), ci] + planes
    L.T360B200_lensBlendMaps.restype = ci
    L.T360B200_lensBlendMaps.argtypes = [C.POINTER(FrameTransformContext), C.POINTER(T360LensRig), C.c_float, C.POINTER(T360Orientation)] + [ci] * 4 + [vp] * 3
    L.T360B200_transformFrameLensBlendAsync.restype = ci
    L.T360B200_transformFrameLensBlendAsync.argtypes = [vp, C.POINTER(T360LensRig), C.c_float, C.POINTER(T360Orientation), ci] + planes
    L.T360B200_lensPhotoMaps.restype = ci
    L.T360B200_lensPhotoMaps.argtypes = [C.POINTER(FrameTransformContext), C.POINTER(T360LensRig), C.POINTER(T360RigPhotometry), C.c_float,
                                         C.POINTER(T360Orientation)] + [ci] * 5 + [vp] * 5
    L.T360B200_transformFrameLensPhotoAsync.restype = ci
    L.T360B200_transformFrameLensPhotoAsync.argtypes = [vp, C.POINTER(T360LensRig), C.POINTER(T360RigPhotometry), C.c_float,
                                                        C.POINTER(T360Orientation), vp, ci] + planes
    L.T360B200_lensMotionMaps.restype = ci
    L.T360B200_lensMotionMaps.argtypes = [C.POINTER(FrameTransformContext), C.POINTER(T360LensRig), C.POINTER(T360RigPhotometry), C.c_float,
                                          C.POINTER(T360Orientation), C.POINTER(T360RigMotion)] + [ci] * 5 + [vp] * 5
    L.T360B200_transformFrameLensMotionAsync.restype = ci
    L.T360B200_transformFrameLensMotionAsync.argtypes = [vp, C.POINTER(T360LensRig), C.POINTER(T360RigPhotometry), C.c_float,
                                                         C.POINTER(T360Orientation), C.POINTER(T360RigMotion), vp, ci] + planes
    L.T360B200_rectilinearMap.restype = ci
    L.T360B200_rectilinearMap.argtypes = [C.POINTER(FrameTransformContext), C.POINTER(T360LensRig), C.POINTER(T360Pose)] + [ci] * 4 + [vp]
    L.T360B200_transformFrameRectilinearAsync.restype = ci
    L.T360B200_transformFrameRectilinearAsync.argtypes = [vp, C.POINTER(T360LensRig), C.POINTER(T360Pose), ci] + planes
    L.T360B200_cameraMap.restype = ci
    L.T360B200_cameraMap.argtypes = [C.POINTER(FrameTransformContext), C.POINTER(T360LensRig), C.POINTER(T360Pose),
                                     C.POINTER(T360Camera)] + [ci] * 4 + [vp]
    L.T360B200_transformFrameCameraAsync.restype = ci
    L.T360B200_transformFrameCameraAsync.argtypes = [vp, C.POINTER(T360LensRig), C.POINTER(T360Pose), C.POINTER(T360Camera), ci] + planes
    L.T360B200_cameraMipMaps.restype = ci
    L.T360B200_cameraMipMaps.argtypes = [C.POINTER(FrameTransformContext), C.POINTER(T360LensRig), C.POINTER(T360Pose),
                                         C.POINTER(T360Camera), C.POINTER(T360Minify)] + [ci] * 4 + [vp] * 4
    L.T360B200_transformFrameCameraMipAsync.restype = ci
    L.T360B200_transformFrameCameraMipAsync.argtypes = [vp, C.POINTER(T360LensRig), C.POINTER(T360Pose), C.POINTER(T360Camera),
                                                        C.POINTER(T360Minify), ci] + planes
    L.T360B200_cameraAnisoMaps.restype = ci
    L.T360B200_cameraAnisoMaps.argtypes = [C.POINTER(FrameTransformContext), C.POINTER(T360LensRig), C.POINTER(T360Pose),
                                           C.POINTER(T360Camera), C.POINTER(T360Minify)] + [ci] * 5 + [vp] * 5
    L.T360B200_transformFrameCameraAnisoAsync.restype = ci
    L.T360B200_transformFrameCameraAnisoAsync.argtypes = [vp, C.POINTER(T360LensRig), C.POINTER(T360Pose), C.POINTER(T360Camera),
                                                          C.POINTER(T360Minify), ci, ci] + planes
    L.T360B200_cameraPhotoMaps.restype = ci
    L.T360B200_cameraPhotoMaps.argtypes = [C.POINTER(FrameTransformContext), C.POINTER(T360LensRig), C.POINTER(T360RigPhotometry), C.c_float,
                                           C.POINTER(T360Pose), C.POINTER(T360Camera), C.POINTER(T360Minify)] + [ci] * 6 + [vp] * 6
    L.T360B200_transformFrameCameraPhotoAsync.restype = ci
    L.T360B200_transformFrameCameraPhotoAsync.argtypes = [vp, C.POINTER(T360LensRig), C.POINTER(T360RigPhotometry), C.c_float,
                                                          C.POINTER(T360Pose), C.POINTER(T360Camera), C.POINTER(T360Minify), vp, ci] + planes
    L.T360B200_cameraMotionMaps.restype = ci
    L.T360B200_cameraMotionMaps.argtypes = [C.POINTER(FrameTransformContext), C.POINTER(T360LensRig), C.POINTER(T360RigPhotometry), C.c_float,
                                            C.POINTER(T360Pose), C.POINTER(T360Camera), C.POINTER(T360Minify), C.POINTER(T360RigMotion)] + [ci] * 6 + [vp] * 6
    L.T360B200_transformFrameCameraMotionAsync.restype = ci
    L.T360B200_transformFrameCameraMotionAsync.argtypes = [vp, C.POINTER(T360LensRig), C.POINTER(T360RigPhotometry), C.c_float,
                                                           C.POINTER(T360Pose), C.POINTER(T360Camera), C.POINTER(T360Minify),
                                                           C.POINTER(T360RigMotion), vp, ci] + planes
    L.T360B200_stereoCameraMaps.restype = ci
    L.T360B200_stereoCameraMaps.argtypes = [C.POINTER(FrameTransformContext), C.POINTER(T360LensRig), C.POINTER(T360RigPhotometry),
                                            C.POINTER(T360Pose), C.POINTER(T360Camera), C.POINTER(T360Minify)] + [ci] * 6 + [vp] * 6
    L.T360B200_transformFrameStereoCameraAsync.restype = ci
    L.T360B200_transformFrameStereoCameraAsync.argtypes = [vp, C.POINTER(T360LensRig), C.POINTER(T360RigPhotometry), C.POINTER(T360Pose),
                                                           C.POINTER(T360Camera), C.POINTER(T360Minify), vp, ci] + planes
    L.T360B200_setPinHostPlanes.restype = None
    L.T360B200_setPinHostPlanes.argtypes = [vp, ci]
    L.T360B200_debugTrace.restype = None
    L.T360B200_debugTrace.argtypes = [vp, ci]
    L.T360B200_debugTraceRead.restype = C.c_ulonglong
    L.T360B200_debugTraceRead.argtypes = [vp, vp, C.c_ulonglong]
    L.T360B200_synchronize.restype = ci
    L.T360B200_synchronize.argtypes = [vp]
    L.T360B200_stream.restype = vp
    L.T360B200_stream.argtypes = [vp]
    L.T360B200_kernelLaunchCount.restype = C.c_ulonglong
    L.T360B200_planDeviceBytes.restype = C.c_ulonglong
    L.T360B200_planDeviceBytes.argtypes = [vp, ci]
    L.T360B200_planTileCounts.restype = ci
    L.T360B200_planTileCounts.argtypes = [vp, ci, C.POINTER(ci)]
    L.T360B200_deviceCount.restype = ci
    L.T360B200_version.restype = C.c_char_p
    if path is None:
        _lib = L
    return L


EXPORTED_SYMBOLS = [
    "VideoFrameTransform_new", "VideoFrameTransform_delete", "VideoFrameTransform_generateMapForPlane",
    "VideoFrameTransform_transformFramePlane", "T360B200_hostPlanCreate", "T360B200_hostPlanCreateFromWarp", "T360B200_hostPlanDestroy",
    "T360B200_generateMapFromWarp", "T360B200_remapFrameAsync",
    "T360B200_hostPlanInfo", "T360B200_hostPlanMap", "T360B200_hostPlanSamples", "T360B200_hostPlanSegment",
    "T360B200_hostPlanGather", "T360B200_hostPlanPoleCaps", "T360B200_hostPlanLaunchExtents", "T360B200_hostPlanWaves", "T360B200_hostPlanDeviceLists", "T360B200_hostPlanBlurLists", "T360B200_weightImage", "T360B200_dealLanes",
    "T360B200_remapTable", "T360B200_transformFramePlaneAsync", "T360B200_transformFrameAsync",
    "T360B200_lowPassPlaneAsync", "T360B200_reconfigure", "T360B200_reconfigureAsync", "T360B200_reconfigureWait",
    "T360B200_transformFrameViewAsync", "T360B200_viewSamples",
    "T360B200_transformFrameOrientedAsync", "T360B200_orientedSamples", "T360B200_transformFramePoseAsync", "T360B200_poseSamples",
    "T360B200_lensMap", "T360B200_transformFrameLensAsync", "T360B200_lensBlendMaps", "T360B200_transformFrameLensBlendAsync",
    "T360B200_lensPhotoMaps", "T360B200_transformFrameLensPhotoAsync",
    "T360B200_rectilinearMap", "T360B200_transformFrameRectilinearAsync", "T360B200_cameraMap", "T360B200_transformFrameCameraAsync",
    "T360B200_cameraMipMaps", "T360B200_transformFrameCameraMipAsync", "T360B200_cameraAnisoMaps", "T360B200_transformFrameCameraAnisoAsync",
    "T360B200_cameraPhotoMaps", "T360B200_transformFrameCameraPhotoAsync",
    "T360B200_stereoCameraMaps", "T360B200_transformFrameStereoCameraAsync",
    "T360B200_lensMotionMaps", "T360B200_transformFrameLensMotionAsync", "T360B200_cameraMotionMaps", "T360B200_transformFrameCameraMotionAsync",
    "T360B200_setPinHostPlanes", "T360B200_debugTrace", "T360B200_debugTraceRead", "T360B200_synchronize", "T360B200_stream", "T360B200_kernelLaunchCount", "T360B200_planDeviceBytes",
    "T360B200_planTileCounts", "T360B200_deviceCount", "T360B200_version",
]


class VideoFrameTransform:
    """The opaque handle of the C-ABI with the reference's method names (VideoFrameTransform.h:40-75)."""

    def __init__(self, ctx: FrameTransformContext):
        self._lib = load()
        self.ctx = ctx
        self._h = self._lib.VideoFrameTransform_new(C.byref(ctx))
        if not self._h:
            raise MemoryError("VideoFrameTransform_new returned NULL")

    def close(self):
        if getattr(self, "_h", None):
            self._lib.VideoFrameTransform_delete(self._h)
            self._h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # -- the reference API ------------------------------------------------------------------------
    def generateMapForPlane(self, inputWidth, inputHeight, outputWidth, outputHeight, transformMatPlaneIndex) -> bool:
        return bool(self._lib.VideoFrameTransform_generateMapForPlane(
            self._h, inputWidth, inputHeight, outputWidth, outputHeight, transformMatPlaneIndex))

    def transformFramePlane(self, inputData, outputData, inputWidth, inputHeight, inputWidthWithPadding,
                            outputWidth, outputHeight, outputWidthWithPadding, transformMatPlaneIndex,
                            imagePlaneIndex) -> bool:
        """inputData / outputData: raw addresses (int) of host or CUDA device memory, as in the C call."""
        return bool(self._lib.VideoFrameTransform_transformFramePlane(
            self._h, inputData, outputData, inputWidth, inputHeight, inputWidthWithPadding, outputWidth,
            outputHeight, outputWidthWithPadding, transformMatPlaneIndex, imagePlaneIndex))

    # -- conveniences over numpy planes (host path of the C-ABI) -----------------------------
    def transform_plane(self, src: np.ndarray, out_w: int, out_h: int, plan_index: int, image_plane: int = 0,
                        out: np.ndarray | None = None) -> np.ndarray:
        assert src.dtype == np.uint8 and src.ndim == 2 and src.strides[1] == 1
        if out is None:
            out = np.zeros((out_h, out_w), np.uint8)
        assert out.dtype == np.uint8 and out.shape == (out_h, out_w) and out.strides[1] == 1
        ok = self.transformFramePlane(src.ctypes.data, out.ctypes.data, src.shape[1], src.shape[0], src.strides[0],
                                      out_w, out_h, out.strides[0], plan_index, image_plane)
        if not ok:
            raise RuntimeError("VideoFrameTransform_transformFramePlane returned 0 (message on stdout)")
        return out

    # -- extensions -------------------------------------------------------------------------------
    def transform_plane_async(self, d_in: int, d_out: int, in_w, in_h, in_pitch, out_w, out_h, out_pitch, plan_index,
                              stream: int = 0) -> bool:
        return bool(self._lib.T360B200_transformFramePlaneAsync(self._h, d_in, d_out, in_w, in_h, in_pitch, out_w,
                                                                out_h, out_pitch, plan_index, stream))

    def _frame_call(self, entry: str, in_planes, out_planes, dims):
        """The argument arrays of the frame entry point `entry` for one (input frame, output frame) pair, prebuilt once.
        Returns (n, enqueue): n planes, and enqueue(lead, stream) -> bool, which calls `entry` with the handle, `lead` (the
        arguments up to the planes, n included) and the planes."""
        n, pin, pout, ptrs, keep = _frame_args(in_planes, out_planes, dims)
        fn, h = getattr(self._lib, entry), self._h

        def enqueue(lead, stream, _keep=keep) -> bool:
            return bool(fn(h, *lead, pin, pout, *ptrs, stream))
        return n, enqueue

    def make_frame_call(self, in_planes, out_planes, dims):
        """Prebuilds the argument arrays of T360B200_transformFrameAsync for one (input frame, output frame) pair.
        in_planes / out_planes: per plane (device_address, pitch); dims: per plane (in_w, in_h, out_w, out_h).
        Returns a callable f(stream) -> bool that enqueues the whole frame."""
        n, enqueue = self._frame_call("T360B200_transformFrameAsync", in_planes, out_planes, dims)
        return lambda stream=0: enqueue((n,), stream)

    def make_view_frame_call(self, in_planes, out_planes, dims):
        """Like make_frame_call, for T360B200_transformFrameViewAsync (FLAT_FIXED transforms): returns a callable
        f(view, stream) -> bool that enqueues the whole frame with `view` (a T360View or (yaw, pitch, hfov, vfov))."""
        n, enqueue = self._frame_call("T360B200_transformFrameViewAsync", in_planes, out_planes, dims)
        return lambda view, stream=0: enqueue((C.byref(as_view(view)), n), stream)

    def make_oriented_frame_call(self, in_planes, out_planes, dims):
        """Like make_frame_call, for T360B200_transformFrameOrientedAsync (cube-map, EAC and equirect outputs): returns a
        callable f(orientation, stream) -> bool that enqueues the whole frame with `orientation` (a T360Orientation or
        (yaw, pitch, roll))."""
        n, enqueue = self._frame_call("T360B200_transformFrameOrientedAsync", in_planes, out_planes, dims)
        return lambda orientation, stream=0: enqueue((C.byref(as_orientation(orientation)), n), stream)

    def make_pose_frame_call(self, in_planes, out_planes, dims):
        """Like make_frame_call, for T360B200_transformFramePoseAsync (every output layout): returns a callable
        f(pose, stream) -> bool that enqueues the whole frame with `pose` (a T360Pose or (yaw, pitch, roll, hfov, vfov))."""
        n, enqueue = self._frame_call("T360B200_transformFramePoseAsync", in_planes, out_planes, dims)
        return lambda pose, stream=0: enqueue((C.byref(as_pose(pose)), n), stream)

    def make_lens_frame_call(self, in_planes, out_planes, dims):
        """Like make_frame_call, for T360B200_transformFrameLensAsync (a fisheye lens rig to any sphere output, no plan
        needed): returns a callable f(rig, orientation, stream) -> bool that enqueues the whole frame with `rig` (a
        T360LensRig) and `orientation` (a T360Orientation or (yaw, pitch, roll))."""
        n, enqueue = self._frame_call("T360B200_transformFrameLensAsync", in_planes, out_planes, dims)
        return lambda rig, orientation, stream=0: enqueue((C.byref(rig), C.byref(as_orientation(orientation)), n), stream)

    def make_lens_blend_frame_call(self, in_planes, out_planes, dims):
        """Like make_lens_frame_call, for T360B200_transformFrameLensBlendAsync (a two-lens rig whose seam is feathered
        across a belt of seam_width degrees): returns a callable f(rig, seam_width, orientation, stream) -> bool that
        enqueues the whole frame."""
        n, enqueue = self._frame_call("T360B200_transformFrameLensBlendAsync", in_planes, out_planes, dims)
        return lambda rig, seam_width, orientation, stream=0: enqueue(
            (C.byref(rig), seam_width, C.byref(as_orientation(orientation)), n), stream)

    def make_lens_photo_frame_call(self, in_planes, out_planes, dims):
        """Like make_lens_frame_call, for T360B200_transformFrameLensPhotoAsync (a rig with photometry: each lens's samples
        corrected before the seam, seam_width 0 for the hard seam): returns a callable f(rig, photometry, seam_width,
        orientation, stream, stats=0) -> bool, `photometry` a T360RigPhotometry and `stats` the device address of
        [planes][6] uint64 sums (0: none)."""
        n, enqueue = self._frame_call("T360B200_transformFrameLensPhotoAsync", in_planes, out_planes, dims)
        return lambda rig, photometry, seam_width, orientation, stream=0, stats=0: enqueue(
            (C.byref(rig), C.byref(photometry), seam_width, C.byref(as_orientation(orientation)), stats or None, n), stream)

    def make_lens_motion_frame_call(self, in_planes, out_planes, dims):
        """Like make_lens_photo_frame_call, for T360B200_transformFrameLensMotionAsync (a rig with photometry and a rig
        motion over the readout): returns a callable f(rig, photometry, seam_width, orientation, motion, stream=0, stats=0)
        -> bool, `motion` a T360RigMotion."""
        n, enqueue = self._frame_call("T360B200_transformFrameLensMotionAsync", in_planes, out_planes, dims)
        return lambda rig, photometry, seam_width, orientation, motion, stream=0, stats=0: enqueue(
            (C.byref(rig), C.byref(photometry), seam_width, C.byref(as_orientation(orientation)), C.byref(motion), stats or None, n), stream)

    def make_rectilinear_frame_call(self, in_planes, out_planes, dims):
        """Like make_frame_call, for T360B200_transformFrameRectilinearAsync (a perspective view, no plan needed): returns a
        callable f(pose, stream, rig=None) -> bool that enqueues the whole frame with `pose` (a T360Pose or (yaw, pitch,
        roll, hfov, vfov)), looking into the context's input, or into `rig` (a T360LensRig) when one is given."""
        n, enqueue = self._frame_call("T360B200_transformFrameRectilinearAsync", in_planes, out_planes, dims)
        return lambda pose, stream=0, rig=None: enqueue((C.byref(rig) if rig is not None else None, C.byref(as_pose(pose)), n), stream)

    def make_camera_frame_call(self, in_planes, out_planes, dims):
        """Like make_rectilinear_frame_call, for T360B200_transformFrameCameraAsync: returns a callable f(pose, camera,
        stream, rig=None) -> bool that enqueues the whole frame with `pose` and `camera` (a T360Camera, a T360_CAMERA_*
        model, or (model, pannini))."""
        n, enqueue = self._frame_call("T360B200_transformFrameCameraAsync", in_planes, out_planes, dims)
        return lambda pose, camera, stream=0, rig=None: enqueue(
            (C.byref(rig) if rig is not None else None, C.byref(as_pose(pose)), C.byref(as_camera(camera)), n), stream)

    def make_camera_mip_frame_call(self, in_planes, out_planes, dims):
        """Like make_camera_frame_call, for T360B200_transformFrameCameraMipAsync (an anti-aliased camera view): returns a
        callable f(pose, camera, minify, stream, rig=None) -> bool, `minify` a T360Minify, a max level, or (max_level,
        lod_bias)."""
        n, enqueue = self._frame_call("T360B200_transformFrameCameraMipAsync", in_planes, out_planes, dims)
        return lambda pose, camera, minify, stream=0, rig=None: enqueue(
            (C.byref(rig) if rig is not None else None, C.byref(as_pose(pose)), C.byref(as_camera(camera)),
             C.byref(as_minify(minify)), n), stream)

    def make_camera_aniso_frame_call(self, in_planes, out_planes, dims):
        """Like make_camera_mip_frame_call, for T360B200_transformFrameCameraAnisoAsync (an anisotropic camera view: up to
        max_probes pyramid probes per pixel along its footprint's longer axis): returns a callable f(pose, camera, minify,
        max_probes, stream, rig=None) -> bool, max_probes 1, 2, 4, 8 or 16."""
        n, enqueue = self._frame_call("T360B200_transformFrameCameraAnisoAsync", in_planes, out_planes, dims)
        return lambda pose, camera, minify, max_probes, stream=0, rig=None: enqueue(
            (C.byref(rig) if rig is not None else None, C.byref(as_pose(pose)), C.byref(as_camera(camera)),
             C.byref(as_minify(minify)), max_probes, n), stream)

    def make_camera_photo_frame_call(self, in_planes, out_planes, dims):
        """Like make_camera_mip_frame_call, for T360B200_transformFrameCameraPhotoAsync (a camera view of a rig with
        photometry: each lens's samples corrected before the hard or feathered seam): returns a callable f(rig, photometry,
        seam_width, pose, camera, minify=None, stream=0, stats=0) -> bool, `minify` as for make_camera_mip_frame_call or None
        (no pyramid) and `stats` the device address of [planes][6] uint64 sums (0: none)."""
        n, enqueue = self._frame_call("T360B200_transformFrameCameraPhotoAsync", in_planes, out_planes, dims)
        return lambda rig, photometry, seam_width, pose, camera, minify=None, stream=0, stats=0: enqueue(
            (C.byref(rig), C.byref(photometry), seam_width, C.byref(as_pose(pose)), C.byref(as_camera(camera)),
             C.byref(as_minify(minify)) if minify is not None else None, stats or None, n), stream)

    def make_camera_motion_frame_call(self, in_planes, out_planes, dims):
        """Like make_camera_photo_frame_call, for T360B200_transformFrameCameraMotionAsync (a camera view of a rig with
        photometry and a rig motion over the readout): returns a callable f(rig, photometry, seam_width, pose, camera,
        minify, motion, stream=0, stats=0) -> bool, `minify` None for no pyramid and `motion` a T360RigMotion."""
        n, enqueue = self._frame_call("T360B200_transformFrameCameraMotionAsync", in_planes, out_planes, dims)
        return lambda rig, photometry, seam_width, pose, camera, minify, motion, stream=0, stats=0: enqueue(
            (C.byref(rig), C.byref(photometry), seam_width, C.byref(as_pose(pose)), C.byref(as_camera(camera)),
             C.byref(as_minify(minify)) if minify is not None else None, C.byref(motion), stats or None, n), stream)

    def make_stereo_camera_frame_call(self, in_planes, out_planes, dims):
        """Like make_camera_photo_frame_call, for T360B200_transformFrameStereoCameraAsync (a camera view of a stereo rig:
        eye e of the context's output_stereo_format takes lens e, no seam): returns a callable f(rig, photometry, pose,
        camera, minify=None, stream=0, stats=0) -> bool."""
        n, enqueue = self._frame_call("T360B200_transformFrameStereoCameraAsync", in_planes, out_planes, dims)
        return lambda rig, photometry, pose, camera, minify=None, stream=0, stats=0: enqueue(
            (C.byref(rig), C.byref(photometry), C.byref(as_pose(pose)), C.byref(as_camera(camera)),
             C.byref(as_minify(minify)) if minify is not None else None, stats or None, n), stream)

    def generate_map_from_warp(self, map, in_w: int, in_h: int, plan_index: int, border: int = BORDER_WRAP) -> bool:
        """T360B200_generateMapFromWarp: installs plan index `plan_index` from a caller's warp map (float32 [h][w][2], the
        source x, y of every output pixel) for input planes of in_w x in_h, sampled with the context's interpolation and
        `border` (BORDER_WRAP or BORDER_TRANSPARENT).  Every frame entry point then serves it.  False: refused (message on
        stdout)."""
        m = _warp_map(map)
        return bool(self._lib.T360B200_generateMapFromWarp(self._h, m.ctypes.data, m.shape[1], m.shape[0], in_w, in_h, border,
                                                           plan_index))

    def make_remap_frame_call(self, in_planes, out_planes, dims, border: int = BORDER_WRAP):
        """Like make_frame_call, for T360B200_remapFrameAsync: returns a callable f(maps, stream) -> bool that enqueues the whole
        frame through one device map per plane, each the size of its output plane.  maps: per plane a CUDA float32 tensor
        [out_h][>= out_w][2] (its row stride gives the pitch), a (device address, pitch in bytes) pair, or a device address
        of a dense map."""
        n, enqueue = self._frame_call("T360B200_remapFrameAsync", in_planes, out_planes, dims)
        dense = [8 * d[2] for d in dims]

        def as_map(m, p):
            if hasattr(m, "data_ptr"):
                return m.data_ptr(), m.stride(0) * m.element_size()
            return (int(m[0]), int(m[1])) if isinstance(m, (tuple, list)) else (int(m), dense[p])

        def call(maps, stream: int = 0) -> bool:
            if len(maps) != n:
                raise ValueError(f"{len(maps)} maps for {n} planes")
            desc = [as_map(m, p) for p, m in enumerate(maps)]
            dmaps, pitches = (C.c_void_p * n)(*[d[0] for d in desc]), (C.c_int * n)(*[d[1] for d in desc])
            return enqueue((n, dmaps, pitches, border), stream)
        return call

    def low_pass_async(self, d_in: int, d_out: int, w, h, in_pitch, out_pitch, plan_index, stream: int = 0) -> bool:
        return bool(self._lib.T360B200_lowPassPlaneAsync(self._h, d_in, d_out, w, h, in_pitch, out_pitch, plan_index,
                                                         stream))

    def reconfigure(self, ctx: FrameTransformContext) -> None:
        """Replaces the context of the running transform (T360B200_reconfigure): frames enqueued before the call use the
        old one, frames enqueued after it the new one; every generated plan index keeps its sizes.  Raises on refusal,
        which leaves the old configuration in effect."""
        if not self._lib.T360B200_reconfigure(self._h, C.byref(ctx)):
            raise RuntimeError("T360B200_reconfigure returned 0 (message on stdout); the old configuration is still in effect")
        self.ctx = ctx

    def reconfigure_async(self, ctx: FrameTransformContext) -> None:
        """Replaces the context without waiting for a re-plan (T360B200_reconfigureAsync): frames enqueued after the call
        use `ctx`, served by the per-frame kernels until its plans, made in the background, are in.  Raises on refusal
        (layouts, stereo formats or scale factors changed, unknown interpolation, non-finite fields, a context the
        low-pass planner refuses), which leaves the old context in effect."""
        if not self._lib.T360B200_reconfigureAsync(self._h, C.byref(ctx)):
            raise RuntimeError("T360B200_reconfigureAsync returned 0 (message on stdout); the old context is still in effect")
        self.ctx = ctx

    def reconfigure_wait(self, block: bool = True) -> int:
        """T360B200_reconfigureWait: 1 when the current context's plans are in effect, 0 while they are pending (only with
        block=False), -1 when the background planner failed (frames are still served, by the per-frame kernels)."""
        return self._lib.T360B200_reconfigureWait(self._h, 1 if block else 0)

    def set_pin_host_planes(self, enable: bool) -> None:
        self._lib.T360B200_setPinHostPlanes(self._h, 1 if enable else 0)

    def debug_trace(self, enable: bool) -> None:
        self._lib.T360B200_debugTrace(self._h, 1 if enable else 0)

    def read_trace(self) -> np.ndarray:
        """[groups][64 jobs][wait start, ready, done (ns), kind] of the last whole-frame gather (after a synchronize); the
        library sizes the trace from the device's SM count."""
        buf = np.zeros(int(self._lib.T360B200_debugTraceRead(self._h, None, 0)), np.uint64)
        n = int(self._lib.T360B200_debugTraceRead(self._h, buf.ctypes.data, buf.size)) if buf.size else 0
        return buf[:n].reshape(-1, 64, 4)

    def synchronize(self) -> bool:
        return bool(self._lib.T360B200_synchronize(self._h))

    @property
    def stream(self) -> int:
        return self._lib.T360B200_stream(self._h) or 0

    def plan_tile_counts(self, plan_index):
        """(gather tiles staged via TMA, gather tiles on the general path, low-pass smem jobs, low-pass direct jobs)"""
        c = (C.c_int * 4)()
        if not self._lib.T360B200_planTileCounts(self._h, plan_index, c):
            raise KeyError(plan_index)
        return tuple(c)

    def plan_device_bytes(self, plan_index) -> int:
        return int(self._lib.T360B200_planDeviceBytes(self._h, plan_index))


class HostPlan:
    """Host-side plan of one plane, computed without touching CUDA (T360B200_hostPlan*)."""

    def __init__(self, ctx: FrameTransformContext, in_w, in_h, out_w, out_h, _handle=None):
        self._lib = load()
        self._h = _handle or self._lib.T360B200_hostPlanCreate(C.byref(ctx), in_w, in_h, out_w, out_h)
        if not self._h:
            raise ValueError("T360B200_hostPlanCreate failed (message on stdout)")
        info = (C.c_int * 6)()
        self._lib.T360B200_hostPlanInfo(self._h, info)
        self.map_w, self.map_h, self.num_segments, self.num_taps, self.kernel_size = info[0], info[1], info[2], info[3], info[4]

    @classmethod
    def from_warp(cls, ctx: FrameTransformContext, map, in_w, in_h, border: int = BORDER_WRAP) -> "HostPlan":
        """The host plan T360B200_generateMapFromWarp installs for a caller's warp map (T360B200_hostPlanCreateFromWarp, no
        CUDA).  Raises ValueError when it is refused (message on stdout)."""
        m = _warp_map(map)
        h = load().T360B200_hostPlanCreateFromWarp(C.byref(ctx), m.ctypes.data, m.shape[1], m.shape[0], in_w, in_h, border)
        if not h:
            raise ValueError("T360B200_hostPlanCreateFromWarp failed (message on stdout)")
        return cls(ctx, in_w, in_h, m.shape[1], m.shape[0], _handle=h)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.T360B200_hostPlanDestroy(self._h)
            self._h = None

    __del__ = close

    @property
    def map(self) -> np.ndarray:
        p = self._lib.T360B200_hostPlanMap(self._h)
        n = self.map_w * self.map_h * 2
        return np.frombuffer((C.c_float * n).from_address(p), np.float32).reshape(self.map_h, self.map_w, 2).copy()

    @property
    def samples(self) -> np.ndarray:
        p = self._lib.T360B200_hostPlanSamples(self._h)
        n = self.map_w * self.map_h * 2
        return np.frombuffer((C.c_int32 * n).from_address(p), np.int32).reshape(self.map_h, self.map_w, 2).copy()

    def gather_plan(self):
        """Jobs and record layout the persistent gather kernel works from (T360B200_hostPlanGather).  Returns a dict:
        tiles_per_row, tile_rows, tile_h (grid of the full records), counts {class0, class1, seam, general, share},
        jobs int32[n][4] = {outX, outY | kind << 24, boxX | boxY << 16 | box variant, recordOffset / 16} (None when the plan is not
        staged), records int32[tiles][tile_h][32][2] (full records), compact uint32[] (compact records)."""
        info = (C.c_int * 10)()
        jobs, recs, comp = C.c_void_p(), C.c_void_p(), C.c_void_p()
        if not self._lib.T360B200_hostPlanGather(self._h, info, C.byref(jobs), C.byref(recs), C.byref(comp)):
            raise ValueError("T360B200_hostPlanGather failed")
        tpr, trows, th, nj = info[0], info[1], info[2], info[3]
        n = tpr * trows * th * 32 * 2
        records = np.frombuffer((C.c_int32 * n).from_address(recs.value), np.int32).reshape(tpr * trows, th, 32, 2).copy()
        j = compact = None
        if nj and jobs.value:
            j = np.frombuffer((C.c_int32 * (nj * 4)).from_address(jobs.value), np.int32).reshape(nj, 4).copy()
        if info[9] and comp.value:
            compact = np.frombuffer((C.c_uint32 * info[9]).from_address(comp.value), np.uint32).copy()
        return dict(tiles_per_row=tpr, tile_rows=trows, tile_h=th, jobs=j, records=records, compact=compact,
                    counts=dict(class0=info[4], class1=info[5], seam=info[6], general=info[7], share=info[8]))

    def pole_caps(self):
        """What the frame kernel runs for the general tiles of gather_plan(), and its launch list
        (T360B200_hostPlanPoleCaps).  Returns a dict: counts {cap, border}, jobs int32[n][4] (pole-cap and border jobs,
        record offsets counting on after gather_plan()'s compact records), records uint32[] (their records), launch
        int32[m][4] (the job list the kernel claims from, in launch order)."""
        info = (C.c_int * 4)()
        jobs, recs, launch = C.c_void_p(), C.c_void_p(), C.c_void_p()
        if not self._lib.T360B200_hostPlanPoleCaps(self._h, info, C.byref(jobs), C.byref(recs), C.byref(launch)):
            raise ValueError("T360B200_hostPlanPoleCaps failed")
        n, m = info[0] + info[1], info[3]
        as_jobs = lambda p, k: np.frombuffer((C.c_int32 * (k * 4)).from_address(p.value), np.int32).reshape(k, 4).copy() if k and p.value else np.zeros((0, 4), np.int32)
        records = np.frombuffer((C.c_uint32 * info[2]).from_address(recs.value), np.uint32).copy() if info[2] and recs.value else np.zeros(0, np.uint32)
        return dict(counts=dict(cap=info[0], border=info[1]), jobs=as_jobs(jobs, n), records=records, launch=as_jobs(launch, m))

    def launch_extents(self):
        """What the planner records per job of pole_caps()["launch"] for streaming a host plane through the device
        (T360B200_hostPlanLaunchExtents): a dict of need_rows int32[m] (the source rows [0, n) the job reads) and rects
        int32[m][4] (x0, y0, x1, y1 of the output pixels it writes, exclusive ends)."""
        n, rows, rects = C.c_int(), C.c_void_p(), C.c_void_p()
        if not self._lib.T360B200_hostPlanLaunchExtents(self._h, C.byref(n), C.byref(rows), C.byref(rects)):
            raise ValueError("T360B200_hostPlanLaunchExtents failed")
        m = n.value
        return dict(need_rows=np.frombuffer((C.c_int32 * m).from_address(rows.value), np.int32).copy() if m else np.zeros(0, np.int32),
                    rects=np.frombuffer((C.c_int32 * (4 * m)).from_address(rects.value), np.int32).reshape(m, 4).copy() if m else np.zeros((0, 4), np.int32))

    def waves(self, chunks=None, need_rows=None):
        """The schedule the synchronous host-pointer call streams a large plane of this plan with (T360B200_hostPlanWaves):
        `chunks` input row bands (None: as many as the call takes for the plan's input size), the planner's need-rows or
        `need_rows` (int per launch job) in their place.  Returns a dict: chunks, chunk_row_end int32[chunks], wave_start
        int32[chunks + 1], order int32[m] (launch-job indices wave by wave), rects int32[r][5] (wave, x0, y0, x1, y1 of each
        output rectangle copied back after that wave)."""
        rows = None
        if need_rows is not None:
            rows = np.ascontiguousarray(need_rows, np.int32)
            if rows.shape != (len(self.pole_caps()["launch"]),):
                raise ValueError("need_rows: one value per launch job")
        info = (C.c_int * 3)()
        ends, starts, order, rects = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        if not self._lib.T360B200_hostPlanWaves(self._h, chunks or 0, None if rows is None else rows.ctypes.data, info, C.byref(ends),
                                                C.byref(starts), C.byref(order), C.byref(rects)):
            raise ValueError("T360B200_hostPlanWaves failed")
        c, m, r = info[0], info[1], info[2]
        arr = lambda p, n: np.frombuffer((C.c_int32 * n).from_address(p.value), np.int32).copy() if n and p.value else np.zeros(0, np.int32)
        return dict(chunks=c, chunk_row_end=arr(ends, c), wave_start=arr(starts, c + 1), order=arr(order, m), rects=arr(rects, 5 * r).reshape(r, 5))

    def device_lists(self):
        """The job list and record buffer the frame kernel reads (T360B200_hostPlanDeviceLists): a dict of jobs int32[m][4]
        (pole_caps()["launch"] with the class-0 box width index in bits 28-31 of recordOffset) and records uint32[]
        (compact records, then the pole caps', a narrow box's window offsets at its pitch)."""
        info = (C.c_int * 2)()
        jobs, recs = C.c_void_p(), C.c_void_p()
        if not self._lib.T360B200_hostPlanDeviceLists(self._h, info, C.byref(jobs), C.byref(recs)):
            raise ValueError("T360B200_hostPlanDeviceLists failed")
        j = np.frombuffer((C.c_int32 * (info[0] * 4)).from_address(jobs.value), np.int32).reshape(-1, 4).copy() if info[0] and jobs.value else np.zeros((0, 4), np.int32)
        r = np.frombuffer((C.c_uint32 * info[1]).from_address(recs.value), np.uint32).copy() if info[1] and recs.value else np.zeros(0, np.uint32)
        return dict(jobs=j, records=r)

    def blur_lists(self, *others, width=0, height=0):
        """The low-pass job lists of this plan -- merged with those of `others` (the other planes of a frame) when given --
        for planes of width x height (0: the planned size), as the device holds them (T360B200_hostPlanBlurLists).  Returns
        a dict: image (bytes), strips (3 arrays int32[n][9]: x0, y0, w, h, kxOffset, kxChunks, kxCount, kyOffset, edge),
        tiles, direct (int32[n][8]: x0, y0, w, h, kxOffset, kxCount, kyOffset, kyCount), taps (float32), offsets (byte
        offsets of strips 1..3, tiles, direct, taps), tile_smem, needs_clear."""
        plans = (C.c_void_p * (1 + len(others)))(self._h, *[o._h for o in others])
        lay, img = (C.c_int * 15)(), C.c_void_p()
        if not self._lib.T360B200_hostPlanBlurLists(plans, len(plans), width, height, lay, C.byref(img)):
            raise ValueError("T360B200_hostPlanBlurLists failed (message on stdout)")
        image = C.string_at(img.value, lay[14]) if lay[14] else b""
        arr = lambda at, n, cols, dt: np.frombuffer(image, dt, n * cols, at).reshape(n, cols).copy()
        return dict(image=image, strips=[arr(lay[8 + c], lay[c], 9, np.int32) for c in range(3)], tiles=arr(lay[11], lay[3], 8, np.int32),
                    direct=arr(lay[12], lay[4], 8, np.int32), taps=np.frombuffer(image, np.float32, lay[5], lay[13]).copy(),
                    offsets=list(lay[8:14]), tile_smem=lay[6], needs_clear=bool(lay[7]))

    def segments(self):
        out = []
        rect, nk = (C.c_int * 4)(), (C.c_int * 2)()
        kx, ky = C.c_void_p(), C.c_void_p()
        for i in range(self.num_segments):
            assert self._lib.T360B200_hostPlanSegment(self._h, i, rect, nk, C.byref(kx), C.byref(ky))
            a = np.frombuffer((C.c_float * nk[0]).from_address(kx.value), np.float32).copy()
            b = np.frombuffer((C.c_float * nk[1]).from_address(ky.value), np.float32).copy()
            out.append((rect[0], rect[1], rect[2], rect[3], a, b))
        return out


def view_samples(ctx: FrameTransformContext, view, in_w, in_h, out_w, out_h) -> np.ndarray:
    """The sampling records the per-view kernel computes for one plane (T360B200_viewSamples, no CUDA):
    int32 [map_h][map_w][2] like HostPlan.samples."""
    return _samples(load().T360B200_viewSamples, ctx, as_view(view), in_w, in_h, out_w, out_h)


def oriented_samples(ctx: FrameTransformContext, orientation, in_w, in_h, out_w, out_h) -> np.ndarray:
    """The sampling records the per-frame orientation kernel computes for one plane (T360B200_orientedSamples, no CUDA):
    int32 [map_h][map_w][2] like HostPlan.samples."""
    return _samples(load().T360B200_orientedSamples, ctx, as_orientation(orientation), in_w, in_h, out_w, out_h)


def pose_samples(ctx: FrameTransformContext, pose, in_w, in_h, out_w, out_h) -> np.ndarray:
    """The sampling records the per-frame kernels compute for one plane with `pose` (T360B200_poseSamples, no CUDA):
    int32 [map_h][map_w][2] like HostPlan.samples."""
    return _samples(load().T360B200_poseSamples, ctx, as_pose(pose), in_w, in_h, out_w, out_h)


def lens_map(ctx: FrameTransformContext, rig: T360LensRig, orientation, in_w, in_h, out_w, out_h) -> np.ndarray:
    """The CV_32FC2 map of one plane of a fisheye lens rig (T360B200_lensMap, no CUDA): float32 [out_h][out_w][2], the
    source x, y of every output pixel in a plane of in_w x in_h, NaN where no lens covers it.  generate_map_from_warp(map,
    in_w, in_h, index, BORDER_TRANSPARENT) plans it for a fixed pose."""
    out = np.zeros((max(out_h, 0), max(out_w, 0), 2), np.float32)
    if not load().T360B200_lensMap(C.byref(ctx), C.byref(rig), C.byref(as_orientation(orientation)), in_w, in_h, out_w, out_h,
                                   out.ctypes.data):
        raise ValueError("T360B200_lensMap refused the arguments (message on stdout)")
    return out


def lens_blend_maps(ctx: FrameTransformContext, rig: T360LensRig, seam_width, orientation, in_w, in_h, out_w,
                    out_h) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """The host twin of one plane of a two-lens rig with a feathered seam (T360B200_lensBlendMaps, no CUDA): (map0, map1,
    weight).  map0 / map1: float32 [out_h][out_w][2] CV_32FC2 maps of lens 0 / lens 1, NaN where that lens does not
    contribute; weight: uint16 [out_h][out_w], the weight w (0..256) of lens 1.  cv::remap of each map under
    BORDER_TRANSPARENT, blended as (a (256 - w) + b w + 128) >> 8 where both are sampled, gives the frame call's plane."""
    shape = (max(out_h, 0), max(out_w, 0))
    map0, map1, weight = np.zeros(shape + (2,), np.float32), np.zeros(shape + (2,), np.float32), np.zeros(shape, np.uint16)
    if not load().T360B200_lensBlendMaps(C.byref(ctx), C.byref(rig), seam_width, C.byref(as_orientation(orientation)), in_w, in_h,
                                         out_w, out_h, map0.ctypes.data, map1.ctypes.data, weight.ctypes.data):
        raise ValueError("T360B200_lensBlendMaps refused the arguments (message on stdout)")
    return map0, map1, weight


def lens_photo_maps(ctx: FrameTransformContext, rig: T360LensRig, photometry: T360RigPhotometry, seam_width, orientation, plane, in_w, in_h,
                    out_w, out_h) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """The host twin of one plane (0 luma, 1 and 2 chroma) of a rig with photometry (T360B200_lensPhotoMaps, no CUDA):
    (map0, map1, weight, gain0, gain1).  map0 / map1: float32 [out_h][out_w][2] CV_32FC2 maps of lens 0 / lens 1, NaN where
    that lens does not cover the pixel; weight: uint16, w of lens 1 (0 or 256 with seam_width 0, the hard seam); gain0 /
    gain1: uint16, each lens's Gq (4096 = 1), 0 where it does not cover the pixel."""
    map0, map1 = np.empty((out_h, out_w, 2), np.float32), np.empty((out_h, out_w, 2), np.float32)
    weight, gain0, gain1 = (np.empty((out_h, out_w), np.uint16) for _ in range(3))
    if not load().T360B200_lensPhotoMaps(C.byref(ctx), C.byref(rig), C.byref(photometry), seam_width, C.byref(as_orientation(orientation)),
                                         plane, in_w, in_h, out_w, out_h, map0.ctypes.data, map1.ctypes.data, weight.ctypes.data,
                                         gain0.ctypes.data, gain1.ctypes.data):
        raise ValueError("T360B200_lensPhotoMaps refused the arguments (message on stdout)")
    return map0, map1, weight, gain0, gain1


def lens_motion_maps(ctx: FrameTransformContext, rig: T360LensRig, photometry: T360RigPhotometry, seam_width, orientation,
                     motion: T360RigMotion, plane, in_w, in_h, out_w, out_h) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """The host twin of one plane of a rig with photometry and a rig motion over the readout (T360B200_lensMotionMaps, no
    CUDA): lens_photo_maps' (map0, map1, weight, gain0, gain1) with each lens's M following the readout time of its point."""
    map0, map1 = np.empty((out_h, out_w, 2), np.float32), np.empty((out_h, out_w, 2), np.float32)
    weight, gain0, gain1 = (np.empty((out_h, out_w), np.uint16) for _ in range(3))
    if not load().T360B200_lensMotionMaps(C.byref(ctx), C.byref(rig), C.byref(photometry), seam_width, C.byref(as_orientation(orientation)),
                                          C.byref(motion), plane, in_w, in_h, out_w, out_h, map0.ctypes.data, map1.ctypes.data,
                                          weight.ctypes.data, gain0.ctypes.data, gain1.ctypes.data):
        raise ValueError("T360B200_lensMotionMaps refused the arguments (message on stdout)")
    return map0, map1, weight, gain0, gain1


def rectilinear_map(ctx: FrameTransformContext, pose, in_w, in_h, out_w, out_h, rig: T360LensRig | None = None) -> np.ndarray:
    """The CV_32FC2 map of one plane of a rectilinear view (T360B200_rectilinearMap, no CUDA): float32 [out_h][out_w][2],
    the source x, y of every output pixel in a plane of in_w x in_h, from the context's input, or from `rig` (NaN where no
    lens covers the pixel).  generate_map_from_warp(map, in_w, in_h, index, BORDER_WRAP, or BORDER_TRANSPARENT with a rig)
    plans it for a fixed pose."""
    out = np.zeros((max(out_h, 0), max(out_w, 0), 2), np.float32)
    if not load().T360B200_rectilinearMap(C.byref(ctx), C.byref(rig) if rig is not None else None, C.byref(as_pose(pose)), in_w, in_h,
                                          out_w, out_h, out.ctypes.data):
        raise ValueError("T360B200_rectilinearMap refused the arguments (message on stdout)")
    return out


def camera_map(ctx: FrameTransformContext, pose, camera, in_w, in_h, out_w, out_h, rig: T360LensRig | None = None) -> np.ndarray:
    """rectilinear_map with a camera model (T360B200_cameraMap, no CUDA): `camera` a T360Camera, a T360_CAMERA_* model, or
    (model, pannini).  generate_map_from_warp plans it for a fixed pose and camera as it plans rectilinear_map's map."""
    out = np.zeros((max(out_h, 0), max(out_w, 0), 2), np.float32)
    if not load().T360B200_cameraMap(C.byref(ctx), C.byref(rig) if rig is not None else None, C.byref(as_pose(pose)),
                                     C.byref(as_camera(camera)), in_w, in_h, out_w, out_h, out.ctypes.data):
        raise ValueError("T360B200_cameraMap refused the arguments (message on stdout)")
    return out


def camera_mip_maps(ctx: FrameTransformContext, pose, camera, minify, in_w, in_h, out_w, out_h,
                    rig: T360LensRig | None = None) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """The host twin of one plane of an anti-aliased camera view (T360B200_cameraMipMaps, no CUDA): (map0, map1, level,
    weight).  map0 / map1: float32 [out_h][out_w][2], each pixel's entry in its level's pixels / in the next level's (NaN
    where the weight is 0); level: uint8 [out_h][out_w]; weight: uint16, the next level's weight w (0..255).  cv::remap of
    each level's entries over the pyramid (cv::resize with INTER_AREA, repeated: mip_level_sizes), blended as
    (a (256 - w) + b w + 128) >> 8, gives the frame call's plane."""
    shape = (max(out_h, 0), max(out_w, 0))
    map0, map1 = np.zeros(shape + (2,), np.float32), np.zeros(shape + (2,), np.float32)
    level, weight = np.zeros(shape, np.uint8), np.zeros(shape, np.uint16)
    if not load().T360B200_cameraMipMaps(C.byref(ctx), C.byref(rig) if rig is not None else None, C.byref(as_pose(pose)),
                                         C.byref(as_camera(camera)), C.byref(as_minify(minify)), in_w, in_h, out_w, out_h,
                                         map0.ctypes.data, map1.ctypes.data, level.ctypes.data, weight.ctypes.data):
        raise ValueError("T360B200_cameraMipMaps refused the arguments (message on stdout)")
    return map0, map1, level, weight


def camera_aniso_maps(ctx: FrameTransformContext, pose, camera, minify, max_probes, in_w, in_h, out_w, out_h,
                      rig: T360LensRig | None = None) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """The host twin of one plane of an anisotropic camera view (T360B200_cameraAnisoMaps, no CUDA): (map0, map1, level,
    weight, probes).  map0 / map1: float32 [max_probes][out_h][out_w][2], probe k's entry in the pixel's level's pixels /
    in the next level's (map1 NaN where the weight is 0, both NaN for k >= probes); level: uint8 [out_h][out_w]; weight:
    uint16, the next level's weight w (0..255), shared by the probes; probes: uint8, the pixel's probe count N.  Each
    probe is camera_mip_maps' composite of its entries; the pixel is their mean (sum + N / 2) // N, with a rig over the
    probes not skipped.  max_probes 1 gives camera_mip_maps' arrays as probe 0."""
    shape = (max(out_h, 0), max(out_w, 0))
    k = max_probes if max_probes in (1, 2, 4, 8, 16) else 1  # (the call refuses other values before it writes)
    map0, map1 = np.zeros((k,) + shape + (2,), np.float32), np.zeros((k,) + shape + (2,), np.float32)
    level, weight, probes = np.zeros(shape, np.uint8), np.zeros(shape, np.uint16), np.zeros(shape, np.uint8)
    if not load().T360B200_cameraAnisoMaps(C.byref(ctx), C.byref(rig) if rig is not None else None, C.byref(as_pose(pose)),
                                           C.byref(as_camera(camera)), C.byref(as_minify(minify)), max_probes, in_w, in_h, out_w, out_h,
                                           map0.ctypes.data, map1.ctypes.data, level.ctypes.data, weight.ctypes.data, probes.ctypes.data):
        raise ValueError("T360B200_cameraAnisoMaps refused the arguments (message on stdout)")
    return map0, map1, level, weight, probes


def camera_photo_maps(ctx: FrameTransformContext, rig: T360LensRig, photometry: T360RigPhotometry, seam_width, pose, camera, minify, lens,
                      plane, in_w, in_h, out_w, out_h) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """The host twin of one lens (0 or 1) of one plane (0 luma, 1 and 2 chroma) of a camera view of a rig with photometry
    (T360B200_cameraPhotoMaps, no CUDA): (map0, map1, level, weight, gain, seam_weight).  The first four are
    camera_mip_maps' arrays for that lens (NaN entries, level 0 and weight 0 where it does not cover the pixel's ray); gain:
    uint16, the lens's Gq (4096 = 1, 0 where it does not cover the ray); seam_weight: uint16, w of lens 1 (0 or 256 with
    seam_width 0, the hard seam).  minify as for camera_mip_maps, or None: no pyramid."""
    shape = (max(out_h, 0), max(out_w, 0))
    map0, map1 = np.zeros(shape + (2,), np.float32), np.zeros(shape + (2,), np.float32)
    level = np.zeros(shape, np.uint8)
    weight, gain, seam_weight = (np.zeros(shape, np.uint16) for _ in range(3))
    if not load().T360B200_cameraPhotoMaps(C.byref(ctx), C.byref(rig), C.byref(photometry), seam_width, C.byref(as_pose(pose)),
                                           C.byref(as_camera(camera)), C.byref(as_minify(minify)) if minify is not None else None, lens,
                                           plane, in_w, in_h, out_w, out_h, map0.ctypes.data, map1.ctypes.data, level.ctypes.data,
                                           weight.ctypes.data, gain.ctypes.data, seam_weight.ctypes.data):
        raise ValueError("T360B200_cameraPhotoMaps refused the arguments (message on stdout)")
    return map0, map1, level, weight, gain, seam_weight


def camera_motion_maps(ctx: FrameTransformContext, rig: T360LensRig, photometry: T360RigPhotometry, seam_width, pose, camera, minify,
                       motion: T360RigMotion, lens, plane, in_w, in_h, out_w, out_h) -> tuple[np.ndarray, ...]:
    """The host twin of one lens of one plane of a camera view of a rig with photometry and a rig motion
    (T360B200_cameraMotionMaps, no CUDA): camera_photo_maps' (map0, map1, level, weight, gain, seam_weight)."""
    shape = (max(out_h, 0), max(out_w, 0))
    map0, map1 = np.zeros(shape + (2,), np.float32), np.zeros(shape + (2,), np.float32)
    level = np.zeros(shape, np.uint8)
    weight, gain, seam_weight = (np.zeros(shape, np.uint16) for _ in range(3))
    if not load().T360B200_cameraMotionMaps(C.byref(ctx), C.byref(rig), C.byref(photometry), seam_width, C.byref(as_pose(pose)),
                                            C.byref(as_camera(camera)), C.byref(as_minify(minify)) if minify is not None else None,
                                            C.byref(motion), lens, plane, in_w, in_h, out_w, out_h, map0.ctypes.data, map1.ctypes.data,
                                            level.ctypes.data, weight.ctypes.data, gain.ctypes.data, seam_weight.ctypes.data):
        raise ValueError("T360B200_cameraMotionMaps refused the arguments (message on stdout)")
    return map0, map1, level, weight, gain, seam_weight


def stereo_camera_maps(ctx: FrameTransformContext, rig: T360LensRig, photometry: T360RigPhotometry, pose, camera, minify, lens, plane,
                       in_w, in_h, out_w, out_h) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """The host twin of one lens (0 or 1) of one plane of a camera view of a stereo rig (T360B200_stereoCameraMaps, no
    CUDA): (map0, map1, level, weight, gain, eye_weight), camera_photo_maps' arrays for that lens wherever it covers the
    ray, and eye_weight (uint16) 0 on eye-0 pixels and 256 on eye-1 pixels.  minify as for camera_mip_maps, or None."""
    shape = (max(out_h, 0), max(out_w, 0))
    map0, map1 = np.zeros(shape + (2,), np.float32), np.zeros(shape + (2,), np.float32)
    level = np.zeros(shape, np.uint8)
    weight, gain, eye_weight = (np.zeros(shape, np.uint16) for _ in range(3))
    if not load().T360B200_stereoCameraMaps(C.byref(ctx), C.byref(rig), C.byref(photometry), C.byref(as_pose(pose)), C.byref(as_camera(camera)),
                                            C.byref(as_minify(minify)) if minify is not None else None, lens, plane, in_w, in_h, out_w, out_h,
                                            map0.ctypes.data, map1.ctypes.data, level.ctypes.data, weight.ctypes.data, gain.ctypes.data,
                                            eye_weight.ctypes.data):
        raise ValueError("T360B200_stereoCameraMaps refused the arguments (message on stdout)")
    return map0, map1, level, weight, gain, eye_weight


def square_pixel_vfov(hfov, width, height) -> float:
    """The vfov in degrees that gives a width x height rectilinear view with horizontal field of view `hfov` square pixels:
    tan(vfov / 2) = tan(hfov / 2) height / width."""
    return float(np.degrees(2.0 * np.arctan(np.tan(np.radians(hfov) / 2.0) * height / width)))


def remap_table(interpolation_alg: int) -> np.ndarray | None:
    L = load()
    p = C.c_void_p()
    k = L.T360B200_remapTable(interpolation_alg, C.byref(p))
    if k < 2:
        return None
    return np.frombuffer((C.c_int16 * (1024 * k * k)).from_address(p.value), np.int16).reshape(1024, k, k).copy()


def deal_lanes(interpolation_alg: int, phases) -> tuple[int, np.ndarray, np.ndarray]:
    """(modelled wavefronts of a weight load, lane of every pixel, table copy of every pixel) for one warp step."""
    L = load()
    ph = np.ascontiguousarray(phases, np.int32)
    lane, copy = np.zeros(ph.size, np.int32), np.zeros(ph.size, np.int32)
    L.T360B200_dealLanes.restype = C.c_int
    L.T360B200_dealLanes.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    w = L.T360B200_dealLanes(interpolation_alg, ph.size, ph.ctypes.data, lane.ctypes.data, copy.ctypes.data)
    if w < 0:
        raise ValueError("T360B200_dealLanes refused the arguments")
    return int(w), lane, copy


def weight_image(interpolation_alg: int) -> np.ndarray | None:
    """The frame kernel's shared-memory image of the interpolation table (bytes)."""
    L = load()
    p = C.c_void_p()
    n = L.T360B200_weightImage(interpolation_alg, C.byref(p))
    if n <= 0:
        return None
    return np.frombuffer((C.c_uint8 * n).from_address(p.value), np.uint8).copy()


def kernel_launch_count() -> int:
    return int(load().T360B200_kernelLaunchCount())


def device_count() -> int:
    return int(load().T360B200_deviceCount())
