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
    L.T360B200_weightImage.restype = ci
    L.T360B200_weightImage.argtypes = [ci, C.POINTER(vp)]
    L.T360B200_remapTable.restype = ci
    L.T360B200_remapTable.argtypes = [ci, C.POINTER(vp)]
    L.T360B200_transformFramePlaneAsync.restype = ci
    L.T360B200_transformFramePlaneAsync.argtypes = [vp, vp, vp] + [ci] * 7 + [vp]
    L.T360B200_transformFrameAsync.restype = ci
    L.T360B200_transformFrameAsync.argtypes = [vp, ci, vp, vp] + [vp] * 6 + [vp]
    L.T360B200_lowPassPlaneAsync.restype = ci
    L.T360B200_lowPassPlaneAsync.argtypes = [vp, vp, vp] + [ci] * 5 + [vp]
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
    "VideoFrameTransform_transformFramePlane", "T360B200_hostPlanCreate", "T360B200_hostPlanDestroy",
    "T360B200_hostPlanInfo", "T360B200_hostPlanMap", "T360B200_hostPlanSamples", "T360B200_hostPlanSegment",
    "T360B200_hostPlanGather", "T360B200_weightImage", "T360B200_dealLanes",
    "T360B200_remapTable", "T360B200_transformFramePlaneAsync", "T360B200_transformFrameAsync",
    "T360B200_lowPassPlaneAsync",
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

    def make_frame_call(self, in_planes, out_planes, dims):
        """Prebuilds the argument arrays of T360B200_transformFrameAsync for one (input frame, output frame) pair.
        in_planes / out_planes: per plane (device_address, pitch); dims: per plane (in_w, in_h, out_w, out_h).
        Returns a callable f(stream) -> bool that enqueues the whole frame."""
        n = len(in_planes)
        VP, IA = C.c_void_p * n, C.c_int * n
        d_in = VP(*[p[0] for p in in_planes])
        d_out = VP(*[p[0] for p in out_planes])
        arrs = [IA(*[d[0] for d in dims]), IA(*[d[1] for d in dims]), IA(*[p[1] for p in in_planes]),
                IA(*[d[2] for d in dims]), IA(*[d[3] for d in dims]), IA(*[p[1] for p in out_planes])]
        fn, h = self._lib.T360B200_transformFrameAsync, self._h
        ptrs = [C.cast(a, C.c_void_p) for a in arrs]
        pin, pout = C.cast(d_in, C.c_void_p), C.cast(d_out, C.c_void_p)

        def call(stream: int = 0, _keep=(d_in, d_out, arrs)) -> bool:
            return bool(fn(h, n, pin, pout, *ptrs, stream))
        return call

    def low_pass_async(self, d_in: int, d_out: int, w, h, in_pitch, out_pitch, plan_index, stream: int = 0) -> bool:
        return bool(self._lib.T360B200_lowPassPlaneAsync(self._h, d_in, d_out, w, h, in_pitch, out_pitch, plan_index,
                                                         stream))

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

    def __init__(self, ctx: FrameTransformContext, in_w, in_h, out_w, out_h):
        self._lib = load()
        self._h = self._lib.T360B200_hostPlanCreate(C.byref(ctx), in_w, in_h, out_w, out_h)
        if not self._h:
            raise ValueError("T360B200_hostPlanCreate failed (message on stdout)")
        info = (C.c_int * 6)()
        self._lib.T360B200_hostPlanInfo(self._h, info)
        self.map_w, self.map_h, self.num_segments, self.num_taps, self.kernel_size = info[0], info[1], info[2], info[3], info[4]

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
