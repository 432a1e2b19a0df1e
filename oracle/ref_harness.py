"""oracle/ref_harness.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Drives ``oracle/_ref/libt360ref.so`` -- the reference's own, unmodified
``VideoFrameTransform.cpp`` / ``VideoFrameTransformHandler.cpp`` compiled against
``oracle/shim/opencv2/opencv.hpp`` -- and points the shim's three pixel hooks
(``cv::remap``, ``cv::sepFilter2D``, ``cv::resize``; reference call sites
VideoFrameTransform.cpp:189-197, 748-754, 763-776) at the real OpenCV in this
image (``cv2`` 4.13.0).  The result is "the reference itself, run here": its
geometry, its low-pass plan, its per-frame control flow, OpenCV's arithmetic.

Only tests/, __graft_entry__.smoke() and bench.py's reference / cpu_baseline
legs may import this module.  Nothing in transform360_b200/ does.
"""
from __future__ import annotations

import ctypes as C
import os
import threading
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
REF_SO = _HERE / "_ref" / "libt360ref.so"

# ---- ABI mirror (reference VideoFrameTransformHelper.h:18-90) -----------------------------
LAYOUT_CUBEMAP_32, LAYOUT_CUBEMAP_23_OFFCENTER, LAYOUT_FLAT_FIXED, LAYOUT_EQUIRECT = 0, 1, 2, 3
LAYOUT_BARREL, LAYOUT_BARREL_SPLIT, LAYOUT_EAC_32, LAYOUT_N = 4, 5, 6, 7
STEREO_FORMAT_TB, STEREO_FORMAT_LR, STEREO_FORMAT_MONO, STEREO_FORMAT_GUESS, STEREO_FORMAT_N = 0, 1, 2, 3, 4
NEAREST, LINEAR, CUBIC, LANCZOS4 = 0, 1, 2, 4


class FrameTransformContext(C.Structure):
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


def default_context(**overrides) -> FrameTransformContext:
    """Filter defaults of the reference's AVOption table (vf_transform360.c:407-987)."""
    ctx = FrameTransformContext(
        input_layout=LAYOUT_EQUIRECT, output_layout=LAYOUT_CUBEMAP_32,
        input_stereo_format=STEREO_FORMAT_MONO, output_stereo_format=STEREO_FORMAT_MONO,
        vflip=0, input_expand_coef=1.01, expand_coef=1.01, interpolation_alg=CUBIC,
        width_scale_factor=1.0, height_scale_factor=1.0, fixed_yaw=0.0, fixed_pitch=0.0,
        fixed_roll=0.0, fixed_hfov=120.0, fixed_vfov=110.0, fixed_cube_offcenter_x=0.0,
        fixed_cube_offcenter_y=0.0, fixed_cube_offcenter_z=0.0, is_horizontal_offset=0,
        enable_low_pass_filter=1, kernel_height_scale_factor=1.0, min_kernel_half_height=1.0,
        max_kernel_half_height=10000.0, enable_multi_threading=1, num_vertical_segments=5,
        num_horizontal_segments=1, adjust_kernel=1, kernel_adjust_factor=1.0)
    for k, v in overrides.items():
        if not hasattr(ctx, k):
            raise AttributeError(k)
        setattr(ctx, k, v)
    return ctx


# ---- synthetic inputs and hashes (SURVEY.md 8d / Appendix D) --------------------------------
def fmix32(h: np.ndarray) -> np.ndarray:
    h = h.astype(np.uint32)
    h ^= h >> np.uint32(16)
    h *= np.uint32(0x85EBCA6B)
    h ^= h >> np.uint32(13)
    h *= np.uint32(0xC2B2AE35)
    h ^= h >> np.uint32(16)
    return h


def noise_plane(w: int, h: int, plane: int = 0, frame: int = 0) -> np.ndarray:
    """v(x,y) = fmix32((x + y*W + plane*W*H + frame*0x9E3779B9) mod 2^32) >> 24, uint8 [h][w]."""
    with np.errstate(over="ignore"):
        idx = np.arange(w * h, dtype=np.uint64)
        idx = (idx + np.uint64(plane) * np.uint64(w * h) + np.uint64(frame) * np.uint64(0x9E3779B9)) & np.uint64(0xFFFFFFFF)
        v = fmix32(idx.astype(np.uint32)) >> np.uint32(24)
    return v.astype(np.uint8).reshape(h, w)


def fnv1a64(buf: bytes | np.ndarray) -> str:
    """FNV-1a 64 over raw bytes (vectorised by 8-bit steps is impossible; use a C loop via numpy-free python for small, chunked ctypes for large)."""
    data = np.ascontiguousarray(buf).view(np.uint8).ravel() if isinstance(buf, np.ndarray) else np.frombuffer(buf, np.uint8)
    lib = _oracle_lib_for_hash()
    if lib is not None:
        return "%016x" % lib.t360o_fnv1a64(data.ctypes.data_as(C.c_void_p), C.c_size_t(data.size))
    h = 0xCBF29CE484222325
    for b in data.tobytes():
        h = ((h ^ b) * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
    return "%016x" % h


_hash_lib = None


def _oracle_lib_for_hash():
    global _hash_lib
    if _hash_lib is None:
        p = _HERE / "libt360oracle.so"
        if p.exists():
            _hash_lib = C.CDLL(str(p))
            _hash_lib.t360o_fnv1a64.restype = C.c_uint64
            _hash_lib.t360o_fnv1a64.argtypes = [C.c_void_p, C.c_size_t]
        else:
            _hash_lib = False
    return _hash_lib or None


def sha16(a: np.ndarray) -> str:
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


# ---- cv2 hooks ---------------------------------------------------------------------------------
_REMAP_T = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.c_int, C.c_int,
                       C.c_size_t, C.c_void_p, C.c_size_t, C.c_int, C.c_int)
_SEP_T = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int,
                     C.c_void_p, C.c_size_t, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int)
_RESIZE_T = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.c_int, C.c_int,
                        C.c_size_t, C.c_int)


def _as_u8(ptr, rows, cols, step):
    buf = (C.c_uint8 * (step * (rows - 1) + cols)).from_address(ptr)
    return np.lib.stride_tricks.as_strided(np.frombuffer(buf, np.uint8), shape=(rows, cols), strides=(step, 1))


def _remap_hook(src, srows, scols, sstep, dst, drows, dcols, dstep, mp, mstep, interp, border):
    try:
        import cv2
        s = _as_u8(src, srows, scols, sstep)
        d = _as_u8(dst, drows, dcols, dstep)
        mbuf = (C.c_float * ((mstep // 4) * (drows - 1) + dcols * 2)).from_address(mp)
        m = np.lib.stride_tricks.as_strided(np.frombuffer(mbuf, np.float32), shape=(drows, dcols, 2),
                                            strides=(mstep, 8, 4))
        # write straight into the caller's plane (a strided view is a valid cv::Mat); under
        # BORDER_TRANSPARENT dst keeps its previous content where unmapped
        out = cv2.remap(s, m, None, interp, dst=d, borderMode=border)
        if not np.shares_memory(out, d):
            d[...] = out
        # the reference remaps a plane right after it has filtered all of its tiles (cpp:727-754): the whole-plane
        # low-pass results cached for that plane (keyed by its address) are dead now, and must not be found again
        # when a later plane or frame is allocated at the same address
        with _sep_lock:
            _SEP_CACHE.clear()
        return 0
    except Exception as e:  # pragma: no cover
        print("remap hook error:", e)
        return 1


# cv2's optimized sepFilter2D mixes fused and unfused multiply-adds depending on where a pixel falls
# in its unrolled loops (whole-plane vs cropped-region calls differ in ~10 px of an 8K plane, always by
# 1 LSB at a rounding tie).  To keep "the reference run here" deterministic, and equal to the
# known-answer hashes of SURVEY.md Appendix D, the hook filters the WHOLE parent plane once per distinct
# (kx, ky) pair and copies each tile out of the matching result (SURVEY.md 8c pitfall i).  When a plan
# has too many distinct kernels for that to be affordable it falls back to filtering the tile grown by
# the kernel half-widths (clipped to the parent, where BORDER_REPLICATE then applies), and cropping.
_SEP_CACHE: dict = {}
_SEP_CACHE_MAX = 48
_sep_lock = threading.Lock()


def _sep_hook(parent, prow, pcol, pstep, rx, ry, rw, rh, dst, dstep, kx, nkx, ky, nky, border):
    try:
        import cv2
        p = _as_u8(parent, prow, pcol, pstep)
        d = _as_u8(dst, rh, rw, dstep)
        kxa = np.frombuffer((C.c_float * nkx).from_address(kx), np.float32).reshape(1, -1).copy()
        kya = np.frombuffer((C.c_float * nky).from_address(ky), np.float32).reshape(1, -1).copy()
        key = (parent, prow, pcol, pstep, kxa.tobytes(), kya.tobytes(), border)
        with _sep_lock:
            full = _SEP_CACHE.get(key)
            if full is None and len(_SEP_CACHE) < _SEP_CACHE_MAX:
                full = cv2.sepFilter2D(np.ascontiguousarray(p), -1, kxa, kya, anchor=(-1, -1), delta=0,
                                       borderType=border)
                _SEP_CACHE[key] = full
        if full is not None:
            d[...] = full[ry:ry + rh, rx:rx + rw]
            return 0
        hx, hy = nkx // 2, nky // 2
        x0, y0 = max(0, rx - hx), max(0, ry - hy)
        x1, y1 = min(pcol, rx + rw + hx), min(prow, ry + rh + hy)
        region = np.ascontiguousarray(p[y0:y1, x0:x1])
        out = cv2.sepFilter2D(region, -1, kxa, kya, anchor=(-1, -1), delta=0, borderType=border)
        d[...] = out[ry - y0: ry - y0 + rh, rx - x0: rx - x0 + rw]
        return 0
    except Exception as e:  # pragma: no cover
        print("sepFilter2D hook error:", e)
        return 1


def _resize_hook(src, srows, scols, sstep, dst, drows, dcols, dstep, interp):
    try:
        import cv2
        s = np.ascontiguousarray(_as_u8(src, srows, scols, sstep))
        d = _as_u8(dst, drows, dcols, dstep)
        d[...] = cv2.resize(s, (dcols, drows), interpolation=interp)
        return 0
    except Exception as e:  # pragma: no cover
        print("resize hook error:", e)
        return 1


_lib = None
_hooks_keepalive = None
_lock = threading.Lock()


def ref_available() -> bool:
    return REF_SO.exists()


def ref_lib():
    """Loads the compiled reference and installs the cv2 hooks (once)."""
    global _lib, _hooks_keepalive
    with _lock:
        if _lib is not None:
            return _lib
        if not REF_SO.exists():
            raise FileNotFoundError(f"{REF_SO} missing: run `make -C oracle ref` where the reference sources exist (REF=... FILTER=...)")
        lib = C.CDLL(str(REF_SO), mode=os.RTLD_LOCAL)
        vp = C.c_void_p
        lib.VideoFrameTransform_new.restype = vp
        lib.VideoFrameTransform_new.argtypes = [C.POINTER(FrameTransformContext)]
        lib.VideoFrameTransform_delete.restype = None
        lib.VideoFrameTransform_delete.argtypes = [vp]
        lib.VideoFrameTransform_generateMapForPlane.restype = C.c_int
        lib.VideoFrameTransform_generateMapForPlane.argtypes = [vp] + [C.c_int] * 5
        lib.VideoFrameTransform_transformFramePlane.restype = C.c_int
        lib.VideoFrameTransform_transformFramePlane.argtypes = [vp, vp, vp] + [C.c_int] * 8
        lib.t360ref_map.restype = vp
        lib.t360ref_map.argtypes = [vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_size_t)]
        lib.t360ref_num_segments.restype = C.c_int
        lib.t360ref_num_segments.argtypes = [vp, C.c_int]
        lib.t360ref_segment.restype = C.c_int
        lib.t360ref_segment.argtypes = [vp, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        lib.t360ref_kernel.restype = C.c_int
        lib.t360ref_kernel.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float), C.c_int]
        lib.t360ref_sizeof_context.restype = C.c_int
        lib.t360ref_set_hooks.restype = None
        lib.t360ref_set_hooks.argtypes = [_REMAP_T, _SEP_T, _RESIZE_T]
        hooks = (_REMAP_T(_remap_hook), _SEP_T(_sep_hook), _RESIZE_T(_resize_hook))
        lib.t360ref_set_hooks(*hooks)
        _hooks_keepalive = hooks
        assert lib.t360ref_sizeof_context() == C.sizeof(FrameTransformContext) == 112
        _lib = lib
        return lib


class RefTransform:
    """The reference ``VideoFrameTransform`` object (handler.h:22-47), driven through its own C-ABI."""

    def __init__(self, ctx: FrameTransformContext):
        self.lib = ref_lib()
        self.ctx = ctx
        self.h = self.lib.VideoFrameTransform_new(C.byref(ctx))
        if not self.h:
            raise MemoryError("VideoFrameTransform_new returned NULL")

    def close(self):
        if self.h:
            self.lib.VideoFrameTransform_delete(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def generate_map(self, in_w, in_h, out_w, out_h, idx) -> bool:
        return bool(self.lib.VideoFrameTransform_generateMapForPlane(self.h, in_w, in_h, out_w, out_h, idx))

    def map(self, idx) -> np.ndarray:
        rows, cols, step = C.c_int(), C.c_int(), C.c_size_t()
        p = self.lib.t360ref_map(self.h, idx, C.byref(rows), C.byref(cols), C.byref(step))
        if not p:
            raise KeyError(idx)
        assert step.value == cols.value * 8
        buf = (C.c_float * (rows.value * cols.value * 2)).from_address(p)
        return np.frombuffer(buf, np.float32).reshape(rows.value, cols.value, 2).copy()

    def segments(self, idx):
        """List of (left, top, width, height, kx float32[], ky float32[]) in the reference's order."""
        out = []
        n = self.lib.t360ref_num_segments(self.h, idx)
        rect = (C.c_int * 4)()
        nk = (C.c_int * 2)()
        for i in range(n):
            assert self.lib.t360ref_segment(self.h, idx, i, rect, nk)
            kx = (C.c_float * nk[0])()
            ky = (C.c_float * nk[1])()
            assert self.lib.t360ref_kernel(self.h, idx, i, 0, kx, nk[0])
            assert self.lib.t360ref_kernel(self.h, idx, i, 1, ky, nk[1])
            out.append((rect[0], rect[1], rect[2], rect[3], np.array(kx, np.float32), np.array(ky, np.float32)))
        return out

    def transform_plane(self, src: np.ndarray, out_w, out_h, idx, image_plane=0, out_pitch=None,
                        prefill=None) -> np.ndarray:
        """Runs the reference's own transformFramePlane (cpp:1319-1351) through the cv2 hooks."""
        assert src.dtype == np.uint8 and src.ndim == 2 and src.strides[1] == 1
        in_h, in_w = src.shape
        pitch = out_pitch or out_w
        dst = np.zeros((out_h, pitch), np.uint8) if prefill is None else np.full((out_h, pitch), prefill, np.uint8)
        with _sep_lock:
            _SEP_CACHE.clear()  # keyed by plane address: only valid within one call
        ok = self.lib.VideoFrameTransform_transformFramePlane(
            self.h, src.ctypes.data, dst.ctypes.data, in_w, in_h, src.strides[0], out_w, out_h, pitch, idx, image_plane)
        with _sep_lock:
            _SEP_CACHE.clear()
        if not ok:
            raise RuntimeError("reference transformFramePlane returned 0")
        return dst[:, :out_w] if out_pitch is None else dst
