"""The position chains of the per-frame kernels (view_gather.cu: FlatPositions, SpherePositions<BARREL>, LensPositions,
LensBlendPositions, RectilinearPositions<LENS>, MapPositions<K, TRANSPARENT>): every pixel's sampling record {col0,
rowPhase}, read back from the device and compared with the host twin record for record, at the breadth of the CPU sweeps
and at the chains' branch points.  The host twins are the planner's samplers, and for rectilinear views and warp maps
HostPlan.from_warp of rectilinear_map's map or of the caller's map.

The chains (flat_view.h, oriented_view.h, libm_ports.h) are the one place where device float code must give the host's
bits, glibc's atan2f / asinf included.  A pixel comparison on noise can miss a record that moved by 1/32 px, and says
nothing about which branch went wrong.  Nothing in the library returns device records, so they are read back through
the public frame entry points from synthetic sources whose bytes encode the position:
  - bilinear (K = 2): a source constant along y whose neighbouring columns differ by 32 gives, for a window inside the
    source's columns, exactly v(col0) + fracX (OpenCV's 1/32 table is (32 - fx)(32 - fy) 32 ..., and the phase-0 entry
    {32767, 0, 0, 1} and BORDER_TRANSPARENT's partial blend round to the same).  Four such sources (32 (x mod 8) and
    32 ((x + 4) mod 8) for the low bits and phase, (x >> 3) & 255 and ((x + 4) >> 3) & 255 for the high bits) give
    col0 mod 2048 and fracX; four more, constant along x, give row0 mod 2048 and fracY;
  - nearest (K = 1): x & 255, x >> 8, y & 255, y >> 8 give the sampled (wrapped) position;
  - an all-zero source into a known pre-fill marks the pixels BORDER_TRANSPARENT leaves alone;
  - the pixels the decode cannot read (a window across a column or row edge, the feathered belt of a blend) are compared
    as bytes, on noise, with remap_u8 of the host twin's records -- at K = 2 and at the case's own K.
The decode is proven on the CPU against remap_u8 before any of it is trusted on the device.

The ledger below classifies every pixel of every case by the chain branch it takes, from exact sources: numpy float32
for the + - * / parts (no contraction), the planner's own float map for ties, saturation and clamps, the lens maps of
single-lens rigs for coverage and lens choice, a float32 replica of the rectilinear chain (which must give rectilinear_map's
bits, or a rig's coverage, on every pixel) and the warp maps' own values.  Each (chain, class, K) must be reached; each
case family must reach one that no other family does; a class that cannot occur is in UNREACHABLE with a CPU test that
proves it.  The rectilinear positions read back are also checked against test_rectilinear's float64 model.
"""
from __future__ import annotations

import ctypes
import ctypes.util
import functools
import math

import numpy as np
import pytest

import transform360_b200 as t360
from oracle import c_oracle as co
from tests.test_lens import LAYOUTS as LENS_LAYOUTS
from tests.test_lens import RIGS, _orientations, directions, make_rig, model
from tests.test_lens_blend import BLEND_RIGS, SEAMS, composite
from tests.test_oriented import _angle
from tests.test_oriented import _sweep_case as oriented_case
from tests.test_pose import _sweep_case as pose_case
from tests.test_rectilinear import CONTEXTS as RECT_CONTEXTS
from tests.test_rectilinear import _in_dims as rect_in_dims
from tests.test_rectilinear import _poses as rect_poses
from tests.test_rectilinear import model as rect_model
from tests.test_rectilinear import rays as rect_model_rays
from tests.test_tile_gather import records_to_map
from tests.test_view import _sweep_case as view_case
from tests.test_view import torch_cuda  # noqa: F401 (fixture)
from tests.test_warp_map import FAMILIES as MAP_FAMILIES
from tests.test_warp_map import _sizes as map_sizes
from transform360_b200.stream import FrameTransformer, StreamSpec

F32 = np.float32
WRAP, TRANSPARENT = t360.BORDER_WRAP, t360.BORDER_TRANSPARENT
INTERP = {1: t360.NEAREST, 2: t360.LINEAR, 4: t360.CUBIC, 8: t360.LANCZOS4}
K_OF = {v: k for k, v in INTERP.items()}
BARRELS = (t360.LAYOUT_BARREL, t360.LAYOUT_BARREL_SPLIT)
MONO, TB, LR = t360.STEREO_FORMAT_MONO, t360.STEREO_FORMAT_TB, t360.STEREO_FORMAT_LR
VIEW_FIELDS = ("fixed_yaw", "fixed_pitch", "fixed_hfov", "fixed_vfov")


# ---- the decode --------------------------------------------------------------------------------------------------------
def coordinate_sources(w, h, k):
    """The w x h planes whose samples encode the position: K = 2, four column sources then four row sources; K = 1, the
    low and high bytes of x, then of y."""
    x, y = np.arange(w), np.arange(h)
    if k == 1:
        axes = [(x & 255, 0), (x >> 8, 0), (y & 255, 1), (y >> 8, 1)]
    else:
        axes = [(f(t), a) for a, t in ((0, x), (1, y)) for f in (lambda t: 32 * (t % 8), lambda t: 32 * ((t + 4) % 8),
                                                                  lambda t: (t >> 3) & 255, lambda t: ((t + 4) >> 3) & 255)]
    out = []
    for v, axis in axes:
        v = v.astype(np.uint8)
        out.append(np.ascontiguousarray(np.broadcast_to(v[None, :], (h, w)) if axis == 0 else np.broadcast_to(v[:, None], (h, w))))
    return out


def _axis_source_values(t):
    return [32 * (t % 8), 32 * ((t + 4) % 8), (t >> 3) & 255, ((t + 4) >> 3) & 255]


@functools.lru_cache(maxsize=None)
def decode_table():
    """(sorted keys, position mod 2048 * 32 + phase) of every first tap and phase of one axis: the bytes the four bilinear
    sources give, key = b0 | b1 << 8 | b2 << 16 | b3 << 24."""
    c = np.repeat(np.arange(2048, dtype=np.int64), 32)
    f = np.tile(np.arange(32, dtype=np.int64), 2048)
    key = np.zeros_like(c)
    for s, (v0, v1) in enumerate(zip(_axis_source_values(c), _axis_source_values(c + 1))):
        key |= (((32 - f) * v0 + f * v1 + 16) >> 5) << (8 * s)
    order = np.argsort(key, kind="stable")
    return key[order], (c * 32 + f)[order]


def decode_axis(b):
    """b: the four byte planes of one axis -> position mod 2048 * 32 + phase, -1 where the bytes are no table entry."""
    keys, vals = decode_table()
    key = b[0].astype(np.int64) | (b[1].astype(np.int64) << 8) | (b[2].astype(np.int64) << 16) | (b[3].astype(np.int64) << 24)
    i = np.clip(np.searchsorted(keys, key), 0, keys.size - 1)
    return np.where(keys[i] == key, vals[i], -1)


def decode(k, planes):
    """The device's fields from the coordinate frames of one plane: K = 2, (col0 mod 2048 * 32 + fracX, row0 mod 2048 *
    32 + fracY); K = 1, (sampled column, sampled row)."""
    if k == 1:
        return planes[0].astype(np.int64) | (planes[1].astype(np.int64) << 8), planes[2].astype(np.int64) | (planes[3].astype(np.int64) << 8)
    return decode_axis(planes[:4]), decode_axis(planes[4:])


def expected_fields(k, rec, w, h):
    """The host records' fields as decode() gives them, and where decode() can read them (column, row)."""
    col0, row0, phase = rec[..., 0].astype(np.int64), rec[..., 1].astype(np.int64) >> 10, rec[..., 1].astype(np.int64) & 1023
    if k == 1:
        return (col0 % w, row0 % h), (np.ones(col0.shape, bool), np.ones(col0.shape, bool))
    return ((col0 % 2048) * 32 + (phase & 31), (row0 % 2048) * 32 + (phase >> 5)), ((col0 >= 0) & (col0 + 1 < w), (row0 >= 0) & (row0 + 1 < h))


def skipped(k, rec, w, h):
    """BORDER_TRANSPARENT: the pixels whose anchor tap lies outside the source (they keep their byte)."""
    col0, row0 = rec[..., 0].astype(np.int64), rec[..., 1].astype(np.int64) >> 10
    return (col0 < 0) | (col0 >= w) | (row0 < 0) | (row0 >= h)


# ---- the cases ---------------------------------------------------------------------------------------------------------
def _unit_scale(ov, sizes):
    """The context at unit scale with the output at the map's size: the frames render at the map's size (no INTER_AREA)."""
    scaled = lambda f, n: int(float(F32(f) * F32(n)) + 0.5)
    iw, ih, ow, oh = sizes
    ow, oh = scaled(ov.get("width_scale_factor", 1.0), ow), scaled(ov.get("height_scale_factor", 1.0), oh)
    ov = {key: v for key, v in ov.items() if key not in ("width_scale_factor", "height_scale_factor", "interpolation_alg")}
    return ov, (iw, ih, ow, oh)


def _chain_case(kind, ov, fields, sizes, own_k):
    ov, sizes = _unit_scale(ov, sizes)
    layout = ov.get("output_layout", t360.LAYOUT_CUBEMAP_32)
    return dict(kind=kind, ov=ov, fields=tuple(fields), sizes=sizes, own_k=own_k,
                border=TRANSPARENT if layout in BARRELS else WRAP)


def view_sweep():
    rng = np.random.default_rng(20261015)
    out = []
    for n in range(600):
        ov, view, sizes = view_case(rng, n)
        out.append(_chain_case("view", ov, view, sizes, K_OF[ov["interpolation_alg"]]))
    return out


def oriented_sweep():
    rng = np.random.default_rng(20261016)
    out = []
    for n in range(384):
        ov, o, sizes = oriented_case(rng, n)
        out.append(_chain_case("oriented", ov, o, sizes, K_OF[ov["interpolation_alg"]]))
    for m in range(16):  # (test_oriented's horizontal off-centre projections with a pixel at a pole's face centre)
        layout = [t360.LAYOUT_CUBEMAP_32, t360.LAYOUT_EAC_32, t360.LAYOUT_CUBEMAP_23_OFFCENTER][m % 3]
        size = (6, 9) if layout == t360.LAYOUT_CUBEMAP_23_OFFCENTER else (9, 6)
        o = (_angle(rng, m, 0), _angle(rng, m, 1), _angle(rng, m, 2))
        ov = dict(enable_low_pass_filter=0, output_layout=layout, fixed_cube_offcenter_x=0.1 * (m % 5), fixed_cube_offcenter_z=-0.5,
                  is_horizontal_offset=1, fixed_yaw=o[0], fixed_pitch=o[1], fixed_roll=o[2])
        out.append(_chain_case("oriented", ov, o, (int(rng.integers(16, 120)) * 2 + 1, 61) + size, [1, 4][m % 2]))
    return out


def pose_sweep():
    rng = np.random.default_rng(20261016)
    out = []
    for n in range(624):
        ov, pose, sizes = pose_case(rng, n)
        out.append(_chain_case("pose", ov, pose, sizes, K_OF[ov["interpolation_alg"]]))
    for m in range(24):  # (test_pose's horizontal off-centre barrels whose cap centre is a pixel centre)
        o = (_angle(rng, m, 0), _angle(rng, m, 1), _angle(rng, m, 2), 120.0, 110.0)
        ov = dict(enable_low_pass_filter=0, output_layout=t360.LAYOUT_BARREL, fixed_cube_offcenter_x=0.1 * (m % 5), fixed_cube_offcenter_z=-0.5,
                  is_horizontal_offset=1, fixed_yaw=o[0], fixed_pitch=o[1], fixed_roll=o[2])
        out.append(_chain_case("pose", ov, o, (int(rng.integers(16, 120)) * 2 + 1, 61, [5, 15, 25][m % 3], [6, 10, 14][(m // 3) % 3]),
                               [1, 4][m % 2]))
    return out


def lens_cases():
    """test_lens's rigs x the six sphere layouts x two seeded orientations, odd sizes."""
    out = []
    for r, rig in enumerate(RIGS):
        for name, layout in sorted(LENS_LAYOUTS.items()):
            for o in _orientations(sum(map(ord, rig + name))):
                out.append(dict(kind="lens", ov=dict(output_layout=layout, enable_low_pass_filter=0), fields=o, rig=rig, sizes=(259, 131, 97, 65),
                                own_k=[4, 8][r % 2], border=TRANSPARENT))
    return out


def blend_cases():
    """test_lens_blend's rigs x the six sphere layouts x its three belt widths, and one large plane."""
    out = []
    for r, rig in enumerate(BLEND_RIGS):
        for name, layout in sorted(LENS_LAYOUTS.items()):
            for s, seam in enumerate(SEAMS):
                o = _orientations(sum(map(ord, rig + name)) + s, 1)[0]
                out.append(dict(kind="blend", ov=dict(output_layout=layout, enable_low_pass_filter=0), fields=o, rig=rig, seam=seam,
                                sizes=(259, 131, 97, 65), own_k=[4, 8][(r + s) % 2], border=TRANSPARENT))
    # and a large plane: record columns above 2048
    out.append(dict(kind="blend", ov=dict(output_layout=t360.LAYOUT_BARREL, enable_low_pass_filter=0), fields=(-40.0, 15.0, 5.0), rig="tilted",
                    seam=10.0, sizes=(7680, 3840, 1920, 960), own_k=4, border=TRANSPARENT))
    return out


def large_cases():
    """7680 x 3840 sources into 1920-wide outputs: record columns above 2048 and long tile loops."""
    big = (7680, 3840, 1920, 960)
    return [_chain_case("view", dict(output_layout=t360.LAYOUT_FLAT_FIXED, enable_low_pass_filter=0), (35.0, -20.0, 110.0, 70.0), big, 4),
            _chain_case("oriented", dict(output_layout=t360.LAYOUT_EQUIRECT, enable_low_pass_filter=0), (-150.0, 30.0, 10.0), big, 8),
            _chain_case("pose", dict(output_layout=t360.LAYOUT_BARREL, enable_low_pass_filter=0), (80.0, -10.0, 5.0, 90.0, 90.0), big, 4),
            dict(kind="lens", ov=dict(output_layout=t360.LAYOUT_EQUIRECT, enable_low_pass_filter=0), fields=(20.0, 5.0, 0.0), rig="pair_190",
                 sizes=(7680, 3840, 1920, 960), own_k=8, border=TRANSPARENT)]


# ---- float32 replicas of the mono CUBEMAP_32 chain, for the classes the maps do not show -----------------
# Every step below is the chain's own IEEE float operation in the chain's order (numpy float32 does not contract), the
# rotation and lens constants are computed in double with glibc's sin / cos as the library computes them, and theta is
# glibc's atan2f (the libm ports equal it bit for bit).  The classifiers check the replica against the host twin's
# weights and coverage on every pixel they classify, so a replica that drifted fails the ledger instead of misleading it.
_LIBM = ctypes.CDLL(ctypes.util.find_library("m"))
_LIBM.atan2f.restype, _LIBM.atan2f.argtypes = ctypes.c_float, (ctypes.c_float, ctypes.c_float)
atan2f = np.vectorize(lambda y, x: F32(_LIBM.atan2f(float(y), float(x))), otypes=[F32])
_CUBE32 = [((.5, -.5, .5), (0, 0, -1), (0, 1, 0)), ((-.5, -.5, -.5), (0, 0, 1), (0, 1, 0)), ((-.5, .5, .5), (1, 0, 0), (0, 0, -1)),
           ((-.5, -.5, -.5), (1, 0, 0), (0, 0, 1)), ((-.5, -.5, .5), (1, 0, 0), (0, 1, 0)), ((.5, -.5, -.5), (-1, 0, 0), (0, 1, 0))]


def rotation_f32(yaw, pitch, roll):
    """oriented_view.h: rotationFromAngles."""
    rad = lambda a: float(F32(a)) * math.pi / 180.0
    s1, s2, s3 = (F32(math.sin(rad(a))) for a in (yaw, pitch, roll))
    c1, c2, c3 = (F32(math.cos(rad(a))) for a in (yaw, pitch, roll))
    return [[c1 * c3 + s1 * s2 * s3, c3 * s1 * s2 - c1 * s3, c2 * s1], [c2 * s3, c2 * c3, -s2],
            [c1 * s2 * s3 - c3 * s1, c1 * c3 * s2 + s1 * s3, c1 * c2]]


def cube_directions(w, h, orientation, expand, offcentre=None):
    """The rotated direction t (spherePoint) of every pixel of a mono w x h CUBEMAP_32 output with expand_coef expand, and with
    an off-centre vector (not horizontal) the ray parameter t of rayToSphere: ([h][w][3] float32, [h][w] float32 or None)."""
    x, y = _centres(w), F32(1.0) - _centres(h)
    col, row = (x * F32(3.0)).astype(np.int64), (y * F32(2.0)).astype(np.int64)
    fx = (x * F32(3.0) - col.astype(F32))[None, :].repeat(h, 0)
    fy = (y * F32(2.0) - row.astype(F32))[:, None].repeat(w, 1)
    face = np.clip(col[None, :] + ((1 - row) * 3)[:, None], 0, 5)
    e = F32(expand)
    fx, fy = (fx - F32(0.5)) * e + F32(0.5), (fy - F32(0.5)) * e + F32(0.5)
    q = np.zeros((h, w, 3), F32)
    for f, (o, du, dv) in enumerate(_CUBE32):
        sel = face == f
        for a in range(3):
            q[..., a][sel] = (F32(o[a]) + F32(du[a]) * fx[sel]) + F32(dv[a]) * fy[sel]
    ray = None
    if offcentre is not None:
        n = np.sqrt((q[..., 0] * q[..., 0] + q[..., 1] * q[..., 1]) + q[..., 2] * q[..., 2])
        q = q / n[..., None]
        o = [F32(v) for v in offcentre]
        along = ((q[..., 0] * -o[0]) + (q[..., 1] * -o[1])) + (q[..., 2] * -o[2])
        d = along * along - ((o[0] * o[0] + o[1] * o[1]) + o[2] * o[2])
        disc = (d.astype(np.float64) + 1.0).astype(F32)
        with np.errstate(invalid="ignore"):
            root = np.sqrt(np.maximum(disc, F32(0.0)))
        ray = np.where((disc <= 0) | (root < along), F32(0.0), root - along).astype(F32)
        hit = ray > 0
        for a in range(3):
            q[..., a] = np.where(hit, q[..., a] * ray - o[a], q[..., a])
    r = rotation_f32(*orientation)
    t = np.stack([(q[..., 0] * r[0][0] - q[..., 1] * r[0][1]) + q[..., 2] * r[0][2],
                  -((q[..., 0] * r[1][0] - q[..., 1] * r[1][1]) + q[..., 2] * r[1][2]),
                  (q[..., 0] * r[2][0] - q[..., 1] * r[2][1]) + q[..., 2] * r[2][2]], -1).astype(F32)
    return t, ray


def lens_matrix(L):
    """video_frame_transform.cpp: lensRigModel's matrix (R^T, y row negated) and thetaMax, in double, stored as float."""
    a, b, g = (float(v) * math.pi / 180.0 for v in (L.yaw, -L.pitch, L.roll))
    ry = [[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]]
    rx = [[1, 0, 0], [0, math.cos(b), -math.sin(b)], [0, math.sin(b), math.cos(b)]]
    rz = [[math.cos(g), -math.sin(g), 0], [math.sin(g), math.cos(g), 0], [0, 0, 1]]
    mul = lambda p, q: [[p[u][0] * q[0][v] + p[u][1] * q[1][v] + p[u][2] * q[2][v] for v in range(3)] for u in range(3)]
    r = mul(mul(ry, rx), rz)
    return [[F32(-r[v][u] if u == 1 else r[v][u]) for v in range(3)] for u in range(3)], F32(float(L.maxAngle) * math.pi / 180.0)


def lens_views(rig, t):
    """Per lens of the rig, (Z, rho, theta, covered) of every direction t (oriented_view.h: lensHit)."""
    out = []
    for i in range(rig.numLenses):
        m, tmax = lens_matrix(rig.lens[i])
        row = lambda u: (m[u][0] * t[..., 0] + m[u][1] * t[..., 1]) + m[u][2] * t[..., 2]
        X, Y, Z = row(0), row(1), row(2)
        rho = np.sqrt(X * X + Y * Y)
        theta = atan2f(rho, Z)
        out.append((Z, rho, theta, theta <= tmax))
    return out


def blend_weight(views, seam):
    """oriented_view.h: lensBlendPosition's w, and tw where both lenses cover."""
    s = F32(1.0 / (2.0 * float(F32(seam)) * math.pi / 180.0))
    (_, _, th0, c0), (_, _, th1, c1) = views
    tw = ((F32(0.5) + (th0 - th1) * s) * F32(256.0)).astype(F32)
    w = np.where(c1, 256, 0)
    both = c0 & c1
    w = np.where(both, np.where(tw <= 0, 0, np.where(tw >= 256, 256, np.rint(tw).astype(np.int64))), w)  # (rint: half to even)
    return w, np.where(both, tw, np.nan)


def exact_cube_case(c):
    """Whether the replicas cover the case: a mono CUBEMAP_32 output without a horizontal offset."""
    ov = c["ov"]
    return ov.get("output_layout") == t360.LAYOUT_CUBEMAP_32 and ov.get("input_stereo_format", MONO) == MONO and not ov.get("is_horizontal_offset")


def _expand(c):
    return case_context(c, 1).expand_coef


def _orientation(c):
    return c["fields"][:3]


def _offcentre(c):
    o = [c["ov"].get(f"fixed_cube_offcenter_{a}", 0.0) for a in "xyz"]
    return o if any(abs(v) > 1e-9 for v in o) else None


def _half_way_search():
    """A back-to-back pair into a CUBEMAP_32 output, searched over orientations and belt widths: the first case with a
    pixel whose tw (both lenses covering) is exactly n + 1/2 with n even, where rounding half to even and rounding half up
    differ."""
    rig = make_rig("pair_190", seed=len("pair_190"))
    seams = np.unique(np.linspace(2.0, 60.0, 40000).astype(F32))
    s = (1.0 / (2.0 * seams.astype(np.float64) * math.pi / 180.0)).astype(F32)
    rng = np.random.default_rng(77)
    for _ in range(200):
        o = tuple(float(F32(v)) for v in (rng.uniform(-180, 180), rng.uniform(-30, 30), rng.uniform(-30, 30)))
        t, _ = cube_directions(48, 32, o, t360.make_context().expand_coef)
        (_, _, th0, c0), (_, _, th1, c1) = lens_views(rig, t)
        both = c0 & c1
        delta = (th0 - th1)[both]
        tw = ((F32(0.5) + delta[:, None] * s[None, :]) * F32(256.0)).astype(F32)
        n = np.floor(tw)
        hit = (tw - n == 0.5) & (n.astype(np.int64) % 2 == 0) & (tw > 0) & (tw < 256)
        if hit.any():
            seam = float(seams[np.nonzero(hit)[1][0]])
            return dict(kind="blend", ov=dict(output_layout=t360.LAYOUT_CUBEMAP_32, enable_low_pass_filter=0), fields=o, rig="pair_190",
                        seam=seam, sizes=(259, 131, 48, 32), own_k=4, border=TRANSPARENT)
    raise AssertionError("no half-way blend weight found")


def _theta_max_search():
    """A back-to-back pair into a 9 x 6 CUBEMAP_32 output at orientation (0, 0, 0) (a face centre on lens 0's axis: rho = 0;
    the pole face centres: z1 == z0), with lens 0's maxAngle searched so that thetaMax equals a pixel's theta exactly."""
    c = dict(kind="lens", ov=dict(output_layout=t360.LAYOUT_CUBEMAP_32, enable_low_pass_filter=0), fields=(0.0, 0.0, 0.0), rig="pair_190",
             sizes=(259, 131, 9, 6), own_k=8, border=TRANSPARENT)
    rig = rig_of(c)
    t, _ = cube_directions(9, 6, (0.0, 0.0, 0.0), t360.make_context().expand_coef)
    theta = lens_views(rig, t)[0][2]
    for th in np.unique(theta[(theta > np.radians(80)) & (theta < np.radians(95))]):
        a0 = F32(float(th) * 180.0 / math.pi)
        for a in a0 + np.arange(-4, 5) * np.spacing(a0):
            if F32(float(a) * math.pi / 180.0) == th:
                return dict(c, max_angle=float(a))
    raise AssertionError("no maxAngle puts thetaMax on a pixel's theta")


def _disc_edge_search():
    """The smallest BARREL outputs (expand_coef 1) with a cap pixel exactly on the disc: dx^2 + dy^2 == 0.25 e e."""
    out = []
    for w in range(3, 120):
        for h in range(3, 60):
            x, y = _centres(w), F32(1.0) - _centres(h)
            cap = x > F32(0.8)
            if not cap.any():
                continue
            half = (y * F32(2.0)).astype(F32).astype(np.int64)
            dx = x[cap] * F32(5.0) - F32(4.0) - F32(0.5)
            dy = y * F32(2.0) - half.astype(F32) - F32(0.5)
            if ((dx[None, :] * dx[None, :] + dy[:, None] * dy[:, None]) == F32(0.25) * F32(1.0) * F32(1.0)).any():
                out.append((w, h))
                if len(out) == 2:
                    return out
    raise AssertionError("no barrel output puts a pixel on the cap's disc")


def boundary_cases():
    """Cases that put pixels exactly on a decision, found by searches on the host or set by hand."""
    cases = {}
    # flatLon beyond the int range: truncToInt gives INT_MIN, the record saturates (x86's cvttss2si, not the device's
    # saturating conversion).  Far beyond (lon ~ 2.8e10) and just beyond: lon = 2^31 + 256, where a saturating conversion would
    # subtract 2^31 and leave an ordinary record
    cases["lon_past_int"] = [_chain_case("view", dict(output_layout=t360.LAYOUT_FLAT_FIXED, enable_low_pass_filter=0), view, (64, 32, 17, 9), 4)
                             for view in ((1.0e13, 10.0, 90.0, 60.0), (-1.0e13, -10.0, 90.0, 60.0),
                                          (float(F32(360.0 * (2 ** 31 + 256))), 10.0, 0.5, 60.0))]
    cases["disc_edge"] = [_chain_case("pose", dict(output_layout=t360.LAYOUT_BARREL, expand_coef=1.0, enable_low_pass_filter=0), (25.0, 10.0, 0.0, 90.0, 90.0),
                                      (64, 32, w, h), 4) for w, h in _disc_edge_search()]
    cases["blend_half_way"] = [_half_way_search()]
    cases["lens_axis_tie_and_edge"] = [_theta_max_search()]
    # an off-centre vector outside the unit sphere: rays that miss it (t == 0) next to rays that meet it
    cases["offcentre_outside"] = [_chain_case("oriented", dict(output_layout=t360.LAYOUT_CUBEMAP_32, fixed_cube_offcenter_x=0.8,
                                                               fixed_cube_offcenter_y=0.3, fixed_cube_offcenter_z=-0.9, enable_low_pass_filter=0),
                                              (15.0, -5.0, 3.0), (96, 64, 27, 18), 8)]
    # cube input where no face takes the direction: a horizontal off-centre projection's NaN at a pole's face centre
    cases["cube_input_no_face"] = [_chain_case("oriented", dict(output_layout=t360.LAYOUT_CUBEMAP_32, input_layout=t360.LAYOUT_CUBEMAP_32,
                                                                fixed_cube_offcenter_z=-0.5, is_horizontal_offset=1, enable_low_pass_filter=0),
                                               (0.0, 0.0, 0.0), (96, 64, 9, 6), 4)]
    # barrels with a (non-horizontal) off-centre vector: rayToSphere's double step on every mapped pixel
    cases["barrel_offcentre"] = [_chain_case("pose", dict(output_layout=lay, fixed_cube_offcenter_x=0.3, fixed_cube_offcenter_y=-0.2,
                                                          fixed_cube_offcenter_z=0.4, expand_coef=1.1, enable_low_pass_filter=0),
                                             (30.0, 12.0, -7.0, 90.0, 90.0), (301, 151, 61, 33), 8) for lay in BARRELS]
    return cases


# ---- rectilinear views and warp maps: the cases -------------------------------------------------------------------------
RECT_CTX = dict(enable_low_pass_filter=0)


def rect_case(inp, pose, sizes, own_k, **extra):
    """A rectilinear view (RectilinearPositions) of `inp`: a context input of test_rectilinear (BORDER_WRAP), a rig of
    test_lens (BORDER_TRANSPARENT) or, with ov= in extra, the context overrides themselves."""
    ov = extra.pop("ov", None)
    if inp in RIGS:
        return dict(kind="rect", ov=dict(RECT_CTX), fields=tuple(pose), rig=inp, sizes=sizes, own_k=own_k, border=TRANSPARENT, **extra)
    return dict(kind="rect", ov=dict(RECT_CTX, **(RECT_CONTEXTS[inp] if ov is None else ov)), fields=tuple(pose), sizes=sizes, own_k=own_k,
                border=WRAP, **extra)


def rectilinear_sweep():
    """test_rectilinear's inputs (four contexts, three rigs) x its seeded and fixed poses, at its sizes."""
    out = []
    for n, inp in enumerate(sorted(RECT_CONTEXTS) + RIGS):
        (iw, ih), _ = rect_in_dims(inp)
        for pose in rect_poses(sum(map(ord, inp))):
            out.append(rect_case(inp, pose, (iw, ih, 97, 65), [4, 8][n % 2]))
    return out


def rectilinear_large():
    """The reframing use: a 7680 x 3840 equirect into a 1920 x 1080 view (90 degrees with square pixels, and 179 degrees
    across the meridian), and a 5760 x 3840 cube map: record columns above 2048, long tile loops and rays up to ~160 times
    longer than a unit vector."""
    hd = (7680, 3840, 1920, 1080)
    return [rect_case("equirect", (35.0, -20.0, 10.0, 90.0, t360.square_pixel_vfov(90.0, 1920, 1080)), hd, 4),
            rect_case("equirect", (-175.0, 50.0, -30.0, 179.0, 150.0), hd, 8),
            rect_case("cube", (120.0, -35.0, 15.0, 100.0, 70.0), (5760, 3840, 1920, 1080), 4, ov=dict(input_layout=t360.LAYOUT_CUBEMAP_32))]


def _meridian_search():
    """Rectilinear views of an odd-width equirect whose ray has t.x == +0 (and another t.x == -0) with t.z < 0: the
    branch cut of atan2f, where u is 1 (column inW - 0.5) or 0 (column -0.5).  Searched over axis-aligned and half-turn
    poses and odd output sizes."""
    found = {}
    angles = (0.0, 90.0, -90.0, 180.0, -180.0, 45.0, -45.0)
    for yaw in angles:
        for pitch in angles:
            for roll in angles:
                for w, h in ((9, 7), (15, 11), (33, 21)):
                    c = rect_case("equirect", (yaw, pitch, roll, 60.0, 40.0), (259, 131, w, h), 4)
                    t, _ = rect_rays(c, 0)
                    cut = (t[..., 0] == 0) & (t[..., 2] < 0)
                    for sign in (False, True):
                        if sign not in found and (cut & (np.signbit(t[..., 0]) == sign)).any():
                            found[sign] = c
                    if len(found) == 2:
                        return [found[False], found[True]]
    raise AssertionError(f"no pose puts a ray on the branch cut with both signs of zero (found {sorted(found)})")


@functools.lru_cache(maxsize=None)
def _pole_search():
    """A view with a ray exactly on a pole, t = (0, y, 0): yaw 0 and roll 0 make the centre column of an odd view t.x = qx =
    0 and t.z = c2 - qy s2, so a row whose qy s2 rounds to c2 is on the pole.  Searched over pitches, output heights and
    rows, with vfov stepped by floats around the angle that aims that row at the pole."""
    for pitch in (45.0, 60.0, 30.0, -45.0, 75.0):
        s2, c2 = (F32(fn(float(F32(pitch)) * math.pi / 180.0)) for fn in (math.sin, math.cos))
        for h in range(3, 40):
            y = F32(1.0) - _centres(h)
            for a in (F32(2.0) * y - F32(1.0))[:h // 2]:
                v0 = F32(2.0 * math.degrees(math.atan(float(c2) / (float(s2) * float(a)))))
                if not 0 < v0 < 179:
                    continue
                for vfov in v0 + np.arange(-256, 257) * np.spacing(v0):
                    ty = F32(math.tan(float(vfov) * math.pi / 360.0))
                    if (a * ty) * s2 == c2:
                        c = rect_case("equirect", (0.0, pitch, 0.0, 60.0, float(vfov)), (259, 131, 9, h), 8)
                        t, _ = rect_rays(c, 0)
                        if ((t[..., 0] == 0) & (t[..., 2] == 0)).any():
                            return c
    return None


def _rect_lens_search():
    """Lens cases through the unnormalised pinhole ray: an unrotated single lens with an odd output, so the centre ray is
    (0, 0, 1) (rho == 0), at 179 x 179 degrees (rays ~160 times longer than a unit vector) with maxAngle searched so that
    thetaMax equals a pixel's theta; and a back-to-back pair with a pose searched for z1 == z0."""
    c = rect_case("single_200", (0.0, 0.0, 0.0, 179.0, 179.0), (259, 131, 33, 21), 8)
    t, _ = rect_rays(c, 0)
    theta = lens_views(rig_of(c), t)[0][2]
    edge = None
    for th in np.unique(theta[(theta > np.radians(85)) & (theta < np.radians(89.5))])[::-1]:
        a0 = F32(float(th) * 180.0 / math.pi)
        hit = [a for a in a0 + np.arange(-4, 5) * np.spacing(a0) if F32(float(a) * math.pi / 180.0) == th]
        if hit:
            edge = dict(c, max_angle=float(hit[0]))
            break
    assert edge is not None, "no maxAngle puts thetaMax on a pixel's theta"
    rig = make_rig("pair_190", seed=len("pair_190"))
    pole = _pole_search()
    cands = [pole] if pole is not None else []
    cands += [rect_case("pair_190", (y, p, r, 60.0, 40.0), (259, 131, 9, h), 4)
              for y in (0.0, 90.0, -90.0, 180.0) for p in (45.0, -45.0, 90.0, 0.0) for r in (0.0, 90.0, 180.0) for h in (7, 11)]
    for c2 in cands:
        c2 = rect_case("pair_190", c2["fields"], c2["sizes"], 4)
        (z0, *_), (z1, *_) = lens_views(rig, rect_rays(c2, 0)[0])
        if (z0 == z1).any():
            return [edge, c2]
    raise AssertionError("no pose gives a ray with z1 == z0 on the back-to-back pair")


def _cube_edge_cases():
    """Cube-map input with input_expand_coef 1: a ray with |gx| == 1 (yaw 45: the centre column's t.x and t.z are the
    same float) and one with |gy| == 1 (pitch 45), the face-selection ties of cubeInputHD."""
    ov = dict(input_layout=t360.LAYOUT_CUBEMAP_32, input_expand_coef=1.0)
    return [rect_case("cube", (45.0, 0.0, 0.0, 60.0, 40.0), (261, 174, 9, 7), 4, ov=ov),
            rect_case("cube", (0.0, 45.0, 0.0, 60.0, 40.0), (261, 174, 9, 7), 8, ov=ov)]


def rectilinear_boundary():
    """Rays put exactly on the chain's decisions, found by the searches above or set by hand, and the one stereo pair the
    sweep lacks (a side-by-side input into a stacked output without the flip)."""
    out = _meridian_search() + _cube_edge_cases() + _rect_lens_search()
    pole = _pole_search()
    if pole is not None:
        out.append(pole)
    out.append(rect_case("lr_to_tb", (-60.0, 10.0, 20.0, 100.0, 80.0), (258, 131, 97, 65), 4,
                         ov=dict(input_layout=t360.LAYOUT_EQUIRECT, input_stereo_format=LR, output_stereo_format=TB)))
    return out


# The warp maps: test_warp_map's families at their sizes, and hand-placed values.  Each plane has its own map (chroma: the
# family at the chroma size, plane 2 mirrored left to right) and its own map pitch (entries of row padding per plane), so
# a plane mix-up or an ignored pitch moves records.
MAP_PITCH_EXTRA = (3, 0, 5)


def _bits(*bits):
    return np.array(bits, np.uint32).view(F32)


# value, and the class it is placed for (at K = 2 the classes of f * 32, at K = 1 those of f)
EXACT_VALUES = [
    (F32(-0.0), "neg_zero"), (F32(1e-40), "subnormal"), (F32(-1e-40), "subnormal"), (_bits(1)[0], "subnormal"),
    (F32(10 + 1 / 64), "tie_even (K 2)"), (F32(10 + 3 / 64), "tie_odd (K 2)"), (F32(12.5), "tie_even (K 1)"), (F32(13.5), "tie_odd (K 1)"),
    (_bits(0x7FC00000)[0], "nan (quiet)"), (_bits(0xFFC00000)[0], "nan (negative)"), (_bits(0x7FC12345)[0], "nan (payload)"),
    (_bits(0x7F800001)[0], "nan (signalling)"), (F32(np.inf), "pos_inf"), (F32(-np.inf), "neg_inf"),
    (F32(40000.5), "sat16_high"), (F32(-40000.5), "sat16_low"),
    (F32(67108860.0), "int_top (K 2: f * 32 = 2147483520)"), (F32(2147483520.0), "int_top (K 1)"),
    (F32(2.0 ** 26), "int_over (K 2: f * 32 = 2^31)"), (F32(2.0 ** 31), "int_over (K 1)"),
    (F32(-(2.0 ** 26)), "int_bottom (K 2: f * 32 = -2^31)"), (F32(-(2.0 ** 31)), "int_bottom (K 1)"),
    (F32(-67108872.0), "int_under (K 2: f * 32 = -2147483904)"), (F32(-2147483904.0), "int_under (K 1)"),
]


def exact_map(ow, oh, iw, ih, p):
    """Ordinary positions inside the source (no window leaves it), with every EXACT_VALUES value once as x and once as y, placed at
    plane-dependent pixels (bits kept: the NaN payloads and signs reach the kernel)."""
    rng = np.random.default_rng(100 + p)
    m = np.stack([rng.uniform(8, iw - 9, (oh, ow)), rng.uniform(8, ih - 9, (oh, ow))], -1).astype(F32)
    bits = m.view(np.uint32)
    for n, (v, _) in enumerate(EXACT_VALUES):
        for axis in range(2):
            i, j = divmod(((2 * n + axis) * 7 + 3 * p + 1) % (ow * oh), ow)
            bits[i, j, axis] = np.array([v], F32).view(np.uint32)[0]
    return m


@functools.lru_cache(maxsize=None)
def _case_map(name, sizes, p):
    iw, ih, ow, oh = StreamSpec(*sizes).plane_dims(p)[:4]
    if name == "exact":
        m = exact_map(ow, oh, iw, ih, p)
    else:
        m = MAP_FAMILIES[name](ow, oh, iw, ih)
        if p == 2:
            m = np.ascontiguousarray(m[:, ::-1])
    m.setflags(write=False)
    return m


def case_map(c, p):
    return _case_map(c["maps"], c["sizes"], p)


def map_families():
    """test_warp_map's six families at their sizes, under both borders (MapPositions<K, false> and <K, true>)."""
    out = []
    for n, name in enumerate(sorted(MAP_FAMILIES)):
        mw, mh, iw, ih = map_sizes(name)
        out += [dict(kind="map", maps=name, ov=dict(RECT_CTX), sizes=(iw, ih, mw, mh), own_k=[4, 8][(n + b) % 2], border=border)
                for b, border in enumerate((WRAP, TRANSPARENT))]
    return out


def map_exact():
    """The hand-placed values into a 2403 x 41 source (plane widths 2403 and 1202 do not divide 65535, so the saturated
    columns 32767 - a and -32768 - a wrap to different columns), under both borders."""
    return [dict(kind="map", maps="exact", ov=dict(RECT_CTX), sizes=(2403, 41, 75, 53), own_k=k, border=border)
            for k, border in ((4, WRAP), (8, TRANSPARENT))]


@functools.lru_cache(maxsize=None)
def families():
    """name -> list of cases: each sweep, the lens and blend sets, the large planes and each boundary search."""
    out = dict(view_sweep=view_sweep(), oriented_sweep=oriented_sweep(), pose_sweep=pose_sweep(), lens=lens_cases(), blend=blend_cases(),
               large=large_cases())
    out.update(boundary_cases())
    out.update(rectilinear_sweep=rectilinear_sweep(), rectilinear_large=rectilinear_large(), rectilinear_boundary=rectilinear_boundary(),
               map_families=map_families(), map_exact=map_exact())
    return out


# ---- the host twin -------------------------------------------------------------------------------------------------------
def plane_dims(c):
    spec = StreamSpec(*c["sizes"])
    return [spec.plane_dims(p)[:4] for p in range(3)]


def case_context(c, k):
    ov = dict(c["ov"], interpolation_alg=INTERP[k])
    if c["kind"] == "view":
        ov.update(zip(VIEW_FIELDS, c["fields"]))
    elif c["kind"] in ("oriented", "pose"):
        ov.update(zip(("fixed_yaw", "fixed_pitch", "fixed_roll", "fixed_hfov", "fixed_vfov"), c["fields"]))
    return t360.make_context(**ov)


def rig_of(c, lens=None):
    rig = make_rig(c["rig"], seed=len(c["rig"]))
    if "max_angle" in c:
        rig.lens[0].maxAngle = c["max_angle"]
    if lens is None:
        return rig
    one = t360.T360LensRig(1, rig.calibWidth, rig.calibHeight)
    one.lens[0] = rig.lens[lens]
    return one


def _quantised(ctx, m, iw, ih, border=TRANSPARENT):
    hp = t360.HostPlan.from_warp(ctx, m, iw, ih, border)
    r = hp.samples
    hp.close()
    return r


def host_plane(c, k, p):
    """dict(rec: the host twin's records (blend: the first record the kernel gathers), map: the float positions they
    quantise, and for lens rigs the maps of each lens alone; blend: map0, map1, weight, rec0, rec1)."""
    iw, ih, ow, oh = plane_dims(c)[p]
    ctx = case_context(c, k)
    kind = c["kind"]
    if kind in ("view", "oriented", "pose"):
        fn = dict(view=t360.view_samples, oriented=t360.oriented_samples, pose=t360.pose_samples)[kind]
        hp = t360.HostPlan(ctx, iw, ih, ow, oh)
        out = dict(rec=fn(ctx, c["fields"], iw, ih, ow, oh), map=hp.map)
        hp.close()
        return out
    warp = t360.make_context(interpolation_alg=INTERP[k], enable_low_pass_filter=0)
    if kind in ("rect", "map"):
        m = t360.rectilinear_map(ctx, c["fields"], iw, ih, ow, oh, rig_of(c) if "rig" in c else None) if kind == "rect" else case_map(c, p)
        return dict(rec=_quantised(warp, m, iw, ih, c["border"]), map=m)
    alone = [t360.lens_map(ctx, rig_of(c, i), c["fields"], iw, ih, ow, oh) for i in range(rig_of(c).numLenses)]
    if kind == "lens":
        m = t360.lens_map(ctx, rig_of(c), c["fields"], iw, ih, ow, oh)
        return dict(rec=_quantised(warp, m, iw, ih), map=m, alone=alone)
    m0, m1, wt = t360.lens_blend_maps(ctx, rig_of(c), c["seam"], c["fields"], iw, ih, ow, oh)
    r0, r1 = _quantised(warp, m0, iw, ih), _quantised(warp, m1, iw, ih)
    first = wt == 256
    return dict(rec=np.where(first[..., None], r1, r0), map=np.where(first[..., None], m1, m0), map0=m0, map1=m1, weight=wt, rec0=r0, rec1=r1,
                alone=alone)


# ---- the ledger ------------------------------------------------------------------------------------------------------------
def tie_classes(m, k):
    f = m[np.isfinite(m)].astype(F32)
    q = f * F32(32.0) if k > 1 else f
    q = q[np.abs(q) < 2.0 ** 30]
    n = np.floor(q)
    tie = q - n == 0.5
    return {f"tie_{'odd' if odd else 'even'}" for odd in np.unique(n[tie].astype(np.int64) & 1)}


def _centres(n):
    return (np.arange(n, dtype=F32) + F32(0.5)) / F32(n)


def _split(t, flip=False):
    eye = t > F32(0.5)
    s = np.where(eye, (t - F32(0.5)) / F32(0.5), t / F32(0.5)).astype(F32)
    if flip:
        s = np.where(eye, F32(1.0) - s, s).astype(F32)
    return s


def _stereo(ov):
    stereo_in = ov.get("input_stereo_format", MONO) != MONO
    out = ov.get("output_stereo_format", MONO)
    return stereo_in and out == LR, stereo_in and out == TB, ov.get("input_stereo_format", MONO)


def flat_classes(c, k, p):
    ov = c["ov"]
    f = c["fields"]
    yaw, pitch, hfov, vfov = (F32(v) for v in (f if len(f) == 4 else f[:2] + f[3:]))  # (a pose: yaw, pitch, roll, hfov, vfov)
    _, _, w, h = plane_dims(c)[p]
    split_lr, split_tb, pack = _stereo(ov)
    x, y = _centres(w), _centres(h)
    if split_lr:
        x = _split(x)
    if split_tb:
        y = _split(y, bool(ov.get("vflip")))
    with np.errstate(all="ignore"):
        lat = (((y - F32(0.5)) * vfov - pitch) / F32(180.0) + F32(0.5)).astype(F32)
        top, bottom = lat >= F32(1.0), lat < F32(0.0)
        out = {n for n, hit in (("fold_none", ~top & ~bottom), ("fold_top", top), ("fold_bottom", bottom)) if hit.any()}
        for fold in (False, True):
            if not (top | bottom).any() and fold or (top | bottom).all() and not fold:
                continue
            lon = (((x - F32(0.5)) * hfov + yaw) / F32(360.0) + F32(0.5)).astype(F32)
            if fold:
                lon = lon + F32(0.5)
            past = np.abs(lon) >= F32(2.0 ** 31)
            just = past & (np.abs(lon) < F32(2.0 ** 32))  # (a saturating conversion would leave an ordinary record)
            out |= {n for n, hit in (("lon_plain", (lon >= 0) & (lon < 1)), ("lon_wrap_down", (lon >= 1) & ~past),
                                     ("lon_wrap_up", (lon < 0) & ~past), ("lon_past_int", past & ~just), ("lon_just_past_int", just))
                    if hit.any()}
    out |= {n for n, hit in (("split_lr", split_lr), ("split_tb", split_tb and not ov.get("vflip")), ("split_tb_vflip", split_tb and ov.get("vflip")),
                             ("pack_lr", pack == LR), ("pack_tb", pack == TB)) if hit}
    return out


CUBE_FACES = {t360.LAYOUT_CUBEMAP_32: "cubemap_32", t360.LAYOUT_EAC_32: "eac_32", t360.LAYOUT_CUBEMAP_23_OFFCENTER: "cubemap_23"}


def _sphere_xy(c, p):
    ov = c["ov"]
    _, _, w, h = plane_dims(c)[p]
    split_lr, split_tb, _ = _stereo(ov)
    x, y = _centres(w), _centres(h)
    if split_lr:
        x = _split(x)
    elif split_tb:
        y = _split(y, bool(ov.get("vflip")))
    return x, (F32(1.0) - y).astype(F32)


def sphere_classes(c, k, p, hp):
    ov = c["ov"]
    layout = ov.get("output_layout", t360.LAYOUT_CUBEMAP_32)
    iw, ih, _, _ = plane_dims(c)[p]
    x, y = _sphere_xy(c, p)
    out = set()
    if layout in CUBE_FACES:
        rows, cols = (3, 2) if layout == t360.LAYOUT_CUBEMAP_23_OFFCENTER else (2, 3)
        ry, cx = (y * F32(rows)).astype(F32), (x * F32(cols)).astype(F32)
        row, col = ry.astype(np.int64), cx.astype(np.int64)
        face = np.clip(col[None, :] + ((rows - 1 - row) * cols)[:, None], 0, 5)
        out |= {f"{CUBE_FACES[layout]}_face{f}" for f in np.unique(face)}
        if (cx == np.floor(cx)).any():
            out.add("column_on_face_edge")
        if (ry == np.floor(ry)).any():
            out.add("row_on_face_edge")
    elif layout == t360.LAYOUT_EQUIRECT:
        out.add("equirect_out")
    mx = hp["map"][..., 0]
    rec = hp["rec"]
    if ov.get("input_layout") == t360.LAYOUT_CUBEMAP_32:
        none = mx == F32(-1.0) * F32(iw) - F32(0.5)
        if none.any():
            out.add("cube_in_none")
        if ov.get("input_stereo_format", MONO) == MONO:
            u, v = (mx.astype(np.float64) + 0.5) / iw, (hp["map"][..., 1].astype(np.float64) + 0.5) / ih
            ok = ~none & np.isfinite(u)
            face = np.clip(np.floor(u[ok] * 3), 0, 2).astype(int) + 3 * np.clip(np.floor(v[ok] * 2), 0, 1).astype(int)
            out |= {f"cube_in_face{f}" for f in np.unique(face)}
    else:
        out.add("equirect_in")
    off = any(abs(ov.get(f"fixed_cube_offcenter_{a}", 0.0)) > 1e-9 for a in "xyz")
    if off:
        nan = (rec[..., 0] <= -32768 - max(k // 2 - 1, 0)) & np.isnan(hp["map"][..., 0])
        out.add("offcentre_horizontal" if ov.get("is_horizontal_offset") else "offcentre")
        if nan.any():
            out.add("offcentre_nan")
        if exact_cube_case(c):
            _, ray = cube_directions(*plane_dims(c)[p][2:], _orientation(c), _expand(c), _offcentre(c))
            out |= {n for n, hit in (("offcentre_t_zero", ray == 0), ("offcentre_t_positive", ray > 0)) if hit.any()}
    return out


def barrel_classes(c, k, p, hp):
    ov = c["ov"]
    layout = ov["output_layout"]
    iw, _, _, _ = plane_dims(c)[p]
    x, y = _sphere_xy(c, p)
    out = set()
    mx = hp["map"][..., 0]
    dead = mx == F32(-1.0) * F32(iw) - F32(0.5)
    if layout == t360.LAYOUT_BARREL:
        band = x <= F32(0.8)
        half = (y * F32(2.0)).astype(F32).astype(np.int64)
        cap = ~band[None, :] & ~dead
        out |= {n for n, hit in (("band", band.any()), ("cap_top", (cap & (half == 1)[:, None]).any()),
                                 ("cap_bottom", (cap & (half != 1)[:, None]).any())) if hit}
        if (x == F32(0.8)).any():
            out.add("band_edge")
        e = F32(_expand(c))
        dx = x * F32(5.0) - F32(4.0) - F32(0.5)
        dy = y * F32(2.0) - half.astype(F32) - F32(0.5)
        if (cap & ((dx[None, :] * dx[None, :] + dy[:, None] * dy[:, None]) == F32(0.25) * e * e)).any():
            out.add("disc_edge")  # (on the disc: mapped; a >= test would make it dead zone)
    else:
        band = F32(3.0) * x <= F32(2.0)
        quarter = (y * F32(4.0)).astype(F32).astype(np.int64)
        cap = ~band[None, :] & ~dead
        out |= {f"quarter{q}" for q in range(4) if (cap & (quarter == q)[:, None]).any()}
        if band.any():
            out.add("band")
        if (F32(3.0) * x == F32(2.0)).any():
            out.add("band_edge")
    if dead.any():
        out.add("dead_zone")
    stereo_in = ov.get("input_stereo_format", MONO)
    if ov.get("input_layout") != t360.LAYOUT_CUBEMAP_32 and stereo_in != LR:
        lo = F32(1.0) / F32(iw) * F32(0.5)
        hi = F32(1.0) - lo
        out |= {n for n, v in (("clamp_low", lo), ("clamp_high", hi)) if (mx == v * F32(iw) - F32(0.5)).any()}
    return out


def lens_classes(c, k, p, hp):
    m, alone = hp["map"], hp["alone"]
    bits = m.view(np.uint32)
    covered = ~np.isnan(m[..., 0])
    out = {"uncovered"} if (~covered).any() else set()
    for i, a in enumerate(alone):
        if (covered & (bits == a.view(np.uint32)).all(-1)).any():
            out.add(f"lens{i}")
    if exact_cube_case(c):
        t, _ = cube_directions(*plane_dims(c)[p][2:], _orientation(c), _expand(c))
        views = lens_views(rig_of(c), t)
        second = views[1][0] > views[0][0] if len(views) > 1 else np.zeros(covered.shape, bool)
        chosen = [np.where(second, b, a) for a, b in zip(views[0], views[-1])]
        assert np.array_equal(chosen[3], covered), f"the lens replica's coverage differs from the host twin's ({c})"
        _, tmax0 = lens_matrix(rig_of(c).lens[0])
        _, tmax1 = lens_matrix(rig_of(c).lens[len(views) - 1])
        out |= {n for n, hit in (("tie", (views[1][0] == views[0][0]) if len(views) > 1 else second), ("rho_zero", covered & (chosen[1] == 0)),
                                 ("theta_at_max", chosen[2] == np.where(second, tmax1, tmax0))) if hit.any()}
    return out


def blend_classes(c, k, p, hp):
    cov0, cov1 = (~np.isnan(a[..., 0]) for a in hp["alone"])
    w = hp["weight"].astype(np.int32)
    both = cov0 & cov1
    out = set()
    if exact_cube_case(c):
        t, _ = cube_directions(*plane_dims(c)[p][2:], _orientation(c), _expand(c))
        views = lens_views(rig_of(c), t)
        rw, tw = blend_weight(views, c["seam"])
        assert np.array_equal(views[0][3], cov0) and np.array_equal(views[1][3], cov1), f"the replica's coverage differs ({c})"
        assert np.array_equal(rw, w), f"the replica's weights differ from the host twin's ({c})"
        with np.errstate(invalid="ignore"):
            n = np.floor(tw)
            if ((tw - n == 0.5) & (np.nan_to_num(n).astype(np.int64) % 2 == 0)).any():
                out.add("half_way_tie_even")  # (half to even keeps n; half up would give n + 1)
    return out | {n for n, hit in (("only_lens0", cov0 & ~cov1 & (w == 0)), ("only_lens1", cov1 & ~cov0 & (w == 256)),
                             ("clamped_low", both & (w == 0)), ("clamped_high", both & (w == 256)), ("ramp", (w > 0) & (w < 256)),
                             ("neither", ~cov0 & ~cov1)) if hit.any()}


_LIBM.asinf.restype, _LIBM.asinf.argtypes = ctypes.c_float, (ctypes.c_float,)
asinf = np.vectorize(lambda x: F32(_LIBM.asinf(float(x))), otypes=[F32])


def rect_rays(c, p):
    """oriented_view.h: rectilinearPoint of every pixel of plane p, in float32: (t [h][w][3], not normalised; eye [h][w])."""
    _, _, w, h = plane_dims(c)[p]
    ov = c["ov"]
    split_lr, split_tb, _ = _stereo(ov)
    x, y = _centres(w), _centres(h)
    eye_x, eye_y = np.zeros(w, bool), np.zeros(h, bool)
    if split_lr:
        eye_x, x = x > F32(0.5), _split(x)
    elif split_tb:
        eye_y, y = y > F32(0.5), _split(y, bool(ov.get("vflip")))
    y = (F32(1.0) - y).astype(F32)
    yaw, pitch, roll, hfov, vfov = (float(F32(v)) for v in c["fields"])
    tx, ty = (F32(math.tan(f * math.pi / 360.0)) for f in (hfov, vfov))  # (video_frame_transform.cpp: rectilinearCamera)
    qx = ((F32(2.0) * x - F32(1.0)) * tx)[None, :].repeat(h, 0)
    qy = ((F32(2.0) * y - F32(1.0)) * ty)[:, None].repeat(w, 1)
    r = rotation_f32(yaw, pitch, roll)
    one = F32(1.0)
    t = np.stack([(qx * r[0][0] - qy * r[0][1]) + one * r[0][2], -((qx * r[1][0] - qy * r[1][1]) + one * r[1][2]),
                  (qx * r[2][0] - qy * r[2][1]) + one * r[2][2]], -1).astype(F32)
    return t, eye_x[None, :] | eye_y[:, None]


_CUBE_IN = [(2, 0, 1, 5, 3, 1, 1), (2, 0, 1, 3, 3, 1, -1), (0, 2, 1, 3, 1, -1, 1), (0, 2, 1, 1, 1, -1, -1), (1, 0, 2, 1, 3, -1, 1),
            (1, 0, 2, 5, 1, 1, 1)]  # cubeInputHD: (major, a, b, col, row, su, sv) of faces 0..5 (even faces: major <= -0.5)


def cube_input(d, e):
    """oriented_view.h: cubeInputHD of unit rays d in float32: (face index or -1, gx, gy, u, v) of the face that takes each."""
    face = np.full(d.shape[:2], -1)
    gx, gy = np.full(d.shape[:2], np.nan, F32), np.full(d.shape[:2], np.nan, F32)
    u, v = np.full(d.shape[:2], F32(-1.0)), np.full(d.shape[:2], F32(0.0))
    with np.errstate(all="ignore"):
        for f, (mj, a, b, col, row, su, sv) in enumerate(_CUBE_IN):
            major = d[..., mj]
            ok = (major <= F32(-0.5)) if f % 2 == 0 else (major >= F32(0.5))
            fx, fy = d[..., a] / major, d[..., b] / major
            win = (face < 0) & ok & (fx >= -1) & (fx <= 1) & (fy >= -1) & (fy <= 1)
            sx, sy = fx / F32(e), fy / F32(e)
            fu = ((F32(col) + sx) if su > 0 else (F32(col) - sx)) / F32(6.0)
            fv = ((F32(row) + sy) if sv > 0 else (F32(row) - sy)) / F32(4.0)
            face, gx, gy = np.where(win, f, face), np.where(win, fx, gx), np.where(win, fy, gy)
            u, v = np.where(win, fu, u).astype(F32), np.where(win, fv, v).astype(F32)
    return face, gx, gy, u, v


_RECT_REPLICA = {}


def rect_classes(c, k, p, hp):
    """The rectilinear chain's branches from its float32 replica, which must give the host twin's map (context inputs: its
    bits; rigs: its coverage) on every pixel.  (The map does not depend on K: the replica runs once per plane.)"""
    key = (repr(sorted(c.items())), p)
    if key not in _RECT_REPLICA:
        _RECT_REPLICA[key] = frozenset(_rect_replica_classes(c, p, hp["map"]))
    out = set(_RECT_REPLICA[key])
    if "rig" not in c and np.isin(hp["rec"][..., 0] + max(k // 2 - 1, 0), (-32768, 32767)).any():
        out.add("input_saturated")
    return out


def _rect_replica_classes(c, p, m):
    ov, f = c["ov"], c["fields"]
    iw, ih, _, _ = plane_dims(c)[p]
    t, eye = rect_rays(c, p)
    split_lr, split_tb, pack = _stereo(ov)
    out = {n for n, hit in (("mono", not (split_lr or split_tb)), ("split_lr", split_lr), ("split_tb", split_tb and not ov.get("vflip")),
                            ("split_tb_vflip", split_tb and ov.get("vflip")), ("pack_lr", pack == LR), ("pack_tb", pack == TB),
                            ("fov_179", max(f[3], f[4]) >= 179.0), ("fov_narrow", min(f[3], f[4]) <= 2.0)) if hit}
    if "rig" in c:
        views = lens_views(rig_of(c), t)
        covered = ~np.isnan(m[..., 0])
        second = views[1][0] > views[0][0] if len(views) > 1 else np.zeros(covered.shape, bool)
        chosen = [np.where(second, b, a) for a, b in zip(views[0], views[-1])]
        assert np.array_equal(chosen[3], covered), f"the lens replica's coverage differs from the host twin's ({c})"
        tmax = np.where(second, lens_matrix(rig_of(c).lens[len(views) - 1])[1], lens_matrix(rig_of(c).lens[0])[1])
        return out | {n for n, hit in (("lens0", covered & ~second), ("lens1", covered & second), ("uncovered", ~covered),
                                       ("tie", (views[1][0] == views[0][0]) if len(views) > 1 else second),
                                       ("rho_zero", covered & (chosen[1] == 0)), ("theta_at_max", chosen[2] == tmax)) if hit.any()}
    tx, ty, tz = t[..., 0], t[..., 1], t[..., 2]
    n = np.sqrt((tx * tx + ty * ty) + tz * tz)
    if ov.get("input_layout") == t360.LAYOUT_CUBEMAP_32:
        face, gx, gy, u, v = cube_input(t / n[..., None], case_context(c, 2).input_expand_coef)
        out |= {f"cube_in_face{i}" for i in np.unique(face) if i >= 0} | ({"cube_in_none"} if (face < 0).any() else set())
        out |= {name for name, g in (("column_on_face_edge", gx), ("row_on_face_edge", gy)) if (np.abs(g) == 1).any()}
    else:
        lon = -atan2f(-tx / n, tz / n)
        lat = asinf(-ty / n)
        u = (lon.astype(np.float64) / (2 * math.pi) + 0.5).astype(F32)
        v = (lat.astype(np.float64) / math.pi + 0.5).astype(F32)
        if pack == LR:
            u = np.where(eye, u * F32(0.5) + F32(0.5), u * F32(0.5)).astype(F32)
        cut = (tx == 0) & (tz < 0)
        wrap = (tz[:, 1:] < 0) & (tz[:, :-1] < 0) & (np.signbit(tx[:, 1:]) != np.signbit(tx[:, :-1]))
        polar = np.hypot(tx.astype(np.float64), tz.astype(np.float64)) < 1e-3 * n
        out |= {name for name, hit in (("lon_plain", tz > 0), ("lon_wrap", wrap), ("lon_cut_pos_zero", cut & ~np.signbit(tx)),
                                       ("lon_cut_neg_zero", cut & np.signbit(tx)), ("near_pole", polar),
                                       ("exact_pole", (tx == 0) & (tz == 0))) if hit.any()}
    if pack == TB:
        v = np.where(eye, v * F32(0.5) + F32(0.5), v * F32(0.5)).astype(F32)
    want = np.stack([u * F32(iw) - F32(0.5), v * F32(ih) - F32(0.5)], -1)
    assert np.array_equal(want.view(np.uint32), m.view(np.uint32)), f"the rectilinear replica's map differs from the host twin's ({c}, plane {p})"
    return out


def map_classes(c, k, p, hp):
    """The map chain's branches from the map values themselves: f * 32 (K >= 2) or f (K = 1) against roundHalfEven's
    int range, the int16 clamp and the special floats."""
    f = hp["map"].reshape(-1)
    with np.errstate(all="ignore"):
        q = (f * F32(32.0)).astype(F32) if k > 1 else f
        fin = np.isfinite(f)
        inside = fin & (q >= F32(-(2.0 ** 31))) & (q < F32(2.0 ** 31))
        r = np.where(inside, np.rint(np.where(inside, q, 0).astype(np.float64)), 0).astype(np.int64)
        first = r >> 5 if k > 1 else r
    hit = {"interior": inside & (first >= -32768) & (first <= 32767), "neg_zero": (f == 0) & np.signbit(f),
           "subnormal": (f != 0) & (np.abs(f) < np.finfo(F32).tiny), "nan": np.isnan(f), "pos_inf": f == np.inf, "neg_inf": f == -np.inf,
           "sat16_high": inside & (first > 32767), "sat16_low": inside & (first < -32768), "int_top": q == F32(2147483520.0),
           "int_over": fin & (q >= F32(2.0 ** 31)), "int_bottom": q == F32(-(2.0 ** 31)), "int_under": fin & (q < F32(-(2.0 ** 31)))}
    out = {n for n, h in hit.items() if h.any()}
    iw, ih, _, _ = plane_dims(c)[p]
    col0, row0 = hp["rec"][..., 0].astype(np.int64), hp["rec"][..., 1].astype(np.int64) >> 10
    span = max(k, 1)
    for first, n, ok in ((col0, iw, inside.reshape(-1, 2)[:, 0]), (row0, ih, inside.reshape(-1, 2)[:, 1])):
        first = first.reshape(-1)
        if (ok & (first > -32768) & (first < 32767 - span) & ((first < 0) | (first + span > n))).any():
            out.add("edge")  # (an ordinary record whose window leaves the source: wrapped, or under BORDER_TRANSPARENT skipped or reflected)
    out.add("border_wrap" if c["border"] == WRAP else "border_transparent")
    if MAP_PITCH_EXTRA[p] > 0:
        out.add("padded_pitch")
    return out


def chain_of(c):
    if c["kind"] in ("lens", "blend"):
        return c["kind"]
    if c["kind"] in ("rect", "map"):
        return {"rect": "rectilinear", "map": "map"}[c["kind"]]
    layout = c["ov"].get("output_layout", t360.LAYOUT_CUBEMAP_32)
    return "flat" if layout == t360.LAYOUT_FLAT_FIXED else ("barrel" if layout in BARRELS else "sphere")


def all_classes(k, hp, iw):
    rec = hp["rec"]
    a = max(k // 2 - 1, 0)
    out = set(tie_classes(hp["map"], k))
    if np.isin(rec[..., 0] + a, (-32768, 32767)).any() or np.isin((rec[..., 1] >> 10) + a, (-32768, 32767)).any():
        out.add("saturated")
    if ((rec[..., 0] >= 2048) & (rec[..., 0] < iw)).any():
        out.add("column_above_2048")
    return out


def plane_classes(c, k, p, hp):
    chain = chain_of(c)
    own = {"flat": lambda: flat_classes(c, k, p), "sphere": lambda: sphere_classes(c, k, p, hp), "barrel": lambda: barrel_classes(c, k, p, hp),
           "lens": lambda: lens_classes(c, k, p, hp), "blend": lambda: blend_classes(c, k, p, hp),
           "rectilinear": lambda: rect_classes(c, k, p, hp), "map": lambda: map_classes(c, k, p, hp)}[chain]()
    if chain == "barrel":
        own |= {f"sphere:{s}" for s in sphere_classes(c, k, p, hp) if s.startswith(("cube_in", "equirect_in", "offcentre"))}
    return {(chain, cls, k) for cls in own | all_classes(k, hp, plane_dims(c)[p][0])}


@functools.lru_cache(maxsize=None)
def family_classes(name):
    out = set()
    for c in families()[name]:
        for k in (1, 2):
            for p in range(3):
                out |= plane_classes(c, k, p, host_plane(c, k, p))
    return frozenset(out)


CLASSES = {
    "flat": ("fold_none", "fold_top", "fold_bottom", "lon_plain", "lon_wrap_down", "lon_wrap_up", "lon_past_int", "lon_just_past_int", "split_lr", "split_tb",
             "split_tb_vflip", "pack_lr", "pack_tb"),
    "sphere": tuple(f"{n}_face{f}" for n in ("cubemap_32", "eac_32", "cubemap_23") for f in range(6)) + (
        "equirect_out", "equirect_in", "cube_in_none", "column_on_face_edge", "row_on_face_edge", "offcentre", "offcentre_horizontal",
        "offcentre_nan", "offcentre_t_zero", "offcentre_t_positive") + tuple(f"cube_in_face{f}" for f in range(6)),
    "barrel": ("band", "cap_top", "cap_bottom", "quarter0", "quarter1", "quarter2", "quarter3", "band_edge", "disc_edge", "dead_zone", "clamp_low",
               "clamp_high", "sphere:equirect_in", "sphere:cube_in_none", "sphere:offcentre", "sphere:offcentre_horizontal", "sphere:offcentre_nan"),
    "lens": ("lens0", "lens1", "uncovered", "tie", "rho_zero", "theta_at_max"),
    "blend": ("only_lens0", "only_lens1", "clamped_low", "clamped_high", "ramp", "neither", "half_way_tie_even"),
    "rectilinear": ("mono", "split_lr", "split_tb", "split_tb_vflip", "pack_lr", "pack_tb", "lon_plain", "lon_wrap", "lon_cut_pos_zero",
                    "lon_cut_neg_zero", "near_pole", "exact_pole") + tuple(f"cube_in_face{f}" for f in range(6)) + (
        "cube_in_none", "column_on_face_edge", "row_on_face_edge", "lens0", "lens1", "uncovered", "tie", "rho_zero", "theta_at_max", "fov_179",
        "fov_narrow", "input_saturated"),
    "map": ("interior", "edge", "neg_zero", "subnormal", "nan", "pos_inf", "neg_inf", "sat16_high", "sat16_low", "int_top", "int_over", "int_bottom",
            "int_under", "padded_pitch", "border_wrap", "border_transparent"),
}
ALL = ("tie_even", "tie_odd", "saturated", "column_above_2048")
UNREACHABLE = {
    ("barrel", "band_edge"): "no pixel centre (j + 0.5) / W, nor its eye-split image, rounds to 0.8f or to a third of 2 for any W < 8192 "
                             "(test_barrel_band_edges_are_not_reached_by_any_size)",
    ("rectilinear", "cube_in_none"): "a unit ray's largest component is at least 1/sqrt(3) > 0.5 after the float normalisation, and "
                                     "|a / major| <= 1 is exact in float division, so its face always takes it "
                                     "(test_every_unit_ray_has_a_cube_input_face)",
    ("rectilinear", "input_saturated"): "u and v of a context input lie within 2^-26 of [0, 1] (equirect) or at most (5 + 1 / e) / 4 "
                                        "from 0 (cube map, input_expand_coef e >= 0.5), so no record of a plane narrower than 8192 columns reaches the int16 clamp "
                                        "(test_context_input_records_stay_inside_the_int16_range)",
}


def required():
    out = set()
    for chain, classes in CLASSES.items():
        for cls in classes + ALL:
            if (chain, cls) not in UNREACHABLE:
                out |= {(chain, cls, k) for k in (1, 2)}
    return out


def ledger(names):
    out = set()
    for n in names:
        out |= family_classes(n)
    return out


def missing_classes(names):
    return sorted(required() - ledger(names), key=str)


# ---- CPU: the decode -----------------------------------------------------------------------------------------------------
def test_linear_table_has_the_closed_form():
    """OpenCV's bilinear table at every 1/32 phase: w = (32 - fx)(32 - fy) 32, fx (32 - fy) 32, (32 - fx) fy 32, fx fy 32,
    except phase 0, {32767, 0, 0, 1} (the saturated 32768 and its correction)."""
    t = t360.remap_table(t360.LINEAR).astype(np.int64)
    fx, fy = np.arange(1024) & 31, np.arange(1024) >> 5
    want = np.stack([np.stack([(32 - fx) * (32 - fy), fx * (32 - fy)], -1), np.stack([(32 - fx) * fy, fx * fy], -1)], 1) * 32
    want[0] = [[32767, 0], [0, 1]]
    assert np.array_equal(t, want)


def test_decode_table_is_one_to_one():
    keys, vals = decode_table()
    assert keys.size == 2048 * 32 and np.unique(keys).size == keys.size and np.unique(vals).size == vals.size


def _random_records(k, w, h, n, rng):
    """Records over the source, across its edges, far outside, saturated and NaN (a NaN map entry quantises to INT_MIN)."""
    col0 = rng.integers(-3, w + 3, n)
    row0 = rng.integers(-3, h + 3, n)
    a = max(k // 2 - 1, 0)
    pick = rng.integers(0, 10, n)
    col0 = np.where(pick == 0, rng.choice([-32768 - a, 32767 - a, -5000, 9000], n), col0)
    row0 = np.where(pick == 1, rng.choice([-32768 - a, 32767 - a, -4000, 7000], n), row0)
    phase = rng.integers(0, 1024, n) if k > 1 else np.zeros(n, np.int64)
    return np.stack([col0, (row0 << 10) | phase], -1).astype(np.int32)


@pytest.mark.parametrize("border", (WRAP, TRANSPARENT))
@pytest.mark.parametrize("k", (1, 2))
def test_decode_reads_back_random_records(k, border):
    """remap_u8 of random records (edge, saturated and NaN ones included) over the coordinate sources decodes back to
    exactly those records wherever expected_fields() claims it can, and BORDER_TRANSPARENT skips exactly skipped()."""
    rng = np.random.default_rng(10 * k + border)
    for w, h in ((37, 23), (2100, 9), (11, 2300), (7680, 3)):
        rec = _random_records(k, w, h, 6000, rng).reshape(60, 100, 2)
        m = records_to_map(rec, k)
        nan = rng.random((60, 100)) < 0.02
        m[nan] = np.nan
        rec = rec.copy()
        rec[nan] = [np.int32(-32768 - max(k // 2 - 1, 0)), np.int32(((-32768 - max(k // 2 - 1, 0)) << 10))]
        planes = [co.remap_u8(s, m, INTERP[k], border, np.full((60, 100), 255, np.uint8)) for s in coordinate_sources(w, h, k)]
        zero = co.remap_u8(np.zeros((h, w), np.uint8), m, INTERP[k], border, np.full((60, 100), 255, np.uint8))
        skip = skipped(k, rec, w, h) if border == TRANSPARENT else np.zeros((60, 100), bool)
        assert np.array_equal(zero == 255, skip), (k, border, w, h)
        got = decode(k, planes)
        want, valid = expected_fields(k, rec, w, h)
        for axis in range(2):
            sel = valid[axis] & ~skip
            assert sel.sum() > 1000
            bad = sel & (got[axis] != want[axis])
            assert not bad.any(), (k, border, w, h, axis, int(bad.sum()))


# ---- CPU: the ledger -----------------------------------------------------------------------------------------------------
def test_the_cases_reach_every_class():
    missing = missing_classes(families())
    assert not missing, f"no case reaches {missing}: those chain branches go unchecked on the device"


def test_unreachable_classes_are_not_produced():
    made = sorted((chain, cls) for chain, cls, _ in ledger(families()) if (chain, cls) in UNREACHABLE)
    assert not made, made


@pytest.mark.parametrize("name", sorted(families()))
def test_every_case_is_needed(name):
    """Each family (a sweep, the lens or blend set, the large planes, a boundary search) reaches a class no other does."""
    missing = missing_classes(set(families()) - {name})
    assert missing, f"{name} reaches no class of its own"


def test_barrel_band_edges_are_not_reached_by_any_size():
    for w in range(2, 8192):
        x = _centres(w)
        for t in (x, _split(x)):
            assert not (t == F32(0.8)).any() and not (F32(3.0) * t == F32(2.0)).any(), w


def test_every_unit_ray_has_a_cube_input_face():
    """cube_in_none is unreachable for a rectilinear ray.  The ray t = R q with q = (qx, qy, 1) is finite and at least ~1 long,
    so n > 0 and d = t / n is a unit vector up to a few float steps; its largest component is then at least 1/sqrt(3) (1 -
    4 eps) > 0.5, which passes that face's major test, and the other two components are no larger in magnitude, so |a /
    major| <= 1 (float division is monotonic and x / x == 1): the largest component's face takes d if no earlier face
    has.  Checked here on the worst case (the eight diagonals and their float neighbours, where the largest component is
    smallest) and on a million random rays of every length a view makes (up to ~160)."""
    rng = np.random.default_rng(3)
    diag = np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)], F32)
    steps = np.array([np.spacing(F32(1.0)) * s for s in range(-4, 5)], F32)
    near_diag = (diag[:, None, :] * (F32(1.0) + steps[None, :, None])).reshape(-1, 3)
    rand = (rng.normal(size=(1000000, 3)) * rng.uniform(1, 160, (1000000, 1))).astype(F32)
    for t in (near_diag, rand):
        t = t[None]
        n = np.sqrt((t[..., 0] * t[..., 0] + t[..., 1] * t[..., 1]) + t[..., 2] * t[..., 2])
        d = t / n[..., None]
        assert (np.abs(d).max(-1) > F32(0.5)).all()
        for e in (1.0, 1.04, 0.9):
            assert (cube_input(d, e)[0] >= 0).all()


def test_context_input_records_stay_inside_the_int16_range():
    """input_saturated is unreachable: atan2f returns at most float(pi) and asinf at most float(pi / 2) in magnitude, and
    the double steps make u = lon / 2pi + 0.5 and v = lat / pi + 0.5 of those extremes lie within 2^-26 of [0, 1] (float(pi)
    is a little above pi: u of -float(pi) is -1.4e-8); a cube-map input gives u = (col +- gx / e) / 6 with col in {1, 3, 5},
    v = (row +- gy / e) / 4 with row in {1, 3}, and |gx|, |gy| <= 1.  So |u inW - 0.5| stays below (5 + 1 / e) inW / 4 + 1,
    and for inW < 8192 and e >= 0.5 every record is far inside -32768 .. 32767 - 3."""
    pi_f, half_pi_f = F32(math.pi), F32(math.pi / 2)
    assert atan2f(F32(0.0), F32(-1.0)) == pi_f and atan2f(F32(-0.0), F32(-1.0)) == -pi_f and asinf(F32(1.0)) == half_pi_f
    ext = [F32(float(a) / (2 * math.pi) + 0.5) for a in (pi_f, -pi_f)] + [F32(float(a) / math.pi + 0.5) for a in (half_pi_f, -half_pi_f)]
    assert all(-(2.0 ** -26) <= a <= 1 + 2.0 ** -26 for a in ext), ext
    for e in (0.5, 1.0, 1.04):
        d = np.array([[[1.0, 1.0, -1.0], [-1.0, -1.0, 1.0], [1.0, -1.0, 1.0], [-1.0, 1.0, -1.0]]], F32) / F32(math.sqrt(3.0))
        _, _, _, u, v = cube_input(d, e)
        assert (np.abs(np.concatenate([u, v])) <= (5 + 1 / e) / 4).all()
    assert 8191 * 7 / 4 + 1 < 32767 - 3
    assert all(c["sizes"][0] < 8192 for cases in families().values() for c in cases if c["kind"] == "rect")


def test_host_twins_equal_the_planner_on_the_added_cases():
    """The large and boundary cases (not in the CPU sweeps): the host twin's records equal the planner's.  (The rectilinear
    families' float32 replica is checked against rectilinear_map on every pixel by rect_classes, through the ledger.)"""
    for name in ("rectilinear_sweep", "rectilinear_large", "rectilinear_boundary"):
        assert family_classes(name)
    for name, cases in families().items():
        if name in ("view_sweep", "oriented_sweep", "pose_sweep", "lens", "blend"):
            continue
        for c in cases:
            if c["kind"] not in ("view", "oriented", "pose"):
                continue
            for k in (1, 2):
                for p in range(3):
                    iw, ih, ow, oh = plane_dims(c)[p]
                    hp = t360.HostPlan(case_context(c, k), iw, ih, ow, oh)
                    assert np.array_equal(host_plane(c, k, p)["rec"], hp.samples), (name, k, p)
                    hp.close()


# ---- GPU -----------------------------------------------------------------------------------------------------------------
def _plane_labels(c, k, p, hp):
    """The ledger classes of a case's plane (for a failure message: the failing pixel's branch is among them)."""
    return sorted(cls for _, cls, _ in plane_classes(c, k, p, hp))


def _run_frames(torch, c, k, frames, prefill_luma):
    """Every frame (a list of three source planes) through the case's per-frame entry point with the case's fields;
    returns the output planes per frame."""
    dims = plane_dims(c)
    ctx = case_context(c, k)
    d_in = [torch.from_numpy(np.stack([f[p] for f in frames])).cuda() for p in range(3)]
    d_out = [torch.full((len(frames), dims[p][3], dims[p][2]), prefill_luma if p == 0 else 0, dtype=torch.uint8, device="cuda") for p in range(3)]
    st = torch.cuda.Stream()
    if c["kind"] in ("view", "oriented", "pose"):
        ft = FrameTransformer(ctx, StreamSpec(*c["sizes"]))
        vft = ft.vft
        make = dict(view=vft.make_view_frame_call, oriented=vft.make_oriented_frame_call, pose=vft.make_pose_frame_call)[c["kind"]]
        args = (c["fields"],)
    elif c["kind"] == "rect":  # (a never-planned transform)
        vft = t360.VideoFrameTransform(ctx)
        rig = rig_of(c) if "rig" in c else None
        make, args = (lambda i, o, d: lambda pose, stream: vft.make_rectilinear_frame_call(i, o, d)(pose, stream, rig)), (c["fields"],)
    elif c["kind"] == "map":
        vft = t360.VideoFrameTransform(ctx)
        make, args = (lambda i, o, d: vft.make_remap_frame_call(i, o, d, c["border"])), (device_maps(torch, c),)
    else:
        vft = t360.VideoFrameTransform(ctx)
        if c["kind"] == "lens":
            make, args = vft.make_lens_frame_call, (rig_of(c), c["fields"])
        else:
            make, args = vft.make_lens_blend_frame_call, (rig_of(c), c["seam"], c["fields"])
    torch.cuda.synchronize()
    for f in range(len(frames)):
        ins = [(d_in[p][f].data_ptr(), dims[p][0]) for p in range(3)]
        outs = [(d_out[p][f].data_ptr(), dims[p][2]) for p in range(3)]
        assert make(ins, outs, dims)(*args, st.cuda_stream), f"{c}: the call was refused"
    st.synchronize()
    got = [d.cpu().numpy() for d in d_out]
    vft.close()
    return [[got[p][f] for p in range(3)] for f in range(len(frames))]


def _oracle(c, k, p, hp, src, prefill):
    if c["kind"] == "blend":
        return composite(src, hp["map0"], hp["map1"], hp["weight"], INTERP[k], prefill)
    m = hp["map"] if c["kind"] == "lens" else records_to_map(hp["rec"], k)
    return co.remap_u8(src, m, INTERP[k], c["border"], prefill.copy())


def _first_bad(what, c, k, p, hp, bad, detail):
    ys, xs = np.nonzero(bad)
    i, j = int(ys[0]), int(xs[0])
    pytest.fail(f"{what}: {int(bad.sum())} px of plane {p} differ, first at x {j} y {i} -- case {c}, K {k}, ledger classes of the plane "
                f"{_plane_labels(c, k, p, hp)}, host record {hp['rec'][i, j].tolist()}: {detail(i, j)}")


def check_case(torch, c, k):
    dims = plane_dims(c)
    noise = [co.noise_plane(*dims[p][:2], plane=p, frame=k) for p in range(3)]
    coords = [coordinate_sources(*dims[p][:2], k) for p in range(3)]
    frames = [[coords[p][s] for p in range(3)] for s in range(len(coords[0]))]
    tones = []
    if c["kind"] == "blend":  # the weight itself: lens 0's half of the source 0 and lens 1's 255, then the other way round
        tones = [[np.where(np.arange(dims[p][0]) * 2 < dims[p][0], lo, 255 - lo).astype(np.uint8)[None, :].repeat(dims[p][1], 0)
                  for p in range(3)] for lo in (0, 255)]
    frames += tones + [[np.zeros(dims[p][1::-1], np.uint8) for p in range(3)], noise]
    got = _run_frames(torch, c, k, frames, 255)
    for f, tone in enumerate(tones):
        for p in range(3):
            hp = host_plane(c, k, p)
            ow, oh = dims[p][2:]
            want = _oracle(c, k, p, hp, tone[p], np.full((oh, ow), 255 if p == 0 else 128, np.uint8))
            g = got[len(frames) - 2 - len(tones) + f][p]
            if not np.array_equal(g, want):
                _first_bad("two-tone bytes (the blend weight)", c, k, p, hp, g != want, lambda i, j: f"device {int(g[i, j])}, host {int(want[i, j])}")
    got = got[:len(got) - 2 - len(tones)] + got[len(got) - 2:]
    transparent = c["border"] == TRANSPARENT
    for p in range(3):
        iw, ih, ow, oh = dims[p]
        hp = host_plane(c, k, p)
        prefill = np.full((oh, ow), 255 if p == 0 or not transparent else 128, np.uint8)
        # the skipped pixels: the zero source leaves them at the pre-fill
        want_zero = _oracle(c, k, p, hp, np.zeros((ih, iw), np.uint8), prefill)
        skip = want_zero != 0
        dev_skip = got[-2][p] != 0
        if not np.array_equal(dev_skip, skip):
            _first_bad("skipped pixels", c, k, p, hp, dev_skip != skip,
                       lambda i, j: f"device {'skips' if dev_skip[i, j] else 'writes'} it, the host twin {'skips' if skip[i, j] else 'writes'} it")
        # bytes on noise, every pixel (the only check of the pixels the decode cannot read)
        want = _oracle(c, k, p, hp, noise[p], prefill)
        if not np.array_equal(got[-1][p], want):
            g = got[-1][p]
            _first_bad("noise bytes", c, k, p, hp, g != want, lambda i, j: f"device {int(g[i, j])}, host {int(want[i, j])}")
        # the records
        dev = decode(k, [f[p] for f in got[:-2]])
        host, valid = expected_fields(k, hp["rec"], iw, ih)
        single = ~skip if c["kind"] != "blend" else ~skip & ((hp["weight"] == 0) | (hp["weight"] == 256))
        for axis, name in enumerate(("column", "row")):
            bad = valid[axis] & single & (dev[axis] != host[axis])
            if bad.any():
                unit = "sampled position" if k == 1 else "position mod 2048 * 32 + phase"
                _first_bad(f"{name} records ({unit})", c, k, p, hp, bad,
                           lambda i, j: f"device {int(dev[axis][i, j])}, host {int(host[axis][i, j])}")
        if c["kind"] == "lens" and k == 2 and p == 0 and iw <= 2048 and ih <= 2048:
            check_against_model(c, hp, dev, valid, ~skip)
        if c["kind"] == "rect" and k == 2 and p == 0:
            check_rect_against_model(c, dev, valid, ~skip)


def device_maps(torch, c):
    """The case's map of each plane on the device, with MAP_PITCH_EXTRA entries of row padding (built in numpy and copied
    whole, so every NaN keeps its bits)."""
    out = []
    for p in range(3):
        m = case_map(c, p)
        padded = np.zeros((m.shape[0], m.shape[1] + MAP_PITCH_EXTRA[p], 2), F32)
        padded[:, :m.shape[1]] = m
        out.append(torch.from_numpy(padded).cuda())
        assert out[-1].stride(0) * 4 == 8 * (m.shape[1] + MAP_PITCH_EXTRA[p])
    return out


def check_rect_against_model(c, dev, valid, written):
    """The device's rectilinear positions (column and row + phase / 32, read back, modulo 2048) against test_rectilinear's
    float64 model of the header's contract, not through the host twin: within 1/64 px of quantisation plus the model's
    0.01 px (0.02 px for rigs), away from its near-threshold and polar pixels.  Plus the float32 pinhole's own slack: 2x - 1
    and 2y' - 1 round to 2^-24 before tan(fov / 2) scales them, a direction error of up to 2^-23 max(tx, ty) rad (1.4e-5 rad
    at 179 degrees), which an equirect input turns into that over 2 pi hypot(x, z) of a row in columns (so a 179-degree view
    of a 7680-wide input moves by pixels near the poles) and over pi hypot(x, z) in rows."""
    iw, ih, ow, oh = plane_dims(c)[0]
    ctx = case_context(c, 2)
    rig = rig_of(c) if "rig" in c else None
    with np.errstate(divide="ignore", invalid="ignore"):  # (the model's cube lookup divides by every component)
        want, near, polar = rect_model(None, ctx, rig, c["fields"], iw, ih, ow, oh)
    d, eye = rect_model_rays(ctx, c["fields"], ow, oh, mono=rig is not None)
    if rig is None and ctx.input_stereo_format == LR:  # (the model leaves side-by-side inputs to the caller: re-pack u)
        want[..., 0] = ((want[..., 0] + 0.5) / iw * 0.5 + np.where(eye, 0.5, 0.0)) * iw - 0.5
    eps = 2.0 ** -23 * max(float(F32(math.tan(float(F32(f)) * math.pi / 360.0))) for f in c["fields"][3:])
    if rig is None and ctx.input_layout != t360.LAYOUT_CUBEMAP_32:
        r = np.maximum(np.hypot(d[..., 0], d[..., 2]), 1e-12)  # (d atan2 and d asin both grow as 1 / r towards the poles)
        slack = [eps * iw / (2 * math.pi * r), eps * ih / (math.pi * r)]
    else:
        slack = [eps * max(iw, ih)] * 2
    ok = ~np.isnan(want[..., 0]) & ~near & ~polar & written
    for axis in range(2):
        sel = ok & valid[axis]
        err = np.abs(dev[axis][sel] / 32.0 - np.mod(want[..., axis][sel], 2048.0))
        err = np.minimum(err, 2048.0 - err)
        over = err - (1 / 64 + (0.02 if rig is not None else 0.01) + np.broadcast_to(slack[axis], want.shape[:2])[sel])
        assert sel.sum() > 0 and over.max() <= 0, (f"rectilinear positions read back differ from the float64 model by up to "
                                                   f"{over.max():.4f} px beyond the bound (axis {axis}, case {c})")


def check_against_model(c, hp, dev, valid, written):
    """The device's lens positions (column and row + phase / 32, read back) against test_lens's float64 model, not through
    the host twin: within 1/64 px of quantisation plus the model's 0.02 px, away from its near-threshold pixels."""
    iw, ih, ow, oh = plane_dims(c)[0]
    d, dead = directions(dict(output_layout=c["ov"]["output_layout"]), c["fields"], ow, oh)
    want, _, near, _ = model(rig_of(c), d, dead, iw, ih)
    ok = ~np.isnan(want[..., 0]) & ~near & written
    for axis in range(2):
        sel = ok & valid[axis]
        err = np.abs(dev[axis][sel] / 32.0 - want[..., axis][sel])
        assert sel.sum() > 0 and err.max() <= 1 / 64 + 0.02, (f"lens positions read back differ from the float64 model by up to "
                                                              f"{err.max():.4f} px (axis {axis}, case {c})")


def check_own_k(torch, c):
    """The case at its own K (4 or 8): every byte on noise against the host twin's records."""
    k, dims = c["own_k"], plane_dims(c)
    if k < 4:
        return
    noise = [co.noise_plane(*dims[p][:2], plane=p, frame=k + 1) for p in range(3)]
    got = _run_frames(torch, c, k, [noise], 255)[0]
    for p in range(3):
        hp = host_plane(c, k, p)
        ow, oh = dims[p][2:]
        prefill = np.full((oh, ow), 255 if p == 0 or c["border"] == WRAP else 128, np.uint8)
        want = _oracle(c, k, p, hp, noise[p], prefill)
        if not np.array_equal(got[p], want):
            _first_bad(f"noise bytes at K {k}", c, k, p, hp, got[p] != want, lambda i, j: f"device {int(got[p][i, j])}, host {int(want[i, j])}")


@pytest.mark.gpu
@pytest.mark.parametrize("k", (1, 2))
@pytest.mark.parametrize("name", sorted(families()))
def test_records_on_the_device(name, k, torch_cuda):
    """Every case of the family through its per-frame entry point: the records read back equal the host twin's, the same
    pixels are skipped, and every byte on noise equals remap_u8 of the host twin's records, at K and (K = 2) at the case's
    own K."""
    for c in families()[name]:
        check_case(torch_cuda, c, k)
        if k == 2:
            check_own_k(torch_cuda, c)
