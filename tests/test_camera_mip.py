"""Anti-aliased camera views: an input pyramid and a per-pixel level from ray differentials (T360B200_cameraMipMaps /
camera_mip_maps, T360B200_transformFrameCameraMipAsync / make_camera_mip_frame_call).

What pins what:
  - the twin's entries against camera_map bit for bit: level 0 is the camera map, every other level is the header's
    scaling of it, and maxLevel 0 is the camera map with level 0 and weight 0;
  - the twin's level of detail against a float64 model of the header's footprint (rays through the pixel edges, the chart
    Jacobians written out in float64 for equirect and cube-map input, a float64 central difference of the lens projection
    for rigs): within 2/256 level of the model's value through the same bit rule, and within 0.05 level of 1/2 log2 rho^2;
  - pyramid sizes and top levels, the odd sizes and the 8-pixel floor;
  - that it anti-aliases: a zone plate on the sphere, seen through a dome and a little planet, against an ideal render;
  - the frames against the oracle's composite of the twin (cv::resize INTER_AREA pyramids, cv::remap per level, the blend),
    and against the camera call where nothing is minified.
Poses, rigs and planes are made from seeds."""
import ctypes as C
import math

import numpy as np
import pytest

import tests.test_lens as tl
import transform360_b200 as t360
from oracle import c_oracle as co
from transform360_b200.handler import as_minify
from tests.test_camera_models import EQUIDISTANT, PANNINI, PINHOLE, STEREOGRAPHIC
from tests.test_lens import make_rig
from tests.test_rectilinear import CONTEXTS, INTERPS, RECT_CTX, _ctx, _pattern, _rig
from tests.test_rectilinear import torch_cuda  # noqa: F401 (fixture)
from tests.test_warp_map import _check, _pitch, _refused, _stdout

WRAP, TRANSPARENT = t360.BORDER_WRAP, t360.BORDER_TRANSPARENT
MODELS = {"pinhole": PINHOLE, "equidistant": EQUIDISTANT, "stereographic": STEREOGRAPHIC, "pannini": PANNINI}
MIP_INPUTS = sorted(CONTEXTS) + ["single_200", "pair_190"]
F32 = lambda v: float(np.float32(v))


def _in_dims(name):
    """Odd luma sizes (so the pyramid has non-integer INTER_AREA levels) and their 4:2:0 chroma; "equirect_even" (a mono
    equirect context) has even sides down to its top level, so every level, the first one read from the caller's plane
    included, takes the exact 2 x 2 cells."""
    if name == "equirect_even":
        return (1024, 512), (512, 256)
    return ((1029, 686), (515, 343)) if name == "cubemap_32" else ((1029, 515), (515, 258))


OUT_DIMS = [(97, 65), (49, 33), (49, 33)]


def wide_pose(model, seed):
    """A seeded pose and camera of `model` wide enough that a 97 x 65 view of a 1029-wide input is minified 2-8 times."""
    rng = np.random.default_rng(seed)
    ang = (float(rng.uniform(-180, 180)), float(rng.uniform(-80, 80)), float(rng.uniform(-180, 180)))
    if model == PINHOLE:
        return (*ang, float(rng.uniform(100, 150)), float(rng.uniform(80, 120))), (PINHOLE, 0.0)
    if model == PANNINI:
        return (*ang, float(rng.uniform(120, 200)), float(rng.uniform(80, 150))), (PANNINI, float(rng.uniform(0.3, 1.0)))
    return (*ang, float(rng.uniform(150, 300)), float(rng.uniform(150, 300))), (model, 0.0)


# ---- the oracle's composite --------------------------------------------------------------------------------------------
def pyramid(src, max_level):
    """Levels 0..T of src: cv::resize with INTER_AREA to half the size, rounded up, repeated."""
    levels = [np.ascontiguousarray(src)]
    for w, h in t360.mip_level_sizes(src.shape[1], src.shape[0], max_level)[1:]:
        levels.append(co.resize_area(levels[-1], w, h))
    return levels


def composite(levels, m0, m1, lv, w, interp, prefill=None):
    """Step 5 of the header from the twin's arrays: cv::remap of each level's entries, blended as (a (256 - w) + b w +
    128) >> 8.  prefill None: BORDER_WRAP; else BORDER_TRANSPARENT into the (non-zero) pre-fill, where one skipped sample
    leaves the other alone and two leave the pre-fill."""
    border = WRAP if prefill is None else TRANSPARENT
    shape = lv.shape
    a, b = np.zeros(shape, np.int32), np.zeros(shape, np.int32)
    skip_a, skip_b = np.zeros(shape, bool), np.zeros(shape, bool)
    for level, src in enumerate(levels):
        for sel, m, val, skip in ((lv == level, m0, a, skip_a), ((lv + 1 == level) & (w > 0), m1, b, skip_b)):
            if not sel.any():
                continue
            mm = np.where(sel[..., None], m, np.float32(0)).astype(np.float32)
            if prefill is None:
                val[sel] = co.remap_u8(src, mm, interp, border)[sel]
            else:
                val[sel] = co.remap_u8(src, mm, interp, border, prefill.copy())[sel]
                skip[sel] = (co.remap_u8(np.zeros_like(src), mm, interp, border, prefill.copy()) != 0)[sel]
    wi = w.astype(np.int32)
    blend = (a * (256 - wi) + b * wi + 128) >> 8
    out = np.where(wi > 0, np.where(skip_a, b, np.where(skip_b, a, blend)), a)
    if prefill is not None:
        out = np.where(skip_a & (skip_b | (wi == 0)), prefill, out)
    return out.astype(np.uint8)


def mip_want(ctx, rig, pose, cam, minify, srcs, out_dims, prefills=None):
    """The oracle composite of every plane of a frame: planes 1 and 2 share the twin's arrays."""
    out = []
    twins = {}
    for p, src in enumerate(srcs):
        key = (src.shape, out_dims[p])
        if key not in twins:
            twins[key] = t360.camera_mip_maps(ctx, pose, cam, minify, src.shape[1], src.shape[0], *out_dims[p], rig)
        m0, m1, lv, w = twins[key]
        levels = pyramid(src, as_minify(minify).maxLevel)
        out.append(composite(levels, m0, m1, lv, w, ctx.interpolation_alg, None if prefills is None else prefills[p]))
    return out


# ---- the float64 model of the footprint --------------------------------------------------------------------------------
def _rotation(pose):
    s1, s2, s3 = np.sin(np.radians(pose[:3]))
    c1, c2, c3 = np.cos(np.radians(pose[:3]))
    return np.array([[c1 * c3 + s1 * s2 * s3, c3 * s1 * s2 - c1 * s3, c2 * s1], [c2 * s3, c2 * c3, -s2],
                     [c1 * s2 * s3 - c3 * s1, c1 * c3 * s2 + s1 * s3, c1 * c2]])


def rays64(pose, camera, X, Y):
    """Rotated, unnormalised rays (float64 [..][3]) of the model at (X, Y), with the library's float32 constants."""
    model, d = camera
    hh, hv = math.radians(pose[3]) / 2, math.radians(pose[4]) / 2
    if model == EQUIDISTANT:
        a, b = X * F32(hh), Y * F32(hv)
        rho = np.hypot(a, b)
        s = np.where(rho > 0, np.sin(rho) / np.where(rho > 0, rho, 1), 1.0)
        q = np.stack([a * s, b * s, np.cos(rho)], -1)
    elif model == STEREOGRAPHIC:
        a, b = X * F32(math.tan(hh / 2)), Y * F32(math.tan(hv / 2))
        q = np.stack([2 * a, 2 * b, 1 - a * a - b * b], -1)
    elif model == PANNINI:
        d = F32(d)
        u, v = X * F32((d + 1) * math.sin(hh) / (d + math.cos(hh))), Y * F32(math.tan(hv))
        k = u * u / (d + 1) ** 2
        c = (-k * d + np.sqrt(1 + k * (1 - d * d))) / (k + 1)
        q = np.stack([u * (d + c) / (d + 1), v * (d + c) / (d + 1), c], -1)
    else:
        q = np.stack([X * F32(math.tan(hh)), Y * F32(math.tan(hv)), np.ones_like(X)], -1)
    rows = _rotation(pose)
    return np.stack([q[..., 0] * r[0] - q[..., 1] * r[1] + q[..., 2] * r[2] for r in rows], -1) * np.array([1.0, -1.0, 1.0])


def pixel_xy(ctx, w, h, mono):
    """X, Y of every pixel's centre and dX / 2, dY / 2 (steps 1-3 and the footprint's steps)."""
    x, y = np.meshgrid((np.arange(w) + 0.5) / w, (np.arange(h) + 0.5) / h)
    stereo = ctx.input_stereo_format != t360.STEREO_FORMAT_MONO and not mono
    hx, hy = 1.0 / w, 1.0 / h
    if stereo and ctx.output_stereo_format == t360.STEREO_FORMAT_LR:
        x, hx = np.where(x > 0.5, (x - 0.5) / 0.5, x / 0.5), 2.0 / w
    elif stereo and ctx.output_stereo_format == t360.STEREO_FORMAT_TB:
        eye = y > 0.5
        y, hy = np.where(eye, (y - 0.5) / 0.5, y / 0.5), 2.0 / h
        if ctx.vflip:
            y = np.where(eye, 1 - y, y)
    return 2 * x - 1, 2 * (1 - y) - 1, hx, hy


def _lens_pixels(rig, d, in_w, in_h):
    """The lens projection of rays d in float64 (test_lens.model's, without its NaN for uncovered rays): (px, py, the
    chosen lens's z, the other lens's z)."""
    n = rig.numLenses
    cams = [d @ tl._rot(rig.lens[i].yaw, rig.lens[i].pitch, rig.lens[i].roll) for i in range(n)]
    cams = [np.stack([c[..., 0], -c[..., 1], c[..., 2]], -1) for c in cams]
    second = (cams[1][..., 2] > cams[0][..., 2]) if n > 1 else np.zeros(d.shape[:-1], bool)
    cam = np.where(second[..., None], cams[1], cams[0]) if n > 1 else cams[0]
    px, py = np.zeros(d.shape[:-1]), np.zeros(d.shape[:-1])
    for i in range(n):
        L = rig.lens[i]
        sel = second if i == 1 else ~second
        X, Y, Z = cam[..., 0], cam[..., 1], cam[..., 2]
        rho = np.hypot(X, Y)
        th = np.arctan2(rho, Z)
        t = th * th
        thd = th * (1 + t * (L.k[0] + t * (L.k[1] + t * (L.k[2] + t * L.k[3]))))
        s = np.where(rho > 0, thd / np.where(rho > 0, rho, 1), 1 / np.where(Z > 0, Z, 1))
        px = np.where(sel, (L.fx * s * X + L.cx + 0.5) / rig.calibWidth * in_w - 0.5, px)
        py = np.where(sel, (L.fy * s * Y + L.cy + 0.5) / rig.calibHeight * in_h - 0.5, py)
    zz = [c[..., 2] for c in cams] + [cams[0][..., 2]]
    return px, py, np.abs(zz[0] - zz[1]) if n > 1 else np.full(d.shape[:-1], np.inf)


def footprint64(ctx, rig, pose, camera, in_w, in_h, w, h):
    """(rho^2 [h][w], unsure [h][w]): the header's footprint in float64, and the pixels where the float32 chain may pick
    another chart (a cube face edge, a lens tie, coverage) or is ill-conditioned (an equirect pole)."""
    X, Y, hx, hy = pixel_xy(ctx, w, h, mono=rig is not None)
    t = rays64(pose, camera, X, Y)
    rx = rays64(pose, camera, X + hx, Y) - rays64(pose, camera, X - hx, Y)
    ry = rays64(pose, camera, X, Y + hy) - rays64(pose, camera, X, Y - hy)
    unsure = np.zeros((h, w), bool)
    if rig is not None:
        n = np.linalg.norm(t, axis=-1, keepdims=True)
        px, py, tie = _lens_pixels(rig, t / n, in_w, in_h)
        outs = []
        for r in (rx, ry):
            eps = 1e-6 * n / np.linalg.norm(r, axis=-1, keepdims=True)
            p1 = _lens_pixels(rig, (t + eps * r) / n, in_w, in_h)
            p0 = _lens_pixels(rig, (t - eps * r) / n, in_w, in_h)
            outs.append(((p1[0] - p0[0]) / (2 * eps[..., 0])) ** 2 + ((p1[1] - p0[1]) / (2 * eps[..., 0])) ** 2)
        unsure |= tie < 1e-4 * n[..., 0]
        return np.maximum(*outs), unsure
    x, y, z = t[..., 0], t[..., 1], t[..., 2]
    if ctx.input_layout == t360.LAYOUT_CUBEMAP_32:
        e = np.float64(np.float32(ctx.input_expand_coef))
        d = t / np.linalg.norm(t, axis=-1, keepdims=True)
        faces = [(2, 0, 1, True), (2, 0, 1, False), (0, 2, 1, True), (0, 2, 1, False), (1, 0, 2, True), (1, 0, 2, False)]
        rho2 = [np.full((h, w), np.nan), np.full((h, w), np.nan)]
        for mj, ai, bi, neg in faces:
            m = d[..., mj]
            ok = (m <= -0.5) if neg else (m >= 0.5)
            gx, gy = d[..., ai] / m, d[..., bi] / m
            unsure |= ok & ((np.abs(np.abs(gx) - 1) < 1e-4) | (np.abs(np.abs(gy) - 1) < 1e-4))
            win = ok & (np.abs(gx) <= 1) & (np.abs(gy) <= 1) & np.isnan(rho2[0])
            for k, r in enumerate((rx, ry)):
                tm, ta, tb = t[..., mj], t[..., ai], t[..., bi]
                du = in_w / (6 * e) * (r[..., ai] * tm - ta * r[..., mj]) / tm ** 2
                dv = in_h / (4 * e) * (r[..., bi] * tm - tb * r[..., mj]) / tm ** 2
                rho2[k] = np.where(win, du * du + dv * dv, rho2[k])
        return np.maximum(*rho2), unsure
    su = in_w / (2 * np.pi) / (2 if ctx.input_stereo_format == t360.STEREO_FORMAT_LR else 1)
    sv = in_h / np.pi / (2 if ctx.input_stereo_format == t360.STEREO_FORMAT_TB else 1)
    h2, r2 = x * x + z * z, x * x + y * y + z * z
    rho2 = []
    for r in (rx, ry):
        du = su * (z * r[..., 0] - x * r[..., 2]) / h2
        dv = sv * (r[..., 1] * h2 - y * (x * r[..., 0] + z * r[..., 2])) / (r2 * np.sqrt(h2))
        rho2.append(du * du + dv * dv)
    unsure |= np.sqrt(h2) < 1e-3 * np.sqrt(r2)
    return np.maximum(*rho2), unsure


def bit_rule(rho2, bias=0.0):
    """lambda256 of the header's step 3 from float64 rho^2 (rounded to float32 first)."""
    bits = np.asarray(rho2, np.float32).view(np.int32).astype(np.int64)
    return ((bits - 0x3F800000) >> 16) + int(math.floor(abs(256 * bias) + 0.5)) * (1 if bias >= 0 else -1)


def check_lod(ctx, rig, pose, cam, in_w, in_h, w, h, max_level=8, bias=0.0, what=""):
    """The twin's lambda256 (256 level + w where it is not clamped) against the model; returns the pixels compared."""
    _, _, lv, wt = t360.camera_mip_maps(ctx, pose, cam, (max_level, bias), in_w, in_h, w, h, rig)
    top = len(t360.mip_level_sizes(in_w, in_h, max_level)) - 1
    rho2, unsure = footprint64(ctx, rig, pose, cam, in_w, in_h, w, h)
    with np.errstate(all="ignore"):
        model = np.where(np.isfinite(rho2), bit_rule(np.where(np.isfinite(rho2), rho2, 1.0), bias), 256 * top)
        exact = 0.5 * np.log2(rho2) + bias
    lam = lv.astype(np.int64) * 256 + wt
    free = (lam > 0) & (lam < 256 * top) & ~unsure & np.isfinite(rho2)
    if rig is not None:
        m0 = t360.camera_map(ctx, pose, cam, in_w, in_h, w, h, rig)
        free &= ~np.isnan(m0[..., 0])
    diff = np.abs(lam - model)[free]
    assert diff.size == 0 or diff.max() <= 2, f"{what}: lambda256 off the model by {diff.max()} at {int((diff > 2).sum())} px"
    err = np.abs(lam / 256.0 - exact)[free]
    assert err.size == 0 or err.max() <= 0.05, f"{what}: level off 1/2 log2 rho^2 by {err.max():.4f}"
    # clamped pixels: the model lies on the same side (within the tolerance)
    low, high = (lam <= 0) & ~unsure, (lam >= 256 * top) & ~unsure
    assert (model[low] <= 2).all(), f"{what}: clamped to level 0 where the model has {model[low].max()}"
    assert (model[high] >= 256 * top - 2).all(), f"{what}: clamped to the top where the model has {model[high].min()}"
    return int(free.sum())


# ---- no GPU needed -----------------------------------------------------------------------------------------------------
def test_entry_points_are_exported_with_their_bindings():
    import subprocess
    from transform360_b200.handler import EXPORTED_SYMBOLS, LIB_PATH
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    L = t360.load()
    for name in ("T360B200_cameraMipMaps", "T360B200_transformFrameCameraMipAsync"):
        assert name in EXPORTED_SYMBOLS and name in defined, name
    P = C.POINTER
    assert L.T360B200_cameraMipMaps.argtypes == [P(t360.FrameTransformContext), P(t360.T360LensRig), P(t360.T360Pose), P(t360.T360Camera),
                                                 P(t360.T360Minify)] + [C.c_int] * 4 + [C.c_void_p] * 4
    assert L.T360B200_transformFrameCameraMipAsync.argtypes == [C.c_void_p, P(t360.T360LensRig), P(t360.T360Pose), P(t360.T360Camera),
                                                                P(t360.T360Minify), C.c_int] + [C.c_void_p] * 9
    assert hasattr(t360.VideoFrameTransform, "make_camera_mip_frame_call") and callable(t360.camera_mip_maps)
    assert C.sizeof(t360.T360Minify) == 8


def same_bits(got, want):
    """float32 arrays equal bit for bit (-0 against +0 included), where a NaN must meet a NaN (of any payload)."""
    g, w = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
    nan = np.isnan(g) & np.isnan(w)
    return g.shape == w.shape and np.array_equal(np.where(nan, 0, g.view(np.uint32)), np.where(nan, 0, w.view(np.uint32)))


@pytest.mark.parametrize("name", MIP_INPUTS)
@pytest.mark.parametrize("model", sorted(MODELS))
def test_level_zero_is_the_camera_map_and_levels_scale_it(model, name):
    """Every pixel at level 0 has camera_map's entry bit for bit; at every level map0 and map1 are the header's scaling of
    camera_map's entry bit for bit; maxLevel 0 is camera_map with level 0 and weight 0."""
    ctx, rig = _ctx(name), _rig(name, seed=3)
    (in_w, in_h), _ = _in_dims(name)
    w, h = 97, 65
    sizes = t360.mip_level_sizes(in_w, in_h, 8)
    sx = [np.float32(s[0] / in_w) for s in sizes]
    sy = [np.float32(s[1] / in_h) for s in sizes]
    for k in range(3):
        pose, cam = wide_pose(MODELS[model], 100 * k + len(name))
        m = t360.camera_map(ctx, pose, cam, in_w, in_h, w, h, rig)
        m0, m1, lv, wt = t360.camera_mip_maps(ctx, pose, cam, (8, 0.5 * k - 0.5), in_w, in_h, w, h, rig)
        assert lv.max() <= len(sizes) - 1 and wt.max() <= 255 and len(np.unique(lv)) > 1, (model, name, pose)
        scaled = lambda p, s: (((p + np.float32(0.5)).astype(np.float32) * s).astype(np.float32) - np.float32(0.5)).astype(np.float32)
        for level in range(len(sizes)):
            sel = lv == level
            want0 = m[sel] if level == 0 else np.stack([scaled(m[sel][:, 0], sx[level]), scaled(m[sel][:, 1], sy[level])], -1)
            assert same_bits(m0[sel], want0), (level, pose)
            sel1 = sel & (wt > 0)
            if level + 1 < len(sizes):
                want1 = np.stack([scaled(m[sel1][:, 0], sx[level + 1]), scaled(m[sel1][:, 1], sy[level + 1])], -1)
                assert same_bits(m1[sel1], want1), (level, pose)
        assert np.isnan(m1[wt == 0]).all()
        z0, z1, zl, zw = t360.camera_mip_maps(ctx, pose, cam, 0, in_w, in_h, w, h, rig)
        assert np.array_equal(z0.view(np.uint32), m.view(np.uint32)) and not zl.any() and not zw.any() and np.isnan(z1).all()


CASES = [(name, model) for name in MIP_INPUTS for model in sorted(MODELS)] + [("tilted", "equidistant")]


@pytest.mark.parametrize("name,model", CASES)
def test_level_of_detail_against_the_float64_model(name, model):
    """lambda256 within 2/256 level of the float64 footprint through the same bit rule, and within 0.05 level of
    1/2 log2 rho^2, for every model, input and output eye split; the bias moves it by round(256 bias)."""
    ctx, rig = _ctx(name), _rig(name, seed=5)
    (in_w, in_h), _ = _in_dims(name)
    n = 0
    for k in range(3):
        pose, cam = wide_pose(MODELS[model], 7 * k + len(name) + 1000)
        n += check_lod(ctx, rig, pose, cam, in_w, in_h, 97, 65, bias=(0.0, -1.0, 1.5)[k], what=f"{name} {model} {pose}")
    assert n > 1000


def test_level_of_detail_at_hand_placed_places():
    """The equirect pole (level T), the seam (no step across it), cube-face edges (no step across them) and rho = 0 of a
    lens (the written-out limit, level as its neighbours)."""
    ctx = _ctx("equirect")
    top = len(t360.mip_level_sizes(4096, 2048, 8)) - 1
    # a pinhole at the zenith of odd size: the centre ray is the pole's direction up to the rotation's rounding
    _, _, lv, wt = t360.camera_mip_maps(ctx, (0.0, 90.0, 0.0, 60.0, 60.0), PINHOLE, 8, 4096, 2048, 65, 65)
    assert lv[32, 32] == top and wt[32, 32] == 0
    check_lod(ctx, None, (0.0, 89.0, 0.0, 60.0, 60.0), (PINHOLE, 0.0), 4096, 2048, 65, 65, what="near the pole")
    # the seam in the middle of the view
    _, _, lv, wt = t360.camera_mip_maps(ctx, (180.0, 0.0, 0.0, 120.0, 90.0), EQUIDISTANT, 8, 1029, 515, 96, 64)
    lam = lv.astype(int) * 256 + wt
    assert np.abs(np.diff(lam[:, 44:52], axis=1)).max() <= 8
    check_lod(ctx, None, (180.0, 0.0, 0.0, 120.0, 90.0), (EQUIDISTANT, 0.0), 1029, 515, 96, 64, what="the seam")
    # a cube map's face edge at yaw 45 (no step across it), and a corner of three faces (where the larger of the two axes'
    # stretches changes axis, so the level may step: only the model is checked)
    cctx = _ctx("cubemap_32")
    for pose in ((45.0, 0.0, 0.0, 60.0, 60.0), (45.0, 35.26, 0.0, 60.0, 60.0)):
        _, _, lv, wt = t360.camera_mip_maps(cctx, pose, PINHOLE, 8, 1029, 686, 96, 96)
        lam = lv.astype(int) * 256 + wt
        if pose[1] == 0.0:
            assert np.abs(np.diff(lam, axis=1)).max() <= 16 and np.abs(np.diff(lam, axis=0)).max() <= 16, pose
        check_lod(cctx, None, pose, (PINHOLE, 0.0), 1029, 686, 96, 96, what=f"cube edge {pose}")
    # rho = 0: a lens on the axis, the centre pixel of an odd view looking along it
    rig = make_rig("single_200", 0)
    rig.lens[0].yaw = rig.lens[0].pitch = rig.lens[0].roll = 0.0
    lctx = _ctx("single_200")
    for cam in (PINHOLE, EQUIDISTANT):
        _, _, lv, wt = t360.camera_mip_maps(lctx, (0.0, 0.0, 0.0, 150.0, 150.0), cam, 8, 1029, 1029, 33, 33, rig)
        lam = lv.astype(int) * 256 + wt
        assert 0 < lam[16, 16] < 256 * 7 and abs(lam[16, 16] - lam[16, 15]) <= 16 and abs(lam[16, 16] - lam[15, 16]) <= 16
        check_lod(lctx, rig, (0.0, 0.0, 0.0, 150.0, 150.0), (cam, 0.0), 1029, 1029, 33, 33, what="rho = 0")


def test_pyramid_sizes_and_top_levels():
    """Each level half the one below rounded up; the top is the last level with both sides >= 8, at most maxLevel; a
    chroma plane stops before its luma plane; the twin never goes past the top."""
    assert t360.mip_level_sizes(1029, 515, 8) == [(1029, 515), (515, 258), (258, 129), (129, 65), (65, 33), (33, 17), (17, 9)]
    assert t360.mip_level_sizes(515, 258, 8)[-1] == (17, 9) and len(t360.mip_level_sizes(515, 258, 8)) == 6
    assert t360.mip_level_sizes(7680, 3840, 4)[-1] == (480, 240) and len(t360.mip_level_sizes(7680, 3840, 8)) == 9
    assert t360.mip_level_sizes(16, 16, 8) == [(16, 16), (8, 8)] and t360.mip_level_sizes(15, 100, 8) == [(15, 100), (8, 50)]
    assert t360.mip_level_sizes(14, 100, 8) == [(14, 100)] and t360.mip_level_sizes(7, 7, 8) == [(7, 7)]
    ctx = _ctx("equirect")
    for (w, h), top in (((1029, 515), 6), ((515, 258), 5), ((33, 17), 1), ((15, 15), 1), ((14, 14), 0)):
        _, _, lv, wt = t360.camera_mip_maps(ctx, (0.0, -90.0, 0.0, 300.0, 300.0), STEREOGRAPHIC, 8, w, h, 97, 97)
        assert lv.max() == top and (wt[lv == top] == 0).all(), (w, h)


# ---- it anti-aliases ---------------------------------------------------------------------------------------------------
ZONE_K = 520.0  # 260 cycles per radian behind the camera (0.8 of the 4096-wide input's Nyquist rate), 130 at 90 degrees


def zone_plate(d):
    """0..255: cos(K (1 - d.z)) on unit directions, a zone plate around the forward axis."""
    return 127.5 + 127.5 * np.cos(ZONE_K * (1.0 - d[..., 2]))


def _zone_equirect(w=4096, h=2048):
    out = np.zeros((h, w))
    for oy in (0.25, 0.75):  # 2 x 2 samples per input pixel
        for ox in (0.25, 0.75):
            lon = ((np.arange(w) + ox) / w - 0.5) * 2 * np.pi
            lat = (0.5 - (np.arange(h) + oy) / h) * np.pi
            lon, lat = np.meshgrid(lon, lat)
            d = np.stack([np.sin(lon) * np.cos(lat), np.sin(lat), np.cos(lon) * np.cos(lat)], -1)
            out += zone_plate(d) / 4
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


def _ideal(pose, cam, w, h, ss=8):
    """The view rendered from the analytic pattern, ss x ss samples per output pixel."""
    acc = np.zeros((h, w))
    for sy in range(ss):
        for sx in range(ss):
            x, y = np.meshgrid((np.arange(w) + (sx + 0.5) / ss) / w, (np.arange(h) + (sy + 0.5) / ss) / h)
            t = rays64(pose, (cam, 0.0), 2 * x - 1, 2 * (1 - y) - 1)
            t = t / np.linalg.norm(t, axis=-1, keepdims=True)
            # the rays looked up in the equirect, y up: the pattern's directions (sin lon cos lat, sin lat, cos lon cos lat)
            acc += zone_plate(np.stack([t[..., 0], -t[..., 1], t[..., 2]], -1))
    return acc / (ss * ss)


@pytest.fixture(scope="module")
def zone():
    return _zone_equirect()


# The bounds on the pyramid's RMS error against the ideal render, as a fraction of the point-sampled view's, set from the
# first run (ratios 0.30 for the dome; 0.66 for the little planet at lodBias 0 and 0.34 at -0.5).  The little planet's
# outer ring looks at the equirect's zenith, whose horizontal stretch the isotropic (max-axis) footprint also applies
# vertically: it over-blurs there, and a negative lodBias trades that back.
AA_BOUNDS = {"dome": [(0.0, 0.4)], "little_planet": [(0.0, 0.75), (-0.5, 0.4)]}


@pytest.mark.parametrize("view,pose,cam", [("dome", (0.0, 0.0, 0.0, 180.0, 180.0), EQUIDISTANT),
                                           ("little_planet", (0.0, -90.0, 0.0, 300.0, 300.0), STEREOGRAPHIC)], ids=["dome", "little_planet"])
def test_it_anti_aliases(view, pose, cam, zone):
    """A zone plate on the sphere in a 4096 x 2048 equirect, seen through a 256^2 view: the oracle composite of the twin has
    at most AA_BOUNDS of the RMS error of camera_map's point-sampled view against an ideal 8 x 8 supersampled render."""
    ctx = _ctx("equirect", t360.CUBIC)
    ideal = _ideal(pose, cam, 256, 256)
    plain = co.remap_u8(zone, t360.camera_map(ctx, pose, cam, 4096, 2048, 256, 256), t360.CUBIC, WRAP)
    e_plain = np.sqrt(np.mean((plain - ideal) ** 2))
    for bias, bound in AA_BOUNDS[view]:
        mip = mip_want(ctx, None, pose, cam, (8, bias), [zone], [(256, 256)])[0]
        e_mip = np.sqrt(np.mean((mip - ideal) ** 2))
        print(f"{view} lodBias {bias}: RMS error point-sampled {e_plain:.2f}, pyramid {e_mip:.2f}, ratio {e_mip / e_plain:.3f}")
        assert e_mip <= bound * e_plain, (bias, e_mip, e_plain)


def test_a_magnified_view_is_the_camera_map(zone):
    """A 512^2 pinhole of 30 degrees magnifies the 4096 x 2048 input everywhere: level 0 and weight 0 everywhere, so the
    composite is camera_map's remap bit for bit."""
    ctx = _ctx("equirect", t360.CUBIC)
    pose = (20.0, 10.0, 5.0, 30.0, 30.0)
    m0, _, lv, wt = t360.camera_mip_maps(ctx, pose, PINHOLE, 8, 4096, 2048, 512, 512)
    assert not lv.any() and not wt.any()
    plain = co.remap_u8(zone, t360.camera_map(ctx, pose, PINHOLE, 4096, 2048, 512, 512), t360.CUBIC, WRAP)
    assert np.array_equal(mip_want(ctx, None, pose, PINHOLE, (8, 0.0), [zone], [(512, 512)])[0], plain)


def _bad_minify():
    nan, inf = float("nan"), float("inf")
    return [("NULL minify", None)] + [(f"maxLevel {m}", (m, 0.0)) for m in (-1, 9, 1000)] + \
        [(f"lodBias {b}", (4, b)) for b in (nan, inf, -inf, 4.01, -4.01)]


def _frame_call(L, vft, rig, pose, camera, minify, n=1, planes=(0x20000,), dims=(64, 32, 8, 8), pitch=(64, 8)):
    P, I = C.c_void_p * 3, C.c_int * 3
    arr = lambda v: I(*([v] * 3))
    mb = C.byref(t360.T360Minify(*minify)) if minify is not None else None
    pb = C.byref(t360.T360Pose(*pose)) if pose is not None else None
    cb = C.byref(t360.T360Camera(*camera)) if camera is not None else None
    return L.T360B200_transformFrameCameraMipAsync(vft._h, C.byref(rig) if rig is not None else None, pb, cb, mb, n,
                                                   P(*(list(planes) * 3)[:3]), P(*(list(planes) * 3)[:3]), arr(dims[0]), arr(dims[1]),
                                                   arr(pitch[0]), arr(dims[2]), arr(dims[3]), arr(pitch[1]), None)


def test_refusals_happen_without_a_gpu(capfd):
    """Every refusal of the twin and of the frame call (the camera views' own, and minify's) comes with a message and
    before any CUDA call, with bogus plane pointers that are never dereferenced and no kernel launched; the limits
    themselves are accepted."""
    from tests.test_camera_models import _bad_calls
    L = t360.load()
    ctx = t360.make_context(**RECT_CTX)
    arrays = [np.zeros((8, 8, 2), np.float32), np.zeros((8, 8, 2), np.float32), np.zeros((8, 8), np.uint8), np.zeros((8, 8), np.uint16)]
    ptrs = [a.ctypes.data for a in arrays]
    n0 = t360.kernel_launch_count()
    ok_pose, ok_cam = (10.0, 5.0, 0.0, 90.0, 60.0), (STEREOGRAPHIC, 0.0)
    cases = [(what, None, ok_pose, ok_cam, m, {}) for what, m in _bad_minify()]
    cases += [(what, rig, pose, cam, (4, 0.0), ov) for what, rig, pose, cam, ov in _bad_calls()]
    for what, rig, pose, cam, minify, ov in cases:
        c = t360.make_context(**{**RECT_CTX, **ov})
        mb = C.byref(t360.T360Minify(*minify)) if minify is not None else None
        pb = C.byref(t360.T360Pose(*pose)) if pose is not None else None
        cb = C.byref(t360.T360Camera(*cam)) if cam is not None else None
        assert not L.T360B200_cameraMipMaps(C.byref(c), C.byref(rig) if rig is not None else None, pb, cb, mb, 64, 32, 8, 8, *ptrs), what
        out = _stdout(capfd)
        assert "Could not compute the camera mip maps" in out, what
        if minify is None or what.startswith(("maxLevel", "lodBias")):
            assert ("minify" in out) or ("maxLevel" in out) or ("lodBias" in out), out
        with t360.VideoFrameTransform(c) as vft:
            assert "anti-aliased camera view" in _refused(capfd, _frame_call, L, vft, rig, pose, cam, minify), what
    mb = C.byref(t360.T360Minify(4, 0.0))
    pb, cb = C.byref(t360.T360Pose(*ok_pose)), C.byref(t360.T360Camera(*ok_cam))
    for args in ((64, 32, 0, 8, *ptrs), (64, 0, 8, 8, *ptrs), (64, 32, 8, 8, None, *ptrs[1:]), (64, 32, 8, 8, *ptrs[:3], None)):
        _refused(capfd, L.T360B200_cameraMipMaps, C.byref(ctx), None, pb, cb, mb, *args)
    _refused(capfd, L.T360B200_cameraMipMaps, None, None, pb, cb, mb, 64, 32, 8, 8, *ptrs)
    with t360.VideoFrameTransform(ctx) as vft:
        for kw in (dict(n=0), dict(n=4), dict(planes=(None,)), dict(dims=(0, 32, 8, 8)), dict(pitch=(63, 8))):
            _refused(capfd, lambda: _frame_call(L, vft, None, ok_pose, ok_cam, (4, 0.0), **kw))
    assert not L.T360B200_transformFrameCameraMipAsync(None, None, None, None, None, 1, *([None] * 9))
    assert t360.kernel_launch_count() == n0
    with pytest.raises(ValueError):
        t360.camera_mip_maps(ctx, ok_pose, ok_cam, (9, 0.0), 64, 32, 8, 8)
    for minify in ((0, -4.0), (8, 4.0), (8, -4.0)):
        t360.camera_mip_maps(ctx, ok_pose, ok_cam, minify, 64, 32, 8, 8)


# ---- on the GPU --------------------------------------------------------------------------------------------------------
def _dev(torch, a, pitch=None):
    pitch = pitch or _pitch(a.shape[1])
    t = torch.zeros((a.shape[0], pitch), dtype=torch.uint8, device="cuda")
    t[:, :a.shape[1]] = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t


class MipFrame:
    """Noise source planes of input `name` (odd sizes), pre-filled outputs and the argument lists of one frame."""

    def __init__(self, torch, name, n=3, seed=0, unaligned=False, in_dims=None, out_dims=None):
        self.torch, self.n = torch, n
        luma, chroma = in_dims or _in_dims(name)
        self.in_dims = [luma, chroma, chroma][:n]
        self.out_dims = (out_dims or OUT_DIMS)[:n]
        self.src = [co.noise_plane(*self.in_dims[p], plane=p, frame=seed) for p in range(n)]
        self.d_src = [_dev(torch, s) for s in self.src]
        self.in_planes = [(t.data_ptr(), t.stride(0)) for t in self.d_src]
        if unaligned:  # plane 0's rows start 1 byte into the buffer, with an odd pitch
            (h, w), pitch = self.src[0].shape, _pitch(self.src[0].shape[1]) + 1
            flat = np.zeros((h + 1) * pitch, np.uint8)
            for r in range(h):
                flat[1 + r * pitch:1 + r * pitch + w] = self.src[0][r]
            self.d_src[0] = torch.from_numpy(flat).cuda()
            self.in_planes[0] = (self.d_src[0].data_ptr() + 1, pitch)
        self.prefill = [_pattern(*self.out_dims[p], p) if p == 0 else np.full(self.out_dims[p][::-1], 128, np.uint8) for p in range(n)]
        self.outs = [torch.zeros((d[1], _pitch(d[0])), dtype=torch.uint8, device="cuda") for d in self.out_dims]
        for p, o in enumerate(self.outs):
            o[:, :self.out_dims[p][0]] = torch.from_numpy(_pattern(*self.out_dims[p], p)).cuda()
        self.dims = [(*self.in_dims[p], *self.out_dims[p]) for p in range(n)]

    @property
    def out_planes(self):
        return [(o.data_ptr(), o.stride(0)) for o in self.outs]

    def host(self):
        return [o[:, :self.out_dims[p][0]].cpu().numpy() for p, o in enumerate(self.outs)]

    def want(self, ctx, rig, pose, cam, minify):
        return mip_want(ctx, rig, pose, cam, minify, self.src, self.out_dims, self.prefill if rig is not None else None)


MINIFIES = [(1, 0.0), (4, -1.0), (8, 1.5)]


@pytest.mark.gpu
@pytest.mark.parametrize("name", MIP_INPUTS + ["equirect_even"])
@pytest.mark.parametrize("interp", INTERPS)
@pytest.mark.parametrize("model", sorted(MODELS))
def test_frames_equal_the_oracle_composite(model, interp, name, torch_cuda):
    """3- and 1-plane frames of noise (one with an unaligned luma plane) equal the oracle's composite of the twin bit for
    bit at maxLevel 1, 4 and 8 and lodBias -1, 0 and 1.5."""
    torch = torch_cuda
    ctx, rig = _ctx(name, interp), _rig(name, seed=interp)
    vft = t360.VideoFrameTransform(ctx)
    st = torch.cuda.Stream()
    for k, minify in enumerate(MINIFIES):
        pose, cam = wide_pose(MODELS[model], 31 * interp + 7 * k + len(name))
        for n, unaligned in ((3, False), (1, False), (3, True)):
            f = MipFrame(torch, name, n, seed=interp + k, unaligned=unaligned)
            want = f.want(ctx, rig, pose, cam, minify)
            torch.cuda.synchronize()
            assert vft.make_camera_mip_frame_call(f.in_planes, f.out_planes, f.dims)(pose, cam, minify, st.cuda_stream, rig)
            st.synchronize()
            for p, got in enumerate(f.host()):
                _check(got, want[p], f"{model} {minify} {pose}, {n} planes{' (unaligned)' if unaligned else ''}, plane {p}")
    vft.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["equirect", "cubemap_32", "pair_190"])
def test_equal_to_the_camera_call_where_nothing_is_minified(name, torch_cuda):
    """maxLevel 0, and a view magnified everywhere at maxLevel 8, give the camera call's bytes; the first takes one launch,
    the second T_max + 1."""
    torch = torch_cuda
    rig = _rig(name, seed=1)
    st = torch.cuda.Stream()
    for interp in INTERPS:
        vft = t360.VideoFrameTransform(_ctx(name, interp))
        for pose, cam, minify, top in (((10.0, 20.0, 30.0, 200.0, 150.0), EQUIDISTANT, (0, 1.5), 0),
                                       ((10.0, 20.0, 30.0, 4.0, 3.0), PINHOLE, (8, 0.0), 6)):
            a, b = MipFrame(torch, name, 3, seed=interp), MipFrame(torch, name, 3, seed=interp)
            torch.cuda.synchronize()
            n0 = t360.kernel_launch_count()
            assert vft.make_camera_mip_frame_call(a.in_planes, a.out_planes, a.dims)(pose, cam, minify, st.cuda_stream, rig)
            n1 = t360.kernel_launch_count()
            assert vft.make_camera_frame_call(b.in_planes, b.out_planes, b.dims)(pose, cam, st.cuda_stream, rig)
            assert (n1 - n0, t360.kernel_launch_count() - n1) == (top + 1, 1), (name, pose)
            st.synchronize()
            for p, (x, y) in enumerate(zip(a.host(), b.host())):
                assert np.array_equal(x, y), (name, interp, pose, p)
        vft.close()


@pytest.mark.gpu
def test_trajectory_on_two_streams(torch_cuda):
    """Two streams enqueue a trajectory without synchronising, model, pose, maxLevel and lodBias changing every frame:
    every frame equals the oracle, every frame takes T_max + 1 launches, and device memory stays bounded."""
    torch = torch_cuda
    ctx = _ctx("tb_to_lr", t360.CUBIC)
    vft = t360.VideoFrameTransform(ctx)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    args = []
    for k in range(24):
        pose, cam = wide_pose(MODELS[sorted(MODELS)[k % 4]], 500 + k)
        args.append((pose, cam, (1 + k % 8, (-1.0, 0.0, 0.75)[k % 3])))
    want_launches = sum(len(t360.mip_level_sizes(*_in_dims("tb_to_lr")[0], m[0])) for _, _, m in args)
    mem = []
    for lap in range(3):
        frames = [MipFrame(torch, "tb_to_lr", 3, seed=k + lap) for k in range(len(args))]
        torch.cuda.synchronize()
        n0 = t360.kernel_launch_count()
        for k, (f, (pose, cam, minify)) in enumerate(zip(frames, args)):
            assert vft.make_camera_mip_frame_call(f.in_planes, f.out_planes, f.dims)(pose, cam, minify, streams[k % 2].cuda_stream)
        torch.cuda.synchronize()
        assert t360.kernel_launch_count() - n0 == want_launches
        mem.append(torch.cuda.mem_get_info()[0])
        for k, (f, (pose, cam, minify)) in enumerate(zip(frames, args)):
            want = f.want(ctx, None, pose, cam, minify)
            for p, got in enumerate(f.host()):
                _check(got, want[p], f"lap {lap} frame {k} plane {p}")
        del frames
    assert abs(mem[2] - mem[1]) < (8 << 20), mem
    vft.close()


@pytest.mark.gpu
def test_refused_calls_launch_nothing_and_leave_the_outputs(torch_cuda, capfd):
    """A refused frame launches no kernel and leaves every output byte as it was."""
    torch = torch_cuda
    ctx = _ctx("equirect")
    vft = t360.VideoFrameTransform(ctx)
    f = MipFrame(torch, "equirect", 3)
    before = f.host()
    call = vft.make_camera_mip_frame_call(f.in_planes, f.out_planes, f.dims)
    n0 = t360.kernel_launch_count()
    for minify in ((9, 0.0), (4, float("nan")), (4, 5.0)):
        assert not call((0.0, 0.0, 0.0, 90.0, 60.0), PINHOLE, minify, 0)
    assert not call((0.0, 0.0, 0.0, 200.0, 60.0), PINHOLE, (4, 0.0), 0)
    torch.cuda.synchronize()
    assert t360.kernel_launch_count() == n0
    assert all(np.array_equal(a, b) for a, b in zip(before, f.host()))
    assert "anti-aliased camera view" in _stdout(capfd)
    vft.close()
