"""Stereo fisheye rigs and the equirect camera model: VR180 views with one lens per eye (T360B200_stereoCameraMaps /
stereo_camera_maps, T360B200_transformFrameStereoCameraAsync / make_stereo_camera_frame_call), and T360_CAMERA_EQUIRECT
through every camera call.

What pins what:
  - the equirect model's camera_map against a float64 model of its header row, for the context inputs and the rigs, and
    its 360 x 180 view at zero pose against the identity grid of an equirect input; camera_mip_maps against camera_map bit
    for bit and its level of detail against test_camera_mip's float64 footprint;
  - the stereo twin with MONO output against camera_photo_maps of the one-lens rig {lens 0} bit for bit; with LR and TB
    output each eye's entries against a float64 projection through that eye's lens, eyeWeight = 256 eye, and the two
    halves of an LR view of a rig of two equal lenses equal bit for bit;
  - the stereo quality: a synthetic stereo rig of a scene at infinity, lens 1 rotated by 2 degrees, vignetted and 1.3x
    brighter, has a mean luma difference between the eyes at most a quarter of the naive one's;
  - the frames and statistics against test_camera_photo's oracle composite of the stereo twin, the MONO frame against the
    camera-photo call, and the eye-combined twin map planned through generateMapFromWarp against the frame.
  - the device build of the equirect ray and of the stereo chain against the host build: tests/stereo_camera_twin_gate.cu,
    run from tests/test_twin_gates.py.
Poses, rigs and planes are made from seeds."""
import ctypes as C
import math
import subprocess

import numpy as np
import pytest

import tests.test_camera_mip as tcm
import tests.test_camera_photo as tcp
import tests.test_lens as tl
import transform360_b200 as t360
from tests.test_camera_mip import MipFrame, _in_dims, check_lod, same_bits
from tests.test_camera_models import EQUIDISTANT, PANNINI, PINHOLE, STEREOGRAPHIC, _bad_calls
from tests.test_camera_photo import lens_pixels64
from tests.test_lens import make_rig
from tests.test_lens_photo import IDENTITY, STATS, _bad_photo_calls, _render_rig, photometry, r_max, rig_photos
from tests.test_rectilinear import INPUTS, INTERPS, RECT_CTX, _ctx, _rig
from tests.test_rectilinear import torch_cuda  # noqa: F401 (fixture)
from tests.test_warp_map import _check, _refused, _stdout

EQUIRECT = t360.T360_CAMERA_EQUIRECT
MODELS = {"pinhole": PINHOLE, "equidistant": EQUIDISTANT, "stereographic": STEREOGRAPHIC, "pannini": PANNINI, "equirect": EQUIRECT}
LR, TB, MONO = t360.STEREO_FORMAT_LR, t360.STEREO_FORMAT_TB, t360.STEREO_FORMAT_MONO
FORMATS = {"mono": dict(output_stereo_format=MONO), "lr": dict(output_stereo_format=LR), "tb": dict(output_stereo_format=TB),
           "tb_vflip": dict(output_stereo_format=TB, vflip=1)}
MINIFIES = [None, (3, 0.0), (4, 1.0)]
W, H = 97, 65
F32 = lambda v: float(np.float32(v))
WRAP, TRANSPARENT = t360.BORDER_WRAP, t360.BORDER_TRANSPARENT


def stereo_rig(name="stereo_190", seed=0):
    """Two forward 190-degree lenses side by side on a 2000 x 1000 frame, lens 1 with a small rectification rotation;
    "swapped": the left eye's circle (lens 0) on the right half; "equal": both lenses the same."""
    rng = np.random.default_rng(seed)
    j = lambda s: float(rng.uniform(-s, s))
    rig = t360.T360LensRig(2, 2000, 1000)
    left, right = (1499.5, 499.5) if name == "swapped" else (499.5, 1499.5)
    rig.lens[0] = tl._lens(rng, 500, left + j(2), 499.5 + j(2), j(1), j(1), j(1), 95)
    rig.lens[1] = tl._lens(rng, 500, right + j(2), 499.5 + j(2), j(2), j(2), j(2), 95)
    if name == "equal":
        rig.lens[1] = rig.lens[0]
    return rig


def eq_pose(seed, model=EQUIRECT):
    """A seeded forward-looking pose of `model` for a stereo rig: the VR180 window, a cropped one, or a wide one."""
    rng = np.random.default_rng(seed)
    ang = (float(rng.uniform(-20, 20)), float(rng.uniform(-20, 20)), float(rng.uniform(-10, 10)))
    if model == EQUIRECT:
        return (*ang, *((180.0, 180.0), (float(rng.uniform(60, 200)), float(rng.uniform(40, 180))))[seed % 2]), (EQUIRECT, 0.0)
    pose, cam = tcm.wide_pose(model, seed)
    return (*ang, *pose[3:]), cam


# ---- the float64 model of the equirect row ---------------------------------------------------------------------------
def rays_any(pose, camera, X, Y):
    """test_camera_mip.rays64 with the equirect row: rotated, unnormalised rays of the model at (X, Y)."""
    if camera[0] != EQUIRECT:
        return tcm.rays64(pose, camera, X, Y)
    lon, lat = X * F32(math.radians(pose[3]) / 2), Y * F32(math.radians(pose[4]) / 2)
    q = np.stack([np.cos(lat) * np.sin(lon), np.sin(lat), np.cos(lat) * np.cos(lon)], -1)
    rows = tcm._rotation(pose)
    return np.stack([q[..., 0] * r[0] - q[..., 1] * r[1] + q[..., 2] * r[2] for r in rows], -1) * np.array([1.0, -1.0, 1.0])


def eye_xy(ctx, w, h, stereo=True):
    """X, Y and the eye of every pixel (steps 1-3 with the stereo call's split of output_stereo_format), and dX / 2, dY / 2."""
    x, y = np.meshgrid((np.arange(w) + 0.5) / w, (np.arange(h) + 0.5) / h)
    eye, hx, hy = np.zeros((h, w), bool), 1.0 / w, 1.0 / h
    if stereo and ctx.output_stereo_format == LR:
        eye, hx = x > 0.5, 2.0 / w
        x = np.where(eye, (x - 0.5) / 0.5, x / 0.5)
    elif stereo and ctx.output_stereo_format == TB:
        eye, hy = y > 0.5, 2.0 / h
        y = np.where(eye, (y - 0.5) / 0.5, y / 0.5)
        if ctx.vflip:
            y = np.where(eye, 1 - y, y)
    return 2 * x - 1, 2 * (1 - y) - 1, eye, hx, hy


def _context_rays(c, pose, camera):
    """test_rectilinear.rays for the equirect camera: unit rays and eyes with the context's own eye split."""
    def rays(ctx, p, w, h, mono=False):
        stereo = ctx.input_stereo_format != MONO and not mono
        X, Y, eye, _, _ = eye_xy(ctx, w, h, stereo)
        t = rays_any(p, camera, X, Y)
        return t / np.linalg.norm(t, axis=-1, keepdims=True), eye
    return rays


def equirect_poses(seed, n=4):
    rng = np.random.default_rng(seed)
    out = [((float(rng.uniform(-180, 180)), float(rng.uniform(-85, 85)), float(rng.uniform(-180, 180)), float(rng.uniform(20, 360)),
             float(rng.uniform(10, 180))), (EQUIRECT, 0.0)) for _ in range(n)]
    return out + [((0.0, 0.0, 0.0, 360.0, 180.0), (EQUIRECT, 0.0)), ((30.0, -60.0, 20.0, 180.0, 180.0), (EQUIRECT, 0.0)),
                  ((-100.0, 20.0, 5.0, 2.0, 1.5), (EQUIRECT, 0.0))]


# ---- the stereo twin and the oracle composite ----------------------------------------------------------------------------
def stereo_twin(ctx, rig, ph, pose, cam, minify, plane, in_w, in_h, w=W, h=H):
    """stereo_camera_maps of both lenses: [(map0, map1, level, weight, gain)] * 2 and eyeWeight."""
    out = [t360.stereo_camera_maps(ctx, rig, ph, pose, cam, minify, lens, plane, in_w, in_h, w, h) for lens in (0, 1)]
    assert np.array_equal(out[0][5], out[1][5])
    return [o[:5] for o in out], out[0][5]


def stereo_want(ctx, rig, ph, pose, cam, minify, srcs, out_dims, prefills):
    """test_camera_photo.photo_want with the stereo twin (eyeWeight as the seam weight): per lens the camera-mip composite,
    then s', then the choice by eye; the statistics over the pixels both lenses cover where neither sample is skipped."""
    with pytest.MonkeyPatch.context() as m:
        m.setattr(tcp, "twin", lambda c, r, p, seam, po, ca, mi, pl, iw, ih, w=W, h=H: stereo_twin(c, r, p, po, ca, mi, pl, iw, ih, w, h))
        return tcp.photo_want(ctx, rig, ph, 0.0, pose, cam, minify, srcs, out_dims, prefills)


# ---- no GPU needed -----------------------------------------------------------------------------------------------------
def test_entry_points_are_exported_with_their_bindings(tmp_path):
    from transform360_b200.handler import EXPORTED_SYMBOLS, LIB_PATH, PKG
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    L = t360.load()
    for name in ("T360B200_stereoCameraMaps", "T360B200_transformFrameStereoCameraAsync"):
        assert name in EXPORTED_SYMBOLS and name in defined, name
    P = C.POINTER
    assert L.T360B200_stereoCameraMaps.argtypes == ([P(t360.FrameTransformContext), P(t360.T360LensRig), P(t360.T360RigPhotometry),
                                                     P(t360.T360Pose), P(t360.T360Camera), P(t360.T360Minify)] + [C.c_int] * 6 + [C.c_void_p] * 6)
    assert L.T360B200_transformFrameStereoCameraAsync.argtypes == ([C.c_void_p, P(t360.T360LensRig), P(t360.T360RigPhotometry), P(t360.T360Pose),
                                                                    P(t360.T360Camera), P(t360.T360Minify), C.c_void_p, C.c_int] + [C.c_void_p] * 9)
    assert hasattr(t360.VideoFrameTransform, "make_stereo_camera_frame_call") and callable(t360.stereo_camera_maps)
    assert EQUIRECT == 5
    src = tmp_path / "decl.c"
    src.write_text('#include "transform360_b200.h"\n'
                   "_Static_assert(T360_CAMERA_EQUIRECT == 5, \"model number\");\n"
                   "int (*maps)(const FrameTransformContext*, const T360LensRig*, const T360RigPhotometry*, const T360Pose*, const T360Camera*, "
                   "const T360Minify*, int, int, int, int, int, int, float*, float*, uint8_t*, uint16_t*, uint16_t*, uint16_t*) = "
                   "T360B200_stereoCameraMaps;\n"
                   "int (*frame)(VideoFrameTransform*, const T360LensRig*, const T360RigPhotometry*, const T360Pose*, const T360Camera*, "
                   "const T360Minify*, unsigned long long*, int, const uint8_t* const*, uint8_t* const*, const int*, const int*, const int*, "
                   "const int*, const int*, const int*, void*) = T360B200_transformFrameStereoCameraAsync;\n")
    subprocess.run(["cc", "-std=c11", "-Wall", "-Werror", "-c", "-I", str(PKG.parent / "include"), "-o", str(tmp_path / "decl.o"), str(src)],
                   check=True)


# the largest |camera_map - model| the equirect row may leave, per input, a margin over what it reaches (7.3e-4 px for the
# stereo top-bottom inputs, 1.8e-4 mono equirect, 3.5e-5 cube map, 1.1e-4 for the rigs).  The top-bottom inputs' largest
# errors lie within a degree of a pole, where the input lookup's longitude atan2(x, z) takes x and z of about 1e-2 of the
# ray: the existing models reach the same there (stereographic 1.1e-3 px on tb_to_lr in test_camera_models).
MAP_BOUNDS = {"equirect": 3e-4, "tb_to_lr": 1e-3, "tb_to_tb": 1e-3, "cubemap_32": 1e-4, "single_200": 2.5e-4, "pair_190": 2.5e-4,
              "tilted": 2.5e-4}


@pytest.mark.parametrize("name", INPUTS)
def test_equirect_camera_map_equals_the_float64_model(name, monkeypatch):
    """camera_map with the equirect model against the float64 model of its row for seeded poses (hfov up to 360, vfov up to
    180) at test_camera_models' odd luma and chroma sizes, away from the same near-threshold and polar pixels: within
    MAP_BOUNDS for the input, and the same NaN pattern elsewhere."""
    import tests.test_rectilinear as tr
    rig = _rig(name, seed=len(name))
    worst, near_total, pixels = 0.0, 0, 0
    for pose, cam in equirect_poses(sum(map(ord, name))):
        for (w, h), (in_w, in_h) in zip(((97, 65), (49, 33)), tr._in_dims(name)):
            ctx = _ctx(name)
            got = t360.camera_map(ctx, pose, cam, in_w, in_h, w, h, rig).astype(np.float64)
            with monkeypatch.context() as m:
                m.setattr(tr, "rays", _context_rays(ctx, pose, cam))
                with np.errstate(divide="ignore", invalid="ignore"):
                    want, near, polar = tr.model(name, ctx, rig, pose, in_w, in_h, w, h)
            gn, wn = np.isnan(got).any(-1), np.isnan(want).any(-1)
            assert not ((gn != wn) & ~near).any(), f"{int(((gn != wn) & ~near).sum())} pixels covered differently (pose {pose})"
            if rig is None:
                assert not gn.any()
            both = ~gn & ~wn & ~near
            dx = np.abs(got[..., 0] - want[..., 0])
            dx = np.minimum(dx, np.abs(dx - in_w))
            dx[polar] = 0.0
            dy = np.abs(got[..., 1] - want[..., 1])
            if both.any():
                worst = max(worst, float(dx[both].max()), float(dy[both].max()))
            near_total += int(near.sum())
            pixels += near.size
    print(f"equirect / {name}: max |delta| {worst:.2e} px")
    assert worst <= MAP_BOUNDS[name], f"max |delta| {worst:.2e} px"
    assert near_total < 0.01 * pixels


@pytest.mark.parametrize("size", [(1024, 512), (517, 259), (97, 65)])
def test_equirect_360_at_zero_pose_is_the_identity(size):
    """A 360 x 180 equirect view at zero pose of an equirect input at its own size maps every pixel to itself: columns
    within 2e-4 px (the wrap column, where the longitude reaches +-pi, compared modulo the width), rows within 1e-3 px
    away from the two pole rows and 4e-3 px on them (where the input lookup's asin of a y near +-1 is ill-conditioned)."""
    w, h = size
    ctx = t360.make_context(**RECT_CTX, input_layout=t360.LAYOUT_EQUIRECT)
    m = t360.camera_map(ctx, (0.0, 0.0, 0.0, 360.0, 180.0), (EQUIRECT, 0.0), w, h, w, h).astype(np.float64)
    jj, ii = np.meshgrid(np.arange(w), np.arange(h))
    dx = np.abs(m[..., 0] - jj)
    dx = np.minimum(dx, np.abs(dx - w))
    dy = np.abs(m[..., 1] - ii)
    cols, rows, poles = float(dx.max()), float(dy[1:-1].max()), float(dy[[0, -1]].max())
    print(f"{w}x{h}: max |map - identity| columns {cols:.2e} px, rows {rows:.2e} px, pole rows {poles:.2e} px")
    assert cols <= 2e-4 and rows <= 1e-3 and poles <= 4e-3, (cols, rows, poles)


@pytest.mark.parametrize("name", ["equirect", "cubemap_32", "pair_190"])
def test_equirect_mip_maps_are_the_camera_map_and_the_footprint(name, monkeypatch):
    """camera_mip_maps with the equirect model: level 0 entries are camera_map's bit for bit and the other levels its
    header scaling; its level of detail is within 2/256 of a level of test_camera_mip's float64 footprint model."""
    ctx, rig = _ctx(name), _rig(name, seed=5)
    (in_w, in_h), _ = tcm._in_dims(name)
    monkeypatch.setattr(tcm, "rays64", rays_any)
    n = 0
    for k, (pose, cam) in enumerate(equirect_poses(31 + len(name), 3)[:5]):
        base = t360.camera_map(ctx, pose, cam, in_w, in_h, W, H, rig)
        m0, m1, lv, wt = t360.camera_mip_maps(ctx, pose, cam, (8, 0.0), in_w, in_h, W, H, rig)
        sizes = t360.mip_level_sizes(in_w, in_h, 8)
        for level in np.unique(lv):
            sel = lv == level
            if level == 0:
                assert same_bits(m0[sel], base[sel])
            else:
                sx, sy = np.float32(sizes[level][0] / in_w), np.float32(sizes[level][1] / in_h)
                want = np.stack([(base[..., 0] + np.float32(0.5)) * sx - np.float32(0.5), (base[..., 1] + np.float32(0.5)) * sy - np.float32(0.5)], -1)
                assert same_bits(m0[sel], want.astype(np.float32)[sel]), (pose, level)
        n += check_lod(ctx, rig, pose, cam, in_w, in_h, W, H, what=f"{name} {pose}")
    assert n > 1000, n


@pytest.mark.parametrize("minify", [None, (3, 0.0), (8, 1.0)])
@pytest.mark.parametrize("model", sorted(MODELS))
def test_mono_twin_is_the_camera_photo_twin_of_lens_0(model, minify):
    """With MONO output, lens 0's arrays equal camera_photo_maps of the one-lens rig {lens 0} with seam 0 bit for bit, with
    and without a pyramid; eyeWeight is 0 everywhere."""
    rig = stereo_rig(seed=3)
    one = t360.T360LensRig(1, rig.calibWidth, rig.calibHeight)
    one.lens[0] = rig.lens[0]
    ph = rig_photos(rig)["falloff"]
    ctx = _ctx("pair_190", output_stereo_format=MONO)
    for k in range(2):
        pose, cam = eq_pose(10 * k + len(model), MODELS[model])
        for plane, (in_w, in_h) in ((0, (1029, 515)), (1, (515, 258))):
            got = t360.stereo_camera_maps(ctx, rig, ph, pose, cam, minify, 0, plane, in_w, in_h, W, H)
            want = t360.camera_photo_maps(ctx, one, ph, 0.0, pose, cam, minify, 0, plane, in_w, in_h, W, H)
            for g, wnt in zip(got[:5], want[:5]):
                assert g.tobytes() == wnt.tobytes(), (model, minify, pose, plane)
            assert not got[5].any()
            assert np.isfinite(got[0]).any()


@pytest.mark.parametrize("fmt", ["lr", "tb", "tb_vflip"])
@pytest.mark.parametrize("model", sorted(MODELS))
def test_each_eye_takes_its_own_lens(model, fmt):
    """With LR and TB (vflip 0 and 1) output, eyeWeight is 256 on eye-1 pixels and 0 on eye-0 pixels; lens e's entries are
    given wherever it covers the ray and match a float64 projection through lens e (within 2e-3 px, away from 1e-5 rad of
    thetaMax), and the pixels of eye e are NaN for lens e exactly where it does not cover."""
    rig = stereo_rig("swapped" if model == "pannini" else "stereo_190", seed=len(model))
    ctx = _ctx("pair_190", **FORMATS[fmt])
    worst, n = 0.0, 0
    for k in range(2):
        pose, cam = eq_pose(20 * k + len(fmt), MODELS[model])
        lenses, ew = stereo_twin(ctx, rig, IDENTITY, pose, cam, None, 0, 1029, 515)
        X, Y, eye, _, _ = eye_xy(ctx, W, H)
        assert np.array_equal(ew, np.where(eye, 256, 0)), (fmt, pose)
        assert eye.any() and (~eye).any()
        d = rays_any(pose, cam, X, Y)
        d /= np.linalg.norm(d, axis=-1, keepdims=True)
        for lens in (0, 1):
            m0 = lenses[lens][0]
            px, py, th = lens_pixels64(rig, lens, d, 1029, 515)
            t_max = np.radians(np.float64(np.float32(rig.lens[lens].maxAngle)))
            sure = np.abs(th - t_max) > 1e-5
            inside = (th < t_max) & sure
            assert np.isfinite(m0[inside]).all() and np.isnan(m0[(th > t_max) & sure]).all()
            err = np.hypot(m0[inside][:, 0] - px[inside], m0[inside][:, 1] - py[inside])
            worst = max(worst, float(err.max()))
            n += int((inside & (eye == bool(lens))).sum())
    print(f"{model} {fmt}: entries within {worst:.2e} px of the float64 lens model over {n} eye pixels")
    assert worst <= 2e-3 and n > 1000


def test_equal_lenses_give_equal_halves():
    """A rig of two equal lenses with equal photometry seen through an LR view whose eye width is a power of two (so both halves' pixel centres
    fold to the same float x): the two halves of every array are equal bit for bit (each eye's pixel takes the same ray
    through the same lens), with and without a pyramid."""
    rig = stereo_rig("equal", seed=9)
    ctx = _ctx("pair_190", output_stereo_format=LR)
    w, h = 2 * 64, 91
    ph = rig_photos(rig)["falloff"]
    ph.lens[1] = ph.lens[0]
    for model in sorted(MODELS):
        pose, cam = eq_pose(7, MODELS[model])
        for minify in (None, (4, 0.5)):
            lenses, ew = stereo_twin(ctx, rig, ph, pose, cam, minify, 0, 1029, 515, w, h)
            for a, b in zip(*lenses):
                assert a[:, :w // 2].tobytes() == b[:, w // 2:].tobytes(), (model, minify)
            assert not ew[:, :w // 2].any() and (ew[:, w // 2:] == 256).all()


def _vr180_eyes(rig, ph, true_rig, in_w=2000, in_h=1000, w=360, h=180):
    """The oracle composite's luma of a 180 x 180 equirect LR view of `rig` with photometry `ph`, of a frame rendered
    through `true_rig` of a smooth scene at infinity with V(r) = 1 - 0.1 r^2 and lens 1 1.3x brighter: (left, right)."""
    scene = lambda d: 100 + 40 * d[..., 1] + 20 * d[..., 0]
    src = _render_rig(true_rig, in_w, in_h, -0.1, (1.0, 1.3), scene)
    ctx = _ctx("pair_190", t360.CUBIC, output_stereo_format=LR)
    want, _ = stereo_want(ctx, rig, ph, (0.0, 0.0, 0.0, 180.0, 180.0), (EQUIRECT, 0.0), None, [src], [(w, h)], [np.zeros((h, w), np.uint8)])
    out = want[0].astype(np.float64)
    return out[:, :w // 2], out[:, w // 2:]


def test_eyes_match_with_the_true_extrinsics_and_photometry():
    """A synthetic stereo rig (equidistant 190-degree lenses, lens 1 rotated by 2 degrees, both vignetted, lens 1 1.3x
    brighter) of a scene at infinity: the mean absolute luma difference between the two eyes' 180-degree halves with the
    true extrinsics and photometry is at most a quarter of the one with the lenses taken as unrotated and no photometry."""
    true_rig = t360.T360LensRig(2, 2000, 1000)
    for i in range(2):
        true_rig.lens[i] = t360.T360Lens(300.0, 300.0, 499.5 + 1000 * i, 499.5, (0, 0, 0, 0), 0.0, 2.0 * i, 0.0, 95)
    naive = t360.T360LensRig(2, 2000, 1000)
    naive.lens[0] = true_rig.lens[0]
    naive.lens[1] = t360.T360Lens(300.0, 300.0, 1499.5, 499.5, (0, 0, 0, 0), 0.0, 0.0, 0.0, 95)
    true_ph = photometry(0, ((-0.1, 0, 0), (-0.1, 0, 0)), ((1.0, 1, 1), (1 / 1.3, 1, 1)))
    diff = lambda lr: float(np.abs(lr[0] - lr[1]).mean())
    before = diff(_vr180_eyes(naive, IDENTITY, true_rig))
    after = diff(_vr180_eyes(true_rig, true_ph, true_rig))
    print(f"mean |left - right| luma: unrotated, no photometry {before:.2f}; true extrinsics and photometry {after:.2f} code values")
    assert before > 10 and after <= before / 4, (before, after)


def _stereo_frame(L, vft, rig, ph, pose, cam, minify, n=1, planes=(0x20000,), dims=(64, 32, 8, 8), pitch=(64, 8)):
    P, I = C.c_void_p * 3, C.c_int * 3
    arr = lambda v: I(*([v] * 3))
    return L.T360B200_transformFrameStereoCameraAsync(
        vft._h, C.byref(rig) if rig is not None else None, C.byref(ph) if ph is not None else None,
        C.byref(t360.T360Pose(*pose)) if pose is not None else None, C.byref(t360.T360Camera(*cam)) if cam is not None else None,
        C.byref(t360.T360Minify(*minify)) if minify is not None else None, 0x40000, n, P(*(list(planes) * 3)[:3]),
        P(*(list(planes) * 3)[:3]), arr(dims[0]), arr(dims[1]), arr(pitch[0]), arr(dims[2]), arr(dims[3]), arr(pitch[1]), None)


def _bad_stereo_calls():
    """(what, rig, photometry, pose, camera, minify, context overrides) the stereo twin and frame call refuse."""
    from tests.test_camera_mip import _bad_minify
    pair = stereo_rig()
    ok_pose, ok_cam = (0.0, 5.0, 0.0, 180.0, 180.0), (EQUIRECT, 0.0)
    cases = [("NULL rig", None, IDENTITY, ok_pose, ok_cam, None, {}), ("one lens", make_rig("single_200"), IDENTITY, ok_pose, ok_cam, None, {})]
    for sf in (t360.STEREO_FORMAT_GUESS, 4, -1):
        cases.append((f"output_stereo_format {sf}", pair, IDENTITY, ok_pose, ok_cam, None, dict(output_stereo_format=sf)))
    for hfov, vfov in ((0.0, 90.0), (360.5, 90.0), (90.0, 0.0), (90.0, 180.5), (float("nan"), 90.0)):
        cases.append((f"equirect fov {hfov} x {vfov}", pair, IDENTITY, (0.0, 0.0, 0.0, hfov, vfov), ok_cam, None, {}))
    cases += [(what, rig or pair, IDENTITY, pose, cam, None, ov) for what, rig, pose, cam, ov in _bad_calls() if what != "bad rig"]
    cases += [(what, rig, ph, ok_pose, ok_cam, (4, 0.0), ov) for what, rig, ph, seam, o, ov in _bad_photo_calls()
              if rig is not None and rig.numLenses == 2 and seam == 0.0 and o is not None and not what.startswith("orientation")
              and "output_layout" not in ov]
    cases += [(what, pair, IDENTITY, ok_pose, ok_cam, m, {}) for what, m in _bad_minify() if m is not None]
    return cases


def test_refusals_happen_without_a_gpu(capfd):
    """Every refusal of the twin and of the frame call comes with a message and before any CUDA call, with bogus plane and
    statistics pointers that are never dereferenced and no kernel launched; the equirect model's limits and model 4."""
    L = t360.load()
    cases = _bad_stereo_calls()
    arrays = [np.zeros((8, 8, 2), np.float32), np.zeros((8, 8, 2), np.float32), np.zeros((8, 8), np.uint8)] + \
        [np.zeros((8, 8), np.uint16) for _ in range(3)]
    ptrs = [a.ctypes.data for a in arrays]
    n0 = t360.kernel_launch_count()
    assert len(cases) > 50
    for what, rig, ph, pose, cam, minify, ov in cases:
        c = t360.make_context(**{**RECT_CTX, "output_stereo_format": LR, **ov})
        pb = C.byref(t360.T360Pose(*pose)) if pose is not None else None
        cb = C.byref(t360.T360Camera(*cam)) if cam is not None else None
        mb = C.byref(t360.T360Minify(*minify)) if minify is not None else None
        assert not L.T360B200_stereoCameraMaps(C.byref(c), C.byref(rig) if rig is not None else None, C.byref(ph) if ph is not None else None,
                                               pb, cb, mb, 0, 0, 64, 32, 8, 8, *ptrs), what
        assert "Could not compute the stereo camera maps" in _stdout(capfd), what
        with t360.VideoFrameTransform(c) as vft:
            assert "stereo rig" in _refused(capfd, _stereo_frame, L, vft, rig, ph, pose, cam, minify), what
    pair = stereo_rig()
    ctx = t360.make_context(**RECT_CTX, output_stereo_format=LR)
    pb, cb = C.byref(t360.T360Pose(0.0, 0.0, 0.0, 180.0, 180.0)), C.byref(t360.T360Camera(EQUIRECT, 0.0))
    for lens, plane in ((-1, 0), (2, 0), (0, -1), (0, 3)):
        _refused(capfd, L.T360B200_stereoCameraMaps, C.byref(ctx), C.byref(pair), C.byref(IDENTITY), pb, cb, None, lens, plane, 64, 32, 8, 8, *ptrs)
    for k in range(6):
        bad = list(ptrs)
        bad[k] = None
        _refused(capfd, L.T360B200_stereoCameraMaps, C.byref(ctx), C.byref(pair), C.byref(IDENTITY), pb, cb, None, 0, 0, 64, 32, 8, 8, *bad)
    _refused(capfd, L.T360B200_stereoCameraMaps, C.byref(ctx), C.byref(pair), C.byref(IDENTITY), pb, cb, None, 0, 0, 0, 32, 8, 8, *ptrs)
    _refused(capfd, L.T360B200_stereoCameraMaps, None, C.byref(pair), C.byref(IDENTITY), pb, cb, None, 0, 0, 64, 32, 8, 8, *ptrs)
    ok = (0.0, 0.0, 0.0, 180.0, 180.0)
    with t360.VideoFrameTransform(ctx) as vft:
        for kw in (dict(n=0), dict(n=4), dict(planes=(None,)), dict(dims=(0, 32, 8, 8)), dict(pitch=(63, 8))):
            _refused(capfd, lambda: _stereo_frame(L, vft, pair, IDENTITY, ok, (EQUIRECT, 0.0), None, **kw))
        _refused(capfd, lambda: _stereo_frame(L, vft, pair, IDENTITY, ok, (EQUIRECT, 0.0), (1, 0.0), dims=(131071, 32, 8, 8), pitch=(131072, 8)))
        assert _stdout(capfd) == ""
    assert not L.T360B200_transformFrameStereoCameraAsync(None, None, None, None, None, None, None, 1, *([None] * 9))
    # the equirect model through the other calls: its limits, and model 4 still refused
    mono = t360.make_context(**RECT_CTX)
    for hfov, vfov in ((360.5, 90.0), (90.0, 180.5), (0.0, 90.0)):
        with pytest.raises(ValueError):
            t360.camera_map(mono, (0.0, 0.0, 0.0, hfov, vfov), EQUIRECT, 64, 32, 8, 8)
    with pytest.raises(ValueError):
        t360.camera_map(mono, (0.0, 0.0, 0.0, 90.0, 60.0), (4, 0.0), 64, 32, 8, 8)
    assert t360.kernel_launch_count() == n0
    # accepted: the limits, a TB output with vflip, a MONO output of a context with a stereo input format
    t360.camera_map(mono, (0.0, 0.0, 0.0, 360.0, 180.0), EQUIRECT, 64, 32, 8, 8)
    for ov in (dict(output_stereo_format=TB, vflip=1), dict(input_stereo_format=TB, output_stereo_format=MONO)):
        c = t360.make_context(**RECT_CTX, **ov)
        for minify in (None, (0, -4.0), (8, 4.0)):
            t360.stereo_camera_maps(c, pair, IDENTITY, ok, EQUIRECT, minify, 1, 2, 64, 32, 8, 8)


# ---- on the GPU --------------------------------------------------------------------------------------------------------
def _call(vft, f):
    return vft.make_stereo_camera_frame_call(f.in_planes, f.out_planes, f.dims)


def _prefill(f, torch):
    for p, o in enumerate(f.outs):
        o[:, :f.out_dims[p][0]] = torch.from_numpy(f.prefill[p]).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("interp", INTERPS)
@pytest.mark.parametrize("model", sorted(MODELS))
def test_frames_and_statistics_equal_the_oracle(model, interp, torch_cuda):
    """MONO, LR and TB (vflip 0 and 1) output, no pyramid, (3, 0) and (4, 1.0), a non-identity photometry, odd sizes:
    3-plane frames equal the oracle's composite bit for bit with and without statistics, and the statistics its sums."""
    torch = torch_cuda
    st = torch.cuda.Stream()
    stats = torch.zeros((3, STATS), dtype=torch.int64, device="cuda")
    rig = stereo_rig("swapped" if interp % 2 else "stereo_190", seed=interp + len(model))
    ph = rig_photos(rig)["falloff"]
    for fmt, ov in FORMATS.items():
        ctx = _ctx("pair_190", interp, **ov)
        vft = t360.VideoFrameTransform(ctx)
        for k, minify in enumerate(MINIFIES):
            pose, cam = eq_pose(31 * interp + 7 * k + len(fmt), MODELS[model])
            f = MipFrame(torch, "pair_190", 3, seed=interp + k)
            want, sums = stereo_want(ctx, rig, ph, pose, cam, minify, f.src, f.out_dims, f.prefill)
            what = f"{fmt} minify {minify} {pose}"
            for with_stats in (False, True):
                _prefill(f, torch)
                stats.fill_(-1)
                torch.cuda.synchronize()
                assert _call(vft, f)(rig, ph, pose, cam, minify, st.cuda_stream, stats.data_ptr() if with_stats else 0)
                st.synchronize()
                for p, got in enumerate(f.host()):
                    _check(got, want[p], f"{what}, statistics {with_stats}, plane {p}")
                got_sums = stats.cpu().numpy()
                if with_stats:
                    for p in range(3):
                        assert got_sums[p].tolist() == sums[p], f"{what}: plane {p} statistics {got_sums[p].tolist()} != {sums[p]}"
                    assert got_sums[0][0] > 0, f"{what}: no overlap pixel"
                else:
                    assert (got_sums == -1).all()
        vft.close()


@pytest.mark.gpu
@pytest.mark.parametrize("interp", INTERPS)
def test_equirect_model_through_the_camera_calls(interp, torch_cuda):
    """The equirect model through the camera call (context inputs and a rig: the oracle's cv::remap of camera_map, and the
    planned camera_map path), the camera-mip call and the camera-photo call: every frame equals its oracle composite."""
    from tests.test_camera_models import _want
    from tests.test_rectilinear import Frame
    torch = torch_cuda
    st = torch.cuda.Stream()
    for name in ("equirect", "tb_to_tb", "cubemap_32", "pair_190"):
        ctx, rig = _ctx(name, interp), _rig(name, seed=interp)
        pose, cam = equirect_poses(interp * 10 + len(name), 1)[0]
        vft = t360.VideoFrameTransform(ctx)
        f = Frame(torch, name, 3, seed=interp)
        want, maps = _want(f, ctx, rig, pose, cam)
        torch.cuda.synchronize()
        assert vft.make_camera_frame_call(f.in_planes, f.out_planes, f.dims)(pose, cam, st.cuda_stream, rig)
        st.synchronize()
        for p, got in enumerate(f.host()):
            _check(got, want[p], f"{name} camera frame, plane {p}")
        g = Frame(torch, name, 3, seed=interp)
        for idx in (0, 1):
            assert vft.generate_map_from_warp(maps[idx], *g.in_dims[idx], idx, TRANSPARENT if rig is not None else WRAP)
        torch.cuda.synchronize()
        assert vft.make_frame_call(g.in_planes, g.out_planes, g.dims)(st.cuda_stream)
        st.synchronize()
        for p, got in enumerate(g.host()):
            _check(got, want[p], f"{name} planned camera frame, plane {p}")
        vft.close()
        if name in ("equirect", "pair_190"):
            vft = t360.VideoFrameTransform(ctx)
            for minify in ((3, 0.0), (8, 1.0)):
                m = MipFrame(torch, name, 3, seed=interp)
                want = m.want(ctx, rig, pose, cam, minify)
                torch.cuda.synchronize()
                assert vft.make_camera_mip_frame_call(m.in_planes, m.out_planes, m.dims)(pose, cam, minify, st.cuda_stream, rig)
                st.synchronize()
                for p, got in enumerate(m.host()):
                    _check(got, want[p], f"{name} camera-mip frame {minify}, plane {p}")
            vft.close()
    ctx, rig = _ctx("pair_190", interp), make_rig("pair_190", seed=interp)
    ph = rig_photos(rig)["falloff"]
    vft = t360.VideoFrameTransform(ctx)
    for seam, minify in ((0.0, None), (4.0, (4, 1.0))):
        pose, cam = (90.0, 10.0, 0.0, 200.0, 120.0), (EQUIRECT, 0.0)
        f = MipFrame(torch, "pair_190", 3, seed=interp)
        want, sums = tcp.photo_want(ctx, rig, ph, seam, pose, cam, minify, f.src, f.out_dims, f.prefill)
        stats = torch.zeros((3, STATS), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        assert vft.make_camera_photo_frame_call(f.in_planes, f.out_planes, f.dims)(rig, ph, seam, pose, cam, minify, st.cuda_stream, stats.data_ptr())
        st.synchronize()
        for p, got in enumerate(f.host()):
            _check(got, want[p], f"camera-photo frame seam {seam}, plane {p}")
        assert stats.cpu().numpy().tolist() == sums
    vft.close()


@pytest.mark.gpu
def test_mono_frame_is_the_camera_photo_call_of_lens_0(torch_cuda):
    """With MONO output and statistics off the stereo frame equals transformFrameCameraPhotoAsync's with the one-lens rig
    {lens 0} and seam 0 byte for byte, with and without a pyramid, every model and interpolator."""
    torch = torch_cuda
    rig = stereo_rig(seed=4)
    one = t360.T360LensRig(1, rig.calibWidth, rig.calibHeight)
    one.lens[0] = rig.lens[0]
    ph = rig_photos(rig)["falloff"]
    st = torch.cuda.Stream()
    for interp in INTERPS:
        vft = t360.VideoFrameTransform(_ctx("pair_190", interp, output_stereo_format=MONO, input_stereo_format=TB))
        for model in sorted(MODELS):
            pose, cam = eq_pose(interp + len(model), MODELS[model])
            for minify in MINIFIES:
                a, b = MipFrame(torch, "pair_190", 3, seed=interp), MipFrame(torch, "pair_190", 3, seed=interp)
                torch.cuda.synchronize()
                assert _call(vft, a)(rig, ph, pose, cam, minify, st.cuda_stream)
                assert vft.make_camera_photo_frame_call(b.in_planes, b.out_planes, b.dims)(one, ph, 0.0, pose, cam, minify, st.cuda_stream)
                st.synchronize()
                for p, (x, y) in enumerate(zip(a.host(), b.host())):
                    assert np.array_equal(x, y), (interp, model, minify, p)
        vft.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["lr", "tb_vflip"])
def test_eye_combined_twin_map_planned_is_the_frame(fmt, torch_cuda):
    """The identity photometry without a pyramid: the twin's two map0 arrays combined by eye, planned with
    generate_map_from_warp(..., BORDER_TRANSPARENT) and served by transformFrameAsync, give the stereo frame byte for byte
    (the VR180 recipe for a fixed pose)."""
    torch = torch_cuda
    rig = stereo_rig(seed=8)
    st = torch.cuda.Stream()
    for interp in INTERPS:
        ctx = _ctx("pair_190", interp, **FORMATS[fmt])
        vft = t360.VideoFrameTransform(ctx)
        pose, cam = (3.0, -2.0, 1.0, 180.0, 180.0), (EQUIRECT, 0.0)
        a, b = MipFrame(torch, "pair_190", 3, seed=interp), MipFrame(torch, "pair_190", 3, seed=interp)
        for idx, (in_w, in_h) in enumerate(a.in_dims[:2]):
            w, h = a.out_dims[idx]
            lenses, ew = stereo_twin(ctx, rig, IDENTITY, pose, cam, None, idx, in_w, in_h, w, h)
            m = np.where((ew == 256)[..., None], lenses[1][0], lenses[0][0])
            assert vft.generate_map_from_warp(m, in_w, in_h, idx, TRANSPARENT)
        torch.cuda.synchronize()
        assert _call(vft, a)(rig, IDENTITY, pose, cam, None, st.cuda_stream)
        assert vft.make_frame_call(b.in_planes, b.out_planes, b.dims)(st.cuda_stream)
        st.synchronize()
        for p, (x, y) in enumerate(zip(a.host(), b.host())):
            assert np.array_equal(x, y), (fmt, interp, p, int((x != y).sum()))
        vft.close()


@pytest.mark.gpu
def test_trajectory_on_two_streams(torch_cuda):
    """Two streams enqueue 24 frames without synchronising, pose, camera model, photometry and minify changing every
    frame, a statistics buffer each frame: every frame and its statistics equal the oracle."""
    torch = torch_cuda
    ctx = _ctx("pair_190", t360.CUBIC, output_stereo_format=LR)
    rig = stereo_rig(seed=61)
    rng = np.random.default_rng(22)
    args = []
    for k in range(24):
        pose, cam = eq_pose(500 + k, MODELS[sorted(MODELS)[k % 5]])
        ph = photometry(16, [tuple(rng.uniform([-0.5, -0.1, 0], [0, 0.1, 0.01]) / r_max(rig.lens[i]) ** np.array([2, 4, 6])) for i in range(2)],
                        [tuple(rng.uniform(0.7, 1.4, 3)) for _ in range(2)], [tuple(rng.uniform(-8, 8, 3)) for _ in range(2)])
        args.append((ph, pose, cam, (None, (2, 0.0), (5, -0.5), (8, 1.0))[k % 4]))
    vft = t360.VideoFrameTransform(ctx)
    frames = [MipFrame(torch, "pair_190", 3, seed=k % 4) for k in range(24)]
    stats = torch.zeros((24, 3, STATS), dtype=torch.int64, device="cuda")
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for k, (f, (ph, pose, cam, minify)) in enumerate(zip(frames, args)):
        assert _call(vft, f)(rig, ph, pose, cam, minify, streams[k % 2].cuda_stream, stats[k].data_ptr())
    torch.cuda.synchronize()
    got_stats = stats.cpu().numpy()
    for k, (f, (ph, pose, cam, minify)) in enumerate(zip(frames, args)):
        want, sums = stereo_want(ctx, rig, ph, pose, cam, minify, f.src, f.out_dims, f.prefill)
        for p, got in enumerate(f.host()):
            _check(got, want[p], f"frame {k}, plane {p}")
            assert got_stats[k, p].tolist() == sums[p], f"frame {k}, plane {p} statistics"
    vft.close()


@pytest.mark.gpu
def test_device_memory_and_launches_stay_bounded(torch_cuda):
    """60 frames after a warm-up, minify and statistics changing: T_max + 1 launches each (1 without a pyramid) and no
    growth of device memory."""
    torch = torch_cuda
    ctx = _ctx("pair_190", t360.LANCZOS4, output_stereo_format=TB, vflip=1)
    rig = stereo_rig(seed=91)
    vft = t360.VideoFrameTransform(ctx)
    f = MipFrame(torch, "pair_190", 3)
    call = _call(vft, f)
    stats = torch.zeros((3, STATS), dtype=torch.int64, device="cuda")
    st = torch.cuda.Stream()
    ph = rig_photos(rig)["falloff"]
    minifies = [None, (3, 0.0), (8, 0.5)]
    tops = [0 if m is None else len(t360.mip_level_sizes(*_in_dims("pair_190")[0], m[0])) - 1 for m in minifies]

    def frame(i):
        return call(rig, ph, (3.0 * (i % 5), 1.0, 0.0, 180.0, 180.0), (EQUIRECT, 0.0), minifies[i % 3], st.cuda_stream,
                    stats.data_ptr() if i % 4 else 0)
    for i in range(6):
        assert frame(i)
    st.synchronize()
    free_before = torch.cuda.mem_get_info()[0]
    n0 = t360.kernel_launch_count()
    for i in range(60):
        assert frame(i)
    launches = t360.kernel_launch_count() - n0
    st.synchronize()
    assert launches == sum(tops[i % 3] + 1 for i in range(60)), launches
    assert torch.cuda.mem_get_info()[0] >= free_before - (2 << 20), "device memory grew"
    vft.close()


@pytest.mark.gpu
def test_refused_calls_launch_nothing_and_leave_the_outputs(torch_cuda, capfd):
    """Refused frames on real planes and a real statistics buffer: no kernel launch, the outputs and the statistics keep
    their bytes."""
    torch = torch_cuda
    f = MipFrame(torch, "pair_190", 3)
    stats = torch.full((3, STATS), 5, dtype=torch.int64, device="cuda")
    before = f.host()
    pair, single = stereo_rig(), make_rig("single_200")
    ok = (0.0, 0.0, 0.0, 180.0, 180.0)
    torch.cuda.synchronize()
    n0 = t360.kernel_launch_count()
    for ov, rig, ph, pose, cam, minify in ((dict(output_stereo_format=LR), single, IDENTITY, ok, EQUIRECT, None),
                                           (dict(output_stereo_format=t360.STEREO_FORMAT_GUESS), pair, IDENTITY, ok, EQUIRECT, None),
                                           (dict(output_stereo_format=LR), pair, photometry(gain=((0, 1, 1), (1, 1, 1))), ok, EQUIRECT, None),
                                           (dict(output_stereo_format=TB), pair, IDENTITY, (0.0, 0.0, 0.0, 180.0, 181.0), EQUIRECT, None),
                                           (dict(output_stereo_format=LR), pair, IDENTITY, ok, EQUIRECT, (9, 0.0))):
        vft = t360.VideoFrameTransform(_ctx("pair_190", **ov))
        _refused(capfd, _call(vft, f), rig, ph, pose, cam, minify, 0, stats.data_ptr())
        vft.close()
    torch.cuda.synchronize()
    assert t360.kernel_launch_count() == n0
    assert all(np.array_equal(a, b) for a, b in zip(before, f.host()))
    assert (stats.cpu().numpy() == 5).all()
