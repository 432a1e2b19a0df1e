"""Camera views of a lens rig with photometry: the rectilinear view, the other camera models and the anti-aliased views
with each lens corrected before a hard or feathered seam (T360B200_cameraPhotoMaps / camera_photo_maps,
T360B200_transformFrameCameraPhotoAsync / make_camera_photo_frame_call).

What pins what:
  - the twin with the identity photometry and seamWidth 0: the closer lens's entries are camera_map's (no pyramid) and
    camera_mip_maps' (with one) bit for bit, its levels and weights too where it covers the ray, its gain 4096;
  - the farther lens's entries and levels against float64 models of its projection and footprint, w and the gains
    against the float64 models of test_lens_photo.py;
  - the seam: a synthetic rig of a smooth scene with a falloff and an exposure mismatch, seen through a pinhole view across
    the seam, has a luma step at most a quarter of the uncorrected hard seam's;
  - the frames and statistics against the oracle's composite of the twin (the camera-mip composite per lens, then s',
    then the seam), and the identity frames against the camera and camera-mip calls byte for byte.
Poses, rigs and planes are made from seeds."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import transform360_b200 as t360
from transform360_b200.handler import as_minify
from tests.test_camera_mip import (MODELS, MipFrame, _in_dims, composite, pixel_xy, pyramid, rays64, same_bits,
                                   wide_pose)
from tests.test_camera_models import EQUIDISTANT, PINHOLE, _bad_calls
from tests.test_lens import _rot, make_rig
from tests.test_lens_photo import (IDENTITY, STATS, _bad_photo_calls, _falloff, _mild, _render_rig, correct, equidistant_pair, offset_q,
                                   photometry, r_max, rig_photos)
from tests.test_rectilinear import INTERPS, RECT_CTX, _ctx
from tests.test_rectilinear import torch_cuda  # noqa: F401 (fixture)
from tests.test_warp_map import _check, _refused, _stdout

RIGS = ["single_200", "pair_190"]
MINIFIES = [None, (3, 0.0), (4, 1.0)]
W, H = 97, 65


def seam_pose(model, seed):
    """wide_pose's pose turned to look along the seam of a back-to-back pair (yaw 90 +- 25), so the view straddles it."""
    pose, cam = wide_pose(model, seed)
    rng = np.random.default_rng(seed + 1)
    return (90.0 + float(rng.uniform(-25, 25)), float(rng.uniform(-30, 30)), pose[2], *pose[3:]), cam


def twin(ctx, rig, ph, seam, pose, cam, minify, plane, in_w, in_h, w=W, h=H):
    """camera_photo_maps of both lenses: [(map0, map1, level, weight, gain)] * 2 and the seam weight."""
    out = [t360.camera_photo_maps(ctx, rig, ph, seam, pose, cam, minify, lens, plane, in_w, in_h, w, h) for lens in (0, 1)]
    assert np.array_equal(out[0][5], out[1][5])
    return [o[:5] for o in out], out[0][5]


# ---- the oracle's composite --------------------------------------------------------------------------------------------
def photo_want(ctx, rig, ph, seam, pose, cam, minify, srcs, out_dims, prefills):
    """The oracle's planes and statistics: per lens the camera-mip composite of its arrays (cv::resize INTER_AREA
    pyramids, cv::remap per level under BORDER_TRANSPARENT, the level blend; sampled into 1 and into 255: where the two
    differ the lens's sample is skipped), s' with its gain, then the seam as in test_lens_photo.photo_composite."""
    interp = ctx.interpolation_alg
    max_level = 0 if minify is None else as_minify(minify).maxLevel
    want, sums = [], []
    for p, src in enumerate(srcs):
        w, h = out_dims[p]
        lenses, wt = twin(ctx, rig, ph, seam, pose, cam, minify, p, src.shape[1], src.shape[0], w, h)
        levels = pyramid(src, max_level)
        pivot = ph.lumaPivot if p == 0 else 128
        val, ok, fin = [], [], []
        for i, (m0, m1, lv, lw, g) in enumerate(lenses):
            lo = composite(levels, m0, m1, lv, lw, interp, np.ones((h, w), np.uint8))
            hi = composite(levels, m0, m1, lv, lw, interp, np.full((h, w), 255, np.uint8))
            val.append(correct(lo, g, offset_q(ph.lens[i].offset[p]), pivot))
            ok.append(lo == hi)
            fin.append(np.isfinite(m0).all(-1))
        (a, b), (va, vb) = val, ok
        wt = wt.astype(np.int64)
        out = prefills[p].astype(np.int64).copy()
        lone0, lone1, mid = wt == 0, wt == 256, (wt > 0) & (wt < 256)
        out[lone0 & va] = a[lone0 & va]
        out[lone1 & vb] = b[lone1 & vb]
        out[mid & va & ~vb] = a[mid & va & ~vb]
        out[mid & vb & ~va] = b[mid & vb & ~va]
        both = mid & va & vb
        out[both] = (a[both] * (256 - wt[both]) + b[both] * wt[both] + 128) >> 8
        ov = fin[0] & fin[1] & va & vb
        want.append(out.astype(np.uint8))
        sums.append([int(ov.sum()), int(a[ov].sum()), int(b[ov].sum()), int((a[ov] ** 2).sum()), int((b[ov] ** 2).sum()),
                     int((a[ov] * b[ov]).sum())])
    return want, sums


# ---- float64 models of one lens --------------------------------------------------------------------------------------
def lens_pixels64(rig, lens, d, in_w, in_h):
    """(px, py, theta) of unit rays d through lens `lens` in float64 (the lens calls' projection, uncovered rays
    included)."""
    L = rig.lens[lens]
    c = d @ _rot(L.yaw, L.pitch, L.roll)
    X, Y, Z = c[..., 0], -c[..., 1], c[..., 2]
    k = [np.float64(np.float32(x)) for x in L.k]
    rho = np.hypot(X, Y)
    th = np.arctan2(rho, Z)
    t = th * th
    thd = th * (1 + t * (k[0] + t * (k[1] + t * (k[2] + t * k[3]))))
    s = np.where(rho > 0, thd / np.where(rho > 0, rho, 1), 1 / np.where(Z > 0, Z, 1))
    px = (L.fx * s * X + L.cx + 0.5) / rig.calibWidth * in_w - 0.5
    py = (L.fy * s * Y + L.cy + 0.5) / rig.calibHeight * in_h - 0.5
    return px, py, th


def lens_footprint64(ctx, rig, lens, pose, camera, in_w, in_h, w, h):
    """test_camera_mip.footprint64 for a chosen lens: rho^2 of the central difference of that lens's projection."""
    X, Y, hx, hy = pixel_xy(ctx, w, h, mono=True)
    t = rays64(pose, camera, X, Y)
    rx = rays64(pose, camera, X + hx, Y) - rays64(pose, camera, X - hx, Y)
    ry = rays64(pose, camera, X, Y + hy) - rays64(pose, camera, X, Y - hy)
    n = np.linalg.norm(t, axis=-1, keepdims=True)
    outs = []
    for r in (rx, ry):
        eps = 1e-6 * n / np.linalg.norm(r, axis=-1, keepdims=True)
        p1 = lens_pixels64(rig, lens, (t + eps * r) / n, in_w, in_h)
        p0 = lens_pixels64(rig, lens, (t - eps * r) / n, in_w, in_h)
        outs.append(((p1[0] - p0[0]) / (2 * eps[..., 0])) ** 2 + ((p1[1] - p0[1]) / (2 * eps[..., 0])) ** 2)
    return np.maximum(*outs), t / n


# ---- no GPU needed -----------------------------------------------------------------------------------------------------
def test_entry_points_are_exported_with_their_bindings(tmp_path):
    from transform360_b200.handler import EXPORTED_SYMBOLS, LIB_PATH, PKG
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    L = t360.load()
    for name in ("T360B200_cameraPhotoMaps", "T360B200_transformFrameCameraPhotoAsync"):
        assert name in EXPORTED_SYMBOLS and name in defined, name
    P = C.POINTER
    assert L.T360B200_cameraPhotoMaps.argtypes == ([P(t360.FrameTransformContext), P(t360.T360LensRig), P(t360.T360RigPhotometry), C.c_float,
                                                    P(t360.T360Pose), P(t360.T360Camera), P(t360.T360Minify)] + [C.c_int] * 6 + [C.c_void_p] * 6)
    assert L.T360B200_transformFrameCameraPhotoAsync.argtypes == ([C.c_void_p, P(t360.T360LensRig), P(t360.T360RigPhotometry), C.c_float,
                                                                   P(t360.T360Pose), P(t360.T360Camera), P(t360.T360Minify), C.c_void_p,
                                                                   C.c_int] + [C.c_void_p] * 9)
    assert hasattr(t360.VideoFrameTransform, "make_camera_photo_frame_call") and callable(t360.camera_photo_maps)
    src = tmp_path / "decl.c"
    src.write_text('#include "transform360_b200.h"\n'
                   "int (*maps)(const FrameTransformContext*, const T360LensRig*, const T360RigPhotometry*, float, const T360Pose*, "
                   "const T360Camera*, const T360Minify*, int, int, int, int, int, int, float*, float*, uint8_t*, uint16_t*, uint16_t*, "
                   "uint16_t*) = T360B200_cameraPhotoMaps;\n"
                   "int (*frame)(VideoFrameTransform*, const T360LensRig*, const T360RigPhotometry*, float, const T360Pose*, const T360Camera*, "
                   "const T360Minify*, unsigned long long*, int, const uint8_t* const*, uint8_t* const*, const int*, const int*, const int*, "
                   "const int*, const int*, const int*, void*) = T360B200_transformFrameCameraPhotoAsync;\n")
    subprocess.run(["cc", "-std=c11", "-Wall", "-Werror", "-c", "-I", str(PKG.parent / "include"), "-o", str(tmp_path / "decl.o"), str(src)],
                   check=True)


def _closer(rig, pose, cam, ctx, w=W, h=H):
    """Whether lens 1 is the closer lens of every pixel's ray (lensPosition's choice in float64; ties are not decided)."""
    X, Y, _, _ = pixel_xy(ctx, w, h, mono=True)
    d = rays64(pose, cam, X, Y)
    if rig.numLenses == 1:
        return np.zeros((h, w), bool), np.zeros((h, w), bool)
    z = [(d @ _rot(rig.lens[i].yaw, rig.lens[i].pitch, rig.lens[i].roll))[..., 2] for i in range(2)]
    return z[1] > z[0], np.abs(z[1] - z[0]) < 1e-5 * np.linalg.norm(d, axis=-1)


@pytest.mark.parametrize("name", RIGS)
@pytest.mark.parametrize("model", sorted(MODELS))
def test_identity_closer_lens_is_the_camera_and_mip_maps(model, name):
    """With the identity photometry and seamWidth 0 the closer lens's entries equal camera_map's without a pyramid and
    camera_mip_maps' with one, bit for bit, and its level and weight where it covers the ray; its gain is 4096 and w
    names it (0 or 256)."""
    ctx, rig = _ctx(name), make_rig(name, seed=3)
    (in_w, in_h), _ = _in_dims(name)
    for k in range(3):
        pose, cam = seam_pose(MODELS[model], 100 * k + len(name))
        for minify in MINIFIES:
            lenses, wt = twin(ctx, rig, IDENTITY, 0.0, pose, cam, minify, 0, in_w, in_h)
            second = wt == 256
            assert set(np.unique(wt)) <= {0, 256}
            pick = lambda a, b: np.where(second[(...,) + (None,) * (a.ndim - 2)], b, a)
            m0, m1, lv, lw, g = (pick(lenses[0][j], lenses[1][j]) for j in range(5))
            covered = np.isfinite(m0).all(-1)
            if minify is None:
                want = t360.camera_map(ctx, pose, cam, in_w, in_h, W, H, rig)
                assert same_bits(m0, want) and np.isnan(m1).all() and not lv.any() and not lw.any(), (model, name, pose)
            else:
                w0, w1, wl, ww = t360.camera_mip_maps(ctx, pose, cam, minify, in_w, in_h, W, H, rig)
                assert same_bits(m0, w0) and same_bits(m1[covered], w1[covered]), (model, name, pose, minify)
                assert np.array_equal(lv[covered], wl[covered]) and np.array_equal(lw[covered], ww[covered]), (model, name, pose, minify)
                assert not lv[~covered].any() and not lw[~covered].any()
                assert len(np.unique(lv[covered])) > 1, "the views are minified"
            assert (g[covered] == 4096).all() and not g[~covered].any()
            if rig.numLenses == 2:
                want_second, tie = _closer(rig, pose, cam, ctx)
                assert np.array_equal(second[~tie], want_second[~tie])
                assert second.any() and (~second).any(), "the view straddles the seam"


@pytest.mark.parametrize("model", sorted(MODELS))
def test_farther_lens_against_the_float64_models(model):
    """Both lenses of a pair, the farther one included: entries within 2e-3 px of a float64 projection through that lens
    and lambda256 within 2/256 level of its float64 footprint through the header's bit rule (pixels where the float32
    chain may differ in coverage, within 1e-5 rad of thetaMax, are left out); NaN entries exactly where it does not
    cover the ray."""
    from tests.test_camera_mip import bit_rule
    ctx, rig = _ctx("pair_190"), make_rig("pair_190", seed=11)
    (in_w, in_h), _ = _in_dims("pair_190")
    worst_px, worst_lam, n = 0.0, 0, 0
    for k in range(3):
        pose, cam = seam_pose(MODELS[model], 40 + k)
        for minify in (None, (8, 0.0)):
            lenses, _ = twin(ctx, rig, IDENTITY, 0.0, pose, cam, minify, 0, in_w, in_h)
            top = len(t360.mip_level_sizes(in_w, in_h, 8)) - 1
            for lens in (0, 1):
                m0, _, lv, lw, _ = lenses[lens]
                rho2, d = lens_footprint64(ctx, rig, lens, pose, cam, in_w, in_h, W, H)
                px, py, th = lens_pixels64(rig, lens, d, in_w, in_h)
                t_max = np.radians(np.float64(np.float32(rig.lens[lens].maxAngle)))
                sure = np.abs(th - t_max) > 1e-5
                inside = (th < t_max) & sure
                assert np.isfinite(m0[inside]).all() and np.isnan(m0[(th > t_max) & sure]).all()
                if minify is None:
                    err = np.hypot(m0[inside][:, 0] - px[inside], m0[inside][:, 1] - py[inside])
                    worst_px = max(worst_px, float(err.max()))
                else:
                    lam = lv.astype(np.int64) * 256 + lw
                    model64 = bit_rule(rho2)
                    free = inside & (lam > 0) & (lam < 256 * top)
                    diff = np.abs(lam - model64)[free]
                    worst_lam = max(worst_lam, int(diff.max()) if diff.size else 0)
                    n += int(free.sum())
    print(f"{model}: entries within {worst_px:.2e} px, lambda256 within {worst_lam}/256 level over {n} px")
    assert worst_px <= 2e-3 and worst_lam <= 2 and n > 1000


@pytest.mark.parametrize("model", sorted(MODELS))
def test_seam_weight_and_gains_against_the_float64_models(model):
    """w of the feathered seam within 1 of 256 clamp(0.5 + (theta0 - theta1) / (2 seamWidth)) and each lens's Gq within 1
    of 4096 gain / V(theta_d) in float64, for seeded falloffs and gains, every plane, pixels within 1e-5 rad of a
    coverage bound left out."""
    rng = np.random.default_rng(len(model))
    rig = _mild(make_rig("pair_190", seed=len(model)))
    ctx = _ctx("pair_190")
    worst_g, worst_w = 0.0, 0.0
    for k in range(2):
        pose, cam = seam_pose(MODELS[model], 7 + k)
        ph = photometry(int(rng.integers(0, 256)), [_falloff(rng, rig.lens[i]) for i in range(2)],
                        [tuple(rng.uniform(0.05, 8.0, 3)) for _ in range(2)], [tuple(rng.uniform(-64, 64, 3)) for _ in range(2)])
        X, Y, _, _ = pixel_xy(ctx, W, H, mono=True)
        d = rays64(pose, cam, X, Y)
        d /= np.linalg.norm(d, axis=-1, keepdims=True)
        ths = [lens_pixels64(rig, i, d, 259, 131)[2] for i in range(2)]
        t_max = [np.radians(np.float64(np.float32(rig.lens[i].maxAngle))) for i in range(2)]
        sure = (np.abs(ths[0] - t_max[0]) > 1e-5) & (np.abs(ths[1] - t_max[1]) > 1e-5)
        for plane in (0, 1, 2):
            for seam in (0.0, 6.0):
                lenses, wt = twin(ctx, rig, ph, seam, pose, cam, (3, 0.0), plane, 259, 131)
                for i in range(2):
                    L = rig.lens[i]
                    k4 = [np.float64(np.float32(x)) for x in L.k]
                    th = ths[i]
                    r2 = (th * (1 + k4[0] * th ** 2 + k4[1] * th ** 4 + k4[2] * th ** 6 + k4[3] * th ** 8)) ** 2
                    v = [np.float64(np.float32(x)) for x in ph.lens[i].vignetting]
                    gm = np.minimum(4096 * np.float64(np.float32(ph.lens[i].gain[plane])) / (1 + r2 * (v[0] + r2 * (v[1] + r2 * v[2]))), 65535)
                    sel = (th < t_max[i]) & sure
                    worst_g = max(worst_g, float(np.abs(lenses[i][4][sel] - gm[sel]).max()))
                    assert not lenses[i][4][(th > t_max[i]) & sure].any()
                if seam > 0:
                    both = (ths[0] < t_max[0]) & (ths[1] < t_max[1]) & sure
                    wm = 256 * np.clip(0.5 + (ths[0] - ths[1]) / (2 * np.radians(seam)), 0, 1)
                    worst_w = max(worst_w, float(np.abs(wt[both] - wm[both]).max()))
                    assert both.sum() > 100
    assert worst_g <= 1.0 and worst_w <= 1.0, (worst_g, worst_w)


def _seam_frame(ph, seam, pose=(90.0, 0.0, 0.0, 60.0, 45.0), w=360, h=270, in_w=2000, in_h=1000):
    """The oracle composite's luma of a pinhole view across the seam of an equidistant pair rendered with V(r) = 1 - 0.1 r^2
    and lens 1 1.3x brighter, of a scene that is smooth across the seam."""
    rig = equidistant_pair()
    scene = lambda d: 100 + 40 * d[..., 1] + 20 * d[..., 0]
    src = _render_rig(rig, in_w, in_h, -0.1, (1.0, 1.3), scene)
    ctx = _ctx("pair_190", t360.CUBIC)
    want, _ = photo_want(ctx, rig, ph, seam, pose, (PINHOLE, 0.0), None, [src], [(w, h)], [np.zeros((h, w), np.uint8)])
    return want[0].astype(np.float64)


def test_seam_step_is_removed():
    """A pinhole view looking along the seam of a synthetic dual-fisheye rig (V(r) = 1 - 0.1 r^2, lens 1 1.3x brighter, a
    scene smooth across the seam): the mean luma step across the seam column with the true photometry and a 4-degree belt
    is at most a quarter of the uncorrected hard seam's."""
    w, h = 360, 270
    c = w // 2  # the seam plane (yaw 90) is the view's centre column
    cols = (c - 16, c + 16)  # 2.7 degrees either side: clear of a 4-degree belt (2 degrees, 12 px, each side)
    rows = slice(h // 4, 3 * h // 4)

    def step(img):
        return float(np.abs(img[rows, cols[0]] - img[rows, cols[1]]).mean())
    hard = step(_seam_frame(IDENTITY, 0.0))
    true = photometry(0, ((-0.1, 0, 0), (-0.1, 0, 0)), ((1.0, 1, 1), (1 / 1.3, 1, 1)))
    fixed = step(_seam_frame(true, 4.0))
    print(f"luma step across the seam: hard, uncorrected {hard:.2f}; true photometry, 4-degree belt {fixed:.2f} code values")
    assert hard > 10 and fixed <= hard / 4, (hard, fixed)


def test_refusals_happen_without_a_gpu(capfd):
    """Every refusal of the twin and of the frame call comes with a message and before any CUDA call, with bogus plane
    and statistics pointers that are never dereferenced and no kernel launched: a NULL rig, the camera views' refusals with
    a rig, the photometric lens call's seam and photometry refusals, and minify's when it is given."""
    from tests.test_camera_mip import _bad_minify
    L = t360.load()
    pair = make_rig("pair_190")
    ok_pose, ok_cam = (80.0, 5.0, 0.0, 90.0, 60.0), (EQUIDISTANT, 0.0)
    cases = [("NULL rig", None, IDENTITY, 0.0, ok_pose, ok_cam, None, {})]
    cases += [(what, rig or pair, IDENTITY, 0.0, pose, cam, None, ov) for what, rig, pose, cam, ov in _bad_calls()]
    cases += [(what, rig, ph, seam, ok_pose, ok_cam, (4, 0.0), ov) for what, rig, ph, seam, o, ov in _bad_photo_calls()
              if rig is not None and o is not None and not what.startswith("orientation") and "output_layout" not in ov]
    cases += [(what, pair, IDENTITY, 4.0, ok_pose, ok_cam, m, {}) for what, m in _bad_minify() if m is not None]
    arrays = [np.zeros((8, 8, 2), np.float32), np.zeros((8, 8, 2), np.float32), np.zeros((8, 8), np.uint8)] + \
        [np.zeros((8, 8), np.uint16) for _ in range(3)]
    ptrs = [a.ctypes.data for a in arrays]
    P, I = C.c_void_p * 3, C.c_int * 3
    arr = lambda v: I(*([v] * 3))

    def frame(vft, rig, ph, seam, pose, cam, minify, n=1, planes=(0x20000,), dims=(64, 32, 8, 8), pitch=(64, 8)):
        return L.T360B200_transformFrameCameraPhotoAsync(
            vft._h, C.byref(rig) if rig is not None else None, C.byref(ph) if ph is not None else None, seam,
            C.byref(t360.T360Pose(*pose)) if pose is not None else None, C.byref(t360.T360Camera(*cam)) if cam is not None else None,
            C.byref(t360.T360Minify(*minify)) if minify is not None else None, 0x40000, n, P(*(list(planes) * 3)[:3]),
            P(*(list(planes) * 3)[:3]), arr(dims[0]), arr(dims[1]), arr(pitch[0]), arr(dims[2]), arr(dims[3]), arr(pitch[1]), None)
    n0 = t360.kernel_launch_count()
    assert len(cases) > 60
    for what, rig, ph, seam, pose, cam, minify, ov in cases:
        c = t360.make_context(**{**RECT_CTX, **ov})
        pb = C.byref(t360.T360Pose(*pose)) if pose is not None else None
        cb = C.byref(t360.T360Camera(*cam)) if cam is not None else None
        mb = C.byref(t360.T360Minify(*minify)) if minify is not None else None
        assert not L.T360B200_cameraPhotoMaps(C.byref(c), C.byref(rig) if rig is not None else None, C.byref(ph) if ph is not None else None,
                                              seam, pb, cb, mb, 0, 0, 64, 32, 8, 8, *ptrs), what
        assert "Could not compute the camera photometry maps" in _stdout(capfd), what
        with t360.VideoFrameTransform(c) as vft:
            assert "photometry" in _refused(capfd, frame, vft, rig, ph, seam, pose, cam, minify), what
    ctx = t360.make_context(**RECT_CTX)
    pb, cb = C.byref(t360.T360Pose(*ok_pose)), C.byref(t360.T360Camera(*ok_cam))
    for lens, plane in ((-1, 0), (2, 0), (0, -1), (0, 3)):
        _refused(capfd, L.T360B200_cameraPhotoMaps, C.byref(ctx), C.byref(pair), C.byref(IDENTITY), 0.0, pb, cb, None, lens, plane, 64, 32, 8, 8, *ptrs)
    for k in range(6):
        bad = list(ptrs)
        bad[k] = None
        _refused(capfd, L.T360B200_cameraPhotoMaps, C.byref(ctx), C.byref(pair), C.byref(IDENTITY), 0.0, pb, cb, None, 0, 0, 64, 32, 8, 8, *bad)
    _refused(capfd, L.T360B200_cameraPhotoMaps, C.byref(ctx), C.byref(pair), C.byref(IDENTITY), 0.0, pb, cb, None, 0, 0, 0, 32, 8, 8, *ptrs)
    _refused(capfd, L.T360B200_cameraPhotoMaps, None, C.byref(pair), C.byref(IDENTITY), 0.0, pb, cb, None, 0, 0, 64, 32, 8, 8, *ptrs)
    with t360.VideoFrameTransform(ctx) as vft:
        for kw in (dict(n=0), dict(n=4), dict(planes=(None,)), dict(dims=(0, 32, 8, 8)), dict(pitch=(63, 8))):
            _refused(capfd, lambda: frame(vft, pair, IDENTITY, 0.0, ok_pose, ok_cam, None, **kw))
        _refused(capfd, lambda: frame(vft, pair, IDENTITY, 0.0, ok_pose, ok_cam, (1, 0.0), dims=(131071, 32, 8, 8), pitch=(131072, 8)))
    assert not L.T360B200_transformFrameCameraPhotoAsync(None, None, None, 0.0, None, None, None, None, 1, *([None] * 9))
    assert t360.kernel_launch_count() == n0
    # accepted: a FLAT_FIXED output layout (the pose replaces it), lens 1 of a one-lens rig (all NaN), the minify limits
    single = make_rig("single_200")
    flat = t360.make_context(**RECT_CTX, output_layout=t360.LAYOUT_FLAT_FIXED)
    m0 = t360.camera_photo_maps(flat, single, IDENTITY, 0.0, ok_pose, ok_cam, None, 1, 0, 64, 32, 8, 8)[0]
    assert np.isnan(m0).all()
    for minify in ((0, -4.0), (8, 4.0)):
        t360.camera_photo_maps(ctx, pair, IDENTITY, 180.0, ok_pose, ok_cam, minify, 0, 2, 64, 32, 8, 8)


# ---- on the GPU --------------------------------------------------------------------------------------------------------
def _call(vft, f):
    return vft.make_camera_photo_frame_call(f.in_planes, f.out_planes, f.dims)


@pytest.mark.gpu
@pytest.mark.parametrize("interp", INTERPS)
@pytest.mark.parametrize("model", sorted(MODELS))
def test_frames_and_statistics_equal_the_oracle(model, interp, torch_cuda):
    """Both rigs, seams 0 and 4 degrees (two lenses), no pyramid, (3, 0) and (4, 1.0), a non-identity photometry: 3-plane
    frames equal the oracle's composite bit for bit with and without statistics (the same bytes), and the statistics equal
    its int64 sums exactly."""
    torch = torch_cuda
    ctx = _ctx("pair_190", interp)
    vft = t360.VideoFrameTransform(ctx)
    st = torch.cuda.Stream()
    stats = torch.zeros((3, STATS), dtype=torch.int64, device="cuda")
    for name in RIGS:
        rig = make_rig(name, seed=interp + len(model))
        ph = rig_photos(rig)["falloff"]
        for seam in ((0.0,) if rig.numLenses == 1 else (0.0, 4.0)):
            for k, minify in enumerate(MINIFIES):
                pose, cam = seam_pose(MODELS[model], 31 * interp + 7 * k + len(name))
                f = MipFrame(torch, name, 3, seed=interp + k)
                want, sums = photo_want(ctx, rig, ph, seam, pose, cam, minify, f.src, f.out_dims, f.prefill)
                what = f"{name} seam {seam} minify {minify} {pose}"
                for with_stats in (False, True):
                    for p, o in enumerate(f.outs):
                        o[:, :f.out_dims[p][0]] = torch.from_numpy(f.prefill[p]).cuda()
                    stats.fill_(-1)
                    torch.cuda.synchronize()
                    assert _call(vft, f)(rig, ph, seam, pose, cam, minify, st.cuda_stream, stats.data_ptr() if with_stats else 0)
                    st.synchronize()
                    for p, got in enumerate(f.host()):
                        _check(got, want[p], f"{what}, statistics {with_stats}, plane {p}")
                    got_sums = stats.cpu().numpy()
                    if with_stats:
                        for p in range(3):
                            assert got_sums[p].tolist() == sums[p], f"{what}: plane {p} statistics {got_sums[p].tolist()} != {sums[p]}"
                        assert rig.numLenses == 1 or got_sums[0][0] > 0, f"{what}: no overlap pixel"
                    else:
                        assert (got_sums == -1).all()
    vft.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", RIGS)
def test_identity_equals_the_camera_and_camera_mip_calls(name, torch_cuda):
    """The identity photometry with seamWidth 0: without a pyramid the camera call's bytes, with one the camera-mip
    call's, every model and interpolator, with statistics on; launches 1 and T_max + 1 (+ the memset, not a kernel)."""
    torch = torch_cuda
    rig = make_rig(name, seed=2)
    st = torch.cuda.Stream()
    stats = torch.zeros((3, STATS), dtype=torch.int64, device="cuda")
    for interp in INTERPS:
        vft = t360.VideoFrameTransform(_ctx(name, interp))
        for model in sorted(MODELS):
            pose, cam = seam_pose(MODELS[model], interp + len(model))
            for minify in MINIFIES:
                a, b = MipFrame(torch, name, 3, seed=interp), MipFrame(torch, name, 3, seed=interp)
                torch.cuda.synchronize()
                n0 = t360.kernel_launch_count()
                assert _call(vft, a)(rig, IDENTITY, 0.0, pose, cam, minify, st.cuda_stream, stats.data_ptr())
                n1 = t360.kernel_launch_count()
                if minify is None:
                    assert vft.make_camera_frame_call(b.in_planes, b.out_planes, b.dims)(pose, cam, st.cuda_stream, rig)
                else:
                    assert vft.make_camera_mip_frame_call(b.in_planes, b.out_planes, b.dims)(pose, cam, minify, st.cuda_stream, rig)
                top = 0 if minify is None else len(t360.mip_level_sizes(*_in_dims(name)[0], minify[0])) - 1
                assert (n1 - n0, t360.kernel_launch_count() - n1) == (top + 1, top + 1), (name, model, minify)
                st.synchronize()
                for p, (x, y) in enumerate(zip(a.host(), b.host())):
                    assert np.array_equal(x, y), (name, interp, model, minify, p)
        vft.close()


@pytest.mark.gpu
def test_trajectory_on_two_streams(torch_cuda):
    """Two streams enqueue 24 frames without synchronising, pose, camera model, photometry, seam and minify changing every
    frame, a statistics buffer each frame: every frame and its statistics equal the oracle."""
    torch = torch_cuda
    ctx = _ctx("pair_190", t360.CUBIC)
    rig = make_rig("pair_190", 61)
    rng = np.random.default_rng(21)
    args = []
    for k in range(24):
        pose, cam = seam_pose(MODELS[sorted(MODELS)[k % 4]], 500 + k)
        ph = photometry(16, [tuple(rng.uniform([-0.5, -0.1, 0], [0, 0.1, 0.01]) / r_max(rig.lens[i]) ** np.array([2, 4, 6])) for i in range(2)],
                        [tuple(rng.uniform(0.7, 1.4, 3)) for _ in range(2)], [tuple(rng.uniform(-8, 8, 3)) for _ in range(2)])
        args.append((ph, (0.0, 3.0, 4.0)[k % 3], pose, cam, (None, (2, 0.0), (5, -0.5), (8, 1.0))[k % 4]))
    vft = t360.VideoFrameTransform(ctx)
    frames = [MipFrame(torch, "pair_190", 3, seed=k % 4) for k in range(24)]
    stats = torch.zeros((24, 3, STATS), dtype=torch.int64, device="cuda")
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for k, (f, (ph, seam, pose, cam, minify)) in enumerate(zip(frames, args)):
        assert _call(vft, f)(rig, ph, seam, pose, cam, minify, streams[k % 2].cuda_stream, stats[k].data_ptr())
    torch.cuda.synchronize()
    got_stats = stats.cpu().numpy()
    for k, (f, (ph, seam, pose, cam, minify)) in enumerate(zip(frames, args)):
        want, sums = photo_want(ctx, rig, ph, seam, pose, cam, minify, f.src, f.out_dims, f.prefill)
        for p, got in enumerate(f.host()):
            _check(got, want[p], f"frame {k}, plane {p}")
            assert got_stats[k, p].tolist() == sums[p], f"frame {k}, plane {p} statistics"
    vft.close()


@pytest.mark.gpu
def test_device_memory_and_launches_stay_bounded(torch_cuda):
    """60 frames after a warm-up, seam, minify and statistics changing: T_max + 1 launches each (1 without a pyramid) and
    no growth of device memory."""
    torch = torch_cuda
    ctx = _ctx("pair_190", t360.LANCZOS4)
    rig = make_rig("pair_190", 91)
    vft = t360.VideoFrameTransform(ctx)
    f = MipFrame(torch, "pair_190", 3)
    call = _call(vft, f)
    stats = torch.zeros((3, STATS), dtype=torch.int64, device="cuda")
    st = torch.cuda.Stream()
    ph = rig_photos(rig)["falloff"]
    minifies = [None, (3, 0.0), (8, 0.5)]
    tops = [0 if m is None else len(t360.mip_level_sizes(*_in_dims("pair_190")[0], m[0])) - 1 for m in minifies]

    def frame(i):
        return call(rig, ph, 4.0 * (i % 2), (90.0 + 3 * i, 1.0, 0.0, 150.0, 120.0), (EQUIDISTANT, 0.0), minifies[i % 3], st.cuda_stream,
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
    ctx = _ctx("pair_190")
    vft = t360.VideoFrameTransform(ctx)
    f = MipFrame(torch, "pair_190", 3)
    stats = torch.full((3, STATS), 5, dtype=torch.int64, device="cuda")
    before = f.host()
    call = _call(vft, f)
    pair, single = make_rig("pair_190"), make_rig("single_200")
    ok = (90.0, 0.0, 0.0, 90.0, 60.0)
    torch.cuda.synchronize()
    n0 = t360.kernel_launch_count()
    for rig, ph, seam, pose, cam, minify in ((single, IDENTITY, 4.0, ok, PINHOLE, None), (pair, IDENTITY, 0.005, ok, PINHOLE, None),
                                             (pair, photometry(gain=((0, 1, 1), (1, 1, 1))), 0.0, ok, PINHOLE, None),
                                             (pair, IDENTITY, 0.0, (0.0, 0.0, 0.0, 200.0, 60.0), PINHOLE, None),
                                             (pair, IDENTITY, 0.0, ok, PINHOLE, (9, 0.0))):
        _refused(capfd, call, rig, ph, seam, pose, cam, minify, 0, stats.data_ptr())
    torch.cuda.synchronize()
    assert t360.kernel_launch_count() == n0
    assert all(np.array_equal(a, b) for a, b in zip(before, f.host()))
    assert (stats.cpu().numpy() == 5).all()
    vft.close()


# ---- the twin gate (tests/camera_photo_twin_gate.cu on tests/twin_gate.cuh) --------------------------------------------
GATE_PROBES = ("lensJacobian<lens>", "cameraPhotoPoint", "cameraPhotoSample<MIP>", "cameraPhotoSample<plain>")


@pytest.fixture(scope="module")
def photo_gate(tmp_path_factory):
    """(name, executable) of the camera photometry gate, built once with the library's nvcc flags."""
    from tests.test_twin_gates import gate_command
    exe = tmp_path_factory.mktemp("camera_photo_twin_gate") / "camera_photo_twin_gate"
    r = subprocess.run(gate_command("camera_photo_twin_gate", exe), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return "camera_photo_twin_gate", exe


def test_gate_builds_for_sm_90a_with_the_library_flags(photo_gate):
    from tests.test_twin_gates import test_gate_builds_for_sm_90a_with_the_library_flags as check
    check(photo_gate)


def test_gate_host_half_does_not_depend_on_the_thread_count(photo_gate):
    from tests.test_twin_gates import THREADS, _fingerprints, run
    one = _fingerprints(run(photo_gate, "--host-only", "--threads", "1").stdout)
    many = _fingerprints(run(photo_gate, "--host-only", "--threads", str(THREADS)).stdout)
    assert [line.split()[1] for line in one] == list(GATE_PROBES), one
    assert one == many


def test_gate_self_test_reports_exactly_the_flipped_element(photo_gate):
    import re
    from tests.test_twin_gates import THREADS, run
    r = run(photo_gate, "--self-test", "--threads", str(THREADS), check=False)
    assert r.returncode == 1, r.stdout + r.stderr
    flipped = re.search(r"self-test: flipped (\S+) (\d+) word (\d+) bit (\d+)", r.stdout)
    assert flipped, r.stdout
    probe, index, word, bit = flipped.group(1), int(flipped.group(2)), int(flipped.group(3)), int(flipped.group(4))
    reports = [line.split() for line in r.stdout.splitlines() if len(line.split()) == 5 and not line.startswith("self-test")]
    assert len(reports) == 1, r.stdout
    name, at, _, host, other = reports[0]
    assert (name, int(at)) == (probe, index)
    h, o = [int(x, 16) for x in host.split(":")], [int(x, 16) for x in other.split(":")]
    assert [x ^ y for x, y in zip(h, o)] == [(1 << bit) if k == word else 0 for k in range(11)]
    assert r.stdout.strip().splitlines()[-1].endswith(" 1 mismatches"), r.stdout


def test_gate_ledger_reaches_every_class(photo_gate):
    """Rays on a used lens's axis, a lens's thetaMax, belt pixels and the infinite footprint of a used lens's back axis are
    all reached by the first 2^20 inputs of cameraPhotoPoint."""
    from tests.test_twin_gates import THREADS, run
    counts = {}
    for line in run(photo_gate, "--ledger", "--threads", str(THREADS)).stdout.splitlines():
        _, probe, cls, n = line.split()
        counts[(probe, cls)] = int(n)
    print(counts)
    assert sorted(counts) == [("cameraPhotoPoint", c) for c in sorted(("belt", "infiniteFootprint", "lensAxis", "thetaMax"))], counts
    assert all(n >= 100 for n in counts.values()), counts


@pytest.mark.gpu
def test_gate_device_twins_equal_the_host_twins(photo_gate):
    import re
    from tests.test_twin_gates import THREADS, run
    r = run(photo_gate, "--threads", str(THREADS), check=False)
    print(r.stdout)
    last = r.stdout.strip().splitlines()[-1]
    m = re.fullmatch(r"(\d+) probes, (\d+) inputs, (\d+) mismatches", last)
    assert m and r.returncode == 0 and m.group(3) == "0", r.stdout + r.stderr
