"""Anisotropic camera views: N pyramid probes along each pixel's longer footprint axis (T360B200_cameraAnisoMaps /
camera_aniso_maps, T360B200_transformFrameCameraAnisoAsync / make_camera_aniso_frame_call).

What pins what:
  - maxProbes 1 against camera_mip_maps bit for bit (so against camera_map where nothing is minified);
  - the level, the probe count and each probe's entry against a float64 model of the header's steps 1-2 (both footprint
    axes, the bit rule, the probe's offset ray looked up in float64);
  - that it anti-aliases better than the isotropic pyramid: the zone plate of test_camera_mip.py through a little planet
    and a dome;
  - the refusals and their order;
  - the twin gate (tests/aniso_twin_gate.cu): the device build of anisoLevelOf, anisoFootprint, anisoCameraPoint and
    anisoCameraSample against the host build the twin runs;
  - on the GPU, frames against the oracle's composite of the twin (cv::resize INTER_AREA pyramids, cv::remap per probe
    and level, the level blend, the probe mean), and against the camera-mip and camera calls where they must agree.
Poses, rigs and planes are made from seeds."""
import ctypes as C
import math
import re
import subprocess

import numpy as np
import pytest

import transform360_b200 as t360
from oracle import c_oracle as co
from transform360_b200.handler import as_minify
from tests.test_camera_mip import (MIP_INPUTS, MipFrame, _bad_minify, _in_dims, _ideal, _lens_pixels, _rotation, bit_rule, mip_want, pixel_xy,
                                   pyramid, same_bits, wide_pose)
from tests.test_camera_mip import rays64 as _rays64
from tests.test_camera_mip import zone  # noqa: F401 (fixture)
from tests.test_camera_models import EQUIDISTANT, PANNINI, PINHOLE, STEREOGRAPHIC, _bad_calls
from tests.test_rectilinear import INTERPS, RECT_CTX, _ctx, _rig
from tests.test_rectilinear import torch_cuda  # noqa: F401 (fixture)
from tests.test_twin_gates import THREADS, gate_command, run
from tests.test_warp_map import _check, _refused, _stdout

WRAP, TRANSPARENT = t360.BORDER_WRAP, t360.BORDER_TRANSPARENT
EQUIRECT = t360.T360_CAMERA_EQUIRECT
MODELS = {"pinhole": PINHOLE, "equidistant": EQUIDISTANT, "stereographic": STEREOGRAPHIC, "pannini": PANNINI, "equirect": EQUIRECT}


def aniso_pose(model, seed):
    """wide_pose of test_camera_mip.py, and for the equirect model a latitude / longitude window of 90-360 x 60-180."""
    if model != EQUIRECT:
        return wide_pose(model, seed)
    rng = np.random.default_rng(seed)
    ang = (float(rng.uniform(-180, 180)), float(rng.uniform(-80, 80)), float(rng.uniform(-180, 180)))
    return (*ang, float(rng.uniform(90, 360)), float(rng.uniform(60, 180))), (EQUIRECT, 0.0)


def rays64(pose, camera, X, Y):
    """test_camera_mip.rays64 with the equirect model: q = (cos lat sin lon, sin lat, cos lat cos lon), lon = X ax, lat = Y ay
    with the library's float32 constants."""
    if camera[0] != EQUIRECT:
        return _rays64(pose, camera, X, Y)
    lon, lat = X * np.float64(np.float32(math.radians(pose[3]) / 2)), Y * np.float64(np.float32(math.radians(pose[4]) / 2))
    q = np.stack([np.cos(lat) * np.sin(lon), np.sin(lat), np.cos(lat) * np.cos(lon)], -1)
    return np.stack([q[..., 0] * r[0] - q[..., 1] * r[1] + q[..., 2] * r[2] for r in _rotation(pose)], -1) * np.array([1.0, -1.0, 1.0])


# ---- the oracle's composite --------------------------------------------------------------------------------------------
def _remap_sel(src, m, sel, interp, prefill):
    """cv::remap of the entries m where sel (value, skipped): BORDER_WRAP with prefill None, else BORDER_TRANSPARENT into
    prefill, skipped where it keeps the pre-fill."""
    mm = np.where(sel[..., None], m, np.float32(0)).astype(np.float32)
    if prefill is None:
        return co.remap_u8(src, mm, interp, WRAP).astype(np.int32), np.zeros(sel.shape, bool)
    val = co.remap_u8(src, mm, interp, TRANSPARENT, prefill.copy()).astype(np.int32)
    return val, co.remap_u8(np.zeros_like(src), mm, interp, TRANSPARENT, prefill.copy()) != 0


def aniso_composite(levels, m0, m1, lv, w, probes, interp, prefill=None):
    """Step 3 of the header from the twin's arrays: each probe's two levels by cv::remap, blended as (a (256 - w) + b w +
    128) >> 8 with a skipped sample leaving the other alone; then the mean (sum + n / 2) // n over the probes that are not
    skipped (all N under BORDER_WRAP), the pre-fill where every probe is skipped."""
    shape, wi = lv.shape, w.astype(np.int32)
    total, count = np.zeros(shape, np.int64), np.zeros(shape, np.int64)
    for k in range(m0.shape[0]):
        live = probes > k
        a, b = np.zeros(shape, np.int32), np.zeros(shape, np.int32)
        skip_a, skip_b = np.ones(shape, bool), np.ones(shape, bool)
        for level, src in enumerate(levels):
            for sel, m, val, skip in ((live & (lv == level), m0[k], a, skip_a), (live & (lv + 1 == level) & (wi > 0), m1[k], b, skip_b)):
                if sel.any():
                    v, s = _remap_sel(src, m, sel, interp, prefill)
                    val[sel], skip[sel] = v[sel], s[sel]
        blend = (a * (256 - wi) + b * wi + 128) >> 8
        two = wi > 0
        v = np.where(two, np.where(skip_a, b, np.where(skip_b, a, blend)), a)
        ok = live & ~(skip_a & (skip_b | ~two))
        total += np.where(ok, v, 0)
        count += ok
    out = (total + count // 2) // np.maximum(count, 1)
    if prefill is not None:
        out = np.where(count == 0, prefill, out)
    return out.astype(np.uint8)


def aniso_want(ctx, rig, pose, cam, minify, max_probes, srcs, out_dims, prefills=None):
    """The oracle composite of every plane of a frame: planes 1 and 2 share the twin's arrays."""
    out, twins = [], {}
    for p, src in enumerate(srcs):
        key = (src.shape, out_dims[p])
        if key not in twins:
            twins[key] = t360.camera_aniso_maps(ctx, pose, cam, minify, max_probes, src.shape[1], src.shape[0], *out_dims[p], rig)
        m0, m1, lv, w, n = twins[key]
        levels = pyramid(src, as_minify(minify).maxLevel)
        out.append(aniso_composite(levels, m0, m1, lv, w, n, ctx.interpolation_alg, None if prefills is None else prefills[p]))
    return out


# ---- the float64 model -------------------------------------------------------------------------------------------------
def axes64(ctx, rig, pose, camera, in_w, in_h, w, h):
    """(aa, bb, unsure): the header's a.a and b.b in float64 (test_camera_mip.footprint64's footprint, both axes kept), and
    the pixels where the float32 chain may pick another chart or is ill-conditioned."""
    X, Y, hx, hy = pixel_xy(ctx, w, h, mono=rig is not None)
    t = rays64(pose, camera, X, Y)
    rs = (rays64(pose, camera, X + hx, Y) - rays64(pose, camera, X - hx, Y), rays64(pose, camera, X, Y + hy) - rays64(pose, camera, X, Y - hy))
    unsure = np.zeros((h, w), bool)
    if rig is not None:
        n = np.linalg.norm(t, axis=-1, keepdims=True)
        _, _, tie = _lens_pixels(rig, t / n, in_w, in_h)
        outs = []
        for r in rs:
            eps = 1e-6 * n / np.linalg.norm(r, axis=-1, keepdims=True)
            p1, p0 = _lens_pixels(rig, (t + eps * r) / n, in_w, in_h), _lens_pixels(rig, (t - eps * r) / n, in_w, in_h)
            outs.append(((p1[0] - p0[0]) / (2 * eps[..., 0])) ** 2 + ((p1[1] - p0[1]) / (2 * eps[..., 0])) ** 2)
        return outs[0], outs[1], unsure | (tie < 1e-4 * n[..., 0])
    x, y, z = t[..., 0], t[..., 1], t[..., 2]
    if ctx.input_layout == t360.LAYOUT_CUBEMAP_32:
        e = np.float64(np.float32(ctx.input_expand_coef))
        d = t / np.linalg.norm(t, axis=-1, keepdims=True)
        ax = [np.full((h, w), np.nan), np.full((h, w), np.nan)]
        for mj, ai, bi, neg in [(2, 0, 1, True), (2, 0, 1, False), (0, 2, 1, True), (0, 2, 1, False), (1, 0, 2, True), (1, 0, 2, False)]:
            m = d[..., mj]
            ok = (m <= -0.5) if neg else (m >= 0.5)
            gx, gy = d[..., ai] / m, d[..., bi] / m
            unsure |= ok & ((np.abs(np.abs(gx) - 1) < 1e-4) | (np.abs(np.abs(gy) - 1) < 1e-4))
            win = ok & (np.abs(gx) <= 1) & (np.abs(gy) <= 1) & np.isnan(ax[0])
            for k, r in enumerate(rs):
                tm, ta, tb = t[..., mj], t[..., ai], t[..., bi]
                du = in_w / (6 * e) * (r[..., ai] * tm - ta * r[..., mj]) / tm ** 2
                dv = in_h / (4 * e) * (r[..., bi] * tm - tb * r[..., mj]) / tm ** 2
                ax[k] = np.where(win, du * du + dv * dv, ax[k])
        return ax[0], ax[1], unsure
    su = in_w / (2 * np.pi) / (2 if ctx.input_stereo_format == t360.STEREO_FORMAT_LR else 1)
    sv = in_h / np.pi / (2 if ctx.input_stereo_format == t360.STEREO_FORMAT_TB else 1)
    h2, r2 = x * x + z * z, x * x + y * y + z * z
    ax = []
    for r in rs:
        du = su * (z * r[..., 0] - x * r[..., 2]) / h2
        dv = sv * (r[..., 1] * h2 - y * (x * r[..., 0] + z * r[..., 2])) / (r2 * np.sqrt(h2))
        ax.append(du * du + dv * dv)
    return ax[0], ax[1], unsure | (np.sqrt(h2) < 1e-3 * np.sqrt(r2))


def model_lod(aa, bb, top, bias, max_log2):
    """(lambda256 before the clamp, e) of the header's step 1 from float64 aa, bb (each rounded to float32 first)."""
    hi, lo = bit_rule(np.maximum(aa, bb)), bit_rule(np.minimum(aa, bb))
    e = np.minimum((hi - lo + 255) >> 8, max_log2)
    return np.maximum(hi - 256 * e, lo) + int(math.floor(abs(256 * bias) + 0.5)) * (1 if bias >= 0 else -1), e, hi - lo


def check_model(ctx, rig, pose, cam, in_w, in_h, w, h, max_probes, max_level=8, bias=0.0, what=""):
    """The twin's lambda256 within 2/256 of the model where it is not clamped, its N equal to the model's where lambda_maj -
    lambda_min is not within 2 of a multiple of 256, away from chart edges and poles; returns the pixels compared."""
    m0, _, lv, wt, n = t360.camera_aniso_maps(ctx, pose, cam, (max_level, bias), max_probes, in_w, in_h, w, h, rig)
    top = len(t360.mip_level_sizes(in_w, in_h, max_level)) - 1
    aa, bb, unsure = axes64(ctx, rig, pose, cam, in_w, in_h, w, h)
    with np.errstate(all="ignore"):
        finite = np.isfinite(aa) & np.isfinite(bb)
        lam, e, spread = model_lod(np.where(finite, aa, 1.0), np.where(finite, bb, 1.0), top, bias, int(math.log2(max_probes)))
    free = finite & ~unsure
    if rig is not None:
        free &= ~np.isnan(m0[0][..., 0])
    got = lv.astype(np.int64) * 256 + wt
    inner = free & (got > 0) & (got < 256 * top)
    diff = np.abs(got - lam)[inner]
    assert diff.size == 0 or diff.max() <= 2, f"{what}: lambda256 off the model by {diff.max()} at {int((diff > 2).sum())} px"
    r = spread % 256
    clear = free & (spread > 2) & (r > 2) & (r < 254)
    clear |= free & (spread == 0) & (np.abs(aa - bb) <= 1e-9 * aa)
    bad = clear & (n != (1 << e))
    assert not bad.any(), f"{what}: N off the model at {int(bad.sum())} px"
    return int(inner.sum()), int(clear.sum())


def entries64(ctx, rig, pose, cam, in_w, in_h, w, h, n, rows, k):
    """Probe k's level-0 entry (px, py) in float64 for pixels with N = n on the given axis: the offset ray looked up in the
    mono equirect, or in a rig's closer lens."""
    X, Y, hx, hy = pixel_xy(ctx, w, h, mono=rig is not None)
    o = (2 * k + 1 - n) / n
    t = rays64(pose, cam, np.where(rows, X, X + o * hx), np.where(rows, Y + o * hy, Y))
    if rig is not None:
        px, py, _ = _lens_pixels(rig, t / np.linalg.norm(t, axis=-1, keepdims=True), in_w, in_h)
        return px, py
    r = np.linalg.norm(t, axis=-1)
    return (0.5 + np.arctan2(t[..., 0], t[..., 2]) / (2 * np.pi)) * in_w - 0.5, (0.5 - np.arcsin(t[..., 1] / r) / np.pi) * in_h - 0.5


# ---- no GPU needed -----------------------------------------------------------------------------------------------------
def test_entry_points_are_exported_with_their_bindings():
    from transform360_b200.handler import EXPORTED_SYMBOLS, LIB_PATH
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    L = t360.load()
    for name in ("T360B200_cameraAnisoMaps", "T360B200_transformFrameCameraAnisoAsync"):
        assert name in EXPORTED_SYMBOLS and name in defined, name
    P = C.POINTER
    assert L.T360B200_cameraAnisoMaps.argtypes == [P(t360.FrameTransformContext), P(t360.T360LensRig), P(t360.T360Pose), P(t360.T360Camera),
                                                   P(t360.T360Minify)] + [C.c_int] * 5 + [C.c_void_p] * 5
    assert L.T360B200_transformFrameCameraAnisoAsync.argtypes == [C.c_void_p, P(t360.T360LensRig), P(t360.T360Pose), P(t360.T360Camera),
                                                                  P(t360.T360Minify), C.c_int, C.c_int] + [C.c_void_p] * 9
    assert hasattr(t360.VideoFrameTransform, "make_camera_aniso_frame_call") and callable(t360.camera_aniso_maps)


@pytest.mark.parametrize("name", MIP_INPUTS)
@pytest.mark.parametrize("model", sorted(MODELS))
def test_one_probe_is_the_camera_mip_maps(model, name):
    """maxProbes 1: probe 0 is camera_mip_maps' four arrays bit for bit and N = 1 everywhere, for several maxLevel and
    lodBias, maxLevel 0 (the camera map) included."""
    ctx, rig = _ctx(name), _rig(name, seed=3)
    (in_w, in_h), _ = _in_dims(name)
    for k, minify in enumerate(((8, 0.0), (4, -1.0), (1, 1.5), (0, 0.5))):
        pose, cam = aniso_pose(MODELS[model], 100 * k + len(name))
        m0, m1, lv, wt, n = t360.camera_aniso_maps(ctx, pose, cam, minify, 1, in_w, in_h, 97, 65, rig)
        w0, w1, wl, ww = t360.camera_mip_maps(ctx, pose, cam, minify, in_w, in_h, 97, 65, rig)
        assert m0.shape == (1, 65, 97, 2) and same_bits(m0[0], w0) and same_bits(m1[0], w1), (minify, pose)
        assert np.array_equal(lv, wl) and np.array_equal(wt, ww) and (n == 1).all(), (minify, pose)


CASES = [(name, model) for name in MIP_INPUTS for model in sorted(MODELS)]


@pytest.mark.parametrize("name,model", CASES)
def test_level_and_probe_count_against_the_float64_model(name, model):
    """lambda256 within 2/256 level of the float64 footprint through the header's rule, and N the model's wherever
    lambda_maj - lambda_min is not within 2 of a multiple of 256, for every model, input and output eye split."""
    ctx, rig = _ctx(name), _rig(name, seed=5)
    (in_w, in_h), _ = _in_dims(name)
    inner = clear = 0
    for k in range(3):
        pose, cam = aniso_pose(MODELS[model], 7 * k + len(name) + 1000)
        a, b = check_model(ctx, rig, pose, cam, in_w, in_h, 97, 65, (16, 4, 2)[k], max_level=(8, 8, 0)[k], bias=(0.0, -1.0, 1.5)[k],
                           what=f"{name} {model} {pose}")
        inner, clear = inner + a, clear + b
    assert clear > 1000 and (inner > 500 or rig is not None), (inner, clear)


@pytest.mark.parametrize("name", ["equirect", "single_200", "pair_190"])
def test_probe_entries_against_the_float64_lookup(name):
    """Each probe's level-0 entry within 1e-3 px of the float64 lookup of its offset ray (away from the equirect's seam
    and poles, and from a rig's lens tie); the probes beyond N are NaN."""
    ctx, rig = _ctx(name), _rig(name, seed=9)
    (in_w, in_h), _ = _in_dims(name)
    checked = 0
    for k in range(4):
        pose, cam = aniso_pose(sorted(MODELS.values())[k + 1], 40 + k)
        m0, m1, lv, wt, n = t360.camera_aniso_maps(ctx, pose, cam, (0, 0.0), 16, in_w, in_h, 97, 65, rig)
        aa, bb, unsure = axes64(ctx, rig, pose, cam, in_w, in_h, 97, 65)
        rows = ~(aa >= bb)
        for p in range(16):
            assert np.isnan(m0[p][n <= p]).all() and np.isnan(m1[p]).all()
            px, py = entries64(ctx, rig, pose, cam, in_w, in_h, 97, 65, n.astype(np.int64), rows, p)
            sel = (n > p) & ~unsure & np.isfinite(m0[p][..., 0]) & np.isfinite(px)
            dx = np.abs(m0[p][..., 0] - px)
            if rig is None:  # (the seam, and 16 rows at the poles, where longitude is ill-conditioned in float)
                sel &= (px > 2) & (px < in_w - 3) & (py > 16) & (py < in_h - 17)
            err = np.maximum(dx, np.abs(m0[p][..., 1] - py))[sel]
            assert err.size == 0 or err.max() <= 1e-3, (name, pose, p, err.max())
            checked += int(sel.sum())
    assert checked > 20000, checked


def test_a_round_footprint_takes_one_probe():
    """A narrow pinhole at the equator of a 2:1 equirect has square footprints: N = 1 wherever the two axes' lambda256
    agree, and at most 2 elsewhere (a 1/256 level apart).  At the zenith the pixel is at the top level with weight 0,
    however many probes its footprint takes."""
    ctx = _ctx("equirect")
    _, _, lv, wt, n = t360.camera_aniso_maps(ctx, (0.0, 0.0, 0.0, 1.0, 1.0), PINHOLE, (8, 0.0), 16, 4096, 2048, 65, 65)
    assert n.max() <= 2 and (n == 1).mean() > 0.5 and n[32, 32] == 1, np.bincount(n.ravel())
    _, _, lv, wt, n = t360.camera_aniso_maps(ctx, (0.0, 90.0, 0.0, 60.0, 60.0), PINHOLE, (8, 0.0), 16, 4096, 2048, 65, 65)
    assert lv[32, 32] == len(t360.mip_level_sizes(4096, 2048, 8)) - 1 and wt[32, 32] == 0


# The bound on the RMS error against the ideal render, as a fraction of the point-sampled view's, set from the first run:
# at lodBias 0 the isotropic pyramid has ratio 0.659 for the little planet and 0.302 for the dome, 16 probes 0.419 and
# 0.268.  The little planet's outer ring, where the isotropic footprint over-blurs across the zenith's horizontal stretch,
# gains most; the dome must be no worse than the isotropic pyramid.
AA_BOUNDS = {"little_planet": 0.5, "dome": None}


@pytest.mark.parametrize("view,pose,cam", [("dome", (0.0, 0.0, 0.0, 180.0, 180.0), EQUIDISTANT),
                                           ("little_planet", (0.0, -90.0, 0.0, 300.0, 300.0), STEREOGRAPHIC)], ids=["dome", "little_planet"])
def test_it_anti_aliases_better_than_the_isotropic_pyramid(view, pose, cam, zone):  # noqa: F811 (fixture)
    """The zone plate of test_camera_mip.test_it_anti_aliases through a 256^2 view at lodBias 0: with maxProbes 16 the
    little planet's RMS error against the ideal render is clearly below the isotropic pyramid's, and the dome's is no
    worse."""
    ctx = _ctx("equirect", t360.CUBIC)
    ideal = _ideal(pose, cam, 256, 256)
    plain = co.remap_u8(zone, t360.camera_map(ctx, pose, cam, 4096, 2048, 256, 256), t360.CUBIC, WRAP)
    e_plain = np.sqrt(np.mean((plain - ideal) ** 2))
    e_mip = np.sqrt(np.mean((mip_want(ctx, None, pose, cam, (8, 0.0), [zone], [(256, 256)])[0] - ideal) ** 2))
    e_aniso = np.sqrt(np.mean((aniso_want(ctx, None, pose, cam, (8, 0.0), 16, [zone], [(256, 256)])[0] - ideal) ** 2))
    print(f"{view}: RMS error point-sampled {e_plain:.2f}, isotropic {e_mip:.2f} ({e_mip / e_plain:.3f}), "
          f"16 probes {e_aniso:.2f} ({e_aniso / e_plain:.3f})")
    assert e_aniso <= e_mip * 1.001, (e_aniso, e_mip)
    if AA_BOUNDS[view] is not None:
        assert e_aniso <= AA_BOUNDS[view] * e_plain, (e_aniso, e_plain)


def _frame_call(L, vft, rig, pose, camera, minify, max_probes, n=1, planes=(0x20000,), dims=(64, 32, 8, 8), pitch=(64, 8)):
    P, I = C.c_void_p * 3, C.c_int * 3
    arr = lambda v: I(*([v] * 3))
    mb = C.byref(t360.T360Minify(*minify)) if minify is not None else None
    pb = C.byref(t360.T360Pose(*pose)) if pose is not None else None
    cb = C.byref(t360.T360Camera(*camera)) if camera is not None else None
    return L.T360B200_transformFrameCameraAnisoAsync(vft._h, C.byref(rig) if rig is not None else None, pb, cb, mb, max_probes, n,
                                                     P(*(list(planes) * 3)[:3]), P(*(list(planes) * 3)[:3]), arr(dims[0]), arr(dims[1]),
                                                     arr(pitch[0]), arr(dims[2]), arr(dims[3]), arr(pitch[1]), None)


def test_refusals_happen_without_a_gpu(capfd):
    """Every refusal of the camera-mip call, then maxProbes 0, 3, 32 and -1, come with a message and before any CUDA call,
    with bogus plane pointers that are never dereferenced and no kernel launched; a bad maxProbes never hides an earlier
    refusal; every allowed maxProbes is accepted."""
    L = t360.load()
    ctx = t360.make_context(**RECT_CTX)
    arrays = [np.zeros((16, 8, 8, 2), np.float32), np.zeros((16, 8, 8, 2), np.float32), np.zeros((8, 8), np.uint8), np.zeros((8, 8), np.uint16),
              np.zeros((8, 8), np.uint8)]
    ptrs = [a.ctypes.data for a in arrays]
    n0 = t360.kernel_launch_count()
    ok_pose, ok_cam = (10.0, 5.0, 0.0, 90.0, 60.0), (STEREOGRAPHIC, 0.0)
    cases = [(what, None, ok_pose, ok_cam, m, 4, {}) for what, m in _bad_minify()]
    cases += [(what, rig, pose, cam, (4, 0.0), 4, ov) for what, rig, pose, cam, ov in _bad_calls()]
    # the same refusals with a bad maxProbes too: the earlier rung's message wins
    cases += [(what + " (and maxProbes 3)", rig, pose, cam, m, 3, ov) for what, rig, pose, cam, m, _, ov in list(cases)]
    cases += [(f"maxProbes {k}", None, ok_pose, ok_cam, (4, 0.0), k, {}) for k in (0, 3, 32, -1)]
    for what, rig, pose, cam, minify, probes, ov in cases:
        c = t360.make_context(**{**RECT_CTX, **ov})
        mb = C.byref(t360.T360Minify(*minify)) if minify is not None else None
        pb = C.byref(t360.T360Pose(*pose)) if pose is not None else None
        cb = C.byref(t360.T360Camera(*cam)) if cam is not None else None
        rb = C.byref(rig) if rig is not None else None
        assert not L.T360B200_cameraAnisoMaps(C.byref(c), rb, pb, cb, mb, probes, 64, 32, 8, 8, *ptrs), what
        out = _stdout(capfd)
        assert "Could not compute the camera aniso maps" in out, what
        assert ("maxProbes" in out) == what.startswith("maxProbes"), (what, out)
        assert not L.T360B200_cameraMipMaps(C.byref(c), rb, pb, cb, mb, 64, 32, 8, 8, *ptrs[:4]) or what.startswith("maxProbes"), what
        mip_out = _stdout(capfd)
        if not what.startswith("maxProbes"):  # the camera-mip twin's message, word for word
            assert out.split("Error: ", 1)[1] == mip_out.split("Error: ", 1)[1], (what, out, mip_out)
        with t360.VideoFrameTransform(c) as vft:
            frame = _refused(capfd, _frame_call, L, vft, rig, pose, cam, minify, probes)
            assert "anisotropic camera view" in frame and ("maxProbes" in frame) == what.startswith("maxProbes"), (what, frame)
    mb = C.byref(t360.T360Minify(4, 0.0))
    pb, cb = C.byref(t360.T360Pose(*ok_pose)), C.byref(t360.T360Camera(*ok_cam))
    for args in ((64, 32, 0, 8, *ptrs), (64, 0, 8, 8, *ptrs), (64, 32, 8, 8, None, *ptrs[1:]), (64, 32, 8, 8, *ptrs[:4], None)):
        _refused(capfd, L.T360B200_cameraAnisoMaps, C.byref(ctx), None, pb, cb, mb, 16, *args)
    _refused(capfd, L.T360B200_cameraAnisoMaps, None, None, pb, cb, mb, 16, 64, 32, 8, 8, *ptrs)
    with t360.VideoFrameTransform(ctx) as vft:
        for kw in (dict(n=0), dict(n=4), dict(planes=(None,)), dict(dims=(0, 32, 8, 8)), dict(pitch=(63, 8))):
            _refused(capfd, lambda: _frame_call(L, vft, None, ok_pose, ok_cam, (4, 0.0), 16, **kw))
    assert not L.T360B200_transformFrameCameraAnisoAsync(None, None, None, None, None, 16, 1, *([None] * 9))
    assert t360.kernel_launch_count() == n0
    for probes in (1, 2, 4, 8, 16):
        t360.camera_aniso_maps(ctx, ok_pose, ok_cam, (0, -4.0), probes, 64, 32, 8, 8)
    with pytest.raises(ValueError):
        t360.camera_aniso_maps(ctx, ok_pose, ok_cam, (4, 0.0), 5, 64, 32, 8, 8)


# ---- the twin gate (tests/aniso_twin_gate.cu on tests/twin_gate.cuh) ---------------------------------------------------
GATE_PROBES = ("anisoLevelOf", "anisoFootprint<ctx>", "anisoFootprint<lens>", "anisoCameraPoint<ctx>", "anisoCameraPoint<lens>",
               "anisoCameraSample<ctx>", "anisoCameraSample<lens>")
GATE_CLASSES = {("anisoLevelOf", c) for c in ("equal", "multipleOf256", "zero", "denormal", "infNaN", "clamped")} | \
    {(p, c) for p in ("anisoFootprint<ctx>", "anisoFootprint<lens>") for c in ("columnAxis", "rowAxis")} | \
    {(f"anisoCamera{k}<ctx>", "faceChange") for k in ("Point", "Sample")} | {(f"anisoCamera{k}<lens>", "lensChange") for k in ("Point", "Sample")}


@pytest.fixture(scope="module")
def aniso_gate(tmp_path_factory):
    exe = tmp_path_factory.mktemp("aniso_twin_gate") / "aniso_twin_gate"
    r = subprocess.run(gate_command("aniso_twin_gate", exe), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return "aniso_twin_gate", exe


def test_gate_builds_for_sm_90a_with_the_library_flags(aniso_gate):
    import os
    from transform360_b200 import build as b
    cmd = gate_command(*aniso_gate)
    assert cmd[cmd.index("-Xcompiler") + 1] == b.HOST_FLAGS and "arch=compute_90a,code=sm_90a" in cmd and "-O3" in cmd
    elf = subprocess.run([os.path.join(os.path.dirname(b.nvcc_path()), "cuobjdump"), "--list-elf", str(aniso_gate[1])], capture_output=True,
                         text=True, check=True).stdout
    assert "sm_90a" in elf


def test_gate_host_half_does_not_depend_on_the_thread_count(aniso_gate):
    fp = lambda out: [line for line in out.splitlines() if line.startswith("fingerprint ")]
    one = fp(run(aniso_gate, "--host-only", "--threads", "1").stdout)
    many = fp(run(aniso_gate, "--host-only", "--threads", str(THREADS)).stdout)
    assert [line.split()[1] for line in one] == list(GATE_PROBES) and one == many


def test_gate_self_test_reports_exactly_the_flipped_element(aniso_gate):
    r = run(aniso_gate, "--self-test", "--threads", str(THREADS), check=False)
    assert r.returncode == 1, r.stdout + r.stderr
    flipped = re.search(r"self-test: flipped (\S+) (\d+) word (\d) bit (\d)", r.stdout)
    assert flipped, r.stdout
    reports = [line.split() for line in r.stdout.splitlines() if len(line.split()) == 5 and not line.startswith("self-test")]
    assert len(reports) == 1 and (reports[0][0], int(reports[0][1])) == (flipped.group(1), int(flipped.group(2))), r.stdout
    h, o = [int(x, 16) for x in reports[0][3].split(":")], [int(x, 16) for x in reports[0][4].split(":")]
    word, bit = int(flipped.group(3)), int(flipped.group(4))
    assert [x ^ y for x, y in zip(h, o)] == [(1 << bit) if k == word else 0 for k in range(len(h))]
    assert r.stdout.strip().splitlines()[-1].endswith(" 1 mismatches"), r.stdout


def test_gate_ledger_reaches_every_class(aniso_gate):
    """anisoLevelOf reaches aa == bb, an exact multiple of 256 between the axes, a zero and a denormal axis, a pole (inf
    or NaN) and N clamped by maxProbes; the footprints take both axes; a probe row crosses a cube face edge and a
    two-lens rig's seam."""
    counts = {}
    for line in run(aniso_gate, "--ledger", "--threads", str(THREADS)).stdout.splitlines():
        _, probe, cls, n = line.split()
        counts[(probe, cls)] = int(n)
    missed = sorted(k for k, n in counts.items() if n == 0)
    assert not missed, missed
    assert GATE_CLASSES <= set(counts), counts


# ---- on the GPU --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gate_device_twins_equal_the_host_twins(aniso_gate):
    r = run(aniso_gate, "--threads", str(THREADS), check=False)
    print(r.stdout)
    m = re.fullmatch(r"(\d+) probes, (\d+) inputs, (\d+) mismatches", r.stdout.strip().splitlines()[-1])
    assert m and r.returncode == 0 and m.group(3) == "0", r.stdout + r.stderr


class AnisoFrame(MipFrame):
    def want(self, ctx, rig, pose, cam, minify, max_probes):
        return aniso_want(ctx, rig, pose, cam, minify, max_probes, self.src, self.out_dims, self.prefill if rig is not None else None)


@pytest.mark.gpu
@pytest.mark.parametrize("name", MIP_INPUTS)
@pytest.mark.parametrize("interp", INTERPS)
@pytest.mark.parametrize("model", sorted(MODELS))
def test_frames_equal_the_oracle_composite(model, interp, name, torch_cuda):
    """3- and 1-plane frames of noise (odd sizes, 4:2:0 chroma) equal the oracle's composite of the twin bit for bit at
    maxProbes 2, 8 and 16, maxLevel 0 (level 0 supersampled), 4 and 8."""
    torch = torch_cuda
    ctx, rig = _ctx(name, interp), _rig(name, seed=interp)
    vft = t360.VideoFrameTransform(ctx)
    st = torch.cuda.Stream()
    for k, (probes, minify) in enumerate(((2, (4, -1.0)), (8, (0, 0.0)), (16, (8, 0.5)))):
        pose, cam = aniso_pose(MODELS[model], 31 * interp + 7 * k + len(name))
        for n in (3, 1):
            f = AnisoFrame(torch, name, n, seed=interp + k)
            want = f.want(ctx, rig, pose, cam, minify, probes)
            torch.cuda.synchronize()
            assert vft.make_camera_aniso_frame_call(f.in_planes, f.out_planes, f.dims)(pose, cam, minify, probes, st.cuda_stream, rig)
            st.synchronize()
            for p, got in enumerate(f.host()):
                _check(got, want[p], f"{model} {probes} probes {minify} {pose}, {n} planes, plane {p}")
    vft.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["equirect", "cubemap_32", "pair_190"])
def test_one_probe_equals_the_camera_mip_and_camera_calls(name, torch_cuda):
    """maxProbes 1 gives the camera-mip call's bytes and launches, and with maxLevel 0 the camera call's."""
    torch = torch_cuda
    rig = _rig(name, seed=1)
    st = torch.cuda.Stream()
    for interp in INTERPS:
        vft = t360.VideoFrameTransform(_ctx(name, interp))
        for k, minify in enumerate(((8, 0.0), (3, -0.5), (0, 1.0))):
            pose, cam = aniso_pose(sorted(MODELS.values())[(k + interp) % 5], 60 + k)
            a, b = MipFrame(torch, name, 3, seed=interp), MipFrame(torch, name, 3, seed=interp)
            torch.cuda.synchronize()
            n0 = t360.kernel_launch_count()
            assert vft.make_camera_aniso_frame_call(a.in_planes, a.out_planes, a.dims)(pose, cam, minify, 1, st.cuda_stream, rig)
            n1 = t360.kernel_launch_count()
            if minify[0]:
                assert vft.make_camera_mip_frame_call(b.in_planes, b.out_planes, b.dims)(pose, cam, minify, st.cuda_stream, rig)
            else:
                assert vft.make_camera_frame_call(b.in_planes, b.out_planes, b.dims)(pose, cam, st.cuda_stream, rig)
            assert n1 - n0 == t360.kernel_launch_count() - n1, (name, minify)
            st.synchronize()
            for p, (x, y) in enumerate(zip(a.host(), b.host())):
                assert np.array_equal(x, y), (name, interp, minify, p)
        vft.close()


@pytest.mark.gpu
def test_trajectory_on_two_streams(torch_cuda):
    """Two streams enqueue a trajectory without synchronising, model, pose, minify and maxProbes changing every frame: every
    frame equals the oracle, takes the camera-mip call's launches, and device memory stays bounded."""
    torch = torch_cuda
    ctx = _ctx("tb_to_lr", t360.CUBIC)
    vft = t360.VideoFrameTransform(ctx)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    args = []
    for k in range(20):
        pose, cam = aniso_pose(sorted(MODELS.values())[k % 5], 700 + k)
        args.append((pose, cam, (k % 9, (-1.0, 0.0, 0.75)[k % 3]), (2, 4, 8, 16, 1)[k % 5]))
    want_launches = sum(len(t360.mip_level_sizes(*_in_dims("tb_to_lr")[0], m[0])) for _, _, m, _ in args)
    mem = []
    for lap in range(3):
        frames = [AnisoFrame(torch, "tb_to_lr", 3, seed=k + lap) for k in range(len(args))]
        torch.cuda.synchronize()
        n0 = t360.kernel_launch_count()
        for k, (f, (pose, cam, minify, probes)) in enumerate(zip(frames, args)):
            assert vft.make_camera_aniso_frame_call(f.in_planes, f.out_planes, f.dims)(pose, cam, minify, probes, streams[k % 2].cuda_stream)
        torch.cuda.synchronize()
        assert t360.kernel_launch_count() - n0 == want_launches
        mem.append(torch.cuda.mem_get_info()[0])
        for k, (f, (pose, cam, minify, probes)) in enumerate(zip(frames, args)):
            want = f.want(ctx, None, pose, cam, minify, probes)
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
    f = AnisoFrame(torch, "equirect", 3)
    before = f.host()
    call = vft.make_camera_aniso_frame_call(f.in_planes, f.out_planes, f.dims)
    n0 = t360.kernel_launch_count()
    for minify, probes in (((9, 0.0), 4), ((4, float("nan")), 4), ((4, 0.0), 0), ((4, 0.0), 3), ((4, 0.0), 32), ((0, 0.0), -1)):
        assert not call((0.0, 0.0, 0.0, 90.0, 60.0), PINHOLE, minify, probes, 0)
    assert not call((0.0, 0.0, 0.0, 200.0, 60.0), PINHOLE, (4, 0.0), 4, 0)
    torch.cuda.synchronize()
    assert t360.kernel_launch_count() == n0
    assert all(np.array_equal(a, b) for a, b in zip(before, f.host()))
    assert "anisotropic camera view" in _stdout(capfd)
    vft.close()
