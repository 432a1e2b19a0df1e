"""Rectilinear views: perspective (pinhole) cameras posed per frame, looking into the context's equirect or cube-map input
or into a fisheye lens rig (T360B200_rectilinearMap / rectilinear_map, T360B200_transformFrameRectilinearAsync /
make_rectilinear_frame_call).

What pins what:
  - the host map against a float64 numpy model written from the header's contract (pinhole ray, rotation, input lookup or
    the lens model of tests/test_lens.py);
  - the whole pinhole -> lens chain against cv2.fisheye.initUndistortRectifyMap for an unrotated single lens;
  - the rotation's sense and handedness against the planner: a 90-degree square view is the FRONT face of a CUBEMAP_32
    output of the same orientation (T360B200_poseSamples);
  - the frames against the plain-C oracle's cv::remap of rectilinear_map's map (BORDER_WRAP for the context's input,
    BORDER_TRANSPARENT into pre-filled planes for a rig), and against the planned path, bit for bit.
Poses, rigs and planes are made from seeds."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import tests.test_gather_plan as tgp
import transform360_b200 as t360
from oracle import c_oracle as co
from tests.golden.cases import SMALL
from tests.test_lens import RIGS, make_rig
from tests.test_lens import model as lens_model
from tests.test_warp_map import _check, _pitch, _refused, _stdout

WRAP, TRANSPARENT = t360.BORDER_WRAP, t360.BORDER_TRANSPARENT
INTERPS = [t360.NEAREST, t360.LINEAR, t360.CUBIC, t360.LANCZOS4]
RECT_CTX = dict(enable_low_pass_filter=0)
# the context inputs: mono equirect, stereo top-bottom equirect into side-by-side and stacked views, a cube map with
# input_expand_coef != 1; the rigs of tests/test_lens.py
CONTEXTS = {
    "equirect": dict(input_layout=t360.LAYOUT_EQUIRECT),
    "tb_to_lr": dict(input_layout=t360.LAYOUT_EQUIRECT, input_stereo_format=t360.STEREO_FORMAT_TB, output_stereo_format=t360.STEREO_FORMAT_LR),
    "tb_to_tb": dict(input_layout=t360.LAYOUT_EQUIRECT, input_stereo_format=t360.STEREO_FORMAT_TB, output_stereo_format=t360.STEREO_FORMAT_TB,
                     vflip=1),
    "cubemap_32": dict(input_layout=t360.LAYOUT_CUBEMAP_32, input_expand_coef=1.04),
}
INPUTS = sorted(CONTEXTS) + RIGS


def _ctx(name, interp=t360.CUBIC, **ov):
    """The context of input `name` (a rig's: a mono equirect context, whose input fields the rig replaces)."""
    return t360.make_context(**RECT_CTX, **CONTEXTS.get(name, {}), interpolation_alg=interp, **ov)


def _rig(name, seed=0):
    return make_rig(name, seed) if name in RIGS else None


def _poses(seed, n=3, w=97, h=65):
    """Seeded poses, large roll included, and fixed narrow, wide and 170-degree ones; vfov square-pixel or free."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        hfov = float(rng.uniform(20, 150))
        vfov = t360.square_pixel_vfov(hfov, w, h) if k % 2 == 0 else float(rng.uniform(15, 120))
        out.append((float(rng.uniform(-180, 180)), float(rng.uniform(-85, 85)), float(rng.uniform(-180, 180)), hfov, vfov))
    out += [(12.0, 70.0, 170.0, 170.0, 150.0), (-100.0, -20.0, 5.0, 2.0, 1.5), (170.0, -89.0, -120.0, 120.0, 170.0)]
    return out


# ---- the float64 model -------------------------------------------------------------------------------------------------
def rays(ctx, pose, w, h, mono=False):
    """Unit rotated rays (float64 [h][w][3]) and output eyes of a w x h view: steps 1-5 of the header's contract."""
    yaw, pitch, roll, hfov, vfov = pose
    x, y = np.meshgrid((np.arange(w) + 0.5) / w, (np.arange(h) + 0.5) / h)
    stereo = ctx.input_stereo_format != t360.STEREO_FORMAT_MONO and not mono
    eye = np.zeros((h, w), bool)
    if stereo and ctx.output_stereo_format == t360.STEREO_FORMAT_LR:
        eye = x > 0.5
        x = np.where(eye, (x - 0.5) / 0.5, x / 0.5)
    elif stereo and ctx.output_stereo_format == t360.STEREO_FORMAT_TB:
        eye = y > 0.5
        y = np.where(eye, (y - 0.5) / 0.5, y / 0.5)
        if ctx.vflip:
            y = np.where(eye, 1 - y, y)
    y = 1 - y
    tx, ty = (float(np.float32(np.tan(np.radians(f) / 2))) for f in (hfov, vfov))
    q = np.stack([(2 * x - 1) * tx, (2 * y - 1) * ty, np.ones_like(x)], -1)
    s1, s2, s3 = np.sin(np.radians([yaw, pitch, roll]))
    c1, c2, c3 = np.cos(np.radians([yaw, pitch, roll]))
    rows = np.array([[c1 * c3 + s1 * s2 * s3, c3 * s1 * s2 - c1 * s3, c2 * s1], [c2 * s3, c2 * c3, -s2],
                     [c1 * s2 * s3 - c3 * s1, c1 * c3 * s2 + s1 * s3, c1 * c2]])
    # t.x = q.x xx - q.y xy + q.z xz, t.y = -(q.x yx - q.y yy + q.z yz), t.z = q.x zx - q.y zy + q.z zz
    t = np.stack([q[..., 0] * r[0] - q[..., 1] * r[1] + q[..., 2] * r[2] for r in rows], -1) * np.array([1.0, -1.0, 1.0])
    return t / np.linalg.norm(t, axis=-1, keepdims=True), eye


def _cube_input(d, e):
    """The 3x2 cube-map lookup of unit rays d: (u, v, near), near where a face test lies within 1e-6 of its threshold."""
    faces = [(2, 0, 1, 5, 3, 1, 1, True), (2, 0, 1, 3, 3, 1, -1, False), (0, 2, 1, 3, 1, -1, 1, True), (0, 2, 1, 1, 1, -1, -1, False),
             (1, 0, 2, 1, 3, -1, 1, True), (1, 0, 2, 5, 1, 1, 1, False)]
    u, v = np.full(d.shape[:2], np.nan), np.full(d.shape[:2], np.nan)
    near = np.zeros(d.shape[:2], bool)
    for mj, a, b, col, row, su, sv, neg in faces:
        major = d[..., mj]
        ok = (major <= -0.5) if neg else (major >= 0.5)
        gx, gy = d[..., a] / major, d[..., b] / major
        near |= ok & ((np.abs(np.abs(gx) - 1) < 1e-6) | (np.abs(np.abs(gy) - 1) < 1e-6))
        win = ok & (np.abs(gx) <= 1) & (np.abs(gy) <= 1) & np.isnan(u)
        u = np.where(win, (col + su * gx / e) / 6, u)
        v = np.where(win, (row + sv * gy / e) / 4, v)
    return u, v, near


def model(name, ctx, rig, pose, in_w, in_h, w, h):
    """The contract in float64: (map [h][w][2], NaN where a rig does not cover; near: pixels within 1e-5 of a lens-choice,
    coverage or cube-face threshold; polar: rays within 1e-3 of the input's poles, where longitude is ill-conditioned)."""
    d, eye = rays(ctx, pose, w, h, mono=rig is not None)
    polar = np.hypot(d[..., 0], d[..., 2]) < 1e-3
    if rig is not None:
        m, _, near, _ = lens_model(rig, d, np.zeros((h, w), bool), in_w, in_h)
        return m, near, np.zeros_like(near)
    if ctx.input_layout == t360.LAYOUT_CUBEMAP_32:
        u, v, near = _cube_input(d, np.float64(np.float32(ctx.input_expand_coef)))
        polar[:] = False
    else:
        u = np.arctan2(d[..., 0], d[..., 2]) / (2 * np.pi) + 0.5
        v = np.arcsin(-d[..., 1]) / np.pi + 0.5
        near = np.zeros((h, w), bool)
    if ctx.input_stereo_format == t360.STEREO_FORMAT_TB:
        v = v * 0.5 + np.where(eye, 0.5, 0.0)
    return np.stack([u * in_w - 0.5, v * in_h - 0.5], -1), near, polar


def _in_dims(name):
    return ((261, 174), (131, 87)) if name == "cubemap_32" else ((259, 131), (130, 66))


# ---- no GPU needed -----------------------------------------------------------------------------------------------------
def test_rectilinear_entry_points_are_exported_with_their_bindings(tmp_path):
    from transform360_b200.handler import EXPORTED_SYMBOLS, LIB_PATH, PKG
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    L = t360.load()
    for name in ("T360B200_rectilinearMap", "T360B200_transformFrameRectilinearAsync"):
        assert name in EXPORTED_SYMBOLS and name in defined, name
    P = C.POINTER
    assert L.T360B200_rectilinearMap.argtypes == [P(t360.FrameTransformContext), P(t360.T360LensRig), P(t360.T360Pose)] + [C.c_int] * 4 + [C.c_void_p]
    assert L.T360B200_transformFrameRectilinearAsync.argtypes == [C.c_void_p, P(t360.T360LensRig), P(t360.T360Pose), C.c_int] + [C.c_void_p] * 9
    assert hasattr(t360.VideoFrameTransform, "make_rectilinear_frame_call") and callable(t360.rectilinear_map)
    # the prototypes compile from C, and the pose has the header's layout
    src = tmp_path / "proto.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "transform360_b200.h"\n'
                   "int (*a)(const FrameTransformContext*, const T360LensRig*, const T360Pose*, int, int, int, int, float*) = "
                   "T360B200_rectilinearMap;\n"
                   "int (*b)(VideoFrameTransform*, const T360LensRig*, const T360Pose*, int, const uint8_t* const*, uint8_t* const*, "
                   "const int*, const int*, const int*, const int*, const int*, const int*, void*) = T360B200_transformFrameRectilinearAsync;\n"
                   'int main(void) {\n  printf("%zu %zu %zu\\n", sizeof(T360Pose), offsetof(T360Pose, hfov), offsetof(T360Pose, vfov));\n'
                   "  return a == 0 || b == 0;\n}\n")
    exe = tmp_path / "proto"
    subprocess.run(["cc", "-Wall", "-Werror", "-I", str(PKG.parent / "include"), "-c", "-o", str(tmp_path / "proto.o"), str(src)], check=True)
    subprocess.run(["cc", "-I", str(PKG.parent / "include"), "-o", str(exe), str(tmp_path / "proto.o"), str(LIB_PATH)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(t360.T360Pose), t360.T360Pose.hfov.offset, t360.T360Pose.vfov.offset]


def test_square_pixel_vfov():
    for hfov, w, h in ((90.0, 1920, 1080), (170.0, 97, 65), (1.0, 640, 480), (60.0, 100, 100)):
        vfov = t360.square_pixel_vfov(hfov, w, h)
        assert np.isclose(np.tan(np.radians(vfov) / 2) / np.tan(np.radians(hfov) / 2), h / w, rtol=1e-12)
    assert t360.square_pixel_vfov(75.0, 64, 64) == pytest.approx(75.0)


@pytest.mark.parametrize("name", INPUTS)
def test_rectilinear_map_equals_the_float64_model(name):
    """rectilinear_map against the float64 model for seeded poses (large roll, narrow, wide and 170-degree fields of view),
    at odd luma and chroma sizes.  Within 0.01 px (context inputs) or 0.02 px (rigs, as tests/test_lens.py), columns taken
    modulo the input width (the equirect seam); the column is not compared within 1e-3 rad of an equirect input's poles,
    where longitude is ill-conditioned.  NaN patterns equal, except pixels within 1e-5 of a lens-choice, coverage or cube
    face threshold (fewer than 0.1 %)."""
    rig = _rig(name, seed=len(name))
    tol = 0.02 if rig is not None else 0.01
    worst, near_total, pixels = 0.0, 0, 0
    for pose in _poses(sum(map(ord, name))):
        for (w, h), (in_w, in_h) in zip(((97, 65), (49, 33)), _in_dims(name)):
            ctx = _ctx(name)
            got = t360.rectilinear_map(ctx, pose, in_w, in_h, w, h, rig).astype(np.float64)
            want, near, polar = model(name, ctx, rig, pose, in_w, in_h, w, h)
            gn, wn = np.isnan(got).any(-1), np.isnan(want).any(-1)
            assert (np.isnan(got[..., 0]) == np.isnan(got[..., 1])).all()
            bad = (gn != wn) & ~near
            assert not bad.any(), f"{int(bad.sum())} pixels covered differently from the model (pose {pose}, {w}x{h})"
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
    assert worst <= tol, f"max |delta| {worst:.5f} px"
    assert near_total < 0.001 * pixels, f"{near_total} of {pixels} pixels near a threshold"


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_lens_undistortion_equals_opencv(seed):
    """A one-lens rig with its lens unrotated, viewed with pose (0, 0, 0, hfov, vfov) at the calibration size, is OpenCV's
    fisheye undistortion: where covered, the map lies within 0.02 px of cv2.fisheye.initUndistortRectifyMap(K, D, I, P)
    with P = [[W / (2 tx), 0, W / 2 - 0.5], [0, H / (2 ty), H / 2 - 0.5], [0, 0, 1]]."""
    cv2 = pytest.importorskip("cv2")
    rig = make_rig("single_200", seed)
    L, W, H = rig.lens[0], rig.calibWidth, rig.calibHeight
    rng = np.random.default_rng(seed)
    for hfov, vfov in ((100.0, t360.square_pixel_vfov(100.0, W, H)), (float(rng.uniform(30, 160)), float(rng.uniform(30, 160))), (170.0, 170.0)):
        got = t360.rectilinear_map(_ctx("single_200"), (0, 0, 0, hfov, vfov), W, H, W, H, rig).astype(np.float64)
        tx, ty = (float(np.float32(np.tan(np.radians(f) / 2))) for f in (hfov, vfov))
        K = np.array([[L.fx, 0, L.cx], [0, L.fy, L.cy], [0, 0, 1]], np.float64)
        D = np.array(list(L.k), np.float64).reshape(4, 1)
        P = np.array([[W / (2 * tx), 0, W / 2 - 0.5], [0, H / (2 * ty), H / 2 - 0.5], [0, 0, 1]], np.float64)
        mx, my = cv2.fisheye.initUndistortRectifyMap(K, D, np.eye(3), P, (W, H), cv2.CV_32FC1)
        covered = ~np.isnan(got).any(-1)
        assert covered.all(), "a 200-degree lens covers every ray of a view narrower than 180 degrees"
        delta = max(np.abs(got[..., 0] - mx).max(), np.abs(got[..., 1] - my).max())
        assert delta <= 0.02, f"hfov {hfov}, vfov {vfov}: {delta:.4f} px from cv2.fisheye.initUndistortRectifyMap"


def _pos32(rec):
    """Positions in 1/32 px (x, y) of int32 records [..][2]: col0 and rowPhase as T360B200_hostPlanSamples holds them."""
    col0, rp = rec[..., 0].astype(np.int64), rec[..., 1].astype(np.int64)
    return col0 * 32 + (rp & 31), (rp >> 10) * 32 + ((rp >> 5) & 31)


def test_square_view_is_the_front_face_of_a_cube_map():
    """50 seeded orientations: the records of an N x N view with hfov = vfov = 90 (rectilinear_map, planned under
    BORDER_WRAP) differ from those of the FRONT face of a 3N x 2N CUBEMAP_32 output with the same orientation
    (T360B200_poseSamples) by at most one 1/32-px step per axis, columns modulo the input width: the rotation has the
    planner's sense and handedness."""
    n, in_w, in_h = 48, 512, 256
    rng = np.random.default_rng(50)
    cube = t360.make_context(**RECT_CTX, output_layout=t360.LAYOUT_CUBEMAP_32, expand_coef=1.0, interpolation_alg=t360.CUBIC)
    for _ in range(50):
        yaw, pitch, roll = (float(v) for v in (rng.uniform(-180, 180), rng.uniform(-90, 90), rng.uniform(-180, 180)))
        m = t360.rectilinear_map(cube, (yaw, pitch, roll, 90.0, 90.0), in_w, in_h, n, n)
        view = t360.HostPlan.from_warp(cube, m, in_w, in_h, WRAP).samples
        face = t360.pose_samples(cube, (yaw, pitch, roll, 0.0, 0.0), in_w, in_h, 3 * n, 2 * n)[n:, n:2 * n]
        (vx, vy), (fx, fy) = _pos32(view), _pos32(face)
        dx = np.abs(vx - fx) % (32 * in_w)
        dx = np.minimum(dx, 32 * in_w - dx)
        assert dx.max() <= 1 and np.abs(vy - fy).max() <= 1, (yaw, pitch, roll, int(dx.max()), int(np.abs(vy - fy).max()))


@pytest.mark.parametrize("name", INPUTS)
@pytest.mark.parametrize("interp", INTERPS)
def test_gather_plans_of_rectilinear_maps_keep_the_invariants(name, interp, monkeypatch):
    """HostPlan.from_warp of each input's map (BORDER_WRAP for a context input, BORDER_TRANSPARENT for a rig) keeps what
    tests/test_gather_plan.py checks for context plans."""
    rig = _rig(name, seed=3)
    (in_w, in_h), _ = _in_dims(name)
    border = TRANSPARENT if rig is not None else WRAP
    m = t360.rectilinear_map(_ctx(name, interp), (20.0, 35.0, -13.0, 110.0, 80.0), in_w, in_h, 161, 81, rig)
    hp = t360.HostPlan.from_warp(t360.make_context(interpolation_alg=interp, **RECT_CTX), m, in_w, in_h, border)
    # test_gather_plan reads the context only to tell staged plans from BORDER_TRANSPARENT ones (the barrel layouts)
    shown = t360.make_context(interpolation_alg=interp, output_layout=t360.LAYOUT_BARREL if border == TRANSPARENT else t360.LAYOUT_EQUIRECT)
    monkeypatch.setitem(SMALL, "__rectilinear", {})
    monkeypatch.setattr(tgp, "_plan", lambda case, plane: (shown, hp, in_w, in_h))
    tgp.test_gather_plan_invariants("small", "__rectilinear", 0)


def _bad_calls():
    """(what, rig or None, pose or None, context overrides) the library refuses."""
    good = make_rig("pair_190")
    ok = (10.0, 5.0, 0.0, 90.0, 60.0)
    cases = [("NULL pose", None, None, {}), ("NULL pose with a rig", good, None, {})]
    for k in range(5):
        for v in (float("nan"), float("inf"), float("-inf")):
            pose = list(ok)
            pose[k] = v
            cases.append((f"pose {pose}", good if k == 2 else None, tuple(pose), {}))
    for hfov, vfov in ((0.0, 60.0), (-5.0, 60.0), (179.01, 60.0), (180.0, 60.0), (90.0, 0.0), (90.0, 179.5), (90.0, -1.0)):
        cases.append((f"fov {hfov} x {vfov}", None, (0.0, 0.0, 0.0, hfov, vfov), {}))

    def rig_with(**kw):
        r = make_rig("pair_190")
        for key, v in kw.items():
            if key == "k":
                r.lens[0].k[:] = v
            elif key in ("numLenses", "calibWidth", "calibHeight"):
                setattr(r, key, v)
            else:
                setattr(r.lens[1 if key.startswith("l1_") else 0], key.removeprefix("l1_"), v)
        return r
    for kw in (dict(numLenses=0), dict(numLenses=3), dict(calibWidth=0), dict(calibHeight=-2), dict(fx=0.0), dict(l1_fy=-1.0),
               dict(cx=float("nan")), dict(l1_yaw=float("inf")), dict(maxAngle=0.0), dict(l1_maxAngle=180.5), dict(k=(-0.2, 0.0, 0.0, 0.0))):
        cases.append((str(kw), rig_with(**kw), ok, {}))
    for ov in (dict(enable_low_pass_filter=1), dict(interpolation_alg=3), dict(interpolation_alg=9)):
        cases.append((str(ov), None, ok, ov))
        cases.append((f"{ov} with a rig", good, ok, ov))
    return cases


def _frame_call(L, vft, rig, pose, n=1, planes=(0x20000,), dims=(64, 32, 8, 8), pitch=(64, 8)):
    P, I = C.c_void_p * 3, C.c_int * 3
    arr = lambda v: I(*([v] * 3))
    pb = C.byref(t360.T360Pose(*pose)) if pose is not None else None
    return L.T360B200_transformFrameRectilinearAsync(vft._h, C.byref(rig) if rig is not None else None, pb, n, P(*(list(planes) * 3)[:3]),
                                                     P(*(list(planes) * 3)[:3]), arr(dims[0]), arr(dims[1]), arr(pitch[0]), arr(dims[2]),
                                                     arr(dims[3]), arr(pitch[1]), None)


def test_refusals_happen_without_a_gpu(capfd):
    """Every refusal of rectilinear_map and of the frame call comes with a message and before any CUDA call (this machine
    may have none): fake device addresses are never dereferenced.  The output layout is not read."""
    L = t360.load()
    m = np.zeros((8, 8, 2), np.float32)
    for what, rig, pose, ov in _bad_calls():
        ctx = t360.make_context(**{**RECT_CTX, **ov})
        pb = C.byref(t360.T360Pose(*pose)) if pose is not None else None
        assert not L.T360B200_rectilinearMap(C.byref(ctx), C.byref(rig) if rig is not None else None, pb, 64, 32, 8, 8, m.ctypes.data), what
        assert _stdout(capfd).strip(), what
        with t360.VideoFrameTransform(ctx) as vft:
            _refused(capfd, _frame_call, L, vft, rig, pose)
    good, pose = make_rig("pair_190"), t360.T360Pose(0, 0, 0, 90, 60)
    ctx = t360.make_context(**RECT_CTX)
    for args in ((64, 32, 0, 8, m.ctypes.data), (64, 0, 8, 8, m.ctypes.data), (-1, 32, 8, 8, m.ctypes.data), (64, 32, 8, 8, None)):
        _refused(capfd, L.T360B200_rectilinearMap, C.byref(ctx), None, C.byref(pose), *args)
    _refused(capfd, L.T360B200_rectilinearMap, None, C.byref(good), C.byref(pose), 64, 32, 8, 8, m.ctypes.data)
    with pytest.raises(ValueError):
        t360.rectilinear_map(t360.make_context(enable_low_pass_filter=1), (0, 0, 0, 90, 60), 64, 32, 8, 8)
    with t360.VideoFrameTransform(ctx) as vft:
        for rig in (None, good):
            for kw in (dict(n=0), dict(n=4), dict(planes=(None,)), dict(dims=(0, 32, 8, 8)), dict(dims=(64, 32, 8, -1)),
                       dict(pitch=(63, 8)), dict(pitch=(64, 7))):
                _refused(capfd, lambda: _frame_call(L, vft, rig, (0, 0, 0, 90, 60), **kw))
    assert not L.T360B200_transformFrameRectilinearAsync(None, None, None, 1, None, None, None, None, None, None, None, None, None)
    # what the pose replaces is not read: every output layout (FLAT_FIXED, barrels, out of range) and the view fields
    for layout in (t360.LAYOUT_FLAT_FIXED, t360.LAYOUT_BARREL, t360.LAYOUT_BARREL_SPLIT, 7, -1):
        c = t360.make_context(**RECT_CTX, output_layout=layout, fixed_hfov=float("nan"), expand_coef=3.0, width_scale_factor=0.5)
        a = t360.rectilinear_map(c, (0, 0, 0, 90, 60), 64, 32, 8, 8)
        assert np.array_equal(a, t360.rectilinear_map(t360.make_context(**RECT_CTX), (0, 0, 0, 90, 60), 64, 32, 8, 8))
        b = t360.rectilinear_map(c, (0, 0, 0, 90, 60), 64, 32, 8, 8, good)
        assert np.array_equal(b, t360.rectilinear_map(t360.make_context(**RECT_CTX), (0, 0, 0, 90, 60), 64, 32, 8, 8, good), equal_nan=True)


# ---- on the GPU --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests must run on an H100 (there is no CPU fallback to test)")
    return torch


OUT_DIMS = [(97, 65), (49, 33), (49, 33)]


def _pattern(w, h, p):
    """What an output holds before the frame: a non-zero pattern (chroma too: a rig's call pre-fills it with 128)."""
    i, j = np.mgrid[:h, :w]
    return (((i * 7 + j * 13 + 29 * p) % 251) + 1).astype(np.uint8)


def _dev(torch, a, pitch=None):
    pitch = pitch or _pitch(a.shape[1])
    t = torch.zeros((a.shape[0], pitch), dtype=torch.uint8, device="cuda")
    t[:, :a.shape[1]] = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t


class Frame:
    """Source planes (host and device) of input `name`, pre-filled outputs and the argument lists of one frame."""

    def __init__(self, torch, name, n=3, seed=0, unaligned=False):
        self.torch, self.n = torch, n
        luma, chroma = _in_dims(name)
        self.in_dims = [luma, chroma, chroma][:n]
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
        self.outs = []
        self.reset()
        self.dims = [(*self.in_dims[p], *OUT_DIMS[p]) for p in range(n)]

    def reset(self):
        torch = self.torch
        self.outs = self.outs or [torch.zeros((OUT_DIMS[p][1], _pitch(OUT_DIMS[p][0])), dtype=torch.uint8, device="cuda") for p in range(self.n)]
        for p, o in enumerate(self.outs):
            o[:, :OUT_DIMS[p][0]] = torch.from_numpy(_pattern(*OUT_DIMS[p], p)).cuda()
        return self

    @property
    def out_planes(self):
        return [(o.data_ptr(), o.stride(0)) for o in self.outs]

    def host(self):
        return [o[:, :OUT_DIMS[p][0]].cpu().numpy() for p, o in enumerate(self.outs)]

    def want(self, ctx, rig, pose):
        """The oracle's cv::remap of rectilinear_map's maps: BORDER_WRAP, or BORDER_TRANSPARENT into the pre-fill (luma: the
        pattern, chroma: 128) with a rig."""
        maps = [t360.rectilinear_map(ctx, pose, *self.in_dims[p], *OUT_DIMS[p], rig) for p in range(min(self.n, 2))]
        out = []
        for p in range(self.n):
            if rig is None:
                out.append(co.remap_u8(self.src[p], maps[min(p, 1)], ctx.interpolation_alg, WRAP))
            else:
                dst = _pattern(*OUT_DIMS[p], p) if p == 0 else np.full(OUT_DIMS[p][::-1], 128, np.uint8)
                out.append(co.remap_u8(self.src[p], maps[min(p, 1)], ctx.interpolation_alg, TRANSPARENT, dst))
        return out, maps


@pytest.mark.gpu
@pytest.mark.parametrize("name", INPUTS)
@pytest.mark.parametrize("interp", INTERPS)
def test_rectilinear_frames_equal_the_oracle_and_the_planned_path(name, interp, torch_cuda, monkeypatch):
    """On a never-planned transform, 3- and 1-plane frames (one with an unaligned luma plane) equal the oracle's cv::remap
    of rectilinear_map's maps bit for bit.  Then rectilinear_map -> generate_map_from_warp on indices 0 and 1:
    transformFrameAsync and the host-pointer ABI (streamed) give the same frames, and rectilinear frames on the transform
    holding those plans still do, while the plans stay in effect."""
    torch = torch_cuda
    monkeypatch.setenv("T360B200_PIPELINE_MIN_BYTES", "0")  # host planes take the streamed path
    ctx = _ctx(name, interp)
    rig = _rig(name, seed=interp)
    pose = _poses(interp * 10 + len(name), 1)[0]
    vft = t360.VideoFrameTransform(ctx)
    st = torch.cuda.Stream()
    for n, unaligned in ((3, False), (1, False), (3, True)):
        f = Frame(torch, name, n, seed=interp, unaligned=unaligned)
        want, _ = f.want(ctx, rig, pose)
        torch.cuda.synchronize()
        assert vft.make_rectilinear_frame_call(f.in_planes, f.out_planes, f.dims)(pose, st.cuda_stream, rig)
        st.synchronize()
        for p, got in enumerate(f.host()):
            _check(got, want[p], f"rectilinear frame of {n} planes{' (unaligned)' if unaligned else ''}, plane {p}")
    # the planned path for the same pose
    border = TRANSPARENT if rig is not None else WRAP
    f = Frame(torch, name, 3, seed=interp)
    want, maps = f.want(ctx, rig, pose)
    for idx in (0, 1):
        assert vft.generate_map_from_warp(maps[idx], *f.in_dims[idx], idx, border)
    torch.cuda.synchronize()
    assert vft.make_frame_call(f.in_planes, f.out_planes, f.dims)(st.cuda_stream)
    st.synchronize()
    for p, got in enumerate(f.host()):
        _check(got, want[p], f"planned frame, plane {p}")
        h_out = _pattern(*OUT_DIMS[p], p) if p == 0 else np.full(OUT_DIMS[p][::-1], 128, np.uint8)
        _check(vft.transform_plane(f.src[p], *OUT_DIMS[p], min(p, 1), p, out=h_out), want[p], f"host-pointer planned plane {p}")
    other = _poses(interp + 99, 1)[0]
    f2 = Frame(torch, name, 3, seed=interp + 1)
    want2, _ = f2.want(ctx, rig, other)
    torch.cuda.synchronize()
    assert vft.make_rectilinear_frame_call(f2.in_planes, f2.out_planes, f2.dims)(other, st.cuda_stream, rig)
    st.synchronize()
    for p, got in enumerate(f2.host()):
        _check(got, want2[p], f"rectilinear frame on a transform holding warp plans, plane {p}")
    f.reset()
    torch.cuda.synchronize()
    assert vft.make_frame_call(f.in_planes, f.out_planes, f.dims)(st.cuda_stream)
    st.synchronize()
    for p, got in enumerate(f.host()):
        _check(got, want[p], f"planned frame after the rectilinear frame, plane {p}")
    vft.close()


@pytest.mark.gpu
def test_pose_trajectory_with_a_rig_change_on_two_streams(torch_cuda):
    """30 frames of a seeded trajectory (pan, tilt, roll and zoom every frame), the rig replaced at frame 15 and the output
    planes recycled, enqueued on two streams in turn with no synchronisation between them; and the same trajectory on the
    context's equirect input: every frame equals the oracle."""
    torch = torch_cuda
    rigs = [make_rig("pair_190", 21), make_rig("tilted", 22)]
    rng = np.random.default_rng(5)
    steps = np.cumsum(rng.normal(0, [6, 2, 3, 3], (30, 4)), 0)
    traj = [(float(a), float(np.clip(b, -80, 80)), float(c), float(np.clip(90 + d, 20, 170))) for a, b, c, d in steps]
    poses = [(a, b, c, hf, t360.square_pixel_vfov(hf, *OUT_DIMS[0])) for a, b, c, hf in traj]
    for name in ("pair_190", "equirect"):
        ctx = _ctx(name, t360.CUBIC)
        vft = t360.VideoFrameTransform(ctx)
        frames = [Frame(torch, name, 3, seed=f % 4) for f in range(30)]
        rig_of = (lambda f: rigs[f >= 15]) if name in RIGS else (lambda f: None)
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        torch.cuda.synchronize()
        for f, fr in enumerate(frames):
            assert vft.make_rectilinear_frame_call(fr.in_planes, fr.out_planes, fr.dims)(poses[f], streams[f % 2].cuda_stream, rig_of(f))
        for s in streams:
            s.synchronize()
        for f, fr in enumerate(frames):
            want, _ = fr.want(ctx, rig_of(f), poses[f])
            for p, got in enumerate(fr.host()):
                _check(got, want[p], f"{name}: frame {f}, plane {p}")
        vft.close()


@pytest.mark.gpu
def test_reconfigure_between_rectilinear_frames_is_frame_exact(torch_cuda):
    """On a transform holding context plans, rectilinear frames and context frames interleaved with reconfigure_async
    (the interpolation, then input_expand_coef) and a reconfigure (the interpolation), all enqueued without synchronising:
    every rectilinear frame equals the oracle for the context current when it was enqueued, every context frame a fresh
    transform's, and the plans are left in effect."""
    torch = torch_cuda
    base = dict(RECT_CTX, **CONTEXTS["cubemap_32"], output_layout=t360.LAYOUT_EQUIRECT, interpolation_alg=t360.CUBIC)
    ctxs = [t360.make_context(**base), t360.make_context(**dict(base, interpolation_alg=t360.LINEAR)),
            t360.make_context(**dict(base, interpolation_alg=t360.LINEAR, input_expand_coef=1.0)),
            t360.make_context(**dict(base, interpolation_alg=t360.LANCZOS4))]
    vft = t360.VideoFrameTransform(ctxs[0])
    luma, chroma = _in_dims("cubemap_32")
    for idx, d in enumerate((luma, chroma)):
        assert vft.generateMapForPlane(*d, *OUT_DIMS[idx], idx)
    rect = [Frame(torch, "cubemap_32", 3, seed=s) for s in range(4)]
    plain = [Frame(torch, "cubemap_32", 3, seed=s) for s in range(4)]
    poses = [(30.0 * s, 5.0 - 10 * s, 20.0 * s, 100.0 - 15 * s, 70.0) for s in range(4)]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for s in range(4):
        if s in (1, 2):
            vft.reconfigure_async(ctxs[s])
        elif s == 3:
            vft.reconfigure(ctxs[s])
        assert vft.make_rectilinear_frame_call(rect[s].in_planes, rect[s].out_planes, rect[s].dims)(poses[s], st.cuda_stream)
        for o in plain[s].outs:
            o.zero_()
        assert vft.make_frame_call(plain[s].in_planes, plain[s].out_planes, plain[s].dims)(st.cuda_stream)
    st.synchronize()
    for s in range(4):
        want, _ = rect[s].want(ctxs[s], None, poses[s])
        for p, got in enumerate(rect[s].host()):
            _check(got, want[p], f"rectilinear frame {s}, plane {p}")
        fresh = t360.VideoFrameTransform(ctxs[s])
        for idx, d in enumerate((luma, chroma)):
            assert fresh.generateMapForPlane(*d, *OUT_DIMS[idx], idx)
        ref = Frame(torch, "cubemap_32", 3, seed=s)
        for o in ref.outs:
            o.zero_()
        assert fresh.make_frame_call(ref.in_planes, ref.out_planes, ref.dims)(0)
        torch.cuda.synchronize()
        for p, (got, w) in enumerate(zip(plain[s].host(), ref.host())):
            _check(got, w, f"context frame {s}, plane {p}")
        fresh.close()
    vft.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["equirect", "tilted"])
def test_device_memory_and_launches_stay_bounded(name, torch_cuda):
    """200 frames after a warm-up, a new pose every frame: one kernel launch each (a rig's chroma pre-fill is a memset) and
    no growth of device memory."""
    torch = torch_cuda
    ctx = _ctx(name, t360.LANCZOS4)
    rig = _rig(name, 41)
    vft = t360.VideoFrameTransform(ctx)
    f = Frame(torch, name, 3)
    call = vft.make_rectilinear_frame_call(f.in_planes, f.out_planes, f.dims)
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for i in range(5):
        assert call((7.0 * i, 1.0, 0.0, 90.0, 60.0), st.cuda_stream, rig)
    st.synchronize()
    free_before = torch.cuda.mem_get_info()[0]
    n0 = t360.kernel_launch_count()
    for i in range(200):
        assert call((7.0 * i, 30.0 * np.sin(i), 3.0 * i, 40.0 + i % 120, 30.0 + i % 100), st.cuda_stream, rig)
    launches = t360.kernel_launch_count() - n0
    st.synchronize()
    assert launches == 200, f"{launches} launches for 200 frames"
    assert torch.cuda.mem_get_info()[0] >= free_before - (2 << 20), "device memory grew over rectilinear frames"
    vft.close()


@pytest.mark.gpu
def test_refused_calls_launch_nothing_and_leave_the_outputs(torch_cuda, capfd):
    """Refused rectilinear frames on real planes: no kernel launch, the outputs keep their bytes (chroma included)."""
    torch = torch_cuda
    L = t360.load()
    for what, rig, pose, ov in _bad_calls():
        ctx = t360.make_context(**{**RECT_CTX, **ov})
        with t360.VideoFrameTransform(ctx) as vft:
            f = Frame(torch, "pair_190", 3)
            before = f.host()
            torch.cuda.synchronize()
            n0 = t360.kernel_launch_count()
            P, I = C.c_void_p * 3, C.c_int * 3
            pb = C.byref(t360.T360Pose(*pose)) if pose is not None else None
            ok = L.T360B200_transformFrameRectilinearAsync(vft._h, C.byref(rig) if rig is not None else None, pb, 3,
                                                           P(*[p[0] for p in f.in_planes]), P(*[p[0] for p in f.out_planes]),
                                                           I(*[d[0] for d in f.dims]), I(*[d[1] for d in f.dims]), I(*[p[1] for p in f.in_planes]),
                                                           I(*[d[2] for d in f.dims]), I(*[d[3] for d in f.dims]), I(*[p[1] for p in f.out_planes]),
                                                           None)
            torch.cuda.synchronize()
            assert not ok, what
            assert _stdout(capfd).strip(), what
            assert t360.kernel_launch_count() == n0, what
            for p, (a, b) in enumerate(zip(before, f.host())):
                assert np.array_equal(a, b), f"{what}: plane {p} changed"
