"""Camera models of the per-frame views: equidistant fisheye, stereographic and Pannini beside the pinhole
(T360B200_cameraMap / camera_map, T360B200_transformFrameCameraAsync / make_camera_frame_call).

What pins what:
  - PINHOLE against rectilinear_map bit for bit, and the camera call against the rectilinear call byte for byte;
  - each model's host map against a float64 model of the header's table, through test_rectilinear's rotation and input
    lookup (its `model`, with the ray replaced);
  - geometry that does not restate the contract: the equidistant angle-to-radius law, the stereographic little planet's
    nadir and rings, Pannini's straight verticals, its d = 0 limit and the forward Pannini projection;
  - sincCos, the equidistant model's sin(rho) / rho and cos(rho), against double over every float of its range (the host
    build; tests/test_twin_gates.py compares the device build with it over every 32-bit input, and cameraRay and the
    rectilinear chains of every model over structured families);
  - the frames against the plain-C oracle's cv::remap of camera_map's map and against the planned path, and the records
    the kernel computes read back through test_position_chains' decode and compared with the host twin's.
Poses, rigs and planes are made from seeds."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import tests.test_gather_plan as tgp
import tests.test_rectilinear as tr
import transform360_b200 as t360
from oracle import c_oracle as co
from tests.golden.cases import SMALL
from tests.test_lens import make_rig
from tests.test_position_chains import _quantised, coordinate_sources, decode, expected_fields
from tests.test_rectilinear import INPUTS, INTERPS, OUT_DIMS, RECT_CTX, Frame, _ctx, _in_dims, _pattern, _poses, _rig
from tests.test_rectilinear import torch_cuda  # noqa: F401 (fixture)
from tests.test_warp_map import _check, _refused, _stdout

WRAP, TRANSPARENT = t360.BORDER_WRAP, t360.BORDER_TRANSPARENT
PINHOLE, EQUIDISTANT, STEREOGRAPHIC, PANNINI = (t360.T360_CAMERA_PINHOLE, t360.T360_CAMERA_EQUIDISTANT, t360.T360_CAMERA_STEREOGRAPHIC,
                                                t360.T360_CAMERA_PANNINI)
MODELS = {"equidistant": EQUIDISTANT, "stereographic": STEREOGRAPHIC, "pannini": PANNINI}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = lambda v: float(np.float32(v))


def pannini_limit(d):
    """The widest hfov (degrees) a Pannini camera with distance d accepts: d + cos(hfov / 2) > 0."""
    return 2.0 * math.degrees(math.acos(-d)) if d < 1 else 360.0


def camera_poses(model, seed, n=3):
    """(pose, camera) pairs of `model`: seeded poses with large roll over the model's range, and fixed wide ones (past 180
    degrees for the fisheye models, near the hfov limit for Pannini)."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        ang = (float(rng.uniform(-180, 180)), float(rng.uniform(-85, 85)), float(rng.uniform(-180, 180)))
        if model == PANNINI:
            d = float(rng.uniform(0, 1))
            h = float(rng.uniform(20, min(300.0, pannini_limit(d) - 1)))
            out.append(((*ang, h, float(rng.uniform(15, 170))), (model, d)))
        else:
            top = 360.0 if model == EQUIDISTANT else 340.0
            out.append(((*ang, float(rng.uniform(20, top)), float(rng.uniform(20, top))), (model, 0.0)))
    if model == EQUIDISTANT:
        out += [((0.0, 0.0, 0.0, 180.0, 180.0), (model, 0.0)), ((30.0, -60.0, 20.0, 360.0, 360.0), (model, 0.0)),
                ((-100.0, 20.0, 5.0, 2.0, 1.5), (model, 0.0))]
    elif model == STEREOGRAPHIC:
        out += [((0.0, -90.0, 0.0, 270.0, 270.0), (model, 0.0)), ((170.0, 45.0, -120.0, 359.0, 200.0), (model, 0.0)),
                ((-100.0, 20.0, 5.0, 2.0, 1.5), (model, 0.0))]
    else:
        out += [((12.0, 10.0, 30.0, pannini_limit(0.3) - 0.5, 100.0), (model, 0.3)), ((-40.0, 0.0, 0.0, 358.0, 179.0), (model, 1.0)),
                ((100.0, -20.0, 5.0, 150.0, 90.0), (model, 0.0))]
    return out


# ---- the float64 model -------------------------------------------------------------------------------------------------
def camera_rays(ctx, pose, camera, w, h, mono=False):
    """Unit rotated rays (float64 [h][w][3]) and output eyes of a w x h view: steps 1-5 of the header's contract with the
    camera's ray in step 4."""
    yaw, pitch, roll, hfov, vfov = pose
    model, d = camera
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
    X, Y = 2 * x - 1, 2 * (1 - y) - 1
    hh, hv = math.radians(hfov) / 2, math.radians(vfov) / 2
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
        c = (-k * d + np.sqrt(k * k * d * d - (k + 1) * (k * d * d - 1))) / (k + 1)
        q = np.stack([u * (d + c) / (d + 1), v * (d + c) / (d + 1), c], -1)
    else:
        q = np.stack([X * F32(math.tan(hh)), Y * F32(math.tan(hv)), np.ones_like(X)], -1)
    s1, s2, s3 = np.sin(np.radians([yaw, pitch, roll]))
    c1, c2, c3 = np.cos(np.radians([yaw, pitch, roll]))
    rows = np.array([[c1 * c3 + s1 * s2 * s3, c3 * s1 * s2 - c1 * s3, c2 * s1], [c2 * s3, c2 * c3, -s2],
                     [c1 * s2 * s3 - c3 * s1, c1 * c3 * s2 + s1 * s3, c1 * c2]])
    t = np.stack([q[..., 0] * r[0] - q[..., 1] * r[1] + q[..., 2] * r[2] for r in rows], -1) * np.array([1.0, -1.0, 1.0])
    return t / np.linalg.norm(t, axis=-1, keepdims=True), eye


def camera_model(name, ctx, rig, pose, camera, in_w, in_h, w, h, monkeypatch):
    """test_rectilinear.model (the input lookup, its near-threshold and polar pixels) with the camera's rays."""
    with monkeypatch.context() as m:
        m.setattr(tr, "rays", lambda c, p, ww, hh, mono=False: camera_rays(c, p, camera, ww, hh, mono))
        with np.errstate(divide="ignore", invalid="ignore"):
            return tr.model(name, ctx, rig, pose, in_w, in_h, w, h)


# ---- no GPU needed -----------------------------------------------------------------------------------------------------
def test_camera_entry_points_are_exported_with_their_bindings(tmp_path):
    from transform360_b200.handler import EXPORTED_SYMBOLS, LIB_PATH, PKG
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    L = t360.load()
    for name in ("T360B200_cameraMap", "T360B200_transformFrameCameraAsync"):
        assert name in EXPORTED_SYMBOLS and name in defined, name
    P = C.POINTER
    assert L.T360B200_cameraMap.argtypes == [P(t360.FrameTransformContext), P(t360.T360LensRig), P(t360.T360Pose), P(t360.T360Camera)] + \
        [C.c_int] * 4 + [C.c_void_p]
    assert L.T360B200_transformFrameCameraAsync.argtypes == [C.c_void_p, P(t360.T360LensRig), P(t360.T360Pose), P(t360.T360Camera), C.c_int] + \
        [C.c_void_p] * 9
    assert hasattr(t360.VideoFrameTransform, "make_camera_frame_call") and callable(t360.camera_map)
    assert C.sizeof(t360.T360Camera) == 8 and (PINHOLE, EQUIDISTANT, STEREOGRAPHIC, PANNINI) == (0, 1, 2, 3)
    src = tmp_path / "proto.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "transform360_b200.h"\n'
                   "int (*a)(const FrameTransformContext*, const T360LensRig*, const T360Pose*, const T360Camera*, int, int, int, int, float*) = "
                   "T360B200_cameraMap;\n"
                   "int (*b)(VideoFrameTransform*, const T360LensRig*, const T360Pose*, const T360Camera*, int, const uint8_t* const*, "
                   "uint8_t* const*, const int*, const int*, const int*, const int*, const int*, const int*, void*) = "
                   "T360B200_transformFrameCameraAsync;\n"
                   'int main(void) {\n  printf("%zu %zu %d %d %d %d\\n", sizeof(T360Camera), offsetof(T360Camera, pannini), T360_CAMERA_PINHOLE, '
                   "T360_CAMERA_EQUIDISTANT, T360_CAMERA_STEREOGRAPHIC, T360_CAMERA_PANNINI);\n  return a == 0 || b == 0;\n}\n")
    exe = tmp_path / "proto"
    subprocess.run(["cc", "-Wall", "-Werror", "-I", str(PKG.parent / "include"), "-c", "-o", str(tmp_path / "proto.o"), str(src)], check=True)
    subprocess.run(["cc", "-I", str(PKG.parent / "include"), "-o", str(exe), str(tmp_path / "proto.o"), str(LIB_PATH)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [8, t360.T360Camera.pannini.offset, 0, 1, 2, 3]


@pytest.mark.parametrize("name", INPUTS)
def test_pinhole_camera_is_the_rectilinear_map(name):
    """camera_map with PINHOLE (the pannini field is not read) equals rectilinear_map bit for bit, NaNs included."""
    rig = _rig(name, seed=len(name))
    for pose in _poses(sum(map(ord, name)) + 1):
        for (w, h), (in_w, in_h) in zip(((97, 65), (49, 33)), _in_dims(name)):
            want = t360.rectilinear_map(_ctx(name), pose, in_w, in_h, w, h, rig)
            for cam in (PINHOLE, (PINHOLE, float("nan")), (PINHOLE, 7.0)):
                got = t360.camera_map(_ctx(name), pose, cam, in_w, in_h, w, h, rig)
                assert got.tobytes() == want.tobytes(), (pose, cam)


@pytest.mark.parametrize("name", INPUTS)
@pytest.mark.parametrize("model", sorted(MODELS))
def test_camera_map_equals_the_float64_model(model, name, monkeypatch):
    """camera_map against the float64 model of the header's table for seeded poses over each model's range (past 180
    degrees for the fisheye models, up to the hfov limit for Pannini), at odd luma and chroma sizes.  Within 0.01 px
    (context inputs) or 0.02 px (rigs), as test_rectilinear, columns modulo the input width, away from the same near-threshold
    and polar pixels; the same NaN pattern elsewhere, and no NaN for a context input."""
    rig = _rig(name, seed=len(name))
    tol = 0.02 if rig is not None else 0.01
    worst, near_total, pixels = 0.0, 0, 0
    for pose, cam in camera_poses(MODELS[model], sum(map(ord, name + model))):
        for (w, h), (in_w, in_h) in zip(((97, 65), (49, 33)), _in_dims(name)):
            ctx = _ctx(name)
            got = t360.camera_map(ctx, pose, cam, in_w, in_h, w, h, rig).astype(np.float64)
            want, near, polar = camera_model(name, ctx, rig, pose, cam, in_w, in_h, w, h, monkeypatch)
            gn, wn = np.isnan(got).any(-1), np.isnan(want).any(-1)
            bad = (gn != wn) & ~near
            assert not bad.any(), f"{int(bad.sum())} pixels covered differently from the model (pose {pose}, {cam}, {w}x{h})"
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
    print(f"{model} / {name}: max |delta| {worst:.2e} px")
    assert worst <= tol, f"max |delta| {worst:.5f} px"
    assert near_total < 0.01 * pixels, f"{near_total} of {pixels} pixels near a threshold"


def _equirect_directions(m, in_w, in_h):
    """(longitude, latitude) in radians of an equirect input's map positions (u = lon / 2pi + 0.5, v = 0.5 - lat / pi)."""
    lon = ((m[..., 0].astype(np.float64) + 0.5) / in_w - 0.5) * 2 * np.pi
    lat = (0.5 - (m[..., 1].astype(np.float64) + 0.5) / in_h) * np.pi
    return lon, lat


BIG = (8192, 4096)  # a large equirect input, so that a map position resolves its direction to ~1e-6 rad


def test_equidistant_180_is_a_dome_master():
    """An N x N equidistant view at 180 degrees, unrotated: the angle of every pixel's ray to the view axis is its distance
    from the plane's centre times 180 / N degrees (so the inscribed circle is the front hemisphere)."""
    for n in (64, 101):
        m = t360.camera_map(_ctx("equirect"), (0, 0, 0, 180, 180), EQUIDISTANT, *BIG, n, n)
        lon, lat = _equirect_directions(m, *BIG)
        angle = np.degrees(np.arccos(np.clip(np.cos(lat) * np.cos(lon), -1, 1)))
        i, j = np.mgrid[:n, :n]
        radius = np.hypot(j + 0.5 - n / 2, i + 0.5 - n / 2)
        err = np.abs(angle - radius * 180.0 / n)
        assert err.max() < 2e-3, f"{n}x{n}: {err.max():.2e} degrees"


def test_stereographic_little_planet_looks_at_the_nadir():
    """A stereographic view at pitch -90 (yaw and roll 0 and seeded): the centre pixel of an odd plane samples the
    equirect's bottom row, and every ring of pixels at one distance from the centre samples one latitude, which falls
    monotonically towards the zenith as the ring grows."""
    n = 101
    rng = np.random.default_rng(7)
    for yaw, roll, fov in ((0.0, 0.0, 270.0), (float(rng.uniform(-180, 180)), float(rng.uniform(-180, 180)), 220.0)):
        m = t360.camera_map(_ctx("equirect"), (yaw, -90.0, roll, fov, fov), STEREOGRAPHIC, *BIG, n, n)
        c = n // 2
        assert BIG[1] - 1 <= m[c, c, 1] < BIG[1], m[c, c]
        lon, lat = _equirect_directions(m, *BIG)
        i, j = np.mgrid[:n, :n]
        r2 = (i - c) ** 2 + (j - c) ** 2
        rings = np.unique(r2)
        lo = np.array([lat[r2 == r].min() for r in rings])
        hi = np.array([lat[r2 == r].max() for r in rings])
        assert (hi - lo).max() < 1e-5, f"a ring spans {(hi - lo).max():.2e} rad of latitude"
        assert (np.diff(lo) > 0).all() and lo[0] < -math.pi / 2 + 1e-3 and lo[-1] > 0  # the far corners look above the horizon


@pytest.mark.parametrize("d", [0.0, 0.25, 0.5, 1.0])
def test_pannini_keeps_verticals_and_projects_forward(d):
    """A Pannini view at pitch = roll = 0: each output column samples one longitude; each ray, projected forward by the
    Pannini formula ((d + 1) sin lon / (d + cos lon), (d + 1) tan lat / (d + cos lon)) and scaled by the plane's edges
    (xe, ye), lands on its pixel's centre to 0.01 px (near the hfov limit a float32 map position of an 8192-wide input
    resolves the longitude to ~1e-6 rad, which the projection stretches to a few thousandths of an output pixel); and
    d = 0 is the pinhole map to about 1e-3 px."""
    w, h = 161, 91
    for yaw, hfov, vfov in ((0.0, 120.0, 80.0), (33.0, min(300.0, pannini_limit(d) - 2.0), 150.0)):
        m = t360.camera_map(_ctx("equirect"), (yaw, 0, 0, hfov, vfov), (PANNINI, d), *BIG, w, h)
        lon, lat = _equirect_directions(m, *BIG)
        col_spread = (m[..., 0].max(0) - m[..., 0].min(0)).max()
        assert col_spread < 2e-3, f"a column spans {col_spread:.2e} px"
        lam = np.angle(np.exp(1j * (lon - math.radians(yaw))))
        dd = F32(d)
        hh = math.radians(hfov) / 2
        xe, ye = F32((dd + 1) * math.sin(hh) / (dd + math.cos(hh))), F32(math.tan(math.radians(vfov) / 2))
        X = (dd + 1) * np.sin(lam) / (dd + np.cos(lam)) / xe
        Y = (dd + 1) * np.tan(lat) / (dd + np.cos(lam)) / ye
        x, y = np.meshgrid(2 * (np.arange(w) + 0.5) / w - 1, 1 - 2 * (np.arange(h) + 0.5) / h)
        err = max(np.abs(X - x).max() * w / 2, np.abs(Y - y).max() * h / 2)
        assert err < 1e-2, f"d {d}, hfov {hfov}: the forward projection misses its pixel by {err:.2e} px"
    if d == 0.0:
        for pose in _poses(3, w=w, h=h):
            if pose[4] <= 179:
                a = t360.camera_map(_ctx("equirect"), pose, (PANNINI, 0.0), 2048, 1024, w, h).astype(np.float64)
                b = t360.rectilinear_map(_ctx("equirect"), pose, 2048, 1024, w, h).astype(np.float64)
                dx = np.abs(a[..., 0] - b[..., 0])
                dx = np.minimum(dx, 2048 - dx)
                d2 = np.hypot(dx, a[..., 1] - b[..., 1])
                lat_ok = np.abs(b[..., 1] - 511.5) < 0.45 * 1024  # (away from the poles, where a column is a degree)
                assert d2[lat_ok].max() < 2e-3, (pose, float(d2[lat_ok].max()))


SINCCOS_GATE = r"""
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>
#include "oriented_view.h"
int main(int argc, char** argv) {
  const int threads = std::atoi(argv[1]);
  const float top = static_cast<float>(M_PI * std::sqrt(2.0));
  uint32_t last;
  std::memcpy(&last, &top, 4);
  std::vector<double> es(threads), ec(threads);
  std::vector<uint32_t> ws(threads), wc(threads);
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; ++t)
    pool.emplace_back([&, t] {
      for (uint32_t b = t; b <= last; b += threads) {
        float r;
        std::memcpy(&r, &b, 4);
        float s, c;
        t360::sincCos(r, &s, &c);
        const double rd = r, ws_ = rd > 0 ? std::sin(rd) / rd : 1.0, wc_ = std::cos(rd);
        const double e1 = std::fabs(s - ws_), e2 = std::fabs(c - wc_);
        if (!(e1 <= es[t])) { es[t] = e1; ws[t] = b; }
        if (!(e2 <= ec[t])) { ec[t] = e2; wc[t] = b; }
      }
    });
  for (auto& p : pool) p.join();
  double s = 0, c = 0;
  uint32_t bs = 0, bc = 0;
  for (int t = 0; t < threads; ++t) {
    if (es[t] > s) { s = es[t]; bs = ws[t]; }
    if (ec[t] > c) { c = ec[t]; bc = wc[t]; }
  }
  float fs, fc;
  std::memcpy(&fs, &bs, 4);
  std::memcpy(&fc, &bc, 4);
  std::printf("%u %.3e %.9g %.3e %.9g\n", last + 1, s, fs, c, fc);
  return 0;
}
"""


def test_sinccos_against_double_over_every_float(tmp_path):
    """sincCos (oriented_view.h), compiled for the host as the library's host code is (-ffp-contract=off), against double
    sin(rho) / rho and cos(rho) over every float rho in [0, pi sqrt 2]: the largest absolute error of each is reported and
    asserted.  Measured: 1.9e-7 for sin(rho) / rho and 9.1e-7 for cos(rho) (the two angle doublings amplify the polynomials'
    rounding), a ray direction within ~1e-6 rad."""
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.fail("no C++ compiler to build the sincCos comparison")
    src, exe = tmp_path / "sinccos_gate.cpp", tmp_path / "sinccos_gate"
    src.write_text(SINCCOS_GATE)
    csrc = os.path.join(ROOT, "transform360_b200", "csrc")
    subprocess.run([cxx, "-std=c++17", "-O2", "-ffp-contract=off", "-fno-builtin", "-pthread", "-I", csrc, "-I", os.path.join(ROOT, "include"),
                    str(src), "-o", str(exe), "-lm"], check=True)
    out = subprocess.run([str(exe), str(max(8, os.cpu_count() or 1))], capture_output=True, text=True, check=True).stdout.split()
    count, es, at_s, ec, at_c = int(out[0]), float(out[1]), float(out[2]), float(out[3]), float(out[4])
    print(f"sincCos over {count} floats: max |sin(r)/r error| {es:.3e} at r = {at_s}, max |cos(r) error| {ec:.3e} at r = {at_c}")
    assert count > 1_000_000_000
    assert es <= 2.5e-7 and ec <= 1.0e-6, (es, ec)


@pytest.mark.parametrize("name", INPUTS)
@pytest.mark.parametrize("model", sorted(MODELS))
def test_gather_plans_of_camera_maps_keep_the_invariants(model, name, monkeypatch):
    """HostPlan.from_warp of each model's map (BORDER_WRAP for a context input, BORDER_TRANSPARENT for a rig) keeps what
    tests/test_gather_plan.py checks for context plans, at every interpolation."""
    rig = _rig(name, seed=3)
    (in_w, in_h), _ = _in_dims(name)
    border = TRANSPARENT if rig is not None else WRAP
    pose, cam = camera_poses(MODELS[model], 11, 1)[0]
    for interp in INTERPS:
        m = t360.camera_map(_ctx(name, interp), pose, cam, in_w, in_h, 161, 81, rig)
        hp = t360.HostPlan.from_warp(t360.make_context(interpolation_alg=interp, **RECT_CTX), m, in_w, in_h, border)
        shown = t360.make_context(interpolation_alg=interp, output_layout=t360.LAYOUT_BARREL if border == TRANSPARENT else t360.LAYOUT_EQUIRECT)
        monkeypatch.setitem(SMALL, "__camera", {})
        monkeypatch.setattr(tgp, "_plan", lambda case, plane: (shown, hp, in_w, in_h))
        tgp.test_gather_plan_invariants("small", "__camera", 0)
        hp.close()


def _bad_calls():
    """(what, rig or None, pose, camera or None, context overrides) the library refuses, beyond the rectilinear refusals."""
    good = make_rig("pair_190")
    ok = (10.0, 5.0, 0.0, 90.0, 60.0)
    nan, inf = float("nan"), float("inf")
    cases = [("NULL camera", None, ok, None, {}), ("NULL camera with a rig", good, ok, None, {})]
    for model in (-1, 4, 1000):
        cases.append((f"model {model}", None, ok, (model, 0.0), {}))
    for d in (nan, inf, -inf, -0.01, 1.01):
        cases.append((f"pannini {d}", None, ok, (PANNINI, d), {}))
    fields = {EQUIDISTANT: ((0.0, 60.0), (360.5, 60.0), (90.0, -1.0), (90.0, 361.0)),
              STEREOGRAPHIC: ((0.0, 60.0), (359.5, 60.0), (90.0, 0.0), (90.0, 360.0)),
              PANNINI: ((0.0, 60.0), (359.5, 60.0), (90.0, 0.0), (90.0, 179.5))}
    for model, fovs in fields.items():
        for hfov, vfov in fovs:
            cases.append((f"model {model} fov {hfov} x {vfov}", None, (0.0, 0.0, 0.0, hfov, vfov), (model, 0.5), {}))
    for d in (0.0, 0.3, 0.9):  # d + cos(hfov / 2) <= 0: just past the limit, and the limit rounded up
        cases.append((f"Pannini {d} past its limit", good, (0.0, 0.0, 0.0, pannini_limit(d) + 0.01, 60.0), (PANNINI, d), {}))
    cases.append(("low-pass", None, ok, (EQUIDISTANT, 0.0), dict(enable_low_pass_filter=1)))
    cases.append(("no interpolation", good, ok, (STEREOGRAPHIC, 0.0), dict(interpolation_alg=3)))
    cases.append(("bad rig", make_rig("pair_190"), ok, (PANNINI, 0.5), {}))
    cases[-1][1].numLenses = 3
    cases.append(("NULL pose", None, None, (EQUIDISTANT, 0.0), {}))
    cases.append(("pose not finite", None, (0.0, nan, 0.0, 90.0, 60.0), (STEREOGRAPHIC, 0.0), {}))
    return cases


def _frame_call(L, vft, rig, pose, camera, n=1, planes=(0x20000,), dims=(64, 32, 8, 8), pitch=(64, 8)):
    P, I = C.c_void_p * 3, C.c_int * 3
    arr = lambda v: I(*([v] * 3))
    pb = C.byref(t360.T360Pose(*pose)) if pose is not None else None
    cb = C.byref(t360.T360Camera(*camera)) if camera is not None else None
    return L.T360B200_transformFrameCameraAsync(vft._h, C.byref(rig) if rig is not None else None, pb, cb, n, P(*(list(planes) * 3)[:3]),
                                                P(*(list(planes) * 3)[:3]), arr(dims[0]), arr(dims[1]), arr(pitch[0]), arr(dims[2]),
                                                arr(dims[3]), arr(pitch[1]), None)


def test_refusals_happen_without_a_gpu(capfd):
    """Every refusal of camera_map and of the camera frame call comes with a message and before any CUDA call, with bogus
    plane pointers that are never dereferenced and no kernel launched; the fields' upper limits themselves are accepted."""
    L = t360.load()
    m = np.zeros((8, 8, 2), np.float32)
    n0 = t360.kernel_launch_count()
    for what, rig, pose, cam, ov in _bad_calls():
        ctx = t360.make_context(**{**RECT_CTX, **ov})
        pb = C.byref(t360.T360Pose(*pose)) if pose is not None else None
        cb = C.byref(t360.T360Camera(*cam)) if cam is not None else None
        assert not L.T360B200_cameraMap(C.byref(ctx), C.byref(rig) if rig is not None else None, pb, cb, 64, 32, 8, 8, m.ctypes.data), what
        assert _stdout(capfd).strip(), what
        with t360.VideoFrameTransform(ctx) as vft:
            _refused(capfd, _frame_call, L, vft, rig, pose, cam)
    ctx = t360.make_context(**RECT_CTX)
    cam = t360.T360Camera(EQUIDISTANT, 0.0)
    for args in ((64, 32, 0, 8, m.ctypes.data), (64, 0, 8, 8, m.ctypes.data), (64, 32, 8, 8, None)):
        _refused(capfd, L.T360B200_cameraMap, C.byref(ctx), None, C.byref(t360.T360Pose(0, 0, 0, 90, 60)), C.byref(cam), *args)
    _refused(capfd, L.T360B200_cameraMap, None, None, C.byref(t360.T360Pose(0, 0, 0, 90, 60)), C.byref(cam), 64, 32, 8, 8, m.ctypes.data)
    with t360.VideoFrameTransform(ctx) as vft:
        for kw in (dict(n=0), dict(n=4), dict(planes=(None,)), dict(dims=(0, 32, 8, 8)), dict(pitch=(63, 8))):
            _refused(capfd, lambda: _frame_call(L, vft, None, (0, 0, 0, 90, 60), (STEREOGRAPHIC, 0.0), **kw))
    assert not L.T360B200_transformFrameCameraAsync(None, None, None, None, 1, None, None, None, None, None, None, None, None, None)
    assert t360.kernel_launch_count() == n0
    with pytest.raises(ValueError):
        t360.camera_map(ctx, (0, 0, 0, 90, 60), (PANNINI, 2.0), 64, 32, 8, 8)
    for pose, cam in (((0, 0, 0, 360, 360), EQUIDISTANT), ((0, 0, 0, 359, 359), STEREOGRAPHIC), ((0, 0, 0, 359, 179), (PANNINI, 1.0)),
                      ((0, 0, 0, pannini_limit(0.5) - 0.01, 179), (PANNINI, 0.5)), ((0, 0, 0, 180, 90), (PANNINI, 0.0))):
        assert not np.isnan(t360.camera_map(ctx, pose, cam, 64, 32, 8, 8)).any(), (pose, cam)


# ---- on the GPU --------------------------------------------------------------------------------------------------------
def _want(f, ctx, rig, pose, cam):
    """Frame.want with camera_map's maps: the oracle's cv::remap, BORDER_WRAP, or BORDER_TRANSPARENT into the pre-fill."""
    maps = [t360.camera_map(ctx, pose, cam, *f.in_dims[p], *OUT_DIMS[p], rig) for p in range(min(f.n, 2))]
    out = []
    for p in range(f.n):
        if rig is None:
            out.append(co.remap_u8(f.src[p], maps[min(p, 1)], ctx.interpolation_alg, WRAP))
        else:
            dst = _pattern(*OUT_DIMS[p], p) if p == 0 else np.full(OUT_DIMS[p][::-1], 128, np.uint8)
            out.append(co.remap_u8(f.src[p], maps[min(p, 1)], ctx.interpolation_alg, TRANSPARENT, dst))
    return out, maps


@pytest.mark.gpu
@pytest.mark.parametrize("name", INPUTS)
@pytest.mark.parametrize("interp", INTERPS)
@pytest.mark.parametrize("model", sorted(MODELS))
def test_camera_frames_equal_the_oracle_and_the_planned_path(model, interp, name, torch_cuda):
    """On a never-planned transform, 3- and 1-plane frames (one with an unaligned luma plane) equal the oracle's cv::remap
    of camera_map's maps bit for bit; then camera_map -> generate_map_from_warp -> transformFrameAsync gives the same frame."""
    torch = torch_cuda
    ctx = _ctx(name, interp)
    rig = _rig(name, seed=interp)
    pose, cam = camera_poses(MODELS[model], interp * 10 + len(name), 1)[0]
    vft = t360.VideoFrameTransform(ctx)
    st = torch.cuda.Stream()
    for n, unaligned in ((3, False), (1, False), (3, True)):
        f = Frame(torch, name, n, seed=interp, unaligned=unaligned)
        want, _ = _want(f, ctx, rig, pose, cam)
        torch.cuda.synchronize()
        assert vft.make_camera_frame_call(f.in_planes, f.out_planes, f.dims)(pose, cam, st.cuda_stream, rig)
        st.synchronize()
        for p, got in enumerate(f.host()):
            _check(got, want[p], f"{model} frame of {n} planes{' (unaligned)' if unaligned else ''}, plane {p}")
    f = Frame(torch, name, 3, seed=interp)
    want, maps = _want(f, ctx, rig, pose, cam)
    for idx in (0, 1):
        assert vft.generate_map_from_warp(maps[idx], *f.in_dims[idx], idx, TRANSPARENT if rig is not None else WRAP)
    torch.cuda.synchronize()
    assert vft.make_frame_call(f.in_planes, f.out_planes, f.dims)(st.cuda_stream)
    st.synchronize()
    for p, got in enumerate(f.host()):
        _check(got, want[p], f"planned {model} frame, plane {p}")
    vft.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", INPUTS)
def test_pinhole_camera_call_is_the_rectilinear_call(name, torch_cuda):
    """PINHOLE through the camera call gives the rectilinear call's bytes, for seeded poses at every interpolation."""
    torch = torch_cuda
    rig = _rig(name, seed=2)
    st = torch.cuda.Stream()
    for interp in INTERPS:
        vft = t360.VideoFrameTransform(_ctx(name, interp))
        for pose in _poses(interp + 40, 2):
            a, b = Frame(torch, name, 3, seed=interp), Frame(torch, name, 3, seed=interp)
            torch.cuda.synchronize()
            assert vft.make_camera_frame_call(a.in_planes, a.out_planes, a.dims)(pose, (PINHOLE, 0.5), st.cuda_stream, rig)
            assert vft.make_rectilinear_frame_call(b.in_planes, b.out_planes, b.dims)(pose, st.cuda_stream, rig)
            st.synchronize()
            for p, (x, y) in enumerate(zip(a.host(), b.host())):
                assert np.array_equal(x, y), (name, interp, pose, p)
        vft.close()


def record_cases():
    """(input, pose, camera, (in_w, in_h, out_w, out_h) of luma, own K) of the record read-back: every input with each model,
    and the branch points -- rho = 0 at the centre pixel of odd planes, rays beyond 90 degrees (equidistant at 360 and
    stereographic at 300 and 359), Pannini within 0.1 degree of its hfov limit and at d = 1 -- plus the reframing size."""
    out = []
    for n, name in enumerate(INPUTS):
        (iw, ih), _ = _in_dims(name)
        for model in sorted(MODELS):
            for pose, cam in camera_poses(MODELS[model], n + len(model), 1):
                out.append((name, pose, cam, (iw, ih, 97, 65), [4, 8][n % 2]))
    out += [("equirect", (0.0, 0.0, 0.0, 180.0, 180.0), (EQUIDISTANT, 0.0), (259, 131, 97, 97), 4),
            ("cubemap_32", (20.0, -30.0, 40.0, 360.0, 360.0), (EQUIDISTANT, 0.0), (261, 174, 97, 65), 8),
            ("tilted", (0.0, 0.0, 0.0, 200.0, 200.0), (EQUIDISTANT, 0.0), (259, 131, 97, 65), 4),
            ("equirect", (0.0, -90.0, 0.0, 300.0, 300.0), (STEREOGRAPHIC, 0.0), (259, 131, 97, 97), 8),
            ("pair_190", (10.0, -80.0, 30.0, 359.0, 359.0), (STEREOGRAPHIC, 0.0), (259, 131, 97, 65), 4),
            ("tb_to_lr", (-30.0, 5.0, 0.0, pannini_limit(0.3) - 0.1, 120.0), (PANNINI, 0.3), (259, 131, 97, 65), 8),
            ("equirect", (150.0, 10.0, -5.0, 358.9, 179.0), (PANNINI, 1.0), (259, 131, 97, 65), 4),
            ("equirect", (35.0, -20.0, 10.0, 180.0, 101.25), (EQUIDISTANT, 0.0), (7680, 3840, 1920, 1080), 4),
            ("equirect", (35.0, 0.0, 0.0, 150.0, 100.0), (PANNINI, 0.7), (7680, 3840, 1920, 1080), 8)]
    return out


def _plane_dims(sizes):
    iw, ih, ow, oh = sizes
    return [(iw, ih, ow, oh), ((iw + 1) // 2, (ih + 1) // 2, (ow + 1) // 2, (oh + 1) // 2)]


def _run(torch, name, pose, cam, k, dims, frames, prefill):
    """Each frame (a list of two source planes) through the camera call on a never-planned transform; the output planes."""
    ctx = _ctx(name, tr.INTERPS[[1, 2, 4, 8].index(k)])
    rig = _rig(name, seed=len(name))
    vft = t360.VideoFrameTransform(ctx)
    d_in = [torch.from_numpy(np.stack([f[p] for f in frames])).cuda() for p in range(2)]
    d_out = [torch.full((len(frames), dims[p][3], dims[p][2]), prefill if p == 0 else 0, dtype=torch.uint8, device="cuda") for p in range(2)]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for f in range(len(frames)):
        ins = [(d_in[p][f].data_ptr(), dims[p][0]) for p in range(2)]
        outs = [(d_out[p][f].data_ptr(), dims[p][2]) for p in range(2)]
        assert vft.make_camera_frame_call(ins, outs, dims)(pose, cam, st.cuda_stream, rig)
    st.synchronize()
    got = [d.cpu().numpy() for d in d_out]
    vft.close()
    return [[got[p][f] for p in range(2)] for f in range(len(frames))], ctx, rig


@pytest.mark.gpu
@pytest.mark.parametrize("k", (1, 2))
def test_records_on_the_device(k, torch_cuda):
    """Every record case through the camera call: the records read back (test_position_chains' coordinate sources and
    decode) equal HostPlan.from_warp of camera_map's map record for record, the same pixels are skipped, every byte on
    noise equals remap_u8 of that map, at K and (K = 2) at the case's own K."""
    torch = torch_cuda
    for name, pose, cam, sizes, own_k in record_cases():
        dims = _plane_dims(sizes)
        rig = _rig(name, seed=len(name))
        border = TRANSPARENT if rig is not None else WRAP
        for kk in ((k, own_k) if k == 2 else (k,)):
            coords = [coordinate_sources(*dims[p][:2], kk) for p in range(2)] if kk <= 2 else None
            noise = [co.noise_plane(*dims[p][:2], plane=p, frame=kk) for p in range(2)]
            frames = ([[coords[p][s] for p in range(2)] for s in range(len(coords[0]))] if coords else []) + \
                [[np.zeros(dims[p][1::-1], np.uint8) for p in range(2)], noise]
            got, ctx, _ = _run(torch, name, pose, cam, kk, dims, frames, 255)
            warp = t360.make_context(interpolation_alg=ctx.interpolation_alg, enable_low_pass_filter=0)
            for p in range(2):
                iw, ih, ow, oh = dims[p]
                m = t360.camera_map(ctx, pose, cam, iw, ih, ow, oh, rig)
                rec = _quantised(warp, m, iw, ih, border)
                what = f"{name} {pose} {cam} K {kk} plane {p}"
                prefill = np.full((oh, ow), 255 if p == 0 or border == WRAP else 128, np.uint8)
                want = co.remap_u8(noise[p], m, ctx.interpolation_alg, border, prefill.copy())
                assert np.array_equal(got[-1][p], want), f"{what}: {int((got[-1][p] != want).sum())} noise bytes differ"
                skip = co.remap_u8(np.zeros((ih, iw), np.uint8), m, ctx.interpolation_alg, border, prefill.copy()) != 0
                assert np.array_equal(got[-2][p] != 0, skip), f"{what}: skipped pixels differ"
                if coords is None:
                    continue
                dev = decode(kk, [f[p] for f in got[:-2]])
                host, valid = expected_fields(kk, rec, iw, ih)
                for axis in range(2):
                    bad = valid[axis] & ~skip & (dev[axis] != host[axis])
                    assert not bad.any(), f"{what}: {int(bad.sum())} {('column', 'row')[axis]} records differ"
                    assert (valid[axis] & ~skip).any(), what


@pytest.mark.gpu
def test_camera_trajectory_on_two_streams(torch_cuda):
    """30 frames whose model, pose and Pannini d change every frame, on the context's equirect input and through a rig,
    enqueued on two streams in turn without synchronising: every frame equals its own reference."""
    torch = torch_cuda
    rng = np.random.default_rng(9)
    models = [PINHOLE, EQUIDISTANT, STEREOGRAPHIC, PANNINI]
    for name in ("equirect", "pair_190"):
        ctx = _ctx(name, t360.CUBIC)
        rig = _rig(name, seed=4)
        vft = t360.VideoFrameTransform(ctx)
        frames = [Frame(torch, name, 3, seed=f % 4) for f in range(30)]
        traj = []
        for f in range(30):
            model = models[f % 4]
            d = float(rng.uniform(0, 1))
            top = {PINHOLE: 179.0, EQUIDISTANT: 360.0, STEREOGRAPHIC: 359.0, PANNINI: min(359.0, pannini_limit(d) - 1)}[model]
            hfov = float(rng.uniform(30, top))
            vfov = float(rng.uniform(30, 179.0 if model in (PINHOLE, PANNINI) else top))
            traj.append(((float(rng.uniform(-180, 180)), float(rng.uniform(-90, 90)), float(rng.uniform(-180, 180)), hfov, vfov), (model, d)))
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        torch.cuda.synchronize()
        for f, fr in enumerate(frames):
            assert vft.make_camera_frame_call(fr.in_planes, fr.out_planes, fr.dims)(*traj[f], streams[f % 2].cuda_stream, rig)
        for s in streams:
            s.synchronize()
        for f, fr in enumerate(frames):
            want, _ = _want(fr, ctx, rig, *traj[f])
            for p, got in enumerate(fr.host()):
                _check(got, want[p], f"{name}: frame {f} {traj[f]}, plane {p}")
        vft.close()


@pytest.mark.gpu
def test_refused_calls_launch_nothing_and_one_launch_per_frame(torch_cuda, capfd):
    """Refused camera frames on real planes launch nothing and leave the outputs' bytes; 200 frames of changing models
    and poses are one launch each, without growth of device memory."""
    torch = torch_cuda
    L = t360.load()
    for what, rig, pose, cam, ov in _bad_calls():
        ctx = t360.make_context(**{**RECT_CTX, **ov})
        with t360.VideoFrameTransform(ctx) as vft:
            f = Frame(torch, "pair_190", 3)
            before = f.host()
            torch.cuda.synchronize()
            n0 = t360.kernel_launch_count()
            P, I = C.c_void_p * 3, C.c_int * 3
            pb = C.byref(t360.T360Pose(*pose)) if pose is not None else None
            cb = C.byref(t360.T360Camera(*cam)) if cam is not None else None
            ok = L.T360B200_transformFrameCameraAsync(vft._h, C.byref(rig) if rig is not None else None, pb, cb, 3,
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
    for name in ("equirect", "tilted"):
        vft = t360.VideoFrameTransform(_ctx(name, t360.LANCZOS4))
        rig = _rig(name, 41)
        f = Frame(torch, name, 3)
        call = vft.make_camera_frame_call(f.in_planes, f.out_planes, f.dims)
        st = torch.cuda.Stream()
        cams = [(EQUIDISTANT, 0.0), (STEREOGRAPHIC, 0.0), (PANNINI, 0.5), (PINHOLE, 0.0)]
        torch.cuda.synchronize()
        for i in range(8):
            assert call((7.0 * i, 1.0, 0.0, 90.0, 60.0), cams[i % 4], st.cuda_stream, rig)
        st.synchronize()
        free_before = torch.cuda.mem_get_info()[0]
        n0 = t360.kernel_launch_count()
        for i in range(200):
            assert call((7.0 * i, 30.0 * np.sin(i), 3.0 * i, 40.0 + i % 120, 30.0 + i % 100), cams[i % 4], st.cuda_stream, rig)
        launches = t360.kernel_launch_count() - n0
        st.synchronize()
        assert launches == 200, f"{launches} launches for 200 frames"
        assert torch.cuda.mem_get_info()[0] >= free_before - (2 << 20), "device memory grew over camera frames"
        vft.close()
