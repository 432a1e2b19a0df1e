"""Rolling-shutter lens rigs: a rig motion over the readout for the photometric lens and camera calls
(T360B200_lensMotionMaps / lens_motion_maps, T360B200_transformFrameLensMotionAsync / make_lens_motion_frame_call,
T360B200_cameraMotionMaps / camera_motion_maps, T360B200_transformFrameCameraMotionAsync / make_camera_motion_frame_call).

What pins what:
  - all-zero deltas against lens_photo_maps / camera_photo_maps: every array bit for bit, for any readout and sample count;
  - a constant delta against the photometric twin of the rig whose lenses are turned by it (the convention);
  - the twin against a float64 model whose fixed point t = readout(project(M(t) d)) is solved to convergence;
  - a synthetic rolling-shutter frame, rendered through a float64 forward model, corrected against the still frame;
  - the frames against the oracle composites of test_lens_photo / test_camera_photo, bit for bit, and the device half of
    the twin gate (tests/motion_twin_gate.cu) against its host half.
Rigs, motions, readouts and poses are made from seeds."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest

import transform360_b200 as t360
from transform360_b200 import synth
import tests.test_camera_photo as camera_photo
from tests.test_camera_mip import MODELS, MipFrame
from tests.test_camera_models import EQUIDISTANT, PINHOLE
from tests.test_camera_photo import photo_want, seam_pose
from tests.test_lens import IN_DIMS, LAYOUTS, LENS_CTX, OUT_DIMS, Frame, _orientations, _pattern, _rot, directions, make_rig
from tests.test_lens_blend import INTERPS
from tests.test_lens_photo import IDENTITY, STATS, equidistant_pair, photo_composite, rig_photos
from tests.test_rectilinear import RECT_CTX, _ctx
from tests.test_twin_gates import THREADS, gate_command, run
from tests.test_warp_map import _check, _refused, _stdout

READOUTS = {"rows": (0.0, 1.0, 0.0), "reversed": (0.0, -1.0, 1.0), "columns": (1.0, 0.0, 0.0), "half": (2.0, 0.0, -1.0)}


def motion(deltas, readouts=((0.0, 1.0, 0.0), (0.0, 1.0, 0.0))):
    return t360.rig_motion([tuple(float(x) for x in d) for d in deltas], readouts)


def zero_motion(n, readouts=((0.0, 1.0, 0.0), (0.0, 1.0, 0.0))):
    return motion([(0.0, 0.0, 0.0)] * n, readouts)


def sweep(n, angle, axis=0, readouts=((0.0, 1.0, 0.0), (0.0, 1.0, 0.0))):
    """A turn of `angle` degrees about one axis (0 yaw, 1 pitch, 2 roll) across the readout, centred on the frame's
    orientation, sampled at n times."""
    d = np.zeros((n, 3))
    d[:, axis] = np.linspace(-angle / 2, angle / 2, n)
    return motion(d, readouts)


def seeded_motion(rng, n, scale=2.0):
    return motion(rng.uniform(-scale, scale, (n, 3)), [tuple(rng.uniform([-1, -1, -0.5], [1, 1, 0.5])) for _ in range(2)])


def same(a, b):
    """Bit for bit, NaNs included."""
    return a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def turned_rig(rig, delta):
    """rig with every lens's extrinsic rotation R turned to Rot(delta) R, as Euler angles (yaw, pitch, roll)."""
    out = t360.T360LensRig(rig.numLenses, rig.calibWidth, rig.calibHeight)
    for i in range(rig.numLenses):
        L = rig.lens[i]
        r = _rot(*delta) @ _rot(L.yaw, L.pitch, L.roll)
        b = np.arcsin(-r[1, 2])
        yaw, roll = np.degrees(np.arctan2(r[0, 2], r[2, 2])), np.degrees(np.arctan2(r[1, 0], r[1, 1]))
        out.lens[i] = t360.T360Lens(L.fx, L.fy, L.cx, L.cy, tuple(L.k), yaw, -np.degrees(b), roll, L.maxAngle)
    return out


# ---- no GPU needed -----------------------------------------------------------------------------------------------------
def test_entry_points_are_exported_with_their_bindings(tmp_path):
    from transform360_b200.handler import EXPORTED_SYMBOLS, LIB_PATH, PKG
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    names = ("T360B200_lensMotionMaps", "T360B200_transformFrameLensMotionAsync", "T360B200_cameraMotionMaps",
             "T360B200_transformFrameCameraMotionAsync")
    for name in names:
        assert name in EXPORTED_SYMBOLS and name in defined, name
    L, P = t360.load(), C.POINTER
    assert L.T360B200_lensMotionMaps.argtypes == ([P(t360.FrameTransformContext), P(t360.T360LensRig), P(t360.T360RigPhotometry), C.c_float,
                                                   P(t360.T360Orientation), P(t360.T360RigMotion)] + [C.c_int] * 5 + [C.c_void_p] * 5)
    assert L.T360B200_transformFrameLensMotionAsync.argtypes == ([C.c_void_p, P(t360.T360LensRig), P(t360.T360RigPhotometry), C.c_float,
                                                                  P(t360.T360Orientation), P(t360.T360RigMotion), C.c_void_p, C.c_int]
                                                                 + [C.c_void_p] * 9)
    assert L.T360B200_cameraMotionMaps.argtypes == ([P(t360.FrameTransformContext), P(t360.T360LensRig), P(t360.T360RigPhotometry), C.c_float,
                                                     P(t360.T360Pose), P(t360.T360Camera), P(t360.T360Minify), P(t360.T360RigMotion)]
                                                    + [C.c_int] * 6 + [C.c_void_p] * 6)
    assert L.T360B200_transformFrameCameraMotionAsync.argtypes == ([C.c_void_p, P(t360.T360LensRig), P(t360.T360RigPhotometry), C.c_float,
                                                                    P(t360.T360Pose), P(t360.T360Camera), P(t360.T360Minify),
                                                                    P(t360.T360RigMotion), C.c_void_p, C.c_int] + [C.c_void_p] * 9)
    assert C.sizeof(t360.T360LensReadout) == 12 and C.sizeof(t360.T360RigMotion) == 220
    assert t360.T360RigMotion.delta.offset == 4 and t360.T360RigMotion.readout.offset == 196
    for m in ("make_lens_motion_frame_call", "make_camera_motion_frame_call"):
        assert hasattr(t360.VideoFrameTransform, m)
    assert callable(t360.lens_motion_maps) and callable(t360.camera_motion_maps)
    src = tmp_path / "decl.c"
    src.write_text('#include <stddef.h>\n#include "transform360_b200.h"\n'
                   "_Static_assert(sizeof(T360LensReadout) == 12 && sizeof(T360RigMotion) == 220 && offsetof(T360RigMotion, delta) == 4 && "
                   "offsetof(T360RigMotion, readout) == 196, \"layout\");\n"
                   "int (*lm)(const FrameTransformContext*, const T360LensRig*, const T360RigPhotometry*, float, const T360Orientation*, "
                   "const T360RigMotion*, int, int, int, int, int, float*, float*, uint16_t*, uint16_t*, uint16_t*) = T360B200_lensMotionMaps;\n"
                   "int (*lf)(VideoFrameTransform*, const T360LensRig*, const T360RigPhotometry*, float, const T360Orientation*, const T360RigMotion*, "
                   "unsigned long long*, int, const uint8_t* const*, uint8_t* const*, const int*, const int*, const int*, const int*, "
                   "const int*, const int*, void*) = T360B200_transformFrameLensMotionAsync;\n"
                   "int (*cm)(const FrameTransformContext*, const T360LensRig*, const T360RigPhotometry*, float, const T360Pose*, const T360Camera*, "
                   "const T360Minify*, const T360RigMotion*, int, int, int, int, int, int, float*, float*, uint8_t*, uint16_t*, uint16_t*, "
                   "uint16_t*) = T360B200_cameraMotionMaps;\n"
                   "int (*cf)(VideoFrameTransform*, const T360LensRig*, const T360RigPhotometry*, float, const T360Pose*, const T360Camera*, "
                   "const T360Minify*, const T360RigMotion*, unsigned long long*, int, const uint8_t* const*, uint8_t* const*, const int*, "
                   "const int*, const int*, const int*, const int*, const int*, void*) = T360B200_transformFrameCameraMotionAsync;\n")
    subprocess.run(["cc", "-std=c11", "-Wall", "-Werror", "-c", "-I", str(PKG.parent / "include"), "-o", str(tmp_path / "decl.o"), str(src)],
                   check=True)


# (rig, seamWidth): one lens, the hard seam of two, the feathered seam
MODES = {"one": ("single_200", 0.0), "hard": ("pair_190", 0.0), "feathered": ("tilted", 8.0)}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_zero_deltas_are_the_photometric_lens_twin(layout):
    """All-zero deltas, any readout and sample count: every array of lens_motion_maps is lens_photo_maps', bit for bit (-0
    entries of the lens matrices included), with 1- and 2-lens rigs, both seams and a non-identity photometry."""
    rng = np.random.default_rng(len(layout))
    for mode, (rig_name, seam) in sorted(MODES.items()):
        rig = make_rig(rig_name, seed=len(layout) + len(mode))
        for ph_name, ph in sorted(rig_photos(rig).items()):
            o = _orientations(len(layout) + len(ph_name), 1)[0]
            n = int(rng.integers(2, 17))
            readouts = [tuple(rng.uniform(-3, 3, 3)) for _ in range(2)]
            ctx = t360.make_context(output_layout=LAYOUTS[layout], interpolation_alg=t360.CUBIC, **LENS_CTX)
            for plane, (in_w, in_h), (w, h) in ((0, (259, 131), (97, 65)), (1, (130, 66), (49, 33))):
                want = t360.lens_photo_maps(ctx, rig, ph, seam, o, plane, in_w, in_h, w, h)
                got = t360.lens_motion_maps(ctx, rig, ph, seam, o, zero_motion(n, readouts), plane, in_w, in_h, w, h)
                for a, b in zip(got, want):
                    assert same(a, b), (layout, mode, ph_name, plane)


@pytest.mark.parametrize("model", sorted(MODELS))
def test_zero_deltas_are_the_photometric_camera_twin(model):
    """All-zero deltas: camera_motion_maps is camera_photo_maps bit for bit, every camera model, with and without a
    pyramid, 1- and 2-lens rigs, hard and feathered seams, both lenses."""
    rng = np.random.default_rng(len(model) + 5)
    for rig_name in ("single_200", "pair_190"):
        rig = make_rig(rig_name, seed=len(model))
        ph = rig_photos(rig)["falloff"]
        ctx = _ctx(rig_name, t360.CUBIC)
        for seam in ((0.0,) if rig.numLenses == 1 else (0.0, 4.0)):
            for k, minify in enumerate((None, (3, 0.0), (4, 1.0))):
                pose, cam = seam_pose(MODELS[model], 3 * k + len(rig_name))
                mo = zero_motion(int(rng.integers(2, 17)), [tuple(rng.uniform(-3, 3, 3)) for _ in range(2)])
                for lens in (0, 1):
                    want = t360.camera_photo_maps(ctx, rig, ph, seam, pose, cam, minify, lens, 0, 400, 200, 97, 65)
                    got = t360.camera_motion_maps(ctx, rig, ph, seam, pose, cam, minify, mo, lens, 0, 400, 200, 97, 65)
                    for a, b in zip(got, want):
                        assert same(a, b), (model, rig_name, seam, minify, lens)


def test_constant_delta_turns_the_rig():
    """delta_k = delta for every k is the rig whose lens extrinsics are turned by delta: the entries agree with the
    photometric twin of that rig within float rounding (1e-4 px), wherever both cover the pixel."""
    worst = 0.0
    for rig_name in ("single_200", "pair_190", "tilted"):
        rig = make_rig(rig_name, seed=4)
        for delta in ((2.0, -1.5, 1.0), (-7.0, 4.0, -3.0)):
            ctx = t360.make_context(output_layout=t360.LAYOUT_EQUIRECT, interpolation_alg=t360.CUBIC, **LENS_CTX)
            o = (20.0, 5.0, -3.0)
            got = t360.lens_motion_maps(ctx, rig, IDENTITY, 0.0, o, motion([delta] * 5, [(0.3, 0.7, 0.0)] * 2), 0, 259, 131, 360, 180)
            want = t360.lens_photo_maps(ctx, turned_rig(rig, delta), IDENTITY, 0.0, o, 0, 259, 131, 360, 180)
            for a, b in ((got[0], want[0]), (got[1], want[1]))[:rig.numLenses]:
                both = np.isfinite(a).all(-1) & np.isfinite(b).all(-1)
                assert both.sum() > 1000
                worst = max(worst, float(np.abs(a[both] - b[both]).max()))
    print(f"constant delta: max |entry - turned rig's entry| {worst:.2e} px")
    assert worst <= 1e-4


def _lens_2880(right_half=False):
    """One equidistant-like 200-degree lens about 2880 rows high (a 5.7K dual-fisheye sensor's lens), mild distortion;
    right_half: the lens of the right half of a 5760 x 2880 side-by-side frame."""
    rig = t360.T360LensRig(1, 5760 if right_half else 2880, 2880)
    th = np.radians(100.0)
    k = (0.01, -0.002, 0.0005, 0.0)
    f = 1440 / (th * (1 + k[0] * th ** 2 + k[1] * th ** 4 + k[2] * th ** 6 + k[3] * th ** 8))
    rig.lens[0] = t360.T360Lens(f, f, 4319.5 if right_half else 1439.5, 1439.5, k, 0.0, 0.0, 0.0, 100.0)
    return rig


def motion_model64(rig, mo, d, in_w, in_h, iterations=60):
    """The contract in float64 for lens 0 with the fixed point solved to convergence: the sample matrices Rot(delta_k) R
    in float64, M(t) interpolated entry by entry, t = clamp(a u + b v + c, 0, 1).  Returns (px, py, theta, t)."""
    L, n = rig.lens[0], mo.numSamples
    R = _rot(L.yaw, L.pitch, L.roll)
    Ms = np.stack([(_rot(mo.delta[k].yaw, mo.delta[k].pitch, mo.delta[k].roll) @ R).T * np.array([[1.0], [-1.0], [1.0]]) for k in range(n)])
    a, b, c = (np.float64(np.float32(x)) for x in (mo.readout[0].a, mo.readout[0].b, mo.readout[0].c))
    kk = [np.float64(np.float32(x)) for x in L.k]
    t = np.full(d.shape[:-1], 0.5)

    def project(t):
        s = t * (n - 1)
        k = np.minimum(np.floor(s), n - 2).astype(int)
        f = (s - k)[..., None, None]
        M = Ms[k] + f * (Ms[k + 1] - Ms[k])
        cam = np.einsum("...ij,...j->...i", M, d)
        X, Y, Z = cam[..., 0], cam[..., 1], cam[..., 2]
        rho = np.hypot(X, Y)
        th = np.arctan2(rho, Z)
        q = th * th
        sc = np.where(rho > 0, th * (1 + q * (kk[0] + q * (kk[1] + q * (kk[2] + q * kk[3])))) / np.where(rho > 0, rho, 1), 0.0)
        u = (L.fx * sc * X + L.cx + 0.5) / rig.calibWidth
        v = (L.fy * sc * Y + L.cy + 0.5) / rig.calibHeight
        return u, v, th
    for _ in range(iterations):
        u, v, th = project(t)
        t = np.clip(a * u + b * v + c, 0.0, 1.0)
    u, v, th = project(t)
    return u * in_w - 0.5, v * in_h - 0.5, th, t


def test_twin_against_the_float64_fixed_point():
    """1, 3 and 6 degrees of turn across the readout (yaw, pitch and roll), row, column, reversed and half-frame readouts
    (the half-frame one on the right lens of a side-by-side frame), on a lens about 2880 rows high: the twin's entries
    against the float64 model solved to convergence.  At 3 degrees the error stays within 0.02 px; the maxima are
    printed (the float chain alone gives about 0.007 px on the pole rows)."""
    ctx = t360.make_context(output_layout=t360.LAYOUT_EQUIRECT, interpolation_alg=t360.CUBIC, **LENS_CTX)
    w, h = 360, 180
    d, dead = directions(dict(output_layout=t360.LAYOUT_EQUIRECT), (0.0, 0.0, 0.0), w, h)
    worst = {}
    for angle in (1.0, 3.0, 6.0):
        for name, r in sorted(READOUTS.items()):
            rig = _lens_2880(right_half=name == "half")
            in_w, in_h = rig.calibWidth, rig.calibHeight
            for axis in (0, 1, 2):
                mo = sweep(9, angle, axis, (r, r))
                m0 = t360.lens_motion_maps(ctx, rig, IDENTITY, 0.0, (0.0, 0.0, 0.0), mo, 0, in_w, in_h, w, h)[0].astype(np.float64)
                px, py, th, _ = motion_model64(rig, mo, d, in_w, in_h)
                sel = (th < np.radians(100.0) - 0.06) & ~dead  # (clear of the rim by more than the turn: every projection covers)
                assert np.isfinite(m0[sel]).all()
                err = np.hypot(m0[..., 0] - px, m0[..., 1] - py)[sel]
                worst[(angle, name)] = max(worst.get((angle, name), 0.0), float(err.max()))
    for k, v in sorted(worst.items()):
        print(f"{k[0]:.0f} degrees, {k[1]} readout: max error {v:.4f} px")
    assert max(v for (a, _), v in worst.items() if a == 3.0) <= 0.02, worst


def _render_rolling(rig, in_w, in_h, scene, turn):
    """A dual-fisheye luma plane of an equidistant rig (k = 0) read top to bottom while the rig turns by `turn` degrees
    of yaw across the readout (centred): each source pixel's ray, turned by the rig's orientation at its own row's readout
    time t = v (u, v its normalised calibration coordinates), shows scene(d), in float64 and rounded."""
    y, x = np.mgrid[:in_h, :in_w].astype(np.float64)
    out = np.zeros((in_h, in_w))
    v = ((y + 0.5) * rig.calibHeight / in_h) / rig.calibHeight  # = (fy y' + cy + 0.5) / calibHeight
    for i in range(2):
        L = rig.lens[i]
        xp = ((x + 0.5) * rig.calibWidth / in_w - 0.5 - L.cx) / L.fx
        yp = ((y + 0.5) * rig.calibHeight / in_h - 0.5 - L.cy) / L.fy
        r = np.hypot(xp, yp)
        inside = (r <= np.radians(L.maxAngle)) & ((x < in_w / 2) if i == 0 else (x >= in_w / 2))
        s = np.where(r > 0, np.sin(r) / np.where(r > 0, r, 1), 1.0)
        cam = np.stack([xp * s, -yp * s, np.cos(r)], -1)
        yaw = np.radians(turn * (v - 0.5))
        d = cam @ _rot(L.yaw, L.pitch, L.roll).T
        dx = np.cos(yaw) * d[..., 0] + np.sin(yaw) * d[..., 2]
        dz = -np.sin(yaw) * d[..., 0] + np.cos(yaw) * d[..., 2]
        d = np.stack([dx, d[..., 1], dz], -1)
        out[inside] = scene(d)[inside]
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


def test_synthetic_rolling_shutter_frame_is_corrected():
    """A dual-fisheye frame of a textured scene rendered through a float64 rolling-shutter model (3 degrees of yaw across
    a top-to-bottom readout), corrected to EQUIRECT with lens_motion_maps and the oracle composite, against the still
    frame's rendering: the mean absolute error over covered pixels is at least 4x lower than without the correction
    (lens_photo_maps).  The ratio is printed."""
    rig = equidistant_pair()
    in_w, in_h, w, h = 2000, 1000, 720, 360
    tex = synth.scene_plane(1440, 720).astype(np.float64)

    def scene(d):  # the texture on the sphere, bilinear
        lon, lat = np.arctan2(d[..., 0], d[..., 2]), np.arcsin(np.clip(d[..., 1] / np.linalg.norm(d, axis=-1), -1, 1))
        fx, fy = (lon / (2 * np.pi) + 0.5) * 1440 - 0.5, (0.5 - lat / np.pi) * 720 - 0.5
        x0, y0 = np.floor(fx).astype(int), np.floor(fy).astype(int)
        ax, ay = fx - x0, fy - y0
        g = lambda yy, xx: tex[np.clip(yy, 0, 719), xx % 1440]
        return (g(y0, x0) * (1 - ax) + g(y0, x0 + 1) * ax) * (1 - ay) + (g(y0 + 1, x0) * (1 - ax) + g(y0 + 1, x0 + 1) * ax) * ay
    still, moving = _render_rolling(rig, in_w, in_h, scene, 0.0), _render_rolling(rig, in_w, in_h, scene, 3.0)
    ctx = t360.make_context(output_layout=t360.LAYOUT_EQUIRECT, interpolation_alg=t360.LINEAR, **LENS_CTX)
    o = (0.0, 0.0, 0.0)
    prefill = np.zeros((h, w), np.uint8)
    plain = t360.lens_photo_maps(ctx, rig, IDENTITY, 0.0, o, 0, in_w, in_h, w, h)
    mo = sweep(5, 3.0, 0, ((0.0, 1.0, 0.0), (0.0, 1.0, 0.0)))
    corrected = t360.lens_motion_maps(ctx, rig, IDENTITY, 0.0, o, mo, 0, in_w, in_h, w, h)
    ref = photo_composite(still, plain, t360.LINEAR, prefill, IDENTITY, 0)[0].astype(np.float64)
    before = photo_composite(moving, plain, t360.LINEAR, prefill, IDENTITY, 0)[0].astype(np.float64)
    after = photo_composite(moving, corrected, t360.LINEAR, prefill, IDENTITY, 0)[0].astype(np.float64)
    cov = np.isfinite(np.where(plain[2][..., None] == 256, plain[1], plain[0])).all(-1)
    cov[:8] = cov[-8:] = False  # (the poles' rows: a few source pixels spread over a whole row)
    mae_before, mae_after = np.abs(before - ref)[cov].mean(), np.abs(after - ref)[cov].mean()
    print(f"rolling shutter, 3 degrees: MAE {mae_before:.3f} uncorrected, {mae_after:.3f} corrected, ratio {mae_before / mae_after:.1f}")
    assert mae_before >= 4 * mae_after, (mae_before, mae_after)


def _bad_motions(rig):
    """(what, motion or None) the calls refuse, for a usable rig."""
    cases = [("NULL motion", None)]
    for n in (0, 1, 17, -3):
        m = zero_motion(2)
        m.numSamples = n
        cases.append((f"numSamples {n}", m))
    for k, field, value in ((0, "yaw", float("nan")), (1, "pitch", float("inf")), (1, "roll", 30.5), (0, "yaw", -31.0)):
        m = zero_motion(3)
        setattr(m.delta[k], field, value)
        cases.append((f"delta[{k}].{field} {value}", m))
    for lens in range(rig.numLenses):
        for field in ("a", "b", "c"):
            m = zero_motion(2)
            setattr(m.readout[lens], field, float("nan"))
            cases.append((f"readout[{lens}].{field} nan", m))
    return cases


def test_refusals_happen_without_a_gpu(capfd):
    """Every motion refusal comes with its message, after every refusal of the call extended, and before any CUDA call
    (bogus device pointers are never dereferenced, no kernel is launched).  A one-lens rig does not read readout[1], and
    deltas of +-30 degrees and delta entries past numSamples are accepted."""
    L = t360.load()
    pair, single = make_rig("pair_190"), make_rig("single_200")
    lens_ctx = t360.make_context(output_layout=t360.LAYOUT_EQUIRECT, **LENS_CTX)
    cam_ctx = t360.make_context(**RECT_CTX)
    m0, m1 = np.zeros((8, 8, 2), np.float32), np.zeros((8, 8, 2), np.float32)
    u8, u16 = np.zeros((8, 8), np.uint8), [np.zeros((8, 8), np.uint16) for _ in range(3)]
    lens_arrays = (m0.ctypes.data, m1.ctypes.data, *(a.ctypes.data for a in u16))
    cam_arrays = (m0.ctypes.data, m1.ctypes.data, u8.ctypes.data, *(a.ctypes.data for a in u16))
    P, I = C.c_void_p * 3, C.c_int * 3
    arr = lambda v: I(*([v] * 3))
    planes = lambda: (1, P(0x20000, 0, 0), P(0x20000, 0, 0), arr(64), arr(32), arr(64), arr(8), arr(8), arr(8), None)
    pose, cam = C.byref(t360.T360Pose(80.0, 5.0, 0.0, 90.0, 60.0)), C.byref(t360.T360Camera(EQUIDISTANT, 0.0))
    o = C.byref(t360.T360Orientation())
    n0 = t360.kernel_launch_count()
    messages = {}
    with t360.VideoFrameTransform(lens_ctx) as lv, t360.VideoFrameTransform(cam_ctx) as cv:
        for rig in (pair, single):
            for what, mo in _bad_motions(rig):
                mb = C.byref(mo) if mo is not None else None
                out = _refused(capfd, L.T360B200_lensMotionMaps, C.byref(lens_ctx), C.byref(rig), C.byref(IDENTITY), 0.0, o, mb, 0, 64, 32, 8, 8,
                               *lens_arrays)
                assert "Could not compute the lens motion maps" in out, what
                messages[what] = out.split("Error: ")[-1].strip()
                out = _refused(capfd, L.T360B200_transformFrameLensMotionAsync, lv._h, C.byref(rig), C.byref(IDENTITY), 0.0, o, mb, 0x40000,
                               *planes())
                assert out.split("Error: ")[-1].strip() == messages[what], what
                out = _refused(capfd, L.T360B200_cameraMotionMaps, C.byref(cam_ctx), C.byref(rig), C.byref(IDENTITY), 0.0, pose, cam, None, mb, 0,
                               0, 64, 32, 8, 8, *cam_arrays)
                assert out.split("Error: ")[-1].strip() == messages[what], what
                out = _refused(capfd, L.T360B200_transformFrameCameraMotionAsync, cv._h, C.byref(rig), C.byref(IDENTITY), 0.0, pose, cam, None, mb,
                               0x40000, *planes())
                assert out.split("Error: ")[-1].strip() == messages[what], what
        assert messages["NULL motion"] == "a NULL motion" and "numSamples 17" in messages["numSamples 17"]
        assert "delta[1]" in messages["delta[1].roll 30.5"] and "readout of lens 1" in messages["readout[1].a nan"]
        # the rungs come after every refusal of the calls extended: their messages win over a bad motion's
        bad = zero_motion(1)
        for what, call in (("seam", lambda: t360.lens_motion_maps(lens_ctx, pair, IDENTITY, 0.005, (0, 0, 0), bad, 0, 64, 32, 8, 8)),
                           ("orientation", lambda: t360.lens_motion_maps(lens_ctx, pair, IDENTITY, 0.0, (float("nan"), 0, 0), bad, 0, 64, 32, 8, 8)),
                           ("photometry gain", lambda: t360.lens_motion_maps(lens_ctx, pair, t360.T360RigPhotometry(16), 0.0, (0, 0, 0), bad, 0, 64, 32,
                                                                             8, 8)),
                           ("pose", lambda: t360.camera_motion_maps(cam_ctx, pair, IDENTITY, 0.0, (0, 0, 0, 200.0, 60.0), PINHOLE, None, bad, 0, 0, 64,
                                                                    32, 8, 8)),
                           ("minify", lambda: t360.camera_motion_maps(cam_ctx, pair, IDENTITY, 0.0, (0, 0, 0, 90.0, 60.0), PINHOLE, (9, 0.0), bad, 0,
                                                                      0, 64, 32, 8, 8))):
            with pytest.raises(ValueError):
                call()
            out = _stdout(capfd)
            assert "Error" in out and "numSamples" not in out, (what, out)
        # the twins' own array and index checks come after the motion's
        assert "numSamples" in _refused(capfd, L.T360B200_lensMotionMaps, C.byref(lens_ctx), C.byref(pair), C.byref(IDENTITY), 0.0, o, C.byref(bad),
                                        7, 64, 32, 8, 8, *lens_arrays)
        assert "plane 7" in _refused(capfd, L.T360B200_lensMotionMaps, C.byref(lens_ctx), C.byref(pair), C.byref(IDENTITY), 0.0, o,
                                     C.byref(zero_motion(2)), 7, 64, 32, 8, 8, *lens_arrays)
        assert "NULL photometry" in _refused(capfd, L.T360B200_transformFrameLensMotionAsync, lv._h, C.byref(pair), None, 0.0, o, None, 0x40000,
                                             *planes())
        assert not L.T360B200_transformFrameLensMotionAsync(None, None, None, 0.0, None, None, None, 1, *([None] * 9))
        assert not L.T360B200_transformFrameCameraMotionAsync(None, None, None, 0.0, None, None, None, None, None, 1, *([None] * 9))
    assert t360.kernel_launch_count() == n0
    # accepted: readout[1] of a one-lens rig, +-30 degrees, junk past numSamples
    mo = motion([(30.0, -30.0, 30.0), (-30.0, 30.0, -30.0)], [(0, 1, 0), (float("nan"), 0, 0)])
    mo.delta[5].yaw = float("nan")
    t360.lens_motion_maps(lens_ctx, single, IDENTITY, 0.0, (0, 0, 0), mo, 0, 64, 32, 8, 8)
    t360.camera_motion_maps(cam_ctx, single, IDENTITY, 0.0, (0, 0, 0, 90.0, 60.0), PINHOLE, None, mo, 0, 0, 64, 32, 8, 8)


# ---- the twin gate (tests/motion_twin_gate.cu on tests/twin_gate.cuh) --------------------------------------------------
GATE_PROBES = ("motionLens", "lensMotionPosition", "lensMotionSample<BARREL>", "lensMotionSample<plain>", "cameraMotionSample<plain>",
               "cameraMotionSample<MIP>")
GATE_CLASSES = {("lensMotionPosition", c) for c in ("clampedAt0", "clampedAt1", "coveredThenUncovered", "segmentBoundary", "hard", "feathered",
                                                    "bothLenses")}


@pytest.fixture(scope="module")
def motion_gate(tmp_path_factory):
    exe = tmp_path_factory.mktemp("motion_twin_gate") / "motion_twin_gate"
    r = subprocess.run(gate_command("motion_twin_gate", exe), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return "motion_twin_gate", exe


def test_gate_builds_for_sm_90a_with_the_library_flags(motion_gate):
    from transform360_b200 import build as b
    cmd = gate_command(*motion_gate)
    assert cmd[cmd.index("-Xcompiler") + 1] == b.HOST_FLAGS and "arch=compute_90a,code=sm_90a" in cmd and "-O3" in cmd
    import os
    elf = subprocess.run([os.path.join(os.path.dirname(b.nvcc_path()), "cuobjdump"), "--list-elf", str(motion_gate[1])], capture_output=True,
                         text=True, check=True).stdout
    assert "sm_90a" in elf


def test_gate_host_half_does_not_depend_on_the_thread_count(motion_gate):
    fp = lambda out: [line for line in out.splitlines() if line.startswith("fingerprint ")]
    one = fp(run(motion_gate, "--host-only", "--threads", "1").stdout)
    many = fp(run(motion_gate, "--host-only", "--threads", str(THREADS)).stdout)
    assert [line.split()[1] for line in one] == list(GATE_PROBES) and one == many


def test_gate_self_test_reports_exactly_the_flipped_element(motion_gate):
    r = run(motion_gate, "--self-test", "--threads", str(THREADS), check=False)
    assert r.returncode == 1, r.stdout + r.stderr
    flipped = re.search(r"self-test: flipped (\S+) (\d+) word (\d) bit (\d)", r.stdout)
    assert flipped, r.stdout
    reports = [line.split() for line in r.stdout.splitlines() if len(line.split()) == 5 and not line.startswith("self-test")]
    assert len(reports) == 1 and (reports[0][0], int(reports[0][1])) == (flipped.group(1), int(flipped.group(2))), r.stdout
    h, o = [int(x, 16) for x in reports[0][3].split(":")], [int(x, 16) for x in reports[0][4].split(":")]
    word, bit = int(flipped.group(3)), int(flipped.group(4))
    assert [x ^ y for x, y in zip(h, o)] == [(1 << bit) if k == word else 0 for k in range(len(h))]
    assert r.stdout.strip().splitlines()[-1].endswith(" 1 mismatches"), r.stdout


def test_gate_ledger_reaches_every_class(motion_gate):
    """The interpolation reaches t = 0, t = 1 and inner segment boundaries; lensMotionPosition reaches t clamped at 0 and
    at 1, the first projection covered with the last one not (the converse cannot happen: an uncovered projection keeps
    t), a projection on a segment boundary, the hard seam, both lenses and the feathered seam."""
    counts = {}
    for line in run(motion_gate, "--ledger", "--threads", str(THREADS)).stdout.splitlines():
        _, probe, cls, n = line.split()
        counts[(probe, cls)] = int(n)
    missed = sorted(k for k, n in counts.items() if n == 0)
    assert not missed, missed
    assert GATE_CLASSES <= set(counts), counts
    assert {("motionLens", c) for c in ("t0", "t1", "boundary")} <= set(counts), counts


# ---- on the GPU --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests must run on an H100 (there is no CPU fallback to test)")
    return torch


@pytest.mark.gpu
def test_gate_device_twins_equal_the_host_twins(motion_gate):
    r = run(motion_gate, "--threads", str(THREADS), check=False)
    print(r.stdout)
    m = re.fullmatch(r"(\d+) probes, (\d+) inputs, (\d+) mismatches", r.stdout.strip().splitlines()[-1])
    assert m and r.returncode == 0 and m.group(3) == "0", r.stdout + r.stderr


def want_motion(f, ctx, rig, ph, seam, o, mo):
    """The oracle's planes of Frame f and the statistics per plane: photo_composite of lens_motion_maps' arrays."""
    want, sums = [], []
    for p in range(f.n):
        maps = t360.lens_motion_maps(ctx, rig, ph, seam, o, mo, p, *IN_DIMS[p], *OUT_DIMS[p])
        prefill = _pattern(*OUT_DIMS[p], p) if p == 0 else np.full(OUT_DIMS[p][::-1], 128, np.uint8)
        out, s = photo_composite(f.src[p], maps, ctx.interpolation_alg, prefill, ph, p)
        want.append(out)
        sums.append(s)
    return want, sums


def camera_motion_want(monkeypatch, mo, *args):
    """test_camera_photo.photo_want with camera_motion_maps' arrays in place of camera_photo_maps'."""
    def twin(ctx, rig, ph, seam, pose, cam, minify, plane, in_w, in_h, w, h):
        out = [t360.camera_motion_maps(ctx, rig, ph, seam, pose, cam, minify, mo, lens, plane, in_w, in_h, w, h) for lens in (0, 1)]
        assert np.array_equal(out[0][5], out[1][5])
        return [x[:5] for x in out], out[0][5]
    with monkeypatch.context() as m:
        m.setattr(camera_photo, "twin", twin)
        return photo_want(*args)


def _lens_call(vft, f):
    return vft.make_lens_motion_frame_call(f.in_planes, f.out_planes, f.dims)


def _camera_call(vft, f):
    return vft.make_camera_motion_frame_call(f.in_planes, f.out_planes, f.dims)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("interp", INTERPS)
def test_lens_frames_and_statistics_equal_the_oracle(layout, interp, torch_cuda):
    """One lens, the hard seam of two and the feathered seam, seeded motions and readouts, a non-identity photometry:
    3-plane frames equal the oracle composite of lens_motion_maps bit for bit, with and without statistics, and the
    statistics its int64 sums."""
    torch = torch_cuda
    ctx = t360.make_context(output_layout=LAYOUTS[layout], interpolation_alg=interp, **LENS_CTX)
    vft = t360.VideoFrameTransform(ctx)
    st = torch.cuda.Stream()
    stats = torch.zeros((3, STATS), dtype=torch.int64, device="cuda")
    rng = np.random.default_rng(interp * 10 + len(layout))
    for m, (mode, (rig_name, seam)) in enumerate(sorted(MODES.items())):
        rig = make_rig(rig_name, seed=interp + 3 * m)
        o = _orientations(interp * 10 + len(layout) + m, 1)[0]
        ph = rig_photos(rig)["falloff"]
        mo = seeded_motion(rng, int(rng.integers(2, 17)))
        f = Frame(torch, 3, seed=interp + m)
        want, sums = want_motion(f, ctx, rig, ph, seam, o, mo)
        for with_stats in (False, True):
            f.reset()
            stats.fill_(-1)
            torch.cuda.synchronize()
            assert _lens_call(vft, f)(rig, ph, seam, o, mo, st.cuda_stream, stats.data_ptr() if with_stats else 0)
            st.synchronize()
            for p, got in enumerate(f.host()):
                _check(got, want[p], f"{mode}, statistics {with_stats}, plane {p}")
            got_sums = stats.cpu().numpy()
            if with_stats:
                for p in range(3):
                    assert got_sums[p].tolist() == sums[p], f"{mode}: plane {p} statistics"
            else:
                assert (got_sums == -1).all()
    vft.close()


@pytest.mark.gpu
@pytest.mark.parametrize("model", sorted(MODELS))
def test_camera_frames_and_statistics_equal_the_oracle(model, torch_cuda, monkeypatch):
    """Both rigs, hard and feathered seams, no pyramid and two pyramids, seeded motions: 3-plane frames and statistics equal
    the oracle composite of camera_motion_maps, every interpolator."""
    torch = torch_cuda
    stats = torch.zeros((3, STATS), dtype=torch.int64, device="cuda")
    rng = np.random.default_rng(len(model) + 77)
    for interp in INTERPS:
        ctx = _ctx("pair_190", interp)
        vft = t360.VideoFrameTransform(ctx)
        for name in ("single_200", "pair_190"):
            rig = make_rig(name, seed=interp + len(model))
            ph = rig_photos(rig)["falloff"]
            for seam in ((0.0,) if rig.numLenses == 1 else (0.0, 4.0)):
                for k, minify in enumerate((None, (3, 0.0), (4, 1.0))):
                    if (k + interp + int(seam)) % 2 and minify is not None:
                        continue
                    pose, cam = seam_pose(MODELS[model], 31 * interp + 7 * k + len(name))
                    mo = seeded_motion(rng, int(rng.integers(2, 17)))
                    f = MipFrame(torch, name, 3, seed=interp + k)
                    want, sums = camera_motion_want(monkeypatch, mo, ctx, rig, ph, seam, pose, cam, minify, f.src, f.out_dims, f.prefill)
                    for p, o in enumerate(f.outs):
                        o[:, :f.out_dims[p][0]] = torch.from_numpy(f.prefill[p]).cuda()
                    stats.fill_(-1)
                    torch.cuda.synchronize()
                    assert _camera_call(vft, f)(rig, ph, seam, pose, cam, minify, mo, 0, stats.data_ptr())
                    torch.cuda.synchronize()
                    what = f"{name} interp {interp} seam {seam} minify {minify}"
                    for p, got in enumerate(f.host()):
                        _check(got, want[p], f"{what}, plane {p}")
                        assert stats[p].cpu().tolist() == sums[p], f"{what}: plane {p} statistics"
        vft.close()


@pytest.mark.gpu
def test_zero_deltas_equal_the_photometric_calls(torch_cuda):
    """All-zero deltas on a 1440x720 dual-fisheye yuv420p frame: the lens-motion call gives the lens-photo call's frame
    and statistics byte for byte (every sphere layout, both seams), the camera-motion call the camera-photo call's (every
    model, with and without a pyramid); the launches are the same."""
    torch = torch_cuda
    rig = make_rig("pair_190", seed=5)
    dims = [(1440, 720, 384, 256), (720, 360, 192, 128), (720, 360, 192, 128)]
    src = [torch.from_numpy(synth.noise_plane(w, h, p, 3)).cuda() for p, (w, h, _, _) in enumerate(dims)]
    outs = [[torch.full((oh, ow), 7 + p, dtype=torch.uint8, device="cuda") for p, (_, _, ow, oh) in enumerate(dims)] for _ in range(2)]
    planes = lambda ts: [(t.data_ptr(), t.stride(0)) for t in ts]
    stats = [torch.zeros((3, STATS), dtype=torch.int64, device="cuda") for _ in range(2)]
    ph = rig_photos(rig)["falloff"]
    mo = zero_motion(7, ((0.3, 0.9, -0.1), (-1.0, 0.5, 0.7)))

    def compare(what, run_a, run_b):
        for a, b in zip(*outs):
            a.fill_(9)
            b.fill_(9)
        torch.cuda.synchronize()
        n0 = t360.kernel_launch_count()
        assert run_a()
        n1 = t360.kernel_launch_count()
        assert run_b()
        torch.cuda.synchronize()
        assert n1 - n0 == t360.kernel_launch_count() - n1, what
        for p, (a, b) in enumerate(zip(*outs)):
            assert torch.equal(a, b), f"{what}, plane {p}: {int((a != b).sum())} bytes differ"
        assert torch.equal(stats[0], stats[1]), what
    for layout in sorted(LAYOUTS):
        ctx = t360.make_context(output_layout=LAYOUTS[layout], interpolation_alg=t360.CUBIC, **LENS_CTX)
        with t360.VideoFrameTransform(ctx) as vft:
            a = vft.make_lens_motion_frame_call(planes(src), planes(outs[0]), dims)
            b = vft.make_lens_photo_frame_call(planes(src), planes(outs[1]), dims)
            for seam, o in ((0.0, (20.0, 5.0, -3.0)), (6.0, (-70.0, 10.0, 2.0))):
                compare(f"{layout} seam {seam}", lambda: a(rig, ph, seam, o, mo, 0, stats[0].data_ptr()),
                        lambda: b(rig, ph, seam, o, 0, stats[1].data_ptr()))
    with t360.VideoFrameTransform(_ctx("pair_190", t360.LANCZOS4)) as vft:
        a = vft.make_camera_motion_frame_call(planes(src), planes(outs[0]), dims)
        b = vft.make_camera_photo_frame_call(planes(src), planes(outs[1]), dims)
        for model in sorted(MODELS):
            pose, cam = seam_pose(MODELS[model], len(model))
            for minify in (None, (3, 0.0)):
                for seam in (0.0, 4.0):
                    compare(f"{model} minify {minify} seam {seam}", lambda: a(rig, ph, seam, pose, cam, minify, mo, 0, stats[0].data_ptr()),
                            lambda: b(rig, ph, seam, pose, cam, minify, 0, stats[1].data_ptr()))


@pytest.mark.gpu
def test_trajectory_on_two_streams_and_bounded_memory(torch_cuda, monkeypatch):
    """A motion, orientation and seam that change every frame, enqueued on two streams in turn without synchronising:
    every lens frame and its statistics equal the per-frame composites, and camera frames too.  Then 60 more frames: one
    gather launch each, and device memory does not grow."""
    torch = torch_cuda
    ctx = t360.make_context(output_layout=t360.LAYOUT_EQUIRECT, interpolation_alg=t360.CUBIC, **LENS_CTX)
    rig = make_rig("pair_190", 61)
    rng = np.random.default_rng(33)
    traj = np.cumsum(rng.normal(0, [6, 2, 2], (16, 3)), 0)
    motions = [seeded_motion(rng, 2 + f % 15, 3.0) for f in range(16)]
    ph = rig_photos(rig)["falloff"]
    vft = t360.VideoFrameTransform(ctx)
    frames = [Frame(torch, 3, seed=f % 4) for f in range(16)]
    stats = torch.zeros((16, 3, STATS), dtype=torch.int64, device="cuda")
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for f, fr in enumerate(frames):
        assert _lens_call(vft, fr)(rig, ph, 3.0 * (f % 2), tuple(traj[f]), motions[f], streams[f % 2].cuda_stream, stats[f].data_ptr())
    torch.cuda.synchronize()
    got_stats = stats.cpu().numpy()
    for f, fr in enumerate(frames):
        want, sums = want_motion(fr, ctx, rig, ph, 3.0 * (f % 2), tuple(traj[f]), motions[f])
        for p, got in enumerate(fr.host()):
            _check(got, want[p], f"frame {f}, plane {p}")
            assert got_stats[f, p].tolist() == sums[p], f"frame {f}, plane {p} statistics"
    cam_ctx = _ctx("pair_190", t360.LINEAR)
    cv = t360.VideoFrameTransform(cam_ctx)
    cframes = [MipFrame(torch, "pair_190", 3, seed=k % 3) for k in range(8)]
    args = [(seam_pose(MODELS[sorted(MODELS)[k % 4]], 900 + k), (None, (3, 0.0))[k % 2], motions[k]) for k in range(8)]
    torch.cuda.synchronize()
    for k, (f, ((pose, cam), minify, mo)) in enumerate(zip(cframes, args)):
        assert _camera_call(cv, f)(rig, ph, 4.0, pose, cam, minify, mo, streams[k % 2].cuda_stream, 0)
    torch.cuda.synchronize()
    for k, (f, ((pose, cam), minify, mo)) in enumerate(zip(cframes, args)):
        want, _ = camera_motion_want(monkeypatch, mo, cam_ctx, rig, ph, 4.0, pose, cam, minify, f.src, f.out_dims, f.prefill)
        for p, got in enumerate(f.host()):
            _check(got, want[p], f"camera frame {k}, plane {p}")
    cv.close()
    f = frames[0]
    call = _lens_call(vft, f)
    st = torch.cuda.Stream()
    for i in range(6):
        assert call(rig, ph, 4.0 * (i % 2), (7.0 * i, 1.0, 0.0), motions[i], st.cuda_stream, stats[0].data_ptr())
    st.synchronize()
    free_before = torch.cuda.mem_get_info()[0]
    n0 = t360.kernel_launch_count()
    for i in range(60):
        assert call(rig, ph, 4.0 * (i % 2), (7.0 * i, 3.0 * np.sin(i), -2.0), motions[i % 16], st.cuda_stream, stats[0].data_ptr() if i % 3 else 0)
    launches = t360.kernel_launch_count() - n0
    st.synchronize()
    assert launches == 60, f"{launches} launches for 60 frames"
    assert torch.cuda.mem_get_info()[0] >= free_before - (2 << 20), "device memory grew over motion frames"
    vft.close()


@pytest.mark.gpu
def test_refused_calls_launch_nothing_and_leave_the_outputs(torch_cuda, capfd):
    """Refused motion frames on real planes and a real statistics buffer: no kernel launch, the outputs and the statistics
    keep their bytes."""
    torch = torch_cuda
    pair = make_rig("pair_190")
    stats = torch.full((3, STATS), 5, dtype=torch.int64, device="cuda")
    lens_ctx = t360.make_context(output_layout=t360.LAYOUT_EQUIRECT, **LENS_CTX)
    with t360.VideoFrameTransform(lens_ctx) as lv, t360.VideoFrameTransform(_ctx("pair_190")) as cv:
        f, g = Frame(torch, 3), MipFrame(torch, "pair_190", 3)
        before, gbefore = f.host(), g.host()
        lcall, ccall = _lens_call(lv, f), _camera_call(cv, g)
        torch.cuda.synchronize()
        n0 = t360.kernel_launch_count()
        for what, mo in _bad_motions(pair)[1:]:
            _refused(capfd, lcall, pair, IDENTITY, 0.0, (0, 0, 0), mo, 0, stats.data_ptr())
            _refused(capfd, ccall, pair, IDENTITY, 0.0, (90.0, 0.0, 0.0, 90.0, 60.0), PINHOLE, (3, 0.0), mo, 0, stats.data_ptr())
        torch.cuda.synchronize()
        assert t360.kernel_launch_count() == n0
        assert all(np.array_equal(a, b) for a, b in zip(before, f.host())) and all(np.array_equal(a, b) for a, b in zip(gbefore, g.host()))
        assert (stats.cpu().numpy() == 5).all()
