"""Fisheye camera input: frames of a rig of one or two OpenCV-calibrated fisheye lenses to every sphere layout, with the
orientation passed per frame (T360B200_lensMap / lens_map, T360B200_transformFrameLensAsync / make_lens_frame_call).

What pins what:
  - the lens half against a float64 numpy model written from the header's contract, and against cv2.fisheye.projectPoints
    where that is defined (Z > 0); the model's directions come from the planner's map for a large mono equirect input,
    whose u, v are by definition the rig frame's atan2 / asin of the direction the output chain hands to the input lookup;
  - the frames against the plain-C oracle's cv::remap of lens_map's map under BORDER_TRANSPARENT, and against the planned
    path (lens_map -> generate_map_from_warp), bit for bit.
Rigs, orientations and planes are made from seeds."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import tests.test_gather_plan as tgp
import transform360_b200 as t360
from oracle import c_oracle as co
from tests.golden.cases import SMALL
from tests.test_warp_map import _check, _pitch, _refused, _stdout

TRANSPARENT = t360.BORDER_TRANSPARENT
INTERPS = [t360.NEAREST, t360.LINEAR, t360.CUBIC, t360.LANCZOS4]
LAYOUTS = {"cubemap_32": t360.LAYOUT_CUBEMAP_32, "cubemap_23_offcenter": t360.LAYOUT_CUBEMAP_23_OFFCENTER, "eac_32": t360.LAYOUT_EAC_32,
           "equirect": t360.LAYOUT_EQUIRECT, "barrel": t360.LAYOUT_BARREL, "barrel_split": t360.LAYOUT_BARREL_SPLIT}
# output fields of the model checks: the six layouts, an off-centre cube map and a barrel with expand_coef != 1
OUTPUTS = {**{name: dict(output_layout=lay) for name, lay in LAYOUTS.items()},
           "cubemap_32_offcentre": dict(output_layout=t360.LAYOUT_CUBEMAP_32, fixed_cube_offcenter_x=0.2, fixed_cube_offcenter_z=-0.35),
           "barrel_expand": dict(output_layout=t360.LAYOUT_BARREL, expand_coef=1.12),
           "equirect_vflip": dict(output_layout=t360.LAYOUT_EQUIRECT, vflip=1)}
LENS_CTX = dict(enable_low_pass_filter=0)


# ---- rigs (seeded) -----------------------------------------------------------------------------------------------------
def _increasing(k, max_angle):
    t2 = np.square(np.linspace(0.0, np.radians(max_angle), 4097))
    return bool(((1 + t2 * (3 * k[0] + t2 * (5 * k[1] + t2 * (7 * k[2] + t2 * 9 * k[3])))) > 0).all())


def _k(rng, max_angle):
    """Distortion in +-0.05 whose theta_d(theta) increases up to max_angle (the library refuses the others)."""
    while True:
        k = rng.uniform(-0.05, 0.05, 4)
        if _increasing(k, max_angle):
            return k


def _lens(rng, radius, cx, cy, yaw, pitch, roll, max_angle, aspect=1.0):
    k = _k(rng, max_angle)
    th = np.radians(max_angle)
    f = radius / (th * (1 + k[0] * th ** 2 + k[1] * th ** 4 + k[2] * th ** 6 + k[3] * th ** 8))
    return t360.T360Lens(f, f * aspect, cx, cy, tuple(k), yaw, pitch, roll, max_angle)


def make_rig(name, seed=0):
    """single_200: one 200-degree lens; pair_190: back-to-back 190-degree lenses side by side (a dual-fisheye frame);
    tilted: a pair with tilt, roll and unequal intrinsics."""
    rng = np.random.default_rng(seed)
    j = lambda s: float(rng.uniform(-s, s))
    if name == "single_200":
        rig = t360.T360LensRig(1, 1000, 1000)
        rig.lens[0] = _lens(rng, 500, 499.5 + j(3), 499.5 + j(3), 0, 0, 0, 100)
    elif name == "pair_190":
        rig = t360.T360LensRig(2, 2000, 1000)
        rig.lens[0] = _lens(rng, 500, 499.5 + j(2), 499.5 + j(2), 0, 0, 0, 95)
        rig.lens[1] = _lens(rng, 500, 1499.5 + j(2), 499.5 + j(2), 180, 0, 0, 95)
    else:
        rig = t360.T360LensRig(2, 1600, 900)
        rig.lens[0] = _lens(rng, 430, 395 + j(5), 452 + j(5), 5 + j(3), 10 + j(3), 15 + j(3), 97, aspect=1.03)
        rig.lens[1] = _lens(rng, 415, 1205 + j(5), 446 + j(5), 172 + j(3), -8 + j(3), -20 + j(3), 93, aspect=0.98)
    return rig


RIGS = ["single_200", "pair_190", "tilted"]


# ---- the float64 model -------------------------------------------------------------------------------------------------
BIG_W, BIG_H = 1 << 20, 1 << 19  # the planner's equirect input for the directions: 7.5e-7 rad per float32 step of its map


def _rot(yaw, pitch, roll):
    """R = Ry(yaw) Rx(-pitch) Rz(roll)."""
    a, b, g = np.radians([yaw, -pitch, roll])
    ry = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    rx = np.array([[1, 0, 0], [0, np.cos(b), -np.sin(b)], [0, np.sin(b), np.cos(b)]])
    rz = np.array([[np.cos(g), -np.sin(g), 0], [np.sin(g), np.cos(g), 0], [0, 0, 1]])
    return ry @ rx @ rz


def directions(out, orientation, w, h):
    """Unit rig-frame directions (float64 [h][w][3]) of a w x h output and the barrel dead zone, from the planner's map for
    a mono BIG_W x BIG_H equirect input: u = atan2(x, z) / 2pi + 0.5, v = 0.5 - asin(y) / pi by the rig frame's definition."""
    ctx = t360.make_context(**out, **LENS_CTX, input_layout=t360.LAYOUT_EQUIRECT, fixed_yaw=orientation[0], fixed_pitch=orientation[1],
                            fixed_roll=orientation[2])
    m = t360.HostPlan(ctx, BIG_W, BIG_H, w, h).map.astype(np.float64)
    u, v = (m[..., 0] + 0.5) / BIG_W, (m[..., 1] + 0.5) / BIG_H
    dead = u < -0.5  # (the dead zone's u = -1)
    lon, lat = (u - 0.5) * 2 * np.pi, (0.5 - v) * np.pi
    return np.stack([np.cos(lat) * np.sin(lon), np.sin(lat), np.cos(lat) * np.cos(lon)], -1), dead


def model(rig, d, dead, in_w, in_h, eps=1e-5):
    """The contract in float64: (map [h][w][2] with NaN where uncovered, camera coordinates [h][w][3] of the chosen lens,
    near: pixels whose lens choice or coverage lies within eps of its threshold, second: lens 1 chosen)."""
    n = rig.numLenses
    lenses = [rig.lens[i] for i in range(n)]
    cams = [d @ _rot(L.yaw, L.pitch, L.roll) for L in lenses]  # (R^T d per pixel)
    cams = [np.stack([c[..., 0], -c[..., 1], c[..., 2]], -1) for c in cams]
    second = (cams[1][..., 2] > cams[0][..., 2]) if n == 2 else np.zeros(d.shape[:2], bool)
    near = (np.abs(cams[1][..., 2] - cams[0][..., 2]) < eps) if n == 2 else np.zeros(d.shape[:2], bool)
    cam = np.where(second[..., None], cams[1], cams[0]) if n == 2 else cams[0]
    out = np.full(d.shape[:2] + (2,), np.nan)
    for i, L in enumerate(lenses):
        sel = (second if i == 1 else ~second) & ~dead
        X, Y, Z = cam[..., 0], cam[..., 1], cam[..., 2]
        rho = np.hypot(X, Y)
        th = np.arctan2(rho, Z)
        t_max = np.radians(np.float64(np.float32(L.maxAngle)))
        near |= sel & (np.abs(th - t_max) < eps)
        k = list(L.k)
        thd = th * (1 + k[0] * th ** 2 + k[1] * th ** 4 + k[2] * th ** 6 + k[3] * th ** 8)
        s = np.where(rho > 0, thd / np.where(rho > 0, rho, 1), 0.0)
        px = (L.fx * s * X + L.cx + 0.5) / rig.calibWidth * in_w - 0.5
        py = (L.fy * s * Y + L.cy + 0.5) / rig.calibHeight * in_h - 0.5
        ok = sel & (th <= t_max)
        out[ok] = np.stack([px, py], -1)[ok]
    return out, cam, near & ~dead, second


def _orientations(seed, n=2):
    rng = np.random.default_rng(seed)
    return [tuple(float(v) for v in (rng.uniform(-180, 180), rng.uniform(-60, 60), rng.uniform(-45, 45))) for _ in range(n)]


# ---- no GPU needed -----------------------------------------------------------------------------------------------------
def test_lens_entry_points_are_exported_with_their_bindings(tmp_path):
    from transform360_b200.handler import EXPORTED_SYMBOLS, LIB_PATH, PKG
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    L = t360.load()
    for name in ("T360B200_lensMap", "T360B200_transformFrameLensAsync"):
        assert name in EXPORTED_SYMBOLS and name in defined, name
    P = C.POINTER
    assert L.T360B200_lensMap.argtypes == [P(t360.FrameTransformContext), P(t360.T360LensRig), P(t360.T360Orientation)] + [C.c_int] * 4 + [C.c_void_p]
    assert L.T360B200_transformFrameLensAsync.argtypes == [C.c_void_p, P(t360.T360LensRig), P(t360.T360Orientation), C.c_int] + [C.c_void_p] * 9
    assert hasattr(t360.VideoFrameTransform, "make_lens_frame_call") and callable(t360.lens_map)
    # the ctypes mirrors have the header's sizes and offsets
    src = tmp_path / "layout.c"
    fields = ["fx", "fy", "cx", "cy", "k", "yaw", "pitch", "roll", "maxAngle"]
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "transform360_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(T360Lens), sizeof(T360LensRig), offsetof(T360LensRig, numLenses), '
                   'offsetof(T360LensRig, calibWidth), offsetof(T360LensRig, calibHeight), offsetof(T360LensRig, lens));\n'
                   + "".join(f'  printf("%zu\\n", offsetof(T360Lens, {f}));\n' for f in fields) + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-I", str(PKG.parent / "include"), "-o", str(exe), str(src)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    R = t360.T360LensRig
    want = [C.sizeof(t360.T360Lens), C.sizeof(R), R.numLenses.offset, R.calibWidth.offset, R.calibHeight.offset, R.lens.offset]
    want += [getattr(t360.T360Lens, f).offset for f in fields]
    assert got == want


def _lens_map(out, rig, o, in_w, in_h, w, h, interp=t360.CUBIC):
    return t360.lens_map(t360.make_context(**out, **LENS_CTX, interpolation_alg=interp), rig, o, in_w, in_h, w, h)


@pytest.mark.parametrize("rig_name", RIGS)
@pytest.mark.parametrize("out_name", sorted(OUTPUTS))
def test_lens_map_equals_the_float64_model(rig_name, out_name):
    """lens_map against the float64 model for seeded orientations, at odd luma and chroma sizes: max |delta| <= 0.02 px
    and the same NaN pattern, except pixels within 1e-5 of a lens-choice or coverage threshold (fewer than 0.1 %)."""
    rig = make_rig(rig_name, seed=len(out_name))
    near_total = pixels = 0
    worst = 0.0
    for o in _orientations(sum(map(ord, rig_name + out_name))):
        for (w, h), (in_w, in_h) in (((97, 65), (259, 131)), ((49, 33), (130, 66))):
            got = _lens_map(OUTPUTS[out_name], rig, o, in_w, in_h, w, h).astype(np.float64)
            d, dead = directions(OUTPUTS[out_name], o, w, h)
            want, _, near, _ = model(rig, d, dead, in_w, in_h)
            gn, wn = np.isnan(got).any(-1), np.isnan(want).any(-1)
            assert (np.isnan(got[..., 0]) == np.isnan(got[..., 1])).all()
            bad = (gn != wn) & ~near
            assert not bad.any(), f"{int(bad.sum())} pixels covered differently from the model (orientation {o}, {w}x{h})"
            both = ~gn & ~wn & ~near
            if both.any():
                worst = max(worst, float(np.abs(got[both] - want[both]).max()))
            near_total += int(near.sum())
            pixels += near.size
            if "barrel" in out_name:
                assert dead.any() and np.isnan(got[dead]).all(), "the barrel dead zone is uncovered"
    assert worst <= 0.02, f"max |delta| {worst:.4f} px"
    assert near_total < 0.001 * pixels, f"{near_total} of {pixels} pixels near a threshold"


@pytest.mark.parametrize("rig_name", RIGS)
def test_lens_map_equals_opencv_fisheye_project_points(rig_name):
    """At the calibration size, covered pixels with Z > 0 lie within 0.02 px of cv2.fisheye.projectPoints of the model's
    camera coordinates: the lens model is OpenCV's."""
    cv2 = pytest.importorskip("cv2")
    rig = make_rig(rig_name, seed=7)
    out = OUTPUTS["equirect"]
    w, h = 181, 91
    for o in _orientations(11, 3):
        got = _lens_map(out, rig, o, rig.calibWidth, rig.calibHeight, w, h).astype(np.float64)
        d, dead = directions(out, o, w, h)
        want, cam, near, second = model(rig, d, dead, rig.calibWidth, rig.calibHeight)
        sel = ~np.isnan(got).any(-1) & ~np.isnan(want).any(-1) & ~near & (cam[..., 2] > 0)
        assert sel.sum() > 0.2 * sel.size
        for i in range(rig.numLenses):
            L = rig.lens[i]
            pick = sel & (second if i == 1 else ~second)
            if not pick.any():
                continue
            K = np.array([[L.fx, 0, L.cx], [0, L.fy, L.cy], [0, 0, 1]], np.float64)
            D = np.array(list(L.k), np.float64).reshape(4, 1)
            pts, _ = cv2.fisheye.projectPoints(cam[pick].reshape(-1, 1, 3), np.zeros(3), np.zeros(3), K, D)
            delta = np.abs(pts.reshape(-1, 2) - got[pick]).max()
            assert delta <= 0.02, f"lens {i}: {delta:.4f} px from cv2.fisheye.projectPoints"


@pytest.mark.parametrize("rig_name", RIGS)
@pytest.mark.parametrize("interp", INTERPS)
def test_gather_plans_of_lens_maps_keep_the_invariants(rig_name, interp, monkeypatch):
    """HostPlan.from_warp of each rig's map (BORDER_TRANSPARENT) keeps what tests/test_gather_plan.py checks for context
    plans."""
    rig = make_rig(rig_name, seed=3)
    m = _lens_map(OUTPUTS["equirect"], rig, (20.0, 5.0, -3.0), 259, 131, 161, 81, interp)
    hp = t360.HostPlan.from_warp(t360.make_context(interpolation_alg=interp, **LENS_CTX), m, 259, 131, TRANSPARENT)
    shown = t360.make_context(interpolation_alg=interp, output_layout=t360.LAYOUT_BARREL)  # (a BORDER_TRANSPARENT plan)
    monkeypatch.setitem(SMALL, "__lens", {})
    monkeypatch.setattr(tgp, "_plan", lambda case, plane: (shown, hp, 259, 131))
    tgp.test_gather_plan_invariants("small", "__lens", 0)


def _bad_rigs():
    """(what, rig or None, orientation or None, context overrides) the library refuses."""
    good = make_rig("pair_190")
    cases = [("NULL rig", None, (0, 0, 0), {}), ("NULL orientation", good, None, {})]

    def rig_with(**kw):
        r = make_rig("pair_190")
        for key, v in kw.items():
            if key.startswith("l1_"):
                setattr(r.lens[1], key[3:], v)
            elif key == "k":
                r.lens[0].k[:] = v
            elif key in ("numLenses", "calibWidth", "calibHeight"):
                setattr(r, key, v)
            else:
                setattr(r.lens[0], key, v)
        return r
    for kw in (dict(numLenses=0), dict(numLenses=3), dict(numLenses=-1), dict(calibWidth=0), dict(calibHeight=-5),
               dict(fx=0.0), dict(fy=-1.0), dict(l1_fx=0.0), dict(cx=float("nan")), dict(l1_cy=float("inf")), dict(yaw=float("nan")),
               dict(l1_roll=float("-inf")), dict(maxAngle=0.0), dict(maxAngle=-10.0), dict(maxAngle=180.5), dict(l1_maxAngle=float("nan")),
               dict(k=(0.0, 0.0, 0.0, float("nan"))), dict(k=(-0.2, 0.0, 0.0, 0.0)), dict(k=(0.0, -0.05, 0.0, 0.0)),
               dict(k=(0.05, 0.0, 0.0, -0.01))):
        cases.append((str(kw), rig_with(**kw), (0, 0, 0), {}))
    for o in ((float("nan"), 0, 0), (0, float("inf"), 0), (0, 0, float("-inf"))):
        cases.append((f"orientation {o}", good, o, {}))
    for ov in (dict(output_layout=t360.LAYOUT_FLAT_FIXED), dict(output_layout=7), dict(output_layout=-1), dict(enable_low_pass_filter=1),
               dict(interpolation_alg=3), dict(interpolation_alg=9)):
        cases.append((str(ov), good, (0, 0, 0), ov))
    return cases


def test_refusals_happen_without_a_gpu(capfd):
    """Every refusal of lens_map and of the lens frame call comes with a message and before any CUDA call (this machine may
    have none): fake device addresses are never dereferenced."""
    L = t360.load()
    m = np.zeros((8, 8, 2), np.float32)
    P, I = C.c_void_p * 3, C.c_int * 3

    def frame(vft, rig, o, n=1, planes=(0x20000,), dims=(64, 32, 8, 8), pitch=(64, 8)):
        arr = lambda v: I(*([v] * 3))
        ob = C.byref(t360.T360Orientation(*o)) if o is not None else None
        return L.T360B200_transformFrameLensAsync(vft._h, C.byref(rig) if rig is not None else None, ob, n, P(*(list(planes) * 3)[:3]),
                                                  P(*(list(planes) * 3)[:3]), arr(dims[0]), arr(dims[1]), arr(pitch[0]), arr(dims[2]),
                                                  arr(dims[3]), arr(pitch[1]), None)
    for what, rig, o, ov in _bad_rigs():
        ctx = t360.make_context(**{**LENS_CTX, "output_layout": t360.LAYOUT_EQUIRECT, **ov})
        ob = C.byref(t360.T360Orientation(*o)) if o is not None else None
        assert not L.T360B200_lensMap(C.byref(ctx), C.byref(rig) if rig is not None else None, ob, 64, 32, 8, 8, m.ctypes.data), what
        assert _stdout(capfd).strip(), what
        with t360.VideoFrameTransform(ctx) as vft:
            _refused(capfd, frame, vft, rig, o)
    good = make_rig("pair_190")
    ctx = t360.make_context(output_layout=t360.LAYOUT_EQUIRECT, **LENS_CTX)
    for args in ((64, 32, 0, 8, m.ctypes.data), (64, 0, 8, 8, m.ctypes.data), (64, 32, 8, 8, None)):
        _refused(capfd, L.T360B200_lensMap, C.byref(ctx), C.byref(good), C.byref(t360.T360Orientation()), *args)
    _refused(capfd, L.T360B200_lensMap, None, C.byref(good), C.byref(t360.T360Orientation()), 64, 32, 8, 8, m.ctypes.data)
    with pytest.raises(ValueError):
        t360.lens_map(t360.make_context(output_layout=t360.LAYOUT_FLAT_FIXED, **LENS_CTX), good, (0, 0, 0), 64, 32, 8, 8)
    with t360.VideoFrameTransform(ctx) as vft:
        for kw in (dict(n=0), dict(n=4), dict(planes=(None,)), dict(dims=(0, 32, 8, 8)), dict(dims=(64, 32, 8, -1)),
                   dict(pitch=(63, 8)), dict(pitch=(64, 7))):
            _refused(capfd, lambda: frame(vft, good, (0, 0, 0), **kw))
    assert not L.T360B200_transformFrameLensAsync(None, None, None, 1, None, None, None, None, None, None, None, None, None)


# ---- on the GPU --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests must run on an H100 (there is no CPU fallback to test)")
    return torch


IN_DIMS = [(259, 131), (130, 66), (130, 66)]  # a dual-fisheye yuv420p frame with odd sizes
OUT_DIMS = [(97, 65), (49, 33), (49, 33)]


def _pattern(w, h, p):
    """What an output holds before the frame: a non-zero pattern (chroma too: the call pre-fills it with 128)."""
    i, j = np.mgrid[:h, :w]
    return (((i * 7 + j * 13 + 29 * p) % 251) + 1).astype(np.uint8)


def _dev(torch, a, pitch=None):
    pitch = pitch or _pitch(a.shape[1])
    t = torch.zeros((a.shape[0], pitch), dtype=torch.uint8, device="cuda")
    t[:, :a.shape[1]] = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t


def _oracle(src, m, interp, p, out_w, out_h):
    """cv::remap of the lens map under BORDER_TRANSPARENT into the pre-filled output (luma: the pattern, chroma: 128)."""
    dst = _pattern(out_w, out_h, p) if p == 0 else np.full((out_h, out_w), 128, np.uint8)
    return co.remap_u8(src, m, interp, TRANSPARENT, dst)


class Frame:
    """Source planes (host and device), pre-filled outputs and the argument lists of one lens frame."""

    def __init__(self, torch, n=3, seed=0, unaligned=False):
        self.torch, self.n = torch, n
        self.src = [co.noise_plane(*IN_DIMS[p], plane=p, frame=seed) for p in range(n)]
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
        self.dims = [(*IN_DIMS[p], *OUT_DIMS[p]) for p in range(n)]

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

    def want(self, ctx, rig, o, interp):
        maps = [t360.lens_map(ctx, rig, o, *IN_DIMS[p], *OUT_DIMS[p]) for p in range(min(self.n, 2))]
        return [_oracle(self.src[p], maps[min(p, 1)], interp, p, *OUT_DIMS[p]) for p in range(self.n)], maps


@pytest.mark.gpu
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("interp", INTERPS)
def test_lens_frames_equal_the_oracle_and_the_planned_path(layout, interp, torch_cuda):
    """On a never-planned transform, 3- and 1-plane lens frames (one with an unaligned luma plane) equal the oracle's
    cv::remap of lens_map's maps bit for bit: uncovered luma keeps the pattern, chroma is 128.  Then lens_map ->
    generate_map_from_warp on indices 0 and 1: transformFrameAsync and the host ABI give the same frames, and lens frames
    on the transform holding those warp plans still do."""
    torch = torch_cuda
    ctx = t360.make_context(output_layout=LAYOUTS[layout], interpolation_alg=interp, **LENS_CTX)
    rig = make_rig("tilted" if interp in (t360.LINEAR, t360.LANCZOS4) else "pair_190", seed=interp)
    o = _orientations(interp * 10 + len(layout), 1)[0]
    vft = t360.VideoFrameTransform(ctx)
    st = torch.cuda.Stream()
    for n, unaligned in ((3, False), (1, False), (3, True)):
        f = Frame(torch, n, seed=interp, unaligned=unaligned)
        want, maps = f.want(ctx, rig, o, interp)
        torch.cuda.synchronize()
        assert vft.make_lens_frame_call(f.in_planes, f.out_planes, f.dims)(rig, o, st.cuda_stream)
        st.synchronize()
        for p, got in enumerate(f.host()):
            _check(got, want[p], f"lens frame of {n} planes{' (unaligned)' if unaligned else ''}, plane {p}")
    if "barrel" in layout:
        assert np.isnan(maps[0]).any()
    # the planned path for the same pose
    f = Frame(torch, 3, seed=interp)
    want, maps = f.want(ctx, rig, o, interp)
    for idx in (0, 1):
        assert vft.generate_map_from_warp(maps[idx], *IN_DIMS[idx], idx, TRANSPARENT)
    torch.cuda.synchronize()
    assert vft.make_frame_call(f.in_planes, f.out_planes, f.dims)(st.cuda_stream)
    st.synchronize()
    for p, got in enumerate(f.host()):
        _check(got, want[p], f"planned frame, plane {p}")
        h_out = _pattern(*OUT_DIMS[p], p) if p == 0 else np.full(OUT_DIMS[p][::-1], 128, np.uint8)
        _check(vft.transform_plane(f.src[p], *OUT_DIMS[p], min(p, 1), p, out=h_out), want[p], f"host-pointer planned plane {p}")
    f.reset()
    torch.cuda.synchronize()
    assert vft.make_lens_frame_call(f.in_planes, f.out_planes, f.dims)(rig, o, st.cuda_stream)
    st.synchronize()
    for p, got in enumerate(f.host()):
        _check(got, want[p], f"lens frame on a transform holding warp plans, plane {p}")
    vft.close()


@pytest.mark.gpu
def test_orientation_trajectory_with_a_rig_change_on_two_streams(torch_cuda):
    """30 frames of a seeded orientation trajectory, the rig replaced at frame 12 and the output pair recycled every frame,
    enqueued on two streams in turn with no synchronisation between them: every frame equals the oracle."""
    torch = torch_cuda
    ctx = t360.make_context(output_layout=t360.LAYOUT_CUBEMAP_32, interpolation_alg=t360.CUBIC, **LENS_CTX)
    rigs = [make_rig("pair_190", 21), make_rig("tilted", 22)]
    rng = np.random.default_rng(5)
    traj = np.cumsum(rng.normal(0, [6, 2, 2], (30, 3)), 0)
    vft = t360.VideoFrameTransform(ctx)
    frames = [Frame(torch, 3, seed=f % 4) for f in range(30)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for f, fr in enumerate(frames):
        assert vft.make_lens_frame_call(fr.in_planes, fr.out_planes, fr.dims)(rigs[f >= 12], tuple(traj[f]), streams[f % 2].cuda_stream)
    for s in streams:
        s.synchronize()
    for f, fr in enumerate(frames):
        want, _ = fr.want(ctx, rigs[f >= 12], tuple(traj[f]), t360.CUBIC)
        for p, got in enumerate(fr.host()):
            _check(got, want[p], f"frame {f}, plane {p}")
    vft.close()


@pytest.mark.gpu
def test_reconfigure_between_lens_frames_is_frame_exact(torch_cuda):
    """On a transform holding context plans, lens frames and context frames interleaved with reconfigure_async (expand_coef,
    then the interpolation) and a reconfigure, all enqueued without synchronising: every lens frame equals the oracle for
    the context current when it was enqueued, every context frame a fresh transform's, and the plans are left in effect."""
    torch = torch_cuda
    base = dict(output_layout=t360.LAYOUT_BARREL, interpolation_alg=t360.CUBIC, input_layout=t360.LAYOUT_EQUIRECT, **LENS_CTX)
    ctxs = [t360.make_context(**base), t360.make_context(**dict(base, expand_coef=1.1)),
            t360.make_context(**dict(base, expand_coef=1.1, interpolation_alg=t360.LINEAR)),
            t360.make_context(**dict(base, interpolation_alg=t360.LANCZOS4))]
    rig = make_rig("pair_190", 31)
    vft = t360.VideoFrameTransform(ctxs[0])
    for idx in (0, 1):
        assert vft.generateMapForPlane(*IN_DIMS[idx], *OUT_DIMS[idx], idx)
    lens = [Frame(torch, 3, seed=s) for s in range(4)]
    plain = [Frame(torch, 3, seed=s) for s in range(4)]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for s in range(4):
        if s in (1, 2):
            vft.reconfigure_async(ctxs[s])
        elif s == 3:
            vft.reconfigure(ctxs[s])
        assert vft.make_lens_frame_call(lens[s].in_planes, lens[s].out_planes, lens[s].dims)(rig, (30.0 * s, 5.0, 0.0), st.cuda_stream)
        for o in plain[s].outs:
            o.zero_()
        assert vft.make_frame_call(plain[s].in_planes, plain[s].out_planes, plain[s].dims)(st.cuda_stream)
    st.synchronize()
    for s in range(4):
        want, _ = lens[s].want(ctxs[s], rig, (30.0 * s, 5.0, 0.0), ctxs[s].interpolation_alg)
        for p, got in enumerate(lens[s].host()):
            _check(got, want[p], f"lens frame {s}, plane {p}")
        fresh = t360.VideoFrameTransform(ctxs[s])
        for idx in (0, 1):
            assert fresh.generateMapForPlane(*IN_DIMS[idx], *OUT_DIMS[idx], idx)
        ref = Frame(torch, 3, seed=s)
        for o in ref.outs:
            o.zero_()
        assert fresh.make_frame_call(ref.in_planes, ref.out_planes, ref.dims)(0)
        torch.cuda.synchronize()
        for p, (got, w) in enumerate(zip(plain[s].host(), ref.host())):
            _check(got, w, f"context frame {s}, plane {p}")
        fresh.close()
    vft.close()


@pytest.mark.gpu
def test_device_memory_and_launches_stay_bounded(torch_cuda):
    """50 lens frames after a warm-up, a new orientation every frame: one kernel launch each (the chroma pre-fill is a
    memset) and no growth of device memory."""
    torch = torch_cuda
    ctx = t360.make_context(output_layout=t360.LAYOUT_EAC_32, interpolation_alg=t360.LANCZOS4, **LENS_CTX)
    rig = make_rig("tilted", 41)
    vft = t360.VideoFrameTransform(ctx)
    f = Frame(torch, 3)
    call = vft.make_lens_frame_call(f.in_planes, f.out_planes, f.dims)
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for i in range(5):
        assert call(rig, (7.0 * i, 1.0, 0.0), st.cuda_stream)
    st.synchronize()
    free_before = torch.cuda.mem_get_info()[0]
    n0 = t360.kernel_launch_count()
    for i in range(50):
        assert call(rig, (7.0 * i, 3.0 * np.sin(i), -2.0), st.cuda_stream)
    launches = t360.kernel_launch_count() - n0
    st.synchronize()
    assert launches == 50, f"{launches} launches for 50 frames"
    assert torch.cuda.mem_get_info()[0] >= free_before - (2 << 20), "device memory grew over lens frames"
    vft.close()


@pytest.mark.gpu
def test_refused_calls_launch_nothing_and_leave_the_outputs(torch_cuda, capfd):
    """Refused lens frames on real planes: no kernel launch, the outputs keep their bytes (chroma included)."""
    torch = torch_cuda
    L = t360.load()
    for what, rig, o, ov in _bad_rigs():
        ctx = t360.make_context(**{**LENS_CTX, "output_layout": t360.LAYOUT_EQUIRECT, **ov})
        with t360.VideoFrameTransform(ctx) as vft:
            f = Frame(torch, 3)
            before = f.host()
            torch.cuda.synchronize()
            n0 = t360.kernel_launch_count()
            P, I = C.c_void_p * 3, C.c_int * 3
            ob = C.byref(t360.T360Orientation(*o)) if o is not None else None
            ok = L.T360B200_transformFrameLensAsync(vft._h, C.byref(rig) if rig is not None else None, ob, 3, P(*[p[0] for p in f.in_planes]),
                                                    P(*[p[0] for p in f.out_planes]), I(*[d[0] for d in f.dims]), I(*[d[1] for d in f.dims]),
                                                    I(*[p[1] for p in f.in_planes]), I(*[d[2] for d in f.dims]), I(*[d[3] for d in f.dims]),
                                                    I(*[p[1] for p in f.out_planes]), None)
            torch.cuda.synchronize()
            assert not ok, what
            assert _stdout(capfd).strip(), what
            assert t360.kernel_launch_count() == n0, what
            for p, (a, b) in enumerate(zip(before, f.host())):
                assert np.array_equal(a, b), f"{what}: plane {p} changed"
