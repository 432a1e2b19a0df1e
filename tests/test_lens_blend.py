"""Fisheye lens rigs with a feathered seam: two lenses blended across a belt of seamWidth degrees (T360B200_lensBlendMaps /
lens_blend_maps, T360B200_transformFrameLensBlendAsync / make_lens_blend_frame_call).

What pins what:
  - the host maps and weights against a float64 model of the header's contract (both lenses' theta, coverage and the
    weight w of lens 1), on the directions tests/test_lens.py derives from the planner;
  - the projection against lens_map: where w is 0 or 256 the contributing map is lens_map's, bit for bit;
  - the frames against a composite of the plain-C oracle's cv::remap of both maps under BORDER_TRANSPARENT, blended with
    the integer rule, bit for bit.
Rigs, orientations and planes are made from seeds."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import transform360_b200 as t360
from oracle import c_oracle as co
from tests.test_lens import IN_DIMS, LAYOUTS, LENS_CTX, OUT_DIMS, Frame, _orientations, _pattern, _rot, directions, make_rig
from tests.test_warp_map import _check, _refused

TRANSPARENT = t360.BORDER_TRANSPARENT
INTERPS = [t360.NEAREST, t360.LINEAR, t360.CUBIC, t360.LANCZOS4]
BLEND_RIGS = ["pair_190", "tilted"]
SEAMS = [2.0, 10.0, 40.0]
NAN = np.float32("nan")


# ---- the float64 model -------------------------------------------------------------------------------------------------
def seam_scale(seam):
    """s = 1 / (2 seamWidth) in radians, computed in double and stored as float, as the library does."""
    return np.float64(np.float32(1.0 / (2.0 * np.float64(np.float32(seam)) * np.pi / 180.0)))


def blend_model(rig, d, dead, in_w, in_h, seam, eps=1e-5):
    """The contract in float64: (map0, map1 [h][w][2] with NaN where the lens does not contribute, w [h][w], near: pixels
    within eps of a coverage threshold or of a weight threshold (theta0 - theta1 where w leaves 0 or reaches 256))."""
    thetas, covers, positions = [], [], []
    near = np.zeros(d.shape[:2], bool)
    for i in range(2):
        L = rig.lens[i]
        c = d @ _rot(L.yaw, L.pitch, L.roll)
        X, Y, Z = c[..., 0], -c[..., 1], c[..., 2]
        rho = np.hypot(X, Y)
        th = np.arctan2(rho, Z)
        t_max = np.radians(np.float64(np.float32(L.maxAngle)))
        k = list(L.k)
        thd = th * (1 + k[0] * th ** 2 + k[1] * th ** 4 + k[2] * th ** 6 + k[3] * th ** 8)
        sc = np.where(rho > 0, thd / np.where(rho > 0, rho, 1), 0.0)
        px = (L.fx * sc * X + L.cx + 0.5) / rig.calibWidth * in_w - 0.5
        py = (L.fy * sc * Y + L.cy + 0.5) / rig.calibHeight * in_h - 0.5
        thetas.append(th)
        covers.append((th <= t_max) & ~dead)
        positions.append(np.stack([px, py], -1))
        near |= np.abs(th - t_max) < eps
    s = seam_scale(seam)
    tw = 256.0 * (0.5 + (thetas[0] - thetas[1]) * s)
    both = covers[0] & covers[1]
    w = np.where(both, np.clip(np.round(tw), 0, 256), np.where(covers[1], 256, 0)).astype(np.int32)
    near |= both & ((np.abs(tw - 0.5) < 256 * s * eps) | (np.abs(tw - 255.5) < 256 * s * eps))
    map0 = np.where((covers[0] & (w < 256))[..., None], positions[0], np.nan)
    map1 = np.where((covers[1] & (w > 0))[..., None], positions[1], np.nan)
    return map0, map1, w, near & ~dead


def _blend_maps(layout, rig, seam, o, in_w, in_h, w, h, interp=t360.CUBIC):
    ctx = t360.make_context(output_layout=layout, interpolation_alg=interp, **LENS_CTX)
    return t360.lens_blend_maps(ctx, rig, seam, o, in_w, in_h, w, h)


# ---- no GPU needed -----------------------------------------------------------------------------------------------------
def test_lens_blend_entry_points_are_exported_with_their_bindings(tmp_path):
    from transform360_b200.handler import EXPORTED_SYMBOLS, LIB_PATH, PKG
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    L = t360.load()
    for name in ("T360B200_lensBlendMaps", "T360B200_transformFrameLensBlendAsync"):
        assert name in EXPORTED_SYMBOLS and name in defined, name
    P = C.POINTER
    assert L.T360B200_lensBlendMaps.argtypes == ([P(t360.FrameTransformContext), P(t360.T360LensRig), C.c_float, P(t360.T360Orientation)]
                                                 + [C.c_int] * 4 + [C.c_void_p] * 3)
    assert L.T360B200_transformFrameLensBlendAsync.argtypes == ([C.c_void_p, P(t360.T360LensRig), C.c_float, P(t360.T360Orientation), C.c_int]
                                                                + [C.c_void_p] * 9)
    assert hasattr(t360.VideoFrameTransform, "make_lens_blend_frame_call") and callable(t360.lens_blend_maps)
    # the header declares both with these prototypes, and compiles as C
    src = tmp_path / "decl.c"
    src.write_text('#include "transform360_b200.h"\n'
                   "int (*maps)(const FrameTransformContext*, const T360LensRig*, float, const T360Orientation*, int, int, int, int, float*, "
                   "float*, uint16_t*) = T360B200_lensBlendMaps;\n"
                   "int (*frame)(VideoFrameTransform*, const T360LensRig*, float, const T360Orientation*, int, const uint8_t* const*, "
                   "uint8_t* const*, const int*, const int*, const int*, const int*, const int*, const int*, void*) = "
                   "T360B200_transformFrameLensBlendAsync;\n")
    subprocess.run(["cc", "-std=c99", "-Wall", "-Werror", "-c", "-I", str(PKG.parent / "include"), "-o", str(tmp_path / "decl.o"), str(src)],
                   check=True)


@pytest.mark.parametrize("rig_name", BLEND_RIGS)
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_lens_blend_maps_equal_the_float64_model(rig_name, layout):
    """lens_blend_maps against the float64 model for seeded orientations, odd luma and chroma sizes and belts of 2, 10 and
    40 degrees: maps within 0.02 px with the same NaN pattern and |delta w| <= 1, except pixels within 1e-5 of a coverage
    or weight threshold (fewer than 0.1 %)."""
    rig = make_rig(rig_name, seed=len(layout))
    out = dict(output_layout=LAYOUTS[layout])
    near_total = pixels = 0
    worst = 0.0
    for o in _orientations(sum(map(ord, rig_name + layout))):
        for (w, h), (in_w, in_h) in (((97, 65), (259, 131)), ((49, 33), (130, 66))):
            d, dead = directions(out, o, w, h)
            for seam in SEAMS:
                m0, m1, wt = _blend_maps(LAYOUTS[layout], rig, seam, o, in_w, in_h, w, h)
                w0, w1, ww, near = blend_model(rig, d, dead, in_w, in_h, seam)
                assert wt.dtype == np.uint16 and int(wt.max()) <= 256
                dw = np.abs(wt.astype(np.int32) - ww)
                assert not (dw[~near] > 1).any(), f"|delta w| {int(dw[~near].max())} (orientation {o}, {w}x{h}, seam {seam})"
                for got, want in ((m0, w0), (m1, w1)):
                    got = got.astype(np.float64)
                    gn, wn = np.isnan(got).any(-1), np.isnan(want).any(-1)
                    assert (np.isnan(got[..., 0]) == np.isnan(got[..., 1])).all()
                    bad = (gn != wn) & ~near
                    assert not bad.any(), f"{int(bad.sum())} entries differ in coverage from the model (orientation {o}, {w}x{h}, seam {seam})"
                    sel = ~gn & ~wn & ~near
                    if sel.any():
                        worst = max(worst, float(np.abs(got[sel] - want[sel]).max()))
                near_total += int(near.sum())
                pixels += near.size
                if "barrel" in layout:
                    assert dead.any() and np.isnan(m0[dead]).all() and np.isnan(m1[dead]).all() and (wt[dead] == 0).all()
    assert worst <= 0.02, f"max |delta| {worst:.4f} px"
    assert near_total < 0.001 * pixels, f"{near_total} of {pixels} pixels near a threshold"


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_single_lens_pixels_equal_lens_map_bit_for_bit(layout):
    """For the back-to-back pair, wherever w is 0 or 256 the contributing map is lens_map's map bit for bit (NaN included),
    and the other map is NaN: the blend and the hard seam share the projection code."""
    rig = make_rig("pair_190", seed=5)
    for o in _orientations(len(layout) + 50, 2):
        for (w, h), (in_w, in_h) in (((97, 65), (259, 131)), ((49, 33), (130, 66))):
            ctx = t360.make_context(output_layout=LAYOUTS[layout], **LENS_CTX)
            hard = t360.lens_map(ctx, rig, o, in_w, in_h, w, h).view(np.uint32)
            m0, m1, wt = t360.lens_blend_maps(ctx, rig, 10.0, o, in_w, in_h, w, h)
            for lone, mine, other in ((wt == 0, m0, m1), (wt == 256, m1, m0)):
                assert lone.any()
                assert np.array_equal(mine.view(np.uint32)[lone], hard[lone]), f"orientation {o}, {w}x{h}"
                assert np.isnan(other[lone]).all()


def test_the_weight_is_a_ramp_across_each_seam():
    """pair_190 to EQUIRECT at orientation (0, 0, 0): along every row w is monotone across each seam (non-increasing over
    the left half, where lens 1's back view gives way to lens 0, non-decreasing over the right half); in the equator row it
    passes from 0 to 256 over seamWidth / 360 x outW columns (+-2), and away from the equator the belt is wider."""
    rig = make_rig("pair_190", seed=9)
    w, h = 720, 361  # (row 180 is the equator)
    for seam in (2.0, 4.0, 10.0):  # (a belt inside both 190-degree lenses' coverage: seamWidth <= 2 (95 - 90))
        _, _, wt = _blend_maps(t360.LAYOUT_EQUIRECT, rig, seam, (0, 0, 0), 2000, 1000, w, h)
        wt = wt.astype(np.int32)
        left, right = wt[:, :w // 2], wt[:, w // 2:]
        assert (np.diff(left, axis=1) <= 0).all() and (np.diff(right, axis=1) >= 0).all(), f"seam {seam}"
        expect = seam / 360 * w
        for half in (left[h // 2], right[h // 2]):
            assert half.min() == 0 and half.max() == 256
            belt = int(((half > 0) & (half < 256)).sum())
            assert abs(belt - expect) <= 2, f"seam {seam}: the equator's belt is {belt} columns, {expect:.1f} expected"
        equator = int(((left[h // 2] > 0) & (left[h // 2] < 256)).sum())
        for row in (h // 4, 3 * h // 4):  # +-45 degrees
            assert int(((left[row] > 0) & (left[row] < 256)).sum()) > equator


def _bad_blend_calls():
    """(what, rig or None, seamWidth, orientation or None, context overrides) the blend calls refuse."""
    good = make_rig("pair_190")

    def rig_with(**kw):
        r = make_rig("pair_190")
        for key, v in kw.items():
            if key in ("numLenses", "calibWidth"):
                setattr(r, key, v)
            else:
                setattr(r.lens[1 if key.startswith("l1_") else 0], key[3:] if key.startswith("l1_") else key, v)
        return r
    cases = [("NULL rig", None, 10.0, (0, 0, 0), {}), ("NULL orientation", good, 10.0, None, {})]
    for kw in (dict(numLenses=1), dict(numLenses=0), dict(numLenses=3), dict(calibWidth=0), dict(fx=0.0), dict(l1_maxAngle=181.0),
               dict(l1_cy=float("nan"))):
        cases.append((str(kw), rig_with(**kw), 10.0, (0, 0, 0), {}))
    single = make_rig("single_200")
    cases.append(("a single-lens rig", single, 10.0, (0, 0, 0), {}))
    for seam in (float("nan"), float("inf"), float("-inf"), 0.0, 0.005, 181.0, -10.0):
        cases.append((f"seamWidth {seam}", good, seam, (0, 0, 0), {}))
    cases.append(("orientation nan", good, 10.0, (float("nan"), 0, 0), {}))
    for ov in (dict(output_layout=t360.LAYOUT_FLAT_FIXED), dict(output_layout=7), dict(enable_low_pass_filter=1), dict(interpolation_alg=3)):
        cases.append((str(ov), good, 10.0, (0, 0, 0), ov))
    return cases


def test_refusals_happen_without_a_gpu(capfd):
    """Every refusal of lens_blend_maps and of the blend frame call comes with a message and before any CUDA call (this
    machine may have none): fake device addresses are never dereferenced."""
    L = t360.load()
    m0, m1, wt = np.zeros((8, 8, 2), np.float32), np.zeros((8, 8, 2), np.float32), np.zeros((8, 8), np.uint16)
    P, I = C.c_void_p * 3, C.c_int * 3

    def frame(vft, rig, seam, o, n=1, planes=(0x20000,), dims=(64, 32, 8, 8), pitch=(64, 8)):
        arr = lambda v: I(*([v] * 3))
        ob = C.byref(t360.T360Orientation(*o)) if o is not None else None
        return L.T360B200_transformFrameLensBlendAsync(vft._h, C.byref(rig) if rig is not None else None, seam, ob, n,
                                                       P(*(list(planes) * 3)[:3]), P(*(list(planes) * 3)[:3]), arr(dims[0]), arr(dims[1]),
                                                       arr(pitch[0]), arr(dims[2]), arr(dims[3]), arr(pitch[1]), None)
    for what, rig, seam, o, ov in _bad_blend_calls():
        ctx = t360.make_context(**{**LENS_CTX, "output_layout": t360.LAYOUT_EQUIRECT, **ov})
        ob = C.byref(t360.T360Orientation(*o)) if o is not None else None
        _refused(capfd, L.T360B200_lensBlendMaps, C.byref(ctx), C.byref(rig) if rig is not None else None, seam, ob, 64, 32, 8, 8,
                 m0.ctypes.data, m1.ctypes.data, wt.ctypes.data)
        with t360.VideoFrameTransform(ctx) as vft:
            _refused(capfd, frame, vft, rig, seam, o)
    good = make_rig("pair_190")
    ctx = t360.make_context(output_layout=t360.LAYOUT_EQUIRECT, **LENS_CTX)
    o = C.byref(t360.T360Orientation())
    for args in ((64, 32, 0, 8, m0.ctypes.data, m1.ctypes.data, wt.ctypes.data), (0, 32, 8, 8, m0.ctypes.data, m1.ctypes.data, wt.ctypes.data),
                 (64, 32, 8, 8, None, m1.ctypes.data, wt.ctypes.data), (64, 32, 8, 8, m0.ctypes.data, None, wt.ctypes.data),
                 (64, 32, 8, 8, m0.ctypes.data, m1.ctypes.data, None)):
        _refused(capfd, L.T360B200_lensBlendMaps, C.byref(ctx), C.byref(good), 10.0, o, *args)
    _refused(capfd, L.T360B200_lensBlendMaps, None, C.byref(good), 10.0, o, 64, 32, 8, 8, m0.ctypes.data, m1.ctypes.data, wt.ctypes.data)
    with pytest.raises(ValueError):
        t360.lens_blend_maps(ctx, good, 0.0, (0, 0, 0), 64, 32, 8, 8)
    with t360.VideoFrameTransform(ctx) as vft:
        for kw in (dict(n=0), dict(n=4), dict(planes=(None,)), dict(dims=(0, 32, 8, 8)), dict(pitch=(63, 8)), dict(pitch=(64, 7))):
            _refused(capfd, lambda: frame(vft, good, 10.0, (0, 0, 0), **kw))
    assert not L.T360B200_transformFrameLensBlendAsync(None, None, 10.0, None, 1, None, None, None, None, None, None, None, None, None)


# ---- on the GPU --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests must run on an H100 (there is no CPU fallback to test)")
    return torch


def composite(src, map0, map1, weight, interp, prefill):
    """The oracle's frame: cv::remap of each map under BORDER_TRANSPARENT twice, into outputs of 0 and of 255 (where the two
    differ, BORDER_TRANSPARENT skipped the pixel), then (a (256 - w) + b w + 128) >> 8 where both were sampled, the one
    that was where only one was, and the pre-fill where neither was."""
    h, w = weight.shape

    def sample(m):
        lo = co.remap_u8(src, m, interp, TRANSPARENT, np.zeros((h, w), np.uint8))
        hi = co.remap_u8(src, m, interp, TRANSPARENT, np.full((h, w), 255, np.uint8))
        return lo.astype(np.int32), lo == hi
    (a, va), (b, vb) = sample(map0), sample(map1)
    wt = weight.astype(np.int32)
    out = prefill.astype(np.int32).copy()
    out[va & ~vb] = a[va & ~vb]
    out[vb & ~va] = b[vb & ~va]
    both = va & vb
    out[both] = (a[both] * (256 - wt[both]) + b[both] * wt[both] + 128) >> 8
    return out.astype(np.uint8)


def want_blend(f, ctx, rig, seam, o):
    """The oracle's planes of Frame f (luma pre-filled with its pattern, chroma with 128), and the luma maps."""
    maps = [t360.lens_blend_maps(ctx, rig, seam, o, *IN_DIMS[p], *OUT_DIMS[p]) for p in range(min(f.n, 2))]
    want = []
    for p in range(f.n):
        prefill = _pattern(*OUT_DIMS[p], p) if p == 0 else np.full(OUT_DIMS[p][::-1], 128, np.uint8)
        want.append(composite(f.src[p], *maps[min(p, 1)], ctx.interpolation_alg, prefill))
    return want, maps[0]


def _blend_call(vft, f):
    return vft.make_lens_blend_frame_call(f.in_planes, f.out_planes, f.dims)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("interp", INTERPS)
def test_blend_frames_equal_the_oracle(layout, interp, torch_cuda):
    """On a never-planned transform, 3- and 1-plane blend frames (one with an unaligned luma plane) equal the oracle's
    composite bit for bit.  Then on the same transform holding context plans (index 0) and a warp plan (index 1): blend
    frames still equal it, and the plans stay in effect (a planned frame is the same before and after)."""
    torch = torch_cuda
    ctx = t360.make_context(output_layout=LAYOUTS[layout], interpolation_alg=interp, **LENS_CTX)
    rig = make_rig("tilted" if interp in (t360.LINEAR, t360.LANCZOS4) else "pair_190", seed=interp + 1)
    seam = (4.0, 10.0, 25.0, 40.0)[INTERPS.index(interp)]
    o = _orientations(interp * 10 + len(layout) + 3, 1)[0]
    vft = t360.VideoFrameTransform(ctx)
    st = torch.cuda.Stream()
    for n, unaligned in ((3, False), (1, False), (3, True)):
        f = Frame(torch, n, seed=interp, unaligned=unaligned)
        want, m0 = want_blend(f, ctx, rig, seam, o)
        torch.cuda.synchronize()
        assert _blend_call(vft, f)(rig, seam, o, st.cuda_stream)
        st.synchronize()
        for p, got in enumerate(f.host()):
            _check(got, want[p], f"blend frame of {n} planes{' (unaligned)' if unaligned else ''}, plane {p}")
    # a transform holding a context plan and a warp plan
    assert vft.generateMapForPlane(*IN_DIMS[0], *OUT_DIMS[0], 0)
    assert vft.generate_map_from_warp(t360.lens_map(ctx, rig, o, *IN_DIMS[1], *OUT_DIMS[1]), *IN_DIMS[1], 1, TRANSPARENT)
    planned = Frame(torch, 3, seed=7)
    torch.cuda.synchronize()
    assert vft.make_frame_call(planned.in_planes, planned.out_planes, planned.dims)(st.cuda_stream)
    st.synchronize()
    before = planned.host()
    f = Frame(torch, 3, seed=interp + 1)
    want, _ = want_blend(f, ctx, rig, seam, o)
    torch.cuda.synchronize()
    assert _blend_call(vft, f)(rig, seam, o, st.cuda_stream)
    st.synchronize()
    for p, got in enumerate(f.host()):
        _check(got, want[p], f"blend frame on a transform holding plans, plane {p}")
    planned.reset()
    torch.cuda.synchronize()
    assert vft.make_frame_call(planned.in_planes, planned.out_planes, planned.dims)(st.cuda_stream)
    st.synchronize()
    for p, (a, b) in enumerate(zip(before, planned.host())):
        _check(b, a, f"planned frame after blend frames, plane {p}")
    vft.close()


@pytest.mark.gpu
def test_trajectory_with_rig_and_seam_changes_on_two_streams(torch_cuda):
    """30 frames with a new orientation every frame, the rig and seamWidth replaced at frame 14 and the frames enqueued on
    two streams in turn with no synchronisation between them: every frame equals the oracle."""
    torch = torch_cuda
    ctx = t360.make_context(output_layout=t360.LAYOUT_EQUIRECT, interpolation_alg=t360.CUBIC, **LENS_CTX)
    rigs, seams = [make_rig("pair_190", 61), make_rig("tilted", 62)], [10.0, 3.5]
    rng = np.random.default_rng(15)
    traj = np.cumsum(rng.normal(0, [6, 2, 2], (30, 3)), 0)
    vft = t360.VideoFrameTransform(ctx)
    frames = [Frame(torch, 3, seed=f % 4) for f in range(30)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for f, fr in enumerate(frames):
        assert _blend_call(vft, fr)(rigs[f >= 14], seams[f >= 14], tuple(traj[f]), streams[f % 2].cuda_stream)
    for s in streams:
        s.synchronize()
    for f, fr in enumerate(frames):
        want, _ = want_blend(fr, ctx, rigs[f >= 14], seams[f >= 14], tuple(traj[f]))
        for p, got in enumerate(fr.host()):
            _check(got, want[p], f"frame {f}, plane {p}")
    vft.close()


@pytest.mark.gpu
def test_reconfigure_between_blend_frames_is_frame_exact(torch_cuda):
    """On a transform holding context plans, blend frames and context frames interleaved with reconfigure_async
    (expand_coef, then the interpolation) and a reconfigure, all enqueued without synchronising: every blend frame equals
    the oracle for the context current when it was enqueued, every context frame a fresh transform's."""
    torch = torch_cuda
    base = dict(output_layout=t360.LAYOUT_BARREL, interpolation_alg=t360.CUBIC, input_layout=t360.LAYOUT_EQUIRECT, **LENS_CTX)
    ctxs = [t360.make_context(**base), t360.make_context(**dict(base, expand_coef=1.1)),
            t360.make_context(**dict(base, expand_coef=1.1, interpolation_alg=t360.LINEAR)),
            t360.make_context(**dict(base, interpolation_alg=t360.LANCZOS4))]
    rig = make_rig("pair_190", 71)
    vft = t360.VideoFrameTransform(ctxs[0])
    for idx in (0, 1):
        assert vft.generateMapForPlane(*IN_DIMS[idx], *OUT_DIMS[idx], idx)
    blend = [Frame(torch, 3, seed=s) for s in range(4)]
    plain = [Frame(torch, 3, seed=s) for s in range(4)]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for s in range(4):
        if s in (1, 2):
            vft.reconfigure_async(ctxs[s])
        elif s == 3:
            vft.reconfigure(ctxs[s])
        assert _blend_call(vft, blend[s])(rig, 8.0, (30.0 * s, 5.0, 0.0), st.cuda_stream)
        for o in plain[s].outs:
            o.zero_()
        assert vft.make_frame_call(plain[s].in_planes, plain[s].out_planes, plain[s].dims)(st.cuda_stream)
    st.synchronize()
    for s in range(4):
        want, _ = want_blend(blend[s], ctxs[s], rig, 8.0, (30.0 * s, 5.0, 0.0))
        for p, got in enumerate(blend[s].host()):
            _check(got, want[p], f"blend frame {s}, plane {p}")
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
def test_two_tone_source_blends_across_the_belt(torch_cuda):
    """A dual-fisheye luma plane whose lens 0 half is flat 60 and lens 1 half flat 200, to EQUIRECT: along the equator
    from lens 0's centre to lens 1's, the blend rises monotonically from 60 to 200 through intermediate values, over the
    belt only; the hard-seam lens call on the same frame jumps from 60 to 200 between two adjacent columns."""
    torch = torch_cuda
    rig = make_rig("pair_190", seed=81)
    in_w, in_h, w, h, seam = 2000, 1000, 720, 361, 6.0  # (a 6-degree belt stays 10 px clear of the circles' rims)
    src = np.full((in_h, in_w), 60, np.uint8)
    src[:, in_w // 2:] = 200
    ctx = t360.make_context(output_layout=t360.LAYOUT_EQUIRECT, interpolation_alg=t360.CUBIC, **LENS_CTX)
    d_src = torch.from_numpy(src).cuda()
    outs = [torch.zeros((h, w), dtype=torch.uint8, device="cuda") for _ in range(2)]
    planes = lambda t: [(t.data_ptr(), t.stride(0))]
    vft = t360.VideoFrameTransform(ctx)
    assert vft.make_lens_blend_frame_call(planes(d_src), planes(outs[0]), [(in_w, in_h, w, h)])(rig, seam, (0, 0, 0), 0)
    assert vft.make_lens_frame_call(planes(d_src), planes(outs[1]), [(in_w, in_h, w, h)])(rig, (0, 0, 0), 0)
    torch.cuda.synchronize()
    blended, hard = (o.cpu().numpy()[h // 2, w // 2:].astype(np.int32) for o in outs)
    assert blended[0] == 60 and blended[-1] == 200 and (np.diff(blended) >= 0).all()
    ramp = int(((blended > 60) & (blended < 200)).sum())
    assert abs(ramp - seam / 360 * w) <= 2, f"{ramp} intermediate columns"
    assert len(np.unique(blended)) >= 8
    _, _, wt = t360.lens_blend_maps(ctx, rig, seam, (0, 0, 0), in_w, in_h, w, h)
    row_w = wt[h // 2, w // 2:].astype(np.int32)
    assert np.array_equal(blended, (60 * (256 - row_w) + 200 * row_w + 128) >> 8)
    steps = np.flatnonzero(np.diff(hard))
    assert hard[0] == 60 and hard[-1] == 200 and len(steps) == 1 and hard[steps[0] + 1] - hard[steps[0]] == 140
    vft.close()


@pytest.mark.gpu
def test_device_memory_and_launches_stay_bounded(torch_cuda):
    """50 blend frames after a warm-up, a new orientation every frame: one kernel launch each (the chroma pre-fill is a
    memset) and no growth of device memory."""
    torch = torch_cuda
    ctx = t360.make_context(output_layout=t360.LAYOUT_CUBEMAP_32, interpolation_alg=t360.LANCZOS4, **LENS_CTX)
    rig = make_rig("tilted", 91)
    vft = t360.VideoFrameTransform(ctx)
    f = Frame(torch, 3)
    call = _blend_call(vft, f)
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for i in range(5):
        assert call(rig, 10.0, (7.0 * i, 1.0, 0.0), st.cuda_stream)
    st.synchronize()
    free_before = torch.cuda.mem_get_info()[0]
    n0 = t360.kernel_launch_count()
    for i in range(50):
        assert call(rig, 4.0 + i % 3, (7.0 * i, 3.0 * np.sin(i), -2.0), st.cuda_stream)
    launches = t360.kernel_launch_count() - n0
    st.synchronize()
    assert launches == 50, f"{launches} launches for 50 frames"
    assert torch.cuda.mem_get_info()[0] >= free_before - (2 << 20), "device memory grew over blend frames"
    vft.close()


@pytest.mark.gpu
def test_refused_calls_launch_nothing_and_leave_the_outputs(torch_cuda, capfd):
    """Refused blend frames on real planes: no kernel launch, the outputs keep their bytes (chroma included)."""
    torch = torch_cuda
    for what, rig, seam, o, ov in _bad_blend_calls():
        if rig is None or o is None:
            continue  # (make_lens_blend_frame_call takes a rig and an orientation; the NULL cases are covered without a GPU)
        ctx = t360.make_context(**{**LENS_CTX, "output_layout": t360.LAYOUT_EQUIRECT, **ov})
        with t360.VideoFrameTransform(ctx) as vft:
            f = Frame(torch, 3)
            before = f.host()
            torch.cuda.synchronize()
            n0 = t360.kernel_launch_count()
            _refused(capfd, _blend_call(vft, f), rig, seam, o, 0)
            torch.cuda.synchronize()
            assert t360.kernel_launch_count() == n0, what
            for p, (a, b) in enumerate(zip(before, f.host())):
                assert np.array_equal(a, b), f"{what}: plane {p} changed"
