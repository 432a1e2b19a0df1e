"""Fisheye lens rigs with photometry: each lens's samples corrected for vignetting, gain and offset before the hard or the
feathered seam, and the overlap's statistics from the same launch (T360B200_lensPhotoMaps / lens_photo_maps,
T360B200_transformFrameLensPhotoAsync / make_lens_photo_frame_call).

What pins what:
  - the identity photometry against lens_map (hard seam) and lens_blend_maps (feathered seam): the twin's maps and weights
    are theirs, bit for bit, and every covered gain is 4096;
  - the gains against a float64 model of the header's falloff, 4096 gain_p / V(theta_d), within 1;
  - the frames against a composite of the plain-C oracle's cv::remap of both maps under BORDER_TRANSPARENT, corrected and
    combined with the header's integer rules, bit for bit; the statistics against the same composite's int64 sums.
Rigs, orientations, photometries and planes are made from seeds."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import transform360_b200 as t360
from oracle import c_oracle as co
from tests.test_lens import IN_DIMS, LAYOUTS, LENS_CTX, OUT_DIMS, Frame, _orientations, _pattern, _rot, directions, make_rig
from tests.test_lens_blend import INTERPS, composite
from tests.test_warp_map import _check, _refused

TRANSPARENT = t360.BORDER_TRANSPARENT
STATS = 6


def photometry(pivot=16, vignetting=((0, 0, 0), (0, 0, 0)), gain=((1, 1, 1), (1, 1, 1)), offset=((0, 0, 0), (0, 0, 0))):
    """A T360RigPhotometry from per-lens triples; the defaults are the identity."""
    ph = t360.T360RigPhotometry(int(pivot))
    for i in range(2):
        ph.lens[i].vignetting[:] = [float(x) for x in vignetting[i]]
        ph.lens[i].gain[:] = [float(x) for x in gain[i]]
        ph.lens[i].offset[:] = [float(x) for x in offset[i]]
    return ph


IDENTITY = photometry()


def r_max(lens):
    """theta_d(maxAngle) of a lens, in double as the library's refusal computes it."""
    t = np.radians(np.float64(lens.maxAngle))
    k = [np.float64(x) for x in lens.k]
    return t * (1 + t * t * (k[0] + t * t * (k[1] + t * t * (k[2] + t * t * k[3]))))


def rig_photos(rig):
    """The photometries of the frame tests, their falloffs scaled to the rig's theta_d(maxAngle) R so that V(R) is what the
    name says whatever the seeded distortion: "identity"; "falloff", V(R) = 0.7 and 0.6 with unequal gains per plane and
    offsets in 1/16 code value steps and between them; "clamps", lens 0 driving its samples into both the 0 and the 255
    clamp, lens 1 reaching Gq's clamp (G >= 16) towards its rim (V(R) = 0.4, gain 8)."""
    R = [r_max(rig.lens[min(i, rig.numLenses - 1)]) ** 2 for i in range(2)]
    return {
        "identity": IDENTITY,
        "falloff": photometry(16, ((-0.36 / R[0], 0.06 / R[0] ** 2, 0.0), (-0.5 / R[1], 0.12 / R[1] ** 2, -0.02 / R[1] ** 3)),
                              ((1.1, 0.95, 1.05), (0.8, 1.2, 0.9)), ((3.3, -2.5, 1.03125), (-4.0, 5.5, -0.53))),
        "clamps": photometry(0, ((0.0, 0.0, 0.0), (-0.6 / R[1], 0.0, 0.0)), ((6.0, 5.0, 7.5), (8.0, 8.0, 8.0)),
                             ((-60.0, -64.0, -50.0), (64.0, 30.0, -10.0))),
    }


# (rig, seamWidth): the hard seam of one and of two lenses, and the feathered seam
MODES = {"one": ("single_200", 0.0), "hard": ("pair_190", 0.0), "feathered": ("tilted", 8.0)}


def offset_q(offset):
    """Oq = round(16 offset), half away from zero (computed in double)."""
    x = 16.0 * np.float64(np.float32(offset))
    return int(np.sign(x) * np.floor(abs(x) + 0.5))


def correct(s, gq, oq, pivot):
    """s' of the header, in int64."""
    s, gq = s.astype(np.int64), gq.astype(np.int64)
    return np.clip(pivot + (((s - pivot) * gq + oq * 256 + 2048) >> 12), 0, 255)


def photo_composite(src, maps, interp, prefill, ph, plane):
    """The oracle's frame and statistics: cv::remap of each map under BORDER_TRANSPARENT (into 0 and into 255: where the
    two differ the sample is skipped), s' per lens, then lens 0's alone where w = 0, lens 1's where w = 256, the blend
    elsewhere (the other alone where one is skipped), the pre-fill where nothing is sampled; the sums n, a', b', a'^2,
    b'^2, a'b' (int64) over the pixels where both maps are finite and neither sample is skipped."""
    map0, map1, weight, g0, g1 = maps
    h, w = weight.shape
    pivot = ph.lumaPivot if plane == 0 else 128

    def sample(m, gq, lens):
        lo = co.remap_u8(src, m, interp, TRANSPARENT, np.zeros((h, w), np.uint8))
        hi = co.remap_u8(src, m, interp, TRANSPARENT, np.full((h, w), 255, np.uint8))
        return correct(lo, gq, offset_q(ph.lens[lens].offset[plane]), pivot), lo == hi
    (a, va), (b, vb) = sample(map0, g0, 0), sample(map1, g1, 1)
    wt = weight.astype(np.int64)
    out = prefill.astype(np.int64).copy()
    lone0, lone1, mid = wt == 0, wt == 256, (wt > 0) & (wt < 256)
    out[lone0 & va] = a[lone0 & va]
    out[lone1 & vb] = b[lone1 & vb]
    out[mid & va & ~vb] = a[mid & va & ~vb]
    out[mid & vb & ~va] = b[mid & vb & ~va]
    both = mid & va & vb
    out[both] = (a[both] * (256 - wt[both]) + b[both] * wt[both] + 128) >> 8
    ov = np.isfinite(map0).all(-1) & np.isfinite(map1).all(-1) & va & vb
    sums = [int(ov.sum()), int(a[ov].sum()), int(b[ov].sum()), int((a[ov] ** 2).sum()), int((b[ov] ** 2).sum()), int((a[ov] * b[ov]).sum())]
    return out.astype(np.uint8), sums


def _maps(layout, rig, ph, seam, o, plane, in_w, in_h, w, h, interp=t360.CUBIC):
    ctx = t360.make_context(output_layout=layout, interpolation_alg=interp, **LENS_CTX)
    return t360.lens_photo_maps(ctx, rig, ph, seam, o, plane, in_w, in_h, w, h)


# ---- no GPU needed -----------------------------------------------------------------------------------------------------
def test_lens_photo_entry_points_are_exported_with_their_bindings(tmp_path):
    from transform360_b200.handler import EXPORTED_SYMBOLS, LIB_PATH, PKG
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    L = t360.load()
    for name in ("T360B200_lensPhotoMaps", "T360B200_transformFrameLensPhotoAsync"):
        assert name in EXPORTED_SYMBOLS and name in defined, name
    P = C.POINTER
    assert L.T360B200_lensPhotoMaps.argtypes == ([P(t360.FrameTransformContext), P(t360.T360LensRig), P(t360.T360RigPhotometry), C.c_float,
                                                  P(t360.T360Orientation)] + [C.c_int] * 5 + [C.c_void_p] * 5)
    assert L.T360B200_transformFrameLensPhotoAsync.argtypes == ([C.c_void_p, P(t360.T360LensRig), P(t360.T360RigPhotometry), C.c_float,
                                                                 P(t360.T360Orientation), C.c_void_p, C.c_int] + [C.c_void_p] * 9)
    assert C.sizeof(t360.T360LensPhotometry) == 36 and C.sizeof(t360.T360RigPhotometry) == 76
    assert hasattr(t360.VideoFrameTransform, "make_lens_photo_frame_call") and callable(t360.lens_photo_maps)
    src = tmp_path / "decl.c"
    src.write_text('#include "transform360_b200.h"\n'
                   "_Static_assert(sizeof(T360LensPhotometry) == 36 && sizeof(T360RigPhotometry) == 76, \"layout\");\n"
                   "int (*maps)(const FrameTransformContext*, const T360LensRig*, const T360RigPhotometry*, float, const T360Orientation*, int, "
                   "int, int, int, int, float*, float*, uint16_t*, uint16_t*, uint16_t*) = T360B200_lensPhotoMaps;\n"
                   "int (*frame)(VideoFrameTransform*, const T360LensRig*, const T360RigPhotometry*, float, const T360Orientation*, "
                   "unsigned long long*, int, const uint8_t* const*, uint8_t* const*, const int*, const int*, const int*, const int*, "
                   "const int*, const int*, void*) = T360B200_transformFrameLensPhotoAsync;\n")
    subprocess.run(["cc", "-std=c11", "-Wall", "-Werror", "-c", "-I", str(PKG.parent / "include"), "-o", str(tmp_path / "decl.o"), str(src)],
                   check=True)


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_identity_hard_seam_is_the_lens_map(layout):
    """Identity photometry, seamWidth 0: wherever lens i carries the pixel (w = 0 for lens 0, 256 for lens 1) map_i is
    lens_map's entry bit for bit (NaN included), the lens choice follows the float64 model's closer lens, and every gain of
    a covered pixel is 4096.  A one-lens rig gives w = 0, map1 NaN and gain1 0 everywhere."""
    for rig_name in ("single_200", "pair_190", "tilted"):
        rig = make_rig(rig_name, seed=len(layout))
        for o in _orientations(len(layout) + 7, 2):
            for (w, h), (in_w, in_h) in (((97, 65), (259, 131)), ((49, 33), (130, 66))):
                ctx = t360.make_context(output_layout=LAYOUTS[layout], **LENS_CTX)
                hard = t360.lens_map(ctx, rig, o, in_w, in_h, w, h).view(np.uint32)
                for plane in (0, 1):
                    m0, m1, wt, g0, g1 = t360.lens_photo_maps(ctx, rig, IDENTITY, 0.0, o, plane, in_w, in_h, w, h)
                    assert set(np.unique(wt)) <= {0, 256}
                    for lone, mine in ((wt == 0, m0), (wt == 256, m1)):
                        assert np.array_equal(mine.view(np.uint32)[lone], hard[lone]), f"{rig_name} {o} {w}x{h}"
                    for m, g in ((m0, g0), (m1, g1)):
                        cov = np.isfinite(m).all(-1)
                        assert (np.isnan(m[~cov]).all()) and (g[cov] == 4096).all() and (g[~cov] == 0).all()
                    if rig.numLenses == 1:
                        assert (wt == 0).all() and np.isnan(m1).all() and (g1 == 0).all()
                    else:
                        d, dead = directions(dict(output_layout=LAYOUTS[layout]), o, w, h)
                        z = [(d @ _rot(rig.lens[i].yaw, rig.lens[i].pitch, rig.lens[i].roll))[..., 2] for i in range(2)]
                        clear = (np.abs(z[1] - z[0]) > 1e-5) & ~dead
                        assert np.array_equal((wt == 256)[clear], (z[1] > z[0])[clear])


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_identity_feathered_seam_is_the_blend_maps(layout):
    """Identity photometry, seamWidth > 0: w is lens_blend_maps' weight, map_i its map_i wherever that one carries weight,
    and every covered gain is 4096."""
    for rig_name in ("pair_190", "tilted"):
        rig = make_rig(rig_name, seed=len(layout) + 3)
        for o in _orientations(len(layout) + 11, 2):
            for seam in (2.0, 10.0, 40.0):
                ctx = t360.make_context(output_layout=LAYOUTS[layout], **LENS_CTX)
                b0, b1, bw = t360.lens_blend_maps(ctx, rig, seam, o, 259, 131, 97, 65)
                m0, m1, wt, g0, g1 = t360.lens_photo_maps(ctx, rig, IDENTITY, seam, o, 0, 259, 131, 97, 65)
                assert np.array_equal(wt, bw), f"{rig_name} {o} seam {seam}"
                for mine, blend, g in ((m0, b0, g0), (m1, b1, g1)):
                    carry = np.isfinite(blend).all(-1)
                    assert np.array_equal(mine.view(np.uint32)[carry], blend.view(np.uint32)[carry])
                    cov = np.isfinite(mine).all(-1)
                    assert (carry <= cov).all() and (g[cov] == 4096).all() and (g[~cov] == 0).all()


def _falloff(rng, lens):
    """v1..v3 in a range around real lenses' falloffs whose V(r) stays positive up to theta_d(maxAngle) (the library refuses
    the others)."""
    t = np.radians(lens.maxAngle)
    k = list(lens.k)
    r2 = np.square(np.linspace(0, t * (1 + t * t * (k[0] + t * t * (k[1] + t * t * (k[2] + t * t * k[3])))), 4097))
    while True:
        v = rng.uniform([-0.15, -0.02, -0.002], [0.05, 0.03, 0.002])
        if (1 + r2 * (v[0] + r2 * (v[1] + r2 * v[2])) > 0.05).all():
            return tuple(v)


def _mild(rig):
    """rig with its distortion scaled to a tenth: theta_d(maxAngle) about 1.1 theta instead of up to 5 theta, as real
    fisheye calibrations have it.  (With the strongest seeded k the model's directions, exact to about 1e-6 rad, move V
    by more than the 1/4096 the comparison resolves.)"""
    for i in range(rig.numLenses):
        rig.lens[i].k[:] = [0.1 * k for k in rig.lens[i].k]
    return rig


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_gains_equal_the_float64_model(layout):
    """The twin's Gq is within 1 of 4096 gain_p / V(theta_d) in float64 (65535 where that reaches the clamp), for seeded
    falloffs and gains, every plane and both seams, except pixels within 1e-5 rad of a lens's coverage bound."""
    rng = np.random.default_rng(sum(map(ord, layout)))
    worst = 0
    for rig_name in ("equidistant", "tilted", "single_200"):
        rig = equidistant_pair() if rig_name == "equidistant" else _mild(make_rig(rig_name, seed=len(layout) + 1))
        for o in _orientations(len(layout) + 19, 2):
            ph = photometry(int(rng.integers(0, 256)), [_falloff(rng, rig.lens[i if i < rig.numLenses else 0]) for i in range(2)],
                            [tuple(rng.uniform(0.05, 8.0, 3)) for _ in range(2)], [tuple(rng.uniform(-64, 64, 3)) for _ in range(2)])
            d, dead = directions(dict(output_layout=LAYOUTS[layout]), o, 97, 65)
            for plane in (0, 1, 2):
                for seam in ((0.0,) if rig.numLenses == 1 else (0.0, 6.0)):
                    m0, m1, wt, g0, g1 = _maps(LAYOUTS[layout], rig, ph, seam, o, plane, 259, 131, 97, 65)
                    for i, (m, g) in enumerate(((m0, g0), (m1, g1))[:rig.numLenses]):
                        L = rig.lens[i]
                        c = d @ _rot(L.yaw, L.pitch, L.roll)
                        th = np.arctan2(np.hypot(c[..., 0], c[..., 1]), c[..., 2])
                        t_max = np.radians(np.float64(np.float32(L.maxAngle)))
                        k = [np.float64(np.float32(x)) for x in L.k]
                        r2 = (th * (1 + k[0] * th ** 2 + k[1] * th ** 4 + k[2] * th ** 6 + k[3] * th ** 8)) ** 2
                        v = [np.float64(np.float32(x)) for x in ph.lens[i].vignetting]
                        model = 4096 * np.float64(np.float32(ph.lens[i].gain[plane])) / (1 + r2 * (v[0] + r2 * (v[1] + r2 * v[2])))
                        model = np.minimum(model, 65535)
                        sel = (th < t_max - 1e-5) & ~dead
                        assert np.isfinite(m[sel]).all() and np.isnan(m[(th > t_max + 1e-5) & ~dead]).all()
                        err = np.abs(g[sel].astype(np.float64) - model[sel])
                        worst = max(worst, float(err.max()))
    assert worst <= 1.0, f"max |Gq - model| {worst:.3f}"


def equidistant_pair():
    """Back-to-back 190-degree equidistant lenses (k = 0, so theta_d = theta: theta_d(95 degrees) = 1.658) side by side on a
    2000x1000 frame."""
    rig = t360.T360LensRig(2, 2000, 1000)
    for i in range(2):
        rig.lens[i] = t360.T360Lens(300.0, 300.0, 499.5 + 1000 * i, 499.5, (0, 0, 0, 0), 180.0 * i, 0, 0, 95)
    return rig


def _bad_photo_calls():
    """(what, rig or None, photometry or None, seamWidth, orientation or None, context overrides) the calls refuse."""
    pair, single = make_rig("pair_190"), make_rig("single_200")

    def ph_with(lens=0, **kw):
        ph = photometry()
        for key, (k, v) in kw.items():
            getattr(ph.lens[lens], key)[k] = v
        return ph
    cases = [("NULL rig", None, IDENTITY, 0.0, (0, 0, 0), {}), ("NULL orientation", pair, IDENTITY, 0.0, None, {}),
             ("NULL photometry", pair, None, 0.0, (0, 0, 0), {}), ("NULL photometry, feathered", pair, None, 10.0, (0, 0, 0), {})]
    r = make_rig("pair_190")
    r.numLenses = 3
    cases.append(("numLenses 3", r, IDENTITY, 0.0, (0, 0, 0), {}))
    r = make_rig("pair_190")
    r.lens[1].maxAngle = 181.0
    cases.append(("maxAngle 181", r, IDENTITY, 0.0, (0, 0, 0), {}))
    cases.append(("a feathered seam on one lens", single, IDENTITY, 10.0, (0, 0, 0), {}))
    for seam in (float("nan"), float("inf"), -1.0, -0.0 - 1e-30, 0.005, 181.0):
        cases.append((f"seamWidth {seam}", pair, IDENTITY, seam, (0, 0, 0), {}))
    for pivot in (-1, 256):
        cases.append((f"lumaPivot {pivot}", pair, photometry(pivot), 0.0, (0, 0, 0), {}))
    for lens in (0, 1):
        for field in ("vignetting", "gain", "offset"):
            cases.append((f"lens {lens} {field} nan", pair, ph_with(lens, **{field: (lens, float("nan"))}), 0.0, (0, 0, 0), {}))
        for g in (0.0, -1.0, 8.001, float("inf")):
            cases.append((f"lens {lens} gain {g}", pair, ph_with(lens, gain=(2, g)), 10.0, (0, 0, 0), {}))
        for off in (-64.01, 64.5):
            cases.append((f"lens {lens} offset {off}", pair, ph_with(lens, offset=(1, off)), 0.0, (0, 0, 0), {}))
    # V(r) <= 0 inside theta_d(maxAngle) = 1.658: 1 - 0.37 r^2 reaches 0 at r = 1.644, 1 - 0.1 r^6 at 1.468
    eq = equidistant_pair()
    for lens in (0, 1):
        cases.append((f"lens {lens} falloff reaches 0", eq, ph_with(lens, vignetting=(0, -0.37)), 0.0, (0, 0, 0), {}))
    cases.append(("falloff reaches 0 through v3", eq, ph_with(0, vignetting=(2, -0.1)), 10.0, (0, 0, 0), {}))
    cases.append(("orientation nan", pair, IDENTITY, 0.0, (float("nan"), 0, 0), {}))
    for ov in (dict(output_layout=t360.LAYOUT_FLAT_FIXED), dict(enable_low_pass_filter=1), dict(interpolation_alg=3)):
        cases.append((str(ov), pair, IDENTITY, 0.0, (0, 0, 0), ov))
    return cases


def _photo_frame(L, vft, rig, ph, seam, o, stats=None, n=1, planes=(0x20000,), dims=(64, 32, 8, 8), pitch=(64, 8)):
    P, I = C.c_void_p * 3, C.c_int * 3
    arr = lambda v: I(*([v] * 3))
    ob = C.byref(t360.T360Orientation(*o)) if o is not None else None
    return L.T360B200_transformFrameLensPhotoAsync(vft._h, C.byref(rig) if rig is not None else None, C.byref(ph) if ph is not None else None,
                                                   seam, ob, stats, n, P(*(list(planes) * 3)[:3]), P(*(list(planes) * 3)[:3]), arr(dims[0]),
                                                   arr(dims[1]), arr(pitch[0]), arr(dims[2]), arr(dims[3]), arr(pitch[1]), None)


def test_refusals_happen_without_a_gpu(capfd):
    """Every refusal of lens_photo_maps and of the photometric frame call comes with a message and before any CUDA call (this
    machine may have none): fake device addresses, the statistics buffer's included, are never dereferenced.  A one-lens rig
    does not read lens[1]'s photometry, and a falloff that stays positive is accepted."""
    L = t360.load()
    m0, m1 = np.zeros((8, 8, 2), np.float32), np.zeros((8, 8, 2), np.float32)
    wt, g0, g1 = (np.zeros((8, 8), np.uint16) for _ in range(3))
    arrays = (m0.ctypes.data, m1.ctypes.data, wt.ctypes.data, g0.ctypes.data, g1.ctypes.data)
    for what, rig, ph, seam, o, ov in _bad_photo_calls():
        ctx = t360.make_context(**{**LENS_CTX, "output_layout": t360.LAYOUT_EQUIRECT, **ov})
        ob = C.byref(t360.T360Orientation(*o)) if o is not None else None
        out = _refused(capfd, L.T360B200_lensPhotoMaps, C.byref(ctx), C.byref(rig) if rig is not None else None,
                       C.byref(ph) if ph is not None else None, seam, ob, 0, 64, 32, 8, 8, *arrays)
        assert "Error" in out, what
        with t360.VideoFrameTransform(ctx) as vft:
            _refused(capfd, _photo_frame, L, vft, rig, ph, seam, o, 0x40000)
    ctx = t360.make_context(output_layout=t360.LAYOUT_EQUIRECT, **LENS_CTX)
    pair, o = make_rig("pair_190"), C.byref(t360.T360Orientation())
    for plane in (-1, 3):
        _refused(capfd, L.T360B200_lensPhotoMaps, C.byref(ctx), C.byref(pair), C.byref(IDENTITY), 0.0, o, plane, 64, 32, 8, 8, *arrays)
    for k in range(5):
        bad = list(arrays)
        bad[k] = None
        _refused(capfd, L.T360B200_lensPhotoMaps, C.byref(ctx), C.byref(pair), C.byref(IDENTITY), 0.0, o, 0, 64, 32, 8, 8, *bad)
    _refused(capfd, L.T360B200_lensPhotoMaps, C.byref(ctx), C.byref(pair), C.byref(IDENTITY), 0.0, o, 0, 0, 32, 8, 8, *arrays)
    _refused(capfd, L.T360B200_lensPhotoMaps, None, C.byref(pair), C.byref(IDENTITY), 0.0, o, 0, 64, 32, 8, 8, *arrays)
    with pytest.raises(ValueError):
        t360.lens_photo_maps(ctx, pair, IDENTITY, 0.005, (0, 0, 0), 0, 64, 32, 8, 8)
    with t360.VideoFrameTransform(ctx) as vft:
        for kw in (dict(n=0), dict(n=4), dict(planes=(None,)), dict(dims=(0, 32, 8, 8)), dict(pitch=(63, 8))):
            _refused(capfd, lambda: _photo_frame(L, vft, pair, IDENTITY, 0.0, (0, 0, 0), **kw))
    assert not L.T360B200_transformFrameLensPhotoAsync(None, None, None, 0.0, None, None, 1, None, None, None, None, None, None, None, None,
                                                       None)
    # accepted: lens[1] of a one-lens rig is not read; a strong falloff that stays positive inside the coverage
    single = make_rig("single_200")
    junk = photometry(gain=((1, 1, 1), (float("nan"), 0, 99)), vignetting=((0, 0, 0), (float("nan"), 0, 0)))
    assert t360.lens_photo_maps(ctx, single, junk, 0.0, (0, 0, 0), 0, 64, 32, 8, 8)[3].max() > 0
    assert t360.lens_photo_maps(ctx, equidistant_pair(), photometry(vignetting=((-0.35, 0, 0), (-0.35, 0, 0))), 0.0, (0, 0, 0), 0, 64, 32, 8, 8)


# ---- on the GPU --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests must run on an H100 (there is no CPU fallback to test)")
    return torch


def want_photo(f, ctx, rig, ph, seam, o):
    """The oracle's planes of Frame f (luma pre-filled with its pattern, chroma with 128) and the statistics per plane."""
    want, sums = [], []
    for p in range(f.n):
        maps = t360.lens_photo_maps(ctx, rig, ph, seam, o, p, *IN_DIMS[p], *OUT_DIMS[p])
        prefill = _pattern(*OUT_DIMS[p], p) if p == 0 else np.full(OUT_DIMS[p][::-1], 128, np.uint8)
        out, s = photo_composite(f.src[p], maps, ctx.interpolation_alg, prefill, ph, p)
        want.append(out)
        sums.append(s)
    return want, sums


def _photo_call(vft, f):
    return vft.make_lens_photo_frame_call(f.in_planes, f.out_planes, f.dims)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("interp", INTERPS)
def test_photo_frames_and_statistics_equal_the_oracle(layout, interp, torch_cuda):
    """For the hard seam of one and of two lenses and the feathered seam, with each photometry: 3-plane frames equal the
    oracle's composite bit for bit, with and without statistics (the same bytes), and the statistics equal its int64 sums
    exactly; a 1-plane frame too."""
    torch = torch_cuda
    ctx = t360.make_context(output_layout=LAYOUTS[layout], interpolation_alg=interp, **LENS_CTX)
    vft = t360.VideoFrameTransform(ctx)
    st = torch.cuda.Stream()
    stats = torch.zeros((3, STATS), dtype=torch.int64, device="cuda")
    for m, (mode, (rig_name, seam)) in enumerate(sorted(MODES.items())):
        rig = make_rig(rig_name, seed=interp + 3 * m)
        o = _orientations(interp * 10 + len(layout) + m, 1)[0]
        for ph_name, ph in sorted(rig_photos(rig).items()):
            for n in (3, 1):
                if n == 1 and ph_name != "falloff":
                    continue
                f = Frame(torch, n, seed=interp + m)
                want, sums = want_photo(f, ctx, rig, ph, seam, o)
                what = f"{mode} seam, photometry {ph_name}, {n} planes"
                for with_stats in (False, True):
                    f.reset()
                    stats.fill_(-1)
                    torch.cuda.synchronize()
                    assert _photo_call(vft, f)(rig, ph, seam, o, st.cuda_stream, stats.data_ptr() if with_stats else 0)
                    st.synchronize()
                    for p, got in enumerate(f.host()):
                        _check(got, want[p], f"{what}, statistics {with_stats}, plane {p}")
                    got_sums = stats.cpu().numpy()
                    if with_stats:
                        for p in range(n):
                            assert got_sums[p].tolist() == sums[p], f"{what}: plane {p} statistics {got_sums[p].tolist()} != {sums[p]}"
                        assert (got_sums[n:] == -1).all(), "the call wrote past its planes' statistics"
                        if rig.numLenses == 1:
                            assert (got_sums[:n] == 0).all()
                        else:
                            assert got_sums[0][0] > 0, f"{what}: no overlap pixel"
                    else:
                        assert (got_sums == -1).all()
    vft.close()


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["equirect", "cubemap_32", "barrel"])
def test_identity_photometry_equals_the_lens_and_blend_calls(layout, torch_cuda):
    """Identity photometry on a 1440x720 dual-fisheye yuv420p frame: seamWidth 0 gives T360B200_transformFrameLensAsync's
    frame and seamWidth > 0 T360B200_transformFrameLensBlendAsync's, byte for byte, every interpolator, with statistics on."""
    torch = torch_cuda
    rig = make_rig("pair_190", seed=5)
    dims = [(1440, 720, 768, 512), (720, 360, 384, 256), (720, 360, 384, 256)]
    src = [torch.from_numpy(co.noise_plane(w, h, plane=p, frame=3)).cuda() for p, (w, h, _, _) in enumerate(dims)]
    outs = [[torch.full((oh, ow), 7 + p, dtype=torch.uint8, device="cuda") for p, (_, _, ow, oh) in enumerate(dims)] for _ in range(2)]
    planes = lambda ts: [(t.data_ptr(), t.stride(0)) for t in ts]
    stats = torch.zeros((3, STATS), dtype=torch.int64, device="cuda")
    for interp in INTERPS:
        ctx = t360.make_context(output_layout=LAYOUTS[layout], interpolation_alg=interp, **LENS_CTX)
        with t360.VideoFrameTransform(ctx) as vft:
            photo = vft.make_lens_photo_frame_call(planes(src), planes(outs[0]), dims)
            for seam, o in ((0.0, (20.0, 5.0, -3.0)), (4.0, (-70.0, 10.0, 2.0)), (10.0, (100.0, -30.0, 0.0))):
                for a, b in zip(*outs):
                    a.fill_(9)
                    b.fill_(9)
                if seam:
                    assert vft.make_lens_blend_frame_call(planes(src), planes(outs[1]), dims)(rig, seam, o, 0)
                else:
                    assert vft.make_lens_frame_call(planes(src), planes(outs[1]), dims)(rig, o, 0)
                assert photo(rig, IDENTITY, seam, o, 0, stats.data_ptr())
                torch.cuda.synchronize()
                for p, (a, b) in enumerate(zip(*outs)):
                    assert torch.equal(a, b), f"interp {interp}, seam {seam}, plane {p}: {int((a != b).sum())} bytes differ"


def _render_rig(rig, in_w, in_h, falloff, exposure, scene):
    """A dual-fisheye luma plane of an equidistant rig (k = 0): each lens's circle shows scene(d) V(r) exposure_i of the
    direction d its pixel sees, V(r) = 1 + falloff r^2, rounded; 0 outside the circles."""
    y, x = np.mgrid[:in_h, :in_w].astype(np.float64)
    out = np.zeros((in_h, in_w))
    for i in range(2):
        L = rig.lens[i]
        xp = ((x + 0.5) * rig.calibWidth / in_w - 0.5 - L.cx) / L.fx
        yp = ((y + 0.5) * rig.calibHeight / in_h - 0.5 - L.cy) / L.fy
        r = np.hypot(xp, yp)
        inside = (r <= np.radians(L.maxAngle)) & ((x < in_w / 2) if i == 0 else (x >= in_w / 2))
        s = np.where(r > 0, np.sin(r) / np.where(r > 0, r, 1), 1.0)
        cam = np.stack([xp * s, -yp * s, np.cos(r)], -1)  # (camera y down -> up)
        d = cam @ _rot(L.yaw, L.pitch, L.roll).T
        out[inside] = (scene(d) * (1 + falloff * r * r) * exposure[i])[inside]
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


@pytest.mark.gpu
def test_auto_exposure_loop_converges(torch_cuda):
    """A back-to-back 190-degree rig whose lens 1 half is rendered 1.3x brighter than lens 0's, both with the falloff
    V(r) = 1 - 0.1 r^2, to EQUIRECT with a 6-degree belt.  Starting from unit gains and the true falloff, the loop of
    INTEGRATION.md (g1 *= sqrt(sum a' / sum b'), g0 *= sqrt(sum b' / sum a'), smoothed by an exponent 0.7) brings the
    overlap's ratio to 1 +- 1 % within 10 frames, and the luma step across the belt below 1 code value (from about 30)."""
    torch = torch_cuda
    rig = equidistant_pair()
    in_w, in_h, w, h, seam = 2000, 1000, 720, 360, 6.0
    scene = lambda d: 110 + 40 * d[..., 1]  # brightness by elevation only: every equirect row is flat
    src = torch.from_numpy(_render_rig(rig, in_w, in_h, -0.1, (1.0, 1.3), scene)).cuda()
    out = torch.zeros((h, w), dtype=torch.uint8, device="cuda")
    stats = torch.zeros((1, STATS), dtype=torch.int64, device="cuda")
    ctx = t360.make_context(output_layout=t360.LAYOUT_EQUIRECT, interpolation_alg=t360.CUBIC, **LENS_CTX)
    vft = t360.VideoFrameTransform(ctx)
    call = vft.make_lens_photo_frame_call([(src.data_ptr(), src.stride(0))], [(out.data_ptr(), out.stride(0))], [(in_w, in_h, w, h)])
    g0, g1 = 1.0, 1.0
    # the belt's outer edges on the equator, 2 degrees clear of it, at both seams (lon -90 and +90: columns w/4 and 3w/4)
    cols = [(int(c - (seam / 2 + 2) * w / 360), int(c + (seam / 2 + 2) * w / 360)) for c in (w // 4, 3 * w // 4)]
    rows = slice(h // 3, 2 * h // 3)

    def step():
        img = out.cpu().numpy().astype(np.float64)
        return max(float(np.abs(img[rows, a] - img[rows, b]).mean()) for a, b in cols)
    ratios, steps = [], []
    for frame in range(10):
        ph = photometry(0, ((-0.1, 0, 0), (-0.1, 0, 0)), ((g0, 1, 1), (g1, 1, 1)))
        assert call(rig, ph, seam, (0, 0, 0), 0, stats.data_ptr())
        torch.cuda.synchronize()
        n, sa, sb = (int(v) for v in stats[0, :3].cpu())
        assert n > 1000
        ratios.append(sa / sb)
        steps.append(step())
        g1 *= (sa / sb) ** (0.7 / 2)
        g0 *= (sb / sa) ** (0.7 / 2)
    print("ratios", [f"{r:.4f}" for r in ratios], "steps", [f"{s:.2f}" for s in steps])
    assert abs(ratios[0] - 1 / 1.3) < 0.03 and steps[0] > 20
    assert abs(ratios[-1] - 1) < 0.01, ratios
    assert steps[-1] < 1.0, steps
    vft.close()


@pytest.mark.gpu
def test_trajectory_with_rig_photometry_and_seam_changes_on_two_streams(torch_cuda):
    """24 frames with a new orientation, photometry and seam every frame (hard and feathered in turn), the rig replaced
    at frame 12, enqueued on two streams in turn with a statistics buffer each frame and no synchronisation between them:
    every frame and its statistics equal the oracle (and so the frames serial calls give)."""
    torch = torch_cuda
    ctx = t360.make_context(output_layout=t360.LAYOUT_EQUIRECT, interpolation_alg=t360.CUBIC, **LENS_CTX)
    rigs = [make_rig("pair_190", 61), make_rig("tilted", 62)]
    rng = np.random.default_rng(21)
    traj = np.cumsum(rng.normal(0, [6, 2, 2], (24, 3)), 0)
    phs = [photometry(16, [tuple(rng.uniform([-0.5, -0.1, 0], [0, 0.1, 0.01]) / r_max(rigs[f >= 12].lens[i]) ** np.array([2, 4, 6]))
                           for i in range(2)],
                      [tuple(rng.uniform(0.7, 1.4, 3)) for _ in range(2)], [tuple(rng.uniform(-8, 8, 3)) for _ in range(2)]) for f in range(24)]
    seams = [0.0 if f % 2 else 3.0 + f % 5 for f in range(24)]
    vft = t360.VideoFrameTransform(ctx)
    frames = [Frame(torch, 3, seed=f % 4) for f in range(24)]
    stats = torch.zeros((24, 3, STATS), dtype=torch.int64, device="cuda")
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for f, fr in enumerate(frames):
        assert _photo_call(vft, fr)(rigs[f >= 12], phs[f], seams[f], tuple(traj[f]), streams[f % 2].cuda_stream, stats[f].data_ptr())
    for s in streams:
        s.synchronize()
    got_stats = stats.cpu().numpy()
    for f, fr in enumerate(frames):
        want, sums = want_photo(fr, ctx, rigs[f >= 12], phs[f], seams[f], tuple(traj[f]))
        for p, got in enumerate(fr.host()):
            _check(got, want[p], f"frame {f}, plane {p}")
            assert got_stats[f, p].tolist() == sums[p], f"frame {f}, plane {p} statistics"
    vft.close()


@pytest.mark.gpu
def test_device_memory_and_launches_stay_bounded(torch_cuda):
    """60 photometric frames after a warm-up, hard and feathered seams, statistics on and off in turn: one kernel launch
    each (zeroing the statistics is a memset) and no growth of device memory."""
    torch = torch_cuda
    ctx = t360.make_context(output_layout=t360.LAYOUT_CUBEMAP_32, interpolation_alg=t360.LANCZOS4, **LENS_CTX)
    rig = make_rig("tilted", 91)
    vft = t360.VideoFrameTransform(ctx)
    f = Frame(torch, 3)
    call = _photo_call(vft, f)
    stats = torch.zeros((3, STATS), dtype=torch.int64, device="cuda")
    st = torch.cuda.Stream()
    ph = rig_photos(rig)["falloff"]
    torch.cuda.synchronize()
    for i in range(6):
        assert call(rig, ph, 4.0 * (i % 2), (7.0 * i, 1.0, 0.0), st.cuda_stream, stats.data_ptr() if i % 3 else 0)
    st.synchronize()
    free_before = torch.cuda.mem_get_info()[0]
    n0 = t360.kernel_launch_count()
    for i in range(60):
        assert call(rig, ph, 4.0 * (i % 2), (7.0 * i, 3.0 * np.sin(i), -2.0), st.cuda_stream, stats.data_ptr() if i % 3 else 0)
    launches = t360.kernel_launch_count() - n0
    st.synchronize()
    assert launches == 60, f"{launches} launches for 60 frames"
    assert torch.cuda.mem_get_info()[0] >= free_before - (2 << 20), "device memory grew over photometric frames"
    vft.close()


@pytest.mark.gpu
def test_refused_calls_launch_nothing_and_leave_the_outputs(torch_cuda, capfd):
    """Refused photometric frames on real planes and a real statistics buffer: no kernel launch, the outputs and the
    statistics keep their bytes."""
    torch = torch_cuda
    L = t360.load()
    stats = torch.full((3, STATS), 5, dtype=torch.int64, device="cuda")
    for what, rig, ph, seam, o, ov in _bad_photo_calls():
        ctx = t360.make_context(**{**LENS_CTX, "output_layout": t360.LAYOUT_EQUIRECT, **ov})
        with t360.VideoFrameTransform(ctx) as vft:
            f = Frame(torch, 3)
            before = f.host()
            torch.cuda.synchronize()
            n0 = t360.kernel_launch_count()
            if rig is None or ph is None or o is None:
                _refused(capfd, _photo_frame, L, vft, rig, ph, seam, o, stats.data_ptr(), 3, [p for p, _ in f.in_planes],
                         tuple(IN_DIMS[0]) + tuple(OUT_DIMS[0]), (f.in_planes[0][1], f.out_planes[0][1]))
            else:
                _refused(capfd, _photo_call(vft, f), rig, ph, seam, o, 0, stats.data_ptr())
            torch.cuda.synchronize()
            assert t360.kernel_launch_count() == n0, what
            for p, (a, b) in enumerate(zip(before, f.host())):
                assert np.array_equal(a, b), f"{what}: plane {p} changed"
            assert (stats.cpu() == 5).all(), f"{what}: the statistics changed"
