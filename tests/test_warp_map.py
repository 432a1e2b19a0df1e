"""Warp-map transforms: frames remapped through the caller's own CV_32FC2 map, planned once (T360B200_generateMapFromWarp,
VideoFrameTransform.generate_map_from_warp, HostPlan.from_warp) or passed per frame in device memory
(T360B200_remapFrameAsync, make_remap_frame_call, FrameTransformer.remap_frame_call).

The split that makes this checkable: the map is the caller's, the sampling is cv::remap's.  The host records are pinned
against cv2.convertMaps, the gather plans of every map family against the invariants tests/test_gather_plan.py checks for
context plans, and the frames of every entry point against the plain-C oracle's cv::remap (oracle.c_oracle.remap_u8), which
tests/test_oracle_pin.py pins against cv2.remap for arbitrary maps.  Maps are made in numpy from a seed."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import tests.test_gather_plan as tgp
import transform360_b200 as t360
from oracle import c_oracle as co
from tests.golden.cases import SMALL
from transform360_b200.stream import FrameTransformer, StreamSpec

WRAP, TRANSPARENT = t360.BORDER_WRAP, t360.BORDER_TRANSPARENT
INTERPS = [t360.NEAREST, t360.LINEAR, t360.CUBIC, t360.LANCZOS4]
KSIZE = {t360.NEAREST: 1, t360.LINEAR: 2, t360.CUBIC: 4, t360.LANCZOS4: 8}
WARP_CTX = dict(enable_low_pass_filter=0)


# ---- map families (numpy, seeded) --------------------------------------------------------------------------------------
def _rotation(yaw, pitch=0.0, roll=0.0):
    y, p, r = np.radians([yaw, pitch, roll])
    ry = np.array([[np.cos(y), 0, np.sin(y)], [0, 1, 0], [-np.sin(y), 0, np.cos(y)]])
    rx = np.array([[1, 0, 0], [0, np.cos(p), -np.sin(p)], [0, np.sin(p), np.cos(p)]])
    rz = np.array([[np.cos(r), -np.sin(r), 0], [np.sin(r), np.cos(r), 0], [0, 0, 1]])
    return ry @ rx @ rz


def dual_fisheye(out_w, out_h, in_w, in_h, fov=190.0, yaw=0.0, pitch=0.0, roll=0.0, outside="nan"):
    """Equirect output from two equidistant fisheye circles side by side (the front lens on the left, the back lens on the
    right, each a circle of diameter in_h).  Each direction is taken from the lens it is closer to the axis of; the last
    2 degrees before 90 off-axis lie outside the usable image circle (a stitcher's mask) and get NaN or (-1, 0)."""
    lon = ((np.arange(out_w) + 0.5) / out_w * 2 - 1) * np.pi
    lat = (0.5 - (np.arange(out_h) + 0.5) / out_h) * np.pi
    lon, lat = np.meshgrid(lon, lat)
    d = np.stack([np.cos(lat) * np.sin(lon), np.sin(lat), np.cos(lat) * np.cos(lon)], -1) @ _rotation(yaw, pitch, roll).T
    front = d[..., 2] >= 0
    dx = np.where(front, d[..., 0], -d[..., 0])
    dz = np.abs(d[..., 2])
    theta = np.arccos(np.clip(dz, -1, 1))
    phi = np.arctan2(d[..., 1], dx)
    radius = in_h / 2.0
    r = theta / np.radians(fov / 2) * radius
    cx = np.where(front, in_w / 4.0, 3 * in_w / 4.0)
    m = np.stack([cx + r * np.cos(phi) - 0.5, in_h / 2.0 - r * np.sin(phi) - 0.5], -1)
    out = theta > np.radians(88.0)
    m[out] = np.nan if outside == "nan" else (-1.0, 0.0)
    return m.astype(np.float32)


def fisheye_undistort(out_w, out_h, in_w, in_h, seed=1):
    """Rectilinear output from one fisheye lens with OpenCV's fisheye model theta_d = theta (1 + k1 t^2 + .. + k4 t^8)."""
    rng = np.random.default_rng(seed)
    k = rng.uniform(-0.05, 0.05, 4)
    f_out = out_w / 2.0 / np.tan(np.radians(50))
    f_in = min(in_w, in_h) / np.pi
    x, y = np.meshgrid((np.arange(out_w) - (out_w - 1) / 2) / f_out, (np.arange(out_h) - (out_h - 1) / 2) / f_out)
    rr = np.hypot(x, y)
    th = np.arctan(rr)
    thd = th * (1 + k[0] * th ** 2 + k[1] * th ** 4 + k[2] * th ** 6 + k[3] * th ** 8)
    s = np.where(rr > 0, thd / np.maximum(rr, 1e-12), 1.0)
    return np.stack([(in_w - 1) / 2 + f_in * s * x, (in_h - 1) / 2 + f_in * s * y], -1).astype(np.float32)


def identity(out_w, out_h, in_w, in_h, seed=0):
    """Every output pixel samples the same position scaled to the input (the plain identity when the sizes agree)."""
    x, y = np.meshgrid((np.arange(out_w) + 0.5) * in_w / out_w - 0.5, (np.arange(out_h) + 0.5) * in_h / out_h - 0.5)
    return np.stack([x, y], -1).astype(np.float32)


def noise(out_w, out_h, in_w, in_h, seed=2):
    """Uniform positions over the whole source: no two neighbours are close, the planner's worst case."""
    rng = np.random.default_rng(seed)
    return np.stack([rng.uniform(-0.5, in_w - 0.5, (out_h, out_w)), rng.uniform(-0.5, in_h - 0.5, (out_h, out_w))], -1).astype(np.float32)


def special(out_w, out_h, in_w, in_h, seed=3):
    """NaN, +-inf, +-1e10, values beyond the int16 range, exact 1/64 ties (round half even on the 1/32 grid) and
    coordinates past every edge, mixed with ordinary ones."""
    rng = np.random.default_rng(seed)
    m = np.stack([rng.uniform(-6, in_w + 6, (out_h, out_w)), rng.uniform(-6, in_h + 6, (out_h, out_w))], -1)
    ties = (rng.integers(-64 * 4, 64 * (max(in_w, in_h) + 4), m.shape) * 2 + 1) / 64.0
    m = np.where(rng.random(m.shape) < 0.3, ties, m)
    bad = np.array([np.nan, np.inf, -np.inf, 1e10, -1e10, 40000.5, -40000.5, 32767.9, -32768.7, 2.0 ** 26, -(2.0 ** 26)])
    pick = rng.random(m.shape) < 0.15
    m[pick] = rng.choice(bad, int(pick.sum()))
    return m.astype(np.float32)


FAMILIES = dict(dual_fisheye=dual_fisheye, dual_fisheye_neg=lambda *a, **k: dual_fisheye(*a, outside="neg"),
                fisheye=fisheye_undistort, identity=identity, noise=noise, special=special)


def _sizes(family, n=0):
    """(map w, map h, input w, input h) per family: odd sizes and map sizes other than the input's."""
    return {"dual_fisheye": (257, 129, 512, 256), "dual_fisheye_neg": (200, 100, 384, 192), "fisheye": (241, 135, 333, 331),
            "identity": (160, 90, 160, 90) if n % 2 == 0 else (131, 77, 263, 154), "noise": (97, 61, 203, 101),
            "special": (75, 53, 67, 41)}[family]


# ---- no GPU needed -----------------------------------------------------------------------------------------------------
def test_warp_entry_points_are_exported_with_their_bindings():
    from transform360_b200.handler import EXPORTED_SYMBOLS, LIB_PATH
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    L = t360.load()
    for name in ("T360B200_generateMapFromWarp", "T360B200_hostPlanCreateFromWarp", "T360B200_remapFrameAsync"):
        assert name in EXPORTED_SYMBOLS and name in defined, name
    assert L.T360B200_generateMapFromWarp.argtypes == [C.c_void_p, C.c_void_p] + [C.c_int] * 6
    assert L.T360B200_remapFrameAsync.argtypes == [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 9
    assert (t360.BORDER_WRAP, t360.BORDER_TRANSPARENT) == (3, 5)
    assert hasattr(FrameTransformer, "remap_frame_call") and hasattr(t360.HostPlan, "from_warp")
    assert hasattr(t360.VideoFrameTransform, "generate_map_from_warp") and hasattr(t360.VideoFrameTransform, "make_remap_frame_call")


def _cv2_records(m, k):
    """What cv2.convertMaps makes of the map, as {col0, row0 << 10 | phase} records (nearest: the rounded position)."""
    cv2 = pytest.importorskip("cv2")
    if k == 1:
        xy, _ = cv2.convertMaps(m, None, cv2.CV_16SC2, nninterpolation=True)
        return np.stack([xy[..., 0].astype(np.int64), xy[..., 1].astype(np.int64) << 10], -1)
    xy, frac = cv2.convertMaps(m, None, cv2.CV_16SC2)
    h = k // 2 - 1
    return np.stack([xy[..., 0].astype(np.int64) - h, ((xy[..., 1].astype(np.int64) - h) << 10) | frac.astype(np.int64)], -1)


@pytest.mark.parametrize("family", sorted(FAMILIES))
@pytest.mark.parametrize("interp", INTERPS)
def test_host_records_equal_cv2_convert_maps(family, interp):
    """hostPlanCreateFromWarp's records equal cv2.convertMaps(map, CV_16SC2) wherever a coordinate is finite and its 1/32
    (nearest: whole) value fits an int; elsewhere cv::remap's INT_MIN -> -32768 rule (test_oracle_pin.py): the axis
    samples -32768 with phase 0."""
    k = KSIZE[interp]
    mw, mh, iw, ih = _sizes(family)
    m = FAMILIES[family](mw, mh, iw, ih)
    for border in (WRAP, TRANSPARENT):
        hp = t360.HostPlan.from_warp(t360.make_context(interpolation_alg=interp, **WARP_CTX), m, iw, ih, border)
        assert (hp.map_w, hp.map_h, hp.kernel_size, hp.num_segments) == (mw, mh, k, 0)
        assert np.array_equal(hp.map, m, equal_nan=True)
        got = hp.samples.astype(np.int64)
        want = _cv2_records(m, k)
        scale = 1.0 if k == 1 else 32.0
        with np.errstate(invalid="ignore", over="ignore"):
            ok = np.isfinite(m) & (np.abs(m.astype(np.float64) * scale) < 2.0 ** 31 - 64)
        both = ok.all(-1)
        assert np.array_equal(got[both], want[both]), f"{int((got[both] != want[both]).any(-1).sum())} records differ from cv2"
        h = max(k // 2 - 1, 0)  # (nearest: the rounded position itself)
        col0, row0, phase = got[..., 0], got[..., 1] >> 10, got[..., 1] & 1023
        assert (col0[~ok[..., 0]] == -32768 - h).all() and (row0[~ok[..., 1]] == -32768 - h).all()
        assert ((phase[~ok[..., 0]] & 31) == 0).all() and ((phase[~ok[..., 1]] >> 5) == 0).all()
        if family == "special":
            assert (~ok).any(), "the special family must reach the INT_MIN rule"


@pytest.mark.parametrize("family", sorted(FAMILIES))
@pytest.mark.parametrize("interp", INTERPS)
@pytest.mark.parametrize("border", [WRAP, TRANSPARENT])
def test_gather_plans_of_warp_maps_keep_the_invariants(family, interp, border, monkeypatch):
    """Every map family's gather plan satisfies what tests/test_gather_plan.py checks for context plans: full records in
    lane order that decode to the samples, staged jobs (k >= 2 under BORDER_WRAP) whose records decode to the samples and
    whose windows lie inside their boxes, and every output pixel written by exactly one launch job."""
    mw, mh, iw, ih = _sizes(family, KSIZE[interp])
    m = FAMILIES[family](mw, mh, iw, ih)
    ctx = t360.make_context(interpolation_alg=interp, **WARP_CTX)
    hp = t360.HostPlan.from_warp(ctx, m, iw, ih, border)
    # test_gather_plan reads the context only to tell staged plans from BORDER_TRANSPARENT ones (the barrel layouts)
    shown = t360.make_context(interpolation_alg=interp, output_layout=t360.LAYOUT_BARREL if border == TRANSPARENT else t360.LAYOUT_EQUIRECT)
    monkeypatch.setitem(SMALL, "__warp", {})
    monkeypatch.setattr(tgp, "_plan", lambda case, plane: (shown, hp, iw, ih))
    tgp.test_gather_plan_invariants("small", "__warp", 0)
    if KSIZE[interp] >= 2 and border == WRAP:
        caps = hp.pole_caps()
        g = hp.gather_plan()
        general = int(((g["jobs"][:, 1] >> tgp.KIND_SHIFT) & 15 == tgp.GENERAL).sum())
        assert len(caps["launch"]) == len(g["jobs"]) - general + len(caps["jobs"])


def _stdout(capfd):
    C.CDLL(None).fflush(None)  # (the library prints with printf: flush the C stream before reading the captured fd)
    return capfd.readouterr().out


def _refused(capfd, fn, *args):
    assert not fn(*args)
    out = _stdout(capfd)
    assert out.strip(), "a refusal prints a message"
    return out


def test_refusals_happen_without_a_gpu(capfd):
    """Every refusal of hostPlanCreateFromWarp, generateMapFromWarp and remapFrameAsync comes with a message and before any
    CUDA call (this machine may have none)."""
    L = t360.load()
    m = identity(8, 4, 8, 4)
    good = t360.make_context(interpolation_alg=t360.CUBIC, **WARP_CTX)
    bad_cases = [  # (context, map pointer, map w, map h, in w, in h, border)
        (good, None, 8, 4, 8, 4, WRAP), (good, m.ctypes.data, 0, 4, 8, 4, WRAP), (good, m.ctypes.data, 8, -1, 8, 4, WRAP),
        (good, m.ctypes.data, 8, 4, 0, 4, WRAP), (good, m.ctypes.data, 8, 4, 8, 0, WRAP),
        (good, m.ctypes.data, 65537, 1, 8, 4, WRAP), (good, m.ctypes.data, 1, 65537, 8, 4, WRAP),
        (good, m.ctypes.data, 8, 4, 8, 4, 0), (good, m.ctypes.data, 8, 4, 8, 4, 4), (good, m.ctypes.data, 8, 4, 8, 4, 1),
        (t360.make_context(interpolation_alg=3, **WARP_CTX), m.ctypes.data, 8, 4, 8, 4, WRAP),
        (t360.make_context(interpolation_alg=t360.CUBIC), m.ctypes.data, 8, 4, 8, 4, WRAP),  # the filter's default: low-pass on
    ]
    for ctx, ptr, mw, mh, iw, ih, border in bad_cases:
        assert not L.T360B200_hostPlanCreateFromWarp(C.byref(ctx), ptr, mw, mh, iw, ih, border)
        assert _stdout(capfd).strip()
        with t360.VideoFrameTransform(ctx) as vft:
            _refused(capfd, L.T360B200_generateMapFromWarp, vft._h, ptr, mw, mh, iw, ih, border, 0)
    with pytest.raises(ValueError):
        t360.HostPlan.from_warp(good, np.zeros((4, 8, 3), np.float32), 8, 4)
    assert L.T360B200_hostPlanCreateFromWarp(None, m.ctypes.data, 8, 4, 8, 4, WRAP) is None
    assert not L.T360B200_generateMapFromWarp(None, m.ctypes.data, 8, 4, 8, 4, WRAP, 0)

    # remapFrameAsync: fake (never dereferenced) device addresses; every check is on the host
    def remap(vft, n=1, maps=(0x10000,), pitches=(64,), border=WRAP, dims=(8, 4, 8, 4), planes=(0x20000,), pitch=(8, 8)):
        P, I = C.c_void_p * 3, C.c_int * 3
        arr = lambda v: I(*([v] * 3))
        return L.T360B200_remapFrameAsync(vft._h, n, P(*(list(maps) * 3)[:3]), I(*(list(pitches) * 3)[:3]), border, P(*(list(planes) * 3)[:3]),
                                          P(*(list(planes) * 3)[:3]), arr(dims[0]), arr(dims[1]), arr(pitch[0]), arr(dims[2]), arr(dims[3]),
                                          arr(pitch[1]), None)
    with t360.VideoFrameTransform(good) as vft:
        for kw in (dict(n=0), dict(n=4), dict(maps=(None,)), dict(maps=(0x10004,)), dict(pitches=(60,)), dict(pitches=(56,)),
                   dict(pitches=(0,)), dict(border=4), dict(border=0), dict(planes=(None,)), dict(dims=(8, 4, 0, 4)),
                   dict(dims=(0, 4, 8, 4)), dict(pitch=(4, 8)), dict(pitch=(8, 4))):
            _refused(capfd, lambda: remap(vft, **kw))
    for ctx in (t360.make_context(interpolation_alg=3, **WARP_CTX), t360.make_context(interpolation_alg=t360.CUBIC)):
        with t360.VideoFrameTransform(ctx) as vft:
            _refused(capfd, lambda: remap(vft))
    assert not L.T360B200_remapFrameAsync(None, 1, None, None, WRAP, None, None, None, None, None, None, None, None, None)


# ---- on the GPU --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests must run on an H100 (there is no CPU fallback to test)")
    return torch


def _pitch(w):
    return (w + 255) // 256 * 256 + 64  # pitched planes, not 256-byte aligned rows


def _dev(torch, a, fill=0):
    t = torch.full((a.shape[0], _pitch(a.shape[1])), fill, dtype=torch.uint8, device="cuda")
    t[:, :a.shape[1]] = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t


def _dev_map(torch, m, extra=3):
    """A device map with a pitch of (w + extra) entries."""
    t = torch.zeros((m.shape[0], m.shape[1] + extra, 2), dtype=torch.float32, device="cuda")
    t[:, :m.shape[1]] = torch.from_numpy(m).cuda()
    return t


LUMA_FILL = 7  # what a luma output holds before the frame: BORDER_TRANSPARENT keeps it where no source pixel lands


def _oracle(src, m, interp, border, plane, out_w, out_h):
    """cv::remap through the oracle, with the pre-fill of the planned path (luma keeps LUMA_FILL, chroma starts at 128), and
    the INTER_AREA resize when the output is not the map's size (the render target pre-filled with 0 / 128)."""
    mh, mw = m.shape[:2]
    if (out_w, out_h) == (mw, mh):
        dst = np.full((mh, mw), 128 if plane else LUMA_FILL, np.uint8)
        return co.remap_u8(src, m, interp, border, dst)
    scaled = np.full((mh, mw), 128 if plane else 0, np.uint8)
    return co.resize_area(co.remap_u8(src, m, interp, border, scaled), out_w, out_h)


def _frame_maps(family, seed=0):
    """Luma and chroma (4:2:0) maps and sizes of one family: (maps per plan index, in sizes, map sizes)."""
    mw, mh, iw, ih = _sizes(family, seed)
    cw, ch, ciw, cih = (mw + 1) // 2, (mh + 1) // 2, (iw + 1) // 2, (ih + 1) // 2
    return [FAMILIES[family](mw, mh, iw, ih), FAMILIES[family](cw, ch, ciw, cih)], [(iw, ih), (ciw, cih)]


def _planned_and_oracle(torch, family, interp, border, out_sizes=None):
    """A transform with both plan indices generated from the family's maps; per plane the source, its device copies, the
    oracle frame and (out w, out h)."""
    maps, ins = _frame_maps(family, KSIZE[interp])
    vft = t360.VideoFrameTransform(t360.make_context(interpolation_alg=interp, **WARP_CTX))
    for idx in (0, 1):
        assert vft.generate_map_from_warp(maps[idx], *ins[idx], idx, border)
    planes = []
    for p in range(3):
        idx = min(p, 1)
        (iw, ih), m = ins[idx], maps[idx]
        src = co.noise_plane(iw, ih, plane=p, frame=interp)
        ow, oh = out_sizes[idx] if out_sizes else (m.shape[1], m.shape[0])
        planes.append(dict(src=src, d_src=_dev(torch, src), map=m, out=(ow, oh), idx=idx,
                           want=_oracle(src, m, interp, border, p, ow, oh)))
    return vft, planes


def _out(torch, pl, p):
    ow, oh = pl["out"]
    return torch.full((oh, _pitch(ow)), 128 if p else LUMA_FILL, dtype=torch.uint8, device="cuda")


def _frame_args(planes, outs):
    in_planes = [(pl["d_src"].data_ptr(), pl["d_src"].stride(0)) for pl in planes]
    out_planes = [(o.data_ptr(), o.stride(0)) for o in outs]
    dims = [(pl["src"].shape[1], pl["src"].shape[0], *pl["out"]) for pl in planes]
    return in_planes, out_planes, dims


def _host(o, pl):
    ow, oh = pl["out"]
    return o[:, :ow].cpu().numpy()


def _check(got, want, what):
    assert np.array_equal(got, want), f"{what}: {int((got != want).sum())} px differ from the oracle"


@pytest.mark.gpu
@pytest.mark.parametrize("family", sorted(FAMILIES))
@pytest.mark.parametrize("interp", INTERPS)
@pytest.mark.parametrize("border", [WRAP, TRANSPARENT])
def test_planned_warp_frames_equal_the_oracle(family, interp, border, torch_cuda):
    """generateMapFromWarp, then every frame entry point: transformFrameAsync with 3 and with 1 plane,
    transformFramePlaneAsync per plane and transformFramePlane with host planes, on pitched planes, all bit for bit the
    oracle's cv::remap (with the pre-fill rule under BORDER_TRANSPARENT)."""
    torch = torch_cuda
    vft, planes = _planned_and_oracle(torch, family, interp, border)
    st = torch.cuda.Stream()
    for n in (3, 1):
        outs = [_out(torch, pl, p) for p, pl in enumerate(planes[:n])]
        torch.cuda.synchronize()
        assert vft.make_frame_call(*_frame_args(planes[:n], outs))(st.cuda_stream)
        st.synchronize()
        for p, pl in enumerate(planes[:n]):
            _check(_host(outs[p], pl), pl["want"], f"{family} frame of {n}, plane {p}")
    for p, pl in enumerate(planes):
        o = _out(torch, pl, p)
        if p == 2:  # (transformFramePlaneAsync pre-fills chroma under BORDER_TRANSPARENT itself)
            o.fill_(0)
        torch.cuda.synchronize()
        (iw, ih), (ow, oh) = pl["src"].shape[::-1], pl["out"]
        assert vft.transform_plane_async(pl["d_src"].data_ptr(), o.data_ptr(), iw, ih, pl["d_src"].stride(0), ow, oh, o.stride(0), pl["idx"],
                                         st.cuda_stream)
        st.synchronize()
        _check(_host(o, pl), pl["want"], f"{family} plane call, plane {p}")
        h_out = np.full((oh, ow + 5), 128 if p else LUMA_FILL, np.uint8)
        h_src = np.zeros((ih, iw + 3), np.uint8)
        h_src[:, :iw] = pl["src"]
        got = vft.transform_plane(h_src[:, :iw], ow, oh, pl["idx"], p, out=h_out[:, :ow])
        _check(got, pl["want"], f"{family} host-pointer call, plane {p}")
    vft.close()


@pytest.mark.gpu
@pytest.mark.parametrize("border", [WRAP, TRANSPARENT])
@pytest.mark.parametrize("interp", [t360.LINEAR, t360.CUBIC])
def test_planned_warp_frames_resized_to_another_output_size(border, interp, torch_cuda):
    """An output size other than the map's takes the INTER_AREA branch: oracle remap into a plane pre-filled with 0 / 128,
    then resize_area."""
    torch = torch_cuda
    vft, planes = _planned_and_oracle(torch, "dual_fisheye", interp, border, out_sizes=[(171, 86), (86, 43)])
    outs = [_out(torch, pl, p) for p, pl in enumerate(planes)]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    assert vft.make_frame_call(*_frame_args(planes, outs))(st.cuda_stream)
    st.synchronize()
    for p, pl in enumerate(planes):
        _check(_host(outs[p], pl), pl["want"], f"resized plane {p}")
        got = vft.transform_plane(pl["src"], *pl["out"], pl["idx"], p)
        _check(got, pl["want"], f"resized host plane {p}")
    vft.close()


@pytest.mark.gpu
@pytest.mark.parametrize("interp", [t360.CUBIC, t360.LINEAR])
def test_streamed_host_plane_of_a_dual_fisheye_map(interp, torch_cuda):
    """A 3840 x 1920 dual-fisheye plane with host pointers is large enough for the streamed path (chunked upload, gather
    waves, chunked download); the first call is captured into a graph for page-locked planes, the second replays it."""
    torch = torch_cuda
    m = dual_fisheye(3840, 1920, 3840, 1920)
    vft = t360.VideoFrameTransform(t360.make_context(interpolation_alg=interp, **WARP_CTX))
    assert vft.generate_map_from_warp(m, 3840, 1920, 0)
    src = co.noise_plane(3840, 1920, frame=interp)
    want = _oracle(src, m, interp, WRAP, 0, 3840, 1920)
    _check(vft.transform_plane(src, 3840, 1920, 0), want, "pageable host planes")
    pin_in = torch.from_numpy(src.copy()).pin_memory()
    pin_out = torch.zeros((1920, 3840), dtype=torch.uint8).pin_memory()
    for rep in range(2):
        pin_out.zero_()
        assert vft.transformFramePlane(pin_in.data_ptr(), pin_out.data_ptr(), 3840, 1920, 3840, 3840, 1920, 3840, 0, 0)
        _check(pin_out.numpy(), want, f"page-locked host planes, call {rep}")
    vft.close()


def _remap_call(vft, planes, outs, border):
    return vft.make_remap_frame_call(*_frame_args(planes, outs), border=border)


@pytest.mark.gpu
@pytest.mark.parametrize("family", sorted(FAMILIES))
@pytest.mark.parametrize("interp", INTERPS)
@pytest.mark.parametrize("border", [WRAP, TRANSPARENT])
def test_per_frame_maps_equal_the_planned_path_and_the_oracle(family, interp, border, torch_cuda):
    """remapFrameAsync with the maps generateMapFromWarp planned gives the same frames, with 3 and with 1 plane."""
    torch = torch_cuda
    vft, planes = _planned_and_oracle(torch, family, interp, border)
    st = torch.cuda.Stream()
    d_maps = [_dev_map(torch, pl["map"], extra=p) for p, pl in enumerate(planes)]
    for n in (3, 1):
        planned = [_out(torch, pl, p) for p, pl in enumerate(planes[:n])]
        per_frame = [_out(torch, pl, p) for p, pl in enumerate(planes[:n])]
        torch.cuda.synchronize()
        assert vft.make_frame_call(*_frame_args(planes[:n], planned))(st.cuda_stream)
        assert _remap_call(vft, planes[:n], per_frame, border)(d_maps[:n], st.cuda_stream)
        st.synchronize()
        for p, pl in enumerate(planes[:n]):
            _check(_host(per_frame[p], pl), pl["want"], f"{family} per-frame map, frame of {n}, plane {p}")
            _check(_host(per_frame[p], pl), _host(planned[p], pl), f"{family} per-frame vs planned, plane {p}")
    # a dense map given by its address, and a (pointer, pitch) pair
    dense = [torch.from_numpy(pl["map"]).cuda() for pl in planes]
    outs = [_out(torch, pl, p) for p, pl in enumerate(planes)]
    torch.cuda.synchronize()
    assert _remap_call(vft, planes, outs, border)([dense[0].data_ptr(), (d_maps[1].data_ptr(), d_maps[1].stride(0) * 4), dense[2]],
                                                 st.cuda_stream)
    st.synchronize()
    for p, pl in enumerate(planes):
        _check(_host(outs[p], pl), pl["want"], f"{family} map arguments, plane {p}")
    vft.close()


@pytest.mark.gpu
def test_rotating_dual_fisheye_sequence_on_two_streams(torch_cuda):
    """A stabilisation-like warp that changes every frame: a rotating dual-fisheye map per frame, frames alternating between
    two streams with no synchronisation between them, each frame equal to the oracle for its own maps."""
    torch = torch_cuda
    spec = StreamSpec(768, 384, 512, 256)
    ft = FrameTransformer(t360.make_context(interpolation_alg=t360.CUBIC, output_layout=t360.LAYOUT_EQUIRECT, **WARP_CTX), spec)
    n = 16
    dims = [spec.plane_dims(p) for p in range(3)]
    srcs = [[co.noise_plane(d[0], d[1], plane=p, frame=f % 3) for p, d in enumerate(dims)] for f in range(3)]
    d_src = [[_dev(torch, a) for a in row] for row in srcs]
    maps = [[dual_fisheye(d[2], d[3], d[0], d[1], yaw=25.0 * f, pitch=7.0 * np.sin(f), roll=3.0 * f) for d in dims[:2]] for f in range(n)]
    d_maps = [[_dev_map(torch, m) for m in row] for row in maps]
    outs = [[torch.zeros((d[3], _pitch(d[2])), dtype=torch.uint8, device="cuda") for d in dims] for _ in range(n)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for f in range(n):
        call = ft.remap_frame_call([(t.data_ptr(), t.stride(0)) for t in d_src[f % 3]], [(t.data_ptr(), t.stride(0)) for t in outs[f]])
        assert call([d_maps[f][0], d_maps[f][1], d_maps[f][1]], streams[f % 2].cuda_stream), f"frame {f}"
    for s in streams:
        s.synchronize()
    for f in range(n):
        for p, d in enumerate(dims):
            want = co.remap_u8(srcs[f % 3][p], maps[f][min(p, 1)], t360.CUBIC, WRAP)
            _check(outs[f][p][:, :d[2]].cpu().numpy(), want, f"frame {f} plane {p}")
    ft.close()


@pytest.mark.gpu
def test_a_warp_plan_refuses_geometry_calls_until_regenerated(torch_cuda, capfd):
    """A transform holding a warp plan refuses reconfigure, reconfigureAsync and the view, orientation and pose calls (0, a
    message) and its next frames are unchanged; generateMapForPlane on each index restores geometry plans whose frames equal
    a fresh transform's."""
    torch = torch_cuda
    L = t360.load()
    ov = dict(interpolation_alg=t360.CUBIC, output_layout=t360.LAYOUT_CUBEMAP_32, **WARP_CTX)
    vft, planes = _planned_and_oracle(torch, "fisheye", t360.CUBIC, WRAP)
    vft.ctx = t360.make_context(**ov)
    outs = [_out(torch, pl, p) for p, pl in enumerate(planes)]
    args = _frame_args(planes, outs)
    frame = vft.make_frame_call(*args)
    _stdout(capfd)
    other = t360.make_context(**dict(ov, interpolation_alg=t360.LINEAR))
    assert "warp map" in _refused(capfd, L.T360B200_reconfigure, vft._h, C.byref(other))
    assert "warp map" in _refused(capfd, L.T360B200_reconfigureAsync, vft._h, C.byref(other))
    for make, arg in ((vft.make_view_frame_call, (0, 0, 90, 90)), (vft.make_oriented_frame_call, (10, 0, 0)),
                      (vft.make_pose_frame_call, (10, 0, 0, 90, 90))):
        assert "warp map" in _refused(capfd, lambda: make(*args)(arg, 0))
    torch.cuda.synchronize()
    assert frame(0)
    torch.cuda.synchronize()
    for p, pl in enumerate(planes):
        _check(_host(outs[p], pl), pl["want"], f"frame after the refusals, plane {p}")
    # geometry plans again: the frames a fresh transform gives
    in_dims = [(pl["src"].shape[1], pl["src"].shape[0]) for pl in planes]
    out_dims = [(96, 64), (48, 32), (48, 32)]
    for idx in (0, 1):
        assert vft.generateMapForPlane(*in_dims[idx], *out_dims[idx], idx)
    fresh = t360.VideoFrameTransform(t360.make_context(**ov))
    for idx in (0, 1):
        assert fresh.generateMapForPlane(*in_dims[idx], *out_dims[idx], idx)
    got, want = [], []
    for t, dst in ((vft, got), (fresh, want)):
        o = [torch.zeros((h, _pitch(w)), dtype=torch.uint8, device="cuda") for w, h in out_dims]
        dims = [(*in_dims[p], *out_dims[p]) for p in range(3)]
        assert t.make_frame_call(args[0], [(x.data_ptr(), x.stride(0)) for x in o], dims)(0)
        torch.cuda.synchronize()
        dst.extend(x[:, :w].cpu().numpy() for x, (w, _) in zip(o, out_dims))
    for p in range(3):
        _check(got[p], want[p], f"regenerated geometry plan, plane {p}")
    vft.reconfigure(t360.make_context(**dict(ov, interpolation_alg=t360.LINEAR)))  # accepted again
    vft.close()
    fresh.close()


@pytest.mark.gpu
def test_device_memory_and_launches_stay_bounded_over_per_frame_maps(torch_cuda):
    """50 per-frame maps after a warm-up: device memory does not grow and every frame is one kernel launch (the gather of
    all three planes), also under BORDER_TRANSPARENT (the chroma pre-fill is a memset)."""
    torch = torch_cuda
    spec = StreamSpec(1024, 512, 640, 320)
    dims = [spec.plane_dims(p) for p in range(3)]
    ft = FrameTransformer(t360.make_context(interpolation_alg=t360.LANCZOS4, output_layout=t360.LAYOUT_EQUIRECT, **WARP_CTX), spec)
    d_src = [_dev(torch, co.noise_plane(d[0], d[1], plane=p)) for p, d in enumerate(dims)]
    outs = [torch.zeros((d[3], _pitch(d[2])), dtype=torch.uint8, device="cuda") for d in dims]
    maps = [[_dev_map(torch, dual_fisheye(d[2], d[3], d[0], d[1], yaw=7.0 * f)) for d in dims[:2]] for f in range(50)]
    st = torch.cuda.Stream()
    for border in (WRAP, TRANSPARENT):
        call = ft.remap_frame_call([(t.data_ptr(), t.stride(0)) for t in d_src], [(t.data_ptr(), t.stride(0)) for t in outs], border)
        torch.cuda.synchronize()
        for f in range(5):
            assert call([maps[f][0], maps[f][1], maps[f][1]], st.cuda_stream)
        st.synchronize()
        free_before = torch.cuda.mem_get_info()[0]
        n0 = t360.kernel_launch_count()
        for f in range(50):
            assert call([maps[f][0], maps[f][1], maps[f][1]], st.cuda_stream)
        launches = t360.kernel_launch_count() - n0
        st.synchronize()
        assert torch.cuda.mem_get_info()[0] >= free_before - (2 << 20), "device memory grew over per-frame maps"
        assert launches == 50, f"{launches} launches for 50 frames"
    ft.close()
