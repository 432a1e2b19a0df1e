"""Per-frame views for FLAT_FIXED output (T360B200_transformFrameViewAsync, VideoFrameTransform.make_view_frame_call) and the
transform360_cuda view commands that use it.

The contract: a frame enqueued with a view equals, bit for bit, what a fresh transform gives for the transform's context
with fixed_yaw / pitch / hfov / vfov replaced by the view -- low-pass and area resize included -- without a re-plan and
without synchronising the device.  The sampling records the kernel computes come from the same host/device functions as the
planner's (csrc/flat_view.h); T360B200_viewSamples exposes them on the host and is checked against the planner here."""
import ctypes as C
import json
import math
import os
import subprocess
import time
import zlib

import numpy as np
import pytest

import transform360_b200 as t360
from oracle import c_oracle as co
from oracle import ff_harness as ff
from oracle import ref_harness as rh
from tests.test_reconfigure import ROOT, _command, _params, command_filter, commands_library  # noqa: F401 (fixtures)
from tests.test_warp_map import _stdout
from transform360_b200.stream import FrameTransformer, StreamSpec

FLAT = dict(output_layout=t360.LAYOUT_FLAT_FIXED)


# ---- no GPU needed ----------------------------------------------------------------------------------------------------
def test_view_entry_points_are_exported_with_their_bindings():
    from transform360_b200.handler import EXPORTED_SYMBOLS, LIB_PATH
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    L = t360.load()
    for name in ("T360B200_transformFrameViewAsync", "T360B200_viewSamples"):
        assert name in EXPORTED_SYMBOLS and name in defined, name
        assert getattr(L, name).restype is C.c_int
    assert C.sizeof(t360.T360View) == 16
    assert L.T360B200_transformFrameViewAsync.argtypes[:3] == [C.c_void_p, C.POINTER(t360.T360View), C.c_int]
    assert L.T360B200_viewSamples.argtypes[:2] == [C.POINTER(t360.FrameTransformContext), C.POINTER(t360.T360View)]
    view = t360.T360View(0, 0, 120, 110)
    assert L.T360B200_transformFrameViewAsync(None, C.byref(view), 1, None, None, None, None, None, None, None, None, None) == 0
    assert L.T360B200_viewSamples(C.byref(t360.make_context(**FLAT)), None, 64, 32, 16, 16, None) == 0


def _sweep_case(rng, n):
    """One seeded (context, view, sizes) of the sample sweep."""
    stereo = [t360.STEREO_FORMAT_MONO, t360.STEREO_FORMAT_TB, t360.STEREO_FORMAT_LR]
    yaw = float(rng.uniform(-1000, 1000))
    pitch = float(rng.choice([90.0, -90.0, 180.0, -180.0, 89.99, -90.01, 179.5, -180.5])) if n % 3 == 0 else float(rng.uniform(-200, 200))
    hfov = float(rng.uniform(-400, 400)) if n % 7 == 0 else float(rng.uniform(1, 400))
    vfov = float(rng.uniform(-250, 250)) if n % 5 == 0 else float(rng.uniform(1, 250))
    ov = dict(FLAT, enable_low_pass_filter=0, interpolation_alg=[t360.NEAREST, t360.LINEAR, t360.CUBIC, t360.LANCZOS4][n % 4],
              input_stereo_format=stereo[(n // 4) % 3], output_stereo_format=stereo[(n // 12) % 3], vflip=int((n // 36) % 2),
              fixed_yaw=yaw, fixed_pitch=pitch, fixed_hfov=hfov, fixed_vfov=vfov)
    if n % 11 == 0:
        ov.update(width_scale_factor=float(rng.choice([0.5, 2.0, 1.5])), height_scale_factor=float(rng.choice([0.5, 2.0, 0.75])))
    sizes = (int(rng.integers(16, 160)) * 2 + 1, int(rng.integers(8, 80)) * 2 + 1, int(rng.integers(3, 48)) * 2 + 1,
             int(rng.integers(3, 40)) * 2 + 1)
    return ov, (yaw, pitch, hfov, vfov), sizes


def test_view_samples_equal_the_planner_over_a_seeded_sweep():
    """600 views: yaw up to +-1000, pitch through +-90 and +-180, hfov up to 400, vfov up to 250, odd plane sizes, mono / TB /
    LR input, TB / LR output with and without vflip, every interpolator, a few scale factors."""
    rng = np.random.default_rng(20261015)
    for n in range(600):
        ov, view, sizes = _sweep_case(rng, n)
        # the base context has another view: the samples must come from `view` alone
        base = t360.make_context(**dict(ov, fixed_yaw=3.0, fixed_pitch=-7.0, fixed_hfov=100.0, fixed_vfov=80.0))
        got = t360.view_samples(base, view, *sizes)
        plan = t360.HostPlan(t360.make_context(**ov), *sizes)
        want = plan.samples
        assert got.shape == want.shape, (n, ov, sizes)
        assert np.array_equal(got, want), f"case {n} {ov} {sizes}: {int((got != want).any(axis=2).sum())} records differ"


def test_view_samples_refuse_other_layouts_and_non_finite_views():
    for layout in (t360.LAYOUT_CUBEMAP_32, t360.LAYOUT_EAC_32, t360.LAYOUT_EQUIRECT, t360.LAYOUT_BARREL):
        with pytest.raises(ValueError):
            t360.view_samples(t360.make_context(output_layout=layout), (0, 0, 120, 110), 64, 32, 16, 16)
    for bad in [(math.nan, 0, 120, 110), (0, math.inf, 120, 110), (0, 0, -math.inf, 110), (0, 0, 120, math.nan)]:
        with pytest.raises(ValueError):
            t360.view_samples(t360.make_context(**FLAT), bad, 64, 32, 16, 16)


def _refused_for(capfd, reason, call, *args):
    """call(*args) is refused (returns 0) with a message that names `reason`."""
    assert not call(*args)
    out = _stdout(capfd)
    assert reason in out, (reason, out)


def _bad_planes_are_refused(capfd, make_call, args, planes, dims):
    """make_call(in_planes, out_planes, dims)(*args) refuses a NULL plane, a plane without pixels and a pitch short of the
    width, naming the plane, before any CUDA call: the fake addresses of `planes` are never dereferenced."""
    def with_plane(rows, p, value):
        return [value if i == p else r for i, r in enumerate(rows)]
    in_w, _, out_w, _ = dims[0]
    cases = [(with_plane(planes, 0, (None, planes[0][1])), planes, dims, 0), (planes, with_plane(planes, 2, (None, planes[2][1])), dims, 2),
             (planes, planes, with_plane(dims, 0, (0,) + dims[0][1:]), 0), (planes, planes, with_plane(dims, 1, dims[1][:3] + (-1,)), 1),
             (with_plane(planes, 0, (planes[0][0], in_w - 1)), planes, dims, 0), (planes, with_plane(planes, 0, (planes[0][0], out_w - 1)), dims, 0)]
    for ins, outs, d, p in cases:
        _refused_for(capfd, f"invalid description of plane {p}", make_call(ins, outs, d), *args)


def test_view_frames_are_refused_before_any_device_work(capfd):
    """A non-FLAT_FIXED transform, a NaN view, plan indices that were never generated and invalid planes are refused (return
    0) before the call touches CUDA, so this needs no device."""
    dummy = [(1 << 20, 512)] * 3
    dims = [(512, 256, 160, 120), (256, 128, 80, 60), (256, 128, 80, 60)]
    cube = t360.VideoFrameTransform(t360.make_context(enable_low_pass_filter=0))
    _refused_for(capfd, "per-frame views need output_layout FLAT_FIXED", cube.make_view_frame_call(dummy, dummy, dims), (10.0, 0.0, 120.0, 110.0))
    cube.close()
    flat = t360.VideoFrameTransform(t360.make_context(**FLAT))
    call = flat.make_view_frame_call(dummy, dummy, dims)
    _refused_for(capfd, "is not finite", call, (math.nan, 0.0, 120.0, 110.0))
    _refused_for(capfd, "is not finite", call, (0.0, 0.0, math.inf, 110.0))
    _refused_for(capfd, "no map was generated for index 0", call, (10.0, 0.0, 120.0, 110.0))
    _bad_planes_are_refused(capfd, flat.make_view_frame_call, ((10.0, 0.0, 120.0, 110.0),), dummy, dims)
    _bad_planes_are_refused(capfd, flat.make_frame_call, (), dummy, dims)
    flat.close()


FILTER_FLAT = "output_layout=flat_fixed:w=320:h=240:interpolation_alg=cubic"
VIEW_VALUES = {"yaw": ("30", 30.0), "pitch": ("-12.5", -12.5), "hfov": ("90", 90.0), "vfov": ("60", 60.0)}


def test_cuda_filter_view_commands_before_the_first_frame_only_set_parameters(command_filter):
    f = command_filter(FILTER_FLAT, 512, 256, device=False)
    for name, (arg, value) in VIEW_VALUES.items():
        before = _params(f)
        assert _command(f, name, arg) == 0, name
        after = _params(f)
        assert after[name] == pytest.approx(value) and after[name] != before[name], name
        assert {k: v for k, v in after.items() if k != name} == {k: v for k, v in before.items() if k != name}, name
    assert _command(f, "yaw", "abc") < 0 and _params(f)["yaw"] == 30.0
    f.close()


# ---- on the GPU ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests must run on an H100 (there is no CPU fallback to test)")
    return torch


def _pitch(w):
    return (w + 255) // 256 * 256


def _inputs(torch, spec, frames):
    srcs, dev = [], []
    for f in range(frames):
        planes = [co.noise_plane(*spec.plane_dims(p)[:2], plane=p, frame=f) for p in range(3)]
        srcs.append(planes)
        row = []
        for a in planes:
            t = torch.zeros((a.shape[0], _pitch(a.shape[1])), dtype=torch.uint8, device="cuda")
            t[:, :a.shape[1]] = torch.from_numpy(a).cuda()
            row.append(t)
        dev.append(row)
    return srcs, dev


def _outputs(torch, spec, frames):
    return [[torch.zeros((spec.plane_dims(p)[3], _pitch(spec.plane_dims(p)[2])), dtype=torch.uint8, device="cuda") for p in range(3)]
            for _ in range(frames)]


def _planes(frame):
    return [(t.data_ptr(), t.stride(0)) for t in frame]


def _host(spec, d_out):
    return [[o[:, :spec.plane_dims(p)[2]].cpu().numpy() for p, o in enumerate(frame)] for frame in d_out]


def _with_view(ov, view):
    return dict(ov, fixed_yaw=view[0], fixed_pitch=view[1], fixed_hfov=view[2], fixed_vfov=view[3])


def _fresh(torch, ov, view, spec, d_in):
    """What a fresh transform made for the context with `view` gives (whole-frame entry point)."""
    ft = FrameTransformer(t360.make_context(**_with_view(ov, view)), spec)
    out = _outputs(torch, spec, 1)
    torch.cuda.synchronize()
    assert ft.frame_call(_planes(d_in), _planes(out[0]))(0)
    torch.cuda.synchronize()
    ft.close()
    return _host(spec, out)[0]


def _oracle(ov, view, spec, src):
    octx = rh.default_context(**_with_view(ov, view))
    plans, row = {}, []
    for p in range(3):
        iw, ih, ow, oh, idx = spec.plane_dims(p)
        if idx not in plans:
            plans[idx] = co.OraclePlan(octx, iw, ih, ow, oh)
        row.append(co.transform_plane(octx, plans[idx], src[p], ow, oh, map_index=idx))
    return row


def _trajectory(seed, n):
    """A seeded camera path: yaw sweeps 720 degrees, pitch crosses a pole (|pitch| > 90 on the way), the field of view
    breathes."""
    rng = np.random.default_rng(seed)
    t = np.linspace(0.0, 1.0, n)
    yaw = -360.0 + 720.0 * t + rng.uniform(-3, 3, n)
    pitch = 110.0 * np.sin(2 * np.pi * t) + rng.uniform(-2, 2, n)
    hfov = 100.0 + 25.0 * np.sin(6 * np.pi * t) + rng.uniform(-1, 1, n)
    vfov = 80.0 + 20.0 * np.cos(4 * np.pi * t) + rng.uniform(-1, 1, n)
    return [tuple(float(np.float32(v)) for v in row) for row in zip(yaw, pitch, hfov, vfov)]


def _assert_planes(got, want, what):
    for p, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g, w), f"{what}: plane {p}: {int((g != w).sum())} px differ"


LOW_PASS_DEFAULT = dict(enable_low_pass_filter=1)  # the filter's defaults: 5 bands, adjust_kernel=1
CONFIGS = {  # name: (context, luma in, luma out, views, oracle frames)
    "full_cubic": (dict(FLAT, interpolation_alg=t360.CUBIC, enable_low_pass_filter=0), (7680, 3840), (1920, 1080), 30, 1),
    "full_cubic_low_pass": (dict(FLAT, interpolation_alg=t360.CUBIC, **LOW_PASS_DEFAULT), (7680, 3840), (1920, 1080), 30, 1),
    "lanczos4_low_pass": (dict(FLAT, interpolation_alg=t360.LANCZOS4, num_horizontal_segments=4, num_vertical_segments=9), (960, 480),
                          (322, 182), 32, 3),
    "nearest": (dict(FLAT, interpolation_alg=t360.NEAREST, enable_low_pass_filter=0), (961, 481), (321, 181), 32, 3),
    "linear_low_pass": (dict(FLAT, interpolation_alg=t360.LINEAR), (960, 480), (320, 180), 30, 2),
    "tb_stereo_vflip": (dict(FLAT, interpolation_alg=t360.CUBIC, input_stereo_format=t360.STEREO_FORMAT_TB,
                             output_stereo_format=t360.STEREO_FORMAT_TB, vflip=1), (960, 960), (320, 360), 30, 2),
    "scale_half": (dict(FLAT, interpolation_alg=t360.CUBIC, width_scale_factor=0.5, height_scale_factor=0.5), (960, 480), (320, 180), 30, 2),
    "scale_two": (dict(FLAT, interpolation_alg=t360.CUBIC, width_scale_factor=2.0, height_scale_factor=2.0), (960, 480), (320, 180), 30, 2),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_view_frames_equal_fresh_transforms(name, torch_cuda):
    """A seeded trajectory enqueued back to back on a non-default stream without synchronisation: every frame equals a
    fresh transform made for its view, and the plain-C oracle on a subset."""
    torch = torch_cuda
    ov, inp, out, n, n_oracle = CONFIGS[name]
    spec = StreamSpec(*inp, *out)
    views = _trajectory(zlib.crc32(name.encode()), n)
    srcs, d_in = _inputs(torch, spec, 2)
    d_out = _outputs(torch, spec, n)
    ft = FrameTransformer(t360.make_context(**ov), spec)
    calls = [ft.view_frame_call(_planes(d_in[f % 2]), _planes(d_out[f])) for f in range(n)]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for f, view in enumerate(views):
        assert calls[f](view, st.cuda_stream), f"frame {f} view {view} refused"
    st.synchronize()
    got = _host(spec, d_out)
    ft.close()
    for f, view in enumerate(views):
        _assert_planes(got[f], _fresh(torch, ov, view, spec, d_in[f % 2]), f"{name} frame {f} view {view}")
    for f in np.linspace(0, n - 1, n_oracle).astype(int):
        _assert_planes(got[f], _oracle(ov, views[f], spec, srcs[f % 2]), f"{name} frame {f} view {views[f]}, oracle")


@pytest.mark.gpu
def test_two_streams_and_a_reconfigure_in_flight(torch_cuda):
    """View frames on two streams, a reconfigure of a non-view field (interpolation, low-pass bands) in the middle: every
    frame has the configuration in effect when it was enqueued, with its own view."""
    torch = torch_cuda
    a = dict(FLAT, interpolation_alg=t360.CUBIC, num_vertical_segments=7, num_horizontal_segments=3)
    b = dict(a, interpolation_alg=t360.LANCZOS4, num_vertical_segments=11)
    spec = StreamSpec(960, 480, 320, 240)
    views = _trajectory(7, 12)
    _, d_in = _inputs(torch, spec, 2)
    d_out = _outputs(torch, spec, 12)
    ft = FrameTransformer(t360.make_context(**a), spec)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for f, view in enumerate(views):
        if f == 6:
            ft.vft.reconfigure(t360.make_context(**b))
        assert ft.view_frame_call(_planes(d_in[f % 2]), _planes(d_out[f]))(view, streams[f % 2].cuda_stream)
    for s in streams:
        s.synchronize()
    got = _host(spec, d_out)
    ft.close()
    for f, view in enumerate(views):
        _assert_planes(got[f], _fresh(torch, a if f < 6 else b, view, spec, d_in[f % 2]), f"frame {f} view {view}")


@pytest.mark.gpu
def test_device_memory_and_launches_stay_bounded(torch_cuda):
    """1000 distinct views: device memory does not grow, and without low-pass a frame is one kernel launch (the gather of
    all three planes)."""
    torch = torch_cuda
    spec = StreamSpec(1920, 960, 640, 360)
    _, d_in = _inputs(torch, spec, 1)
    d_out = _outputs(torch, spec, 1)
    views = _trajectory(11, 1000)
    st = torch.cuda.Stream()
    for ov in (dict(FLAT, enable_low_pass_filter=0), dict(FLAT, num_vertical_segments=9, num_horizontal_segments=4)):
        ft = FrameTransformer(t360.make_context(**ov), spec)
        call = ft.view_frame_call(_planes(d_in[0]), _planes(d_out[0]))
        torch.cuda.synchronize()
        for view in views[:50]:  # first use of every scratch plane and ring entry
            assert call(view, st.cuda_stream)
        st.synchronize()
        free_before = torch.cuda.mem_get_info()[0]
        n0 = t360.kernel_launch_count()
        for view in views:
            assert call(view, st.cuda_stream)
        launches = t360.kernel_launch_count() - n0
        st.synchronize()
        free_after = torch.cuda.mem_get_info()[0]
        ft.close()
        assert free_before - free_after <= 4 << 20, f"{(free_before - free_after) >> 20} MB of device memory not released ({ov})"
        if not ov.get("enable_low_pass_filter", 1):
            assert launches == len(views), f"{launches} launches for {len(views)} frames"
        else:
            assert launches <= 4 * len(views), f"{launches} launches for {len(views)} frames"


RECORDS = ROOT / "tests" / "golden" / "view_reference.json"
FILTER_ARGS = FILTER_FLAT  # with the filter's default low-pass


def _reference_filter_frame(args, w, h, planes):
    """The reference software filter's frame for `args` (oracle/_ref): live where it is built, checked against its digests
    in view_reference.json, else those digests.  T360_RECORD_LIVE_REFERENCE=1 rewrites the record."""
    key = f"reference_filter/{args}/{w}x{h}"
    records = json.loads(RECORDS.read_text()) if RECORDS.exists() else {}
    if not ff.available("ref"):
        assert key in records, f"no recorded reference result for {key}"
        return records[key]
    ref = ff.Filter("ref", args, w, h)
    frame = ref.filter(planes)
    ref.close()
    got = {"size": [ref.out_w, ref.out_h], "planes": [rh.sha16(p) for p in frame]}
    if os.environ.get("T360_RECORD_LIVE_REFERENCE") == "1":
        records[key] = got
        RECORDS.write_text(json.dumps(records, indent=1, sort_keys=True) + "\n")
    else:
        assert records.get(key) == got, f"the live reference no longer gives its recorded result for {key}"
    return got


def _filter_planes(w, h):
    return [co.noise_plane(w, h, 0, 5), co.noise_plane((w + 1) // 2, (h + 1) // 2, 1, 5), co.noise_plane((w + 1) // 2, (h + 1) // 2, 2, 5)]


@pytest.mark.gpu
def test_cuda_filter_yaw_command_takes_the_view_path(command_filter):
    """transform360_cuda, FLAT_FIXED: three frames, `yaw 30`, three more: the reference software filter's frames without and
    then with yaw=30.  The command re-plans nothing: it returns far faster than a reconfigure (tens of milliseconds)."""
    w, h = 512, 256
    planes = _filter_planes(w, h)
    want = [_reference_filter_frame(FILTER_ARGS, w, h, planes), _reference_filter_frame(FILTER_ARGS + ":yaw=30", w, h, planes)]
    import torch
    if not torch.cuda.is_available():
        pytest.fail("needs a CUDA device")
    dev = [torch.from_numpy(p).cuda() for p in planes]
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        gpu = command_filter(FILTER_ARGS + ":sync=0", w, h, stream=stream)
        assert [gpu.out_w, gpu.out_h] == want[0]["size"] == want[1]["size"]
        got = []
        for frame in range(6):
            if frame == 3:
                t0 = time.perf_counter()
                assert _command(gpu, "yaw", "30") == 0
                elapsed = time.perf_counter() - t0
            got.append(gpu.filter(dev))
        stream.synchronize()
        for frame, out in enumerate(got):
            for p in range(3):
                assert rh.sha16(out[p].cpu().numpy()) == want[1 if frame >= 3 else 0]["planes"][p], f"plane {p} of frame {frame}"
        assert elapsed < 0.005, f"the view command took {elapsed * 1e3:.1f} ms: it should not re-plan"
        assert _params(gpu)["yaw"] == 30.0
        gpu.close()
