"""Reconfiguring a running transform between frames (T360B200_reconfigure, VideoFrameTransform.reconfigure) and the runtime
commands of the transform360_cuda filter that use it.

The contract: work enqueued before the call completes with the old context, work enqueued after it with the new one,
bit-identical to a fresh transform made with that context; a refused context leaves the old one in effect; the old
plans are released without a leak.  The GPU tests enqueue on a non-default stream and never synchronise between the
frames before and after the call."""
import ctypes as C
import errno
import json
import os
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

import transform360_b200 as t360
from oracle import c_oracle as co
from oracle import ff_harness as ff
from oracle import ref_harness as rh
from tests.golden.cases import FULL
from transform360_b200.stream import FrameTransformer, StreamSpec

ENOSYS, EINVAL = -errno.ENOSYS, -errno.EINVAL


# ---- no GPU needed ----------------------------------------------------------------------------------------------------
def test_reconfigure_is_exported_with_its_binding():
    from transform360_b200.handler import EXPORTED_SYMBOLS, LIB_PATH
    assert "T360B200_reconfigure" in EXPORTED_SYMBOLS
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    assert "T360B200_reconfigure" in {line.split()[-1] for line in out.splitlines() if " T " in line}
    fn = t360.load().T360B200_reconfigure
    assert fn.restype is C.c_int
    assert fn.argtypes == [C.c_void_p, C.POINTER(t360.FrameTransformContext)]
    assert fn(None, C.byref(t360.make_context())) == 0


def test_reconfigure_before_any_plan_needs_no_device():
    """Before generateMapForPlane the call only replaces the context: no CUDA call, so it succeeds without a device."""
    vft = t360.VideoFrameTransform(t360.make_context(enable_low_pass_filter=0))
    b = t360.make_context(fixed_yaw=30.0, interpolation_alg=t360.LANCZOS4, output_layout=t360.LAYOUT_EAC_32)
    vft.reconfigure(b)
    assert vft.ctx is b
    assert vft._lib.T360B200_reconfigure(vft._h, None) == 0
    vft.close()


def test_the_refused_context_of_the_gpu_tests_is_refused_by_the_planner():
    with pytest.raises(ValueError):
        t360.HostPlan(t360.make_context(**REFUSED), 512, 256, 192, 128)


# transform360_cuda through the libavfilter stand-in, configured without a device
RUNTIME_VALUES = {  # option -> (command argument, value it stands for); every value differs from the default
    "yaw": ("30", 30.0), "pitch": ("-12.5", -12.5), "roll": ("7", 7.0), "hfov": ("90", 90.0), "vfov": ("60", 60.0),
    "cube_offcenter_x": ("0.1", 0.1), "cube_offcenter_y": ("-0.2", -0.2), "cube_offcenter_z": ("-0.3", -0.3),
    "expand_coef": ("1.05", 1.05), "input_expand_coef": ("1.02", 1.02), "vflip": ("true", 1), "is_horizontal_offset": ("1", 1),
    "interpolation_alg": ("lanczos4", t360.LANCZOS4), "enable_low_pass_filter": ("0", 0), "num_vertical_segments": ("9", 9),
    "num_horizontal_segments": ("4", 4), "kernel_height_scale_factor": ("2.5", 2.5), "min_kernel_half_height": ("2", 2.0),
    "max_kernel_half_height": ("40", 40.0), "adjust_kernel": ("0", 0), "kernel_adjust_factor": ("1.5", 1.5),
}
SIZE_OR_FORMAT = {"size": "300x200", "s": "300x200", "w": "300", "width": "300", "h": "200", "height": "200",
                  "cube_edge_length": "128", "max_cube_edge_length": "512", "input_layout": "cubemap_32",
                  "output_layout": "eac_32", "input_stereo_format": "tb", "output_stereo_format": "lr",
                  "width_scale_factor": "2", "height_scale_factor": "2"}
INVALID = [("num_vertical_segments", "1"), ("yaw", "abc"), ("yaw", "400"), ("interpolation_alg", "bogus"),
           ("enable_low_pass_filter", "2"), ("hfov", "")]
NUMERIC = sorted(set(RUNTIME_VALUES) | {"cube_edge_length", "max_cube_edge_length", "input_layout", "output_layout", "input_stereo_format",
                                        "output_stereo_format", "width_scale_factor", "height_scale_factor", "sync",
                                        "enable_multi_threading", "max_output_w", "max_output_h"})
ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="session")
def commands_library(tmp_path_factory):
    """transform360_cuda around oracle/ff_driver.c, compiled against the stand-in plus tests/filter_commands (runtime
    options and process_command), with the driver's command entry points; built under a temporary directory."""
    cc = os.environ.get("CC") or shutil.which("gcc") or shutil.which("cc")
    assert cc, "a C compiler is needed to build the filter with runtime commands"
    out = tmp_path_factory.mktemp("filter_commands") / "libvf_t360_cuda_commands.so"
    lib_dir = ROOT / "transform360_b200" / "lib"
    subprocess.run([cc, "-std=gnu11", "-O2", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter", "-Wno-missing-field-initializers",
                    "-Werror", "-shared", "-fvisibility=hidden", "-DFF_FILTER=ff_vf_transform360_cuda",
                    "-I", str(ROOT / "tests" / "filter_commands"), "-I", str(ROOT / "oracle" / "ffshim"), "-I", str(ROOT / "include"),
                    "-o", str(out), str(ROOT / "oracle" / "ff_driver.c"), str(ROOT / "transform360_b200" / "filter" / "vf_transform360_cuda.c"),
                    str(ROOT / "tests" / "filter_commands" / "commands.c"), "-L", str(lib_dir), "-lTransform360",
                    f"-Wl,-rpath,{lib_dir}", "-lm"], check=True, capture_output=True, text=True)
    return out


@pytest.fixture
def command_filter(commands_library, monkeypatch):
    """ff_harness.CudaFilter, on the build of the filter that has runtime commands."""
    monkeypatch.setitem(ff._LIBS, "cuda", commands_library)
    monkeypatch.setattr(ff, "_loaded", {})
    L = ff._lib("cuda")
    L.t360f_command.restype = C.c_int
    L.t360f_command.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
    L.t360f_option.restype = C.c_int
    L.t360f_option.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_double)]
    return ff.CudaFilter


def _command(f, cmd, arg):
    return f.L.t360f_command(f.h, cmd.encode(), arg.encode())


def _params(f):
    out = {}
    for name in NUMERIC:
        v = C.c_double()
        assert f.L.t360f_option(f.h, name.encode(), C.byref(v)) == 0, name
        out[name] = v.value
    return out


def test_cuda_filter_runtime_commands_without_a_device(command_filter):
    """Every view and quality option is a runtime command that changes the filter's parameters; options that could
    change the output link's size or format are ENOSYS, invalid values EINVAL, and neither refusal changes anything."""
    f = command_filter("cube_edge_length=64", 512, 256, device=False)
    size = (f.out_w, f.out_h)
    for name, (arg, value) in RUNTIME_VALUES.items():
        before = _params(f)
        assert _command(f, name, arg) == 0, name
        after = _params(f)
        assert after[name] == pytest.approx(float(np.float32(value))) and after[name] != before[name], name
        assert {k: v for k, v in after.items() if k != name} == {k: v for k, v in before.items() if k != name}, name
    for name, arg in list(SIZE_OR_FORMAT.items()) + [("sync", "0"), ("enable_multi_threading", "0"), ("nonexistent", "1")]:
        before = _params(f)
        assert _command(f, name, arg) == ENOSYS, name
        assert _params(f) == before, name
    for name, arg in INVALID:
        before = _params(f)
        assert _command(f, name, arg) == EINVAL, (name, arg)
        assert _params(f) == before, (name, arg)
    w, h = C.c_int(), C.c_int()
    f.L.t360f_out_size(f.h, C.byref(w), C.byref(h))
    assert (w.value, h.value) == size
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


def _inputs(torch, spec, frames, first=0):
    """Per frame: the source planes (numpy) and their pitched device copies (decoder surfaces: 256-byte rows)."""
    srcs, dev = [], []
    for f in range(first, first + frames):
        planes = [co.noise_plane(*spec.plane_dims(p)[:2], plane=p, frame=f) for p in range(3)]
        srcs.append(planes)
        row = []
        for p, a in enumerate(planes):
            t = torch.zeros((a.shape[0], _pitch(a.shape[1])), dtype=torch.uint8, device="cuda")
            t[:, :a.shape[1]] = torch.from_numpy(a).cuda()
            row.append(t)
        dev.append(row)
    return srcs, dev


def _outputs(torch, spec, frames):
    return [[torch.zeros((spec.plane_dims(p)[3], _pitch(spec.plane_dims(p)[2])), dtype=torch.uint8, device="cuda") for p in range(3)]
            for _ in range(frames)]


def _frame_call(vft, spec, d_in, d_out):
    dims = [spec.plane_dims(p)[:4] for p in range(3)]
    return vft.make_frame_call([(t.data_ptr(), t.stride(0)) for t in d_in], [(t.data_ptr(), t.stride(0)) for t in d_out], dims)


def _host(spec, d_out):
    return [[o[:, :spec.plane_dims(p)[2]].cpu().numpy() for p, o in enumerate(frame)] for frame in d_out]


def _fresh(torch, ctx, spec, d_in):
    """What a transform made with `ctx` gives for these frames (whole-frame entry point)."""
    ft = FrameTransformer(ctx, spec)
    outs = _outputs(torch, spec, len(d_in))
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for f in range(len(d_in)):
        assert _frame_call(ft.vft, spec, d_in[f], outs[f])(st.cuda_stream)
    st.synchronize()
    ft.close()
    return _host(spec, outs)


def _oracle(ov, spec, srcs, planes=(0, 1, 2)):
    octx = rh.default_context(**ov)
    plans = {}
    out = []
    for frame in srcs:
        row = {}
        for p in planes:
            iw, ih, ow, oh, idx = spec.plane_dims(p)
            if idx not in plans:
                plans[idx] = co.OraclePlan(octx, iw, ih, ow, oh)
            row[p] = co.transform_plane(octx, plans[idx], frame[p], ow, oh, map_index=idx)
        out.append(row)
    return out


def _assert_frames(got, want, what):
    for f, (g, w) in enumerate(zip(got, want)):
        for p in (w.keys() if isinstance(w, dict) else range(len(w))):
            assert np.array_equal(g[p], w[p]), f"{what}: frame {f} plane {p}: {int((g[p] != w[p]).sum())} px differ"


CUBIC_NO_LP = dict(interpolation_alg=t360.CUBIC, enable_low_pass_filter=0)
LOW_PASS = dict(interpolation_alg=t360.CUBIC, enable_low_pass_filter=1, num_vertical_segments=15, num_horizontal_segments=8)
REFUSED = dict(LOW_PASS, num_vertical_segments=0)
PAIRS = {  # name: (context A, context B, luma in, luma out)
    "cube_yaw_pitch_roll": (CUBIC_NO_LP, dict(CUBIC_NO_LP, fixed_yaw=30.0, fixed_pitch=-20.0, fixed_roll=12.5), (512, 256), (192, 128)),
    "flat_fixed_yaw_hfov": (dict(CUBIC_NO_LP, output_layout=t360.LAYOUT_FLAT_FIXED, fixed_yaw=100.0, fixed_pitch=50.0),
                            dict(CUBIC_NO_LP, output_layout=t360.LAYOUT_FLAT_FIXED, fixed_yaw=140.0, fixed_pitch=50.0, fixed_hfov=80.0),
                            (512, 256), (160, 120)),
    "cubic_to_lanczos4": (CUBIC_NO_LP, dict(CUBIC_NO_LP, interpolation_alg=t360.LANCZOS4), (512, 256), (192, 128)),
    "low_pass_off_to_on": (CUBIC_NO_LP, LOW_PASS, (960, 480), (240, 160)),
    "low_pass_on_to_off": (LOW_PASS, CUBIC_NO_LP, (960, 480), (240, 160)),
    "cubic_to_nearest": (CUBIC_NO_LP, dict(CUBIC_NO_LP, interpolation_alg=t360.NEAREST), (512, 256), (192, 128)),
    "nearest_to_cubic": (dict(CUBIC_NO_LP, interpolation_alg=t360.NEAREST), CUBIC_NO_LP, (512, 256), (192, 128)),
    "cubemap_to_eac": (CUBIC_NO_LP, dict(CUBIC_NO_LP, output_layout=t360.LAYOUT_EAC_32), (512, 256), (192, 128)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(PAIRS))
def test_frames_switch_view_exactly_at_the_call(name, torch_cuda):
    """Frames 0-2 enqueued with A, reconfigure(B), frames 3-5: A's frames for 0-2 and B's for 3-5, bit for bit against
    fresh transforms, and B's against the plain-C oracle."""
    torch = torch_cuda
    a, b, inp, out = PAIRS[name]
    spec = StreamSpec(*inp, *out)
    srcs, d_in = _inputs(torch, spec, 6)
    d_out = _outputs(torch, spec, 6)
    ft = FrameTransformer(t360.make_context(**a), spec)
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for f in range(3):
        assert _frame_call(ft.vft, spec, d_in[f], d_out[f])(st.cuda_stream)
    ft.vft.reconfigure(t360.make_context(**b))
    for f in range(3, 6):
        assert _frame_call(ft.vft, spec, d_in[f], d_out[f])(st.cuda_stream)
    st.synchronize()
    got = _host(spec, d_out)
    bytes_after = [ft.vft.plan_device_bytes(i) for i in (0, 1)]
    ft.close()
    _assert_frames(got[:3], _fresh(torch, t360.make_context(**a), spec, d_in[:3]), f"{name} before the call")
    _assert_frames(got[3:], _fresh(torch, t360.make_context(**b), spec, d_in[3:]), f"{name} after the call")
    _assert_frames(got[3:], _oracle(b, spec, srcs[3:]), f"{name} after the call, oracle")
    fresh = FrameTransformer(t360.make_context(**b), spec)
    assert bytes_after == [fresh.vft.plan_device_bytes(i) for i in (0, 1)]
    fresh.close()


@pytest.mark.gpu
def test_full_size_cfg2_view_change(torch_cuda):
    """cfg2 (7680x3840 -> 3840x2560, all three planes) with a yaw/pitch/roll change between frames in flight."""
    torch = torch_cuda
    case = FULL["cfg2"]
    a, b = case["ov"], dict(case["ov"], fixed_yaw=30.0, fixed_pitch=-10.0, fixed_roll=5.0)
    spec = StreamSpec(*case["inp"], *case["out"])
    srcs, d_in = _inputs(torch, spec, 4)
    d_out = _outputs(torch, spec, 4)
    ft = FrameTransformer(t360.make_context(**a), spec)
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for f in range(2):
        assert _frame_call(ft.vft, spec, d_in[f], d_out[f])(st.cuda_stream)
    ft.vft.reconfigure(t360.make_context(**b))
    for f in range(2, 4):
        assert _frame_call(ft.vft, spec, d_in[f], d_out[f])(st.cuda_stream)
    st.synchronize()
    got = _host(spec, d_out)
    ft.close()
    _assert_frames(got[:2], _fresh(torch, t360.make_context(**a), spec, d_in[:2]), "cfg2 before the call")
    _assert_frames(got[2:], _fresh(torch, t360.make_context(**b), spec, d_in[2:]), "cfg2 after the call")
    _assert_frames(got[2:3], _oracle(b, spec, srcs[2:3]), "cfg2 after the call, oracle")


LP_SPEC = StreamSpec(960, 480, 240, 160)
LP_A = LOW_PASS
LP_B = dict(LOW_PASS, interpolation_alg=t360.LANCZOS4, num_vertical_segments=9, num_horizontal_segments=4, fixed_yaw=20.0)


@pytest.mark.gpu
def test_every_entry_point_switches_at_the_call(torch_cuda):
    """transformFramePlane (device pointers), transformFramePlaneAsync, transformFrameAsync and lowPassPlaneAsync, all
    enqueued before and after the call."""
    torch = torch_cuda
    spec = LP_SPEC
    srcs, d_in = _inputs(torch, spec, 6)
    d_out = _outputs(torch, spec, 6)
    blurred = [torch.zeros((spec.in_h, spec.in_w), dtype=torch.uint8, device="cuda") for _ in range(2)]
    vft = t360.VideoFrameTransform(t360.make_context(**LP_A))
    for p in (0, 1):
        assert vft.generateMapForPlane(*spec.plane_dims(p)[:4], p)
    st = torch.cuda.Stream()
    torch.cuda.synchronize()

    def enqueue(first, lp):
        assert _frame_call(vft, spec, d_in[first], d_out[first])(st.cuda_stream)
        for p in range(3):
            iw, ih, ow, oh, idx = spec.plane_dims(p)
            i, o = d_in[first + 1][p], d_out[first + 1][p]
            assert vft.transform_plane_async(i.data_ptr(), o.data_ptr(), iw, ih, i.stride(0), ow, oh, o.stride(0), idx, st.cuda_stream)
        for p in range(3):  # synchronous, on the transform's own stream
            iw, ih, ow, oh, idx = spec.plane_dims(p)
            i, o = d_in[first + 2][p], d_out[first + 2][p]
            assert vft.transformFramePlane(i.data_ptr(), o.data_ptr(), iw, ih, i.stride(0), ow, oh, o.stride(0), idx, p)
        i = d_in[first][0]
        assert vft.low_pass_async(i.data_ptr(), lp.data_ptr(), spec.in_w, spec.in_h, i.stride(0), lp.stride(0), 0, st.cuda_stream)

    enqueue(0, blurred[0])
    vft.reconfigure(t360.make_context(**LP_B))
    enqueue(3, blurred[1])
    st.synchronize()
    got = _host(spec, d_out)
    vft.close()
    _assert_frames(got[:3], _fresh(torch, t360.make_context(**LP_A), spec, d_in[:3]), "before the call")
    _assert_frames(got[3:], _fresh(torch, t360.make_context(**LP_B), spec, d_in[3:]), "after the call")
    _assert_frames(got[3:], _oracle(LP_B, spec, srcs[3:]), "after the call, oracle")
    for k, ov in enumerate((LP_A, LP_B)):
        octx = rh.default_context(**ov)
        plan = co.OraclePlan(octx, *spec.plane_dims(0)[:4])
        want = co.filter_plane(octx, srcs[3 * k][0], plan.segs, plan.nsegs, plan.taps)
        assert np.array_equal(blurred[k].cpu().numpy(), want), f"low-pass {'after' if k else 'before'} the call"


@pytest.mark.gpu
def test_host_pointer_path_replays_before_and_recaptures_after(torch_cuda, monkeypatch):
    """The synchronous host-pointer path: a streamed plane with page-locked buffers (its captured graph is replayed before
    the call and captured again after it), and pageable planes through the plain path."""
    torch = torch_cuda
    monkeypatch.setenv("T360B200_PIPELINE_MIN_BYTES", "0")
    a, b = CUBIC_NO_LP, dict(CUBIC_NO_LP, fixed_yaw=30.0, interpolation_alg=t360.LANCZOS4)
    spec = StreamSpec(512, 256, 192, 128)
    srcs, d_in = _inputs(torch, spec, 4)
    vft = t360.VideoFrameTransform(t360.make_context(**a))
    for p in (0, 1):
        assert vft.generateMapForPlane(*spec.plane_dims(p)[:4], p)
    pinned_in = [torch.empty(spec.plane_dims(p)[1::-1], dtype=torch.uint8, pin_memory=True) for p in range(3)]
    pinned_out = [torch.zeros(spec.plane_dims(p)[3:1:-1], dtype=torch.uint8, pin_memory=True) for p in range(3)]
    got = []
    for f in range(4):
        if f == 2:
            vft.reconfigure(t360.make_context(**b))
        row = []
        for p in range(3):
            iw, ih, ow, oh, idx = spec.plane_dims(p)
            if p == 0:  # the same page-locked buffers every frame: captured once, then replayed
                pinned_in[p].numpy()[...] = srcs[f][p]
                assert vft.transformFramePlane(pinned_in[p].data_ptr(), pinned_out[p].data_ptr(), iw, ih, iw, ow, oh, ow, idx, p)
                row.append(pinned_out[p].numpy().copy())
            else:
                row.append(vft.transform_plane(srcs[f][p], ow, oh, idx, image_plane=p))
        got.append(row)
    vft.close()
    _assert_frames(got[:2], _fresh(torch, t360.make_context(**a), spec, d_in[:2]), "before the call")
    _assert_frames(got[2:], _fresh(torch, t360.make_context(**b), spec, d_in[2:]), "after the call")
    _assert_frames(got[2:], _oracle(b, spec, srcs[2:]), "after the call, oracle")


@pytest.mark.gpu
def test_two_streams_with_frames_in_flight(torch_cuda):
    torch = torch_cuda
    spec = LP_SPEC
    _, d_in = _inputs(torch, spec, 12)
    d_out = _outputs(torch, spec, 12)
    ft = FrameTransformer(t360.make_context(**LP_A), spec)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for f in range(12):
        if f == 6:
            ft.vft.reconfigure(t360.make_context(**LP_B))
        assert _frame_call(ft.vft, spec, d_in[f], d_out[f])(streams[f % 2].cuda_stream)
    for s in streams:
        s.synchronize()
    got = _host(spec, d_out)
    ft.close()
    _assert_frames(got[:6], _fresh(torch, t360.make_context(**LP_A), spec, d_in[:6]), "before the call")
    _assert_frames(got[6:], _fresh(torch, t360.make_context(**LP_B), spec, d_in[6:]), "after the call")


@pytest.mark.gpu
def test_refused_context_keeps_the_old_configuration(torch_cuda):
    torch = torch_cuda
    spec = LP_SPEC
    _, d_in = _inputs(torch, spec, 6)
    d_out = _outputs(torch, spec, 6)
    ft = FrameTransformer(t360.make_context(**LP_A), spec)
    bytes_before = [ft.vft.plan_device_bytes(i) for i in (0, 1)]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for f in range(6):
        if f == 3:
            with pytest.raises(RuntimeError):
                ft.vft.reconfigure(t360.make_context(**REFUSED))
        assert _frame_call(ft.vft, spec, d_in[f], d_out[f])(st.cuda_stream)
    st.synchronize()
    got = _host(spec, d_out)
    assert [ft.vft.plan_device_bytes(i) for i in (0, 1)] == bytes_before
    ft.close()
    _assert_frames(got, _fresh(torch, t360.make_context(**LP_A), spec, d_in), "after a refused context")


@pytest.mark.gpu
def test_context_replaced_before_the_first_plan(torch_cuda):
    torch = torch_cuda
    spec = LP_SPEC
    _, d_in = _inputs(torch, spec, 1)
    vft = t360.VideoFrameTransform(t360.make_context(**LP_A))
    vft.reconfigure(t360.make_context(**LP_B))
    for p in (0, 1):
        assert vft.generateMapForPlane(*spec.plane_dims(p)[:4], p)
    out = _outputs(torch, spec, 1)
    torch.cuda.synchronize()
    assert _frame_call(vft, spec, d_in[0], out[0])(0)
    torch.cuda.synchronize()
    vft.close()
    _assert_frames(_host(spec, out), _fresh(torch, t360.make_context(**LP_B), spec, d_in), "planned after the call")


@pytest.mark.gpu
def test_repeated_reconfigures_release_the_old_plans(torch_cuda):
    """Twenty alternating reconfigures (kernel size, low-pass on and off, view), frames in between: device memory does not
    grow, and each index holds the device bytes of a fresh transform's plan."""
    torch = torch_cuda
    spec = StreamSpec(1920, 960, 768, 512)
    a = dict(LOW_PASS)
    b = dict(CUBIC_NO_LP, interpolation_alg=t360.LANCZOS4, fixed_yaw=45.0)
    _, d_in = _inputs(torch, spec, 1)
    d_out = _outputs(torch, spec, 1)
    ft = FrameTransformer(t360.make_context(**a), spec)
    st = torch.cuda.Stream()
    call = _frame_call(ft.vft, spec, d_in[0], d_out[0])

    def cycle(ov):
        ft.vft.reconfigure(t360.make_context(**ov))
        assert call(st.cuda_stream)

    torch.cuda.synchronize()
    assert call(st.cuda_stream)
    for ov in (b, a):  # first use of every table and scratch plane
        cycle(ov)
    st.synchronize()
    free_before = torch.cuda.mem_get_info()[0]
    for k in range(20):
        cycle(b if k % 2 == 0 else a)
    st.synchronize()
    free_after = torch.cuda.mem_get_info()[0]
    assert free_before - free_after <= 4 << 20, f"{(free_before - free_after) >> 20} MB of device memory not released"
    got = [ft.vft.plan_device_bytes(i) for i in (0, 1)]
    ft.close()
    fresh = FrameTransformer(t360.make_context(**a), spec)
    assert got == [fresh.vft.plan_device_bytes(i) for i in (0, 1)]
    fresh.close()


FILTER_ARGS = "cube_edge_length=64:interpolation_alg=cubic:enable_low_pass_filter=0"


RECORDS = ROOT / "tests" / "golden" / "reconfigure_reference.json"


def _reference_filter_frame(args, w, h, planes):
    """The reference software filter's frame for `args` (oracle/_ref): live where it is built, checked against its
    digests in reconfigure_reference.json, else those digests.  T360_RECORD_LIVE_REFERENCE=1 rewrites the record."""
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


@pytest.mark.gpu
def test_cuda_filter_yaw_command_between_frames(command_filter):
    """transform360_cuda: three frames, the command `yaw 30`, three more frames: the reference software filter's frames
    without and then with yaw=30.  A command before the first frame only sets the parameter."""
    w, h = 512, 256
    planes = [co.noise_plane(w, h, 0, 3), co.noise_plane((w + 1) // 2, (h + 1) // 2, 1, 3), co.noise_plane((w + 1) // 2, (h + 1) // 2, 2, 3)]
    want = [_reference_filter_frame(FILTER_ARGS, w, h, planes), _reference_filter_frame(FILTER_ARGS + ":yaw=30", w, h, planes)]
    import torch
    if not torch.cuda.is_available():
        pytest.fail("needs a CUDA device")
    dev = [torch.from_numpy(p).cuda() for p in planes]
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):  # (the output frames are allocated and cleared on the filter's stream)
        gpu = command_filter(FILTER_ARGS + ":sync=0", w, h, stream=stream)
        assert [gpu.out_w, gpu.out_h] == want[0]["size"] == want[1]["size"]
        got = []
        for frame in range(6):  # no synchronisation between the frames (sync=0)
            if frame == 3:
                assert _command(gpu, "yaw", "30") == 0
            got.append(gpu.filter(dev))
        stream.synchronize()
        for frame, out in enumerate(got):
            for p in range(3):
                assert rh.sha16(out[p].cpu().numpy()) == want[1 if frame >= 3 else 0]["planes"][p], f"plane {p} of frame {frame}"
        assert _command(gpu, "output_layout", "eac_32") == ENOSYS
        assert _command(gpu, "yaw", "abc") == EINVAL
        assert _params(gpu)["yaw"] == 30.0
        gpu.close()
        early = command_filter(FILTER_ARGS, w, h, stream=stream)
        assert _command(early, "yaw", "30") == 0
        out = early.filter(dev)
        stream.synchronize()
        assert [rh.sha16(o.cpu().numpy()) for o in out] == want[1]["planes"]
        early.close()
