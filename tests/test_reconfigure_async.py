"""Replacing the context of a running transform without waiting for a re-plan (T360B200_reconfigureAsync,
T360B200_reconfigureWait, VideoFrameTransform.reconfigure_async / reconfigure_wait) and the transform360_cuda commands that
use it.

The contract: every frame enqueued after the call equals, bit for bit, what a fresh transform made with the new context
gives -- first from the per-frame kernels, then, once the background planner has swapped the new plans in, from the planned
frame kernel -- and every frame enqueued before it is the old context's.  A refused context leaves the old one in effect
and enqueues nothing.  Outputs are pre-filled with a non-zero pattern, so that pixels a path leaves untouched are seen."""
import ctypes as C
import errno
import json
import math
import os
import shutil
import subprocess
import threading
import time
from pathlib import Path

import numpy as np
import pytest

import transform360_b200 as t360
from oracle import c_oracle as co
from oracle import ff_harness as ff
from oracle import ref_harness as rh
from transform360_b200.stream import FrameTransformer, StreamSpec

ROOT = Path(__file__).resolve().parents[1]
ENOSYS, EINVAL = -errno.ENOSYS, -errno.EINVAL
BARREL, SPLIT = t360.LAYOUT_BARREL, t360.LAYOUT_BARREL_SPLIT
TB = t360.STEREO_FORMAT_TB


# ---- no GPU needed ----------------------------------------------------------------------------------------------------
def test_async_calls_are_exported_with_their_bindings():
    from transform360_b200.handler import EXPORTED_SYMBOLS, LIB_PATH
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    L = t360.load()
    for name in ("T360B200_reconfigureAsync", "T360B200_reconfigureWait"):
        assert name in EXPORTED_SYMBOLS and name in defined, name
        assert getattr(L, name).restype is C.c_int
    assert L.T360B200_reconfigureAsync.argtypes == [C.c_void_p, C.POINTER(t360.FrameTransformContext)]
    assert L.T360B200_reconfigureWait.argtypes == [C.c_void_p, C.c_int]
    assert L.T360B200_reconfigureAsync(None, C.byref(t360.make_context())) == 0
    assert L.T360B200_reconfigureWait(None, 0) == -1 and L.T360B200_reconfigureWait(None, 1) == -1
    vft = t360.VideoFrameTransform(t360.make_context())
    assert L.T360B200_reconfigureAsync(vft._h, None) == 0
    vft.close()


def test_reconfigure_async_before_any_plan_needs_no_device():
    """Before generateMapForPlane the call only stores the context: no CUDA call, so it succeeds without a device, and
    nothing is pending.  The host-side refusals need no plan either."""
    vft = t360.VideoFrameTransform(t360.make_context(enable_low_pass_filter=0))
    b = t360.make_context(fixed_yaw=30.0, interpolation_alg=t360.LANCZOS4, expand_coef=1.05)
    vft.reconfigure_async(b)
    assert vft.ctx is b
    assert vft.reconfigure_wait(False) == 1 and vft.reconfigure_wait(True) == 1
    for bad in (dict(output_layout=t360.LAYOUT_EAC_32), dict(input_stereo_format=TB), dict(width_scale_factor=2.0),
                dict(interpolation_alg=3), dict(fixed_pitch=math.nan), dict(expand_coef=math.inf),
                dict(enable_low_pass_filter=1, num_vertical_segments=0)):
        with pytest.raises(RuntimeError):
            vft.reconfigure_async(t360.make_context(**dict(dict(fixed_yaw=30.0, interpolation_alg=t360.LANCZOS4, expand_coef=1.05), **bad)))
        assert vft.ctx is b
    vft.close()


# ---- on the GPU ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests must run on an H100 (there is no CPU fallback to test)")
    return torch


def _pitch(w):
    return (w + 255) // 256 * 256


def _pattern(w, h, plane):
    return co.noise_plane(w, h, plane=plane, frame=4242) | np.uint8(1)


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
    return [[torch.from_numpy(_pattern(_pitch(spec.plane_dims(p)[2]), spec.plane_dims(p)[3], p)).cuda() for p in range(3)]
            for _ in range(frames)]


def _planes(frame):
    return [(t.data_ptr(), t.stride(0)) for t in frame]


def _host(spec, d_out):
    return [[o[:, :spec.plane_dims(p)[2]].cpu().numpy() for p, o in enumerate(frame)] for frame in d_out]


def _fresh(torch, ov, spec, d_in):
    """What a fresh transform made with `ov` gives for each input frame (whole-frame entry point, pre-filled outputs)."""
    ft = FrameTransformer(t360.make_context(**ov), spec)
    out = _outputs(torch, spec, len(d_in))
    torch.cuda.synchronize()
    for f, frame in enumerate(d_in):
        assert ft.frame_call(_planes(frame), _planes(out[f]))(0)
    torch.cuda.synchronize()
    ft.close()
    return _host(spec, out)


def _oracle(ov, spec, src):
    octx = rh.default_context(**ov)
    plans, row = {}, []
    for p in range(3):
        iw, ih, ow, oh, idx = spec.plane_dims(p)
        if idx not in plans:
            plans[idx] = co.OraclePlan(octx, iw, ih, ow, oh)
        row.append(co.transform_plane(octx, plans[idx], src[p], ow, oh, map_index=idx, prefill=_pattern(_pitch(ow), oh, p)[:, :ow]))
    return row


def _assert_planes(got, want, what):
    for p, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g, w), f"{what}: plane {p}: {int((g != w).sum())} px differ"


CUBIC = dict(interpolation_alg=t360.CUBIC, enable_low_pass_filter=0)
LOW_PASS = dict(interpolation_alg=t360.CUBIC, enable_low_pass_filter=1, num_vertical_segments=9, num_horizontal_segments=4)
FLAT = dict(CUBIC, output_layout=t360.LAYOUT_FLAT_FIXED, fixed_yaw=100.0, fixed_pitch=20.0)
BARREL_CUBIC = dict(CUBIC, output_layout=BARREL)
OFFCENTRE = dict(CUBIC, output_layout=t360.LAYOUT_CUBEMAP_23_OFFCENTER, fixed_cube_offcenter_z=-0.4)
STEREO_TB = dict(BARREL_CUBIC, input_stereo_format=TB, output_stereo_format=TB)
CUBE_IN = dict(CUBIC, input_layout=t360.LAYOUT_CUBEMAP_32, output_layout=BARREL)
PAIRS = {  # name: (context A, context B, luma in, luma out)
    "cube_pose": (CUBIC, dict(CUBIC, fixed_yaw=30.0, fixed_pitch=-20.0, fixed_roll=12.5), (960, 480), (480, 320)),
    "flat_fixed_pose": (FLAT, dict(FLAT, fixed_yaw=140.0, fixed_pitch=-30.0, fixed_hfov=80.0, fixed_vfov=60.0), (960, 480), (320, 180)),
    "barrel_pose": (BARREL_CUBIC, dict(BARREL_CUBIC, fixed_yaw=-45.0, fixed_pitch=10.0, fixed_roll=5.0), (960, 480), (640, 256)),
    "barrel_expand_coef": (BARREL_CUBIC, dict(BARREL_CUBIC, expand_coef=1.1), (960, 480), (640, 256)),
    "split_expand_coef": (dict(BARREL_CUBIC, output_layout=SPLIT), dict(BARREL_CUBIC, output_layout=SPLIT, expand_coef=0.95), (960, 480), (480, 320)),
    "cube_input_expand_coef": (CUBE_IN, dict(CUBE_IN, input_expand_coef=1.05), (768, 512), (640, 256)),
    "offcentre": (OFFCENTRE, dict(OFFCENTRE, fixed_cube_offcenter_x=0.2, fixed_cube_offcenter_z=-0.6), (960, 480), (320, 480)),
    "offcentre_horizontal": (OFFCENTRE, dict(OFFCENTRE, fixed_cube_offcenter_x=0.3, is_horizontal_offset=1), (960, 480), (320, 480)),
    "vflip_tb_stereo": (STEREO_TB, dict(STEREO_TB, vflip=1), (960, 960), (640, 514)),
    "cubic_to_lanczos4": (CUBIC, dict(CUBIC, interpolation_alg=t360.LANCZOS4), (960, 480), (480, 320)),
    "cubic_to_nearest": (CUBIC, dict(CUBIC, interpolation_alg=t360.NEAREST), (960, 480), (480, 320)),
    "nearest_to_cubic": (dict(CUBIC, interpolation_alg=t360.NEAREST), CUBIC, (960, 480), (480, 320)),
    "low_pass_off_to_on": (CUBIC, LOW_PASS, (960, 480), (240, 160)),
    "low_pass_on_to_off": (LOW_PASS, CUBIC, (960, 480), (240, 160)),
    "segment_counts": (LOW_PASS, dict(LOW_PASS, num_vertical_segments=15, num_horizontal_segments=8), (960, 480), (240, 160)),
    "segment_counts_uncovered": (dict(LOW_PASS, adjust_kernel=1, num_horizontal_segments=8),
                                 dict(LOW_PASS, adjust_kernel=1, num_horizontal_segments=0), (960, 480), (240, 160)),
    "adjust_kernel_on": (dict(OFFCENTRE, **{k: v for k, v in LOW_PASS.items() if k != "interpolation_alg"}, adjust_kernel=0),
                         dict(OFFCENTRE, **{k: v for k, v in LOW_PASS.items() if k != "interpolation_alg"}, adjust_kernel=1,
                              kernel_adjust_factor=1.5), (960, 480), (320, 480)),
    "barrel_low_pass_and_lanczos4": (BARREL_CUBIC, dict(BARREL_CUBIC, enable_low_pass_filter=1, interpolation_alg=t360.LANCZOS4,
                                                        expand_coef=1.05), (960, 480), (640, 256)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(PAIRS))
def test_frames_switch_at_the_call_and_stay_exact_across_the_swap(name, torch_cuda):
    """Three frames with A, reconfigure_async(B), three frames served while B's plan is pending, the wait, three more frames
    on B's plans -- on a non-default stream, never synchronised in between: A's frames, then B's, bit for bit against fresh
    transforms and a sample against the plain-C oracle; the plans then hold a fresh B's device bytes."""
    torch = torch_cuda
    a, b, inp, out = PAIRS[name]
    spec = StreamSpec(*inp, *out)
    srcs, d_in = _inputs(torch, spec, 9)
    d_out = _outputs(torch, spec, 9)
    ft = FrameTransformer(t360.make_context(**a), spec)
    calls = [ft.frame_call(_planes(d_in[f]), _planes(d_out[f])) for f in range(9)]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for f in range(3):
        assert calls[f](st.cuda_stream)
    ft.vft.reconfigure_async(t360.make_context(**b))
    for f in range(3, 6):
        assert calls[f](st.cuda_stream)
    assert ft.vft.reconfigure_wait(False) == 0, "the plan should still be pending (settle interval)"
    assert ft.vft.reconfigure_wait(True) == 1
    for f in range(6, 9):
        assert calls[f](st.cuda_stream)
    st.synchronize()
    got = _host(spec, d_out)
    bytes_after = [ft.vft.plan_device_bytes(i) for i in (0, 1)]
    ft.close()
    want_a, want_b = _fresh(torch, a, spec, d_in[:3]), _fresh(torch, b, spec, d_in[3:])
    for f in range(9):
        _assert_planes(got[f], want_a[f] if f < 3 else want_b[f - 3], f"{name} frame {f}")
    for f in (4, 7):
        _assert_planes(got[f], _oracle(b, spec, srcs[f]), f"{name} frame {f}, oracle")
    fresh = FrameTransformer(t360.make_context(**b), spec)
    assert bytes_after == [fresh.vft.plan_device_bytes(i) for i in (0, 1)]
    fresh.close()


LP_SPEC = StreamSpec(960, 480, 240, 160)


@pytest.mark.gpu
def test_refused_contexts_enqueue_nothing_and_keep_the_old_one(torch_cuda):
    torch = torch_cuda
    spec = LP_SPEC
    _, d_in = _inputs(torch, spec, 2)
    d_out = _outputs(torch, spec, 2)
    ft = FrameTransformer(t360.make_context(**LOW_PASS), spec)
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    assert ft.frame_call(_planes(d_in[0]), _planes(d_out[0]))(st.cuda_stream)
    st.synchronize()
    n0 = t360.kernel_launch_count()
    for bad in (dict(output_layout=t360.LAYOUT_EAC_32), dict(input_layout=t360.LAYOUT_CUBEMAP_32), dict(input_stereo_format=TB),
                dict(output_stereo_format=TB), dict(width_scale_factor=2.0), dict(height_scale_factor=0.5), dict(num_vertical_segments=0),
                dict(num_vertical_segments=-3), dict(interpolation_alg=3), dict(fixed_yaw=math.nan), dict(kernel_adjust_factor=math.nan),
                dict(fixed_cube_offcenter_x=math.inf)):
        with pytest.raises(RuntimeError):
            ft.vft.reconfigure_async(t360.make_context(**dict(dict(LOW_PASS, fixed_yaw=20.0), **bad)))
    assert t360.kernel_launch_count() == n0, "a refused context enqueued device work"
    assert ft.vft.reconfigure_wait(False) == 1
    assert ft.frame_call(_planes(d_in[1]), _planes(d_out[1]))(st.cuda_stream)
    st.synchronize()
    got = _host(spec, d_out)
    ft.close()
    want = _fresh(torch, LOW_PASS, spec, d_in)
    for f in range(2):
        _assert_planes(got[f], want[f], f"frame {f} after the refusals")


@pytest.mark.gpu
def test_superseded_plans_are_discarded(torch_cuda):
    """A -> B -> C with frames between the calls, B's plan started (settle interval over) before C arrives: every frame has
    the context in effect when it was enqueued, and C's plan is the one in effect (its device bytes, not B's)."""
    torch = torch_cuda
    spec = StreamSpec(3840, 1920, 1536, 1024)
    a, b, c = CUBIC, dict(LOW_PASS, fixed_yaw=30.0), dict(CUBIC, interpolation_alg=t360.LANCZOS4, fixed_pitch=-15.0)
    _, d_in = _inputs(torch, spec, 2)
    d_out = _outputs(torch, spec, 8)
    ft = FrameTransformer(t360.make_context(**a), spec)
    calls = [ft.frame_call(_planes(d_in[f % 2]), _planes(d_out[f])) for f in range(8)]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    assert calls[0](st.cuda_stream) and calls[1](st.cuda_stream)
    ft.vft.reconfigure_async(t360.make_context(**b))
    assert calls[2](st.cuda_stream) and calls[3](st.cuda_stream)
    time.sleep(0.3)  # (B's plan is being made now)
    ft.vft.reconfigure_async(t360.make_context(**c))
    assert calls[4](st.cuda_stream) and calls[5](st.cuda_stream)
    assert ft.vft.reconfigure_wait(True) == 1
    assert calls[6](st.cuda_stream) and calls[7](st.cuda_stream)
    st.synchronize()
    got = _host(spec, d_out)
    bytes_after = [ft.vft.plan_device_bytes(i) for i in (0, 1)]
    ft.close()
    for ov, frames in ((a, (0, 1)), (b, (2, 3)), (c, (4, 5, 6, 7))):
        want = _fresh(torch, ov, spec, d_in)
        for f in frames:
            _assert_planes(got[f], want[f % 2], f"frame {f}")
    fresh_b, fresh_c = (FrameTransformer(t360.make_context(**ov), spec) for ov in (b, c))
    assert bytes_after == [fresh_c.vft.plan_device_bytes(i) for i in (0, 1)]
    assert bytes_after != [fresh_b.vft.plan_device_bytes(i) for i in (0, 1)]
    fresh_b.close()
    fresh_c.close()


@pytest.mark.gpu
def test_swap_under_two_enqueuing_streams(torch_cuda):
    """Two threads enqueue whole frames back to back, each on its own stream and draining it after every frame as a
    filter does, while a third waits for the plan: the frames served before and after the swap equal a fresh B's, and no
    enqueue call takes longer than 50 ms (the re-plan takes far longer)."""
    torch = torch_cuda
    spec = StreamSpec(3840, 1920, 1536, 1024)
    a, b = CUBIC, dict(LOW_PASS, interpolation_alg=t360.LANCZOS4, fixed_yaw=25.0)
    _, d_in = _inputs(torch, spec, 2)
    want = [[torch.from_numpy(p).cuda() for p in frame] for frame in _fresh(torch, b, spec, d_in)]
    ft = FrameTransformer(t360.make_context(**a), spec)
    ring = 32  # output frames per thread, reused round robin: slot f % ring always receives input f % 2
    outs = [_outputs(torch, spec, ring) for _ in range(2)]
    calls = [[ft.frame_call(_planes(d_in[f % 2]), _planes(outs[k][f])) for f in range(ring)] for k in range(2)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    swapped, started = threading.Event(), threading.Barrier(3)
    times, before, after = [[], []], [0, 0], [0, 0]
    wrong = []

    def enqueue(k):
        started.wait()
        f = 0
        while after[k] < 2 * ring and f < 100000:
            done = swapped.is_set()
            t0 = time.perf_counter()
            if not calls[k][f % ring](streams[k].cuda_stream):
                wrong.append((k, f))
                return
            times[k].append(time.perf_counter() - t0)
            streams[k].synchronize()
            if done:
                after[k] += 1
            else:
                before[k] += 1
            f += 1

    def wait():
        started.wait()
        time.sleep(0.05)
        assert ft.vft.reconfigure_wait(True) == 1
        swapped.set()

    ft.vft.reconfigure_async(t360.make_context(**b))
    threads = [threading.Thread(target=enqueue, args=(k,)) for k in range(2)] + [threading.Thread(target=wait)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    ft.close()
    assert not wrong, f"refused frames: {wrong}"
    assert swapped.is_set() and min(before) > 0 and min(after) == 2 * ring, f"{before} frames before the swap, {after} after"
    for k in range(2):
        for f in range(ring):
            for p in range(3):
                got = outs[k][f][p][:, :spec.plane_dims(p)[2]]
                assert torch.equal(got, want[f % 2][p]), f"stream {k} slot {f} plane {p}"
    slowest = max(max(t) for t in times)
    assert slowest < 0.05, f"an enqueue call took {slowest * 1e3:.1f} ms during the swap"


@pytest.mark.gpu
def test_per_plane_entry_points_wait_for_the_plan(torch_cuda):
    """transformFramePlane (device pointers), transformFramePlaneAsync and lowPassPlaneAsync called while B's plan is
    pending give B's planes."""
    torch = torch_cuda
    spec = LP_SPEC
    a, b = LOW_PASS, dict(LOW_PASS, interpolation_alg=t360.LANCZOS4, num_vertical_segments=5, num_horizontal_segments=3, fixed_yaw=20.0)
    srcs, d_in = _inputs(torch, spec, 1)
    d_out = _outputs(torch, spec, 2)
    blurred = torch.zeros((spec.in_h, spec.in_w), dtype=torch.uint8, device="cuda")
    vft = t360.VideoFrameTransform(t360.make_context(**a))
    for p in (0, 1):
        assert vft.generateMapForPlane(*spec.plane_dims(p)[:4], p)
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    vft.reconfigure_async(t360.make_context(**b))
    for p in range(3):
        iw, ih, ow, oh, idx = spec.plane_dims(p)
        i, o = d_in[0][p], d_out[0][p]
        assert vft.transform_plane_async(i.data_ptr(), o.data_ptr(), iw, ih, i.stride(0), ow, oh, o.stride(0), idx, st.cuda_stream)
    st.synchronize()
    for p in range(3):
        iw, ih, ow, oh, idx = spec.plane_dims(p)
        i, o = d_in[0][p], d_out[1][p]
        assert vft.transformFramePlane(i.data_ptr(), o.data_ptr(), iw, ih, i.stride(0), ow, oh, o.stride(0), idx, p)
    i = d_in[0][0]
    assert vft.low_pass_async(i.data_ptr(), blurred.data_ptr(), spec.in_w, spec.in_h, i.stride(0), blurred.stride(0), 0, st.cuda_stream)
    st.synchronize()
    assert vft.reconfigure_wait(False) == 1
    got = _host(spec, d_out)
    vft.close()
    want = _fresh(torch, b, spec, d_in)[0]
    for f in range(2):
        _assert_planes(got[f], want, f"per-plane call {f}")
    octx = rh.default_context(**b)
    plan = co.OraclePlan(octx, *spec.plane_dims(0)[:4])
    assert np.array_equal(blurred.cpu().numpy(), co.filter_plane(octx, srcs[0][0], plan.segs, plan.nsegs, plan.taps)), "low-pass"


@pytest.mark.gpu
def test_repeated_async_cycles_release_the_old_plans(torch_cuda):
    torch = torch_cuda
    spec = StreamSpec(1920, 960, 768, 512)
    a, b = dict(LOW_PASS), dict(CUBIC, interpolation_alg=t360.LANCZOS4, fixed_yaw=45.0, expand_coef=1.05)
    _, d_in = _inputs(torch, spec, 1)
    d_out = _outputs(torch, spec, 1)
    ft = FrameTransformer(t360.make_context(**a), spec)
    st = torch.cuda.Stream()
    call = ft.frame_call(_planes(d_in[0]), _planes(d_out[0]))

    def cycle(ov):
        ft.vft.reconfigure_async(t360.make_context(**ov))
        assert call(st.cuda_stream)
        assert ft.vft.reconfigure_wait(True) == 1
        assert call(st.cuda_stream)

    torch.cuda.synchronize()
    for ov in (b, a):  # first use of every table, scratch plane and ring entry
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


def _tasks():
    return len(os.listdir("/proc/self/task"))


@pytest.mark.gpu
def test_close_with_a_pending_plan_leaves_no_thread(torch_cuda):
    torch = torch_cuda
    spec = StreamSpec(3840, 1920, 1536, 1024)
    _, d_in = _inputs(torch, spec, 1)
    d_out = _outputs(torch, spec, 1)

    def run(wait):
        ft = FrameTransformer(t360.make_context(**CUBIC), spec)
        ft.vft.reconfigure_async(t360.make_context(**dict(LOW_PASS, fixed_yaw=10.0)))
        assert ft.frame_call(_planes(d_in[0]), _planes(d_out[0]))(0)
        if wait:
            assert ft.vft.reconfigure_wait(True) == 1
        else:
            time.sleep(0.3)  # (the plan is being made)
        t0 = time.perf_counter()
        ft.close()
        return time.perf_counter() - t0

    run(True)  # the driver's and the runtime's own threads exist from here on
    torch.cuda.synchronize()
    before = _tasks()
    took = run(False)
    assert _tasks() == before, f"{_tasks() - before} threads left behind"
    assert took < 30, f"close() took {took:.1f} s"


# ---- transform360_cuda ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="session")
def commands_library(tmp_path_factory):
    """transform360_cuda around oracle/ff_driver.c, compiled against the stand-in plus tests/filter_commands (runtime options
    and process_command); built under a temporary directory."""
    cc = os.environ.get("CC") or shutil.which("gcc") or shutil.which("cc")
    assert cc, "a C compiler is needed to build the filter with runtime commands"
    out = tmp_path_factory.mktemp("filter_commands_async") / "libvf_t360_cuda_commands.so"
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
    monkeypatch.setitem(ff._LIBS, "cuda", commands_library)
    monkeypatch.setattr(ff, "_loaded", {})
    L = ff._lib("cuda")
    L.t360f_command.restype = C.c_int
    L.t360f_command.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
    return ff.CudaFilter


RECORDS = ROOT / "tests" / "golden" / "reconfigure_async_reference.json"
FILTER_ARGS = "cube_edge_length=64:interpolation_alg=cubic:enable_low_pass_filter=0"
COMMANDS = [("yaw", "30"), ("expand_coef", "1.05"), ("interpolation_alg", "lanczos4"), ("enable_low_pass_filter", "1")]


def _filter_planes(w, h):
    return [co.noise_plane(w, h, 0, 7), co.noise_plane((w + 1) // 2, (h + 1) // 2, 1, 7), co.noise_plane((w + 1) // 2, (h + 1) // 2, 2, 7)]


def _reference_filter_frame(args, w, h, planes):
    """The reference software filter's frame for `args` (oracle/_ref): live where it is built, checked against its digests
    in reconfigure_async_reference.json, else those digests.  T360_RECORD_LIVE_REFERENCE=1 rewrites the record."""
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


def _reference_after(k):
    """The filter arguments with the first k commands applied."""
    return FILTER_ARGS + "".join(f":{name}={arg}" for name, arg in COMMANDS[:k])


def test_reference_digests_are_recorded():
    w, h = 512, 256
    planes = _filter_planes(w, h)
    for k in range(len(COMMANDS) + 1):
        _reference_filter_frame(_reference_after(k), w, h, planes)


@pytest.mark.gpu
def test_cuda_filter_commands_take_effect_at_the_next_frame(command_filter):
    """transform360_cuda: two frames, then each command followed by two frames, then -- after the settle interval and the
    plan -- two more: the reference software filter's frames for the commands given so far.  Every command returns in under
    5 ms: none re-plans on the caller's thread."""
    w, h = 512, 256
    planes = _filter_planes(w, h)
    want = [_reference_filter_frame(_reference_after(k), w, h, planes) for k in range(len(COMMANDS) + 1)]
    import torch
    if not torch.cuda.is_available():
        pytest.fail("needs a CUDA device")
    dev = [torch.from_numpy(p).cuda() for p in planes]
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        gpu = command_filter(FILTER_ARGS + ":sync=0", w, h, stream=stream)
        assert [gpu.out_w, gpu.out_h] == want[0]["size"] == want[-1]["size"]
        got, expected, elapsed = [], [], []
        for k in range(len(COMMANDS) + 1):
            if k:
                t0 = time.perf_counter()
                assert gpu.L.t360f_command(gpu.h, COMMANDS[k - 1][0].encode(), COMMANDS[k - 1][1].encode()) == 0
                elapsed.append(time.perf_counter() - t0)
            for _ in range(2):
                got.append(gpu.filter(dev))
                expected.append(want[k]["planes"])
        time.sleep(1.5)  # the settle interval and the plan of a 512 x 256 frame
        for _ in range(2):
            got.append(gpu.filter(dev))
            expected.append(want[-1]["planes"])
        stream.synchronize()
        for frame, (out, digests) in enumerate(zip(got, expected)):
            for p in range(3):
                assert rh.sha16(out[p].cpu().numpy()) == digests[p], f"plane {p} of frame {frame}"
        assert max(elapsed) < 0.005, f"the commands took {[round(e * 1e3, 2) for e in elapsed]} ms"
        assert gpu.L.t360f_command(gpu.h, b"output_layout", b"eac_32") == ENOSYS
        assert gpu.L.t360f_command(gpu.h, b"yaw", b"abc") == EINVAL
        gpu.close()
