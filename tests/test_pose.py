"""Per-frame poses for every output layout (T360B200_transformFramePoseAsync, VideoFrameTransform.make_pose_frame_call,
FrameTransformer.pose_frame_call) and the transform360_cuda pose commands that use it.

The contract: a frame enqueued with a pose (yaw, pitch, roll, hfov, vfov) equals, bit for bit, what a fresh transform gives
for the transform's context with its five view fields replaced by the pose -- low-pass, area resize and the barrel layouts'
transparent border included -- without a re-plan and without synchronising the device.  FLAT_FIXED goes through the
per-view kernel, every other layout through the per-frame orientation kernel, which here gains BARREL and BARREL_SPLIT
(csrc/oriented_view.h: barrelPoint) and BORDER_TRANSPARENT.  T360B200_poseSamples runs the same position chains on the
host and is checked against the planner."""
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
from tests.test_oriented import _angle, _jitter, _sweep
from tests.test_reconfigure import ROOT, _command, _params, command_filter, commands_library  # noqa: F401 (fixtures)
from tests.test_view import _assert_planes, _bad_planes_are_refused, _host, _inputs, _pitch, _planes, _refused_for, torch_cuda  # noqa: F401 (fixture)
from transform360_b200.stream import FrameTransformer, StreamSpec

BARREL, SPLIT = t360.LAYOUT_BARREL, t360.LAYOUT_BARREL_SPLIT
ALL_OUTPUTS = [t360.LAYOUT_CUBEMAP_32, t360.LAYOUT_CUBEMAP_23_OFFCENTER, t360.LAYOUT_FLAT_FIXED, t360.LAYOUT_EQUIRECT,
               BARREL, SPLIT, t360.LAYOUT_EAC_32]


# ---- no GPU needed ----------------------------------------------------------------------------------------------------
def test_pose_entry_points_are_exported_with_their_bindings():
    from transform360_b200.handler import EXPORTED_SYMBOLS, LIB_PATH
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    L = t360.load()
    for name in ("T360B200_transformFramePoseAsync", "T360B200_poseSamples"):
        assert name in EXPORTED_SYMBOLS and name in defined, name
        assert getattr(L, name).restype is C.c_int
    assert C.sizeof(t360.T360Pose) == 20
    assert [f[0] for f in t360.T360Pose._fields_] == ["yaw", "pitch", "roll", "hfov", "vfov"]
    assert L.T360B200_transformFramePoseAsync.argtypes == [C.c_void_p, C.POINTER(t360.T360Pose), C.c_int] + [C.c_void_p] * 9
    assert L.T360B200_poseSamples.argtypes == [C.POINTER(t360.FrameTransformContext), C.POINTER(t360.T360Pose)] + [C.c_int] * 4 + [C.c_void_p]
    pose = t360.T360Pose(0, 0, 0, 120, 110)
    assert L.T360B200_transformFramePoseAsync(None, C.byref(pose), 1, None, None, None, None, None, None, None, None, None) == 0
    assert L.T360B200_poseSamples(C.byref(t360.make_context()), None, 64, 32, 16, 16, None) == 0
    assert L.T360B200_poseSamples(None, C.byref(pose), 64, 32, 16, 16, None) == 0
    assert hasattr(FrameTransformer, "pose_frame_call")


def _sweep_case(rng, n):
    """One seeded (context, pose, sizes) of the sample sweep: half of the cases barrel, the rest spread over the other five
    layouts."""
    stereo = [t360.STEREO_FORMAT_MONO, t360.STEREO_FORMAT_TB, t360.STEREO_FORMAT_LR]
    layout = [BARREL, SPLIT][n % 2] if n % 4 < 2 else ALL_OUTPUTS[[0, 1, 2, 3, 6][(n // 4) % 5]]
    pose = (_angle(rng, n, 0), _angle(rng, n, 1), _angle(rng, n, 2), float(rng.uniform(1, 400)), float(rng.uniform(1, 250)))
    ov = dict(enable_low_pass_filter=0, output_layout=layout,
              input_layout=[t360.LAYOUT_EQUIRECT, t360.LAYOUT_CUBEMAP_32, t360.LAYOUT_EAC_32][(n // 3) % 3],
              interpolation_alg=[t360.NEAREST, t360.LINEAR, t360.CUBIC, t360.LANCZOS4][(n // 5) % 4],
              input_stereo_format=stereo[(n // 7) % 3], output_stereo_format=stereo[(n // 11) % 3], vflip=int((n // 2) % 2),
              fixed_yaw=pose[0], fixed_pitch=pose[1], fixed_roll=pose[2], fixed_hfov=pose[3], fixed_vfov=pose[4])
    if n % 6 == 1:  # off-centre projections, horizontal ones with NaN records at the poles
        ov.update(fixed_cube_offcenter_x=float(rng.uniform(-0.6, 0.6)), fixed_cube_offcenter_y=float(rng.uniform(-0.6, 0.6)),
                  fixed_cube_offcenter_z=float(rng.uniform(-0.9, 0.9)), is_horizontal_offset=int(n % 12 == 1))
    if n % 5 == 3:  # expand coefficients above and below 1 (the barrel discs shrink below 1 and grow past the square above)
        ov.update(expand_coef=float(rng.choice([1.01, 1.2, 0.9, 0.75])), input_expand_coef=float(rng.choice([1.01, 1.05])))
    if n % 13 == 0:
        ov.update(width_scale_factor=float(rng.choice([0.5, 2.0])), height_scale_factor=float(rng.choice([0.5, 2.0])))
    sizes = (int(rng.integers(16, 120)) * 2 + int(n % 2), int(rng.integers(8, 60)) * 2 + 1, int(rng.integers(3, 40)) * 2 + int(n % 3 == 0),
             int(rng.integers(3, 30)) * 2 + 1)
    return ov, pose, sizes


def test_pose_samples_equal_the_planner_over_a_seeded_sweep():
    """648 poses over all seven output layouts (half of them BARREL or BARREL_SPLIT), EQUIRECT, CUBEMAP_32 and EAC_32 input
    (the planner reads it as equirect), mono / TB / LR input and output with and without vflip, every interpolator, expand
    coefficients above and below 1, off-centre vectors with and without is_horizontal_offset, scale factors 0.5 and 2, odd
    sizes and test_oriented's special angles.  The sweep must reach the barrel dead zones, both sides of the equirect-input
    clamp, every quarter of BARREL_SPLIT's caps and the NaN records of a barrel plan."""
    rng = np.random.default_rng(20261016)
    cases = [_sweep_case(rng, n) for n in range(624)]
    for m in range(24):  # horizontal off-centre barrels whose cap centre is a pixel centre: the pole, a NaN record
        o = (_angle(rng, m, 0), _angle(rng, m, 1), _angle(rng, m, 2), 120.0, 110.0)
        cases.append((dict(enable_low_pass_filter=0, output_layout=BARREL, interpolation_alg=[t360.NEAREST, t360.CUBIC][m % 2],
                           fixed_cube_offcenter_x=0.1 * (m % 5), fixed_cube_offcenter_z=-0.5, is_horizontal_offset=1,
                           fixed_yaw=o[0], fixed_pitch=o[1], fixed_roll=o[2]), o,
                      (int(rng.integers(16, 120)) * 2 + 1, 61, [5, 15, 25][m % 3], [6, 10, 14][(m // 3) % 3])))
    assert sum(ov["output_layout"] in (BARREL, SPLIT) for ov, _, _ in cases) * 2 >= len(cases)
    reached = dict(dead=0, nan=0, clamp_lo=0, clamp_hi=0, quarters=set())
    for n, (ov, pose, sizes) in enumerate(cases):
        base = t360.make_context(**dict(ov, fixed_yaw=3.0, fixed_pitch=-7.0, fixed_roll=11.0, fixed_hfov=100.0, fixed_vfov=80.0))
        got = t360.pose_samples(base, pose, *sizes)  # the samples come from `pose` alone
        plan = t360.HostPlan(t360.make_context(**ov), *sizes)
        want = plan.samples
        assert got.shape == want.shape, (n, ov, sizes)
        assert np.array_equal(got, want), f"case {n} {ov} {sizes}: {int((got != want).any(axis=2).sum())} records differ"
        if ov["output_layout"] not in (BARREL, SPLIT):
            continue
        col0 = want[..., 0]
        dead = (col0 > -32768) & (col0 < -8)  # u = -1: a whole plane width left of the source
        reached["dead"] += int(dead.sum())
        reached["nan"] += int((col0 <= -32768).sum())
        in_w = sizes[0]
        in_layout, in_stereo = ov.get("input_layout", t360.LAYOUT_EQUIRECT), ov.get("input_stereo_format", t360.STEREO_FORMAT_MONO)
        if in_layout != t360.LAYOUT_CUBEMAP_32 and in_stereo != t360.STEREO_FORMAT_LR:  # (u not re-packed)
            w = np.float32(1.0) / np.float32(in_w)
            lo = w * np.float32(0.5)
            hi = np.float32(1.0) - lo
            x = plan.map[..., 0]
            reached["clamp_lo"] += int((x == lo * np.float32(in_w) - np.float32(0.5)).sum())
            reached["clamp_hi"] += int((x == hi * np.float32(in_w) - np.float32(0.5)).sum())
        if ov["output_layout"] == SPLIT and in_stereo == t360.STEREO_FORMAT_MONO:  # (no output eye split)
            map_w, map_h = want.shape[1], want.shape[0]
            x = (np.arange(map_w, dtype=np.float32) + np.float32(0.5)) / np.float32(map_w)
            y = np.float32(1.0) - (np.arange(map_h, dtype=np.float32) + np.float32(0.5)) / np.float32(map_h)
            cap = np.float32(3.0) * x > np.float32(2.0)
            quarter = (y * np.float32(4.0)).astype(np.int32)
            for q in range(4):
                if (~dead[quarter == q][:, cap]).any():
                    reached["quarters"].add(q)
    assert reached["dead"] > 0, "the sweep should reach the barrel dead zones"
    assert reached["nan"] > 0, "the sweep should reach the NaN records of a horizontal off-centre barrel"
    assert reached["clamp_lo"] > 0 and reached["clamp_hi"] > 0, f"the sweep should reach both sides of the equirect clamp: {reached}"
    assert reached["quarters"] == {0, 1, 2, 3}, f"BARREL_SPLIT cap quarters reached: {sorted(reached['quarters'])}"


def test_pose_samples_refuse_non_finite_poses_and_unknown_layouts():
    for bad in [(math.nan, 0, 0, 120, 110), (0, math.inf, 0, 120, 110), (0, 0, -math.inf, 120, 110), (0, 0, 0, math.nan, 110),
                (0, 0, 0, 120, math.inf)]:
        with pytest.raises(ValueError):
            t360.pose_samples(t360.make_context(output_layout=BARREL), bad, 64, 32, 16, 16)
    with pytest.raises(ValueError):
        t360.pose_samples(t360.make_context(output_layout=7), (0, 0, 0, 120, 110), 64, 32, 16, 16)
    with pytest.raises(ValueError):
        t360.pose_samples(t360.make_context(output_layout=BARREL, interpolation_alg=3), (0, 0, 0, 120, 110), 64, 32, 16, 16)


def test_pose_frames_are_refused_before_any_device_work(capfd):
    """Non-finite poses (each of the five fields), plane counts outside 1..3, plan indices that were never generated and
    invalid planes are refused (return 0) before the call touches CUDA, so this needs no device.  (A transform without
    interpolation algorithm needs a generated plan: tested on the GPU.)"""
    dummy = [(1 << 20, 512)] * 3
    dims = [(512, 256, 160, 64), (256, 128, 80, 32), (256, 128, 80, 32)]
    for layout in ALL_OUTPUTS:
        vft = t360.VideoFrameTransform(t360.make_context(output_layout=layout, enable_low_pass_filter=0))
        call = vft.make_pose_frame_call(dummy, dummy, dims)
        for f in range(5):
            for bad in (math.nan, math.inf, -math.inf):
                pose = [10.0, 0.0, 5.0, 120.0, 110.0]
                pose[f] = bad
                _refused_for(capfd, "is not finite", call, pose)
        _refused_for(capfd, "no map was generated for index 0", call, (10.0, 0.0, 5.0, 120.0, 110.0))
        _refused_for(capfd, "0 planes", vft.make_pose_frame_call([], [], []), (10.0, 0.0, 5.0, 120.0, 110.0))
        _refused_for(capfd, "6 planes", vft.make_pose_frame_call(dummy * 2, dummy * 2, dims * 2), (10.0, 0.0, 5.0, 120.0, 110.0))
        _bad_planes_are_refused(capfd, vft.make_pose_frame_call, ((10.0, 0.0, 5.0, 120.0, 110.0),), dummy, dims)
        vft.close()


FILTER_BARREL = "output_layout=barrel:w=640:h=256:interpolation_alg=cubic"
FILTER_CUBE = "cube_edge_length=128:interpolation_alg=cubic"


def test_cuda_filter_pose_commands_before_the_first_frame_only_set_parameters(command_filter):
    f = command_filter(FILTER_BARREL, 512, 256, device=False)
    for name, (arg, value) in {"yaw": ("30", 30.0), "roll": ("15", 15.0), "pitch": ("-12.5", -12.5)}.items():
        before = _params(f)
        assert _command(f, name, arg) == 0, name
        after = _params(f)
        assert after[name] == pytest.approx(value) and after[name] != before[name], name
        assert {k: v for k, v in after.items() if k != name} == {k: v for k, v in before.items() if k != name}, name
    assert _command(f, "roll", "abc") < 0 and _params(f)["roll"] == 15.0
    f.close()


# ---- on the GPU ---------------------------------------------------------------------------------------------------------
def _pattern(w, h, plane):
    """The seeded, nowhere-zero bytes every output buffer holds before a frame, so that "left untouched" is visible."""
    return co.noise_plane(w, h, plane=plane, frame=4242) | np.uint8(1)


def _outputs(torch, spec, frames):
    out = []
    for _ in range(frames):
        row = []
        for p in range(3):
            ow, oh = spec.plane_dims(p)[2:4]
            row.append(torch.from_numpy(_pattern(_pitch(ow), oh, p)).cuda())
        out.append(row)
    return out


def _with_pose(ov, pose):
    return dict(ov, fixed_yaw=pose[0], fixed_pitch=pose[1], fixed_roll=pose[2], fixed_hfov=pose[3], fixed_vfov=pose[4])


def _fresh(torch, ov, pose, spec, d_in):
    """What a fresh transform made for the context with `pose` gives (whole-frame entry point, same pre-filled output)."""
    ft = FrameTransformer(t360.make_context(**_with_pose(ov, pose)), spec)
    out = _outputs(torch, spec, 1)
    torch.cuda.synchronize()
    assert ft.frame_call(_planes(d_in), _planes(out[0]))(0)
    torch.cuda.synchronize()
    ft.close()
    return _host(spec, out)[0]


def _oracle(ov, pose, spec, src):
    octx = rh.default_context(**_with_pose(ov, pose))
    plans, row = {}, []
    for p in range(3):
        iw, ih, ow, oh, idx = spec.plane_dims(p)
        if idx not in plans:
            plans[idx] = co.OraclePlan(octx, iw, ih, ow, oh)
        row.append(co.transform_plane(octx, plans[idx], src[p], ow, oh, map_index=idx, prefill=_pattern(_pitch(ow), oh, p)[:, :ow]))
    return row


def _trajectory(name, n):
    """A shaky pan, then a 720-degree yaw sweep over a pole with roll (test_oriented), the field of view breathing."""
    seed = zlib.crc32(name.encode())
    half = n // 2
    rng = np.random.default_rng(seed + 2)
    fov = [(float(np.float32(100 + 25 * math.sin(f))), float(np.float32(80 + 20 * math.cos(f)))) for f in rng.uniform(0, 6.3, n)]
    return [o + f for o, f in zip(_jitter(seed, half) + _sweep(seed + 1, n - half), fov)]


LOW_PASS = dict(enable_low_pass_filter=1, num_horizontal_segments=8, num_vertical_segments=9)
CONFIGS = {  # name: (context, luma in, luma out, poses, oracle frames)
    "barrel_full_cubic": (dict(output_layout=BARREL, interpolation_alg=t360.CUBIC, enable_low_pass_filter=0), (7680, 3840), (5760, 2304), 6, 1),
    "split_linear_low_pass": (dict(output_layout=SPLIT, interpolation_alg=t360.LINEAR, **LOW_PASS), (961, 481), (723, 482), 14, 2),
    "barrel_nearest": (dict(output_layout=BARREL, interpolation_alg=t360.NEAREST, enable_low_pass_filter=0), (961, 481), (641, 257), 14, 2),
    "split_lanczos4_low_pass": (dict(output_layout=SPLIT, interpolation_alg=t360.LANCZOS4, **LOW_PASS), (1920, 960), (960, 640), 12, 2),
    "barrel_tb_stereo_vflip": (dict(output_layout=BARREL, interpolation_alg=t360.CUBIC, input_stereo_format=t360.STEREO_FORMAT_TB,
                                    output_stereo_format=t360.STEREO_FORMAT_TB, vflip=1), (960, 960), (640, 514), 14, 2),
    "split_lr_stereo_input": (dict(output_layout=SPLIT, interpolation_alg=t360.CUBIC, input_stereo_format=t360.STEREO_FORMAT_LR,
                                   output_stereo_format=t360.STEREO_FORMAT_TB, enable_low_pass_filter=0), (1922, 480), (721, 480), 14, 2),
    "cube_input_to_barrel": (dict(input_layout=t360.LAYOUT_CUBEMAP_32, output_layout=BARREL, interpolation_alg=t360.CUBIC,
                                  enable_low_pass_filter=0), (1536, 1024), (800, 320), 14, 2),
    "barrel_horizontal_offcentre": (dict(output_layout=BARREL, interpolation_alg=t360.CUBIC, enable_low_pass_filter=0, fixed_cube_offcenter_x=0.3,
                                         fixed_cube_offcenter_z=-0.5, is_horizontal_offset=1), (960, 480), (645, 258), 14, 2),
    "barrel_scale_half": (dict(output_layout=BARREL, interpolation_alg=t360.CUBIC, width_scale_factor=0.5, height_scale_factor=0.5),
                          (960, 480), (640, 256), 12, 2),
    "split_scale_two": (dict(output_layout=SPLIT, interpolation_alg=t360.CUBIC, width_scale_factor=2.0, height_scale_factor=2.0,
                             enable_low_pass_filter=0), (960, 480), (480, 320), 12, 2),
    "cubemap": (dict(interpolation_alg=t360.CUBIC, **LOW_PASS), (1920, 960), (960, 640), 12, 1),
    "flat_fixed": (dict(output_layout=t360.LAYOUT_FLAT_FIXED, interpolation_alg=t360.CUBIC, **LOW_PASS), (1920, 960), (640, 360), 12, 1),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_pose_frames_equal_fresh_transforms(name, torch_cuda):
    """A seeded trajectory (a shaky pan, then a 720-degree yaw sweep over a pole with roll) enqueued back to back on a
    non-default stream without synchronisation, into outputs pre-filled with a non-zero pattern: every frame equals a fresh
    transform made for its pose, and the plain-C oracle on a subset."""
    torch = torch_cuda
    ov, inp, out, n, n_oracle = CONFIGS[name]
    spec = StreamSpec(*inp, *out)
    poses = _trajectory(name, n)
    srcs, d_in = _inputs(torch, spec, 2)
    d_out = _outputs(torch, spec, n)
    ft = FrameTransformer(t360.make_context(**ov), spec)
    calls = [ft.pose_frame_call(_planes(d_in[f % 2]), _planes(d_out[f])) for f in range(n)]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for f, pose in enumerate(poses):
        assert calls[f](pose, st.cuda_stream), f"frame {f} pose {pose} refused"
    st.synchronize()
    got = _host(spec, d_out)
    ft.close()
    for f, pose in enumerate(poses):
        _assert_planes(got[f], _fresh(torch, ov, pose, spec, d_in[f % 2]), f"{name} frame {f} pose {pose}")
    for f in np.linspace(0, n - 1, n_oracle).astype(int):
        _assert_planes(got[f], _oracle(ov, poses[f], spec, srcs[f % 2]), f"{name} frame {f} pose {poses[f]}, oracle")


@pytest.mark.gpu
def test_two_streams_and_a_reconfigure_in_flight(torch_cuda):
    """Pose frames on two streams, a reconfigure (BARREL cubic -> BARREL_SPLIT Lanczos4 with other low-pass bands) in the
    middle: every frame has the configuration in effect when it was enqueued, with its own pose."""
    torch = torch_cuda
    a = dict(output_layout=BARREL, interpolation_alg=t360.CUBIC, num_vertical_segments=7, num_horizontal_segments=3)
    b = dict(a, output_layout=SPLIT, interpolation_alg=t360.LANCZOS4, num_vertical_segments=11)
    spec = StreamSpec(960, 480, 720, 480)
    poses = _trajectory("two_streams", 12)
    _, d_in = _inputs(torch, spec, 2)
    d_out = _outputs(torch, spec, 12)
    ft = FrameTransformer(t360.make_context(**a), spec)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for f, pose in enumerate(poses):
        if f == 6:
            ft.vft.reconfigure(t360.make_context(**b))
        assert ft.pose_frame_call(_planes(d_in[f % 2]), _planes(d_out[f]))(pose, streams[f % 2].cuda_stream)
    for s in streams:
        s.synchronize()
    got = _host(spec, d_out)
    ft.close()
    for f, pose in enumerate(poses):
        _assert_planes(got[f], _fresh(torch, a if f < 6 else b, pose, spec, d_in[f % 2]), f"frame {f} pose {pose}")


@pytest.mark.gpu
def test_device_memory_and_launches_stay_bounded(torch_cuda):
    """1000 distinct poses: device memory does not grow, and without low-pass a barrel frame is one kernel launch (the
    gather of all three planes; the chroma pre-fill is a memset, not a kernel)."""
    torch = torch_cuda
    spec = StreamSpec(1920, 960, 1280, 512)
    _, d_in = _inputs(torch, spec, 1)
    d_out = _outputs(torch, spec, 1)
    poses = _trajectory("bounded", 1000)
    st = torch.cuda.Stream()
    for ov in (dict(output_layout=BARREL, enable_low_pass_filter=0), dict(output_layout=SPLIT, num_vertical_segments=9, num_horizontal_segments=4)):
        ft = FrameTransformer(t360.make_context(**ov), spec)
        call = ft.pose_frame_call(_planes(d_in[0]), _planes(d_out[0]))
        torch.cuda.synchronize()
        for pose in poses[:50]:  # first use of every scratch plane and ring entry
            assert call(pose, st.cuda_stream)
        st.synchronize()
        free_before = torch.cuda.mem_get_info()[0]
        n0 = t360.kernel_launch_count()
        for pose in poses:
            assert call(pose, st.cuda_stream)
        launches = t360.kernel_launch_count() - n0
        st.synchronize()
        free_after = torch.cuda.mem_get_info()[0]
        ft.close()
        assert free_before - free_after <= 4 << 20, f"{(free_before - free_after) >> 20} MB of device memory not released ({ov})"
        if not ov.get("enable_low_pass_filter", 1):
            assert launches == len(poses), f"{launches} launches for {len(poses)} frames"
        else:
            assert launches <= 4 * len(poses), f"{launches} launches for {len(poses)} frames"


@pytest.mark.gpu
def test_refusals_of_generated_transforms(torch_cuda):
    """A transform without interpolation algorithm and input planes of another size are refused with no kernel launched."""
    torch = torch_cuda
    spec = StreamSpec(960, 480, 640, 256)
    _, d_in = _inputs(torch, spec, 1)
    d_out = _outputs(torch, spec, 1)
    none = FrameTransformer(t360.make_context(output_layout=BARREL, interpolation_alg=3, enable_low_pass_filter=0), spec)
    ft = FrameTransformer(t360.make_context(output_layout=BARREL, enable_low_pass_filter=0), spec)
    dims = [spec.plane_dims(p)[:4] for p in range(3)]
    dims[0] = (dims[0][0] - 2, dims[0][1], dims[0][2], dims[0][3])
    n0 = t360.kernel_launch_count()
    assert not none.pose_frame_call(_planes(d_in[0]), _planes(d_out[0]))((1.0, 2.0, 3.0, 120.0, 110.0), 0)
    assert not ft.vft.make_pose_frame_call(_planes(d_in[0]), _planes(d_out[0]), dims)((1.0, 2.0, 3.0, 120.0, 110.0))
    assert t360.kernel_launch_count() == n0
    assert ft.pose_frame_call(_planes(d_in[0]), _planes(d_out[0]))((1.0, 2.0, 3.0, 120.0, 110.0), 0)
    torch.cuda.synchronize()
    none.close()
    ft.close()


RECORDS = ROOT / "tests" / "golden" / "pose_reference.json"


def _reference_filter_frame(args, w, h, planes):
    """The reference software filter's frame for `args` (oracle/_ref): live where it is built, checked against its digests
    in pose_reference.json, else those digests.  T360_RECORD_LIVE_REFERENCE=1 rewrites the record."""
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
@pytest.mark.parametrize("args, commands", [(FILTER_BARREL, [("yaw", "30"), ("roll", "15")]), (FILTER_CUBE, [("yaw", "30")])],
                         ids=["barrel", "cubemap"])
def test_cuda_filter_pose_commands_take_the_pose_path(command_filter, args, commands):
    """transform360_cuda: three frames, the commands, three more: the reference software filter's frames without and then
    with the new pose.  The commands re-plan nothing: each returns in under 5 ms."""
    w, h = 512, 256
    planes = _filter_planes(w, h)
    moved = args + "".join(f":{name}={arg}" for name, arg in commands)
    want = [_reference_filter_frame(args, w, h, planes), _reference_filter_frame(moved, w, h, planes)]
    import torch
    if not torch.cuda.is_available():
        pytest.fail("needs a CUDA device")
    dev = [torch.from_numpy(p).cuda() for p in planes]
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        gpu = command_filter(args + ":sync=0", w, h, stream=stream)
        assert [gpu.out_w, gpu.out_h] == want[0]["size"] == want[1]["size"]
        got, elapsed = [], []
        for frame in range(6):
            if frame == 3:
                for name, arg in commands:
                    t0 = time.perf_counter()
                    assert _command(gpu, name, arg) == 0
                    elapsed.append(time.perf_counter() - t0)
            got.append(gpu.filter(dev))
        stream.synchronize()
        for frame, out in enumerate(got):
            for p in range(3):
                assert rh.sha16(out[p].cpu().numpy()) == want[1 if frame >= 3 else 0]["planes"][p], f"plane {p} of frame {frame}"
        assert max(elapsed) < 0.005, f"the pose commands took {[round(e * 1e3, 1) for e in elapsed]} ms: they should not re-plan"
        for name, arg in commands:
            assert _params(gpu)[name] == float(arg)
        gpu.close()
