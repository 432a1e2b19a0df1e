"""Per-frame orientation for cube-map, EAC and equirect outputs (T360B200_transformFrameOrientedAsync,
VideoFrameTransform.make_oriented_frame_call, FrameTransformer.oriented_frame_call).

The contract: a frame enqueued with an orientation equals, bit for bit, what a fresh transform gives for the transform's
context with fixed_yaw / pitch / roll replaced by it -- low-pass and area resize included -- without a re-plan and without
synchronising the device.  The kernel computes each pixel's sampling record with csrc/oriented_view.h, whose equirect input
lookup needs atan2f and asinf exactly as the host libm computes them: csrc/libm_ports.h ports them, and the first test
compares the ports with the library over every float input (asinf, atanf) and 10^8 seeded pairs (atan2f, drawn by
tests/atan2_pairs.h).  That pins the host build; tests/test_twin_gates.py pins the device build to it, bit for bit.
T360B200_orientedSamples runs the chain on the host and is checked against the planner here."""
import ctypes as C
import math
import os
import shutil
import subprocess
import zlib

import numpy as np
import pytest

import transform360_b200 as t360
from tests.test_view import (_assert_planes, _bad_planes_are_refused, _host, _inputs, _outputs, _planes, _refused_for,  # noqa: F401 (fixture)
                             torch_cuda)
from oracle import c_oracle as co
from oracle import ref_harness as rh
from transform360_b200.stream import FrameTransformer, StreamSpec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "transform360_b200", "csrc")
SPHERE_OUTPUTS = [t360.LAYOUT_CUBEMAP_32, t360.LAYOUT_CUBEMAP_23_OFFCENTER, t360.LAYOUT_EAC_32, t360.LAYOUT_EQUIRECT]


# ---- no GPU needed ----------------------------------------------------------------------------------------------------
def test_libm_ports_equal_the_host_libm_bit_for_bit(tmp_path):
    """asinf and atanf over all 2^32 bit patterns, atan2f over 10^8 seeded pairs plus every pair of +-0, +-inf, NaNs,
    subnormals, the extreme normals and the arguments at the algorithms' range splits."""
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.fail("no C++ compiler to build the libm comparison")
    exe = tmp_path / "libm_gate"
    subprocess.run([cxx, "-std=c++17", "-O2", "-ffp-contract=off", "-fno-builtin", "-pthread", "-I", CSRC,
                    os.path.join(ROOT, "tests", "libm_gate.cpp"), "-o", str(exe), "-lm"], check=True)
    threads = max(8, os.cpu_count() or 1)
    r = subprocess.run([str(exe), str(threads), str(100_000_000), "20261015"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 mismatches" in r.stdout, r.stdout


def test_oriented_entry_points_are_exported_with_their_bindings():
    from transform360_b200.handler import EXPORTED_SYMBOLS, LIB_PATH
    out = subprocess.run(["nm", "-D", "--defined-only", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    defined = {line.split()[-1] for line in out.splitlines() if " T " in line}
    L = t360.load()
    for name in ("T360B200_transformFrameOrientedAsync", "T360B200_orientedSamples"):
        assert name in EXPORTED_SYMBOLS and name in defined, name
        assert getattr(L, name).restype is C.c_int
    assert C.sizeof(t360.T360Orientation) == 12
    assert L.T360B200_transformFrameOrientedAsync.argtypes[:3] == [C.c_void_p, C.POINTER(t360.T360Orientation), C.c_int]
    assert L.T360B200_orientedSamples.argtypes[:2] == [C.POINTER(t360.FrameTransformContext), C.POINTER(t360.T360Orientation)]
    o = t360.T360Orientation(0, 0, 0)
    assert L.T360B200_transformFrameOrientedAsync(None, C.byref(o), 1, None, None, None, None, None, None, None, None, None) == 0
    assert L.T360B200_orientedSamples(C.byref(t360.make_context()), None, 64, 32, 16, 16, None) == 0
    assert hasattr(FrameTransformer, "oriented_frame_call")


def _angle(rng, n, k):
    """Seeded angles: ordinary ones, then every so often +-90, +-180, -0.0, angles far outside +-180 and huge ones."""
    special = [90.0, -90.0, 180.0, -180.0, -0.0, 0.0, 89.999, -90.001, 270.0, -450.0, 720.0, 12345.678, -98765.4, 1.0e6]
    if (n + k) % 4 == 0:
        return float(rng.choice(special))
    return float(rng.uniform(-1000, 1000)) if (n + k) % 3 == 0 else float(rng.uniform(-200, 200))


def _sweep_case(rng, n):
    """One seeded (context, orientation, sizes) of the sample sweep."""
    stereo = [t360.STEREO_FORMAT_MONO, t360.STEREO_FORMAT_TB, t360.STEREO_FORMAT_LR]
    orientation = (_angle(rng, n, 0), _angle(rng, n, 1), _angle(rng, n, 2))
    ov = dict(enable_low_pass_filter=0, output_layout=SPHERE_OUTPUTS[n % 4],
              input_layout=t360.LAYOUT_CUBEMAP_32 if (n // 4) % 3 == 2 else t360.LAYOUT_EQUIRECT,
              interpolation_alg=[t360.NEAREST, t360.LINEAR, t360.CUBIC, t360.LANCZOS4][(n // 3) % 4],
              input_stereo_format=stereo[(n // 5) % 3], output_stereo_format=stereo[(n // 7) % 3], vflip=int((n // 2) % 2),
              fixed_yaw=orientation[0], fixed_pitch=orientation[1], fixed_roll=orientation[2])
    if n % 6 == 1:  # off-centre projections, horizontal ones with NaN records at the poles
        ov.update(fixed_cube_offcenter_x=float(rng.uniform(-0.6, 0.6)), fixed_cube_offcenter_y=float(rng.uniform(-0.6, 0.6)),
                  fixed_cube_offcenter_z=float(rng.uniform(-0.9, 0.9)), is_horizontal_offset=int(n % 12 == 1))
    if n % 5 == 3:
        ov.update(expand_coef=float(rng.choice([1.01, 1.1, 0.95])), input_expand_coef=float(rng.choice([1.01, 1.05])))
    if n % 11 == 0:
        ov.update(width_scale_factor=float(rng.choice([0.5, 2.0])), height_scale_factor=float(rng.choice([0.5, 2.0])))
    sizes = (int(rng.integers(16, 120)) * 2 + 1, int(rng.integers(8, 60)) * 2 + 1, int(rng.integers(3, 40)) * 2 + 1,
             int(rng.integers(3, 30)) * 2 + 1)
    return ov, orientation, sizes


def test_oriented_samples_equal_the_planner_over_a_seeded_sweep():
    """400 orientations (special angles, outside +-180, +-90 pitch, -0.0, 1e6) crossed with the four output layouts, both
    input layouts, mono / TB / LR input and output with and without vflip, every interpolator, off-centre vectors with
    and without is_horizontal_offset, expand coefficients, scale factors 0.5 and 2, odd plane sizes."""
    rng = np.random.default_rng(20261016)
    cases = [_sweep_case(rng, n) for n in range(384)]
    for m in range(16):  # horizontal off-centre projections whose map has a pixel at a pole's face centre: a NaN record
        layout = [t360.LAYOUT_CUBEMAP_32, t360.LAYOUT_EAC_32, t360.LAYOUT_CUBEMAP_23_OFFCENTER][m % 3]
        out = (6, 9) if layout == t360.LAYOUT_CUBEMAP_23_OFFCENTER else (9, 6)
        o = (_angle(rng, m, 0), _angle(rng, m, 1), _angle(rng, m, 2))
        cases.append((dict(enable_low_pass_filter=0, output_layout=layout, interpolation_alg=[t360.NEAREST, t360.CUBIC][m % 2],
                           fixed_cube_offcenter_x=0.1 * (m % 5), fixed_cube_offcenter_z=-0.5, is_horizontal_offset=1,
                           fixed_yaw=o[0], fixed_pitch=o[1], fixed_roll=o[2]), o, (int(rng.integers(16, 120)) * 2 + 1, 61) + out))
    nan_records = 0
    for n, (ov, orientation, sizes) in enumerate(cases):
        base = t360.make_context(**dict(ov, fixed_yaw=3.0, fixed_pitch=-7.0, fixed_roll=11.0))  # samples from `orientation` alone
        got = t360.oriented_samples(base, orientation, *sizes)
        want = t360.HostPlan(t360.make_context(**ov), *sizes).samples
        assert got.shape == want.shape, (n, ov, sizes)
        assert np.array_equal(got, want), f"case {n} {ov} {sizes}: {int((got != want).any(axis=2).sum())} records differ"
        nan_records += int((want[..., 0] <= -32768).sum()) if ov.get("is_horizontal_offset") else 0  # (NaN: INT_MIN >> 5, saturated)
    assert nan_records > 0, "the sweep should reach the NaN records of a horizontal off-centre projection"


def test_oriented_samples_refuse_other_layouts_and_non_finite_orientations():
    for layout in (t360.LAYOUT_FLAT_FIXED, t360.LAYOUT_BARREL, t360.LAYOUT_BARREL_SPLIT):
        with pytest.raises(ValueError):
            t360.oriented_samples(t360.make_context(output_layout=layout), (0, 0, 0), 64, 32, 16, 16)
    for bad in [(math.nan, 0, 0), (0, math.inf, 0), (0, 0, -math.inf)]:
        with pytest.raises(ValueError):
            t360.oriented_samples(t360.make_context(), bad, 64, 32, 16, 16)


def test_oriented_frames_are_refused_before_any_device_work(capfd):
    """FLAT_FIXED, BARREL and BARREL_SPLIT transforms, non-finite orientations, plan indices that were never generated and
    invalid planes are refused (return 0) before the call touches CUDA, so this needs no device."""
    dummy = [(1 << 20, 512)] * 3
    dims = [(512, 256, 192, 128), (256, 128, 96, 64), (256, 128, 96, 64)]
    for layout in (t360.LAYOUT_FLAT_FIXED, t360.LAYOUT_BARREL, t360.LAYOUT_BARREL_SPLIT):
        vft = t360.VideoFrameTransform(t360.make_context(output_layout=layout, enable_low_pass_filter=0))
        _refused_for(capfd, "per-frame orientations need", vft.make_oriented_frame_call(dummy, dummy, dims), (10.0, 0.0, 0.0))
        vft.close()
    cube = t360.VideoFrameTransform(t360.make_context())
    call = cube.make_oriented_frame_call(dummy, dummy, dims)
    _refused_for(capfd, "is not finite", call, (math.nan, 0.0, 0.0))
    _refused_for(capfd, "is not finite", call, (0.0, math.inf, 0.0))
    _refused_for(capfd, "is not finite", call, (0.0, 0.0, -math.inf))
    _refused_for(capfd, "no map was generated for index 0", call, (10.0, 0.0, 5.0))
    _bad_planes_are_refused(capfd, cube.make_oriented_frame_call, ((10.0, 0.0, 5.0),), dummy, dims)
    cube.close()


# ---- on the GPU ---------------------------------------------------------------------------------------------------------
def _with_orientation(ov, o):
    return dict(ov, fixed_yaw=o[0], fixed_pitch=o[1], fixed_roll=o[2])


def _fresh(torch, ov, o, spec, d_in):
    """What a fresh transform made for the context with orientation `o` gives (whole-frame entry point)."""
    ft = FrameTransformer(t360.make_context(**_with_orientation(ov, o)), spec)
    out = _outputs(torch, spec, 1)
    torch.cuda.synchronize()
    assert ft.frame_call(_planes(d_in), _planes(out[0]))(0)
    torch.cuda.synchronize()
    ft.close()
    return _host(spec, out)[0]


def _oracle(ov, o, spec, src):
    octx = rh.default_context(**_with_orientation(ov, o))
    plans, row = {}, []
    for p in range(3):
        iw, ih, ow, oh, idx = spec.plane_dims(p)
        if idx not in plans:
            plans[idx] = co.OraclePlan(octx, iw, ih, ow, oh)
        row.append(co.transform_plane(octx, plans[idx], src[p], ow, oh, map_index=idx))
    return row


def _jitter(seed, n):
    """Stabilisation-like: a slow pan with a few degrees of per-frame shake on every axis."""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    yaw = 20.0 + 0.5 * t + rng.uniform(-3, 3, n)
    pitch = -5.0 + rng.uniform(-3, 3, n)
    roll = rng.uniform(-4, 4, n)
    return [tuple(float(np.float32(v)) for v in row) for row in zip(yaw, pitch, roll)]


def _sweep(seed, n):
    """Yaw sweeps 720 degrees, pitch crosses a pole (|pitch| > 90 on the way), roll turns."""
    rng = np.random.default_rng(seed)
    t = np.linspace(0.0, 1.0, n)
    yaw = -360.0 + 720.0 * t + rng.uniform(-2, 2, n)
    pitch = 110.0 * np.sin(2 * np.pi * t) + rng.uniform(-2, 2, n)
    roll = 90.0 * np.sin(4 * np.pi * t) + rng.uniform(-2, 2, n)
    return [tuple(float(np.float32(v)) for v in row) for row in zip(yaw, pitch, roll)]


def _trajectory(name, n):
    seed = zlib.crc32(name.encode())
    half = n // 2
    return _jitter(seed, half) + _sweep(seed + 1, n - half)


CUBE, EAC, EQUI = t360.LAYOUT_CUBEMAP_32, t360.LAYOUT_EAC_32, t360.LAYOUT_EQUIRECT
LOW_PASS = dict(enable_low_pass_filter=1, num_horizontal_segments=32, num_vertical_segments=15, adjust_kernel=1)
CONFIGS = {  # name: (context, luma in, luma out, orientations, oracle frames)
    "cfg2": (dict(interpolation_alg=t360.CUBIC, enable_low_pass_filter=0), (7680, 3840), (3840, 2560), 8, 1),
    "cfg2_low_pass": (dict(interpolation_alg=t360.CUBIC, **LOW_PASS), (7680, 3840), (3840, 2560), 6, 1),
    "eac_lanczos4_low_pass": (dict(output_layout=EAC, interpolation_alg=t360.LANCZOS4, enable_low_pass_filter=1,
                                   num_horizontal_segments=8, num_vertical_segments=9), (1920, 960), (960, 640), 16, 2),
    "offcenter_z": (dict(output_layout=t360.LAYOUT_CUBEMAP_23_OFFCENTER, interpolation_alg=t360.CUBIC, enable_low_pass_filter=0,
                         fixed_cube_offcenter_z=-0.7), (1920, 960), (640, 960), 16, 2),
    "equirect_to_equirect": (dict(output_layout=EQUI, interpolation_alg=t360.CUBIC), (1920, 960), (961, 481), 16, 2),
    "cube_input_to_equirect": (dict(input_layout=CUBE, output_layout=EQUI, interpolation_alg=t360.CUBIC, enable_low_pass_filter=0),
                               (1536, 1024), (960, 480), 16, 2),
    "nearest": (dict(interpolation_alg=t360.NEAREST, enable_low_pass_filter=0), (961, 481), (483, 321), 16, 2),
    "linear_low_pass": (dict(interpolation_alg=t360.LINEAR), (960, 480), (480, 320), 16, 2),
    "tb_stereo_vflip": (dict(interpolation_alg=t360.CUBIC, input_stereo_format=t360.STEREO_FORMAT_TB,
                             output_stereo_format=t360.STEREO_FORMAT_TB, vflip=1), (960, 960), (480, 640), 16, 2),
    "scale_half": (dict(output_layout=EAC, interpolation_alg=t360.CUBIC, width_scale_factor=0.5, height_scale_factor=0.5),
                   (960, 480), (480, 320), 12, 2),
    "scale_two": (dict(interpolation_alg=t360.CUBIC, width_scale_factor=2.0, height_scale_factor=2.0), (960, 480), (480, 320), 12, 2),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_oriented_frames_equal_fresh_transforms(name, torch_cuda):
    """A seeded trajectory (a shaky pan, then a 720-degree yaw sweep over a pole) enqueued back to back on a non-default
    stream without synchronisation: every frame equals a fresh transform made for its orientation, and the plain-C oracle
    on a subset."""
    torch = torch_cuda
    ov, inp, out, n, n_oracle = CONFIGS[name]
    spec = StreamSpec(*inp, *out)
    orientations = _trajectory(name, n)
    srcs, d_in = _inputs(torch, spec, 2)
    d_out = _outputs(torch, spec, n)
    ft = FrameTransformer(t360.make_context(**ov), spec)
    calls = [ft.oriented_frame_call(_planes(d_in[f % 2]), _planes(d_out[f])) for f in range(n)]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for f, o in enumerate(orientations):
        assert calls[f](o, st.cuda_stream), f"frame {f} orientation {o} refused"
    st.synchronize()
    got = _host(spec, d_out)
    ft.close()
    for f, o in enumerate(orientations):
        _assert_planes(got[f], _fresh(torch, ov, o, spec, d_in[f % 2]), f"{name} frame {f} orientation {o}")
    for f in np.linspace(0, n - 1, n_oracle).astype(int):
        _assert_planes(got[f], _oracle(ov, orientations[f], spec, srcs[f % 2]), f"{name} frame {f} orientation {orientations[f]}, oracle")


@pytest.mark.gpu
def test_two_streams_and_a_reconfigure_in_flight(torch_cuda):
    """Oriented frames on two streams, a reconfigure (output layout, interpolation, low-pass bands) in the middle: every
    frame has the configuration in effect when it was enqueued, with its own orientation."""
    torch = torch_cuda
    a = dict(interpolation_alg=t360.CUBIC, num_vertical_segments=7, num_horizontal_segments=3)
    b = dict(a, output_layout=EAC, interpolation_alg=t360.LANCZOS4, num_vertical_segments=11)
    spec = StreamSpec(960, 480, 480, 320)
    orientations = _trajectory("two_streams", 12)
    _, d_in = _inputs(torch, spec, 2)
    d_out = _outputs(torch, spec, 12)
    ft = FrameTransformer(t360.make_context(**a), spec)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for f, o in enumerate(orientations):
        if f == 6:
            ft.vft.reconfigure(t360.make_context(**b))
        assert ft.oriented_frame_call(_planes(d_in[f % 2]), _planes(d_out[f]))(o, streams[f % 2].cuda_stream)
    for s in streams:
        s.synchronize()
    got = _host(spec, d_out)
    ft.close()
    for f, o in enumerate(orientations):
        _assert_planes(got[f], _fresh(torch, a if f < 6 else b, o, spec, d_in[f % 2]), f"frame {f} orientation {o}")


@pytest.mark.gpu
def test_device_memory_and_launches_stay_bounded(torch_cuda):
    """1000 distinct orientations: device memory does not grow, and without low-pass a frame is one kernel launch (the
    gather of all three planes)."""
    torch = torch_cuda
    spec = StreamSpec(1920, 960, 960, 640)
    _, d_in = _inputs(torch, spec, 1)
    d_out = _outputs(torch, spec, 1)
    orientations = _trajectory("bounded", 1000)
    st = torch.cuda.Stream()
    for ov in (dict(enable_low_pass_filter=0), dict(output_layout=EAC, num_vertical_segments=9, num_horizontal_segments=4)):
        ft = FrameTransformer(t360.make_context(**ov), spec)
        call = ft.oriented_frame_call(_planes(d_in[0]), _planes(d_out[0]))
        torch.cuda.synchronize()
        for o in orientations[:50]:  # first use of every scratch plane and ring entry
            assert call(o, st.cuda_stream)
        st.synchronize()
        free_before = torch.cuda.mem_get_info()[0]
        n0 = t360.kernel_launch_count()
        for o in orientations:
            assert call(o, st.cuda_stream)
        launches = t360.kernel_launch_count() - n0
        st.synchronize()
        free_after = torch.cuda.mem_get_info()[0]
        ft.close()
        assert free_before - free_after <= 4 << 20, f"{(free_before - free_after) >> 20} MB of device memory not released ({ov})"
        if not ov.get("enable_low_pass_filter", 1):
            assert launches == len(orientations), f"{launches} launches for {len(orientations)} frames"
        else:
            assert launches <= 4 * len(orientations), f"{launches} launches for {len(orientations)} frames"


@pytest.mark.gpu
def test_input_planes_of_another_size_are_refused(torch_cuda):
    torch = torch_cuda
    spec = StreamSpec(960, 480, 480, 320)
    _, d_in = _inputs(torch, spec, 1)
    d_out = _outputs(torch, spec, 1)
    ft = FrameTransformer(t360.make_context(enable_low_pass_filter=0), spec)
    dims = [spec.plane_dims(p)[:4] for p in range(3)]
    dims[0] = (dims[0][0] - 2, dims[0][1], dims[0][2], dims[0][3])
    assert not ft.vft.make_oriented_frame_call(_planes(d_in[0]), _planes(d_out[0]), dims)((1.0, 2.0, 3.0))
    assert ft.oriented_frame_call(_planes(d_in[0]), _planes(d_out[0]))((1.0, 2.0, 3.0), 0)
    torch.cuda.synchronize()
    ft.close()
