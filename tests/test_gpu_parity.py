"""GPU parity: the CUDA path, called through the drop-in C-ABI, against the oracle.

Bars (task spec / BASELINE.json north_star):
  * gather (cv::remap replacement): integer arithmetic -> BIT-EXACT for all four interpolators;
  * segmented low-pass (cv::sepFilter2D replacement): float32 -> tolerance 1 LSB per north_star, but the
    kernel follows the oracle's operation order, so these tests also demand bit-exactness;
  * end to end vs the recorded outputs of the reference itself (tests/golden/golden.json).
Nothing here reads the reference sources.
"""
import numpy as np
import pytest

import transform360_b200 as t360
from oracle import c_oracle as co
from oracle import ref_harness as rh
from tests.golden.cases import FULL, SMALL, plane_dims

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests must run on an H100 (there is no CPU fallback to test)")
    assert t360.device_count() >= 1
    return torch


def _ctxs(case):
    return t360.make_context(**case["ov"]), rh.default_context(**case["ov"])


def _prefill(ctx):
    return 7 if ctx.output_layout in (t360.LAYOUT_BARREL, t360.LAYOUT_BARREL_SPLIT) else 0


@pytest.mark.parametrize("name", sorted(SMALL))
def test_small_cases_bit_exact_through_c_abi(name, golden, torch_cuda):
    case = SMALL[name]
    ctx, octx = _ctxs(case)
    launches0 = t360.kernel_launch_count()
    with t360.VideoFrameTransform(ctx) as vft:
        for idx in (0, 1):
            iw, ih, ow, oh, _ = plane_dims(case, idx)
            assert vft.generateMapForPlane(iw, ih, ow, oh, idx)
        for plane in (0, 1, 2):
            iw, ih, ow, oh, idx = plane_dims(case, plane)
            src = co.noise_plane(iw, ih, plane=plane, frame=0)
            out = np.full((oh, ow), _prefill(ctx), np.uint8)
            vft.transform_plane(src, ow, oh, idx, image_plane=plane, out=out)
            plan = co.OraclePlan(octx, iw, ih, ow, oh)
            want = co.transform_plane(octx, plan, src, ow, oh, map_index=idx, prefill=_prefill(ctx))
            bad = int((out != want).sum())
            assert bad == 0, f"{name} plane {plane}: {bad} px differ from the oracle (max |d| {np.abs(out.astype(int) - want).max()})"
            if plane < 2:
                g = golden["small"][name]["planes"][str(plane)]
                assert rh.sha16(out) == g["out_sha"], f"{name} plane {plane}: differs from the reference's recorded output"
    assert t360.kernel_launch_count() > launches0, "no kernel of this library was launched"


def test_host_pitch_and_padding_untouched(torch_cuda):
    """linesize > width on both sides (ffmpeg planes): only `width` bytes per row are read / written."""
    case = SMALL["lp_tiles"]
    ctx, octx = _ctxs(case)
    iw, ih, ow, oh, idx = plane_dims(case, 0)
    src = co.noise_plane(iw, ih, plane=0, frame=2, pitch=iw + 37)
    src[:, iw:] = 0xAB
    out = np.full((oh, ow + 19), 0xCD, np.uint8)
    with t360.VideoFrameTransform(ctx) as vft:
        assert vft.generateMapForPlane(iw, ih, ow, oh, 0)
        assert vft.transformFramePlane(src.ctypes.data, out.ctypes.data, iw, ih, src.strides[0], ow, oh, out.strides[0], 0, 0)
    plan = co.OraclePlan(octx, iw, ih, ow, oh)
    want = co.transform_plane(octx, plan, np.ascontiguousarray(src[:, :iw]), ow, oh)
    assert np.array_equal(out[:, :ow], want)
    assert (out[:, ow:] == 0xCD).all()


@pytest.mark.parametrize("name", ["cube_cubic_odd", "eac_tb_lanczos", "lp_tiles", "cube_linear", "cube_nearest"])
def test_device_pointer_path_with_unaligned_pitch(name, torch_cuda):
    """Zero-copy path: device planes with a pitch and base address that are not multiples of 4."""
    torch = torch_cuda
    case = SMALL[name]
    ctx, octx = _ctxs(case)
    iw, ih, ow, oh, idx = plane_dims(case, 0)
    src = co.noise_plane(iw, ih, plane=0, frame=5)
    in_pitch, out_pitch = iw + 13, ow + 7
    d_in = torch.zeros(in_pitch * ih + 64, dtype=torch.uint8, device="cuda")
    d_out = torch.full((out_pitch * oh + 64,), 0xEE, dtype=torch.uint8, device="cuda")
    off_in, off_out = 3, 1
    view = d_in[off_in:off_in + in_pitch * ih].view(ih, in_pitch)
    view[:, :iw] = torch.from_numpy(src).cuda()
    with t360.VideoFrameTransform(ctx) as vft:
        assert vft.generateMapForPlane(iw, ih, ow, oh, 0)
        # synchronous ABI call with device pointers
        assert vft.transformFramePlane(d_in.data_ptr() + off_in, d_out.data_ptr() + off_out, iw, ih, in_pitch, ow, oh, out_pitch, 0, 0)
        got = d_out[off_out:off_out + out_pitch * oh].view(oh, out_pitch).cpu().numpy()
        # asynchronous extension on the transform's stream
        d_out2 = torch.full_like(d_out, 0xEE)
        torch.cuda.synchronize()
        assert vft.transform_plane_async(d_in.data_ptr() + off_in, d_out2.data_ptr() + off_out, iw, ih, in_pitch, ow, oh, out_pitch, 0)
        assert vft.synchronize()
        got2 = d_out2[off_out:off_out + out_pitch * oh].view(oh, out_pitch).cpu().numpy()
    plan = co.OraclePlan(octx, iw, ih, ow, oh)
    want = co.transform_plane(octx, plan, src, ow, oh)
    assert np.array_equal(got[:, :ow], want)
    assert (got[:, ow:] == 0xEE).all()
    assert np.array_equal(got2, got)


EXTRA_LP = {
    # vertical sigma 0.25 -> a single vertical tap (hy = 0), horizontal kernels of every size up to the pole
    "lp_single_vertical_tap": dict(ov=dict(min_kernel_half_height=0.5, num_vertical_segments=9, num_horizontal_segments=1),
                                   inp=(328, 164), out=(480, 320)),
    # odd plane width, tiles narrower than a strip, kernels differing per tile (off-centre): unaligned byte stores
    "lp_odd_offcentre": dict(ov=dict(fixed_cube_offcenter_z=-0.25, num_vertical_segments=7, num_horizontal_segments=5),
                             inp=(1003, 501), out=(384, 256)),
    # wide plane: interior strips (aligned word loads) and edge strips (clamped loads) in the same launch
    "lp_wide": dict(ov=dict(num_vertical_segments=15, num_horizontal_segments=32), inp=(3840, 480), out=(1536, 256)),
}


@pytest.mark.parametrize("name", ["lp_default", "lp_tiles", "lp_even_segments", "lp_big_kernels", "lr_stereo", "eac_tb_lanczos",
                                  "offcenter_adjust"] + sorted(EXTRA_LP))
def test_low_pass_stage_alone(name, torch_cuda):
    torch = torch_cuda
    case = SMALL.get(name) or EXTRA_LP[name]
    ctx, octx = _ctxs(case)
    iw, ih, ow, oh, idx = plane_dims(case, 0)
    src = co.noise_plane(iw, ih, plane=0, frame=9)
    d_in = torch.from_numpy(src).cuda()
    d_out = torch.full((ih, iw), 0x55, dtype=torch.uint8, device="cuda")
    with t360.VideoFrameTransform(ctx) as vft:
        assert vft.generateMapForPlane(iw, ih, ow, oh, 0)
        assert vft.low_pass_async(d_in.data_ptr(), d_out.data_ptr(), iw, ih, iw, iw, 0)
        assert vft.synchronize()
    plan = co.OraclePlan(octx, iw, ih, ow, oh)
    want = co.filter_plane(octx, src, plan.segs, plan.nsegs, plan.taps)
    got = d_out.cpu().numpy()
    d = np.abs(got.astype(int) - want.astype(int))
    assert d.max() <= 1, "north_star tolerance: 1 LSB"
    assert int((d != 0).sum()) == 0, "kernel follows the oracle's FMA order: expected bit-exact"


def test_huge_kernels_take_the_direct_path(torch_cuda):
    """sigma can reach half the plane width (reference cpp:219); tiles that do not fit shared memory still match."""
    ov = dict(interpolation_alg=t360.CUBIC, num_vertical_segments=300, num_horizontal_segments=1, adjust_kernel=0,
              min_kernel_half_height=40.0)
    ctx, octx = t360.make_context(**ov), rh.default_context(**ov)
    iw, ih, ow, oh = 640, 320, 96, 64
    src = co.noise_plane(iw, ih, frame=4)
    with t360.VideoFrameTransform(ctx) as vft:
        assert vft.generateMapForPlane(iw, ih, ow, oh, 0)
        got = vft.transform_plane(src, ow, oh, 0)
    plan = co.OraclePlan(octx, iw, ih, ow, oh)
    want = co.transform_plane(octx, plan, src, ow, oh)
    assert np.array_equal(got, want)


def test_recurring_pageable_planes_can_be_pinned_in_place(torch_cuda):
    """Opt-in cudaHostRegister of recycled caller buffers: same bytes before and after the buffer gets page-locked."""
    case = SMALL["lp_tiles"]
    ctx, octx = _ctxs(case)
    iw, ih, ow, oh, idx = plane_dims(case, 0)
    src = np.ascontiguousarray(co.noise_plane(iw, ih, frame=1))
    out = np.zeros((oh, ow), np.uint8)
    plan = co.OraclePlan(octx, iw, ih, ow, oh)
    with t360.VideoFrameTransform(ctx) as vft:
        vft.set_pin_host_planes(True)
        assert vft.generateMapForPlane(iw, ih, ow, oh, 0)
        for frame in range(4):  # the same two buffers every frame, like a frame pool
            src[...] = co.noise_plane(iw, ih, frame=frame)
            vft.transform_plane(src, ow, oh, 0, out=out)
            assert np.array_equal(out, co.transform_plane(octx, plan, src, ow, oh))


def test_errors_follow_the_reference_contract(torch_cuda):
    ctx = t360.make_context(enable_low_pass_filter=0)
    src = np.zeros((32, 64), np.uint8)
    with t360.VideoFrameTransform(ctx) as vft:
        with pytest.raises(RuntimeError):  # never generated: reference fails on the empty map (SURVEY 8b)
            vft.transform_plane(src, 24, 16, 0)
        assert vft.generateMapForPlane(64, 32, 24, 16, 0)
        assert vft.transform_plane(src, 24, 16, 0).shape == (16, 24)
        assert not vft.transformFramePlane(0, 0, 64, 32, 64, 24, 16, 24, 0, 0)  # NULL planes
        assert vft.generateMapForPlane(64, 32, 24, 16, 0)  # re-plan replaces, does not append


@pytest.mark.parametrize("name", ["cfg2", "cfg3", "cfg4"])
def test_full_size_configs_luma(name, golden, torch_cuda):
    """BASELINE.json configs at full size: every output pixel of the luma plane against the oracle and
    against the reference's recorded SHA."""
    case = FULL[name]
    ctx, octx = _ctxs(case)
    iw, ih, ow, oh, idx = plane_dims(case, 0)
    src = co.noise_plane(iw, ih)
    with t360.VideoFrameTransform(ctx) as vft:
        assert vft.generateMapForPlane(iw, ih, ow, oh, 0)
        got = vft.transform_plane(src, ow, oh, 0)
    plan = co.OraclePlan(octx, iw, ih, ow, oh)
    want = co.transform_plane(octx, plan, src, ow, oh)
    d = np.abs(got.astype(np.int16) - want.astype(np.int16))
    assert d.max() <= 1
    assert int((d != 0).sum()) == 0
    assert rh.sha16(got) == golden["full"][name]["planes"]["0"]["out_sha"]


def test_full_size_cfg3_chroma_and_frame_seeds(torch_cuda):
    """cfg3 chroma planes (plan index 1) and a second frame seed; linearity-free property: the same frame
    gives the same bytes on repeated calls (no state leaks between frames, SURVEY 8e)."""
    case = FULL["cfg3"]
    ctx, octx = _ctxs(case)
    iw, ih, ow, oh, idx = plane_dims(case, 1)
    with t360.VideoFrameTransform(ctx) as vft:
        assert vft.generateMapForPlane(iw, ih, ow, oh, 1)
        plan = co.OraclePlan(octx, iw, ih, ow, oh)
        outs = []
        for plane, frame in ((1, 0), (2, 0), (1, 599), (1, 0)):
            src = co.noise_plane(iw, ih, plane=plane, frame=frame)
            got = vft.transform_plane(src, ow, oh, 1, image_plane=plane)
            assert np.array_equal(got, co.transform_plane(octx, plan, src, ow, oh, map_index=1))
            outs.append(got)
        assert np.array_equal(outs[0], outs[3])


@pytest.mark.parametrize("name", ["lp_tiles", "cube_cubic_odd", "eac_tb_lanczos"])
def test_whole_frame_entry_point_matches_per_plane_calls(name, torch_cuda):
    """T360B200_transformFrameAsync (planes concurrently on internal lanes) == three reference-ABI calls."""
    torch = torch_cuda
    from transform360_b200.stream import FrameTransformer, StreamSpec
    case = SMALL[name]
    ctx, _ = _ctxs(case)
    spec = StreamSpec(case["inp"][0], case["inp"][1], case["out"][0], case["out"][1])
    ft = FrameTransformer(ctx, spec)
    srcs = [co.noise_plane(*spec.plane_dims(p)[:2], plane=p, frame=3) for p in range(3)]
    want = [ft.vft.transform_plane(srcs[p], spec.plane_dims(p)[2], spec.plane_dims(p)[3], spec.plane_dims(p)[4], image_plane=p)
            for p in range(3)]
    d_in = [torch.from_numpy(a).cuda() for a in srcs]
    d_out = [torch.zeros((spec.plane_dims(p)[3], spec.plane_dims(p)[2]), dtype=torch.uint8, device="cuda") for p in range(3)]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for _ in range(3):  # repeated frames reuse the lanes' scratch buffers and events
        ft.transform_frame_device([(t.data_ptr(), t.stride(0)) for t in d_in], [(t.data_ptr(), t.stride(0)) for t in d_out],
                                  st.cuda_stream)
    st.synchronize()
    for p in range(3):
        assert np.array_equal(d_out[p].cpu().numpy(), want[p]), f"plane {p}"
    ft.close()


def _pitched(torch, arr, pitch):
    """Device copy of a 2-D uint8 array with the given row pitch (bytes); returns (base tensor, view)."""
    h, w = arr.shape
    base = torch.zeros((h, pitch), dtype=torch.uint8, device="cuda")
    base[:, :w] = torch.from_numpy(np.ascontiguousarray(arr)).cuda()
    return base


def test_debug_trace_has_a_row_per_consumer_group_of_the_device(torch_cuda):
    """The frame gather's debug trace is sized by the library from the device's SM count (one CTA per SM, three consumer
    groups per CTA for bicubic); the binding reads all of it, and the traced jobs have ordered timestamps."""
    torch = torch_cuda
    from transform360_b200.stream import FrameTransformer, StreamSpec
    case = SMALL["cube_cubic"]
    ctx, _ = _ctxs(case)
    spec = StreamSpec(case["inp"][0], case["inp"][1], case["out"][0], case["out"][1])
    ft = FrameTransformer(ctx, spec)
    pitch = lambda w: (w + 255) // 256 * 256
    d_in = [_pitched(torch, co.noise_plane(*spec.plane_dims(p)[:2], plane=p, frame=2), pitch(spec.plane_dims(p)[0])) for p in range(3)]
    d_out = [torch.zeros((spec.plane_dims(p)[3], pitch(spec.plane_dims(p)[2])), dtype=torch.uint8, device="cuda") for p in range(3)]
    torch.cuda.synchronize()
    ft.vft.debug_trace(True)
    ft.transform_frame_device([(t.data_ptr(), t.stride(0)) for t in d_in], [(t.data_ptr(), t.stride(0)) for t in d_out], 0)
    torch.cuda.synchronize()
    tr = ft.vft.read_trace().astype(np.int64)
    ft.vft.debug_trace(False)
    ft.close()
    assert tr.shape == (torch.cuda.get_device_properties(0).multi_processor_count * 3, 64, 4)
    used = tr[..., 2] > 0
    assert used.any()
    assert (tr[..., 1][used] >= tr[..., 0][used]).all() and (tr[..., 2][used] >= tr[..., 1][used]).all()


@pytest.mark.parametrize("name,planes", [("cube_cubic", 3), ("cube_linear", 3), ("cube_lanczos", 3), ("cube_cubic", 2), ("cube_cubic", 1),
                                         ("rotated", 3), ("cube_to_equirect", 3), ("scaled_2x2", 3), ("scaled_fractional_lp", 3),
                                         ("barrel", 3), ("cube_nearest", 3), ("lr_stereo", 3)])
def test_frame_entry_point_every_path(name, planes, torch_cuda):
    """The whole-frame entry point against the oracle, plane by plane, with TMA-describable planes (256-byte pitch):
    staged plans gather all planes in ONE launch; barrel / nearest plans take the per-plane general kernels; scaled
    plans resize after the shared gather.  Frames are enqueued back to back (programmatic dependent launch, self
    re-arming tile scheduler) into distinct outputs and every one of them is checked."""
    torch = torch_cuda
    from transform360_b200.stream import FrameTransformer, StreamSpec
    case = SMALL[name]
    ctx, octx = _ctxs(case)
    spec = StreamSpec(case["inp"][0], case["inp"][1], case["out"][0], case["out"][1])
    ft = FrameTransformer(ctx, spec)
    frames = 6
    pitch = lambda w: (w + 255) // 256 * 256
    fill = _prefill(ctx)
    plans = {}
    d_in, d_out, want = [], [], []
    for f in range(frames):
        ins, outs, exp = [], [], []
        for p in range(planes):
            iw, ih, ow, oh, idx = spec.plane_dims(p)
            if idx not in plans:
                plans[idx] = co.OraclePlan(octx, iw, ih, ow, oh)
            src = co.noise_plane(iw, ih, plane=p, frame=f)
            ins.append(_pitched(torch, src, pitch(iw)))
            outs.append(torch.full((oh, pitch(ow)), fill, dtype=torch.uint8, device="cuda"))
            exp.append(co.transform_plane(octx, plans[idx], src, ow, oh, map_index=idx, prefill=fill))
        d_in.append(ins); d_out.append(outs); want.append(exp)
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    n0 = t360.kernel_launch_count()
    dims = [spec.plane_dims(p)[:4] for p in range(planes)]
    for f in range(frames):
        call = ft.vft.make_frame_call([(t.data_ptr(), t.stride(0)) for t in d_in[f]], [(t.data_ptr(), t.stride(0)) for t in d_out[f]], dims)
        assert call(st.cuda_stream), "T360B200_transformFrameAsync failed"
    st.synchronize()
    launches = (t360.kernel_launch_count() - n0) / frames
    staged = ctx.interpolation_alg != t360.NEAREST and not fill and not ctx.enable_low_pass_filter \
        and ctx.width_scale_factor == 1 and ctx.height_scale_factor == 1
    staged = staged and all(ft.vft.plan_tile_counts(i)[0] > 0 for i in ((0, 1) if planes > 1 else (0,)))
    if staged and planes > 1:
        assert launches == 1, f"{launches} launches per frame: the planes were not gathered in one launch"
    for f in range(frames):
        for p in range(planes):
            ow = spec.plane_dims(p)[2]
            got = d_out[f][p][:, :ow].cpu().numpy()
            assert np.array_equal(got, want[f][p]), f"frame {f} plane {p}: {(got != want[f][p]).sum()} px differ"
            if d_out[f][p].shape[1] > ow:
                pad = d_out[f][p][:, ow:]
                assert int(pad.min().item()) == fill and int(pad.max().item()) == fill, "row padding was written"
    ft.close()


def test_frame_entry_point_survives_map_regeneration(torch_cuda):
    """generateMapForPlane again (other parameters) between frames: the merged job list is rebuilt."""
    torch = torch_cuda
    from transform360_b200.stream import FrameTransformer, StreamSpec
    case = SMALL["cube_cubic"]
    spec = StreamSpec(case["inp"][0], case["inp"][1], case["out"][0], case["out"][1])
    ctx, octx = _ctxs(case)
    ft = FrameTransformer(ctx, spec)
    pitch = lambda w: (w + 255) // 256 * 256
    srcs = [co.noise_plane(*spec.plane_dims(p)[:2], plane=p, frame=11) for p in range(3)]
    d_in = [_pitched(torch, srcs[p], pitch(spec.plane_dims(p)[0])) for p in range(3)]
    st = torch.cuda.Stream()
    for out_size in (case["out"], (96, 64), case["out"]):
        spec2 = StreamSpec(case["inp"][0], case["inp"][1], out_size[0], out_size[1])
        for idx in (0, 1):
            iw, ih, ow, oh, _ = spec2.plane_dims(idx)
            assert ft.vft.generateMapForPlane(iw, ih, ow, oh, idx)
        d_out = [torch.zeros((spec2.plane_dims(p)[3], pitch(spec2.plane_dims(p)[2])), dtype=torch.uint8, device="cuda") for p in range(3)]
        dims = [spec2.plane_dims(p)[:4] for p in range(3)]
        call = ft.vft.make_frame_call([(t.data_ptr(), t.stride(0)) for t in d_in], [(t.data_ptr(), t.stride(0)) for t in d_out], dims)
        for _ in range(2):
            assert call(st.cuda_stream)
        st.synchronize()
        for p in range(3):
            iw, ih, ow, oh, idx = spec2.plane_dims(p)
            exp = co.transform_plane(octx, co.OraclePlan(octx, iw, ih, ow, oh), srcs[p], ow, oh, map_index=idx)
            assert np.array_equal(d_out[p][:, :ow].cpu().numpy(), exp), f"out {out_size} plane {p}"
    ft.close()


def test_nan_map_entries_sample_like_opencv(torch_cuda):
    """Off-centre + is_horizontal_offset divides by zero at the poles (ref:1203-1206): the map holds NaN for a few
    pixels, which cv::remap rounds to INT_MIN and saturates to column / row -32768 under BORDER_WRAP.  Parameters
    found by the random sweep against the compiled reference (tests/test_host_plan.py)."""
    ov = dict(input_layout=3, output_layout=6, input_stereo_format=1, output_stereo_format=1, input_expand_coef=1.03,
              expand_coef=1.01, interpolation_alg=2, fixed_yaw=-164.79200291974115, fixed_pitch=13.155720951654928,
              fixed_roll=-42.12975619832986, fixed_cube_offcenter_x=0.2557402424642103, fixed_cube_offcenter_y=-0.15772665724832016,
              fixed_cube_offcenter_z=-0.41284091691208313, is_horizontal_offset=1, enable_low_pass_filter=0)
    iw, ih, ow, oh = 194, 240, 198, 142
    for interp in (t360.NEAREST, t360.LINEAR, t360.CUBIC, t360.LANCZOS4):
        ov["interpolation_alg"] = interp
        ctx, octx = t360.make_context(**ov), rh.default_context(**ov)
        plan = co.OraclePlan(octx, iw, ih, ow, oh)
        assert np.isnan(plan.map).any(), "this case is here for its NaN map entries"
        src = co.noise_plane(iw, ih, plane=0, frame=3)
        want = co.transform_plane(octx, plan, src, ow, oh, map_index=0)
        with t360.VideoFrameTransform(ctx) as vft:
            assert vft.generateMapForPlane(iw, ih, ow, oh, 0)
            got = vft.transform_plane(src, ow, oh, 0)
        assert np.array_equal(got, want), f"interp {interp}: {(got != want).sum()} px differ"


def _rank_worker(rank, world, port, q):
    import os
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from transform360_b200.stream import FrameTransformer, StreamSpec, broadcast_parameters, frames_for_rank
        ctx = spec = None
        if rank == 0:
            ctx = t360.make_context(interpolation_alg=t360.CUBIC, num_vertical_segments=15, num_horizontal_segments=8)
            spec = StreamSpec(960, 480, 384, 256)
        ctx, spec = broadcast_parameters(ctx, spec, rank, world, device=torch.device("cuda", rank))
        ft = FrameTransformer(ctx, spec)
        out = {}
        for k in list(frames_for_rank(6, rank, world)) + [5 - rank]:  # own frames + one frame of the other rank
            planes = []
            for p in range(3):
                iw, ih, ow, oh, idx = spec.plane_dims(p)
                src = co.noise_plane(iw, ih, plane=p, frame=k)
                planes.append(rh.sha16(ft.vft.transform_plane(src, ow, oh, idx, image_plane=p)))
            out[k] = planes
        q.put((rank, out))
        ft.close()
    finally:
        dist.destroy_process_group()


def test_frame_bytes_do_not_depend_on_the_gpu(torch_cuda):
    """SURVEY.md 4 item 4 / 8e: frame k gives identical planes whichever rank (GPU) processes it."""
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import socket
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctxm = mp.get_context("spawn")
    q = ctxm.Queue()
    procs = [ctxm.Process(target=_rank_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=300) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    shared = set(res[0]) & set(res[1])
    assert shared, "test must compare at least one frame processed on both GPUs"
    for k in shared:
        assert res[0][k] == res[1][k], f"frame {k} differs between GPUs"


# ---- round 2: the paths the bench times, at the sizes it times them -----------------------------------------------
@pytest.mark.parametrize("name", ["cfg2", "cfg3", "cfg4"])
def test_full_size_frames_through_the_frame_entry_point(name, golden, torch_cuda):
    """What bench.py's device-resident leg runs: T360B200_transformFrameAsync on BASELINE configs[1..3] at full size,
    ALL THREE planes, six frames back to back (programmatic dependent launch, self re-arming scheduler); the first and
    the last frame completely, and every luma plane of cfg2, against the oracle; frame 0 luma also against the
    reference's recorded SHA."""
    torch = torch_cuda
    from transform360_b200.stream import FrameTransformer, StreamSpec
    case = FULL[name]
    ctx, octx = _ctxs(case)
    spec = StreamSpec(case["inp"][0], case["inp"][1], case["out"][0], case["out"][1])
    ft = FrameTransformer(ctx, spec)
    pitch = lambda w: (w + 255) // 256 * 256
    frames = 6
    plans = {idx: co.OraclePlan(octx, *spec.plane_dims(p)[:4]) for p, idx in ((0, 0), (1, 1))}
    st = torch.cuda.Stream()
    d_in, d_out, srcs = [], [], []
    for f in range(frames):
        planes = [co.noise_plane(*spec.plane_dims(p)[:2], plane=p, frame=f) for p in range(3)]
        srcs.append(planes)
        d_in.append([_pitched(torch, planes[p], pitch(spec.plane_dims(p)[0])) for p in range(3)])
        d_out.append([torch.zeros((spec.plane_dims(p)[3], pitch(spec.plane_dims(p)[2])), dtype=torch.uint8, device="cuda") for p in range(3)])
    dims = [spec.plane_dims(p)[:4] for p in range(3)]
    torch.cuda.synchronize()
    for f in range(frames):
        call = ft.vft.make_frame_call([(t.data_ptr(), t.stride(0)) for t in d_in[f]], [(t.data_ptr(), t.stride(0)) for t in d_out[f]], dims)
        assert call(st.cuda_stream)
    st.synchronize()
    for f in range(frames):
        for p in range(3):
            iw, ih, ow, oh, idx = spec.plane_dims(p)
            got = d_out[f][p][:, :ow].cpu().numpy()
            if f in (0, frames - 1) or (p == 0 and name == "cfg2"):  # (the oracle takes seconds per 8K plane)
                want = co.transform_plane(octx, plans[idx], srcs[f][p], ow, oh, map_index=idx)
                assert np.array_equal(got, want), f"{name} frame {f} plane {p}: {(got != want).sum()} px differ"
            if f == 0 and p == 0:
                assert rh.sha16(got) == golden["full"][name]["planes"]["0"]["out_sha"]
    ft.close()


def test_random_contexts_product_vs_oracle(torch_cuda):
    """Seeded sweep over the whole option space (all layouts both ways, stereo, rotation, off-centre, scale factors, every
    interpolator, low-pass on and off, odd sizes), small planes, product through the C-ABI against the oracle on the GPU."""
    from tests.test_host_plan import _random_context
    rng = np.random.default_rng(2024)
    checked = refused = 0
    for i in range(220):
        ov = _random_context(rng)
        iw, ih = int(rng.integers(100, 400)) * 2, int(rng.integers(60, 200)) * 2
        ow, oh = int(rng.integers(30, 160)) * 2 + int(rng.random() < 0.3), int(rng.integers(24, 120)) * 2 + int(rng.random() < 0.3)
        plane = int(rng.integers(0, 3))
        idx = 1 if plane else 0
        ctx, octx = t360.make_context(**ov), rh.default_context(**ov)
        try:
            plan = co.OraclePlan(octx, iw, ih, ow, oh)
        except Exception:
            plan = None
        with t360.VideoFrameTransform(ctx) as vft:
            ok = vft.generateMapForPlane(iw, ih, ow, oh, idx)
            if plan is None or not ok:
                assert plan is None and not ok, f"case {i}: product and oracle disagree on whether the plan exists ({ov})"
                refused += 1
                continue
            src = co.noise_plane(iw, ih, plane=plane, frame=i)
            fill = _prefill(ctx)
            out = np.full((oh, ow), fill, np.uint8)
            vft.transform_plane(src, ow, oh, idx, image_plane=plane, out=out)
        want = co.transform_plane(octx, plan, src, ow, oh, map_index=idx, prefill=fill)
        assert np.array_equal(out, want), f"case {i}: {(out != want).sum()} px differ ({ov}, {iw}x{ih} -> {ow}x{oh}, plane {plane})"
        checked += 1
    assert checked >= 200, (checked, refused)


@pytest.mark.parametrize("name", ["cube_cubic", "cube_linear", "cube_lanczos", "rotated", "eac_mono_cubic", "cube_to_equirect", "cube_cubic_odd"])
def test_streamed_host_path_on_small_planes(name, torch_cuda, monkeypatch):
    """Large host planes are streamed through the device in row bands (chunked H2D || gather waves || D2H of finished
    rectangles).  T360B200_PIPELINE_MIN_BYTES=0 sends small planes down that path too: same bytes as the oracle."""
    monkeypatch.setenv("T360B200_PIPELINE_MIN_BYTES", "0")
    case = SMALL[name]
    ctx, octx = _ctxs(case)
    with t360.VideoFrameTransform(ctx) as vft:
        for idx in (0, 1):
            iw, ih, ow, oh, _ = plane_dims(case, idx)
            assert vft.generateMapForPlane(iw, ih, ow, oh, idx)
        for plane in (0, 1, 2):
            iw, ih, ow, oh, idx = plane_dims(case, plane)
            plan = co.OraclePlan(octx, iw, ih, ow, oh)
            for frame in (0, 1):
                src = co.noise_plane(iw, ih, plane=plane, frame=frame, pitch=iw + 5)
                out = np.full((oh, ow + 3), 0x5A, np.uint8)
                assert vft.transformFramePlane(src.ctypes.data, out.ctypes.data, iw, ih, src.strides[0], ow, oh, out.strides[0], idx, plane)
                want = co.transform_plane(octx, plan, np.ascontiguousarray(src[:, :iw]), ow, oh, map_index=idx)
                assert np.array_equal(out[:, :ow], want), f"{name} plane {plane} frame {frame}: {(out[:, :ow] != want).sum()} px differ"
                assert (out[:, ow:] == 0x5A).all()


def test_concurrent_calls_on_different_planes(torch_cuda):
    """The reference object is safe for concurrent transformFramePlane calls on different planes after init
    (VideoFrameTransform.h:150-159: read-only maps); three host threads, one plane each, several frames."""
    import threading
    case = SMALL["lp_tiles"]
    ctx, octx = _ctxs(case)
    with t360.VideoFrameTransform(ctx) as vft:
        for idx in (0, 1):
            iw, ih, ow, oh, _ = plane_dims(case, idx)
            assert vft.generateMapForPlane(iw, ih, ow, oh, idx)
        results, errors = {}, []

        def work(plane):
            try:
                iw, ih, ow, oh, idx = plane_dims(case, plane)
                for frame in range(6):
                    src = co.noise_plane(iw, ih, plane=plane, frame=frame)
                    results[(plane, frame)] = (src, vft.transform_plane(src, ow, oh, idx, image_plane=plane))
            except Exception as e:  # noqa: BLE001
                errors.append(repr(e))
        threads = [threading.Thread(target=work, args=(p,)) for p in range(3)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors
    for (plane, frame), (src, got) in results.items():
        iw, ih, ow, oh, idx = plane_dims(case, plane)
        want = co.transform_plane(octx, co.OraclePlan(octx, iw, ih, ow, oh), src, ow, oh, map_index=idx)
        assert np.array_equal(got, want), f"plane {plane} frame {frame}"


@pytest.mark.parametrize("name,out2,in2", [("cube_cubic", (150, 90), None), ("cube_linear", (250, 200), None), ("lp_tiles", (240, 160), (900, 440)),
                                           ("lp_default", (200, 100), (600, 300)), ("scaled_2x2", (96, 64), (480, 250))])
def test_sizes_that_differ_from_the_generated_map(name, out2, in2, torch_cuda):
    """The reference decides per call (cpp:735-737): an output size other than the map's takes the render + cv::resize
    (INTER_AREA, shrinking or enlarging) branch; an input plane of another size is sampled with BORDER_WRAP against ITS
    size, and its low-pass applies the planned segments that still fit (cpp:173-204)."""
    case = SMALL[name]
    ctx, octx = _ctxs(case)
    iw, ih, ow, oh, _ = plane_dims(case, 0)
    iw2, ih2 = in2 or (iw, ih)
    src = co.noise_plane(iw2, ih2, plane=0, frame=4)
    with t360.VideoFrameTransform(ctx) as vft:
        assert vft.generateMapForPlane(iw, ih, ow, oh, 0)
        got = vft.transform_plane(src, out2[0], out2[1], 0)
        again = vft.transform_plane(src, out2[0], out2[1], 0)
    plan = co.OraclePlan(octx, iw, ih, ow, oh)
    want = co.transform_plane(octx, plan, src, out2[0], out2[1])
    assert np.array_equal(got, want), f"{(got != want).sum()} px differ"
    assert np.array_equal(again, got)


def test_async_entry_points_on_several_streams(torch_cuda):
    """Per-plane and whole-frame asynchronous calls interleaved on three streams (scratch planes and job schedulers are
    kept per stream): every output still matches the oracle."""
    torch = torch_cuda
    from transform360_b200.stream import FrameTransformer, StreamSpec
    case = SMALL["lp_tiles"]
    ctx, octx = _ctxs(case)
    spec = StreamSpec(case["inp"][0], case["inp"][1], case["out"][0], case["out"][1])
    ft = FrameTransformer(ctx, spec)
    pitch = lambda w: (w + 255) // 256 * 256
    plans = {idx: co.OraclePlan(octx, *spec.plane_dims(p)[:4]) for p, idx in ((0, 0), (1, 1))}
    streams = [torch.cuda.Stream() for _ in range(3)]
    dims = [spec.plane_dims(p)[:4] for p in range(3)]
    work = []
    for f in range(9):
        srcs = [co.noise_plane(*spec.plane_dims(p)[:2], plane=p, frame=f) for p in range(3)]
        d_in = [_pitched(torch, srcs[p], pitch(spec.plane_dims(p)[0])) for p in range(3)]
        d_out = [torch.zeros((spec.plane_dims(p)[3], pitch(spec.plane_dims(p)[2])), dtype=torch.uint8, device="cuda") for p in range(3)]
        work.append((srcs, d_in, d_out))
    torch.cuda.synchronize()
    for f, (srcs, d_in, d_out) in enumerate(work):
        st = streams[f % 3].cuda_stream
        if f % 2:
            call = ft.vft.make_frame_call([(t.data_ptr(), t.stride(0)) for t in d_in], [(t.data_ptr(), t.stride(0)) for t in d_out], dims)
            assert call(st)
        else:
            for p in range(3):
                iw, ih, ow, oh, idx = spec.plane_dims(p)
                assert ft.vft.transform_plane_async(d_in[p].data_ptr(), d_out[p].data_ptr(), iw, ih, d_in[p].stride(0), ow, oh, d_out[p].stride(0), idx, st)
    torch.cuda.synchronize()
    for f, (srcs, d_in, d_out) in enumerate(work):
        for p in range(3):
            iw, ih, ow, oh, idx = spec.plane_dims(p)
            want = co.transform_plane(octx, plans[idx], srcs[p], ow, oh, map_index=idx)
            assert np.array_equal(d_out[p][:, :ow].cpu().numpy(), want), f"frame {f} plane {p}"
    ft.close()
