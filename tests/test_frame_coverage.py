"""Which paths of the frame gather the GPU tests reach, and whole frames through T360B200_transformFrameAsync at the
shapes, layouts and job counts where the kernel, the merged job list or the scheduler could go wrong.

gatherFrameKernel<K, COPIES, GROUPS> has one consumer branch per job kind (share, share-stay, class 0 as a whole 32 x 32
tile or one 16 x 16 quadrant, class 1, seam, pole cap, border), is instantiated for K = 2, 4 and 8, and claims jobs
statically (two per producer warp) and then from an atomic counter that the last producer re-arms.  The ledger below
plans the frames of the GPU tests on the host and lists the (K, kind) pairs in their launch lists, so that a planner
change which moves jobs away from a kind fails here, on a CPU, instead of leaving that branch untested on the GPU.
"""
from __future__ import annotations

import functools

import numpy as np
import pytest

import transform360_b200 as t360
from oracle import c_oracle as co
from oracle import ref_harness as rh
from transform360_b200.stream import FrameTransformer, StreamSpec

KIND_SHIFT = 24
KIND_NAMES = {1: "class1", 3: "share_stay", 4: "share", 7: "seam", 8: "cap", 9: "border"}  # 0: "tile" / "quad"
KINDS = ("tile", "quad", "class1", "cap", "border", "seam", "share", "share_stay")
# (K, kind) pairs the planner cannot produce, and why
UNREACHABLE = {
    (2, "share"): "shareBlock() takes 64 x 32 share blocks for kernel sizes >= 4 only",
    (2, "share_stay"): "shareBlock() takes 64 x 32 share blocks for kernel sizes >= 4 only",
}
REQUIRED = {(k, kind) for k in (2, 4, 8) for kind in KINDS} - set(UNREACHABLE)


def kind_name(job) -> str:
    kind = (int(job[1]) >> KIND_SHIFT) & 15
    return KIND_NAMES.get(kind) or ("quad" if int(job[0]) & 7 else "tile")


@functools.lru_cache(maxsize=None)
def _host_plan(ov_items, iw, ih, ow, oh):
    """(kernel size, launch list kinds, map size) of one plane's plan."""
    hp = t360.HostPlan(t360.make_context(**dict(ov_items)), iw, ih, ow, oh)
    launch = hp.pole_caps()["launch"]
    out = (hp.kernel_size, tuple(kind_name(j) for j in launch), (hp.map_w, hp.map_h))
    hp.close()
    return out


def plane_plan(case, p):
    iw, ih, ow, oh, _ = case_spec(case).plane_dims(p)
    return _host_plan(tuple(sorted(case["ov"].items())), iw, ih, ow, oh)


def case_spec(case) -> StreamSpec:
    return StreamSpec(*case["inp"], *case["out"], num_planes=case["planes"])


def staged(case, p) -> bool:
    """Does plane p run in the frame kernel?  Its plan has a launch list, and its source is TMA-describable: the low-pass
    output (the library's own 256-byte-pitch plane) or a caller plane with a 16-byte aligned base and pitch."""
    _, kinds, _ = plane_plan(case, p)
    in_off, in_pitch = case["layout"][p][:2]
    return bool(kinds) and (bool(case["ov"].get("enable_low_pass_filter", 1)) or (in_off % 16 == 0 and in_pitch % 16 == 0))


def ledger(cases) -> dict:
    """(K, kind) -> number of cases whose frame kernel launches hold a job of that kind."""
    seen: dict = {}
    for case in cases:
        pairs = set()
        for p in range(case["planes"]):
            if staged(case, p):
                k, kinds, _ = plane_plan(case, p)
                pairs.update((k, kind) for kind in kinds)
        for pair in pairs:
            seen[pair] = seen.get(pair, 0) + 1
    return seen


def assert_required(cases, what):
    seen = ledger(cases)
    missing = sorted(REQUIRED - set(seen))
    assert not missing, f"{what} reach no job of {missing} (K, kind): the frame kernel's branches for them go untested"


# ---- the sweep: whole frames, seeded ----------------------------------------------------------------------------------
def _pitch(w, kind, rng):
    """A row pitch for a plane of width w: 'page' (256-byte multiple), 'row16' (16-byte multiple, not 256) or 'odd'."""
    if kind == "page":
        return (w + 255) // 256 * 256 + 256 * int(rng.integers(0, 2))
    if kind == "row16":
        p = (w + 15) // 16 * 16 + 16 * int(rng.integers(0, 4))
        return p + 16 if p % 256 == 0 else p
    return w + 1 + 2 * int(rng.integers(0, 8))


def page_layout(case):
    """Every plane at offset 0 with a 256-byte-multiple pitch."""
    page = lambda w: (w + 255) // 256 * 256
    return [(0, page(d[0]), 0, page(d[2])) for d in map(case_spec(case).plane_dims, range(case["planes"]))]


def _layout(case, rng, unaligned_plane=None):
    """Per plane (input base offset, input pitch, output base offset, output pitch) in bytes."""
    spec = case_spec(case)
    out = []
    for p in range(case["planes"]):
        iw, _, ow, _, _ = spec.plane_dims(p)
        kind = "odd" if p == unaligned_plane else str(rng.choice(["page", "page", "row16"]))
        in_off = 16 * int(rng.integers(0, 2)) if kind != "odd" else int(rng.choice([0, 16]))
        out_kind = str(rng.choice(["page", "row16", "odd"]))
        out_off = int(rng.choice([0, 16, 16, 5]))
        out.append((in_off, _pitch(iw, kind, rng), out_off, _pitch(ow, out_kind, rng)))
    return out


NAMED = [  # (context overrides, luma in, luma out, planes): the frames that give the ledger its pairs at small sizes
    (dict(interpolation_alg=t360.CUBIC), (832, 416), (384, 256), 3),                       # K 4: seam, share, caps, border
    (dict(output_layout=6, interpolation_alg=t360.LANCZOS4), (832, 416), (384, 256), 3),  # K 8: seam, share, caps, border
    (dict(output_layout=3, interpolation_alg=t360.CUBIC), (832, 416), (384, 256), 2),
    (dict(output_layout=0, interpolation_alg=t360.LANCZOS4), (832, 416), (383, 255), 3),
    (dict(output_layout=2, interpolation_alg=t360.CUBIC), (832, 416), (384, 256), 3),      # share + share-stay only
    (dict(output_layout=2, interpolation_alg=t360.LANCZOS4), (832, 416), (384, 256), 1),
    (dict(output_layout=0, interpolation_alg=t360.LINEAR), (960, 480), (240, 160), 3),     # class 1 of each K
    (dict(output_layout=6, interpolation_alg=t360.CUBIC), (960, 480), (240, 160), 2),
    (dict(output_layout=6, interpolation_alg=t360.LANCZOS4), (960, 480), (240, 160), 3),
    (dict(interpolation_alg=t360.LINEAR), (1024, 512), (384, 256), 3),                     # K 2: quadrants, caps
    (dict(output_layout=6, interpolation_alg=t360.LINEAR), (976, 340), (282, 245), 3),     # K 2: seam
    (dict(fixed_cube_offcenter_z=-0.3, is_horizontal_offset=1, fixed_yaw=10.0, interpolation_alg=t360.LINEAR),
     (512, 256), (192, 128), 3),                                                           # K 2: border
    (dict(interpolation_alg=t360.CUBIC), (1920, 960), (768, 512), 3),                      # 950 jobs: dynamic claims
    (dict(interpolation_alg=t360.LANCZOS4, num_vertical_segments=9, num_horizontal_segments=4), (1920, 960), (768, 512), 2),
]
NUM_SWEEP = 75


def _random_overrides(rng):
    from tests.test_host_plan import _random_context
    ov = _random_context(rng)
    ov["input_layout"] = int(rng.choice([3, 3, 3, 3, 0, 6]))
    ov["output_layout"] = int(rng.choice([0, 0, 1, 2, 3, 6, 6, 4, 5]))
    ov["interpolation_alg"] = int(rng.choice([1, 1, 2, 2, 4, 4, 0]))
    ov["enable_low_pass_filter"] = int(rng.random() < 0.4)
    if rng.random() < 0.15:
        ov["width_scale_factor"] = float(rng.choice([1.5, 2.0]))
        ov["height_scale_factor"] = float(rng.choice([1.0, 1.25, 2.0]))
    else:
        ov.pop("width_scale_factor", None)
        ov.pop("height_scale_factor", None)
    return ov


@functools.lru_cache(maxsize=None)
def sweep_cases():
    rng = np.random.default_rng(20261016)
    cases = []

    def add(ov, inp, out, planes):
        case = dict(ov=dict(ov, **({} if "enable_low_pass_filter" in ov else {"enable_low_pass_filter": 0})),
                    inp=inp, out=out, planes=planes)
        try:
            for p in range(min(planes, 2)):
                plane_plan(case, p)
        except ValueError:  # the planner refuses what the reference refuses
            return
        unaligned = int(rng.integers(0, planes)) if planes > 1 and rng.random() < 0.2 else None
        case["layout"] = _layout(case, rng, unaligned)
        cases.append(case)

    for ov, inp, out, planes in NAMED:
        add(ov, inp, out, planes)
    while len(cases) < NUM_SWEEP:
        ov = _random_overrides(rng)
        if rng.random() < 0.5:  # wide planes: seam and share jobs
            iw = int(rng.integers(52, 129)) * 16
            ih = int(rng.integers(iw // 32, iw // 8 + 1)) * 4
        else:
            iw, ih = int(rng.integers(200, 800)), int(rng.integers(100, 400))
        ow = int(rng.integers(32, 400)) * 2 + int(rng.random() < 0.3)
        oh = int(rng.integers(24, 300)) * 2 + int(rng.random() < 0.3)
        add(ov, (iw, ih), (ow, oh), int(rng.choice([1, 2, 3, 3])))
    return cases


def expected_gather_launches(case):
    """Kernel launches of one frame besides the low-pass: ONE gather for all planes when every plane is staged and there are
    several, else one per plane; and an area resize per plane whose requested size is not its map's."""
    planes, spec = case["planes"], case_spec(case)
    gathers = 1 if planes > 1 and all(staged(case, p) for p in range(planes)) else planes
    resizes = sum(plane_plan(case, p)[2] != spec.plane_dims(p)[2:4] for p in range(planes))
    return gathers + resizes


# ---- boundary job counts of the scheduler -----------------------------------------------------------------------------
def groups_of(k):
    return 2 if k == 8 else 3


def boundary_targets(k, planes, num_sms):
    """Launch-list lengths around the static capacity S = N * G * 2 (two static jobs per producer warp)."""
    g = groups_of(k)
    s = num_sms * g * 2
    # (a 3-plane frame has a job per plane at least; for K = 8, where 2G - 1 = 3, it takes 2G: one CTA's producers full)
    small = [1, 2 * g - 1] if planes == 1 else [3, max(2 * g - 1, 4)]
    return small + [s - 1, s, s + 1, 2 * s + 1]


def _flat_ov(k, ow, oh, iw, ih):
    """FLAT_FIXED, no rotation, with the field of view scaled to the output so that the view is a little denser than the
    source: share blocks wherever the output is at least 64 x 32."""
    interp = {4: t360.CUBIC, 8: t360.LANCZOS4}[k]
    hfov = float(min(150.0, max(4.0, ow * 360.0 / iw / 1.25)))
    vfov = float(min(150.0, max(4.0, oh * 180.0 / ih / 1.25)))
    return dict(output_layout=2, interpolation_alg=interp, enable_low_pass_filter=0, fixed_hfov=hfov, fixed_vfov=vfov)


FLAT_IN = (1920, 960)


def boundary_case(k, planes, ow, oh):
    ov = _flat_ov(k, ow, oh, *FLAT_IN)
    return dict(ov=ov, inp=FLAT_IN, out=(ow, oh), planes=planes)


def frame_jobs(k, planes, ow, oh):
    case = boundary_case(k, planes, ow, oh)
    return sum(len(plane_plan(case, p)[1]) for p in range(planes))


def flat_plane_jobs(w, h):
    """Jobs of a plane of these views (_flat_ov): 64 x 32 share blocks, a 32 x 32 tile per row for the columns they leave,
    and a tile per 32 columns for the rows they leave."""
    w, h = np.asarray(w), np.asarray(h)
    rows = h // 32
    return (w // 64) * rows + -(-(w % 64) // 32) * rows + np.where(h % 32 > 0, -(-w // 32), 0)


@functools.lru_cache(maxsize=None)
def boundary_size(k, planes, n):
    """A luma output size (ow, oh) of about 3:2 whose frame's merged launch list holds exactly n jobs, predicted by
    flat_plane_jobs and confirmed by the planner (None: none found)."""
    ow, oh = np.meshgrid(np.arange(16, 2561, 2), np.arange(16, 2561, 2), indexing="ij")
    total = flat_plane_jobs(ow, oh)
    if planes == 3:
        total = total + 2 * flat_plane_jobs((ow + 1) // 2, (oh + 1) // 2)
    cand = np.argwhere(total == n)
    aspect = np.abs(np.log(ow[tuple(cand.T)] / oh[tuple(cand.T)] / 1.5))
    for i in np.argsort(aspect, kind="stable")[:8]:
        size = int(ow[tuple(cand[i])]), int(oh[tuple(cand[i])])
        if frame_jobs(k, planes, *size) == n:
            return size
    return None


BOUNDARY = [(k, planes, i) for k in (4, 8) for planes in (1, 3) for i in range(6)]


# ---- CPU: the ledger --------------------------------------------------------------------------------------------------
def test_kind_names_split_class0_by_quadrant_bits():
    assert kind_name((64, 32 << 0, 0, 0)) == "tile" and kind_name((64 | 3, 0, 0, 0)) == "quad"
    assert kind_name((0, (7 << KIND_SHIFT) | 32, 0, 0)) == "seam" and kind_name((0, 9 << KIND_SHIFT, 0, 0)) == "border"


def test_unreachable_pairs_are_not_produced():
    """The pairs listed as unreachable really never occur, in any frame of the sweep."""
    seen = ledger(sweep_cases())
    assert not set(seen) & set(UNREACHABLE), sorted(set(seen) & set(UNREACHABLE))


def test_sweep_and_boundary_frames_reach_every_required_pair():
    """The GPU frames of this module (the sweep, and the boundary frames of a 132-SM H100) reach every (K, kind) pair."""
    cases = list(sweep_cases())
    for k, planes, i in BOUNDARY:
        size = boundary_size(k, planes, boundary_targets(k, planes, 132)[i])
        if size:
            case = boundary_case(k, planes, *size)
            cases.append(dict(case, layout=page_layout(case)))
    assert_required(cases, "the frames of tests/test_frame_coverage.py")


def test_sweep_has_the_shapes_it_is_meant_to_have():
    cases = sweep_cases()
    assert len(cases) == NUM_SWEEP
    wide = [c for c in cases if c["inp"][0] % 16 == 0 and c["inp"][0] >= 832]
    assert 2 * len(wide) >= len(cases), "at least half the frames have planes wide enough for seam and share jobs"
    assert {c["planes"] for c in cases} == {1, 2, 3}
    assert any(c["out"][0] % 2 for c in cases) and any(c["out"][1] % 2 for c in cases)
    ks = {plane_plan(c, 0)[0] for c in cases}
    assert {1, 2, 4, 8} <= ks, ks
    merged = [c for c in cases if c["planes"] > 1 and all(staged(c, p) for p in range(c["planes"]))]
    mixed = [c for c in cases if c["planes"] > 1 and any(staged(c, p) for p in range(c["planes"]))
             and not all(staged(c, p) for p in range(c["planes"]))]
    assert len(merged) >= 20 and len(mixed) >= 3, (len(merged), len(mixed))
    assert any(c["ov"]["enable_low_pass_filter"] and c["planes"] > 1 for c in merged)
    assert any(expected_gather_launches(c) > (1 if c in merged else c["planes"]) for c in cases), "no frame with a resize"
    pitches = [lay[1] for c in cases for lay in c["layout"]]
    assert any(p % 256 == 0 for p in pitches) and any(p % 16 == 0 and p % 256 for p in pitches)
    assert any(lay[0] == 16 for c in cases for lay in c["layout"])


@pytest.mark.parametrize("num_sms", [132, 114])
def test_boundary_job_counts_are_found(num_sms):
    """The host search finds output sizes whose merged launch lists hold exactly the job counts around the static capacity
    (an SXM H100 has 132 SMs, a PCIe one 114)."""
    for k in (4, 8):
        for planes in (1, 3):
            for n in boundary_targets(k, planes, num_sms):
                size = boundary_size(k, planes, n)
                assert size is not None and frame_jobs(k, planes, *size) == n, (k, planes, n)


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests must run on an H100 (there is no CPU fallback to test)")
    return torch


def _prefill(ov):
    return 7 if ov.get("output_layout") in (t360.LAYOUT_BARREL, t360.LAYOUT_BARREL_SPLIT) else 0


PAD = 0xCD


class FrameBuffers:
    """The device planes of one frame laid out as (base offset, pitch) says; input padding holds noise, output padding and
    the bytes before the output base hold PAD."""

    def __init__(self, torch, spec, layout, srcs, fill):
        self.torch, self.spec, self.layout = torch, spec, layout
        self.ins, self.outs, self.in_ptrs, self.out_ptrs = [], [], [], []
        g = torch.Generator(device="cpu").manual_seed(1)
        for p, src in enumerate(srcs):
            iw, ih, ow, oh, _ = spec.plane_dims(p)
            in_off, in_pitch, out_off, out_pitch = layout[p]
            buf = torch.randint(0, 256, (in_off + in_pitch * ih + 64,), dtype=torch.uint8, generator=g).cuda()
            buf[in_off:in_off + in_pitch * ih].view(ih, in_pitch)[:, :iw] = torch.from_numpy(np.ascontiguousarray(src)).cuda()
            out = torch.full((out_off + out_pitch * oh + 64,), PAD, dtype=torch.uint8, device="cuda")
            out[out_off:out_off + out_pitch * oh].view(oh, out_pitch)[:, :ow] = fill
            self.ins.append(buf)
            self.outs.append(out)
            self.in_ptrs.append((buf.data_ptr() + in_off, in_pitch))
            self.out_ptrs.append((out.data_ptr() + out_off, out_pitch))

    def output(self, p):
        """(plane pixels, everything else of the buffer)"""
        _, _, ow, oh, _ = self.spec.plane_dims(p)
        out_off, out_pitch = self.layout[p][2:]
        host = self.outs[p].cpu().numpy()
        rows = host[out_off:out_off + out_pitch * oh].reshape(oh, out_pitch)
        rest = np.concatenate([host[:out_off], rows[:, ow:].ravel(), host[out_off + out_pitch * oh:]])
        return rows[:, :ow], rest


@functools.lru_cache(maxsize=8)
def _oracle_plan(octx_key, iw, ih, ow, oh):
    return co.OraclePlan(rh.default_context(**dict(octx_key)), iw, ih, ow, oh)


def oracle_plane(ov, spec, p, src, fill):
    iw, ih, ow, oh, idx = spec.plane_dims(p)
    key = tuple(sorted(ov.items()))
    return co.transform_plane(rh.default_context(**ov), _oracle_plan(key, iw, ih, ow, oh), src, ow, oh, map_index=idx, prefill=fill)


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(NUM_SWEEP))
def test_sweep_frames_through_the_frame_entry_point(i, torch_cuda):
    """Frame i of the sweep: two frames (different inputs) back to back on a non-default stream with no synchronise in
    between, every pixel of every plane of both against the oracle, bit-exact; the row padding and the bytes around the
    output planes untouched; the kernel launches of one frame as the planes' layouts and plans predict."""
    torch = torch_cuda
    cases = sweep_cases()
    if i == 0:  # what the sweep reaches, before any GPU work
        assert_required(cases, "the sweep's frames")
    case = cases[i]
    ov, spec = case["ov"], case_spec(case)
    ctx = t360.make_context(**ov)
    fill = _prefill(ov)
    ft = FrameTransformer(ctx, spec)
    dims = [spec.plane_dims(p)[:4] for p in range(case["planes"])]
    frames, calls = [], []
    for f in range(2):
        srcs = [co.noise_plane(*spec.plane_dims(p)[:2], plane=p, frame=100 * i + f) for p in range(case["planes"])]
        bufs = FrameBuffers(torch, spec, case["layout"], srcs, fill)
        frames.append((srcs, bufs))
        calls.append(ft.vft.make_frame_call(bufs.in_ptrs, bufs.out_ptrs, dims))
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    n0 = t360.kernel_launch_count()
    for call in calls:
        assert call(st.cuda_stream), "T360B200_transformFrameAsync failed"
    launches = t360.kernel_launch_count() - n0
    st.synchronize()
    want = expected_gather_launches(case)
    if ov["enable_low_pass_filter"]:  # (plus the low-pass launches, one per vertical kernel size and job list)
        assert launches >= 2 * want, f"{launches} launches for two frames with low-pass, expected {2 * want} and more"
    else:
        assert launches == 2 * want, f"{launches} launches for two frames, expected {2 * want}"
    for f, (srcs, bufs) in enumerate(frames):
        for p in range(case["planes"]):
            got, rest = bufs.output(p)
            exp = oracle_plane(ov, spec, p, srcs[p], fill)
            assert np.array_equal(got, exp), f"frame {f} plane {p}: {int((got != exp).sum())} px differ from the oracle"
            assert (rest == PAD).all(), f"frame {f} plane {p}: bytes outside the plane were written"
    ft.close()


@pytest.mark.gpu
@pytest.mark.parametrize("k,planes,i", BOUNDARY)
def test_scheduler_boundaries(k, planes, i, torch_cuda):
    """Merged launch lists of 1 job, fewer jobs than one CTA's producers hold, S - 1, S, S + 1 and 2S + 1 jobs for the
    static capacity S = SMs * groups * 2 of this device: the frame three times back to back on one stream (a wrong re-arm
    of the claim counter shows on the second or third launch), every output against the oracle."""
    torch = torch_cuda
    num_sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = boundary_targets(k, planes, num_sms)[i]
    size = boundary_size(k, planes, n)
    assert size is not None, f"no output size gives a frame of {n} jobs"
    case = boundary_case(k, planes, *size)
    spec = case_spec(case)
    case["layout"] = page_layout(case)
    assert all(staged(case, p) for p in range(planes))
    ft = FrameTransformer(t360.make_context(**case["ov"]), spec)
    srcs = [co.noise_plane(*spec.plane_dims(p)[:2], plane=p, frame=n) for p in range(planes)]
    dims = [spec.plane_dims(p)[:4] for p in range(planes)]
    runs = [FrameBuffers(torch, spec, case["layout"], srcs, 0) for _ in range(3)]
    calls = [ft.vft.make_frame_call(runs[0].in_ptrs, b.out_ptrs, dims) for b in runs]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    n0 = t360.kernel_launch_count()
    for call in calls:
        assert call(st.cuda_stream)
    assert t360.kernel_launch_count() - n0 == 3, "one launch per frame"
    st.synchronize()
    for p in range(planes):
        exp = oracle_plane(case["ov"], spec, p, srcs[p], 0)
        for r, b in enumerate(runs):
            got, rest = b.output(p)
            assert np.array_equal(got, exp), f"{n} jobs, run {r} plane {p}: {int((got != exp).sum())} px differ"
            assert (rest == PAD).all()
    ft.close()


CACHE_CASE = dict(ov=dict(interpolation_alg=t360.CUBIC, enable_low_pass_filter=0), inp=(512, 256), out=(192, 128), planes=3)


@pytest.mark.gpu
def test_tensor_map_cache_evicts_and_reencodes(torch_cuda):
    """40 distinct source frames (more than the 32 planes a lane remembers) twice through one transform: every lookup of
    the second pass misses, evicts and re-encodes.  Every output against the oracle."""
    torch = torch_cuda
    case = dict(CACHE_CASE, layout=page_layout(CACHE_CASE))
    ov, spec = case["ov"], case_spec(case)
    ft = FrameTransformer(t360.make_context(**ov), spec)
    dims = [spec.plane_dims(p)[:4] for p in range(3)]
    srcs = [[co.noise_plane(*spec.plane_dims(p)[:2], plane=p, frame=300 + f) for p in range(3)] for f in range(40)]
    ins = [FrameBuffers(torch, spec, case["layout"], s, 0) for s in srcs]
    outs = [[FrameBuffers(torch, spec, case["layout"], srcs[0], 0) for _ in range(40)] for _ in range(2)]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    for rnd in range(2):
        for f in range(40):
            assert ft.vft.make_frame_call(ins[f].in_ptrs, outs[rnd][f].out_ptrs, dims)(st.cuda_stream)
    st.synchronize()
    for f in range(40):
        for p in range(3):
            exp = oracle_plane(ov, spec, p, srcs[f][p], 0)
            for rnd in range(2):
                got, _ = outs[rnd][f].output(p)
                assert np.array_equal(got, exp), f"pass {rnd} frame {f} plane {p}: {int((got != exp).sum())} px differ"
    ft.close()


@pytest.mark.gpu
@pytest.mark.parametrize("interp", [t360.CUBIC, t360.LANCZOS4])
def test_reused_input_surface_refilled_on_the_stream(interp, torch_cuda):
    """A decoder's surface pool: one set of input planes, refilled by a device copy on the calling stream before every frame
    call, no synchronise; each frame's output in its own buffers matches the oracle for the content it was given."""
    torch = torch_cuda
    case = dict(ov=dict(interpolation_alg=interp, enable_low_pass_filter=0), inp=(832, 416), out=(384, 256), planes=3)
    case["layout"] = page_layout(case)
    ov, spec = case["ov"], case_spec(case)
    ft = FrameTransformer(t360.make_context(**ov), spec)
    dims = [spec.plane_dims(p)[:4] for p in range(3)]
    srcs = [[co.noise_plane(*spec.plane_dims(p)[:2], plane=p, frame=500 + f) for p in range(3)] for f in range(6)]
    surface = FrameBuffers(torch, spec, case["layout"], srcs[0], 0)
    staging = [FrameBuffers(torch, spec, case["layout"], s, 0) for s in srcs]  # what the decoder writes from
    outs = [FrameBuffers(torch, spec, case["layout"], srcs[0], 0) for _ in range(6)]
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(st):
        for f in range(6):
            for p in range(3):
                surface.ins[p].copy_(staging[f].ins[p], non_blocking=True)
            assert ft.vft.make_frame_call(surface.in_ptrs, outs[f].out_ptrs, dims)(st.cuda_stream)
    st.synchronize()
    for f in range(6):
        for p in range(3):
            got, rest = outs[f].output(p)
            exp = oracle_plane(ov, spec, p, srcs[f][p], 0)
            assert np.array_equal(got, exp), f"frame {f} plane {p}: {int((got != exp).sum())} px differ"
            assert (rest == PAD).all()
    ft.close()
