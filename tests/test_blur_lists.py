"""The low-pass job lists as the device holds them (T360B200_hostPlanBlurLists, no GPU): every pixel of every segment that
fits the plane is filtered by exactly one job with its segment's taps, the lists of a frame's planes merge into one list
with rebased tap offsets and plane tags, and the packed images equal the recorded ones (tests/golden/blur_lists.json).
One GPU test runs merged frame lists of two plane counts interleaved on two streams against the oracle."""
import json
from pathlib import Path

import numpy as np
import pytest

import transform360_b200 as t360
from tests.golden.cases import FULL, SMALL, chroma

GOLDEN = Path(__file__).resolve().parent / "golden" / "blur_lists.json"

VIEWS = [(0.0, 0.0, 120.0, 110.0), (-150.0, 85.0, 140.0, 100.0), (10.0, -80.0, 170.0, 150.0)]  # (three different lists)
FLAT = dict(output_layout=t360.LAYOUT_FLAT_FIXED, interpolation_alg=t360.CUBIC)
CASES = {  # name: (context overrides, luma in, luma out, plane size the lists are cut for: None = planned)
    "cfg3": (FULL["cfg3"]["ov"], FULL["cfg3"]["inp"], FULL["cfg3"]["out"], None),
    "cfg4": (FULL["cfg4"]["ov"], FULL["cfg4"]["inp"], FULL["cfg4"]["out"], None),
    "lp_tiles": (SMALL["lp_tiles"]["ov"], SMALL["lp_tiles"]["inp"], SMALL["lp_tiles"]["out"], None),
    "lp_big_kernels": (SMALL["lp_big_kernels"]["ov"], SMALL["lp_big_kernels"]["inp"], SMALL["lp_big_kernels"]["out"], None),
    "huge_sigma": (dict(interpolation_alg=t360.CUBIC, num_vertical_segments=300, num_horizontal_segments=1, adjust_kernel=0,
                        min_kernel_half_height=40.0), (1280, 640), (192, 128), None),
    "lr_stereo": (SMALL["lr_stereo"]["ov"], SMALL["lr_stereo"]["inp"], SMALL["lr_stereo"]["out"], None),
    "eac_tb_lanczos": (SMALL["eac_tb_lanczos"]["ov"], SMALL["eac_tb_lanczos"]["inp"], SMALL["eac_tb_lanczos"]["out"], None),
    "lp_default_other_size": (SMALL["lp_default"]["ov"], SMALL["lp_default"]["inp"], SMALL["lp_default"]["out"], (700, 350)),
    **{f"flat_view{i}": (dict(FLAT, fixed_yaw=v[0], fixed_pitch=v[1], fixed_hfov=v[2], fixed_vfov=v[3]), (1920, 960), (640, 360), None)
       for i, v in enumerate(VIEWS)},
}
_plans = {}


def _plans_of(name):
    """(luma plan, chroma plan) of a case, made once per session."""
    if name not in _plans:
        ov, inp, out, _ = CASES[name]
        ctx = t360.make_context(**ov)
        _plans[name] = (t360.HostPlan(ctx, *inp, *out), t360.HostPlan(ctx, *chroma(inp), *chroma(out)))
    return _plans[name]


def _lists(name, plane):
    """The lists of plane 0 (luma) or 1 (chroma) of a case, and the segments that fit the plane they were cut for
    (both stereo passes), and its size."""
    ov, inp, _, size = CASES[name]
    plan = _plans_of(name)[plane]
    w, h = size if size and not plane else (inp if not plane else chroma(inp))
    lists = plan.blur_lists(width=w, height=h) if size and not plane else plan.blur_lists()
    stereo = ov.get("input_stereo_format", t360.STEREO_FORMAT_MONO)
    passes = [(0, 0)] + ([(int(0.5 * w), 0)] if stereo == t360.STEREO_FORMAT_LR else [(0, int(0.5 * h))] if stereo == t360.STEREO_FORMAT_TB else [])
    out = []
    for ox, oy in passes:
        for left, top, sw, sh, kx, ky in plan.segments():
            l, t = left + ox, top + oy
            if l >= 0 and t >= 0 and sw > 0 and sh > 0 and l + sw <= w and t + sh <= h:
                out.append((l, t, sw, sh, kx, ky))
    return lists, out, w, h


def _jobs(lists):
    """Every job as ((kind, strip list), row)."""
    for c, strips in enumerate(lists["strips"]):
        for r in strips:
            yield ("strip", c), r
    for kind in ("tiles", "direct"):
        for r in lists[kind]:
            yield (kind, None), r


PLANE_CASES = [(n, p) for n in sorted(CASES) for p in (0, 1)]


@pytest.mark.parametrize("name,plane", PLANE_CASES)
def test_every_pixel_of_every_fitting_segment_is_filtered_by_one_job(name, plane):
    lists, segs, w, h = _lists(name, plane)
    count = np.zeros((h, w), np.uint8)
    for _, r in _jobs(lists):
        x0, y0, jw, jh = (int(v) for v in r[:4])
        assert jw > 0 and jh > 0 and x0 >= 0 and y0 >= 0 and x0 + jw <= w and y0 + jh <= h
        count[y0:y0 + jh, x0:x0 + jw] += 1
    inside = np.zeros((h, w), bool)
    for l, t, sw, sh, _, _ in segs:
        inside[t:t + sh, l:l + sw] = True
    assert (count[inside] == 1).all(), f"{int((count[inside] != 1).sum())} px of fitting segments not filtered exactly once"
    assert not count[~inside].any(), "a job filters pixels outside every fitting segment"
    assert lists["needs_clear"] == bool((count == 0).any())


@pytest.mark.parametrize("name,plane", PLANE_CASES)
def test_every_job_reads_its_segments_taps(name, plane):
    lists, segs, w, h = _lists(name, plane)
    owner = np.full((h, w), -1, np.int32)
    for i, (l, t, sw, sh, _, _) in enumerate(segs):
        owner[t:t + sh, l:l + sw] = i
    taps, tap_at = lists["taps"], lists["offsets"][5]
    assert tap_at % 16 == 0
    for (kind, c), r in _jobs(lists):
        _, _, _, _, kx, ky = segs[owner[r[1], r[0]]]
        if kind == "strip":
            _, _, _, _, kx_off, chunks, kx_count, ky_off, edge = (int(v) for v in r)
            assert len(kx) % 2 == 1 and len(ky) % 2 == 1 and max(len(ky) // 2, 1) == c + 1 and edge in (0, 1)
            assert kx_count == len(kx) and chunks == (len(kx) + 3) // 4 and (tap_at + 4 * kx_off) % 16 == 0
            assert np.array_equal(taps[kx_off:kx_off + 4 * chunks], np.concatenate([kx, np.zeros(4 * chunks - len(kx), np.float32)]))
            want_ky = np.array([0.0, ky[0], 0.0], np.float32) if len(ky) == 1 else ky
            assert np.array_equal(taps[ky_off:ky_off + len(want_ky)], want_ky)
        else:
            _, _, _, _, kx_off, kx_count, ky_off, ky_count = (int(v) for v in r)
            assert (kx_count, ky_count) == (len(kx), len(ky))
            assert np.array_equal(taps[kx_off:kx_off + kx_count], kx) and np.array_equal(taps[ky_off:ky_off + ky_count], ky)
    assert (lists["tile_smem"] > 0) == (len(lists["tiles"]) > 0)


def _weight(r):
    return (int(r[5]) + 2) * int(r[3]) * (1 + 3 * (int(r[8]) & 1))


@pytest.mark.parametrize("name", sorted(n for n in CASES if CASES[n][3] is None))
@pytest.mark.parametrize("num_planes", [2, 3])
def test_merged_lists_are_the_plane_lists_rebased_and_heaviest_first(name, num_planes):
    luma, chroma_plan = _plans_of(name)
    planes = [luma] + [chroma_plan] * (num_planes - 1)
    merged = luma.blur_lists(*planes[1:])
    per_plane = [p.blur_lists() for p in planes]
    base, bases = 0, []
    for p, lists in enumerate(per_plane):
        base = (base + 3) // 4 * 4
        bases.append(base)
        assert np.array_equal(merged["taps"][base:base + len(lists["taps"])], lists["taps"])
        base += len(lists["taps"])
    assert len(merged["taps"]) == base and not len(merged["tiles"]) and not len(merged["direct"])
    for c in range(3):
        want = []
        for p, lists in enumerate(per_plane):
            for r in lists["strips"][c]:
                r = r.copy()
                r[4] += bases[p]
                r[7] += bases[p]
                r[8] |= p << 8
                want.append(r)
        want.sort(key=lambda r: -_weight(r))  # (stable: planes in order inside one weight)
        got = merged["strips"][c]
        assert np.array_equal(got, np.array(want, np.int32).reshape(-1, 9)), f"strips of half-size {c + 1}"
        assert all(_weight(a) >= _weight(b) for a, b in zip(got, got[1:]))


def fnv1a64(data: bytes) -> str:
    h = 0xCBF29CE484222325
    for b in data:
        h = ((h ^ b) * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
    return f"{h:016x}"


def all_list_hashes():
    """FNV-1a 64 of every packed image the tests above look at: per plane, and merged for 2 and 3 planes."""
    out = {}
    for name in sorted(CASES):
        for plane in (0, 1):
            out[f"{name}/plane{plane}"] = fnv1a64(_lists(name, plane)[0]["image"])
        if CASES[name][3] is None:
            luma, chroma_plan = _plans_of(name)
            for n in (2, 3):
                out[f"{name}/merged{n}"] = fnv1a64(luma.blur_lists(*[chroma_plan] * (n - 1))["image"])
    return out


def test_packed_lists_equal_the_recorded_images():
    want = json.loads(GOLDEN.read_text())
    got = all_list_hashes()
    assert sorted(got) == sorted(want)
    diff = [k for k in got if got[k] != want[k]]
    assert not diff, f"packed low-pass lists changed: {diff}"


@pytest.mark.gpu
def test_two_and_three_plane_frames_interleaved_on_two_streams():
    """3-plane and 2-plane low-pass frames enqueued alternately on two streams without synchronising in between: each
    plane count launches its own merged lists, and every output equals the oracle."""
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests must run on an H100 (there is no CPU fallback to test)")
    from oracle import c_oracle as co
    from oracle import ref_harness as rh
    from transform360_b200.stream import FrameTransformer, StreamSpec
    ov = dict(interpolation_alg=t360.CUBIC, num_horizontal_segments=4, num_vertical_segments=9)
    spec = StreamSpec(960, 480, 320, 240)
    ft = FrameTransformer(t360.make_context(**ov), spec)
    octx = rh.default_context(**ov)
    plans = {idx: co.OraclePlan(octx, *spec.plane_dims(p)[:4]) for p, idx in ((0, 0), (1, 1))}
    pitch = lambda w: (w + 255) // 256 * 256
    frames, calls = [], []
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for f in range(8):
        n = 3 if f % 2 == 0 else 2
        srcs = [co.noise_plane(*spec.plane_dims(p)[:2], plane=p, frame=f) for p in range(n)]
        d_in, d_out = [], []
        for p, a in enumerate(srcs):
            t = torch.zeros((a.shape[0], pitch(a.shape[1])), dtype=torch.uint8, device="cuda")
            t[:, :a.shape[1]] = torch.from_numpy(a).cuda()
            d_in.append(t)
            d_out.append(torch.zeros((spec.plane_dims(p)[3], pitch(spec.plane_dims(p)[2])), dtype=torch.uint8, device="cuda"))
        dims = [spec.plane_dims(p)[:4] for p in range(n)]
        calls.append(ft.vft.make_frame_call([(t.data_ptr(), t.stride(0)) for t in d_in], [(t.data_ptr(), t.stride(0)) for t in d_out], dims))
        frames.append((srcs, d_in, d_out))
    torch.cuda.synchronize()
    for f, call in enumerate(calls):
        assert call(streams[f % 2].cuda_stream), f"frame {f} refused"
    torch.cuda.synchronize()
    for f, (srcs, _, d_out) in enumerate(frames):
        for p, src in enumerate(srcs):
            iw, ih, ow, oh, idx = spec.plane_dims(p)
            want = co.transform_plane(octx, plans[idx], src, ow, oh, map_index=idx)
            got = d_out[p][:, :ow].cpu().numpy()
            assert np.array_equal(got, want), f"frame {f} ({len(srcs)} planes) plane {p}: {int((got != want).sum())} px differ"
    ft.close()
