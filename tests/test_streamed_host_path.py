"""The streamed host-plane path: VideoFrameTransform_transformFramePlane with host pointers and a plane of 6 MB or more.

The call cuts the input into 2-8 row bands (chunks) copied on one stream, runs the frame kernel in waves -- wave c is one
launch of the jobs whose source rows have all arrived with chunk c -- and copies the output back in 32-row bands of the
full width, each after the last wave that writes into it (csrc/gather_plan.cpp: scheduleWaves).  For page-locked caller
planes the whole sequence is captured into a CUDA graph once per (plan, buffers, staging planes) and replayed.

Whether the result is right depends on two per-job facts the planner records (launchNeedRows, launchRects).  A job one
row short, or a rectangle that misses a row it writes, still gives the right bytes whenever the upload wins its race
against the kernel, which on an idle card is almost always.  So the CPU tests below check the schedule against what the
plan samples, derived here without trusting either fact: per output pixel the rows its window reads (from the samples)
and the one launch job that writes it (from the job's tile, quadrant or share block, or from the pixel positions a
pole-cap or border job carries).  The GPU tests run the path with T360B200_PIPELINE_STRICT, a legal order in which
every such mistake gives wrong bytes on every call: the staging planes start out poisoned, chunk c + 1 is uploaded only
after wave c, and wave c + 1 runs only after wave c's bands are back on the host.
"""
from __future__ import annotations

import functools

import numpy as np
import pytest

import transform360_b200 as t360
from oracle import c_oracle as co
from oracle import ref_harness as rh
from tests.golden.cases import FULL, SMALL, plane_dims
from transform360_b200.handler import T360_CAMERA_EQUIDISTANT, T360_CAMERA_PANNINI

KIND_SHIFT, ROW_MASK = 24, (1 << 24) - 1
CLASS0, CLASS1, SHARE_STAY, SHARE, SEAM, CAP, BORDER = 0, 1, 3, 4, 7, 8, 9
RECORD_SKIP = 0x8000
CAP_STEP_WORDS, BORDER_PIXEL_WORDS = 64, 4  # kernels.cuh: kCapStepBytes = 256, kBorderPixelBytes = 16
SHARE_W, SHARE_H, TILE = 64, 32, 32          # kShareW, shareH(k) = 4 * shareRows(k), kGatherTileW = kFrameTileH
MIN_BYTES = 6 << 20                          # the default size from which a host plane is streamed
WRAP = t360.BORDER_WRAP


# ---- what the plan samples, derived without the planner's per-job facts -----------------------------------------------
def read_rows(hp, in_h) -> np.ndarray:
    """int64 [mapH][mapW]: per output pixel the end (exclusive) of the source rows its window reads.  A window that leaves
    the plane vertically (BORDER_WRAP) reads up to the last row."""
    row0 = hp.samples[..., 1].astype(np.int64) >> 10
    k = hp.kernel_size
    return np.where((row0 < 0) | (row0 + k > in_h), in_h, row0 + k)


def writer_map(hp) -> np.ndarray:
    """int64 [mapH][mapW]: per output pixel the index of the launch job that writes it; asserts there is exactly one."""
    mw, mh = hp.map_w, hp.map_h
    launch = hp.pole_caps()["launch"].astype(np.int64)
    g = hp.gather_plan()
    pc = hp.pole_caps()
    compact_words = 0 if g["compact"] is None else g["compact"].size
    recs = pc["records"].astype(np.int64)
    writer = np.full((mh, mw), -1, np.int64)
    count = np.zeros((mh, mw), np.int32)
    for j, (ox, oy, _, rec_off) in enumerate(launch):
        kind = (oy >> KIND_SHIFT) & 15
        if kind in (CAP, BORDER):
            at = rec_off * 4 - compact_words
            if kind == CAP:
                words = recs[at:at + ox * CAP_STEP_WORDS].reshape(-1, 2)
                xy = words[(words[:, 0] & RECORD_SKIP) == 0, 1]
            else:
                xy = recs[at:at + ox * BORDER_PIXEL_WORDS].reshape(-1, 4)[:, 2]
            xs, ys = xy & 0xFFFF, xy >> 16
            np.add.at(count, (ys, xs), 1)
            writer[ys, xs] = j
            continue
        x0, y0, quad = ox & ~7, oy & ROW_MASK, (ox & 7) - 1
        if quad >= 0:
            x0, y0, w, h = x0 + 16 * (quad & 1), y0 + 16 * (quad >> 1), 16, 16
        elif kind in (SHARE, SHARE_STAY):
            w, h = SHARE_W, SHARE_H
        else:
            assert kind in (CLASS0, CLASS1, SEAM), f"launch job {j}: kind {kind}"
            w, h = TILE, TILE
        count[y0:y0 + h, x0:x0 + w] += 1
        writer[y0:y0 + h, x0:x0 + w] = j
    assert (count == 1).all(), f"{int((count != 1).sum())} output pixels do not have exactly one writer"
    return writer


class Plane:
    """One plan and what it samples: the launch list's need-rows and rects next to the reads and writers derived here."""

    def __init__(self, hp, in_w, in_h, what):
        self.hp, self.in_w, self.in_h, self.what = hp, in_w, in_h, what
        self.jobs = len(hp.pole_caps()["launch"])

    @functools.cached_property
    def reads(self):
        return read_rows(self.hp, self.in_h)

    @functools.cached_property
    def writer(self):
        return writer_map(self.hp)

    @functools.cached_property
    def _by_job(self):
        """(pixel indices sorted by writer, start of each job's run): every job writes at least one pixel"""
        flat = self.writer.ravel()
        idx = np.argsort(flat, kind="stable")
        starts = np.searchsorted(flat[idx], np.arange(self.jobs))
        assert np.array_equal(np.bincount(flat, minlength=self.jobs) > 0, np.ones(self.jobs, bool)), f"{self.what}: a job writes nothing"
        return idx, starts

    def per_job(self, values, ufunc):
        idx, starts = self._by_job
        return ufunc.reduceat(values.ravel()[idx], starts)

    @functools.cached_property
    def job_reads(self) -> np.ndarray:
        """per launch job the end of the source rows its pixels read"""
        return self.per_job(self.reads, np.maximum)

    @functools.cached_property
    def job_bounds(self) -> np.ndarray:
        """per launch job the bounding rectangle {x0, y0, x1, y1} of the pixels it writes"""
        ys, xs = np.indices(self.writer.shape)
        return np.stack([self.per_job(xs, np.minimum), self.per_job(ys, np.minimum), self.per_job(xs, np.maximum) + 1,
                         self.per_job(ys, np.maximum) + 1], 1)

    @functools.cached_property
    def writer_rows(self):
        """per launch job the output rows it writes"""
        b = self.job_bounds
        return [np.arange(b[j, 1], b[j, 3]) for j in range(self.jobs)]

    def schedule(self, chunks=None, need_rows=None):
        return self.hp.waves(chunks, need_rows)


def job_waves(s) -> np.ndarray:
    wave = np.empty(len(s["order"]), np.int64)
    for c in range(s["chunks"]):
        wave[s["order"][s["wave_start"][c]:s["wave_start"][c + 1]]] = c
    return wave


def check_schedule(p: Plane, s):
    """The four invariants of a streamed plane's schedule; an AssertionError names the chunk, job or band that breaks one."""
    in_h, mh, mw, chunks = p.in_h, p.hp.map_h, p.hp.map_w, s["chunks"]
    ends, starts, order = s["chunk_row_end"].astype(np.int64), s["wave_start"].astype(np.int64), s["order"].astype(np.int64)
    # 1. chunk ends: non-decreasing multiples of 8 (or the plane's end), the last one the plane's end
    assert len(ends) == chunks and ends[-1] == in_h, f"{p.what}: chunk ends {ends.tolist()} do not end at row {in_h}"
    assert (np.diff(ends) >= 0).all() and ((ends % 8 == 0) | (ends == in_h)).all(), f"{p.what}: chunk ends {ends.tolist()}"
    # 4. the waves: a permutation of the launch list, launch order inside each wave
    assert starts[0] == 0 and starts[-1] == p.jobs and (np.diff(starts) >= 0).all(), f"{p.what}: wave starts {starts.tolist()}"
    assert np.array_equal(np.sort(order), np.arange(p.jobs)), f"{p.what}: the waves are not a permutation of the launch list"
    for c in range(chunks):
        w = order[starts[c]:starts[c + 1]]
        if (np.diff(w) <= 0).any():
            j = int(w[1:][np.diff(w) <= 0][0])
            raise AssertionError(f"{p.what}: wave {c} does not keep launch order at job {j}")
    wave = job_waves(s)
    # 2. every pixel's rows have arrived before its writer's wave runs
    pix_wave = wave[p.writer]
    late = p.reads > ends[pix_wave]
    if late.any():
        y, x = (int(v[0]) for v in np.nonzero(late))
        j = int(p.writer[y, x])
        raise AssertionError(f"{p.what}: job {j} runs in wave {wave[j]}, after chunk rows [0, {ends[wave[j]]}), but output pixel "
                             f"({x}, {y}) reads rows up to {int(p.reads[y, x])} (chunks={chunks})")
    # 3. every output row copied exactly once, full width, after a wave no earlier than any of its writers'
    copied = np.zeros(mh, np.int64)
    copy_wave = np.full(mh, -1, np.int64)
    for c, x0, y0, x1, y1 in s["rects"].astype(np.int64):
        assert x0 == 0 and x1 == mw and 0 <= y0 < y1 <= mh, f"{p.what}: band rows {y0}-{y1} x {x0}-{x1} is not a full-width band"
        assert 0 <= c < chunks
        copied[y0:y1] += 1
        copy_wave[y0:y1] = c
    if (copied != 1).any():
        y = int(np.nonzero(copied != 1)[0][0])
        raise AssertionError(f"{p.what}: output row {y} is copied back {int(copied[y])} times")
    row_last = pix_wave.max(axis=1)
    early = copy_wave < row_last
    if early.any():
        y = int(np.nonzero(early)[0][0])
        band = next(r for r in s["rects"] if r[2] <= y < r[4])
        j = int(p.writer[y][pix_wave[y] == row_last[y]][0])
        raise AssertionError(f"{p.what}: band rows {band[2]}-{band[4]} is copied back after wave {band[0]}, but job {j} writes "
                             f"row {y} in wave {int(row_last[y])} (chunks={chunks})")


def check_extents(p: Plane):
    """The planner's need-rows and rects against the reads and writers derived here: a wrong one is named by its job."""
    ext = p.hp.launch_extents()
    need, rects = ext["need_rows"].astype(np.int64), ext["rects"].astype(np.int64)
    short = np.nonzero(need < p.job_reads)[0]
    assert not short.size, (f"{p.what}: job {int(short[0])} records need-rows {int(need[short[0]])}, its pixels read rows up to "
                            f"{int(p.job_reads[short[0]])}")
    b = p.job_bounds
    outside = np.nonzero((b[:, 0] < rects[:, 0]) | (b[:, 1] < rects[:, 1]) | (b[:, 2] > rects[:, 2]) | (b[:, 3] > rects[:, 3]))[0]
    if outside.size:
        j = int(outside[0])
        raise AssertionError(f"{p.what}: job {j} writes the pixels of {b[j].tolist()}, outside its rect {rects[j].tolist()}")


# ---- the plans --------------------------------------------------------------------------------------------------------
def context_plane(ov, inp, out, plane, what):
    case = dict(ov=ov, inp=inp, out=out)
    iw, ih, ow, oh, _ = plane_dims(case, plane)
    return Plane(t360.HostPlan(t360.make_context(**ov), iw, ih, ow, oh), iw, ih, what)


def warp_plane(ctx_ov, m, in_w, in_h, what):
    return Plane(t360.HostPlan.from_warp(t360.make_context(**ctx_ov), m, in_w, in_h, WRAP), in_w, in_h, what)


def _named_planes():
    out = [(f"small:{n}:{p}", ("small", n, p)) for n in sorted(SMALL) for p in (0, 1)]
    out += [(f"full:{n}:{p}", ("full", n, p)) for n in ("cfg2", "cfg3", "cfg4") for p in (0, 1)]
    return out


NAMED = _named_planes()


def random_contexts():
    """The contexts of tests/test_gather_plan.py's random sweep (same seed): every layout in both directions, stereo,
    rotation, off-centre with NaN map entries, scale factors, odd sizes."""
    from tests.test_host_plan import _random_context
    rng = np.random.default_rng(500)
    out = []
    for _ in range(30):
        ov = _random_context(rng)
        iw, ih = int(rng.integers(200, 700)) * 2, int(rng.integers(100, 300)) * 2
        ow, oh = int(rng.integers(40, 200)) * 2 + int(rng.random() < 0.3), int(rng.integers(30, 150)) * 2 + int(rng.random() < 0.3)
        if rng.random() < 0.5:
            iw = (iw + 15) // 16 * 16
        out.append((ov, (iw, ih), (ow, oh), int(rng.integers(0, 2))))
    return out


def warp_planes():
    from tests.test_warp_map import FAMILIES, _sizes
    for family in sorted(FAMILIES):
        for interp in (t360.LINEAR, t360.CUBIC, t360.LANCZOS4):
            mw, mh, iw, ih = _sizes(family, {t360.LINEAR: 2, t360.CUBIC: 4, t360.LANCZOS4: 8}[interp])
            yield warp_plane(dict(interpolation_alg=interp, enable_low_pass_filter=0), FAMILIES[family](mw, mh, iw, ih), iw, ih,
                             f"warp:{family}:{interp}")


def view_planes():
    """Plans of rectilinear_map and camera_map views installed as warp maps (BORDER_WRAP)."""
    for name, ov in (("equirect", dict(input_layout=t360.LAYOUT_EQUIRECT)),
                     ("tb_to_lr", dict(input_layout=t360.LAYOUT_EQUIRECT, input_stereo_format=t360.STEREO_FORMAT_TB,
                                       output_stereo_format=t360.STEREO_FORMAT_LR)),
                     ("cubemap_32", dict(input_layout=t360.LAYOUT_CUBEMAP_32))):
        for interp in (t360.CUBIC, t360.LANCZOS4):
            ctx_ov = dict(ov, interpolation_alg=interp, enable_low_pass_filter=0)
            ctx = t360.make_context(**ctx_ov)
            iw, ih = (1536, 1024) if name == "cubemap_32" else (2048, 1024)
            m = t360.rectilinear_map(ctx, (30.0, 60.0, 10.0, 120.0, 80.0), iw, ih, 640, 360)
            yield warp_plane(ctx_ov, m, iw, ih, f"rectilinear:{name}:{interp}")
            for cam in ((T360_CAMERA_EQUIDISTANT, 0.0), (T360_CAMERA_PANNINI, 0.7)):
                m = t360.camera_map(ctx, (-40.0, -75.0, 0.0, 170.0, 120.0), cam, iw, ih, 480, 320)
                yield warp_plane(ctx_ov, m, iw, ih, f"camera:{name}:{interp}:{cam[0]}")


def check_plane(p: Plane) -> int:
    """Extents and schedule for every chunk count of the path; returns the launch jobs checked (0: the plan takes the
    plain path, it has no launch list)."""
    if not p.jobs:
        return 0
    check_extents(p)
    for chunks in range(2, 9):
        check_schedule(p, p.schedule(chunks))
    return p.jobs


# ---- CPU: invariants ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("what,key", NAMED, ids=[n for n, _ in NAMED])
def test_schedule_of_named_planes(what, key):
    group, name, plane = key
    case = (SMALL if group == "small" else FULL)[name]
    p = context_plane(case["ov"], case["inp"], case["out"], plane, what)
    n = check_plane(p)
    staged = p.hp.kernel_size >= 2 and t360.make_context(**case["ov"]).output_layout not in (t360.LAYOUT_BARREL, t360.LAYOUT_BARREL_SPLIT)
    assert (n > 0) == staged


def test_schedule_of_random_contexts():
    checked = 0
    for i, (ov, inp, out, plane) in enumerate(random_contexts()):
        try:
            p = context_plane(ov, inp, out, plane, f"random {i}")
        except ValueError:  # the planner refuses what the reference refuses
            continue
        checked += check_plane(p) > 0
    assert checked >= 15, checked


def test_schedule_of_warp_maps():
    ks = set()
    for p in warp_planes():
        if check_plane(p):
            ks.add(p.hp.kernel_size)
    assert ks == {2, 4, 8}


def test_schedule_of_rectilinear_and_camera_views():
    assert sum(check_plane(p) > 0 for p in view_planes()) == 18


def test_chunk_rule_and_default_schedule():
    """waves() without a chunk count takes the call's rule: one chunk per 3 MiB of input, 2 to 8."""
    for (iw, ih), want in (((832, 416), 2), ((4096, 2048), 2), ((4608, 2304), 3), ((5120, 2560), 4), ((5760, 2881), 5),
                           ((7680, 3840), 8), ((15360, 7680), 8)):
        hp = t360.HostPlan(t360.make_context(interpolation_alg=t360.LINEAR, enable_low_pass_filter=0), iw, ih, 96, 64)
        assert hp.waves()["chunks"] == want, (iw, ih)


# ---- CPU: the checker catches what it is meant to catch ----------------------------------------------------------------
def mutation_plane():
    return gpu_plane("eq5120_cube_cubic_rot")


def with_waves(s, wave):
    """s with the launch jobs regrouped into the waves `wave` (launch order inside each)."""
    order = np.concatenate([np.nonzero(wave == c)[0] for c in range(s["chunks"])]).astype(np.int32)
    starts = np.concatenate([[0], np.cumsum(np.bincount(wave, minlength=s["chunks"]))]).astype(np.int32)
    return dict(s, order=order, wave_start=starts)


def test_checker_names_a_job_moved_one_wave_later():
    p = mutation_plane()
    s = p.schedule(4)
    wave = job_waves(s)
    copy_wave = np.zeros(p.hp.map_h, np.int64)
    for c, _, y0, _, y1 in s["rects"]:
        copy_wave[y0:y1] = c
    last_writer = [j for j in range(p.jobs) if wave[j] + 1 < s["chunks"] and (copy_wave[p.writer_rows[j]] == wave[j]).any()]
    j = last_writer[len(last_writer) // 2]
    moved = wave.copy()
    moved[j] += 1
    bad = with_waves(s, moved)
    check_schedule(p, with_waves(s, wave))
    with pytest.raises(AssertionError, match=rf"job {j} writes row \d+ in wave {int(wave[j]) + 1}"):
        check_schedule(p, bad)


def test_checker_names_a_band_copied_one_wave_early():
    p = mutation_plane()
    s = p.schedule(4)
    i = next(i for i, r in enumerate(s["rects"]) if r[0] > 0)
    bad = dict(s, rects=s["rects"].copy())
    bad["rects"][i, 0] -= 1
    y0, y1 = int(s["rects"][i][2]), int(s["rects"][i][4])
    with pytest.raises(AssertionError, match=rf"band rows {y0}-{y1} is copied back after wave {int(s['rects'][i][0]) - 1}"):
        check_schedule(p, bad)


def test_checker_names_a_job_one_need_row_short():
    """A need-row one short on a job whose last window row is that row, at a chunk boundary: the product's schedule for
    the corrupted need-rows runs the job a wave early, and the checker names it."""
    p = mutation_plane()
    need = p.hp.launch_extents()["need_rows"]
    for chunks in range(2, 9):
        ends = p.schedule(chunks)["chunk_row_end"]
        hit = np.nonzero(np.isin(need - 1, ends[:-1]) & (p.job_reads == need))[0]
        if hit.size:
            break
    assert hit.size, "no job ends one row past a chunk boundary"
    j = int(hit[0])
    check_schedule(p, p.schedule(chunks))
    bad = need.copy()
    bad[j] -= 1
    with pytest.raises(AssertionError, match=rf"job {j} runs in wave"):
        check_schedule(p, p.schedule(chunks, bad))


# ---- the GPU cases, and what they reach -------------------------------------------------------------------------------
EQ, CUBE, EAC = t360.LAYOUT_EQUIRECT, t360.LAYOUT_CUBEMAP_32, t360.LAYOUT_EAC_32
NO_LP = dict(enable_low_pass_filter=0)
# name -> (context overrides, luma input, luma output) or, for a warp map, ("warp", interpolation, input, map size)
PLANES = {
    "eq4096_cube_linear": (dict(NO_LP, interpolation_alg=t360.LINEAR), (4096, 2048), (1536, 1024)),
    "eq4608_eac_lanczos": (dict(NO_LP, interpolation_alg=t360.LANCZOS4, output_layout=EAC), (4608, 2304), (1536, 1024)),
    "eq5120_cube_cubic_rot": (dict(NO_LP, interpolation_alg=t360.CUBIC, fixed_yaw=30.0, fixed_pitch=20.0), (5120, 2560), (1920, 1280)),
    "eq5760_odd_eac_cubic": (dict(NO_LP, interpolation_alg=t360.CUBIC, output_layout=EAC), (5760, 2881), (1536, 1024)),
    "eq7680_tb_cube_cubic": (dict(NO_LP, interpolation_alg=t360.CUBIC, input_stereo_format=t360.STEREO_FORMAT_TB,
                                  output_stereo_format=t360.STEREO_FORMAT_TB), (7680, 3840), (1536, 2048)),
    "cube4608_eq_cubic": (dict(NO_LP, interpolation_alg=t360.CUBIC, input_layout=CUBE, output_layout=EQ), (4608, 3072), (2048, 1024)),
    "dual_fisheye_wrap": ("warp", t360.CUBIC, (5760, 2880), (2048, 1024)),
    # a narrow view of the equator: every job reads the middle chunk, the first and the last wave have no jobs
    "eq4608_flat_cubic": (dict(NO_LP, interpolation_alg=t360.CUBIC, output_layout=t360.LAYOUT_FLAT_FIXED, fixed_hfov=60.0,
                               fixed_vfov=34.0), (4608, 2304), (1280, 720)),
}
STATIC_CLAIMS = {2: 132 * 3 * 2, 4: 132 * 3 * 2, 8: 132 * 2 * 2}  # a 132-SM H100: SMs x groups x two jobs per producer


@functools.lru_cache(maxsize=None)
def dual_fisheye_map(in_w, in_h, mw, mh):
    from tests.test_warp_map import dual_fisheye
    return dual_fisheye(mw, mh, in_w, in_h)


@functools.lru_cache(maxsize=None)
def gpu_plane(name, plan_index=0) -> Plane:
    spec = PLANES[name]
    if spec[0] == "warp":
        _, interp, (iw, ih), (mw, mh) = spec
        return warp_plane(dict(NO_LP, interpolation_alg=interp), dual_fisheye_map(iw, ih, mw, mh), iw, ih, name)
    ov, inp, out = spec
    return context_plane(ov, inp, out, plan_index, f"{name}:{plan_index}")


def ledger(names) -> dict:
    seen = dict(chunks=set(), empty_wave=0, short_wave=0, border_last=0, band_last=0)
    for name in names:
        p = gpu_plane(name)
        s = p.schedule()
        launch = p.hp.pole_caps()["launch"]
        sizes = np.diff(s["wave_start"])
        last = s["chunks"] - 1
        seen["chunks"].add(s["chunks"])
        seen["empty_wave"] += int((sizes == 0).any())
        seen["short_wave"] += int(((sizes > 0) & (sizes < STATIC_CLAIMS[p.hp.kernel_size])).any())
        kinds = (launch[:, 1] >> KIND_SHIFT) & 15
        border = np.nonzero(kinds == BORDER)[0]
        seen["border_last"] += int(border.size > 0 and (job_waves(s)[border] == last).any())
        seen["band_last"] += int((s["rects"][:, 0] == last).any())
    return seen


def test_gpu_cases_reach_every_schedule_shape():
    """The planes of the GPU tests below reach chunk counts 2, 3, 4, 5 and 8 with the default threshold, a wave with no
    jobs, a wave with fewer jobs than one launch's static claims, border jobs that wrap vertically and so wait for the
    last chunk, and a band that completes only in the last wave."""
    names = sorted(PLANES)
    for name in names:
        check_plane(gpu_plane(name))
        p = gpu_plane(name)
        assert p.in_w * p.in_h >= MIN_BYTES, name
    seen = ledger(names)
    assert {2, 3, 4, 5, 8} <= seen["chunks"], seen
    assert seen["empty_wave"] and seen["short_wave"] and seen["border_last"] and seen["band_last"], seen


# ---- GPU ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests must run on an H100 (there is no CPU fallback to test)")
    return torch


SENTINEL = 0x5A


def nonempty_waves(p: Plane) -> int:
    return int((np.diff(p.schedule()["wave_start"]) > 0).sum())


class HostBuffers:
    """A caller's input and output plane with pitches wider than the planes: pageable (numpy) or page-locked (torch), the
    output padding holding SENTINEL."""

    def __init__(self, torch, iw, ih, ow, oh, pinned):
        self.iw, self.ih, self.ow, self.oh = iw, ih, ow, oh
        in_pitch, out_pitch = iw + 5, ow + 3
        if pinned:
            self._in = torch.empty((ih, in_pitch), dtype=torch.uint8, pin_memory=True)
            self._out = torch.empty((oh, out_pitch), dtype=torch.uint8, pin_memory=True)
            self.src, self.dst = self._in.numpy(), self._out.numpy()
        else:
            self.src, self.dst = np.empty((ih, in_pitch), np.uint8), np.empty((oh, out_pitch), np.uint8)

    def fill(self, src):
        self.src[:, :self.iw] = src
        self.src[:, self.iw:] = 0x33
        self.dst[...] = SENTINEL

    def call(self, vft, plan_index, image_plane):
        assert vft.transformFramePlane(self.src.ctypes.data, self.dst.ctypes.data, self.iw, self.ih, self.src.strides[0], self.ow,
                                       self.oh, self.dst.strides[0], plan_index, image_plane)

    def check(self, want, what):
        got = self.dst[:, :self.ow]
        assert np.array_equal(got, want), f"{what}: {int((got != want).sum())} px differ from the oracle"
        assert (self.dst[:, self.ow:] == SENTINEL).all(), f"{what}: the output padding was written"


def _transform(monkeypatch, strict, min_bytes=None):
    monkeypatch.setenv("T360B200_PIPELINE_STRICT", "1" if strict else "0")
    if min_bytes is not None:
        monkeypatch.setenv("T360B200_PIPELINE_MIN_BYTES", str(min_bytes))
    else:
        monkeypatch.delenv("T360B200_PIPELINE_MIN_BYTES", raising=False)


class Oracle:
    def __init__(self, name, plan_index=0):
        spec = PLANES[name]
        self.warp = spec[0] == "warp"
        if self.warp:
            _, self.interp, (iw, ih), (mw, mh) = spec
            self.map = dual_fisheye_map(iw, ih, mw, mh)
            self.dims = (iw, ih, mw, mh)
        else:
            ov, inp, out = spec
            iw, ih, ow, oh, _ = plane_dims(dict(ov=ov, inp=inp, out=out), plan_index)
            self.octx = rh.default_context(**ov)
            self.plan = co.OraclePlan(self.octx, iw, ih, ow, oh)
            self.dims, self.index = (iw, ih, ow, oh), plan_index

    def __call__(self, src):
        if self.warp:
            from tests.test_warp_map import _oracle
            return _oracle(src, self.map, self.interp, WRAP, 0, self.map.shape[1], self.map.shape[0])
        return co.transform_plane(self.octx, self.plan, src, self.dims[2], self.dims[3], map_index=self.index)


def _install(vft, name, plan_index=0):
    spec = PLANES[name]
    if spec[0] == "warp":
        _, _, (iw, ih), (mw, mh) = spec
        assert vft.generate_map_from_warp(dual_fisheye_map(iw, ih, mw, mh), iw, ih, plan_index)
    else:
        ov, inp, out = spec
        iw, ih, ow, oh, _ = plane_dims(dict(ov=ov, inp=inp, out=out), plan_index)
        assert vft.generateMapForPlane(iw, ih, ow, oh, plan_index)


def _context(name):
    spec = PLANES[name]
    return t360.make_context(**(dict(NO_LP, interpolation_alg=spec[1]) if spec[0] == "warp" else spec[0]))


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True], ids=["free", "strict"])
@pytest.mark.parametrize("name", sorted(PLANES))
def test_streamed_planes_equal_the_oracle(name, strict, torch_cuda, monkeypatch):
    """One plane of each GPU case, pageable and page-locked, with caller pitches wider than the planes: two calls with
    new content each (page-locked: the first captures the graph, the second replays it), every pixel against the oracle,
    the output padding untouched, and one gather launch per non-empty wave of the exported schedule on every call."""
    torch = torch_cuda
    _transform(monkeypatch, strict)
    p, oracle = gpu_plane(name), Oracle(name)
    iw, ih, ow, oh = oracle.dims
    waves = nonempty_waves(p)
    with t360.VideoFrameTransform(_context(name)) as vft:
        _install(vft, name)
        for pinned in (False, True):
            buf = HostBuffers(torch, iw, ih, ow, oh, pinned)
            for frame in range(2):
                src = co.noise_plane(iw, ih, frame=10 * pinned + frame)
                buf.fill(src)
                n0 = t360.kernel_launch_count()
                buf.call(vft, 0, 0)
                assert t360.kernel_launch_count() - n0 == waves, f"{'page-locked' if pinned else 'pageable'} call {frame}: not streamed"
                buf.check(oracle(src), f"{name} {'page-locked' if pinned else 'pageable'} call {frame}")


SMALL_STREAMED = ["cube_cubic", "cube_linear", "cube_lanczos", "rotated", "eac_mono_cubic", "cube_to_equirect", "cube_cubic_odd"]


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True], ids=["free", "strict"])
@pytest.mark.parametrize("name", SMALL_STREAMED)
def test_streamed_small_planes(name, strict, torch_cuda, monkeypatch):
    """T360B200_PIPELINE_MIN_BYTES=0 sends small planes down the streamed path too (always 2 chunks): all three planes of
    a frame, two frames, pageable, caller pitches wider than the planes, same bytes as the oracle."""
    _transform(monkeypatch, strict, min_bytes=0)
    case = SMALL[name]
    ctx, octx = t360.make_context(**case["ov"]), rh.default_context(**case["ov"])
    with t360.VideoFrameTransform(ctx) as vft:
        for idx in (0, 1):
            iw, ih, ow, oh, _ = plane_dims(case, idx)
            assert vft.generateMapForPlane(iw, ih, ow, oh, idx)
        for plane in (0, 1, 2):
            iw, ih, ow, oh, idx = plane_dims(case, plane)
            plan = co.OraclePlan(octx, iw, ih, ow, oh)
            buf = HostBuffers(torch_cuda, iw, ih, ow, oh, pinned=False)
            for frame in (0, 1):
                src = co.noise_plane(iw, ih, plane=plane, frame=frame)
                buf.fill(src)
                buf.call(vft, idx, plane)
                buf.check(co.transform_plane(octx, plan, src, ow, oh, map_index=idx), f"{name} plane {plane} frame {frame}")


LRU_CASE = SMALL["cube_cubic"]


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True], ids=["free", "strict"])
def test_graph_cache_evicts_and_recaptures(strict, torch_cuda, monkeypatch):
    """A pool of 10 page-locked buffer pairs for each of a frame's 3 planes, rotated twice with new content every call: 30
    graphs for a cache of 24, so the second round evicts and captures again.  Every output against the oracle."""
    _transform(monkeypatch, strict, min_bytes=0)
    case = LRU_CASE
    ctx, octx = t360.make_context(**case["ov"]), rh.default_context(**case["ov"])
    with t360.VideoFrameTransform(ctx) as vft:
        for idx in (0, 1):
            assert vft.generateMapForPlane(*plane_dims(case, idx)[:4], idx)
        plans = [co.OraclePlan(octx, *plane_dims(case, idx)[:4]) for idx in (0, 1)]
        pool = [[HostBuffers(torch_cuda, *plane_dims(case, plane)[:4], pinned=True) for plane in range(3)] for _ in range(10)]
        for rnd in range(2):
            for i, bufs in enumerate(pool):
                for plane, buf in enumerate(bufs):
                    iw, ih, ow, oh, idx = plane_dims(case, plane)
                    src = co.noise_plane(iw, ih, plane=plane, frame=100 * rnd + i)
                    buf.fill(src)
                    buf.call(vft, idx, plane)
                    buf.check(co.transform_plane(octx, plans[idx], src, ow, oh, map_index=idx), f"round {rnd} buffers {i} plane {plane}")


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True], ids=["free", "strict"])
def test_staging_growth_drops_the_chroma_graph(strict, torch_cuda, monkeypatch):
    """Chroma first: its graph is captured with staging planes of the chroma size.  The luma call grows them, so the
    chroma graph is stale and must be captured again, not replayed, on the next chroma call (new content)."""
    _transform(monkeypatch, strict)
    name = "eq7680_tb_cube_cubic"
    ov, inp, out = PLANES[name]
    case = dict(ov=ov, inp=inp, out=out)
    dims = [plane_dims(case, idx)[:4] for idx in (0, 1)]
    assert dims[1][0] * dims[1][1] >= MIN_BYTES, "the chroma plane is streamed too"
    with t360.VideoFrameTransform(_context(name)) as vft:
        for idx in (0, 1):
            _install(vft, name, idx)
        oracles = [Oracle(name, idx) for idx in (0, 1)]
        bufs = [HostBuffers(torch_cuda, *dims[idx], pinned=True) for idx in (0, 1)]
        for step, idx in enumerate((1, 0, 1, 0)):
            src = co.noise_plane(*dims[idx][:2], plane=idx, frame=step)
            bufs[idx].fill(src)
            bufs[idx].call(vft, idx, idx)
            bufs[idx].check(oracles[idx](src), f"step {step} plan {idx}")


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True], ids=["free", "strict"])
def test_new_plan_with_the_same_buffers_is_not_replayed(strict, torch_cuda, monkeypatch):
    """generateMapForPlane, a warp map and generateMapForPlane again on plan index 0, each followed by two calls with the
    same page-locked buffers: each plan's first call captures its own graph (an old plan's graph would give the old
    geometry), its second replays it."""
    from tests.test_warp_map import _oracle
    _transform(monkeypatch, strict)
    name = "eq4096_cube_linear"
    ov, (iw, ih), (ow, oh) = PLANES[name]
    m = dual_fisheye_map(iw, ih, ow, oh)
    with t360.VideoFrameTransform(_context(name)) as vft:
        buf = HostBuffers(torch_cuda, iw, ih, ow, oh, pinned=True)
        plain = Oracle(name)
        for step, warp in enumerate((False, True, False)):
            if warp:
                assert vft.generate_map_from_warp(m, iw, ih, 0)
            else:
                assert vft.generateMapForPlane(iw, ih, ow, oh, 0)
            for call in range(2):
                src = co.noise_plane(iw, ih, frame=10 * step + call)
                want = _oracle(src, m, t360.LINEAR, WRAP, 0, ow, oh) if warp else plain(src)
                buf.fill(src)
                buf.call(vft, 0, 0)
                buf.check(want, f"plan {step} ({'warp map' if warp else 'context'}) call {call}")
