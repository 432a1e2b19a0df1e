"""The two float32 kernels -- the segmented low-pass and the INTER_AREA resize -- at every job shape and ratio class they
have, on the device against the oracle, and the oracle against cv2 and a float64 model.

The low-pass runs as strip jobs (blurFrameStripKernel<HY, MULTI>: a 12-register horizontal ring with straight-line code
for 1-3 chunks of 4 taps and a loop for 4 and more, interior strips reading aligned words through a funnel shift and edge
strips replicating bytes, lanes with fewer than 8 columns, an 8-byte store only where destination, pitch and column are
8-aligned, HY = 0 padded to 3 vertical taps), tile jobs and direct jobs.  The resize takes the 2 x 2 fast path, the other
integer cells, the table of fractional ratios (which also catches ratios whose double quotient misses an integer) or, when
an axis enlarges, OpenCV's bilinear "area mode".  Those kernels are bit-exact only because they follow the oracle's order of
operations, so a wrong ring slot, funnel shift or rounding shows as a few differing pixels at the shapes that reach it.

The ledger below plans the cases of the GPU tests on the host and lists the classes their job lists and size pairs reach,
so that a case removed from the sweep, or a planner change that stops producing a class, fails here, on a CPU, naming it.
"""
from __future__ import annotations

import functools
import math
import sys

import numpy as np
import pytest

import transform360_b200 as t360
from oracle import c_oracle as co
from oracle import ref_harness as rh
from transform360_b200.stream import FrameTransformer, StreamSpec

STRIP_W, LANE_PX, PLANE_SHIFT = 256, 8, 8  # kernels.cuh: kStripW, kStripLanePx, kStripPlaneShift
PAD = 0xCD


def chroma(dim):
    return (dim[0] + 1) >> 1, (dim[1] + 1) >> 1


# ---- the low-pass sweep -----------------------------------------------------------------------------------------------
def _pinned(x, nv, **more):
    """Vertical kernel pinned to int(2 * 0.5x) * 2 + 1 taps in every band (min = max half height, no per-tile adjustment):
    the horizontal kernel grows as sigma / cos(latitude) towards the poles, through every chunk count."""
    return dict(dict(interpolation_alg=t360.LINEAR, min_kernel_half_height=x, max_kernel_half_height=x, adjust_kernel=0,
                     num_vertical_segments=nv), **more)


# name: (context overrides, luma in, luma out, another plane size for the stage alone or None, planes of the frame call)
LOW_PASS = {
    # vertical half-size 0 (one tap padded to {0, k, 0}); 800 = 3 strips + 32 columns
    "hy0": (_pinned(0.8, 62), (800, 200), (768, 512), (803, 197), 3),
    # half-size 1 on an odd width (3 strips + 235 columns)
    "hy1": (_pinned(1.5, 45), (1003, 220), (960, 640), (1029, 211), 2),
    # half-size 2: 773 = 3 strips + 5 columns (lanes with fewer than 8 columns, a job narrower than 8)
    "hy2": (_pinned(2.5, 37), (773, 460), (768, 512), (767, 459), 1),
    # half-size 3 on a whole number of strips
    "hy3": (_pinned(3.5, 25), (1024, 240), (960, 640), (1021, 250), 3),
    # half-size 3 on a plane a single strip wide, and 2 strips + 9 columns
    "hy3_narrow": (_pinned(3.7, 25, interpolation_alg=t360.CUBIC), (265, 150), (384, 256), (200, 150), 3),
    # half-size 1 and 2 per tile (off-centre, adjusted kernels): segments of 125 / 126 columns, not multiples of 8
    "offcentre": (dict(interpolation_alg=t360.CUBIC, fixed_cube_offcenter_z=-0.3, fixed_cube_offcenter_x=0.1,
                       num_horizontal_segments=6, num_vertical_segments=9), (751, 300), (576, 384), (640, 300), 3),
    # segments of 240 columns: interior jobs narrower than a strip, a multiple of 8 wide
    "offcentre_mul8": (dict(interpolation_alg=t360.LINEAR, fixed_cube_offcenter_z=-0.3, num_vertical_segments=5,
                            num_horizontal_segments=5), (1200, 240), (768, 512), None, 1),
    # stereo: the segments applied to both halves
    "lr_stereo": (dict(interpolation_alg=t360.CUBIC, input_stereo_format=t360.STEREO_FORMAT_LR, output_stereo_format=t360.STEREO_FORMAT_LR,
                       num_vertical_segments=5, num_horizontal_segments=2, min_kernel_half_height=1.2), (1030, 256), (768, 256), None, 3),
    "tb_stereo": (dict(interpolation_alg=t360.LINEAR, input_stereo_format=t360.STEREO_FORMAT_TB, output_stereo_format=t360.STEREO_FORMAT_TB,
                       output_layout=t360.LAYOUT_EAC_32, num_vertical_segments=9, num_horizontal_segments=3), (600, 602), (576, 768), None, 3),
    # vertical half-size above 3: tile jobs (and a frame whose planes are not merged)
    "tiles": (dict(interpolation_alg=t360.CUBIC, num_vertical_segments=41, num_horizontal_segments=3, min_kernel_half_height=4.5),
              (800, 400), (576, 384), (803, 397), 3),
    # kernels too large for a shared-memory tile: direct jobs
    "direct": (dict(interpolation_alg=t360.CUBIC, num_vertical_segments=300, num_horizontal_segments=1, adjust_kernel=0,
                    min_kernel_half_height=40.0), (640, 320), (480, 320), None, 1),
}

STRIP_HY = (0, 1, 2, 3)
CHUNKS = (1, 2, 3, "4+0", "4+1", "4+2")  # >= 4 chunks by kxChunks % 3: where the loop leaves the ring
WIDTHS = ("256", "mul8", "ragged", "lt8")
HEIGHTS = ("full", "tail")
# The strip classes are (hy, chunks, edge, width, height).  The full product (384) would take hundreds of planes; what the
# kernel's branches depend on jointly is required pairwise: the vertical ring with the horizontal one, the reader (edge or
# interior) with the ring loop and with the store, and the row pipeline with the row budget.
STRIP_PATTERNS = ([(hy, c, None, None, None) for hy in STRIP_HY for c in CHUNKS]
                  + [(None, c, e, None, None) for c in CHUNKS for e in (0, 1)]
                  + [(None, None, e, w, None) for e in (0, 1) for w in WIDTHS]
                  + [(hy, None, None, None, h) for hy in STRIP_HY for h in HEIGHTS]
                  + [(None, c, None, None, h) for c in CHUNKS for h in HEIGHTS])
UNREACHABLE = {
    (2, 1, None, None, None): "the horizontal sigma is sigma_y / cos(latitude) (or half the plane width): 5 vertical taps "
                              "come with at least 5 horizontal ones, 2 chunks, on planes wider than 2 pixels",
    (3, 1, None, None, None): "likewise 7 vertical taps come with at least 7 horizontal ones, 2 chunks",
}
JOB_CLASSES = ("tile", "direct", "merged2", "merged3", "per_plane3", "stereo_lr", "stereo_tb", "one_strip_plane")


def strip_class(pattern) -> str:
    names = ("hy", "chunks", "edge", "width", "height")
    return ", ".join(f"{n}={v}" for n, v in zip(names, pattern) if v is not None)


def row_budget(plane_w, plane_h, chunks):
    """lowpass_jobs.cpp: rows per strip job for a plane size and a horizontal chunk count."""
    wanted = plane_h * ((plane_w + STRIP_W - 1) // STRIP_W) // 5000
    rows = 32 if wanted >= 32 else (16 if wanted >= 16 else 8)
    return min(rows, 32 if chunks <= 3 else (16 if chunks <= 8 else 8))


def strip_classes(lists, sizes):
    """(hy, chunks, edge, width, height) of every strip job of a job list; sizes: plane size of each plane tag."""
    taps, out = lists["taps"], set()
    for c, strips in enumerate(lists["strips"]):
        for x0, y0, w, h, kxo, chunks, kxc, kyo, edge in (tuple(int(v) for v in r) for r in strips):
            hy = 0 if c == 0 and taps[kyo] == 0 and taps[kyo + 2] == 0 else c + 1
            cc = chunks if chunks <= 3 else f"4+{chunks % 3}"
            wc = "256" if w == STRIP_W else ("lt8" if w < LANE_PX else ("mul8" if w % LANE_PX == 0 else "ragged"))
            hc = "full" if h == row_budget(*sizes[edge >> PLANE_SHIFT], chunks) else "tail"
            out.add((hy, cc, edge & 1, wc, hc))
    return out


def matches(pattern, cls):
    return all(p is None or p == c for p, c in zip(pattern, cls))


@functools.lru_cache(maxsize=None)
def _plans(name):
    """(luma plan, chroma plan or None for a frame of one plane)"""
    ov, inp, out, _, planes = LOW_PASS[name]
    ctx = t360.make_context(**ov)
    return t360.HostPlan(ctx, *inp, *out), t360.HostPlan(ctx, *chroma(inp), *chroma(out)) if planes > 1 else None


@functools.lru_cache(maxsize=None)
def low_pass_ledger(names):
    """strip classes -> cases, and whole-job classes -> cases, of the job lists the GPU tests of these cases run: the luma
    plane alone at its size and the other size, every plane of the frame call, and its merged list."""
    strips, jobs = {}, {}
    for name in names:
        ov, inp, _, other, planes = LOW_PASS[name]
        stereo = {t360.STEREO_FORMAT_LR: "stereo_lr", t360.STEREO_FORMAT_TB: "stereo_tb"}.get(ov.get("input_stereo_format"))
        if stereo:  # (the segments applied to both halves)
            jobs.setdefault(stereo, set()).add(name)
        luma, chro = _plans(name)
        lists = [(luma.blur_lists(), [inp])] + ([(chro.blur_lists(), [chroma(inp)])] if chro else [])
        if other:
            lists.append((luma.blur_lists(width=other[0], height=other[1]), [other]))
        if planes > 1:
            merged = luma.blur_lists(*[chro] * (planes - 1))
            if sum(len(s) for s in merged["strips"]):
                tags = {int(r[8]) >> PLANE_SHIFT for s in merged["strips"] for r in s}
                jobs.setdefault(f"merged{len(tags)}", set()).add(name)
            lists.append((merged, [inp] + [chroma(inp)] * (planes - 1)))
            if planes == 3 and any(len(l[k]) for l, _ in lists[:2] for k in ("tiles", "direct")):
                jobs.setdefault("per_plane3", set()).add(name)  # (not mergeable: one launch set per plane)
        for l, sizes in lists:
            for cls in strip_classes(l, sizes):
                strips.setdefault(cls, set()).add(name)
            if sum(len(s) for s in l["strips"]) and min(w for w, _ in sizes) <= STRIP_W:
                jobs.setdefault("one_strip_plane", set()).add(name)  # (every strip both a left and a right edge)
            for kind, key in (("tile", "tiles"), ("direct", "direct")):
                if len(l[key]):
                    jobs.setdefault(kind, set()).add(name)
    return strips, jobs


def low_pass_missing(names):
    strips, jobs = low_pass_ledger(tuple(names))
    missing = [strip_class(p) for p in STRIP_PATTERNS if p not in UNREACHABLE and not any(matches(p, c) for c in strips)]
    return missing + [k for k in JOB_CLASSES if k not in jobs]


# ---- the resize sweep -------------------------------------------------------------------------------------------------
def near_integer_ratio():
    """(n, d): a shrink by the integer n whose double quotient 1 / (d / (n * d)) misses n by DBL_EPSILON or more, so that
    buildAreaResize takes the table path for integer cells (smallest n * d)."""
    found = [(n * d, n, d) for n in range(2, 100) for d in range(1, 8)
             if abs(1.0 / (d / (n * d)) - n) >= sys.float_info.epsilon]
    _, n, d = min(found)
    return n, d


NEAR_N, NEAR_D = near_integer_ratio()
# (map size, requested output size) pairs, luma; the whole-frame call adds the chroma pairs
RESIZE = [
    ((160, 96), (80, 48)),      # 2 x 2
    ((162, 96), (54, 32)),      # 3 x 3
    ((150, 96), (150, 24)),     # 1 x 4, width unchanged
    ((160, 70), (32, 70)),      # 5 x 1, height unchanged
    ((120, 96), (100, 80)),     # fractional both ways: 6 / 5, weights in 36ths (exact .5 sums, rounded as float32 ones)
    ((160, 97), (80, 61)),      # integer 2 across, fractional down
    ((NEAR_N * NEAR_D, 40), (NEAR_D, 20)),  # n x 2 with a quotient that misses n: the table
    ((97, 61), (160, 99)),      # enlarging both ways
    ((97, 200), (160, 51)),     # enlarging across, shrinking down
    ((200, 64), (120, 101)),    # shrinking across, enlarging down
    ((130, 90), (61, 1)),       # one output row: fractional across, 90 down
]  # (the one output column: the near-integer pair)
RESIZE_CLASSES = ("2x2", "int_square", "1xn", "nx1", "table_both", "table_int_x", "table_int_y", "near_integer",
                  "enlarge_both", "enlarge_x_shrink_y", "shrink_x_enlarge_y", "unchanged_x", "unchanged_y", "one_row", "one_col")


def resize_classes(src, dst):
    """The branches buildAreaResize (sampling.cpp) takes for a map of size src requested at size dst."""
    (sw, sh), (dw, dh) = src, dst
    out = set()
    if dh == 1:
        out.add("one_row")
    if dw == 1:
        out.add("one_col")
    if src == dst:
        return out
    if sw == dw:
        out.add("unchanged_x")
    if sh == dh:
        out.add("unchanged_y")
    sx, sy = 1.0 / (dw / sw), 1.0 / (dh / sh)
    if sx < 1.0 or sy < 1.0:
        out.add("enlarge_both" if sx < 1.0 and sy < 1.0 else "enlarge_x_shrink_y" if sx < 1.0 and sy > 1.0
                else "shrink_x_enlarge_y" if sy < 1.0 and sx > 1.0 else "enlarge_one")
        return out
    ix, iy = round(sx), round(sy)  # (lrint: only ties could differ, and they are not integers)
    exact_x, exact_y = abs(sx - ix) < sys.float_info.epsilon, abs(sy - iy) < sys.float_info.epsilon
    if exact_x and exact_y:
        out.add("2x2" if (ix, iy) == (2, 2) else "1xn" if ix == 1 else "nx1" if iy == 1 else "int_square" if ix == iy else "int_cells")
    elif sw % dw == 0 and sh % dh == 0:
        out.add("near_integer")
    elif exact_x or exact_y:
        out.add("table_int_x" if exact_x else "table_int_y")
    else:
        out.add("table_both")
    return out


def resize_pairs(pairs):
    """Every (map size, output size) pair the GPU tests run: each luma pair and its chroma pair."""
    return [q for src, dst in pairs for q in ((src, dst), (chroma(src), chroma(dst)))]


def resize_missing(pairs):
    seen = set().union(*[resize_classes(*q) for q in resize_pairs(pairs)]) if pairs else set()
    return [c for c in RESIZE_CLASSES if c not in seen]


# ---- CPU: the ledger --------------------------------------------------------------------------------------------------
def test_low_pass_sweep_reaches_every_class():
    missing = low_pass_missing(sorted(LOW_PASS))
    assert not missing, f"the low-pass sweep reaches no strip job of class {missing}: those kernel paths go untested"


def test_unreachable_low_pass_classes_are_not_produced():
    strips, _ = low_pass_ledger(tuple(sorted(LOW_PASS)))
    made = [strip_class(p) for p in UNREACHABLE if any(matches(p, c) for c in strips)]
    assert not made, f"classes listed as unreachable are produced: {made}"


@pytest.mark.parametrize("name", sorted(LOW_PASS))
def test_every_low_pass_case_is_needed(name):
    """Each case reaches a class no other case does, so a case removed from the sweep fails the ledger."""
    missing = low_pass_missing(sorted(set(LOW_PASS) - {name}))
    assert missing, f"{name} reaches no class of its own"


def test_resize_sweep_reaches_every_class():
    missing = resize_missing(RESIZE)
    assert not missing, f"the resize sweep reaches no size pair of class {missing}: those kernel paths go untested"


@pytest.mark.parametrize("i", range(len(RESIZE)))
def test_every_resize_pair_is_needed(i):
    missing = resize_missing(RESIZE[:i] + RESIZE[i + 1:])
    assert missing, f"resize pair {RESIZE[i]} reaches no class of its own"


def test_near_integer_ratio_takes_the_table():
    n, d = NEAR_N, NEAR_D
    assert 1.0 / (d / (n * d)) != n and resize_classes((n * d, 2), (d, 1)) >= {"near_integer"}
    assert resize_classes((98, 2), (1, 1)) >= {"near_integer"}, "sw = 49 * dw: 1 / (1 / 49) is not 49.0"


# ---- CPU: the oracle against cv2 and float64 models ---------------------------------------------------------------------
def _noise(w, h, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w), dtype=np.uint8)


@pytest.mark.parametrize("pair", resize_pairs(RESIZE), ids=str)
def test_resize_pairs_oracle_vs_cv2(pair):
    cv2 = pytest.importorskip("cv2")
    (sw, sh), (dw, dh) = pair
    src = _noise(sw, sh, sw * 31 + dh)
    assert np.array_equal(co.resize_area(src, dw, dh), cv2.resize(src, (dw, dh), interpolation=cv2.INTER_AREA))


def _box_weights(s, d):
    """[d][s]: the share of source pixel i in output cell j of an axis shrunk from s to d (exact area overlap)."""
    scale = s / d
    j = np.arange(d)[:, None]
    i = np.arange(s)[None, :]
    lo, hi = j * scale, np.minimum((j + 1) * scale, s)
    return np.clip(np.minimum(i + 1, hi) - np.maximum(i, lo), 0, None) / (hi - lo)


def _linear_weights(s, d):
    """[d][s]: OpenCV's bilinear "area mode" weights in float64: source pixel floor(j * scale) and the next, the next one
    weighted by the (fractional) part of output cell j beyond their boundary, clamped at the last pixel.  The scale is
    1 / (d / s) as cv::resize computes it: where j * scale lands next to an integer, that double decides the pixel."""
    scale, w = 1.0 / (d / s), np.zeros((d, s))
    for j in range(d):
        i = math.floor(j * scale)
        f = (j + 1) - (i + 1) * (d / s)
        f = 0.0 if f <= 0 else f - math.floor(f)
        if i + 1 >= s:
            i, f = min(i, s - 1), 0.0
        w[j, i] += 1 - f
        if f:
            w[j, i + 1] += f
    return w


def resize_model(src, dw, dh):
    """float64 INTER_AREA: the box average when both axes shrink (rounded half up on 2 x 2 cells, as the integer fast path
    does, else half to even), the area-mode bilinear when an axis enlarges."""
    sh, sw = src.shape
    if dw <= sw and dh <= sh:
        v = _box_weights(sh, dh) @ src.astype(np.float64) @ _box_weights(sw, dw).T
        return np.floor(v + 0.5) if (sw, sh) == (2 * dw, 2 * dh) else np.rint(v)
    return np.rint(_linear_weights(sh, dh) @ src.astype(np.float64) @ _linear_weights(sw, dw).T)


# fraction of pixels at +-1 from the float64 model, observed on these noise planes
RESIZE_MODEL_BOUND = dict(shrink=0.04, enlarge=0.15)


def test_resize_oracle_vs_float64_model():
    """Every pair of the sweep, max |d| <= 1.  Shrinking: at most 4 % at +-1 (observed: none on integer cells, 0.18 to
    0.32 % on the table at 160 / 80 x 97 / 61, 3.3 % at 6 / 5 both ways, where one exact sum in 36 is a .5 that the float32
    weights and sums put on either side); enlarging: at most 15 % (observed: 7.3 to 13.2 %, the 11-bit weights and the
    truncating shifts of OpenCV's fixed-point bilinear kernel)."""
    worst = dict(shrink=0.0, enlarge=0.0)
    for (sw, sh), (dw, dh) in resize_pairs(RESIZE):
        src = _noise(sw, sh, sw + 7 * dh)
        got, want = co.resize_area(src, dw, dh).astype(int), resize_model(src, dw, dh)
        d = np.abs(got - want)
        assert d.max() <= 1, ((sw, sh), (dw, dh), d.max())
        kind = "shrink" if dw <= sw and dh <= sh else "enlarge"
        worst[kind] = max(worst[kind], float((d != 0).mean()))
    for kind, bound in RESIZE_MODEL_BOUND.items():
        assert worst[kind] <= bound, (kind, worst[kind])


def low_pass_model(ctx, src, segs):
    """float64 separable Gaussian with each segment's float32 taps, BORDER_REPLICATE against the plane, per fitting segment
    and stereo pass in plan order, rounded half to even; pixels under no segment are 0."""
    h, w = src.shape
    out = np.zeros((h, w))
    passes = [(0, 0)]
    if ctx.input_stereo_format == rh.STEREO_FORMAT_LR:
        passes.append((int(0.5 * w), 0))
    elif ctx.input_stereo_format == rh.STEREO_FORMAT_TB:
        passes.append((0, int(0.5 * h)))
    s64 = src.astype(np.float64)
    for ox, oy in passes:
        for left, top, sw, sh, kx, ky in segs:
            l, t = left + ox, top + oy
            if l < 0 or t < 0 or l + sw > w or t + sh > h:
                continue
            hx, hy = len(kx) // 2, len(ky) // 2
            rows = s64[np.clip(np.arange(t - hy, t + sh + hy), 0, h - 1)][:, np.clip(np.arange(l - hx, l + sw + hx), 0, w - 1)]
            r = sum(float(k) * rows[:, i:i + sw] for i, k in enumerate(kx))
            out[t:t + sh, l:l + sw] = sum(float(k) * r[i:i + sh] for i, k in enumerate(ky))
    return np.clip(np.rint(out), 0, 255)


LOW_PASS_MODEL_BOUND = 5e-5  # fraction of pixels at +-1 from the float64 model


@pytest.mark.parametrize("name", sorted(LOW_PASS))
def test_low_pass_oracle_vs_float64_model(name):
    """co.filter_plane on the luma plane of every case, at its size and the other size: max |d| <= 1, and at most 0.005 %
    of the pixels at +-1 (observed: 0 to 0.0025 %, float32 sums that land on the other side of a .5)."""
    ov, inp, out, other, _ = LOW_PASS[name]
    octx = rh.default_context(**ov)
    plan = co.OraclePlan(octx, *inp, *out)
    segs = co.plan_as_list(plan.segs, plan.nsegs, plan.taps)
    for w, h in [inp] + ([other] if other else []):
        src = co.noise_plane(w, h, frame=11)
        got = co.filter_plane(octx, src, plan.segs, plan.nsegs, plan.taps).astype(int)
        d = np.abs(got - low_pass_model(octx, src, segs))
        assert d.max() <= 1, (name, (w, h), d.max())
        assert (d != 0).mean() <= LOW_PASS_MODEL_BOUND, (name, (w, h), float((d != 0).mean()))


# ---- GPU --------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests must run on an H100 (there is no CPU fallback to test)")
    return torch


class Plane:
    """One device plane at base offset `off` with row pitch `pitch`; PAD in the row padding and around it."""

    def __init__(self, torch, w, h, off, pitch, content=None):
        self.w, self.h, self.off, self.pitch = w, h, off, pitch
        self.buf = torch.full((off + pitch * h + 64,), PAD, dtype=torch.uint8, device="cuda")
        if content is not None:
            self.rows()[:, :w] = torch.from_numpy(np.ascontiguousarray(content)).cuda()

    def rows(self):
        return self.buf[self.off:self.off + self.pitch * self.h].view(self.h, self.pitch)

    @property
    def ptr(self):
        return self.buf.data_ptr() + self.off

    def read(self):
        """(pixels, whether every byte outside them is still PAD)"""
        host = self.buf.cpu().numpy()
        rows = host[self.off:self.off + self.pitch * self.h].reshape(self.h, self.pitch)
        rest = np.concatenate([host[:self.off], rows[:, self.w:].ravel(), host[self.off + self.pitch * self.h:]])
        return rows[:, :self.w].copy(), bool((rest == PAD).all())


# base offset and pitch over the row width, in and out: odd (byte stores, funnel shifts) or 8-aligned (wide stores)
LAYOUTS = {"odd": ((3, 13), (5, 7)), "aligned8": ((8, 24), (16, 40))}


def _pitched(torch, src, layout, side):
    off, extra = LAYOUTS[layout][side]
    return Plane(torch, src.shape[1], src.shape[0], off, src.shape[1] + extra, src)


def _assert_plane(plane, want, what):
    got, pad_ok = plane.read()
    bad = got != want
    if bad.any():
        ys, xs = np.nonzero(bad)
        pytest.fail(f"{what}: {int(bad.sum())} px differ from the oracle (first at x {xs[0]} y {ys[0]}, max |d| "
                    f"{int(np.abs(got.astype(int) - want).max())})")
    assert pad_ok, f"{what}: bytes outside the plane were written"


@functools.lru_cache(maxsize=16)
def _oracle_plan(key, iw, ih, ow, oh):
    return co.OraclePlan(rh.default_context(**dict(key)), iw, ih, ow, oh)


def _oracle_frame(ov, spec, srcs, dims):
    """Every plane of a frame from the oracle: plans at the spec's sizes, outputs at dims' sizes."""
    key, out = tuple(sorted(ov.items())), []
    for p, src in enumerate(srcs):
        iw, ih, ow, oh, idx = spec.plane_dims(p)
        out.append(co.transform_plane(rh.default_context(**ov), _oracle_plan(key, iw, ih, ow, oh), src, dims[p][2], dims[p][3],
                                      map_index=idx))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(LOW_PASS))
def test_low_pass_cases_on_the_device(name, torch_cuda):
    """The stage alone (odd and 8-aligned bases and pitches, the planned size and another), the whole frame with the case's
    plane count, and the per-plane call: every output bit-exact against the oracle, padding untouched."""
    torch = torch_cuda
    if name == sorted(LOW_PASS)[0]:
        missing = low_pass_missing(sorted(LOW_PASS))
        assert not missing, missing
    ov, inp, out, other, planes = LOW_PASS[name]
    octx = rh.default_context(**ov)
    spec = StreamSpec(*inp, *out, num_planes=planes)
    ft = FrameTransformer(t360.make_context(**ov), spec)
    oplan = _oracle_plan(tuple(sorted(ov.items())), *inp, *out)
    st = torch.cuda.Stream()
    # the stage alone
    runs = []
    for w, h in [inp] + ([other] if other else []):
        src = co.noise_plane(w, h, frame=w + h)
        for layout in LAYOUTS:
            d_in, d_out = _pitched(torch, src, layout, 0), Plane(torch, w, h, *LAYOUTS[layout][1][:1], w + LAYOUTS[layout][1][1])
            runs.append((src, layout, d_in, d_out))
    torch.cuda.synchronize()
    for src, layout, d_in, d_out in runs:
        assert ft.vft.low_pass_async(d_in.ptr, d_out.ptr, d_in.w, d_in.h, d_in.pitch, d_out.pitch, 0, st.cuda_stream)
    # the whole frame, then each plane on its own
    srcs = [co.noise_plane(*spec.plane_dims(p)[:2], plane=p, frame=3) for p in range(planes)]
    dims = [spec.plane_dims(p)[:4] for p in range(planes)]
    f_in = [_pitched(torch, s, "odd" if p == planes - 1 else "aligned8", 0) for p, s in enumerate(srcs)]
    f_out = [Plane(torch, d[2], d[3], 16, d[2] + 16 + (p % 2)) for p, d in enumerate(dims)]
    p_out = [Plane(torch, d[2], d[3], 1, d[2] + 3) for d in dims]
    assert ft.vft.make_frame_call([(b.ptr, b.pitch) for b in f_in], [(b.ptr, b.pitch) for b in f_out], dims)(st.cuda_stream)
    for p, (iw, ih, ow, oh) in enumerate(dims):
        assert ft.vft.transform_plane_async(f_in[p].ptr, p_out[p].ptr, iw, ih, f_in[p].pitch, ow, oh, p_out[p].pitch,
                                            spec.plane_dims(p)[4], st.cuda_stream)
    st.synchronize()
    for src, layout, _, d_out in runs:
        want = co.filter_plane(octx, src, oplan.segs, oplan.nsegs, oplan.taps)
        _assert_plane(d_out, want, f"{name} low-pass alone {src.shape[1]}x{src.shape[0]} {layout}")
    want = _oracle_frame(ov, spec, srcs, dims)
    for p in range(planes):
        _assert_plane(f_out[p], want[p], f"{name} frame of {planes} plane {p}")
        _assert_plane(p_out[p], want[p], f"{name} per-plane call, plane {p}")
    ft.close()


# ---- the per-view low-pass cache ----------------------------------------------------------------------------------------
VIEW_OV = dict(output_layout=t360.LAYOUT_FLAT_FIXED, interpolation_alg=t360.CUBIC, num_vertical_segments=7,
               num_horizontal_segments=3)
VIEW_SPEC = (1280, 640, 320, 180)
# the kernels follow the horizontal field of view: the same tap counts with other weights from 124 to 132 degrees, from 144
# to 152 and from 184 to 192
VIEW_CANDIDATES = [(15.0 * i, 0.0, hfov, 110.0) for i, hfov in enumerate((124.0, 128.0, 132.0, 144.0, 148.0, 152.0, 184.0, 188.0))]


def _with_view(ov, view):
    return dict(ov, fixed_yaw=view[0], fixed_pitch=view[1], fixed_hfov=view[2], fixed_vfov=view[3])


@functools.lru_cache(maxsize=None)
def view_key_and_taps(view):
    """What viewLowPass keys its cached job lists on (per plan index: the tap count and, per segment, its rectangle, tap
    counts and whether its taps equal its left neighbour's), and the taps themselves."""
    ctx = t360.make_context(**_with_view(VIEW_OV, view))
    iw, ih, ow, oh = VIEW_SPEC
    key, taps = [], []
    for dims in ((iw, ih, ow, oh), chroma((iw, ih)) + chroma((ow, oh))):
        hp = t360.HostPlan(ctx, *dims)
        key.append(hp.num_taps)
        prev = None
        for l, t, w, h, kx, ky in hp.segments():
            same = prev is not None and np.array_equal(kx, prev[0]) and np.array_equal(ky, prev[1])
            key.append((l, t, w, h, len(kx), len(ky), same))
            taps.append(np.concatenate([kx, ky]))
            prev = (kx, ky)
        hp.close()
    return tuple(key), np.concatenate(taps).tobytes()


def view_groups():
    """Views grouped by key, each group's views with pairwise different taps: within a group the cache refills the taps,
    across groups it cuts the jobs again."""
    groups = {}
    for v in VIEW_CANDIDATES:
        key, taps = view_key_and_taps(v)
        g = groups.setdefault(key, {})
        g.setdefault(taps, v)
    return [list(g.values()) for g in groups.values() if len(g) >= 2]


def view_sequences():
    (a0, a1), (b0, b1) = [g[:2] for g in view_groups()[:2]]
    return [a0, a1, b0, b1, a1, a0, b1, b0], [b0, b1, a0, a1, b1, b0, a1, a0]


def test_view_sequences_refill_and_rebuild():
    """The view sequences alternate refills (same key, other taps) and rebuilds (other key)."""
    assert len(view_groups()) >= 2, "fewer than two view keys with several tap sets"
    for seq in view_sequences():
        kinds = set()
        for a, b in zip(seq, seq[1:]):
            (ka, ta), (kb, tb) = view_key_and_taps(a), view_key_and_taps(b)
            kinds.add("refill" if ka == kb and ta != tb else "rebuild" if ka != kb else "same")
        assert kinds == {"refill", "rebuild"}, kinds


@pytest.mark.gpu
@pytest.mark.parametrize("streams", [1, 2])
def test_view_low_pass_cache_refills_and_rebuilds(streams, torch_cuda):
    """View frames that alternate between refilling the cached low-pass taps and cutting new jobs, on one stream or split
    over two (each stream keeps its own cache), enqueued without a synchronise: every frame equals a fresh transform of
    its view and the oracle."""
    torch = torch_cuda
    seqs = view_sequences()
    order = [(0, v) for v in seqs[0]] if streams == 1 else [(i % 2, seqs[i % 2][i // 2]) for i in range(2 * len(seqs[0]))]
    spec = StreamSpec(*VIEW_SPEC)
    srcs = [co.noise_plane(*spec.plane_dims(p)[:2], plane=p, frame=21) for p in range(3)]
    dims = [spec.plane_dims(p)[:4] for p in range(3)]
    d_in = [_pitched(torch, s, "aligned8", 0) for s in srcs]
    outs = [[Plane(torch, d[2], d[3], 0, d[2] + 8) for d in dims] for _ in order]
    ft = FrameTransformer(t360.make_context(**VIEW_OV), spec)
    sts = [torch.cuda.Stream() for _ in range(streams)]
    ins = [(b.ptr, b.pitch) for b in d_in]
    torch.cuda.synchronize()
    for (s, view), out in zip(order, outs):
        assert ft.view_frame_call(ins, [(b.ptr, b.pitch) for b in out])(view, sts[s].cuda_stream), view
    torch.cuda.synchronize()
    ft.close()
    fresh = {}
    for (s, view), out in zip(order, outs):
        if view not in fresh:
            ov = _with_view(VIEW_OV, view)
            f = FrameTransformer(t360.make_context(**ov), spec)
            ref = [Plane(torch, d[2], d[3], 0, d[2] + 8) for d in dims]
            assert f.frame_call(ins, [(b.ptr, b.pitch) for b in ref])(0)
            torch.cuda.synchronize()
            f.close()
            fresh[view] = [r.read()[0] for r in ref]
            for p, (w, o) in enumerate(zip(fresh[view], _oracle_frame(ov, spec, srcs, dims))):
                assert np.array_equal(w, o), f"fresh transform of {view} plane {p} differs from the oracle"
        for p in range(3):
            _assert_plane(out[p], fresh[view][p], f"stream {s} view {view} plane {p}")


# ---- the resize sweep on the device -------------------------------------------------------------------------------------
RESIZE_OV = dict(interpolation_alg=t360.LINEAR, enable_low_pass_filter=0)
RESIZE_LOW_PASS = dict(interpolation_alg=t360.CUBIC, num_vertical_segments=9, num_horizontal_segments=2)
RESIZE_IN = (320, 160)


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(RESIZE) + 1))
def test_resize_pairs_on_the_device(i, torch_cuda):
    """The map generated at one size, the planes requested at another: the per-plane sync call, the per-plane async call on
    odd and 8-aligned device planes and the whole frame of 3 planes, bit-exact against the oracle, padding untouched.  The
    last case runs the low-pass before a fractional shrink."""
    torch = torch_cuda
    if i == 0:
        missing = resize_missing(RESIZE)
        assert not missing, missing
    (mw, mh), (dw, dh) = RESIZE[i] if i < len(RESIZE) else ((161, 97), (100, 60))
    ov = RESIZE_OV if i < len(RESIZE) else RESIZE_LOW_PASS
    spec = StreamSpec(*RESIZE_IN, mw, mh)
    dims = [spec.plane_dims(0)[:2] + (dw, dh)] + [spec.plane_dims(p)[:2] + chroma((dw, dh)) for p in (1, 2)]
    srcs = [co.noise_plane(*spec.plane_dims(p)[:2], plane=p, frame=i) for p in range(3)]
    want = _oracle_frame(ov, spec, srcs, dims)
    ft = FrameTransformer(t360.make_context(**ov), spec)
    got = ft.vft.transform_plane(srcs[0], dw, dh, 0)
    assert np.array_equal(got, want[0]), f"{RESIZE[i % len(RESIZE)]}: per-plane sync call, {int((got != want[0]).sum())} px differ"
    st = torch.cuda.Stream()
    planes = {layout: (_pitched(torch, srcs[0], layout, 0), Plane(torch, dw, dh, LAYOUTS[layout][1][0], dw + LAYOUTS[layout][1][1]))
              for layout in LAYOUTS}
    f_in = [_pitched(torch, s, "odd" if p else "aligned8", 0) for p, s in enumerate(srcs)]
    f_out = [Plane(torch, d[2], d[3], 16 * p + 1, d[2] + 5) for p, d in enumerate(dims)]
    torch.cuda.synchronize()
    for d_in, d_out in planes.values():
        assert ft.vft.transform_plane_async(d_in.ptr, d_out.ptr, *RESIZE_IN, d_in.pitch, dw, dh, d_out.pitch, 0, st.cuda_stream)
    assert ft.vft.make_frame_call([(b.ptr, b.pitch) for b in f_in], [(b.ptr, b.pitch) for b in f_out], dims)(st.cuda_stream)
    st.synchronize()
    ft.close()
    for layout, (_, d_out) in planes.items():
        _assert_plane(d_out, want[0], f"{(mw, mh)} -> {(dw, dh)} per-plane async, {layout}")
    for p in range(3):
        _assert_plane(f_out[p], want[p], f"{(mw, mh)} -> {(dw, dh)} frame plane {p}")
