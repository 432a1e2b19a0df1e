"""The L1 gather: the tile loop of the per-frame kernels (view_gather.cu: gatherViewTiles with its five record policies) and
the whole-plane kernels (kernels.cu: gatherKernel / nearestKernel), both sampling through gatherPixel
(gather_common.cuh), at every window path, source alignment and tile edge, on the device against the oracle's cv::remap.

gatherPixel takes one of several paths per pixel: the interior fold reads aligned words (so the source base's
misalignment and the row's end matter), the per-tap path wraps (BORDER_WRAP) or reflects (BORDER_TRANSPARENT) each tap,
BORDER_TRANSPARENT skips a pixel whose anchor lies outside and, for bilinear, renormalises the taps that exist.  The tile
loop stores 32 columns x viewTileRows(K) rows per tile over the planes of a frame, persistent over more tiles than
resident CTAs.  A wrong path, shift or bound shows as a few differing pixels or a byte written outside the plane, at the
shapes that reach it.

The ledger below computes every case's sampling records on the host -- the per-frame kernels' host twins, the caller's
map quantised as cv::convertMaps does, or records placed by hand -- and classifies each pixel's window from OpenCV's
semantics, so that a case removed from the sweep, or a host change that stops producing a class, fails here, on a CPU,
naming the pairs that went missing.  The GPU half runs every case through its public entry point on guarded device
buffers and compares bit for bit with remap_u8 of the records written back as an exact CV_32FC2 map.
"""
from __future__ import annotations

import functools
import itertools
import zlib

import numpy as np
import pytest

import transform360_b200 as t360
from oracle import c_oracle as co
from tests.test_lens_blend import composite
from transform360_b200.stream import FrameTransformer, StreamSpec

WRAP, TRANSPARENT = t360.BORDER_WRAP, t360.BORDER_TRANSPARENT
INTERP = {1: t360.NEAREST, 2: t360.LINEAR, 4: t360.CUBIC, 8: t360.LANCZOS4}
KS = (1, 2, 4, 8)
NO_LOW_PASS = dict(enable_low_pass_filter=0)
FULL_SMS = 144  # GH100 with every SM enabled: a tile count above FULL_SMS * 2048 / threads exceeds the resident CTAs of any H100


def gather_threads(k):  # kernels.cuh: gatherThreads
    return 512 if k == 8 else 256


def view_tile_rows(k):  # kernels.cuh: viewTileRows (kViewRowsPerThread = 8)
    return gather_threads(k) // 32 * 8


def plane_tile_rows(k):  # kernels.cuh: gatherTileH (4 rows per thread; nearest runs 256 threads)
    return gather_threads(k) // 32 * 4


def resident_bound(k):
    return FULL_SMS * 2048 // gather_threads(k)


# ---- the window classifier --------------------------------------------------------------------------------------------
# What cv::remap does with one K x K window {col0, row0} (first tap, before any border handling) over a w x h source, split
# where an implementation has to take a different path:
#   interior    every tap inside, and the aligned 32-bit words that hold the window's row (col0 & ~3 up to the word after
#               col0 + K - 1; two words for K = 2) inside the row too: a tight pitch may end the row there
#   slack       every tap inside, but those words would reach past the row's last byte
#   edge_* / corner_*   BORDER_WRAP, the window crosses one edge / two edges of the plane
#   outside     BORDER_WRAP, no tap column (or row) inside: the window wraps whole, once or several times
#   span        BORDER_WRAP, the plane is narrower (or shorter) than the window and it crosses both edges
#   skip        BORDER_TRANSPARENT, the anchor tap (K / 2 - 1, K / 2 - 1) lies outside: the pixel keeps its byte
#   reflect     BORDER_TRANSPARENT, anchor inside, taps outside: reflected (BORDER_REFLECT_101), K = 4 and 8
#   reflect_span  as reflect, on a plane narrower or shorter than the window (the reflection bounces more than once)
#   partial_col / partial_row / partial_corner  bilinear under BORDER_TRANSPARENT with the anchor on the last column / row /
#               both: the taps that exist, renormalised by their weight
#   saturated   a coordinate that did not fit (NaN, infinities, beyond the int16 range): cv::remap samples -32768 or 32767
#   K = 1 (nearest): inside, wrapped (BORDER_WRAP), skip (BORDER_TRANSPARENT), saturated
WRAP_CLASSES = ("interior", "slack", "edge_left", "edge_right", "edge_top", "edge_bottom", "corner_tl", "corner_tr", "corner_bl",
                "corner_br", "outside", "span", "saturated")


def window_vocabulary(k, border):
    if k == 1:
        return ("inside", "wrapped" if border == WRAP else "skip", "saturated")
    if border == WRAP:
        return WRAP_CLASSES
    if k == 2:
        return ("interior", "slack", "skip", "partial_col", "partial_row", "partial_corner", "saturated")
    return ("interior", "slack", "skip", "reflect", "reflect_span", "saturated")


def window_labels(k, border, col0, row0, w, h):
    """Class name of every record {col0, row0} (arrays) over a w x h source, as an object array."""
    col0, row0 = np.asarray(col0, np.int64), np.asarray(row0, np.int64)
    a = max(k // 2 - 1, 0)  # the anchor tap (cv::remap's integer position) and the saturation values it carries
    sat = np.isin(col0 + a, (-32768, 32767)) | np.isin(row0 + a, (-32768, 32767))
    out = np.empty(col0.shape, object)
    if k == 1:
        inside = (col0 >= 0) & (col0 < w) & (row0 >= 0) & (row0 < h)
        out[:] = "wrapped" if border == WRAP else "skip"
        out[inside] = "inside"
        out[sat] = "saturated"
        return out
    in_x, in_y = (col0 >= 0) & (col0 + k <= w), (row0 >= 0) & (row0 + k <= h)
    words = 8 if k == 2 else k + 4
    interior = in_x & in_y & (col0 + words <= w)
    span_x, span_y = (col0 < 0) & (col0 + k > w), (row0 < 0) & (row0 + k > h)
    out[:] = "slack"
    if border == TRANSPARENT:
        anchor = (col0 + a >= 0) & (col0 + a < w) & (row0 + a >= 0) & (row0 + a < h)
        crossing = anchor & ~(in_x & in_y)
        if k == 2:
            xo, yo = col0 + 1 >= w, row0 + 1 >= h
            out[crossing & xo & ~yo] = "partial_col"
            out[crossing & ~xo & yo] = "partial_row"
            out[crossing & xo & yo] = "partial_corner"
        else:
            out[crossing] = "reflect"
            out[crossing & (span_x | span_y)] = "reflect_span"
        out[~anchor] = "skip"
    else:
        left, right, top, bottom = col0 < 0, col0 + k > w, row0 < 0, row0 + k > h
        side = {(True, False, False, False): "edge_left", (False, True, False, False): "edge_right",
                (False, False, True, False): "edge_top", (False, False, False, True): "edge_bottom",
                (True, False, True, False): "corner_tl", (False, True, True, False): "corner_tr",
                (True, False, False, True): "corner_bl", (False, True, False, True): "corner_br"}
        for (l, r, t, b), name in side.items():
            out[(left == l) & (right == r) & (top == t) & (bottom == b)] = name
        out[span_x | span_y] = "span"
        out[(col0 >= w) | (col0 + k <= 0) | (row0 >= h) | (row0 + k <= 0)] = "outside"
    out[interior] = "interior"
    out[sat] = "saturated"
    return out


def window_classes(k, border, records, w, h):
    labels = window_labels(k, border, records[..., 0], records[..., 1] >> 10, w, h)
    return set(np.unique(labels).tolist()) if labels.size else set()


def records_to_map(records, k):
    """The exact CV_32FC2 map whose cv::convertMaps gives these records: x = col0 + K / 2 - 1 + fracX / 32, y likewise
    (nearest: the position itself).  The saturated records come back as -32768 / 32767 + fraction."""
    a = max(k // 2 - 1, 0)
    col0, row0, phase = records[..., 0].astype(np.int64), records[..., 1] >> 10, records[..., 1] & 1023
    fx, fy = (phase & 31, phase >> 5) if k > 1 else (0 * phase, 0 * phase)
    return np.stack([(col0 + a) + fx / 32.0, (row0 + a) + fy / 32.0], -1).astype(np.float32)


def records_from(col0, row0, k, rng):
    """Records {col0, row0 << 10 | phase} with random phases (none for nearest)."""
    phase = rng.integers(0, 1024, np.shape(col0)) if k > 1 else np.zeros(np.shape(col0), np.int64)
    return np.stack([np.asarray(col0, np.int64), (np.asarray(row0, np.int64) << 10) | phase], -1).astype(np.int32)


# ---- hand-built records -----------------------------------------------------------------------------------------------
def axis_positions(k, n, saturate=True):
    """First-tap positions along an axis of n pixels that reach every class: inside (interior and the slack band), crossing
    each edge, wholly outside (adjacent, one and several planes away) and, with saturate, the saturated ends."""
    a = max(k // 2 - 1, 0)
    inside = sorted({0, 1, 2, 3, max(n - k, 0), max(n - k - 1, 0), max(n - k - 3, 0), max(n - 9, 0), n // 2})
    crossing = [-1, -(k - 1), n - k + 1, n - 1] if k > 1 else []
    outside = [-k, -k - 3, n, n + 5, 2 * n + 3, -3 * n - 2] if k > 1 else [-1, -5, n, n + 3, 3 * n + 1, -2 * n - 1]
    sat = [-32768 - a, 32767 - a] if saturate else []
    return inside + crossing + outside + sat


def grid_records(k, w, h, mw, mh, seed, saturate=True):
    """A mw x mh map whose records run through every (column position, row position) pair of axis_positions, cycling."""
    rng = np.random.default_rng(seed)
    pairs = list(itertools.product(axis_positions(k, w, saturate), axis_positions(k, h, saturate)))
    order = rng.permutation(mw * mh) % len(pairs)
    col0 = np.array([pairs[i][0] for i in order]).reshape(mh, mw)
    row0 = np.array([pairs[i][1] for i in order]).reshape(mh, mw)
    return records_from(col0, row0, k, rng)


def spread_records(k, w, h, mw, mh, seed):
    """A mw x mh map of records spread over the source and a band of k + 2 around it: mostly interior windows."""
    rng = np.random.default_rng(seed)
    return records_from(rng.integers(-k - 2, w + 2, (mh, mw)), rng.integers(-k - 2, h + 2, (mh, mw)), k, rng)


# ---- the cases --------------------------------------------------------------------------------------------------------
# Source layouts: base misalignment 0-3 (bytes past a 4-byte boundary; misalignment 0 sits 4 bytes past a 16-byte boundary, so
# that no planned plane is TMA-describable and every one takes the whole-plane kernel) and the pitch: tight (= width), odd,
# or padded by at least 32 columns (then the output's padding also holds a whole tile column of guard bytes).
PITCHES = ("tight", "odd", "padded")
LAYOUTS = [(m, p) for m in range(4) for p in PITCHES]


def pitch_of(kind, w):
    return w if kind == "tight" else ((w + 3) | 1 if kind == "odd" else (w + 32 + 15) // 16 * 16 + 16)


POLICIES = ("flat", "sphere", "barrel", "map", "lens", "blend", "plane")
LARGE = (1000, 1580)  # more view tiles than resident CTAs for every K with its 4:2:0 chroma (and whole-plane tiles alone)
LARGE_MAP = (1100, 2100)  # the same on its own (a map frame's other planes are small)


def _cases():
    """name -> dict(policy, k, border, planes: [(in w, in h, out w, out h)], and what the records come from)."""
    cases = {}
    for k in KS:
        # flat views across the +-180 degree seam, a small frame (narrow, short chroma) and a large one
        for size, out in (("small", (40, 14)), ("large", LARGE)):
            cases[f"flat_k{k}_{size}"] = dict(policy="flat", k=k, border=WRAP, spec=(96 if size == "small" else 512, 48 if size == "small" else 256, *out),
                                              view=(172.0, 25.0, 120.0, 100.0))
        cases[f"sphere_k{k}"] = dict(policy="sphere", k=k, border=WRAP, spec=(96, 48, 60, 14), orientation=(150.0, 30.0, 10.0))
        cases[f"barrel_k{k}"] = dict(policy="barrel", k=k, border=TRANSPARENT, spec=(96, 48, 60, 14), pose=(40.0, 20.0, 5.0, 90.0, 90.0))
        cases[f"lens_k{k}"] = dict(policy="lens", k=k, border=TRANSPARENT, spec=(130, 66, 60, 14), orientation=(30.0, 60.0, 0.0))
        cases[f"blend_k{k}"] = dict(policy="blend", k=k, border=TRANSPARENT, spec=(130, 66, 60, 14), orientation=(20.0, 70.0, 15.0), seam=40.0)
        for border in (WRAP, TRANSPARENT):
            b = "wrap" if border == WRAP else "transparent"
            # per-frame maps: a large plane, a narrow and short one on a source smaller than the window, every window class
            cases[f"map_k{k}_{b}"] = dict(policy="map", k=k, border=border, planes=[
                (301, 199, *LARGE_MAP, "spread"), (max(k - 2, 1), max(k // 2 - 1, 1), 20, 5, "grid"), (37, 23, 45, 40, "grid")])
            # planned whole planes: every window class; narrow and short on a source smaller than the window and of another
            # size than the plan's; large (one border per K where the border adds no window class: the tile loop does not
            # depend on it)
            cases[f"plane_k{k}_{b}_windows"] = dict(policy="plane", k=k, border=border, planes=[(37, 23, 45, 40, "grid")])
            if k >= 4 or (border == WRAP) != (k in (2, 8)):  # (K <= 2: no window spans the narrow source)
                cases[f"plane_k{k}_{b}_narrow"] = dict(policy="plane", k=k, border=border, planes=[(max(k - 3, 1), 3, 29, 6, "grid_in_range")],
                                                       plan_in=(max(k - 3, 1) + 3, 5))
            if (border == WRAP) == (k in (2, 8)):
                cases[f"plane_k{k}_{b}_large"] = dict(policy="plane", k=k, border=border, planes=[(301, 199, *LARGE, "spread")])
    per_policy = {}
    for name, c in cases.items():  # a fixed layout per plane, cycling through LAYOUTS within each policy
        i = per_policy.setdefault(c["policy"], [0])
        c["layouts"] = [LAYOUTS[(i[0] + p) % len(LAYOUTS)] for p in range(3)]
        i[0] += 3 if c["policy"] != "plane" else 1
    return cases


CASES = _cases()
CTX_BASE = dict(flat=dict(output_layout=t360.LAYOUT_FLAT_FIXED), sphere=dict(output_layout=t360.LAYOUT_EQUIRECT),
                barrel=dict(output_layout=t360.LAYOUT_BARREL), lens=dict(output_layout=t360.LAYOUT_EQUIRECT),
                blend=dict(output_layout=t360.LAYOUT_BARREL), map={}, plane={})


def case_context(c):
    return t360.make_context(interpolation_alg=INTERP[c["k"]], **NO_LOW_PASS, **CTX_BASE[c["policy"]])


def blend_rig():
    """Two 190-degree lenses whose image circles are cut by the frame (radius 560 in a 1000-pixel-high calibration), pitched
    apart: covered directions that fall outside the source, so the feathered belt holds pixels where one lens's record is
    skipped by BORDER_TRANSPARENT and the other stands alone."""
    rig = t360.T360LensRig(2, 2000, 1000)
    for i, (cx, yaw, pitch, radius) in enumerate(((500.0, 0.0, 12.0, 560.0), (1500.0, 180.0, -9.0, 530.0))):
        f = radius / np.radians(95.0)
        rig.lens[i] = t360.T360Lens(f, f, cx, 499.5, (0.0, 0.0, 0.0, 0.0), yaw, pitch, 0.0, 95.0)
    return rig


def case_dims(c):
    """(in w, in h, out w, out h) of every plane."""
    if "spec" in c:
        spec = StreamSpec(*c["spec"])
        return [spec.plane_dims(p)[:4] for p in range(3)]
    return [p[:4] for p in c["planes"]]


def _warp_records(ctx, m, iw, ih, border):
    hp = t360.HostPlan.from_warp(ctx, m, iw, ih, border)
    r = hp.samples
    hp.close()
    return r


@functools.lru_cache(maxsize=None)
def case_records(name):
    """Per plane: records [h][w][2] (for the blend: (records of lens 0, records of lens 1, weight, map0, map1))."""
    c = CASES[name]
    k, ctx, out = c["k"], case_context(c), []
    warp_ctx = t360.make_context(interpolation_alg=INTERP[k], **NO_LOW_PASS)
    for p, (iw, ih, ow, oh) in enumerate(case_dims(c)):
        pol = c["policy"]
        if pol == "flat":
            out.append(t360.view_samples(ctx, c["view"], iw, ih, ow, oh))
        elif pol == "sphere":
            out.append(t360.oriented_samples(ctx, c["orientation"], iw, ih, ow, oh))
        elif pol == "barrel":
            out.append(t360.pose_samples(ctx, c["pose"], iw, ih, ow, oh))
        elif pol == "lens":
            m = t360.lens_map(ctx, blend_rig(), c["orientation"], iw, ih, ow, oh)
            out.append(_warp_records(warp_ctx, m, iw, ih, TRANSPARENT))
        elif pol == "blend":
            m0, m1, wt = t360.lens_blend_maps(ctx, blend_rig(), c["seam"], c["orientation"], iw, ih, ow, oh)
            out.append((_warp_records(warp_ctx, m0, iw, ih, TRANSPARENT), _warp_records(warp_ctx, m1, iw, ih, TRANSPARENT), wt, m0, m1))
        else:
            kind = c["planes"][p][4]
            seed = zlib.crc32(f"{name}/{p}".encode())
            if kind == "spread":
                out.append(spread_records(k, iw, ih, ow, oh, seed))
            else:
                out.append(grid_records(k, iw, ih, ow, oh, seed, saturate=kind == "grid"))
    return out


def blend_belt_classes(k, r0, r1, wt, iw, ih):
    """Classes of the feathered belt (0 < w < 256), where the tile loop gathers both records: both sampled, the first
    (lens 0) skipped and the second alone, the second skipped and the first alone."""
    belt = (wt > 0) & (wt < 256)
    s0 = window_labels(k, TRANSPARENT, r0[..., 0], r0[..., 1] >> 10, iw, ih)
    s1 = window_labels(k, TRANSPARENT, r1[..., 0], r1[..., 1] >> 10, iw, ih)
    sk0, sk1 = np.isin(s0, ("skip", "saturated")), np.isin(s1, ("skip", "saturated"))
    out = set()
    for name, m in (("belt_both", ~sk0 & ~sk1), ("belt_first_skipped", sk0 & ~sk1), ("belt_second_skipped", ~sk0 & sk1)):
        if (belt & m).any():
            out.add(name)
    return out


def tile_classes(c):
    """Tile-loop classes of a case: partial last tile in x / y, a map narrower than a tile / shorter than 8 rows, more tiles
    than resident CTAs (the persistent loop takes further tiles), and with several planes a CTA whose tiles cross a plane."""
    k, rows = c["k"], (plane_tile_rows if c["policy"] == "plane" else view_tile_rows)(c["k"])
    out, tiles = set(), 0
    for _, _, ow, oh in case_dims(c):
        out |= {n for n, hit in (("partial_x", ow % 32), ("partial_y", oh % rows), ("narrow", ow < 32), ("short", oh < 8)) if hit}
        tiles += -(-ow // 32) * -(-oh // rows)
    if tiles > resident_bound(k):
        out.add("many_tiles")
        if len(case_dims(c)) > 1:
            out.add("plane_cross")  # (more tiles than CTAs: CTA t takes tile t and tile t + grid, across the plane boundary)
    return out


def case_tiles(c):
    rows = (plane_tile_rows if c["policy"] == "plane" else view_tile_rows)(c["k"])
    return sum(-(-ow // 32) * -(-oh // rows) for _, _, ow, oh in case_dims(c))


@functools.lru_cache(maxsize=None)
def case_pairs(name):
    """(window pairs, layout pairs, tile pairs) of one case."""
    c = CASES[name]
    pol, k, border = c["policy"], c["k"], c["border"]
    win, lay = set(), set()
    for p, ((iw, ih, _, _), rec) in enumerate(zip(case_dims(c), case_records(name))):
        if pol == "blend":
            r0, r1, wt = rec[:3]
            first = np.where((wt == 256)[..., None], r1, r0)
            second = r1[(wt > 0) & (wt < 256)]
            classes = window_classes(k, border, first, iw, ih) | window_classes(k, border, second, iw, ih)
            classes |= blend_belt_classes(k, r0, r1, wt, iw, ih)
        else:
            classes = window_classes(k, border, rec, iw, ih)
        win |= {(pol, k, border, cls) for cls in classes}
        lay.add((pol, *c["layouts"][p]))
    return frozenset(win), frozenset(lay), frozenset((pol, k, t) for t in tile_classes(c))


# ---- what the ledger requires -----------------------------------------------------------------------------------------
BORDERS = {"flat": (WRAP,), "sphere": (WRAP,), "barrel": (TRANSPARENT,), "lens": (TRANSPARENT,), "blend": (TRANSPARENT,),
           "map": (WRAP, TRANSPARENT), "plane": (WRAP, TRANSPARENT)}
BELT = ("belt_both", "belt_first_skipped", "belt_second_skipped")
TILE_CLASSES = ("partial_x", "partial_y", "narrow", "short", "many_tiles", "plane_cross")


def _window_product():
    return {(pol, k, b, cls) for pol in POLICIES for k in KS for b in (WRAP, TRANSPARENT)
            for cls in window_vocabulary(k, b) + (BELT if pol == "blend" and b == TRANSPARENT else ())}


def _unreachable():
    out = {}
    for pol, k, b, cls in _window_product():
        if b not in BORDERS[pol]:
            out[(pol, k, b, cls)] = ("FLAT_FIXED and the non-barrel sphere layouts gather under BORDER_WRAP only" if b == TRANSPARENT
                                     else "barrel layouts and lens rigs always gather under BORDER_TRANSPARENT")
        elif cls == "saturated" and pol in ("flat", "sphere", "barrel"):
            out[(pol, k, b, cls)] = "the geometry's positions are finite and within a few planes of the source"
        elif cls == "span" and k == 2:
            out[(pol, k, b, cls)] = "a 2 x 2 window crosses both edges of an axis only where the plane has no pixel on it"
        elif cls in ("outside", "span", "reflect_span") and pol in ("flat", "sphere", "barrel", "lens", "blend"):
            out[(pol, k, b, cls)] = "sphere and lens positions lie on or next to the source plane, which is wider and taller than any window"
    for k in KS:
        out[("plane", k, "plane_cross")] = "the whole-plane kernel gathers one plane per launch"
    return out


UNREACHABLE = _unreachable()
# Reachable but not required: the persistent loop over many tiles is gatherViewTiles' own, run by the large flat and map
# frames; the sphere, barrel and lens policies differ from the map policy only in record(), and none of them synchronises
# in beginTile as the flat policy does
NOT_REQUIRED = {(pol, k, t) for pol in ("sphere", "barrel", "lens", "blend") for k in KS for t in ("many_tiles", "plane_cross")}
# Geometry policies reach what their positions produce; the classes below are the ones a wrong path would show in
REQUIRED_GEOMETRY = {
    "flat": ("interior", "slack", "edge_left", "edge_right"),
    "sphere": ("interior", "slack", "edge_left", "edge_right"),
    "barrel": ("interior", "slack", "skip"),
    "lens": ("interior", "slack", "skip"),
    "blend": ("interior", "slack", "skip", "belt_both", "belt_first_skipped", "belt_second_skipped"),
}


def required_windows():
    """Every reachable pair of the hand-built policies; the geometry policies' REQUIRED_GEOMETRY classes (nearest: inside,
    and skip where transparent, in its own vocabulary)."""
    out = {q for q in _window_product() if q not in UNREACHABLE and q[0] not in REQUIRED_GEOMETRY}
    for pol, classes in REQUIRED_GEOMETRY.items():
        for b in BORDERS[pol]:
            for k in KS:
                vocab = window_vocabulary(k, b) + (BELT if pol == "blend" else ())
                out |= {(pol, k, b, cls) for cls in classes if cls in vocab}
                if k == 1:
                    out.add((pol, k, b, "inside"))
    return out


def required_layouts():
    return {(pol, m, p) for pol in POLICIES for m, p in LAYOUTS}


def required_tiles():
    return {(pol, k, t) for pol in POLICIES for k in KS for t in TILE_CLASSES if (pol, k, t) not in UNREACHABLE and (pol, k, t) not in NOT_REQUIRED}


@functools.lru_cache(maxsize=None)
def ledger(names):
    win, lay, til = set(), set(), set()
    for n in names:
        w, l, t = case_pairs(n)
        win |= w
        lay |= l
        til |= t
    return win, lay, til


def missing_pairs(names):
    win, lay, til = ledger(tuple(sorted(names)))
    return sorted(required_windows() - win, key=str) + sorted(required_layouts() - lay, key=str) + sorted(required_tiles() - til, key=str)


# ---- CPU: the ledger --------------------------------------------------------------------------------------------------
def test_the_sweep_reaches_every_required_pair():
    missing = missing_pairs(CASES)
    assert not missing, f"no case reaches {missing}: those gather paths go untested"


def test_unreachable_pairs_are_not_produced():
    win, lay, til = ledger(tuple(sorted(CASES)))
    made = sorted((win | til) & set(UNREACHABLE), key=str)
    assert not made, f"pairs listed as unreachable are produced: {made}"


@pytest.mark.parametrize("name", sorted(CASES))
def test_every_case_is_needed(name):
    """Each case reaches a required pair no other case does, so a case removed from the sweep fails the ledger, naming
    exactly the pairs it alone supplied."""
    missing = missing_pairs(set(CASES) - {name})
    assert missing, f"{name} reaches no pair of its own"
    others = ledger(tuple(sorted(set(CASES) - {name})))
    own = set().union(*case_pairs(name)) - set().union(*others)
    assert set(missing) == own & (required_windows() | required_layouts() | required_tiles()), (name, missing)


def test_window_classifier_on_hand_placed_windows():
    """The classifier against windows placed by hand on a 10 x 6 source."""
    cases = [(4, WRAP, 0, 0, "interior"), (4, WRAP, 3, 0, "slack"), (4, WRAP, 6, 2, "slack"), (4, WRAP, -1, 1, "edge_left"),
             (4, WRAP, 7, 1, "edge_right"), (4, WRAP, 1, -2, "edge_top"), (4, WRAP, 1, 3, "edge_bottom"), (4, WRAP, -1, -1, "corner_tl"),
             (4, WRAP, 8, 5, "corner_br"), (4, WRAP, 10, 0, "outside"), (4, WRAP, -4, 0, "outside"), (4, WRAP, -32769, 0, "saturated"),
             (2, WRAP, 2, 0, "interior"), (2, WRAP, 3, 0, "slack"), (8, WRAP, -1, -1, "span"),
             (2, TRANSPARENT, 9, 2, "partial_col"), (2, TRANSPARENT, 3, 5, "partial_row"), (2, TRANSPARENT, 9, 5, "partial_corner"),
             (2, TRANSPARENT, -1, 2, "skip"), (4, TRANSPARENT, -1, 2, "reflect"), (4, TRANSPARENT, -2, 2, "skip"),
             (8, TRANSPARENT, -3, -1, "reflect_span"), (1, WRAP, 10, 0, "wrapped"), (1, TRANSPARENT, 9, 5, "inside"),
             (1, TRANSPARENT, 9, 6, "skip"), (1, WRAP, 32767, 0, "saturated")]
    for k, b, c0, r0, want in cases:
        got = window_labels(k, b, np.array([c0]), np.array([r0]), 10, 6)[0]
        assert got == want, (k, b, c0, r0, got, want)
        assert want in window_vocabulary(k, b)


def _pin_records(k, records, iw, ih):
    ctx = t360.make_context(interpolation_alg=INTERP[k], **NO_LOW_PASS)
    got = _warp_records(ctx, records_to_map(records, k), iw, ih, WRAP)
    assert np.array_equal(got, records), f"K = {k}: {int((got != records).any(-1).sum())} records do not survive the map"


@pytest.mark.parametrize("k", KS)
def test_records_written_as_a_map_quantise_back(k):
    """records_to_map is exact: the map quantises back to the same records, saturated ones included, so remap_u8 of it is
    the oracle of every policy's records."""
    rec = grid_records(k, 37, 23, 45, 40, seed=k)
    assert window_classes(k, WRAP, rec, 37, 23) >= ({"saturated", "wrapped", "inside"} if k == 1 else {"saturated", "outside", "interior"})
    _pin_records(k, rec, 37, 23)
    for name, c in CASES.items():
        if c["k"] == k and c["policy"] in ("flat", "sphere", "barrel"):
            for (iw, ih, ow, oh), r in zip(case_dims(c), case_records(name)):
                if ow * oh <= 20000:
                    _pin_records(k, r, iw, ih)


# ---- GPU --------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests must run on an H100 (there is no CPU fallback to test)")
    return torch


SENTINEL = 0xA5
GUARD_ROWS = 128  # one whole tile of rows (viewTileRows(8)) after the last row
FRONT = 64


class Guarded:
    """A w x h plane at `misalign` bytes past a 4-byte boundary (misalignment 0: 4 bytes past a 16-byte one) in a buffer with
    FRONT guard bytes before it, the row padding of its pitch and GUARD_ROWS rows after it.  Inputs hold noise in every
    guard byte, outputs SENTINEL."""

    def __init__(self, torch, w, h, layout, pixels, guard=None, seed=0):
        misalign, kind = layout
        self.w, self.h, self.pitch = w, h, pitch_of(kind, w)
        self.off = FRONT + (misalign or 4)
        n = self.off + self.pitch * (h + GUARD_ROWS) + 16
        host = np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8) if guard is None else np.full(n, guard, np.uint8)
        rows = host[self.off:self.off + self.pitch * h].reshape(h, self.pitch)
        rows[:, :w] = pixels
        self.host = host
        self.buf = torch.from_numpy(host.copy()).cuda()

    @property
    def ptr(self):
        return self.buf.data_ptr() + self.off

    def check(self, want, what):
        got = self.buf.cpu().numpy()
        rows = got[self.off:self.off + self.pitch * self.h].reshape(self.h, self.pitch)
        pix = rows[:, :self.w]
        bad = pix != want
        if bad.any():
            ys, xs = np.nonzero(bad)
            pytest.fail(f"{what}: {int(bad.sum())} of {bad.size} px differ from the oracle (first at x {xs[0]} y {ys[0]}: "
                        f"{int(pix[ys[0], xs[0]])} for {int(want[ys[0], xs[0]])})")
        mask = np.ones(got.size, bool)
        mask[self.off:self.off + self.pitch * self.h] = np.tile(np.arange(self.pitch) >= self.w, self.h)
        moved = np.nonzero(mask & (got != self.host))[0]
        assert moved.size == 0, (f"{what}: {moved.size} guard bytes written, the first at byte {int(moved[0]) - self.off} from the "
                                 f"plane's base (row {(int(moved[0]) - self.off) // self.pitch})")


def _prefill(c, p, ow, oh):
    """What an output plane holds before the call and keeps where BORDER_TRANSPARENT skips: the caller's bytes, except the
    chroma planes of a per-frame call (pre-filled with 128)."""
    if c["border"] == TRANSPARENT and p > 0 and c["policy"] != "plane":
        return np.full((oh, ow), 128, np.uint8)
    return np.random.default_rng(1000 + p).integers(0, 256, (oh, ow), dtype=np.uint8)


def _oracle(c, name, p, src, prefill):
    k, rec = c["k"], case_records(name)[p]
    if c["policy"] == "blend":
        return composite(src, rec[3], rec[4], rec[2], INTERP[k], prefill)
    return co.remap_u8(src, records_to_map(rec, k), INTERP[k], c["border"], prefill.copy())


def _enqueue(torch, c, name, ins, outs, st):
    """The case through its public entry point; returns the objects the call needs kept alive."""
    pol, k, ctx = c["policy"], c["k"], case_context(c)
    dims = case_dims(c)
    pin = [(g.ptr, g.pitch) for g in ins]
    pout = [(g.ptr, g.pitch) for g in outs]
    if pol in ("flat", "sphere", "barrel"):
        ft = FrameTransformer(ctx, StreamSpec(*c["spec"]))
        torch.cuda.synchronize()
        if pol == "flat":
            ok = ft.vft.make_view_frame_call(pin, pout, dims)(c["view"], st.cuda_stream)
        elif pol == "sphere":
            ok = ft.vft.make_oriented_frame_call(pin, pout, dims)(c["orientation"], st.cuda_stream)
        else:
            ok = ft.vft.make_pose_frame_call(pin, pout, dims)(c["pose"], st.cuda_stream)
        return ok, ft.vft
    vft = t360.VideoFrameTransform(ctx)
    torch.cuda.synchronize()
    if pol == "lens":
        return vft.make_lens_frame_call(pin, pout, dims)(blend_rig(), c["orientation"], st.cuda_stream), vft
    if pol == "blend":
        return vft.make_lens_blend_frame_call(pin, pout, dims)(blend_rig(), c["seam"], c["orientation"], st.cuda_stream), vft
    maps = [records_to_map(r, k) for r in case_records(name)]
    if pol == "map":
        d_maps = []
        for p, m in enumerate(maps):
            t = torch.zeros((m.shape[0], m.shape[1] + p, 2), dtype=torch.float32, device="cuda")
            t[:, :m.shape[1]] = torch.from_numpy(m).cuda()
            d_maps.append(t)
        torch.cuda.synchronize()
        return vft.make_remap_frame_call(pin, pout, dims, border=c["border"])(d_maps, st.cuda_stream) and d_maps, vft
    iw, ih, ow, oh = dims[0]
    assert vft.generate_map_from_warp(maps[0], *c.get("plan_in", (iw, ih)), 0, c["border"])
    return vft.transform_plane_async(ins[0].ptr, outs[0].ptr, iw, ih, ins[0].pitch, ow, oh, outs[0].pitch, 0, st.cuda_stream), vft


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_cases_on_the_device(name, torch_cuda):
    """Every case through its entry point on guarded planes: each output pixel equals the oracle bit for bit, no guard byte
    of any output changes (row padding, the bytes before the base, a tile of rows after the last)."""
    torch = torch_cuda
    c = CASES[name]
    if name == sorted(CASES)[0]:
        missing = missing_pairs(CASES)
        assert not missing, missing
    if "many_tiles" in tile_classes(c):
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        threads = 256 if c["k"] == 1 else gather_threads(c["k"])
        assert case_tiles(c) > sms * 2048 // threads, f"{name}: {case_tiles(c)} tiles fit the {sms} SMs' resident CTAs"
    dims = case_dims(c)
    n = 1 if c["policy"] == "plane" else 3
    ins, outs, wants = [], [], []
    for p in range(n):
        iw, ih, ow, oh = dims[p]
        src = co.noise_plane(iw, ih, plane=p, frame=len(name))
        prefill = _prefill(c, p, ow, oh)
        ins.append(Guarded(torch, iw, ih, c["layouts"][p], src, seed=p + 7))
        fill = np.random.default_rng(1000 + p).integers(0, 256, (oh, ow), dtype=np.uint8)  # (the call pre-fills chroma itself)
        outs.append(Guarded(torch, ow, oh, c["layouts"][(p + 1) % 3], fill, guard=SENTINEL))
        wants.append(_oracle(c, name, p, src, prefill))
    st = torch.cuda.Stream()
    ok, keep = _enqueue(torch, c, name, ins, outs, st)
    assert ok, f"{name}: the call was refused"
    st.synchronize()
    for p in range(n):
        outs[p].check(wants[p], f"{name} plane {p}")
    keep.close()
