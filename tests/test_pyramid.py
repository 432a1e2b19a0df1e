"""The anti-aliased camera views' input pyramid, read back level by level: pyramidLevelKernel (csrc/kernels.cu) through
tests/pyramid_gate.cu, and VideoFrameTransform::buildPyramids through T360B200_transformFrameCameraMipAsync.

The frame tests (test_camera_mip.py, test_camera_aniso.py, test_per_frame_full_size.py) see a pyramid pixel only where an
output pixel's footprint reads it, often blended with a weight below 256.  Here every byte of every level is compared.

What pins what:
  - the gate: one level of 1-3 planes in one launchPyramidLevel call, on torch buffers whose base offsets, pitches and
    sizes the case table chooses, with the tap tables packed as buildPyramids packs them (pyramid_gate.cu).  Every output
    byte equals oracle.c_oracle.resize_area (the plain-C INTER_AREA, pinned to cv2) bit for bit, and the float64 area
    mean: 2 x 2 cells floor(mean + 0.5) exactly; tap levels within 1 LSB of the exact mean over the whole cell, and exact
    against the mean of the taps OpenCV keeps wherever it is more than 1e-3 from a .5 tie.  Every byte around a plane's
    rows (pitch padding and guard bands) keeps its sentinel;
  - the chains: every level of the production inputs (7680 x 3840 luma with its 3840 x 1920 chroma, 5760 x 2880,
    2880 x 2880, 1029 x 515), each level read from the previous one at a 256-byte pitch, as the frame call lays them out;
  - the path ledger: the kernel's own selection rule restated here (taps or 2 x 2 cells; dx + 4 <= dstW; the two source
    rows 8-byte aligned; the destination word 4-byte aligned) reaches, over the case table, the word store, the scalar
    tail, the misaligned-source and misaligned-destination fallbacks and the taps in each parity class;
  - the tap tables the gate packs against OpenCV's computeResizeAreaTab restated in float64 and against the exact
    overlaps of each destination cell;
  - buildPyramids: anti-aliased frames on one stream and on two, with no synchronisation between them, while the input
    sizes (even / odd / mixed parity), maxLevel and the luma plane's alignment change every frame, against the oracle
    composite; a coverage ledger from the host twin shows every level of every plane is read by the views.

Without a GPU: the gate builds for sm_90a with the library flags and links no undefined library symbol, the path ledger
reaches every class, the packed tap tables match, and the coverage ledger holds."""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
from dataclasses import dataclass

import numpy as np
import pytest

import transform360_b200 as t360
from oracle import c_oracle as co
from tests.test_camera_mip import MipFrame
from tests.test_camera_models import STEREOGRAPHIC
from tests.test_rectilinear import _ctx
from tests.test_rectilinear import torch_cuda  # noqa: F401 (fixture)
from transform360_b200 import build as b

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GATE_SOURCES = ("kernels.cu", "sampling.cpp", "geometry.cpp", "lowpass_plan.cpp")  # (sampling.cpp's plan step calls the other two)
BLOCK_W, BLOCK_H = 128, 8  # kPyramidBlockW, kPyramidBlockH (kernels.cuh)
GUARD = 256  # padding bytes before and after every buffer; buffers start 256-byte aligned
# the padding of a source and of the destinations of each level: a level whose source padding leaks into its padding
# (a 2 x 2 cell past the row's end) writes a byte that differs from its sentinel
SOURCE_PAD, SENTINELS = 0x3C, (0xA7, 0x59)


def _pitch256(w):
    return (w + 255) // 256 * 256


# ---- the case table ---------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Plane:
    """One plane of a launch: a srcW x srcH source to its ceil-half level.  src_off / dst_off: the rows' start past a
    256-byte aligned address; pitches default to the frame call's 256-byte pitch."""
    w: int
    h: int
    src_off: int = 0
    src_pitch: int = 0
    dst_off: int = 0
    dst_pitch: int = 0

    @property
    def dw(self):
        return (self.w + 1) // 2

    @property
    def dh(self):
        return (self.h + 1) // 2

    @property
    def sp(self):
        return self.src_pitch or _pitch256(self.w)

    @property
    def dp(self):
        return self.dst_pitch or _pitch256(self.dw)

    @property
    def taps(self):
        return self.w % 2 == 1 or self.h % 2 == 1

    @property
    def blocks(self):
        return -(-self.dw // BLOCK_W) * -(-self.dh // BLOCK_H)


def _cases():
    cases = {}

    def add(name, *planes):
        assert name not in cases
        cases[name] = tuple(planes)

    # parity classes: (even, even) takes the 2 x 2 cells, any odd side the taps
    for w, h in ((200, 100), (201, 100), (200, 101), (201, 101)):
        add(f"parity-{w}x{h}", Plane(w, h))
    # dstW mod 4 on the word path (the scalar tail), and on the taps
    for dw in (64, 65, 66, 67):
        add(f"tail-{dw}", Plane(2 * dw, 38))
        add(f"tail-taps-{dw}", Plane(2 * dw - 1, 38))
    # dstW around the 128-column block, dstH around the 8-row block, on both paths
    for dw in (127, 128, 129, 255, 256, 257):
        add(f"blockW-{dw}", Plane(2 * dw, 22))
        add(f"blockW-taps-{dw}", Plane(2 * dw - 1, 21))
    for dh in (7, 8, 9, 15, 16, 17):
        add(f"blockH-{dh}", Plane(258, 2 * dh))
        add(f"blockH-taps-{dh}", Plane(257, 2 * dh - 1))
    # the smallest levels the pyramid has (sides of 8 from 15 and 16, and 9 from 17), every parity mix
    for w in (15, 16, 17):
        for h in (15, 16, 17):
            add(f"smallest-{w}x{h}", Plane(w, h))
    # level-1 sources at every base offset mod 8, with pitches = 0, 4 and odd mod 8 in one launch: only offset 0 with a
    # pitch = 0 mod 8 has both rows of every 2 x 2 cell 8-byte aligned; the rest take the scalar fallback
    for off in range(8):
        add(f"src-align-{off}", Plane(266, 42, src_off=off, src_pitch=512), Plane(266, 42, src_off=off, src_pitch=516),
            Plane(266, 42, src_off=off, src_pitch=519 + 2 * off))
    # destinations whose rows are not 4-byte aligned: a base offset of 1-3, and an odd pitch that moves every row's start
    for off in (1, 2, 3):
        add(f"dst-align-{off}", Plane(264, 40, dst_off=off), Plane(264, 40, dst_pitch=133 + 2 * off))
    add("dst-align-taps", Plane(263, 39, dst_off=1, dst_pitch=135))
    # several planes in one launch: blocks cross the firstBlock boundaries between 2 x 2 cells and taps, plane 2 with
    # fewer blocks than plane 1
    add("planes-2", Plane(520, 72), Plane(259, 35))
    add("planes-3", Plane(520, 72), Plane(259, 35), Plane(131, 19))
    add("planes-3-taps-first", Plane(515, 71), Plane(516, 70), Plane(33, 17, src_off=3, src_pitch=37))
    add("planes-3-unaligned", Plane(1030, 516, src_off=1, src_pitch=1031), Plane(515, 258), Plane(515, 258))
    return cases


CASES = _cases()
FILLS = ("noise", "zeros", "ones", "tie", "ramp-x", "ramp-y")
# chains: every level of every plane to the top, each from the one below at a 256-byte pitch (level 1 from the
# caller's plane); a yuv420p frame's planes in one launch per level, as the frame call runs them
CHAINS = {
    "7680x3840-yuv420p": [(7680, 3840), (3840, 1920), (3840, 1920)],
    "5760x2880": [(5760, 2880)],
    "2880x2880": [(2880, 2880)],
    "1029x515-yuv420p": [(1029, 515), (515, 258), (515, 258)],
}
MAX_LEVEL = 8


def fill(kind, w, h, seed):
    """A w x h source: seeded noise, all 0, all 255, 2 x 2 cells whose sums are 2 mod 4 (the rounding tie of
    (sum + 2) >> 2), or a column / row ramp (the area mean of a ramp is its value at the cell centre, which for an odd
    side sits just below a .5 for the first cells of every ramp period)."""
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (h, w), dtype=np.uint8)
    if kind == "zeros":
        return np.zeros((h, w), np.uint8)
    if kind == "ones":
        return np.full((h, w), 255, np.uint8)
    if kind == "tie":
        a = rng.integers(0, 255, ((h + 1) // 2, (w + 1) // 2)).repeat(2, 0).repeat(2, 1)[:h, :w]
        return (a + (np.arange(h)[:, None] % 2)).astype(np.uint8)  # a, a over a + 1, a + 1: sum 4a + 2
    x, y = np.meshgrid(np.arange(w), np.arange(h))
    return ((x if kind == "ramp-x" else y) & 255).astype(np.uint8)


# ---- the float64 model ------------------------------------------------------------------------------------------------
def axis_overlaps(s, d, kept_only):
    """Destination i's cell [i s / d, (i + 1) s / d) against sources j, j + 1, j + 2 from j = floor(i s / d): (index, overlap)
    [d][3], overlaps in 1/d source pixels (exact integers).  kept_only: without the slivers of at most 1e-3 source pixel
    that computeResizeAreaTab leaves out."""
    i = np.arange(d, dtype=np.int64)
    lo, hi = i * s, (i + 1) * s
    idx = lo[:, None] // d + np.arange(3)
    ov = np.clip(np.minimum(hi[:, None], (idx + 1) * d) - np.maximum(lo[:, None], idx * d), 0, None)
    ov[idx >= s] = 0
    if kept_only:
        ov[(ov < d) & (ov * 1000 <= d)] = 0
    return np.minimum(idx, s - 1), ov


def area_numerators(src, dw, dh, kept_only):
    """(N, D): the area mean of every destination pixel is N / D exactly (N int64 [dh][dw], D = srcW * srcH)."""
    h, w = src.shape
    ix, wx = axis_overlaps(w, dw, kept_only)
    iy, wy = axis_overlaps(h, dh, kept_only)
    out = np.empty((dh, dw), np.int64)
    s = src.astype(np.int64)
    for r0 in range(0, dh, 256):
        r1 = min(dh, r0 + 256)
        v = sum(wy[r0:r1, k, None] * s[iy[r0:r1, k]] for k in range(3))
        out[r0:r1] = sum(wx[None, :, k] * v[:, ix[:, k]] for k in range(3))
    return out, w * h


def check_float64(got, src, what):
    """2 x 2 cells: floor(mean + 0.5) exactly.  Taps: within 1 LSB of the exact cell mean, and equal to the kept taps'
    mean rounded wherever that is more than 1e-3 from a .5 tie."""
    dh, dw = got.shape
    g = got.astype(np.int64)
    if src.shape[1] % 2 == 0 and src.shape[0] % 2 == 0:
        n, d = area_numerators(src, dw, dh, kept_only=False)
        want = (2 * n + d) // (2 * d)
        bad = np.argwhere(g != want)
        assert not bad.size, f"{what}: {len(bad)} px differ from floor(mean + 0.5), first at {tuple(bad[0])}"
        return
    n, d = area_numerators(src, dw, dh, kept_only=False)
    far = np.abs(g * d - n) > d  # |got - mean| > 1
    bad = np.argwhere(far)
    assert not bad.size, f"{what}: {len(bad)} px more than 1 LSB off the area mean, first at {tuple(bad[0])}"
    n, d = area_numerators(src, dw, dh, kept_only=True)
    frac = (n % d) / d
    sure = np.abs(frac - 0.5) > 1e-3
    want = (2 * n + d) // (2 * d)
    bad = np.argwhere(sure & (g != want))
    assert not bad.size, f"{what}: {len(bad)} px off the kept taps' rounded mean, first at {tuple(bad[0])}"


# ---- the path ledger --------------------------------------------------------------------------------------------------
def path_classes(p: Plane):
    """{class: count of 4-pixel groups (word path) or rows (taps)} of one plane, by the kernel's selection rule, for
    buffers that start 256-byte aligned: xTaps == nullptr; dx + 4 <= dstW; (r0 | r1) & 7; (drow + dx) & 3."""
    if p.taps:
        return {f"taps-{'oe'[p.w % 2 == 0]}{'oe'[p.h % 2 == 0]}": p.dh}
    dy, dx = np.meshgrid(np.arange(p.dh), np.arange(0, p.dw, 4), indexing="ij")
    r0 = p.src_off + 2 * dy * p.sp + 2 * dx
    r1 = r0 + p.sp
    full = dx + 4 <= p.dw
    src_ok = ((r0 | r1) & 7) == 0
    dst_ok = ((p.dst_off + dy * p.dp + dx) & 3) == 0
    return {"word": int((full & src_ok & dst_ok).sum()), "tail": int((~full).sum()), "src-misaligned": int((full & ~src_ok).sum()),
            "dst-misaligned": int((full & src_ok & ~dst_ok).sum())}


LEDGER_CLASSES = ("word", "tail", "src-misaligned", "dst-misaligned", "taps-oe", "taps-eo", "taps-oo")


def ledger(cases):
    counts = {c: 0 for c in LEDGER_CLASSES}
    for planes in cases.values():
        for p in planes:
            for c, n in path_classes(p).items():
                counts[c] += n
    return counts


# ---- the gate ---------------------------------------------------------------------------------------------------------
def gate_command(out):
    """The gate's nvcc command: the library's architecture, optimisation and host flags (build.py)."""
    return [b.nvcc_path(), *b.ARCH, "-O3", "-lineinfo", "-std=c++17", "--shared", "-Xcompiler", b.HOST_FLAGS, "-I",
            os.path.join(ROOT, "include"), "-I", str(b.CSRC), os.path.join(ROOT, "tests", "pyramid_gate.cu"),
            *[str(b.CSRC / s) for s in GATE_SOURCES], "-o", str(out)]


class GatePlane(C.Structure):
    _fields_ = [("src", C.c_ulonglong), ("dst", C.c_ulonglong), ("srcW", C.c_int), ("srcH", C.c_int), ("srcPitch", C.c_int),
                ("dstW", C.c_int), ("dstH", C.c_int), ("dstPitch", C.c_int)]


@pytest.fixture(scope="module")
def gate(tmp_path_factory):
    """(path, ctypes library) of the gate, built once."""
    so = tmp_path_factory.mktemp("pyramid_gate") / "pyramid_gate.so"
    r = subprocess.run(gate_command(so), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lib = C.CDLL(str(so))
    ull, ci = C.POINTER(C.c_ulonglong), C.POINTER(C.c_int)
    lib.pyramidGateTaps.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_size_t, ull, ci]
    lib.pyramidGateLevel.argtypes = [C.c_int, C.POINTER(GatePlane)]
    return so, lib


def packed_taps(lib, w, h, dw, dh):
    """The gate's packed tables of one level: None for exact 2 x 2 cells, else (xTaps, xFirst, yTaps, yFirst) as
    int32 [n][2] {src, float bits}, int32 [dw + 1], int32 [n][2], int32 [dh + 1]."""
    at, n = (C.c_ulonglong * 4)(), (C.c_int * 4)()
    r = lib.pyramidGateTaps(w, h, dw, dh, None, 0, at, n)
    if r == 1:
        return None
    assert r == 0, (w, h, r)
    buf = np.zeros(at[0], np.uint8)
    assert lib.pyramidGateTaps(w, h, dw, dh, buf.ctypes.data, buf.size, at, n) == 0
    assert all(a % 8 == 0 for a in at)
    get = lambda k, per: buf[at[k]:at[k] + 4 * per * n[k]].view(np.int32).reshape(-1, per) if per == 2 else buf[at[k]:at[k] + 4 * n[k]].view(np.int32)
    return get(0, 2), get(1, 1), get(2, 2), get(3, 1)


def area_tab(ssize, dsize):
    """OpenCV's computeResizeAreaTab for one axis, in float64 as OpenCV computes it: ([(src, float32 alpha)], first)."""
    scale = 1.0 / (dsize / ssize)
    taps, first = [], []
    for d in range(dsize):
        first.append(len(taps))
        f1 = d * scale
        f2 = f1 + scale
        cell = min(scale, ssize - f1)
        s2 = min(math.floor(f2), ssize - 1)
        s1 = min(math.ceil(f1), s2)
        if s1 - f1 > 1e-3:
            taps.append((s1 - 1, np.float32((s1 - f1) / cell)))
        taps += [(s, np.float32(1.0 / cell)) for s in range(s1, s2)]
        if f2 - s2 > 1e-3:
            taps.append((s2, np.float32(min(f2 - s2, 1.0, cell) / cell)))
    first.append(len(taps))
    return taps, first


# ---- no GPU needed ----------------------------------------------------------------------------------------------------
def test_gate_builds_for_sm_90a_with_the_library_flags(gate):
    cmd = gate_command(gate[0])
    assert "-ffp-contract=off" in b.HOST_FLAGS and "-fno-fast-math" in b.HOST_FLAGS
    assert cmd[cmd.index("-Xcompiler") + 1] == b.HOST_FLAGS and "arch=compute_90a,code=sm_90a" in cmd and "-O3" in cmd
    assert not any("fast-math" in c and "no" not in c or "ftz" in c for c in cmd)
    assert str(b.CSRC / "kernels.cu") in cmd and set(GATE_SOURCES) <= set(b.SOURCES)
    elf = subprocess.run([os.path.join(os.path.dirname(b.nvcc_path()), "cuobjdump"), "--list-elf", str(gate[0])], capture_output=True,
                         text=True, check=True).stdout
    assert "sm_90a" in elf, elf
    undefined = subprocess.run(["nm", "-DC", "--undefined-only", str(gate[0])], capture_output=True, text=True, check=True).stdout
    assert "t360::" not in undefined, undefined
    sass = subprocess.run([os.path.join(os.path.dirname(b.nvcc_path()), "cuobjdump"), "--list-text", str(gate[0])], capture_output=True,
                          text=True, check=True).stdout
    assert "pyramidLevelKernel" in sass


def test_path_ledger_reaches_every_class():
    """The case table reaches the word store, the scalar tail, both misaligned fallbacks and the taps in each parity class,
    and the sizes, offsets and launches the cases are named for."""
    counts = ledger(CASES)
    missed = [c for c, n in counts.items() if n == 0]
    assert not missed, (missed, counts)
    planes = [p for ps in CASES.values() for p in ps]
    word = [p for p in planes if not p.taps]
    assert {p.dw % 4 for p in word} == {0, 1, 2, 3} and {p.dw % 4 for p in planes if p.taps} == {0, 1, 2, 3}
    for path in (word, [p for p in planes if p.taps]):
        assert {127, 128, 129, 255, 256, 257} <= {p.dw for p in path}
        assert {7, 8, 9, 15, 16, 17} <= {p.dh for p in path}
    assert (8, 8) in {(p.dw, p.dh) for p in word}
    assert {(8, 8), (8, 9), (9, 8), (9, 9)} <= {(p.dw, p.dh) for p in planes if p.taps}
    assert {(w, h) for w in (15, 16, 17) for h in (15, 16, 17)} <= {(p.w, p.h) for p in planes}
    assert {p.src_off % 8 for p in word} == set(range(8)) and {p.sp % 8 for p in word} >= {0, 4, 1, 3, 5, 7}
    assert {p.dst_off % 4 for p in planes} == {0, 1, 2, 3} and any(p.dp % 2 for p in word)
    multi = [ps for ps in CASES.values() if len(ps) > 1]
    assert any(len(ps) == 2 and not ps[0].taps and ps[1].taps for ps in multi)
    assert any(len(ps) == 3 and not ps[0].taps and ps[1].taps and ps[2].taps and ps[2].blocks < ps[1].blocks for ps in multi)
    assert any(len(ps) == 3 and ps[0].taps and not ps[1].taps for ps in multi)
    # the chains reach both paths and the sides of 8 at their tops
    chain_planes = [Plane(*s) for c in CHAINS.values() for w, h in c for s in t360.mip_level_sizes(w, h, MAX_LEVEL)[:-1]]
    assert any(p.taps for p in chain_planes) and any(not p.taps for p in chain_planes)


def _tap_sizes():
    sizes = {(p.w, p.h) for ps in CASES.values() for p in ps}
    sizes |= {s for c in CHAINS.values() for w, h in c for s in t360.mip_level_sizes(w, h, MAX_LEVEL)[:-1]}
    return sorted(sizes)


def test_packed_tap_tables_match_inter_area(gate):
    """Every level the gate runs: exact 2 x 2 cells pass no tables; otherwise the packed {src, alpha bits} and first[]
    arrays are computeResizeAreaTab's, and each destination's taps are the sources its cell overlaps by more than 1e-3
    pixel, with alpha within one float32 ulp of the exact overlap over the cell."""
    lib = gate[1]
    n_taps = 0
    for w, h in _tap_sizes():
        dw, dh = (w + 1) // 2, (h + 1) // 2
        t = packed_taps(lib, w, h, dw, dh)
        assert (t is None) == (w % 2 == 0 and h % 2 == 0), (w, h)
        if t is None:
            continue
        for (taps, first), (s, d) in zip(((t[0], t[1]), (t[2], t[3])), ((w, dw), (h, dh))):
            want, want_first = area_tab(s, d)
            assert first.tolist() == want_first, (s, d)
            assert taps[:, 0].tolist() == [j for j, _ in want], (s, d)
            assert np.array_equal(taps[:, 1], np.array([a for _, a in want], np.float32).view(np.int32)), (s, d)
            idx, ov = axis_overlaps(s, d, kept_only=True)
            alpha = taps[:, 1].copy().view(np.float32).astype(np.float64)
            for i in range(d):
                k = ov[i] > 0
                assert taps[first[i]:first[i + 1], 0].tolist() == idx[i][k].tolist(), (s, d, i)
                exact = ov[i][k] / s
                assert (np.abs(alpha[first[i]:first[i + 1]] - exact) <= np.spacing(exact.astype(np.float32))).all(), (s, d, i)
            n_taps += len(taps)
    assert n_taps > 10000


# ---- on the GPU -------------------------------------------------------------------------------------------------------
class DevBuffer:
    """A torch byte buffer of rows at `off` past a 256-byte aligned address with `pitch`; every byte outside the rows
    (GUARD bytes before and after, the pitch's padding) holds `pad`."""

    def __init__(self, torch, w, h, pitch, off, content=None, pad=SOURCE_PAD):
        self.w, self.h, self.pitch, self.off = w, h, pitch, off
        self.size = GUARD + off + h * pitch + GUARD
        host = np.full(self.size, pad, np.uint8)
        if content is not None:
            host[GUARD + off:GUARD + off + h * pitch].reshape(h, pitch)[:, :w] = content
        self.t = torch.from_numpy(host).cuda()
        assert self.t.data_ptr() % 256 == 0  # the ledger's addresses
        self.addr = self.t.data_ptr() + GUARD + off
        self.initial = host

    def read(self):
        """(rows [h][w], None or where the first byte outside the rows that changed lies)"""
        host = self.t.cpu().numpy()
        rows = host[GUARD + self.off:GUARD + self.off + self.h * self.pitch].reshape(self.h, self.pitch)[:, :self.w].copy()
        outside = np.ones(self.size, bool)
        outside[GUARD + self.off:GUARD + self.off + self.h * self.pitch].reshape(self.h, self.pitch)[:, :self.w] = False
        changed = np.flatnonzero(outside & (host != self.initial))
        if not changed.size:
            return rows, None
        i = int(changed[0]) - GUARD - self.off
        return rows, f"(y {i // self.pitch}, x {i % self.pitch}) of pitch {self.pitch}, {changed.size} bytes in all"


def run_level(torch, lib, planes, what, pad=SENTINELS[0]):
    """One launchPyramidLevel of the planes [(source DevBuffer, Plane)] into destinations padded with `pad`: the
    destination (DevBuffer, rows) of each plane, after checking that nothing around its rows was written."""
    dsts = [DevBuffer(torch, p.dw, p.dh, p.dp, p.dst_off, pad=pad) for _, p in planes]
    args = (GatePlane * len(planes))(*[GatePlane(s.addr, d.addr, p.w, p.h, s.pitch, p.dw, p.dh, p.dp) for (s, p), d in zip(planes, dsts)])
    torch.cuda.synchronize()
    assert lib.pyramidGateLevel(len(planes), args) == 0
    out = []
    for k, d in enumerate(dsts):
        rows, written = d.read()
        assert written is None, f"{what} plane {k} ({d.w}x{d.h}): wrote outside its rows, first at {written}"
        out.append((d, rows))
    return out


def first_difference(got, want):
    bad = np.argwhere(got != want)
    if not bad.size:
        return ""
    y, x = bad[0]
    return f"{len(bad)} px differ, first at (y {y}, x {x}): got {got[y, x]}, want {want[y, x]}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_case_levels_equal_inter_area(case, gate, torch_cuda):
    """Every plane of the case, for every fill, equals co.resize_area bit for bit and the float64 model, and writes
    nothing outside its rows."""
    torch, lib = torch_cuda, gate[1]
    planes = CASES[case]
    for f, kind in enumerate(FILLS):
        srcs = [fill(kind, p.w, p.h, seed=1000 * f + 10 * k + len(case)) for k, p in enumerate(planes)]
        bufs = [DevBuffer(torch, p.w, p.h, p.sp, p.src_off, s) for s, p in zip(srcs, planes)]
        for k, ((_, got), src, p) in enumerate(zip(run_level(torch, lib, list(zip(bufs, planes)), f"{case} {kind}"), srcs, planes)):
            what = f"{case} {kind} plane {k} ({p.w}x{p.h} -> {p.dw}x{p.dh})"
            want = co.resize_area(src, p.dw, p.dh)
            assert np.array_equal(got, want), f"{what}: {first_difference(got, want)}"
            check_float64(got, src, what)


@pytest.mark.gpu
@pytest.mark.parametrize("chain", list(CHAINS))
def test_chains_to_the_top_level(chain, gate, torch_cuda):
    """Every level 1..T of every plane of a production input (T for maxLevel 8), each level's planes in one launch and
    each read from the gate's level below at a 256-byte pitch, equals the oracle's pyramid bit for bit and the float64
    model."""
    torch, lib = torch_cuda, gate[1]
    dims = CHAINS[chain]
    srcs = [co.noise_plane(w, h, plane=p, frame=7) for p, (w, h) in enumerate(dims)]
    sizes = [t360.mip_level_sizes(w, h, MAX_LEVEL) for w, h in dims]
    # level 1 from the caller's planes: the last one with an odd pitch (the scalar fallback where its level is 2 x 2 cells)
    below = [DevBuffer(torch, w, h, _pitch256(w) + (p == 2), 0, s) for p, ((w, h), s) in enumerate(zip(dims, srcs))]
    host_below = srcs
    for level in range(1, max(len(z) for z in sizes)):
        live = [p for p in range(len(dims)) if level < len(sizes[p])]
        planes = [(below[p], Plane(below[p].w, below[p].h, src_pitch=below[p].pitch)) for p in live]
        out = run_level(torch, lib, planes, f"{chain} level {level}", pad=SENTINELS[level % 2])
        for p, (d, got) in zip(live, out):
            assert got.shape == sizes[p][level][::-1]
            what = f"{chain} plane {p} level {level} ({below[p].w}x{below[p].h} -> {d.w}x{d.h})"
            want = co.resize_area(host_below[p], d.w, d.h)
            assert np.array_equal(got, want), f"{what}: {first_difference(got, want)}"
            check_float64(got, host_below[p], what)
            below[p], host_below[p] = d, got
        torch.cuda.synchronize()


# ---- buildPyramids through the frame call -------------------------------------------------------------------------------
# (luma, chroma) input sizes: even / even, odd / odd, and mixed parities; the views: a 300-degree stereographic view tilted
# down, small against the inputs, whose footprints reach every level of every plane (test_coverage_ledger)
SIZES = {"A": ((1024, 512), (512, 256)), "B": ((1029, 515), (515, 258)), "C": ((1031, 514), (516, 257))}
VIEW_POSE, VIEW_CAMERA = (0.0, -60.0, 0.0, 300.0, 300.0), (STEREOGRAPHIC, 0.0)
VIEW_OUT = [(97, 97), (49, 49), (49, 49)]
# (sizes, maxLevel, luma unaligned): sizes and maxLevel change every frame
SEQUENCE = [("A", 8, False), ("B", 2, True), ("A", 8, True), ("C", 5, False)]
COVERAGE_MIN = 0.005  # the least fraction of a plane's output pixels that read each of its levels 1..T


def coverage(ctx, in_dims, out_dims, max_level):
    """{(plane, level): fraction of the plane's output pixels whose level or next level (weight > 0) is `level`}."""
    out = {}
    for p, ((iw, ih), (ow, oh)) in enumerate(zip(in_dims, out_dims)):
        _, _, lv, w = t360.camera_mip_maps(ctx, VIEW_POSE, VIEW_CAMERA, (max_level, 0.0), iw, ih, ow, oh)
        top = len(t360.mip_level_sizes(iw, ih, max_level)) - 1
        for level in range(1, top + 1):
            out[(p, level)] = float(((lv == level) | ((lv + 1 == level) & (w > 0))).mean())
    return out


def test_coverage_ledger():
    """Every level 1..T of every plane of every frame of the sequence is read by at least COVERAGE_MIN of its output."""
    ctx = _ctx("equirect", t360.CUBIC)
    for name, max_level, _ in SEQUENCE:
        luma, chroma = SIZES[name]
        cov = coverage(ctx, [luma, chroma, chroma], VIEW_OUT, max_level)
        for p, (w, h) in enumerate([luma, chroma, chroma]):
            top = len(t360.mip_level_sizes(w, h, max_level)) - 1
            assert top == min(max_level, 6 if p == 0 else 5) and all((p, lv) in cov for lv in range(1, top + 1)), (name, p, top)
        low = {k: v for k, v in cov.items() if v < COVERAGE_MIN}
        assert not low, (name, max_level, low)


def _frames(torch, order, seed):
    """MipFrames of the sequence entries `order`, each with its own planes."""
    return [MipFrame(torch, "equirect", 3, seed=seed + k, unaligned=SEQUENCE[i][2], in_dims=SIZES[SEQUENCE[i][0]], out_dims=VIEW_OUT)
            for k, i in enumerate(order)]


def _top_max(i):
    name, max_level, _ = SEQUENCE[i]
    return max(len(t360.mip_level_sizes(w, h, max_level)) - 1 for w, h in SIZES[name])


def _enqueue_and_check(torch, ctx, vft, frames, order, streams, what):
    torch.cuda.synchronize()
    n0 = t360.kernel_launch_count()
    for f, i, st in zip(frames, order, streams):
        assert vft.make_camera_mip_frame_call(f.in_planes, f.out_planes, f.dims)(VIEW_POSE, VIEW_CAMERA, (SEQUENCE[i][1], 0.0), st.cuda_stream)
    torch.cuda.synchronize()
    assert t360.kernel_launch_count() - n0 == sum(_top_max(i) + 1 for i in order)
    for k, (f, i) in enumerate(zip(frames, order)):
        want = f.want(ctx, None, VIEW_POSE, VIEW_CAMERA, (SEQUENCE[i][1], 0.0))
        for p, got in enumerate(f.host()):
            assert np.array_equal(got, want[p]), f"{what}: frame {k} ({SEQUENCE[i]}) plane {p}: {first_difference(got, want[p])}"


@pytest.mark.gpu
def test_size_and_level_changes_on_one_stream(torch_cuda):
    """The sequence twice on one stream, nothing synchronised between frames: every frame equals the oracle composite and
    takes T_max pyramid launches and one gather."""
    torch = torch_cuda
    ctx = _ctx("equirect", t360.CUBIC)
    vft = t360.VideoFrameTransform(ctx)
    st = torch.cuda.Stream()
    order = list(range(len(SEQUENCE))) * 2
    _enqueue_and_check(torch, ctx, vft, _frames(torch, order, 0), order, [st] * len(order), "one stream")
    vft.close()


@pytest.mark.gpu
def test_size_and_level_changes_on_two_streams(torch_cuda):
    """The sequence on two streams, interleaved and one frame apart (so the two slots hold different sizes and tap tables
    at every step), nothing synchronised: every frame equals the oracle composite."""
    torch = torch_cuda
    ctx = _ctx("equirect", t360.LINEAR)
    vft = t360.VideoFrameTransform(ctx)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    n = len(SEQUENCE)
    order = [i for k in range(2 * n) for i in (k % n, (k + 1) % n)]
    _enqueue_and_check(torch, ctx, vft, _frames(torch, order, 100), order, [streams[k % 2] for k in range(len(order))], "two streams")
    vft.close()
