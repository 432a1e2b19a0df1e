"""Per-frame gathers at production sizes: every instantiation of perFrameGatherKernel<K, FLAG, Positions>
(csrc/view_gather.cu) on frames large enough that its persistent tile loop wraps, against the oracle.

The other per-frame tests render outputs of about 97 x 65, twelve tiles: every CTA does one tile and stops.  Here every
case is a 3-plane yuv420p frame of the size the profiles time (7680 x 3840 equirect and cube-map inputs, 5760 x 2880
dual-fisheye inputs; 1920 x 1080 views, 2048 x 2048 domes, sphere and barrel layouts of 3840 x 1920 and the like), so that
  - the grid, min(numSMs x perSM, numTiles), is smaller than the frame's tiles whatever the occupancy: CTAs take a second
    tile (tile += gridDim.x), and go from luma to chroma tiles (which changes the plane's pyramid and photometry);
  - partial tiles (widths not a multiple of 32, heights not a multiple of the tile rows) come after a CTA's full ones;
  - the overlap statistics of the photometric sources pass 2^32, where a 32-bit accumulation would wrap.

What pins what:
  - the instantiation gate: the library's sm_90a functions list 100 perFrameGatherKernel instantiations, and the case
    table launches exactly that set (the launcher's choice of FLAG is restated per case: the barrel layout, the border,
    the rig or the pyramid);
  - the scheduling ledger: the launcher's tile arithmetic at 114 and 132 SMs and every occupancy the __launch_bounds__
    allow (kernels.cuh's gatherThreads and kViewRowsPerThread, read from the header);
  - the frames: each case once on the device into pre-filled outputs, every plane bit for bit against the oracle
    composite of the host twin the other tests use, and the statistics exactly as int64."""
import functools
import os
import re
import subprocess
from dataclasses import dataclass

import numpy as np
import pytest

import transform360_b200 as t360
from oracle import c_oracle as co
from oracle import ref_harness as rh
from tests.test_camera_aniso import aniso_pose, aniso_want
from tests.test_camera_mip import mip_want, wide_pose
from tests.test_camera_models import EQUIDISTANT, PANNINI, PINHOLE, STEREOGRAPHIC
from tests.test_camera_photo import photo_want, seam_pose
from tests.test_lens import _orientations, make_rig
from tests.test_lens_blend import composite as blend_composite
from tests.test_lens_photo import photo_composite, rig_photos
from tests.test_rectilinear import _poses
from tests.test_rig_motion import camera_motion_want, seeded_motion
from tests.test_stereo_camera import EQUIRECT as EQUIRECT_CAMERA
from tests.test_stereo_camera import eq_pose, stereo_rig, stereo_want
from tests.test_warp_map import dual_fisheye
from transform360_b200 import build as b

WRAP, TRANSPARENT = t360.BORDER_WRAP, t360.BORDER_TRANSPARENT
K_OF = {t360.NEAREST: 1, t360.LINEAR: 2, t360.CUBIC: 4, t360.LANCZOS4: 8}
INTERP_OF = {k: i for i, k in K_OF.items()}
SMS = (114, 132)  # H100 PCIe and SXM
STATS = 6
EQ_IN, CUBE_IN, FISH_IN, ONE_LENS_IN = (7680, 3840), (5760, 3840), (5760, 2880), (2880, 2880)
HD, HD_ODD, DOME, DOME_ODD = (1920, 1080), (1918, 1078), (2048, 2048), (2046, 2046)
NO_LOW_PASS = dict(enable_low_pass_filter=0)


def plane_dims(w, h):
    """The planes of a yuv420p frame: luma, then two chroma planes of half the size rounded up."""
    return [(w, h), ((w + 1) // 2, (h + 1) // 2), ((w + 1) // 2, (h + 1) // 2)]


@dataclass(frozen=True)
class Case:
    """One production-size frame call and the instantiation it launches.  source: the call (PerFrameSource);
    positions / k / flag: perFrameGatherKernel<k, flag, positions>; loop: the pinhole or the model loop of
    RectilinearPositions; ctx: the context's fields; args: the call's rig, seam, photometry, pose, minify, motion and
    maxProbes; unaligned: the luma input starts 1 byte into its buffer with an odd pitch."""
    source: str
    positions: str
    k: int
    flag: bool
    ctx: tuple
    inp: tuple
    out: tuple
    args: tuple = ()
    loop: str = ""
    unaligned: bool = False

    @property
    def id(self):
        flag = "" if self.positions == "FlatPositions" else f"-{str(self.flag).lower()}"
        loop = f"-{self.loop}" if self.loop else ""
        return f"{self.source}-K{self.k}{flag}{loop}-{self.inp[0]}x{self.inp[1]}-to-{self.out[0]}x{self.out[1]}"

    @property
    def interp(self):
        return INTERP_OF[self.k]

    @property
    def kw(self):
        return dict(self.args)

    def context(self, **extra):
        return t360.make_context(**dict(self.ctx), interpolation_alg=self.interp, **extra)


def _case(source, positions, k, flag, ctx, inp, out, loop="", unaligned=False, **args):
    return Case(source, positions, k, flag, tuple(sorted(dict(NO_LOW_PASS, **ctx).items())), inp, out, tuple(sorted(args.items())), loop,
                unaligned)


# ---- the case table ------------------------------------------------------------------------------------------------------
# Positions policy of each call, and what FLAG is for it (launchPerFrameGather)
POSITIONS = {"view": "FlatPositions", "sphere": "SpherePositions", "map": "MapPositions", "lens": "LensPositions",
             "lens_blend": "LensBlendPositions", "rectilinear": "RectilinearPositions", "camera_mip": "MipCameraPositions",
             "camera_aniso": "AnisoCameraPositions", "lens_photo": "LensPhotoPositions", "camera_photo": "CameraPhotoPositions",
             "stereo": "StereoCameraPositions", "lens_motion": "LensMotionPositions", "camera_motion": "CameraMotionPositions"}
BARREL_SIZES = {t360.LAYOUT_BARREL: (3842, 1538), t360.LAYOUT_BARREL_SPLIT: (2883, 1922)}
SPHERE_SIZES = {t360.LAYOUT_EQUIRECT: (3842, 1922), t360.LAYOUT_CUBEMAP_32: (3843, 2562), t360.LAYOUT_EAC_32: (3840, 2560),
                t360.LAYOUT_CUBEMAP_23_OFFCENTER: (2562, 3843)}
SPHERES = [t360.LAYOUT_EQUIRECT, t360.LAYOUT_CUBEMAP_32, t360.LAYOUT_EAC_32, t360.LAYOUT_CUBEMAP_23_OFFCENTER]
BARRELS = [t360.LAYOUT_BARREL, t360.LAYOUT_BARREL_SPLIT, t360.LAYOUT_BARREL, t360.LAYOUT_BARREL_SPLIT]
KS = (1, 2, 4, 8)
VIEW_OUTS = [HD_ODD, DOME, HD, DOME_ODD]  # (one per K; the dome makes every CTA take two tiles)
CAMERA_MODELS = [EQUIDISTANT, STEREOGRAPHIC, PANNINI, EQUIDISTANT]


def _rig_input(rig):
    return ONE_LENS_IN if rig == "single_200" else FISH_IN


def _layout_out(layout):
    return BARREL_SIZES.get(layout) or SPHERE_SIZES[layout]


def build_cases():
    cases = []
    add = lambda *a, **kw: cases.append(_case(*a, **kw))
    for i, k in enumerate(KS):
        # FLAT_FIXED: no flag; equirect input
        add("view", "FlatPositions", k, False, dict(output_layout=t360.LAYOUT_FLAT_FIXED), EQ_IN, VIEW_OUTS[i], unaligned=i == 3,
            view=(-150.0 + 97.0 * i, -70.0 + 45.0 * i, 100.0 + 10 * i, 60.0 + 12 * i))
        for flag in (False, True):
            layout = (BARRELS if flag else SPHERES)[i]
            ox = _orientations(100 + 10 * k + flag, 1)[0]
            # sphere and barrel outputs of a posed context; one of a cube-map input
            cube = i == 2 and not flag
            add("sphere", "SpherePositions", k, flag, dict(output_layout=layout, **(dict(input_layout=t360.LAYOUT_CUBEMAP_32) if cube else {})),
                CUBE_IN if cube else EQ_IN, _layout_out(layout), unaligned=i == 1, pose=(*ox, 120.0, 110.0))
            # a caller's map: the dual-fisheye remap of test_warp_map, BORDER_WRAP or BORDER_TRANSPARENT
            add("map", "MapPositions", k, flag, {}, FISH_IN, [HD_ODD, (3840, 1920), DOME, DOME_ODD][i], unaligned=i == 0,
                map_pose=(30.0 * i - 40.0, 10.0 * flag - 5.0, 7.0 * i), border=TRANSPARENT if flag else WRAP)
            # lens rigs to sphere and barrel layouts
            rig = ["single_200", "pair_190", "tilted", "pair_190"][i]
            add("lens", "LensPositions", k, flag, dict(output_layout=layout), _rig_input(rig), _layout_out(layout), unaligned=i == 2,
                rig=rig, orientation=ox)
            add("lens_blend", "LensBlendPositions", k, flag, dict(output_layout=layout), FISH_IN, _layout_out(layout), unaligned=i == 3,
                rig=["pair_190", "tilted"][i % 2], seam=[4.0, 10.0, 2.0, 25.0][i], orientation=ox)
            mode = [("single_200", 0.0), ("pair_190", 0.0), ("tilted", 8.0), ("pair_190", 4.0)][(i + flag) % 4]
            photo = ["falloff", "clamps"][(i + flag) % 2] if mode[0] != "single_200" else "falloff"
            add("lens_photo", "LensPhotoPositions", k, flag, dict(output_layout=layout), _rig_input(mode[0]), _layout_out(layout),
                unaligned=i == 0, rig=mode[0], seam=mode[1], photo=photo, orientation=ox)
            add("lens_motion", "LensMotionPositions", k, flag, dict(output_layout=layout), _rig_input(mode[0]), _layout_out(layout),
                unaligned=i == 1, rig=mode[0], seam=mode[1], photo="falloff", orientation=ox, motion=(4 + 4 * i, 1.5 + i))
            # camera views: the context's input (equirect or cube map) or a rig (LENS)
            rig = ["pair_190", "single_200", "tilted", "pair_190"][i] if flag else None
            name = rig or ["equirect", "cubemap_32", "equirect", "cubemap_32"][i]
            inp = _rig_input(rig) if rig else (EQ_IN if name == "equirect" else CUBE_IN)
            for loop, out in (("pinhole", [HD, DOME_ODD, HD_ODD, DOME][i]), ("model", [DOME, HD_ODD, DOME_ODD, HD][i])):
                add("rectilinear", "RectilinearPositions", k, flag, dict(_input_ctx(name)), inp, out, loop=loop, unaligned=i == 3 and loop == "model",
                    rig=rig, camera=PINHOLE if loop == "pinhole" else CAMERA_MODELS[i], pose_seed=1000 + 17 * k + 3 * flag + (loop == "model"))
            add("camera_mip", "MipCameraPositions", k, flag, dict(_input_ctx(name)), inp, [DOME_ODD, HD, DOME, HD_ODD][i], unaligned=i == 2,
                rig=rig, camera=CAMERA_MODELS[(i + flag) % 4], pose_seed=2000 + 17 * k + flag, minify=[(8, 0.0), (4, -1.0), (8, 1.5), (3, 0.5)][i])
            # (maxProbes x output pixels bounded: 4 probes at 1080p and on a dome, 16 on 1280 x 1280, which still wraps)
            probes, out = [(4, HD_ODD), (16, (1282, 1282)), (4, DOME), (2, HD)][i]
            add("camera_aniso", "AnisoCameraPositions", k, flag, dict(_input_ctx(name)), inp, out, unaligned=i == 0, rig=rig,
                camera=[EQUIDISTANT, EQUIRECT_CAMERA, PINHOLE, PANNINI][(i + flag) % 4], pose_seed=3000 + 17 * k + flag, max_probes=probes,
                minify=[(8, 0.0), (4, -1.0), (8, 0.5), (2, 0.0)][i])
            # rigs with photometry through a camera view; MIP: a pyramid (FLAG is "some plane has a level").  (The oracle composites
            # every level of both lenses twice: the pyramid cases of the motion and stereo views stay at 1080p.)
            minify = [(8, 0.0), (3, 0.0), (4, 1.0), (8, -0.5)][i] if flag else None
            rig, seam = [("pair_190", 0.0), ("pair_190", 4.0), ("single_200", 0.0), ("pair_190", 10.0)][(i + flag) % 4]
            add("camera_photo", "CameraPhotoPositions", k, flag, dict(_input_ctx(rig)), _rig_input(rig), [DOME, HD_ODD, HD, DOME_ODD][i],
                unaligned=i == 1, rig=rig, seam=seam, photo="falloff", camera=CAMERA_MODELS[i], pose_seed=4000 + 17 * k + flag, minify=minify)
            out = [HD, HD_ODD, HD_ODD, HD][i] if flag else [HD, DOME_ODD, HD_ODD, DOME][i]
            add("camera_motion", "CameraMotionPositions", k, flag, dict(_input_ctx(rig)), _rig_input(rig), out, unaligned=i == 2, rig=rig,
                seam=seam, photo="falloff", camera=CAMERA_MODELS[(i + 1) % 4], pose_seed=5000 + 17 * k + flag, minify=minify,
                motion=(2 + 4 * i, 1.0 + i))
            fmt = [t360.STEREO_FORMAT_MONO, t360.STEREO_FORMAT_LR, t360.STEREO_FORMAT_TB, t360.STEREO_FORMAT_LR][i]
            out = [HD, HD_ODD, HD, HD_ODD][i] if flag else [DOME_ODD, HD, DOME, HD_ODD][i]
            add("stereo", "StereoCameraPositions", k, flag, dict(_input_ctx("pair_190"), output_stereo_format=fmt), FISH_IN, out,
                unaligned=i == 3, rig=["stereo_190", "swapped"][(i + flag) % 2], photo="falloff",
                camera=[EQUIRECT_CAMERA, EQUIDISTANT, EQUIRECT_CAMERA, PINHOLE][i], pose_seed=6000 + 17 * k + flag, minify=minify)
    return cases


def _input_ctx(name):
    """test_rectilinear's contexts of the camera views' inputs (a rig's: a mono equirect context)."""
    return {"cubemap_32": dict(input_layout=t360.LAYOUT_CUBEMAP_32, input_expand_coef=1.04)}.get(name, dict(input_layout=t360.LAYOUT_EQUIRECT))


CASES = build_cases()
CASE_IDS = [c.id for c in CASES]


# ---- the scheduling ledger -------------------------------------------------------------------------------------------------
@functools.lru_cache(None)
def launch_constants():
    """(threads per CTA, tile rows) of each K from kernels.cuh: gatherThreads(k) and viewTileRows(k) = gatherThreads(k) / 32
    x kViewRowsPerThread."""
    text = (b.CSRC / "kernels.cuh").read_text()
    threads = re.search(r"constexpr int gatherThreads\(int k\) \{ return k == 8 \? (\d+) : (\d+); \}", text)
    rows = re.search(r"constexpr int kViewRowsPerThread = (\d+);", text)
    assert threads and rows, "gatherThreads / kViewRowsPerThread not found in kernels.cuh"
    assert "viewTileRows(int k) { return gatherThreads(k) / 32 * kViewRowsPerThread; }" in text
    out = {}
    for k in KS:
        t = int(threads.group(1)) if k == 8 else int(threads.group(2))
        out[k] = (t, t // 32 * int(rows.group(1)))
    return out


def plane_tiles(case):
    """Tiles of each plane, in plane order, as launchPerFrameGather counts them."""
    rows = launch_constants()[case.k][1]
    return [((w + 31) // 32) * ((h + rows - 1) // rows) for w, h in plane_dims(*case.out)]


def max_per_sm(k):
    return 2048 // launch_constants()[k][0]


def schedule(case, sms, per_sm):
    """(grid, every CTA takes >= 2 tiles, some CTA takes tiles of two planes) of the launch at sms SMs and per_sm CTAs per SM."""
    tiles = plane_tiles(case)
    total = sum(tiles)
    grid = min(sms * per_sm, total)
    first = np.arange(grid)
    last = first + (total - 1 - first) // grid * grid
    starts = np.cumsum([0] + tiles[:-1])
    plane = lambda t: np.searchsorted(starts, t, side="right") - 1
    return grid, total >= 2 * grid, bool((plane(first) != plane(last)).any())


def test_case_table_sizes_and_pitches():
    """Every source has an output whose luma and chroma widths are not multiples of 32 and whose heights are not multiples
    of the tile rows, and a case with an unaligned luma plane; cases are unique."""
    assert len(set(CASE_IDS)) == len(CASE_IDS), "duplicate case ids"
    for source in POSITIONS:
        mine = [c for c in CASES if c.source == source]
        rows = lambda c: launch_constants()[c.k][1]
        odd = [c for c in mine if all(w % 32 and h % rows(c) for w, h in plane_dims(*c.out))]
        assert odd, f"{source}: no output with widths off a multiple of 32 and heights off the tile rows in every plane"
        assert any(c.unaligned for c in mine), f"{source}: no unaligned input plane"
    rect = {(c.k, c.flag, c.loop) for c in CASES if c.source == "rectilinear"}
    assert rect == {(k, f, loop) for k in KS for f in (False, True) for loop in ("pinhole", "model")}


def test_scheduling_ledger_every_case_wraps():
    """At 114 and 132 SMs and every occupancy from 1 to 2048 / gatherThreads(K) CTAs per SM, every case has more tiles
    than CTAs; per source, some case has every CTA take two tiles or more at every occupancy, and some case has a CTA take
    tiles of two planes at every occupancy."""
    two, planes = set(), set()
    for c in CASES:
        every_two = crosses = True
        for sms in SMS:
            for per_sm in range(1, max_per_sm(c.k) + 1):
                grid, all_two, cross = schedule(c, sms, per_sm)
                assert sum(plane_tiles(c)) > grid, f"{c.id}: {sum(plane_tiles(c))} tiles for a grid of {grid} at {sms} SMs x {per_sm}"
                every_two &= all_two
                crosses &= cross
        if every_two:
            two.add(c.source)
        if crosses:
            planes.add(c.source)
    assert two == set(POSITIONS), f"no case where every CTA takes two tiles: {sorted(set(POSITIONS) - two)}"
    assert planes == set(POSITIONS), f"no case where a CTA crosses planes: {sorted(set(POSITIONS) - planes)}"


def test_scheduling_ledger_arithmetic():
    """The ledger's numbers for the sizes the table is built from: a 1920 x 1080 frame has 1560 tiles at K <= 4 and 840 at
    K = 8, a 2048 x 2048 dome 3072 and 1536; 132 SMs take at most 1056 and 528 CTAs."""
    hd = lambda k: _case("view", "FlatPositions", k, False, {}, EQ_IN, HD)
    dome = lambda k: _case("view", "FlatPositions", k, False, {}, EQ_IN, DOME)
    assert [sum(plane_tiles(hd(k))) for k in KS] == [1560, 1560, 1560, 840]
    assert [sum(plane_tiles(dome(k))) for k in KS] == [3072, 3072, 3072, 1536]
    assert [132 * max_per_sm(k) for k in KS] == [1056, 1056, 1056, 528]
    assert schedule(dome(4), 132, 8) == (1056, True, True)
    assert schedule(hd(8), 132, 4)[:2] == (528, False)


# ---- the instantiation gate ------------------------------------------------------------------------------------------------
def library_instantiations():
    """(Positions, K, FLAG) of every perFrameGatherKernel function in the library's sm_90a code (cuobjdump's function list,
    demangled by cu++filt from the same toolkit)."""
    from transform360_b200.handler import LIB_PATH
    tools = os.path.dirname(b.nvcc_path())
    elf = subprocess.run([os.path.join(tools, "cuobjdump"), "--list-elf", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    assert "sm_90a" in elf, elf
    usage = subprocess.run([os.path.join(tools, "cuobjdump"), "-res-usage", str(LIB_PATH)], capture_output=True, text=True, check=True).stdout
    names = [m.group(1) for m in re.finditer(r"^\s*Function (\S*perFrameGatherKernel\S*?):", usage, re.M)]
    demangled = subprocess.run([os.path.join(tools, "cu++filt")], input="\n".join(names), capture_output=True, text=True, check=True).stdout
    found = []
    for line in demangled.splitlines():
        m = re.search(r"perFrameGatherKernel<\(int\)(\d+), \(bool\)([01]), t360::[^:]+::(\w+)>", line)
        assert m, f"unparsed instantiation {line!r}"
        found.append((m.group(3), int(m.group(1)), m.group(2) == "1"))
    return found


def test_instantiation_gate():
    """The library holds 100 perFrameGatherKernel instantiations -- FlatPositions for the 4 K, the other twelve policies
    for 4 K x FLAG -- and the case table launches exactly those."""
    t360.load()
    found = library_instantiations()
    assert len(found) == len(set(found)) == 100, f"{len(found)} perFrameGatherKernel instantiations in the library"
    table = {(c.positions, c.k, c.flag) for c in CASES}
    missing = sorted(set(found) - table)
    extra = sorted(table - set(found))
    assert not missing, f"instantiations without a production-size case: {missing}"
    assert not extra, f"cases of instantiations the library does not have: {extra}"


# ---- the oracle ------------------------------------------------------------------------------------------------------------
def _pattern(w, h, p):
    """What an output holds before the frame: a non-zero pattern."""
    i, j = np.mgrid[:h, :w]
    return (((i * 7 + j * 13 + 29 * p) % 251) + 1).astype(np.uint8)


def _rig(case):
    name = case.kw.get("rig")
    if name is None:
        return None
    return stereo_rig(name, seed=case.k) if case.source == "stereo" else make_rig(name, seed=case.k + 7 * case.flag)


def _lens_call(case):
    """A rig's call: BORDER_TRANSPARENT into the pre-fill, the call's own 128 in the chroma planes."""
    return case.kw.get("rig") is not None


def device_prefill(case):
    """What each output plane holds before the call: the pattern; a caller's map's chroma planes 128, as the planned path
    starts them."""
    dims = plane_dims(*case.out)
    return [_pattern(w, h, p) if p == 0 or case.source != "map" else np.full((h, w), 128, np.uint8) for p, (w, h) in enumerate(dims)]


def oracle_prefill(case):
    """What BORDER_TRANSPARENT leaves in each plane: the pre-fill, the chroma planes of a rig's call 128 (the call's own
    pre-fill)."""
    fill = device_prefill(case)
    if _lens_call(case):
        fill[1:] = [np.full_like(f, 128) for f in fill[1:]]
    return fill


def sources(case):
    return [co.noise_plane(w, h, plane=p, frame=case.k + 4 * case.flag) for p, (w, h) in enumerate(plane_dims(*case.inp))]


def _photometry(case, rig):
    return rig_photos(rig)[case.kw["photo"]]


def _motion(case):
    n, scale = case.kw["motion"]
    return seeded_motion(np.random.default_rng(n * 31 + case.k), n, scale)


def _camera_pose(case):
    """A seeded pose and camera of the case's model (test_rectilinear's poses for the pinhole, the mip tests' wide poses for
    the others; along the seam of a pair for the photometric views)."""
    model, seed = case.kw["camera"], case.kw["pose_seed"]
    if case.source == "rectilinear" and model == PINHOLE:
        return _poses(seed, 1, *case.out)[0], (PINHOLE, 0.0)
    if case.source == "camera_aniso":
        return aniso_pose(model, seed)
    if case.source == "stereo":
        return eq_pose(seed, model)
    if case.source in ("camera_photo", "camera_motion") and case.kw["rig"] != "single_200":
        return seam_pose(model, seed)
    return wide_pose(model, seed)


def _pose_ctx(case, pose):
    return dict(dict(case.ctx), interpolation_alg=case.interp, fixed_yaw=pose[0], fixed_pitch=pose[1], fixed_roll=pose[2],
                fixed_hfov=pose[3], fixed_vfov=pose[4])


def _view_pose(case):
    yaw, pitch, hfov, vfov = case.kw["view"]
    return yaw, pitch, 0.0, hfov, vfov


def _warp_maps(case):
    yaw, pitch, roll = case.kw["map_pose"]
    return [dual_fisheye(w, h, iw, ih, yaw=yaw, pitch=pitch, roll=roll) for (w, h), (iw, ih) in zip(plane_dims(*case.out), plane_dims(*case.inp))]


def oracle(case, srcs):
    """The oracle's planes of the case's frame and, for the photometric calls, its int64 statistics per plane."""
    ctx, interp, kw = case.context(), case.interp, case.kw
    outs, ins = plane_dims(*case.out), plane_dims(*case.inp)
    fill = oracle_prefill(case)
    rig = _rig(case)
    if case.source in ("view", "sphere"):
        pose = _view_pose(case) if case.source == "view" else kw["pose"]
        octx = rh.default_context(**_pose_ctx(case, pose))
        plans = [co.OraclePlan(octx, *ins[min(p, 1)], *outs[min(p, 1)]) for p in range(2)]
        return [co.transform_plane(octx, plans[min(p, 1)], srcs[p], *outs[p], map_index=min(p, 1), prefill=fill[p]) for p in range(3)], None
    if case.source == "map":
        maps = _warp_maps(case)
        return [co.remap_u8(srcs[p], maps[p], interp, kw["border"], fill[p].copy()) for p in range(3)], None
    if case.source == "lens":
        return [co.remap_u8(srcs[p], t360.lens_map(ctx, rig, kw["orientation"], *ins[p], *outs[p]), interp, TRANSPARENT, fill[p].copy())
                for p in range(3)], None
    if case.source == "lens_blend":
        return [blend_composite(srcs[p], *t360.lens_blend_maps(ctx, rig, kw["seam"], kw["orientation"], *ins[p], *outs[p]), interp, fill[p])
                for p in range(3)], None
    if case.source in ("lens_photo", "lens_motion"):
        ph = _photometry(case, rig)
        want, sums = [], []
        for p in range(3):
            if case.source == "lens_photo":
                maps = t360.lens_photo_maps(ctx, rig, ph, kw["seam"], kw["orientation"], p, *ins[p], *outs[p])
            else:
                maps = t360.lens_motion_maps(ctx, rig, ph, kw["seam"], kw["orientation"], _motion(case), p, *ins[p], *outs[p])
            out, s = photo_composite(srcs[p], maps, interp, fill[p], ph, p)
            want.append(out)
            sums.append(s)
        return want, sums
    pose, cam = _camera_pose(case)
    if case.source == "rectilinear":
        want = []
        for p in range(3):
            if kw["camera"] == PINHOLE:
                m = t360.rectilinear_map(ctx, pose, *ins[p], *outs[p], rig)
            else:
                m = t360.camera_map(ctx, pose, cam, *ins[p], *outs[p], rig)
            want.append(co.remap_u8(srcs[p], m, interp, WRAP) if rig is None else co.remap_u8(srcs[p], m, interp, TRANSPARENT, fill[p].copy()))
        return want, None
    if case.source == "camera_mip":
        return mip_want(ctx, rig, pose, cam, kw["minify"], srcs, outs, fill if rig is not None else None), None
    if case.source == "camera_aniso":
        return aniso_want(ctx, rig, pose, cam, kw["minify"], kw["max_probes"], srcs, outs, fill if rig is not None else None), None
    ph = _photometry(case, rig)
    if case.source == "camera_photo":
        return photo_want(ctx, rig, ph, kw["seam"], pose, cam, kw["minify"], srcs, outs, fill)
    if case.source == "stereo":
        return stereo_want(ctx, rig, ph, pose, cam, kw["minify"], srcs, outs, fill)
    return camera_motion_want(pytest.MonkeyPatch, _motion(case), ctx, rig, ph, kw["seam"], pose, cam, kw["minify"], srcs, outs, fill)


def test_statistics_pass_2_to_the_32():
    """Some lens-photo, camera-photo, stereo, lens-motion and camera-motion case has an overlap sum above 2^32 in the
    oracle's statistics: a 32-bit accumulation anywhere between a thread's sums and the 64-bit totals would show."""
    for source, name in BIG_STATS.items():
        case = CASES[CASE_IDS.index(name)]
        assert case.source == source
        _, sums = oracle(case, sources(case))
        assert max(max(s) for s in sums) > 2 ** 32, f"{name}: the largest statistics sum is {max(max(s) for s in sums)}"


# the case of each photometric source whose statistics pass 2^32
BIG_STATS = {"lens_photo": "lens_photo-K4-false-5760x2880-to-3840x2560", "lens_motion": "lens_motion-K4-false-5760x2880-to-3840x2560",
             "camera_photo": "camera_photo-K1-true-5760x2880-to-2048x2048", "stereo": "stereo-K2-false-5760x2880-to-1920x1080",
             "camera_motion": "camera_motion-K2-false-5760x2880-to-2046x2046"}


# ---- on the GPU ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the GPU tests must run on an H100 (there is no CPU fallback to test)")
    return torch


def _pitch(w):
    return (w + 255) // 256 * 256 + 64  # pitched planes, not 256-byte aligned rows


class DeviceFrame:
    """The case's source planes on the device (the luma plane 1 byte into its buffer with an odd pitch where the case says
    unaligned) and its pre-filled outputs."""

    def __init__(self, torch, case, srcs):
        self.case = case
        self.d_src, self.in_planes = [], []
        for p, s in enumerate(srcs):
            h, w = s.shape
            if case.unaligned and p == 0:
                pitch = _pitch(w) + 1
                flat = np.zeros((h + 1) * pitch, np.uint8)
                flat[1:1 + h * pitch].reshape(h, pitch)[:, :w] = s
                t = torch.from_numpy(flat).cuda()
                self.in_planes.append((t.data_ptr() + 1, pitch))
            else:
                t = torch.zeros((h, _pitch(w)), dtype=torch.uint8, device="cuda")
                t[:, :w] = torch.from_numpy(np.ascontiguousarray(s)).cuda()
                self.in_planes.append((t.data_ptr(), t.stride(0)))
            self.d_src.append(t)
        self.outs = []
        for (w, h), fill in zip(plane_dims(*case.out), device_prefill(case)):
            o = torch.zeros((h, _pitch(w)), dtype=torch.uint8, device="cuda")
            o[:, :w] = torch.from_numpy(fill).cuda()
            self.outs.append(o)
        self.out_planes = [(o.data_ptr(), o.stride(0)) for o in self.outs]
        self.dims = [(*i, *o) for i, o in zip(plane_dims(*case.inp), plane_dims(*case.out))]

    def host(self):
        return [o[:, :w].cpu().numpy() for o, (w, _) in zip(self.outs, plane_dims(*self.case.out))]


def run(torch, case, f, vft, stats, keep):
    """Enqueues the case's frame call on the default stream; stats: the device address of [3][6] int64 sums."""
    kw, ctx = case.kw, case.context()
    rig = _rig(case)
    if case.source in ("view", "sphere"):
        for idx in (0, 1):
            assert vft.generateMapForPlane(*f.dims[idx], idx)
        if case.source == "view":
            return vft.make_view_frame_call(f.in_planes, f.out_planes, f.dims)(kw["view"])
        return vft.make_pose_frame_call(f.in_planes, f.out_planes, f.dims)(kw["pose"])
    if case.source == "map":
        keep.extend(torch.from_numpy(m).cuda() for m in _warp_maps(case))
        return vft.make_remap_frame_call(f.in_planes, f.out_planes, f.dims, kw["border"])(keep[-3:])
    if case.source == "lens":
        return vft.make_lens_frame_call(f.in_planes, f.out_planes, f.dims)(rig, kw["orientation"])
    if case.source == "lens_blend":
        return vft.make_lens_blend_frame_call(f.in_planes, f.out_planes, f.dims)(rig, kw["seam"], kw["orientation"])
    if case.source == "lens_photo":
        return vft.make_lens_photo_frame_call(f.in_planes, f.out_planes, f.dims)(rig, _photometry(case, rig), kw["seam"], kw["orientation"], 0, stats)
    if case.source == "lens_motion":
        return vft.make_lens_motion_frame_call(f.in_planes, f.out_planes, f.dims)(rig, _photometry(case, rig), kw["seam"], kw["orientation"],
                                                                                  _motion(case), 0, stats)
    pose, cam = _camera_pose(case)
    if case.source == "rectilinear":
        if kw["camera"] == PINHOLE:
            return vft.make_rectilinear_frame_call(f.in_planes, f.out_planes, f.dims)(pose, 0, rig)
        return vft.make_camera_frame_call(f.in_planes, f.out_planes, f.dims)(pose, cam, 0, rig)
    if case.source == "camera_mip":
        return vft.make_camera_mip_frame_call(f.in_planes, f.out_planes, f.dims)(pose, cam, kw["minify"], 0, rig)
    if case.source == "camera_aniso":
        return vft.make_camera_aniso_frame_call(f.in_planes, f.out_planes, f.dims)(pose, cam, kw["minify"], kw["max_probes"], 0, rig)
    ph = _photometry(case, rig)
    if case.source == "camera_photo":
        return vft.make_camera_photo_frame_call(f.in_planes, f.out_planes, f.dims)(rig, ph, kw["seam"], pose, cam, kw["minify"], 0, stats)
    if case.source == "stereo":
        return vft.make_stereo_camera_frame_call(f.in_planes, f.out_planes, f.dims)(rig, ph, pose, cam, kw["minify"], 0, stats)
    return vft.make_camera_motion_frame_call(f.in_planes, f.out_planes, f.dims)(rig, ph, kw["seam"], pose, cam, kw["minify"], _motion(case), 0,
                                                                                stats)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_frame_equals_the_oracle(case, torch_cuda):
    """The case's frame call, once, into pre-filled outputs: every plane equals the oracle bit for bit (pixels
    BORDER_TRANSPARENT leaves alone keep the pre-fill), the statistics equal its int64 sums, and the device's SM count puts
    the launch in the regime the ledger counts on."""
    torch = torch_cuda
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    total = sum(plane_tiles(case))
    assert total > sms * max_per_sm(case.k), f"{total} tiles do not wrap a grid of {sms} SMs x {max_per_sm(case.k)}"
    if all(schedule(case, n, max_per_sm(case.k))[1] for n in SMS):
        assert total >= 2 * sms * max_per_sm(case.k), f"{total} tiles: a CTA of {sms} SMs x {max_per_sm(case.k)} takes one tile"
    srcs = sources(case)
    f = DeviceFrame(torch, case, srcs)
    stats = torch.full((3, STATS), -1, dtype=torch.int64, device="cuda")
    keep = []
    vft = t360.VideoFrameTransform(case.context())
    torch.cuda.synchronize()
    n0 = t360.kernel_launch_count()
    assert run(torch, case, f, vft, stats.data_ptr(), keep), f"{case.id}: the call was refused"
    torch.cuda.synchronize()
    assert t360.kernel_launch_count() > n0
    got = f.host()
    got_sums = stats.cpu().numpy()
    vft.close()
    want, sums = oracle(case, srcs)
    for p, (g, w) in enumerate(zip(got, want)):
        if not np.array_equal(g, w):
            bad = np.argwhere(g != w)
            rows = launch_constants()[case.k][1]
            tiles = sorted({(int(i) // rows, int(j) // 32) for i, j in bad[:4096]})[:8]
            raise AssertionError(f"{case.id}: plane {p}: {len(bad)} px differ from the oracle, first at (row, col) {bad[0].tolist()}; "
                                 f"tiles (row, col) {tiles}")
    if sums is not None:
        for p in range(3):
            assert got_sums[p].tolist() == sums[p], f"{case.id}: plane {p} statistics {got_sums[p].tolist()} != {sums[p]}"
    else:
        assert (got_sums == -1).all()
