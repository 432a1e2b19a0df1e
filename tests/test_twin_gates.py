"""The device build of every float function of the per-frame position chains against its host build, bit for bit.

The per-frame kernels (view_gather.cu) compute each pixel's sampling record with the T360_HD functions of flat_view.h,
libm_ports.h and oriented_view.h; the planner and the host twins compute the same records with their host build.  Each
float step is an explicit _rn intrinsic on the device and a plain operator under -ffp-contract=off on the host, and
libmAtan2f / libmAsinf / libmAtanf (ports of glibc) and sincCos (+ - * / only) are written so both builds agree.  Seven
gates on one harness (tests/twin_gate.cuh) check that rule directly: the same probe code runs on the device and on the
host, and every output word must match (every NaN equals every NaN, nothing else is excused).
  - tests/twin_gate.cu, the position chains:
      - tier A, every 32-bit pattern: libmAtanf, libmAsinf, fSqrt, sincCos, truncToInt, roundHalfEven, quantizeAxis
        (K = 1, 2, 4, 8);
      - tier B, structured families of 2^27-2^28 inputs (all floats in [-1, 2] for toPixel, every j < n <= 16384 for
        pixelCentre): libmAtan2f (tests/atan2_pairs.h, the pairs the glibc gate of test_oriented.py draws), rotateHD,
        rayToSphereHD, warpOffCentreHD, sphereInputHD, lensPosition, lensBlendPosition, cameraRay;
      - tier C, 2^26 (geometry, pixel) samples per chain over seeded contexts and their buildSphereTables tables:
        flatSample, sphereSample, lensSample, lensBlendSample and rectilinearSample in every instantiation the kernels use.
  - tests/mip_twin_gate.cu, the anti-aliased camera views: mipLevelOf for every 32-bit pattern of rho^2;
    rayDifferential for every camera model, equirectJacobian, cubeInputFace with cubeJacobian, lensJacobian (rays on a
    lens's axis, rho = 0, included) and mipScale over 2^26 drawn inputs each; mipCameraPoint and mipCameraSample, LENS =
    false and true, over 2^24 (geometry, pixel) samples each.
  - tests/photo_twin_gate.cu, the lens photometry: lensGain, the falloff and Gq's quantisation, over 2^28 drawn lens
    hits, falloffs and gains; lensPhotoPosition over 2^26 drawn rig directions, hard (closer lens only, or both) and
    feathered seams; lensPhotoSample, BARREL = true and false, over 2^24 (geometry, pixel) samples each of every sphere
    output layout.
  - tests/camera_photo_twin_gate.cu, the camera views of a rig with photometry: lensJacobian of a chosen lens (the
    farther one included) over 2^26 drawn rig directions; cameraPhotoPoint and both instantiations of cameraPhotoSample
    over 2^24 (geometry, camera, rig, photometry, pixel) samples each, with a ledger of rays on a used lens's axis, a
    lens's thetaMax, belt pixels and the back-axis infinite footprint.
  - tests/stereo_camera_twin_gate.cu, the stereo rigs and the equirect camera: cameraRay's equirect case over 2^26 drawn
    pixels, and the stereo chain (cameraPhotoPoint<MIP, true> and both instantiations of cameraPhotoSample<MIP, true>)
    over 2^24 samples each, with a ledger of the eye boundaries, each lens's thetaMax, lon = +-pi, lat near +-90, TB with
    vflip and the back-axis infinite footprint.
  - tests/motion_twin_gate.cu, the rolling-shutter lens rigs: motionLens over 2^26 drawn tables and readout times;
    lensMotionPosition over 2^24 drawn rig directions, motions and readouts; lensMotionSample (BARREL = true and false)
    and cameraMotionSample (MIP = false and true) over 2^22 samples each.
  - tests/aniso_twin_gate.cu, the anisotropic camera views: anisoLevelOf over 2^28 drawn footprint axes; anisoFootprint,
    anisoCameraPoint and anisoCameraSample, LENS = false and true, over 2^24 (geometry, pixel) samples each.
The host builds are the ones test_oriented.py pins to glibc, test_camera_models.py to double, test_camera_mip.py to
camera_map and a float64 model, test_lens_photo.py to lens_map, lens_blend_maps and a float64 model,
test_camera_photo.py, test_stereo_camera.py and test_camera_aniso.py to the camera twins they extend and float64
models, test_rig_motion.py to the photometric twins and a float64 fixed point, and the planner tests to the reference, so
those pins carry over to the device.

Without a GPU: each gate builds with the library's nvcc flags (transform360_b200/build.py), its host half gives the same
fingerprints on one thread and on many, its fingerprint and drill-down path reports exactly one injected bit flip, and
the ledgers show the input families reach every class they are meant to cover (a generator change that stops reaching
one fails here).
"""
from __future__ import annotations

import os
import re
import subprocess
import time
from dataclasses import dataclass, field

import pytest

from transform360_b200 import build as b

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
THREADS = max(8, os.cpu_count() or 1)


@dataclass(frozen=True)
class Gate:
    probes: tuple  # the --host-only probes, in order (twin_gate's tier A runs in the full gate only)
    out_words: int  # the compared words per element (kOut)
    ledger: dict = field(default_factory=dict)  # {(probe, class): the least count}, every class the gate's kInfo names


def classes(probes, names, least=1):
    """Ledger entries: {(probe, class): least} for each probe of `probes` (one name or a tuple) and each class in the
    space-separated `names`."""
    return {(p, c): least for p in ((probes,) if isinstance(probes, str) else probes) for c in names.split()}


_TWIN_PROBES = ("libmAtan2f", "pixelCentre", "toPixel", "rotateHD", "rayToSphereHD", "warpOffCentreHD", "sphereInputHD", "lensPosition",
                "lensBlendPosition0", "lensBlendPosition1", "cameraRay", "flatSample", "sphereSample<BARREL>", "sphereSample<plain>",
                "lensSample<BARREL>", "lensSample<plain>", "lensBlendSample<BARREL>", "lensBlendSample<plain>", "rectilinearSample<ctx,any>",
                "rectilinearSample<ctx,pinhole>", "rectilinearSample<lens,any>", "rectilinearSample<lens,pinhole>")
_LAYOUTS = "cube32 cube23 eac equirect"  # the sphere layouts of a chain's plain instantiation; BARREL adds the barrels
_BARREL_LAYOUTS = _LAYOUTS + " barrel barrelSplit"
_CHAIN = "offCentreHorizontal offCentreFull splitLR splitTBvflip packLR packTB cubeInput oddMap oddInput K1 K2 K4 K8"
_CAMERA_MODELS = "pinhole equidistant stereographic pannini"
GATES = {
    "twin_gate": Gate(
        _TWIN_PROBES, 4,
        ledger={  # pixelCentre and toPixel walk fixed grids and name no class
            **classes("libmAtan2f", "nan xIsOne zero inf ratioAbove2^60 negativeXRatioBelow2^-60 atanfTiny atanfBelow7/16 atanfBelow11/16 "
                                    "atanfBelow19/16 atanfBelow39/16 atanfBelow2^24 atanfAbove2^24 atanfNearSplit"),
            **classes("rotateHD", "angles rawMatrix signedZeroQ"),
            **classes("rayToSphereHD", "discNotPositive discBelowAlong ordinary"),
            **classes("warpOffCentreHD", "horizontalWarped horizontalUnwarped fullWarped fullUnwarped"),
            **classes("sphereInputHD", "cutPlusZero cutMinusZero pole barrelClampLow barrelClampHigh barrelNaN packLR0 packLR1 packTB0 packTB1 "
                                       "face0 face1 face2 face3 face4 face5 gIsOne majorIsHalf noFace noFaceWithoutNaN pickedMajorIsHalf"),
            **classes("lensPosition", "oneLens secondLens z1EqualsZ0 covered uncovered rhoZero thetaIsThetaMax thetaMaxPi"),
            **classes(("lensBlendPosition0", "lensBlendPosition1"), "bothCoveredW0 bothCoveredW256 ramp tie only0 only1 neither"),
            **classes("cameraRay", "equidistantRho0 equidistantRhoAbovePi/2 equidistantRhoAbovePi stereoBelow1 stereoAt1 stereoAbove1 panniniD0 "
                                   "panniniD1 panniniKAbove1e7 equidistantZeroXY stereoZeroXY panniniZeroXY"),
            **classes("flatSample", f"{_CHAIN} fold noFold"),
            **classes("sphereSample<BARREL>", f"{_BARREL_LAYOUTS} {_CHAIN} deadZone"),
            **classes("sphereSample<plain>", f"{_LAYOUTS} {_CHAIN}"),
            **classes("lensSample<BARREL>", f"{_BARREL_LAYOUTS} {_CHAIN} covered uncovered"),
            **classes("lensSample<plain>", f"{_LAYOUTS} {_CHAIN} covered uncovered"),
            **classes("lensBlendSample<BARREL>", f"{_BARREL_LAYOUTS} {_CHAIN} w0 w256 ramp"),
            **classes("lensBlendSample<plain>", f"{_LAYOUTS} {_CHAIN} w0 w256 ramp"),
            **classes(("rectilinearSample<ctx,any>", "rectilinearSample<lens,any>"), f"{_CHAIN} {_CAMERA_MODELS}"),
            **classes(("rectilinearSample<ctx,pinhole>", "rectilinearSample<lens,pinhole>"), f"{_CHAIN} pinhole"),
        }),
    "mip_twin_gate": Gate(
        ("mipLevelOf", "rayDifferential", "equirectJacobian", "cubeJacobian", "lensJacobian", "mipScale", "mipCameraPoint<ctx>",
         "mipCameraPoint<lens>", "mipCameraSample<ctx>", "mipCameraSample<lens>"), 6),
    "photo_twin_gate": Gate(
        ("lensGain", "lensPhotoPosition", "lensPhotoSample<BARREL>", "lensPhotoSample<plain>"), 6,
        ledger=classes("lensGain", "r0 thetaMax nearBound clamp uncovered", 1000)),  # thousands of each edge class of the gain
    "camera_photo_twin_gate": Gate(
        ("lensJacobian<lens>", "cameraPhotoPoint", "cameraPhotoSample<MIP>", "cameraPhotoSample<plain>"), 11,
        # rays on a used lens's axis, a lens's thetaMax, belt pixels and the infinite footprint of a used lens's back axis
        ledger=classes("cameraPhotoPoint", "lensAxis thetaMax belt infiniteFootprint", 100)),
    "stereo_camera_twin_gate": Gate(
        ("cameraRay<equirect>", "cameraPhotoPoint<stereo>", "cameraPhotoSample<MIP,stereo>", "cameraPhotoSample<plain,stereo>"), 11,
        # lon = +-pi at hfov 360 and lat within 0.1 degree of +-90; the eye boundary columns and rows, each lens's thetaMax,
        # the flipped eye of a TB vflip view and the infinite footprint of a used lens's back axis
        ledger={**classes("cameraRay<equirect>", "lonPi latPole", 10000),
                **classes("cameraPhotoPoint<stereo>", "eyeBoundaryCol eyeBoundaryRow thetaMax0 thetaMax1 tbVflip infiniteFootprint", 10000)}),
    "motion_twin_gate": Gate(
        ("motionLens", "lensMotionPosition", "lensMotionSample<BARREL>", "lensMotionSample<plain>", "cameraMotionSample<plain>",
         "cameraMotionSample<MIP>"), 11,
        # the interpolation at t = 0, t = 1 and inner segment boundaries; t clamped at 0 and at 1, the first projection
        # covered with the last one not (the converse cannot happen: an uncovered projection keeps t), a projection on a
        # segment boundary, the hard seam, the feathered seam and both lenses
        ledger={**classes("motionLens", "t0 t1 boundary"),
                **classes("lensMotionPosition", "clampedAt0 clampedAt1 coveredThenUncovered segmentBoundary hard feathered bothLenses")}),
    "aniso_twin_gate": Gate(
        ("anisoLevelOf", "anisoFootprint<ctx>", "anisoFootprint<lens>", "anisoCameraPoint<ctx>", "anisoCameraPoint<lens>",
         "anisoCameraSample<ctx>", "anisoCameraSample<lens>"), 9,
        # aa == bb, an exact multiple of 256 between the axes, a zero and a denormal axis, a pole (inf or NaN) and N clamped
        # by maxProbes; the footprints take both axes; a probe row crosses a cube face edge and a two-lens rig's seam
        ledger={**classes("anisoLevelOf", "equal multipleOf256 zero denormal infNaN clamped"),
                **classes(("anisoFootprint<ctx>", "anisoFootprint<lens>"), "columnAxis rowAxis"),
                **classes(("anisoCameraPoint<ctx>", "anisoCameraSample<ctx>"), "faceChange"),
                **classes(("anisoCameraPoint<lens>", "anisoCameraSample<lens>"), "lensChange")}),
}
every_gate = pytest.mark.parametrize("gate", list(GATES), indirect=True)


def gate_command(name, out):
    """A gate's nvcc command: the library's architecture, optimisation and host flags (build.py)."""
    return [b.nvcc_path(), *b.ARCH, "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", b.HOST_FLAGS, "-I", os.path.join(ROOT, "include"),
            "-I", str(b.CSRC), os.path.join(ROOT, "tests", f"{name}.cu"), "-o", str(out)]


_built = {}


@pytest.fixture(scope="module")
def gate(request, tmp_path_factory):
    """(name, executable) of the gate the test is parametrised with.  Each gate is built once, in whatever order pytest
    sets the fixture up for its parameters."""
    name = request.param
    if name not in _built:
        exe = tmp_path_factory.mktemp(name) / name
        t0 = time.monotonic()
        r = subprocess.run(gate_command(name, exe), capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        print(f"{name} built in {time.monotonic() - t0:.1f} s")
        _built[name] = exe
    return name, _built[name]


def run(gate, *args, check=True):
    r = subprocess.run([str(gate[1]), *args], capture_output=True, text=True)
    if check:
        assert r.returncode == 0, r.stdout + r.stderr
    return r


# ---- no GPU needed ----------------------------------------------------------------------------------------------------
@every_gate
def test_gate_builds_for_sm_90a_with_the_library_flags(gate):
    cmd = gate_command(*gate)
    assert "-ffp-contract=off" in b.HOST_FLAGS and "-fno-fast-math" in b.HOST_FLAGS
    assert cmd[cmd.index("-Xcompiler") + 1] == b.HOST_FLAGS and "arch=compute_90a,code=sm_90a" in cmd and "-O3" in cmd
    assert not any("fast-math" in c and "no" not in c or "ftz" in c for c in cmd)
    elf = subprocess.run([os.path.join(os.path.dirname(b.nvcc_path()), "cuobjdump"), "--list-elf", str(gate[1])], capture_output=True,
                         text=True, check=True).stdout
    assert "sm_90a" in elf, elf


def _fingerprints(out):
    return [line for line in out.splitlines() if line.startswith("fingerprint ")]


@every_gate
def test_host_half_does_not_depend_on_the_thread_count(gate):
    one = _fingerprints(run(gate, "--host-only", "--threads", "1").stdout)
    many = _fingerprints(run(gate, "--host-only", "--threads", str(THREADS)).stdout)
    assert [line.split()[1] for line in one] == list(GATES[gate[0]].probes), one
    assert one == many


@every_gate
def test_self_test_reports_exactly_the_flipped_element(gate):
    r = run(gate, "--self-test", "--threads", str(THREADS), check=False)
    assert r.returncode == 1, r.stdout + r.stderr
    flipped = re.search(r"self-test: flipped (\S+) (\d+) word (\d+) bit (\d+)", r.stdout)
    assert flipped, r.stdout
    probe, index, word, bit = flipped.group(1), int(flipped.group(2)), int(flipped.group(3)), int(flipped.group(4))
    reports = [line.split() for line in r.stdout.splitlines() if len(line.split()) == 5 and not line.startswith("self-test")]
    assert len(reports) == 1, r.stdout
    name, at, _, host, other = reports[0]
    assert (name, int(at)) == (probe, index)
    h, o = [int(x, 16) for x in host.split(":")], [int(x, 16) for x in other.split(":")]
    assert [x ^ y for x, y in zip(h, o)] == [(1 << bit) if k == word else 0 for k in range(GATES[gate[0]].out_words)]
    assert r.stdout.strip().splitlines()[-1].endswith(" 1 mismatches"), r.stdout


@pytest.mark.parametrize("gate", [name for name, g in GATES.items() if g.ledger], indirect=True)
def test_ledger_reaches_every_class(gate):
    """The gate names exactly the classes of its ledger entry, and its families' first 2^20 inputs (a prefix of the full
    gate's) reach each at least as often as the entry asks, and never zero times."""
    spec = GATES[gate[0]]
    counts = {}
    for line in run(gate, "--ledger", "--threads", str(THREADS)).stdout.splitlines():
        _, probe, cls, n = line.split()
        counts[(probe, cls)] = int(n)
    assert set(counts) == set(spec.ledger), ("reported, not in the ledger:", sorted(set(counts) - set(spec.ledger)),
                                             "in the ledger, not reported:", sorted(set(spec.ledger) - set(counts)))
    short = sorted((k, n, spec.ledger[k]) for k, n in counts.items() if n == 0 or n < spec.ledger[k])
    assert not short, short


# ---- GPU --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@every_gate
def test_device_twins_equal_the_host_twins(gate):
    t0 = time.monotonic()
    r = run(gate, "--threads", str(THREADS), check=False)
    wall = time.monotonic() - t0
    print(r.stdout)
    last = r.stdout.strip().splitlines()[-1]
    m = re.fullmatch(r"(\d+) probes, (\d+) inputs, (\d+) mismatches", last)
    assert m, r.stdout + r.stderr
    times = re.search(r"device ([\d.]+) s, host ([\d.]+) s on (\d+) threads", r.stdout)
    print(f"{gate[0]}: {m.group(1)} probes, {m.group(2)} inputs; device {times.group(1)} s, host {times.group(2)} s on {times.group(3)} threads, "
          f"{wall:.1f} s wall")
    assert r.returncode == 0 and m.group(3) == "0", r.stdout + r.stderr
