"""The device build of every float function of the per-frame position chains against its host build, bit for bit.

The per-frame kernels (view_gather.cu) compute each pixel's sampling record with the T360_HD functions of flat_view.h,
libm_ports.h and oriented_view.h; the planner and the host twins compute the same records with their host build.  Each
float step is an explicit _rn intrinsic on the device and a plain operator under -ffp-contract=off on the host, and
libmAtan2f / libmAsinf / libmAtanf (ports of glibc) and sincCos (+ - * / only) are written so both builds agree.  Three
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
The host builds are the ones test_oriented.py pins to glibc, test_camera_models.py to double, test_camera_mip.py to
camera_map and a float64 model, test_lens_photo.py to lens_map, lens_blend_maps and a float64 model, and the planner
tests to the reference, so those pins carry over to the device.

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
    ledger_probes: tuple = ()  # the probes that name ledger classes; every class of theirs must be reached
    ledger_min: dict = field(default_factory=dict)  # {(probe, class): the least count}


_TWIN_PROBES = ("libmAtan2f", "pixelCentre", "toPixel", "rotateHD", "rayToSphereHD", "warpOffCentreHD", "sphereInputHD", "lensPosition",
                "lensBlendPosition0", "lensBlendPosition1", "cameraRay", "flatSample", "sphereSample<BARREL>", "sphereSample<plain>",
                "lensSample<BARREL>", "lensSample<plain>", "lensBlendSample<BARREL>", "lensBlendSample<plain>", "rectilinearSample<ctx,any>",
                "rectilinearSample<ctx,pinhole>", "rectilinearSample<lens,any>", "rectilinearSample<lens,pinhole>")
GATES = {
    "twin_gate": Gate(
        _TWIN_PROBES, 4,
        ledger_probes=tuple(p for p in _TWIN_PROBES if p not in ("pixelCentre", "toPixel")),  # those two walk fixed grids
        ledger_min={k: 1 for k in (("sphereInputHD", "majorIsHalf"), ("sphereInputHD", "pickedMajorIsHalf"), ("sphereInputHD", "noFaceWithoutNaN"),
                                   ("lensPosition", "thetaIsThetaMax"), ("lensBlendPosition0", "tie"), ("cameraRay", "stereoAt1"),
                                   ("cameraRay", "panniniKAbove1e7"))}),
    "mip_twin_gate": Gate(
        ("mipLevelOf", "rayDifferential", "equirectJacobian", "cubeJacobian", "lensJacobian", "mipScale", "mipCameraPoint<ctx>",
         "mipCameraPoint<lens>", "mipCameraSample<ctx>", "mipCameraSample<lens>"), 6),
    "photo_twin_gate": Gate(
        ("lensGain", "lensPhotoPosition", "lensPhotoSample<BARREL>", "lensPhotoSample<plain>"), 6,
        ledger_probes=("lensGain",),  # thousands of each edge class of the gain
        ledger_min={("lensGain", c): 1000 for c in ("r0", "thetaMax", "nearBound", "clamp", "uncovered")}),
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
    flipped = re.search(r"self-test: flipped (\S+) (\d+) word (\d) bit (\d)", r.stdout)
    assert flipped, r.stdout
    probe, index, word, bit = flipped.group(1), int(flipped.group(2)), int(flipped.group(3)), int(flipped.group(4))
    reports = [line.split() for line in r.stdout.splitlines() if len(line.split()) == 5 and not line.startswith("self-test")]
    assert len(reports) == 1, r.stdout
    name, at, _, host, other = reports[0]
    assert (name, int(at)) == (probe, index)
    h, o = [int(x, 16) for x in host.split(":")], [int(x, 16) for x in other.split(":")]
    assert [x ^ y for x, y in zip(h, o)] == [(1 << bit) if k == word else 0 for k in range(GATES[gate[0]].out_words)]
    assert r.stdout.strip().splitlines()[-1].endswith(" 1 mismatches"), r.stdout


@pytest.mark.parametrize("gate", [name for name, g in GATES.items() if g.ledger_probes], indirect=True)
def test_ledger_reaches_every_class(gate):
    """Every class a gate names is reached by its families' first 2^20 inputs (a prefix of the full gate's)."""
    spec = GATES[gate[0]]
    counts = {}
    for line in run(gate, "--ledger", "--threads", str(THREADS)).stdout.splitlines():
        _, probe, cls, n = line.split()
        counts[(probe, cls)] = int(n)
    assert sorted({p for p, _ in counts}) == sorted(spec.ledger_probes), counts
    missed = sorted(k for k, n in counts.items() if n == 0)
    assert not missed, missed
    for k, least in spec.ledger_min.items():
        assert counts.get(k, 0) >= least, (k, counts)


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
