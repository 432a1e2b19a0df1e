"""The device build of every float function of the per-frame position chains against its host build, bit for bit.

The per-frame kernels (view_gather.cu) compute each pixel's sampling record with the T360_HD functions of flat_view.h,
libm_ports.h and oriented_view.h; the planner computes the same records with their host build.  Each float step is an
explicit _rn intrinsic on the device and a plain operator under -ffp-contract=off on the host, and libmAtan2f / libmAsinf /
libmAtanf (ports of glibc) and sincCos (+ - * / only) are written so both builds agree.  tests/twin_gate.cu checks that
rule directly: the same probe code runs on the device and on the host, and every output word must match (every NaN equals
every NaN, nothing else is excused):
  - tier A, every 32-bit pattern: libmAtanf, libmAsinf, fSqrt, sincCos, truncToInt, roundHalfEven, quantizeAxis (K = 1, 2,
    4, 8);
  - tier B, structured families of 2^27-2^28 inputs (all floats in [-1, 2] for toPixel, every j < n <= 16384 for
    pixelCentre): libmAtan2f (tests/atan2_pairs.h, the pairs the glibc gate of test_oriented.py draws), rotateHD,
    rayToSphereHD, warpOffCentreHD, sphereInputHD, lensPosition, lensBlendPosition, cameraRay;
  - tier C, 2^26 (geometry, pixel) samples per chain over seeded contexts and their buildSphereTables tables: flatSample,
    sphereSample, lensSample, lensBlendSample and rectilinearSample in every instantiation the kernels use.
The host build is the one test_oriented.py pins to glibc, test_camera_models.py to double and the planner tests to the
reference, so those pins carry over to the device.

Without a GPU: the gate builds with the library's nvcc flags (transform360_b200/build.py), its host half gives the same
fingerprints on one thread and on many, its fingerprint and drill-down path reports exactly one injected bit flip, and its
input families reach every class the gate is meant to cover (a generator change that stops reaching one fails here).
"""
from __future__ import annotations

import os
import re
import subprocess
import time

import pytest

from transform360_b200 import build as b

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GATE_SRC = os.path.join(ROOT, "tests", "twin_gate.cu")
THREADS = max(8, os.cpu_count() or 1)

def gate_command(out):
    """The gate's nvcc command: the library's architecture, optimisation and host flags (build.py)."""
    return [b.nvcc_path(), *b.ARCH, "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", b.HOST_FLAGS, "-I", os.path.join(ROOT, "include"),
            "-I", str(b.CSRC), GATE_SRC, "-o", str(out)]


@pytest.fixture(scope="module")
def gate(tmp_path_factory):
    exe = tmp_path_factory.mktemp("twin_gate") / "twin_gate"
    t0 = time.monotonic()
    r = subprocess.run(gate_command(exe), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    print(f"twin_gate built in {time.monotonic() - t0:.1f} s")
    return exe


def run(gate, *args, check=True):
    r = subprocess.run([str(gate), *args], capture_output=True, text=True)
    if check:
        assert r.returncode == 0, r.stdout + r.stderr
    return r


# ---- no GPU needed ----------------------------------------------------------------------------------------------------
def test_gate_builds_for_sm_90a_with_the_library_flags(gate):
    cmd = gate_command(gate)
    assert "-ffp-contract=off" in b.HOST_FLAGS and "-fno-fast-math" in b.HOST_FLAGS
    assert cmd[cmd.index("-Xcompiler") + 1] == b.HOST_FLAGS and "arch=compute_90a,code=sm_90a" in cmd and "-O3" in cmd
    assert not any("fast-math" in c and "no" not in c or "ftz" in c for c in cmd)
    elf = subprocess.run([os.path.join(os.path.dirname(b.nvcc_path()), "cuobjdump"), "--list-elf", str(gate)], capture_output=True, text=True,
                         check=True).stdout
    assert "sm_90a" in elf, elf


def _fingerprints(out):
    return [line for line in out.splitlines() if line.startswith("fingerprint ")]


def test_host_half_does_not_depend_on_the_thread_count(gate):
    one = _fingerprints(run(gate, "--host-only", "--threads", "1").stdout)
    many = _fingerprints(run(gate, "--host-only", "--threads", str(THREADS)).stdout)
    assert len(one) >= 20, one
    assert one == many


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
    assert [x ^ y for x, y in zip(h, o)] == [(1 << bit) if k == word else 0 for k in range(4)]
    assert r.stdout.strip().splitlines()[-1].endswith(" 1 mismatches"), r.stdout


def _ledger(gate):
    counts = {}
    for line in run(gate, "--ledger", "--threads", str(THREADS)).stdout.splitlines():
        _, probe, cls, n = line.split()
        counts[(probe, cls)] = int(n)
    return counts


def test_ledger_reaches_every_class(gate):
    """Every class the gate names is reached by its families' first 2^20 inputs (a prefix of the full gate's)."""
    counts = _ledger(gate)
    for probe in ("libmAtan2f", "rotateHD", "rayToSphereHD", "warpOffCentreHD", "sphereInputHD", "lensPosition", "lensBlendPosition0",
                  "lensBlendPosition1", "cameraRay", "flatSample", "sphereSample<BARREL>", "sphereSample<plain>", "lensSample<BARREL>",
                  "lensSample<plain>", "lensBlendSample<BARREL>", "lensBlendSample<plain>", "rectilinearSample<ctx,any>",
                  "rectilinearSample<ctx,pinhole>", "rectilinearSample<lens,any>", "rectilinearSample<lens,pinhole>"):
        assert any(p == probe for p, _ in counts), probe
    missed = sorted(k for k, n in counts.items() if n == 0)
    assert not missed, missed
    for probe, cls in (("sphereInputHD", "majorIsHalf"), ("sphereInputHD", "pickedMajorIsHalf"), ("sphereInputHD", "noFaceWithoutNaN"), ("lensPosition", "thetaIsThetaMax"),
                       ("lensBlendPosition0", "tie"), ("cameraRay", "stereoAt1"), ("cameraRay", "panniniKAbove1e7")):
        assert counts[(probe, cls)] > 0, (probe, cls)


# ---- GPU --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_twins_equal_the_host_twins(gate):
    t0 = time.monotonic()
    r = run(gate, "--threads", str(THREADS), check=False)
    wall = time.monotonic() - t0
    print(r.stdout)
    last = r.stdout.strip().splitlines()[-1]
    m = re.fullmatch(r"(\d+) probes, (\d+) inputs, (\d+) mismatches", last)
    assert m, r.stdout + r.stderr
    times = re.search(r"device ([\d.]+) s, host ([\d.]+) s on (\d+) threads", r.stdout)
    print(f"{m.group(1)} probes, {m.group(2)} inputs; device {times.group(1)} s, host {times.group(2)} s on {times.group(3)} threads, "
          f"{wall:.1f} s wall")
    assert r.returncode == 0 and m.group(3) == "0", r.stdout + r.stderr
