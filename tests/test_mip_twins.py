"""The device build of the anti-aliased camera views' float functions against their host build, bit for bit.

tests/mip_twin_gate.cu runs the same probe code on the device and in a host thread pool (tests/twin_gate.cu's design:
hash-drawn inputs, per-block fingerprints, element re-evaluation on a mismatch) over:
  - mipLevelOf, the level-of-detail rule, for every 32-bit pattern of rho^2;
  - rayDifferential for every camera model, equirectJacobian, cubeInputFace with cubeJacobian, lensJacobian (rays on a
    lens's axis, rho = 0, included) and mipScale over 2^26 drawn inputs each;
  - mipCameraPoint and mipCameraSample, LENS = false and true, over 2^24 (geometry, pixel) samples each.
The host build is the one T360B200_cameraMipMaps runs and tests/test_camera_mip.py pins to camera_map and to a float64
model, so those pins carry over to the kernel.

Without a GPU: the gate builds with the library's nvcc flags (transform360_b200/build.py), its host half gives the same
fingerprints on one thread and on many, and its fingerprint and drill-down path reports exactly one injected bit flip."""
from __future__ import annotations

import os
import re
import subprocess
import time

import pytest

from transform360_b200 import build as b

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GATE_SRC = os.path.join(ROOT, "tests", "mip_twin_gate.cu")
THREADS = max(8, os.cpu_count() or 1)
PROBES = ("mipLevelOf", "rayDifferential", "equirectJacobian", "cubeJacobian", "lensJacobian", "mipScale", "mipCameraPoint<ctx>",
          "mipCameraPoint<lens>", "mipCameraSample<ctx>", "mipCameraSample<lens>")


def gate_command(out):
    """The gate's nvcc command: the library's architecture, optimisation and host flags (build.py)."""
    return [b.nvcc_path(), *b.ARCH, "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", b.HOST_FLAGS, "-I", os.path.join(ROOT, "include"),
            "-I", str(b.CSRC), GATE_SRC, "-o", str(out)]


@pytest.fixture(scope="module")
def gate(tmp_path_factory):
    exe = tmp_path_factory.mktemp("mip_twin_gate") / "mip_twin_gate"
    r = subprocess.run(gate_command(exe), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
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
    elf = subprocess.run([os.path.join(os.path.dirname(b.nvcc_path()), "cuobjdump"), "--list-elf", str(gate)], capture_output=True, text=True,
                         check=True).stdout
    assert "sm_90a" in elf, elf


def _fingerprints(out):
    return [line for line in out.splitlines() if line.startswith("fingerprint ")]


def test_host_half_does_not_depend_on_the_thread_count(gate):
    one = _fingerprints(run(gate, "--host-only", "--threads", "1").stdout)
    many = _fingerprints(run(gate, "--host-only", "--threads", str(THREADS)).stdout)
    assert [line.split()[1] for line in one] == list(PROBES), one
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
    assert [x ^ y for x, y in zip(h, o)] == [(1 << bit) if k == word else 0 for k in range(6)]
    assert r.stdout.strip().splitlines()[-1].endswith(" 1 mismatches"), r.stdout


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
