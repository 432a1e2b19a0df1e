"""The device build of the lens photometry's float function and chains against their host build, bit for bit.

tests/photo_twin_gate.cu runs the same probe code on the device and in a host thread pool (tests/twin_gate.cu's design:
hash-drawn inputs, per-block fingerprints, element re-evaluation on a mismatch) over:
  - lensGain, the falloff and Gq's quantisation, over 2^28 drawn lens hits, falloffs and gains;
  - lensPhotoPosition over 2^26 drawn rig directions, hard (closer lens only, or both) and feathered seams;
  - lensPhotoSample, BARREL = true and false, over 2^24 (geometry, pixel) samples each of every sphere output layout.
The host build is the one T360B200_lensPhotoMaps runs and tests/test_lens_photo.py pins to lens_map, lens_blend_maps
and a float64 model, so those pins carry over to the kernel.

Without a GPU: the gate builds with the library's nvcc flags (transform360_b200/build.py), its host half gives the same
fingerprints on one thread and on many, its fingerprint and drill-down path reports exactly one injected bit flip, and its
ledger shows lensGain's inputs reach every edge class: r = 0, theta = thetaMax, V near the refusal bound, Gq at its clamp,
and rays the lens does not cover."""
from __future__ import annotations

import os
import re
import subprocess
import time

import pytest

from transform360_b200 import build as b

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GATE_SRC = os.path.join(ROOT, "tests", "photo_twin_gate.cu")
THREADS = max(8, os.cpu_count() or 1)
PROBES = ("lensGain", "lensPhotoPosition", "lensPhotoSample<BARREL>", "lensPhotoSample<plain>")
GAIN_CLASSES = ("r0", "thetaMax", "nearBound", "clamp", "uncovered")


def gate_command(out):
    """The gate's nvcc command: the library's architecture, optimisation and host flags (build.py)."""
    return [b.nvcc_path(), *b.ARCH, "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", b.HOST_FLAGS, "-I", os.path.join(ROOT, "include"),
            "-I", str(b.CSRC), GATE_SRC, "-o", str(out)]


@pytest.fixture(scope="module")
def gate(tmp_path_factory):
    exe = tmp_path_factory.mktemp("photo_twin_gate") / "photo_twin_gate"
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


def test_ledger_reaches_every_edge_class_of_the_gain(gate):
    """lensGain's first 2^20 inputs (a prefix of the full gate's) reach each edge class thousands of times."""
    counts = {}
    for line in run(gate, "--ledger", "--threads", str(THREADS)).stdout.splitlines():
        _, probe, cls, n = line.split()
        counts[(probe, cls)] = int(n)
    for cls in GAIN_CLASSES:
        assert counts.get(("lensGain", cls), 0) >= 1000, (cls, counts)


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
