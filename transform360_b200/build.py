"""Builds transform360_b200/lib/libTransform360.so (the drop-in C-ABI library) in-tree with nvcc for sm_90a (H100).

    python -m transform360_b200.build [--force] [--verbose] [--out=PATH]

The artifact name follows the reference's CMake target (Transform360/CMakeLists.txt:9: libTransform360).
The .so is a build product (git-ignored): build() makes it in the tree.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
ROOT = PKG.parent
CSRC = PKG / "csrc"
LIB_DIR = PKG / "lib"
LIB = LIB_DIR / "libTransform360.so"
SOURCES = ["geometry.cpp", "lowpass_plan.cpp", "lowpass_jobs.cpp", "sampling.cpp", "gather_plan.cpp", "kernels.cu", "gather_frame.cu", "view_gather.cu", "video_frame_transform.cpp"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
# host code: -ffp-contract=off keeps the planner's float sequence identical to the reference's build, and the host twins
# of the per-frame position chains (csrc/flat_view.h, libm_ports.h, oriented_view.h) plain IEEE operations.
# tests/test_twin_gates.py builds its host / device comparisons with the same string.
HOST_FLAGS = "-fPIC,-fvisibility=hidden,-ffp-contract=off,-fno-fast-math,-Wall"


def nvcc_path() -> str:
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(p).exists():
        raise FileNotFoundError("nvcc not found (needed to build libTransform360.so)")
    return p


def needs_build() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    deps = list(CSRC.glob("*")) + list((ROOT / "include").rglob("*.h")) + [Path(__file__)]
    return any(d.stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False, out: Path | None = None) -> Path:
    """out: a library built elsewhere than LIB (e.g. a parent commit's build for an A/B run), loaded with
    T360B200_LIB=<path>; it is always built."""
    if out is None and not force and not needs_build():
        return LIB
    out = out or LIB
    LIB_DIR.mkdir(exist_ok=True)
    cmd = [nvcc_path(), *ARCH, "-O3", "-lineinfo", "-std=c++17", "--shared", "-Xcompiler", HOST_FLAGS,
           "-Xptxas", "-v" if verbose else "-warn-spills", "-I", str(ROOT / "include"), "-I", str(CSRC),
           "-o", str(out)] + [str(CSRC / s) for s in SOURCES]
    env = dict(os.environ)
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    if verbose or r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed building libTransform360.so")
    return out


def build_static(verbose: bool = False) -> Path:
    """lib/libTransform360.a, the artifact name of the reference's CMake target (Transform360/CMakeLists.txt:9):
    objects with relocatable device code already linked, so that a plain `cc ... -lTransform360 -lcudart_static -ldl
    -lrt -lpthread -lstdc++` (ffmpeg's --extra-libs) resolves everything."""
    LIB_DIR.mkdir(exist_ok=True)
    obj_dir = LIB_DIR / "obj"
    obj_dir.mkdir(exist_ok=True)
    objs = []
    for src in SOURCES:
        o = obj_dir / (Path(src).stem + ".o")
        cmd = [nvcc_path(), *ARCH, "-O3", "-lineinfo", "-std=c++17", "-c", "-Xcompiler", HOST_FLAGS, "-I", str(ROOT / "include"),
               "-I", str(CSRC), "-o", str(o), str(CSRC / src)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or r.returncode != 0:
            sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}")
        objs.append(str(o))
    out = LIB_DIR / "libTransform360.a"
    if out.exists():
        out.unlink()
    subprocess.run(["ar", "rcs", str(out), *objs], check=True)
    return out


def install(prefix: str) -> None:
    """The reference's install layout (Transform360/CMakeLists.txt:15-16): <prefix>/lib/libTransform360.{so,a},
    <prefix>/include/Transform360/*.h (+ the lower-case forwarding headers the filter source includes)."""
    import shutil as sh
    pre = Path(prefix)
    (pre / "lib").mkdir(parents=True, exist_ok=True)
    sh.copy2(build(), pre / "lib" / "libTransform360.so")
    sh.copy2(build_static(), pre / "lib" / "libTransform360.a")
    for sub in ("Transform360", "transform360"):
        (pre / "include" / sub).mkdir(parents=True, exist_ok=True)
        for h in (ROOT / "include" / sub).glob("*.h"):
            sh.copy2(h, pre / "include" / sub / h.name)
    sh.copy2(ROOT / "include" / "transform360_b200.h", pre / "include" / "transform360_b200.h")
    (pre / "share" / "transform360").mkdir(parents=True, exist_ok=True)  # the CUDA-frame ffmpeg filter goes into an ffmpeg tree as source
    sh.copy2(PKG / "filter" / "vf_transform360_cuda.c", pre / "share" / "transform360" / "vf_transform360_cuda.c")


if __name__ == "__main__":
    if "--static" in sys.argv:
        print(build_static(verbose="--verbose" in sys.argv))
        sys.exit(0)
    pre = [a.split("=", 1)[1] for a in sys.argv[1:] if a.startswith("--install=")]
    if pre:
        install(pre[0])
        print("installed under", pre[0])
        sys.exit(0)
    outs = [a.split("=", 1)[1] for a in sys.argv[1:] if a.startswith("--out=")]
    p = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv, out=Path(outs[0]) if outs else None)
    print(p)
