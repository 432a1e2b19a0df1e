"""Compares the SASS of every perFrameGatherKernel instantiation of view_gather.cu with a base revision's.

    python profiles/view_gather_sass.py [--base REV]      (default HEAD~1, the parent of the checked-out commit)

A change that adds a per-frame source should leave the kernels of the existing sources exactly as they were.  This builds
view_gather.cu of the working tree and of REV (git archive) to cubins for sm_90a with the library's nvcc flags
(transform360_b200/build.py), splits `cuobjdump -sass` by function, and compares each instantiation the base has,
instruction and encoding words included.  Prints one line per differing or missing kernel and a summary; exit status 1
if any differs.  Needs nvcc and git, no GPU.
"""
from __future__ import annotations

import argparse
import io
import os
import re
import subprocess
import sys
import tarfile
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from transform360_b200 import build as b  # noqa: E402


def cubin(tree: Path, out: Path) -> None:
    cmd = [b.nvcc_path(), "-cubin", *b.ARCH, "-O3", "-std=c++17", "-Xcompiler", b.HOST_FLAGS, "-I", str(tree / "include"),
           "-I", str(tree / "transform360_b200" / "csrc"), "-o", str(out), str(tree / "transform360_b200" / "csrc" / "view_gather.cu")]
    subprocess.run(cmd, check=True)


# the anonymous namespace's mangled name carries a hash of the source, which differs between the two builds
ANON = re.compile(r"\d+_GLOBAL__N__[0-9a-f]+_\d+_view_gather_cu_[0-9a-f]+")


def kernels(path: Path) -> dict[str, str]:
    """mangled name (anonymous namespace normalised) -> its SASS (the per-frame gather kernels only)"""
    cuobjdump = os.path.join(os.path.dirname(b.nvcc_path()), "cuobjdump")
    sass = ANON.sub("(anon)", subprocess.run([cuobjdump, "-sass", str(path)], capture_output=True, text=True, check=True).stdout)
    out = {}
    for part in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = part.split("\n", 1)
        if "perFrameGatherKernel" in name:
            out[name.strip()] = body.strip()
    return out


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", default="HEAD~1")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        tmp = Path(tmp)
        archive = subprocess.run(["git", "-C", str(ROOT), "archive", args.base, "include", "transform360_b200/csrc"], capture_output=True,
                                 check=True).stdout
        with tarfile.open(fileobj=io.BytesIO(archive)) as tar:
            tar.extractall(tmp / "base", filter="data")
        cubin(tmp / "base", tmp / "base.cubin")
        cubin(ROOT, tmp / "new.cubin")
        base, new = kernels(tmp / "base.cubin"), kernels(tmp / "new.cubin")
    differ = 0
    for name, body in sorted(base.items()):
        if name not in new:
            print("missing", name)
            differ += 1
        elif new[name] != body:
            print("differs", name)
            differ += 1
    added = sorted(set(new) - set(base))
    print(f"{len(base) - differ} of {len(base)} perFrameGatherKernel instantiations of {args.base} have identical SASS; "
          f"{len(added)} added")
    return 1 if differ else 0


if __name__ == "__main__":
    sys.exit(main())
