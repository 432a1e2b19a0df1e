#!/usr/bin/env python
"""Generates tests/golden/golden.json from THE REFERENCE ITSELF:
``oracle/_ref/libt360ref.so`` (unmodified reference sources + oracle/shim) driving cv2 4.13.0.

    python tests/golden/make_golden.py            # small cases (+ cfg1)
    python tests/golden/make_golden.py --full     # also cfg2/cfg3/cfg4 luma known answers

Needs the reference sources (to build oracle/_ref) and cv2; the output is committed so that the tests do not.
Input planes are the integer-hash ``noise`` generator of SURVEY.md 8(d); plane p of a case uses
noise(w, h, plane=p, frame=0).
"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

from oracle import ref_harness as rh  # noqa: E402
from tests.golden.cases import FULL, SMALL, plane_dims  # noqa: E402


def run_case(name, case, planes=(0, 1)):
    ctx = rh.default_context(**case["ov"])
    ref = rh.RefTransform(ctx)
    rec = {"planes": {}}
    for plane in planes:
        iw, ih, ow, oh, idx = plane_dims(case, plane)
        assert ref.generate_map(iw, ih, ow, oh, idx)
        m = ref.map(idx)
        segs = ref.segments(idx)
        taps = np.concatenate([np.concatenate([s[4], s[5]]) for s in segs]) if segs else np.zeros(0, np.float32)
        rects = np.array([s[:4] for s in segs], np.int32) if segs else np.zeros((0, 4), np.int32)
        src = rh.noise_plane(iw, ih, plane=plane, frame=0)
        barrel = ctx.output_layout in (rh.LAYOUT_BARREL, rh.LAYOUT_BARREL_SPLIT)
        out = ref.transform_plane(src, ow, oh, idx, image_plane=plane, prefill=0 if not barrel else 7)
        rec["planes"][str(plane)] = {
            "dims": [iw, ih, ow, oh, idx],
            "map_fnv": rh.fnv1a64(m),
            "map_corners": [float(m[0, 0, 0]), float(m[0, 0, 1]), float(m[-1, -1, 0]), float(m[-1, -1, 1])],
            "nsegs": len(segs),
            "rects_fnv": rh.fnv1a64(rects),
            "taps_fnv": rh.fnv1a64(taps),
            "ntaps": int(taps.size),
            "src_sha": rh.sha16(src),
            "out_sha": rh.sha16(out),
            "out_sum": int(out.sum(dtype=np.int64)),
            "out_head": [int(v) for v in out[0, :8]],
        }
        print(name, plane, rec["planes"][str(plane)]["out_sha"], rec["planes"][str(plane)]["out_sum"], flush=True)
    ref.close()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--full", action="store_true")
    args = ap.parse_args()
    path = Path(__file__).with_name("golden.json")
    gold = json.loads(path.read_text()) if path.exists() else {}
    gold.setdefault("_meta", {})
    import cv2
    import platform
    gold["_meta"] = {"cv2": cv2.__version__, "glibc": platform.libc_ver()[1], "generator": "tests/golden/make_golden.py",
                     "note": "hashes depend on host libm (sinf/cosf/expf/atan2f/asinf) -- regenerate if the image changes"}
    gold.setdefault("small", {})
    for name, case in SMALL.items():
        gold["small"][name] = run_case(name, case)
    if args.full:
        gold.setdefault("full", {})
        for name in ("cfg2", "cfg3", "cfg4"):
            gold["full"][name] = run_case(name, FULL[name], planes=(0,))
    path.write_text(json.dumps(gold, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    main()
