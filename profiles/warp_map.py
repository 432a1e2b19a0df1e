"""What warp-map transforms cost on the GPU machine: the planned path (T360B200_generateMapFromWarp, then the whole-frame
entry point) against per-frame device maps (T360B200_remapFrameAsync) for the same maps.  Needs a GPU.

    python profiles/warp_map.py [--frames 100] [--windows 3] [--out FILE]

Cases (yuv420p frames, maps from tests/test_warp_map.py's seeded generators, chroma maps made at chroma size):
- dual_fisheye_8k: two 190-degree equidistant fisheye circles side by side, 7680x3840 in -> 7680x3840 equirect, cubic;
- undistort_4k: one fisheye lens undistorted to a rectilinear 3840x2160 view from a 3840x2160 plane, bilinear.
For each case:
- generate_ms: wall time of generateMapFromWarp for plan index 0 and 1 (host planning, gather plan and upload);
- planned_ms / per_frame_ms: CUDA-event GPU time per frame of `--frames` frames enqueued back to back on one stream after a
  warm-up, `--windows` windows each, the two paths alternated window by window;
- identical: whether the two paths' outputs are equal, plane by plane;
- jobs: the luma plan's frame-kernel jobs by kind (T360B200_planTileCounts: staged, border).
Prints one JSON line (also appended to --out) with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

CUBIC, LINEAR = 2, 1


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().split(", ")
    return {"gpu": q[0], "power_limit_w": float(q[1])} if len(q) == 2 else {"gpu": None, "power_limit_w": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100, help="frames per timed window")
    ap.add_argument("--windows", type=int, default=3, help="timed windows per path")
    ap.add_argument("--out", help="append the JSON line to this file")
    args = ap.parse_args()
    import numpy as np
    import torch
    import transform360_b200 as t360
    from oracle import c_oracle as co
    from tests.test_warp_map import dual_fisheye, fisheye_undistort

    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    info = gpu_info()
    cases = {
        "dual_fisheye_8k": (CUBIC, (7680, 3840), (7680, 3840), dual_fisheye),
        "undistort_4k": (LINEAR, (3840, 2160), (3840, 2160), fisheye_undistort),
    }
    result = dict(info, frames=args.frames, windows=args.windows, cases={})
    for name, (interp, (iw, ih), (ow, oh), make) in cases.items():
        dims = [(iw, ih, ow, oh), ((iw + 1) // 2, (ih + 1) // 2, (ow + 1) // 2, (oh + 1) // 2)]
        dims.append(dims[1])
        maps = [make(d[2], d[3], d[0], d[1]) for d in dims[:2]]
        vft = t360.VideoFrameTransform(t360.make_context(interpolation_alg=interp, enable_low_pass_filter=0))
        generate_ms = []
        for idx in (0, 1):
            t0 = time.perf_counter()
            assert vft.generate_map_from_warp(maps[idx], *dims[idx][:2], idx)
            generate_ms.append((time.perf_counter() - t0) * 1e3)
        counts = vft.plan_tile_counts(0)
        pitch = lambda w: (w + 255) // 256 * 256
        src = []
        for p, d in enumerate(dims):
            t = torch.zeros((d[1], pitch(d[0])), dtype=torch.uint8, device="cuda")
            t[:, :d[0]] = torch.from_numpy(co.noise_plane(d[0], d[1], plane=p)).cuda()
            src.append(t)
        outs = {k: [torch.zeros((d[3], pitch(d[2])), dtype=torch.uint8, device="cuda") for d in dims] for k in ("planned", "per_frame")}
        d_maps = [torch.from_numpy(m).cuda() for m in maps]
        in_planes = [(t.data_ptr(), t.stride(0)) for t in src]
        calls = {
            "planned": (lambda c: lambda s: c(s))(vft.make_frame_call(in_planes, [(t.data_ptr(), t.stride(0)) for t in outs["planned"]], dims)),
            "per_frame": (lambda c: lambda s: c([d_maps[0], d_maps[1], d_maps[1]], s))(
                vft.make_remap_frame_call(in_planes, [(t.data_ptr(), t.stride(0)) for t in outs["per_frame"]], dims)),
        }
        st = torch.cuda.Stream()
        torch.cuda.synchronize()
        for call in calls.values():  # warm-up: first launches, weight tables, scratch
            for _ in range(10):
                assert call(st.cuda_stream)
        st.synchronize()
        identical = [bool(torch.equal(a[:, :d[2]], b[:, :d[2]])) for a, b, d in zip(outs["planned"], outs["per_frame"], dims)]
        times = {k: [] for k in calls}
        for _ in range(args.windows):
            for k, call in calls.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(st)
                for _ in range(args.frames):
                    assert call(st.cuda_stream)
                b.record(st)
                b.synchronize()
                times[k].append(round(a.elapsed_time(b) / args.frames, 4))
        result["cases"][name] = dict(interp=interp, input=[iw, ih], output=[ow, oh], generate_ms=[round(v, 1) for v in generate_ms],
                                     planned_ms=times["planned"], per_frame_ms=times["per_frame"], identical=identical,
                                     luma_jobs=dict(staged=counts[0], border=counts[1]),
                                     nan_share=round(float(np.isnan(maps[0][..., 0]).mean()), 4))
        vft.close()
        del d_maps, src, outs
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
