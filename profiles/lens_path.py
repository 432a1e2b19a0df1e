"""What a fisheye lens rig costs on the GPU machine: the per-frame lens call (T360B200_transformFrameLensAsync, a new
orientation every frame) against the planned path for a fixed pose (T360B200_lensMap -> T360B200_generateMapFromWarp ->
T360B200_transformFrameAsync), against T360B200_remapFrameAsync with the same maps resident on the device, and (--blend)
against the feathered seam (T360B200_transformFrameLensBlendAsync) with belts of 4 and 10 degrees.  Needs a GPU.

    python profiles/lens_path.py [--frames 100] [--windows 3] [--blend] [--out FILE]

Workload: a 5760x2880 yuv420p dual-fisheye frame, two 2880-pixel circles side by side from back-to-back 190-degree lenses
with seeded small k1..k4 (calibrated at 5760x2880), bicubic, to EQUIRECT 5760x2880 and to CUBEMAP_32 3840x2560.  Inputs
come from a ring of frames larger than the L2 cache.  Per target:
- lens_map_ms / generate_ms: host wall time of lensMap and of generateMapFromWarp, per plan index;
- lens_ms / planned_ms / remap_ms: CUDA-event GPU time per frame of `--frames` frames enqueued back to back on one stream
  after a warm-up, `--windows` windows per arm, the arms alternated window by window (the lens call with a new orientation
  every frame, the other two with the fixed pose their maps were made for);
- blend4_ms / blend10_ms (--blend): the same for the feathered seam with seamWidth 4 and 10 degrees, a new orientation
  every frame, alternated with the other arms; blend_share: the share of luma pixels in the belt (0 < w < 256) at the
  fixed pose, per seamWidth;
- identical: whether the three arms' outputs for the fixed pose are equal, byte for byte, plane by plane;
- nan_share: the share of luma map entries no lens covers.
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

CUBIC, EQUIRECT, CUBEMAP_32 = 2, 3, 0
RING = 4  # input frames of 24.9 MB: 99.5 MB, twice the H100's 50 MB L2


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().split(", ")
    return {"gpu": q[0], "power_limit_w": float(q[1])} if len(q) == 2 else {"gpu": None, "power_limit_w": None}


def dual_fisheye_rig(seed=0):
    import numpy as np
    import transform360_b200 as t360
    from tests.test_lens import _lens
    rng = np.random.default_rng(seed)
    rig = t360.T360LensRig(2, 5760, 2880)
    rig.lens[0] = _lens(rng, 1440, 1439.5, 1439.5, 0, 0, 0, 95)
    rig.lens[1] = _lens(rng, 1440, 4319.5, 1439.5, 180, 0, 0, 95)
    return rig


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100, help="frames per timed window")
    ap.add_argument("--windows", type=int, default=3, help="timed windows per arm")
    ap.add_argument("--blend", action="store_true", help="add the feathered-seam arms")
    ap.add_argument("--out", help="append the JSON line to this file")
    args = ap.parse_args()
    import numpy as np
    import torch
    import transform360_b200 as t360
    from oracle import c_oracle as co

    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    info = gpu_info()
    rig = dual_fisheye_rig()
    fixed = (35.0, -10.0, 5.0)
    rng = np.random.default_rng(1)
    path = [tuple(float(v) for v in o) for o in np.cumsum(rng.normal(0, [3.0, 1.0, 1.0], (args.frames, 3)), 0) + fixed]
    iw, ih = 5760, 2880
    targets = {"equirect_5760x2880": (EQUIRECT, 5760, 2880), "cubemap_32_3840x2560": (CUBEMAP_32, 3840, 2560)}
    pitch = lambda w: (w + 255) // 256 * 256
    in_dims = [(iw, ih), (iw // 2, ih // 2), (iw // 2, ih // 2)]
    ring = []
    for f in range(RING):
        frame = []
        for p, (w, h) in enumerate(in_dims):
            t = torch.zeros((h, pitch(w)), dtype=torch.uint8, device="cuda")
            t[:, :w] = torch.from_numpy(co.noise_plane(w, h, plane=p, frame=f)).cuda()
            frame.append(t)
        ring.append(frame)
    in_planes = [[(t.data_ptr(), t.stride(0)) for t in frame] for frame in ring]
    result = dict(info, frames=args.frames, windows=args.windows, input=[iw, ih], ring_frames=RING, interp=CUBIC, cases={})
    for name, (layout, ow, oh) in targets.items():
        ctx = t360.make_context(output_layout=layout, interpolation_alg=CUBIC, enable_low_pass_filter=0)
        dims = [(*in_dims[0], ow, oh), (*in_dims[1], ow // 2, oh // 2), (*in_dims[2], ow // 2, oh // 2)]
        lens_map_ms, generate_ms, maps = [], [], []
        vft = t360.VideoFrameTransform(ctx)
        for idx in (0, 1):
            t0 = time.perf_counter()
            maps.append(t360.lens_map(ctx, rig, fixed, *dims[idx]))
            lens_map_ms.append(round((time.perf_counter() - t0) * 1e3, 1))
            t0 = time.perf_counter()
            assert vft.generate_map_from_warp(maps[idx], *dims[idx][:2], idx, t360.BORDER_TRANSPARENT)
            generate_ms.append(round((time.perf_counter() - t0) * 1e3, 1))
        d_maps = [torch.from_numpy(m).cuda() for m in maps]
        outs = {k: [torch.zeros((d[3], pitch(d[2])), dtype=torch.uint8, device="cuda") for d in dims] for k in ("lens", "planned", "remap", "blend")}
        out_planes = {k: [(t.data_ptr(), t.stride(0)) for t in v] for k, v in outs.items()}
        lens = [vft.make_lens_frame_call(in_planes[f], out_planes["lens"], dims) for f in range(RING)]
        planned = [vft.make_frame_call(in_planes[f], out_planes["planned"], dims) for f in range(RING)]
        remap = [vft.make_remap_frame_call(in_planes[f], out_planes["remap"], dims, t360.BORDER_TRANSPARENT) for f in range(RING)]
        st = torch.cuda.Stream()
        s = st.cuda_stream
        # the fixed pose on every arm, from the same input and identically pre-filled outputs
        for v in outs.values():
            for t in v:
                t.fill_(7)
        torch.cuda.synchronize()
        assert lens[0](rig, fixed, s) and planned[0](s) and remap[0]([d_maps[0], d_maps[1], d_maps[1]], s)
        st.synchronize()
        identical = [bool(torch.equal(a[:, :d[2]], b[:, :d[2]]) and torch.equal(a[:, :d[2]], c[:, :d[2]]))
                     for a, b, c, d in zip(outs["lens"], outs["planned"], outs["remap"], dims)]
        arms = {
            "lens_ms": lambda i: lens[i % RING](rig, path[i], s),
            "planned_ms": lambda i: planned[i % RING](s),
            "remap_ms": lambda i: remap[i % RING]([d_maps[0], d_maps[1], d_maps[1]], s),
        }
        extra = {}
        if args.blend:
            blend = [vft.make_lens_blend_frame_call(in_planes[f], out_planes["blend"], dims) for f in range(RING)]
            for seam in (4.0, 10.0):
                arms[f"blend{seam:g}_ms"] = lambda i, seam=seam: blend[i % RING](rig, seam, path[i], s)
            extra["blend_share"] = {f"{seam:g}": round(float(((w > 0) & (w < 256)).mean()), 4)
                                    for seam in (4.0, 10.0) for w in [t360.lens_blend_maps(ctx, rig, seam, fixed, *dims[0])[2]]}
        for call in arms.values():  # warm-up: first launches, weight tables, the lens call's table upload
            for i in range(10):
                assert call(i)
        st.synchronize()
        times = {k: [] for k in arms}
        for _ in range(args.windows):
            for k, call in arms.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(st)
                for i in range(args.frames):
                    assert call(i)
                b.record(st)
                b.synchronize()
                times[k].append(round(a.elapsed_time(b) / args.frames, 4))
        result["cases"][name] = dict(layout=layout, output=[ow, oh], lens_map_ms=lens_map_ms, generate_ms=generate_ms, **times,
                                     identical=identical, nan_share=round(float(np.isnan(maps[0][..., 0]).mean()), 4), **extra)
        vft.close()
        del d_maps, outs
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
