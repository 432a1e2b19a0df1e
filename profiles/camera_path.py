"""What the camera models cost on the GPU machine: the per-frame call (T360B200_transformFrameCameraAsync, a new pose every
frame) against the planned path for one pose (T360B200_cameraMap -> T360B200_generateMapFromWarp ->
T360B200_transformFrameAsync).  Needs a GPU.

    python profiles/camera_path.py [--frames 100] [--windows 3] [--out FILE]

Workloads, yuv420p from a 7680x3840 equirect (chroma 3840x1920), without low-pass:
- <model>_cubic / <model>_lanczos4: a 1920x1080 view (chroma 960x540) with each of the four camera models (pinhole and
  Pannini d = 0.5 at 100 degrees across, equidistant and stereographic at 180), bicubic and Lanczos4;
- dome_4096: a 4096x4096 equidistant 180-degree dome master, bicubic;
- little_planet_2048: a 2048x2048 stereographic view of 270 degrees looking at the nadir, bicubic.
Inputs come from a ring of frames larger than the L2 cache.  Per workload:
- map_ms / generate_ms: host wall time of cameraMap and of generateMapFromWarp, per plan index;
- cam_ms / planned_ms: CUDA-event GPU time per frame of `--frames` frames enqueued back to back on one stream after a
  warm-up, `--windows` windows per arm, the arms alternated window by window (the camera call with a new pose every frame,
  the planned path with the fixed pose its maps were made for);
- identical: whether the per-frame call and the planned path give the same bytes for the fixed pose, plane by plane.
Prints one JSON line (also appended to --out) with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from profiles.rectilinear_path import RING, gpu_info  # noqa: E402

CUBIC, LANCZOS4 = 2, 4
IN_W, IN_H = 7680, 3840
PINHOLE, EQUIDISTANT, STEREOGRAPHIC, PANNINI = 0, 1, 2, 3


def workloads():
    """name -> (interpolation, camera, fixed pose, output luma size, the per-frame path's pose at frame i)"""
    import numpy as np
    import transform360_b200 as t360
    out = {}
    vfov90 = t360.square_pixel_vfov(90.0, 1920, 1080)
    views = {"pinhole": ((PINHOLE, 0.0), 90.0, vfov90), "equidistant": ((EQUIDISTANT, 0.0), 180.0, 101.25),
             "stereographic": ((STEREOGRAPHIC, 0.0), 180.0, 101.25), "pannini": ((PANNINI, 0.5), 100.0, vfov90)}
    rng = np.random.default_rng(1)
    steps = np.cumsum(rng.normal(0, [3.0, 1.0, 1.0], (1000, 3)), 0)
    for model, (cam, hfov, vfov) in views.items():
        for interp, iname in ((CUBIC, "cubic"), (LANCZOS4, "lanczos4")):
            out[f"{model}_{iname}"] = (interp, cam, (35.0, -10.0, 5.0, hfov, vfov), (1920, 1080),
                                       lambda i, h=hfov, v=vfov: (35.0 + steps[i, 0], float(np.clip(-10.0 + steps[i, 1], -80, 80)), 5.0 + steps[i, 2], h, v))
    out["dome_4096"] = (CUBIC, (EQUIDISTANT, 0.0), (0.0, 20.0, 0.0, 180.0, 180.0), (4096, 4096),
                        lambda i: (steps[i, 0], float(np.clip(20.0 + steps[i, 1], -80, 80)), 0.0, 180.0, 180.0))
    out["little_planet_2048"] = (CUBIC, (STEREOGRAPHIC, 0.0), (0.0, -90.0, 0.0, 270.0, 270.0), (2048, 2048),
                                 lambda i: (steps[i, 0], -90.0, steps[i, 2], 270.0, 270.0))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100, help="frames per timed window")
    ap.add_argument("--windows", type=int, default=3, help="timed windows per arm")
    ap.add_argument("--out", help="append the JSON line to this file")
    args = ap.parse_args()
    import torch
    import transform360_b200 as t360
    from oracle import c_oracle as co

    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    info = gpu_info()
    pitch = lambda w: (w + 255) // 256 * 256
    in_dims = [(IN_W, IN_H), (IN_W // 2, IN_H // 2), (IN_W // 2, IN_H // 2)]
    ring = []
    for f in range(RING):
        frame = []
        for p, (w, h) in enumerate(in_dims):
            t = torch.zeros((h, pitch(w)), dtype=torch.uint8, device="cuda")
            t[:, :w] = torch.from_numpy(co.noise_plane(w, h, plane=p, frame=f)).cuda()
            frame.append(t)
        ring.append(frame)
    in_planes = [[(t.data_ptr(), t.stride(0)) for t in frame] for frame in ring]
    result = dict(info, frames=args.frames, windows=args.windows, input=[IN_W, IN_H], ring_frames=RING, cases={})
    for name, (interp, cam, fixed, (ow, oh), path) in workloads().items():
        dims = [(*in_dims[0], ow, oh), (*in_dims[1], ow // 2, oh // 2), (*in_dims[2], ow // 2, oh // 2)]
        ctx = t360.make_context(interpolation_alg=interp, enable_low_pass_filter=0)
        vft = t360.VideoFrameTransform(ctx)
        map_ms, generate_ms = [], []
        for idx in (0, 1):
            t0 = time.perf_counter()
            m = t360.camera_map(ctx, fixed, cam, *dims[idx])
            map_ms.append(round((time.perf_counter() - t0) * 1e3, 1))
            t0 = time.perf_counter()
            assert vft.generate_map_from_warp(m, *dims[idx][:2], idx, t360.BORDER_WRAP)
            generate_ms.append(round((time.perf_counter() - t0) * 1e3, 1))
        outs = {k: [torch.zeros((d[3], pitch(d[2])), dtype=torch.uint8, device="cuda") for d in dims] for k in ("cam", "planned")}
        out_planes = {k: [(t.data_ptr(), t.stride(0)) for t in v] for k, v in outs.items()}
        camera = [vft.make_camera_frame_call(in_planes[f], out_planes["cam"], dims) for f in range(RING)]
        planned = [vft.make_frame_call(in_planes[f], out_planes["planned"], dims) for f in range(RING)]
        st = torch.cuda.Stream()
        s = st.cuda_stream
        for v in outs.values():
            for t in v:
                t.fill_(7)
        torch.cuda.synchronize()
        assert camera[0](fixed, cam, s) and planned[0](s)
        st.synchronize()
        identical = [bool(torch.equal(a[:, :d[2]], b[:, :d[2]])) for a, b, d in zip(outs["cam"], outs["planned"], dims)]
        arms = {"cam_ms": lambda i: camera[i % RING](path(i), cam, s), "planned_ms": lambda i: planned[i % RING](s)}
        for call in arms.values():  # warm-up: first launches, weight tables
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
        result["cases"][name] = dict(interp=interp, camera=list(cam), pose=list(fixed), output=[ow, oh], map_ms=map_ms, generate_ms=generate_ms,
                                     **times, identical=identical)
        vft.close()
        del outs
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
