"""What the anti-aliased camera views cost on the GPU machine: T360B200_transformFrameCameraMipAsync at maxLevel 0 (the
camera call itself), 4 and 6, a new pose every frame.  Needs a GPU.

    python profiles/camera_mip_path.py [--frames 100] [--windows 3] [--out FILE]

Workloads, yuv420p from a 7680x3840 equirect (chroma 3840x1920), bicubic, without low-pass:
- pinhole_1080p: a 1920x1080 pinhole view of 90 degrees across (no minification: the cost of leaving the option on);
- pinhole_540p: a 960x540 pinhole view of 100 degrees across (a preview or thumbnail);
- dome_1024: a 1024x1024 equidistant 180-degree dome master;
- little_planet_1080: a 1080x1080 stereographic view of 300 degrees looking at the nadir.
Inputs come from a ring of frames larger than the L2 cache.  Per workload and maxLevel, mip<L>_ms: CUDA-event GPU time
per frame of `--frames` frames enqueued back to back on one stream after a warm-up, `--windows` windows per arm, the arms
alternated window by window; launches: kernel launches per frame.  pyramid<L>_ms: the same call rendering a 16x16 view
(chroma 8x8), i.e. the pyramid of the whole input and a negligible gather.  Prints one JSON line (also appended to
--out) with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from profiles.rectilinear_path import RING, gpu_info  # noqa: E402

CUBIC = 2
IN_W, IN_H = 7680, 3840
PINHOLE, EQUIDISTANT, STEREOGRAPHIC = 0, 1, 2
LEVELS = (0, 4, 6)


def workloads():
    """name -> (camera, output luma size, the pose at frame i)"""
    import numpy as np
    import transform360_b200 as t360
    rng = np.random.default_rng(1)
    steps = np.cumsum(rng.normal(0, [3.0, 1.0, 1.0], (1000, 3)), 0)
    walk = lambda h, v, pitch=-10.0: (lambda i: (35.0 + steps[i, 0], float(np.clip(pitch + steps[i, 1], -80, 80)), 5.0 + steps[i, 2], h, v))
    return {
        "pinhole_1080p": ((PINHOLE, 0.0), (1920, 1080), walk(90.0, t360.square_pixel_vfov(90.0, 1920, 1080))),
        "pinhole_540p": ((PINHOLE, 0.0), (960, 540), walk(100.0, t360.square_pixel_vfov(100.0, 960, 540))),
        "dome_1024": ((EQUIDISTANT, 0.0), (1024, 1024), walk(180.0, 180.0, 20.0)),
        "little_planet_1080": ((STEREOGRAPHIC, 0.0), (1080, 1080), lambda i: (steps[i, 0], -90.0, steps[i, 2], 300.0, 300.0)),
    }


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
    result = dict(info, frames=args.frames, windows=args.windows, input=[IN_W, IN_H], ring_frames=RING, interp="cubic", cases={})
    ctx = t360.make_context(interpolation_alg=CUBIC, enable_low_pass_filter=0)
    vft = t360.VideoFrameTransform(ctx)
    st = torch.cuda.Stream()
    s = st.cuda_stream

    def timed(arms):
        for call in arms.values():  # warm-up: first launches, scratch, tap tables
            for i in range(10):
                assert call(i)
        st.synchronize()
        times = {k: [] for k in arms}
        launches = {}
        for _ in range(args.windows):
            for k, call in arms.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                n0 = t360.kernel_launch_count()
                a.record(st)
                for i in range(args.frames):
                    assert call(i)
                b.record(st)
                b.synchronize()
                launches[k] = (t360.kernel_launch_count() - n0) / args.frames
                times[k].append(round(a.elapsed_time(b) / args.frames, 4))
        return times, launches

    for name, (cam, (ow, oh), path) in workloads().items():
        dims = [(*in_dims[0], ow, oh), (*in_dims[1], ow // 2, oh // 2), (*in_dims[2], ow // 2, oh // 2)]
        outs = [torch.zeros((d[3], pitch(d[2])), dtype=torch.uint8, device="cuda") for d in dims]
        out_planes = [(t.data_ptr(), t.stride(0)) for t in outs]
        calls = [vft.make_camera_mip_frame_call(in_planes[f], out_planes, dims) for f in range(RING)]
        arms = {f"mip{L}_ms": (lambda i, L=L: calls[i % RING](path(i), cam, (L, 0.0), s)) for L in LEVELS}
        times, launches = timed(arms)
        result["cases"][name] = dict(camera=list(cam), output=[ow, oh], **times, launches=launches)
        del outs
    tiny = [(*in_dims[0], 16, 16), (*in_dims[1], 8, 8), (*in_dims[2], 8, 8)]
    outs = [torch.zeros((d[3], pitch(d[2])), dtype=torch.uint8, device="cuda") for d in tiny]
    out_planes = [(t.data_ptr(), t.stride(0)) for t in outs]
    calls = [vft.make_camera_mip_frame_call(in_planes[f], out_planes, tiny) for f in range(RING)]
    arms = {f"pyramid{L}_ms": (lambda i, L=L: calls[i % RING]((float(i), -10.0, 0.0, 90.0, 90.0), PINHOLE, (L, 0.0), s)) for L in LEVELS}
    times, launches = timed(arms)
    result["pyramid"] = dict(output=[16, 16], **times, launches=launches)
    vft.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
