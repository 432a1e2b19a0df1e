"""What the anisotropic camera views cost on the GPU machine: T360B200_transformFrameCameraAnisoAsync at maxProbes 1 (the
camera-mip call itself), 4, 8 and 16, maxLevel 6, a new pose every frame.  Needs a GPU.

    python profiles/camera_aniso_path.py [--frames 100] [--windows 3] [--out FILE]

Workloads: camera_mip_path.py's (yuv420p from a 7680x3840 equirect, bicubic, without low-pass; a 1920x1080 pinhole of
90 degrees, a 960x540 pinhole of 100 degrees, a 1024x1024 equidistant 180-degree dome, a 1080x1080 stereographic
300-degree little planet).  Inputs come from a ring of frames larger than the L2 cache.  Per workload and maxProbes N,
aniso<N>_ms: CUDA-event GPU time per frame of `--frames` frames enqueued back to back on one stream after a warm-up,
`--windows` windows per arm, the arms alternated window by window; launches: kernel launches per frame; mean_probes: the
mean probe count of the luma plane's pixels (from the host twin, at frame 0's pose).  Prints one JSON line (also
appended to --out) with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from profiles.camera_mip_path import CUBIC, IN_H, IN_W, workloads  # noqa: E402
from profiles.rectilinear_path import RING, gpu_info  # noqa: E402

MAX_LEVEL = 6
PROBES = (1, 4, 8, 16)


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
    result = dict(info, frames=args.frames, windows=args.windows, input=[IN_W, IN_H], ring_frames=RING, interp="cubic", max_level=MAX_LEVEL,
                  cases={})
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
        calls = [vft.make_camera_aniso_frame_call(in_planes[f], out_planes, dims) for f in range(RING)]
        arms = {f"aniso{n}_ms": (lambda i, n=n: calls[i % RING](path(i), cam, (MAX_LEVEL, 0.0), n, s)) for n in PROBES}
        times, launches = timed(arms)
        mean_probes = {f"aniso{n}_ms": round(float(t360.camera_aniso_maps(ctx, path(0), cam, (MAX_LEVEL, 0.0), n, IN_W, IN_H, ow, oh)[4].mean()), 3)
                       for n in PROBES}
        result["cases"][name] = dict(camera=list(cam), output=[ow, oh], **times, launches=launches, mean_probes=mean_probes)
        del outs
    vft.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
