"""What a VR180 view of a stereo fisheye rig costs on the GPU machine: T360B200_transformFrameStereoCameraAsync, a new pose
every frame.  Needs a GPU.

    python profiles/stereo_camera_path.py [--frames 100] [--windows 3] [--out FILE]

Workload: a synthetic 8192x4096 yuv420p side-by-side frame of two forward 190-degree lenses (lens 0 the left eye on the
left half, lens 1 the right eye with a 1-degree rectification rotation), bicubic, inputs from a ring of frames larger than
the L2 cache.  Output: 7680x3840 LR, each eye a 180 x 180 degree equirect (T360_CAMERA_EQUIRECT), a drifting pose.  Arms,
each the CUDA-event GPU time per frame of `--frames` frames enqueued back to back on one stream after a warm-up,
`--windows` windows per arm, the arms alternated window by window:
- identity_ms: the identity photometry, no pyramid;
- photo_ms / photo_stats_ms: a non-identity photometry (falloff, unequal gains, offsets), without and with statistics;
- mip_ms: the non-identity photometry with minify (3, 0).
Prints one JSON line (also appended to --out) with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from profiles.lens_path import CUBIC, gpu_info  # noqa: E402
from profiles.lens_photo_path import photometries  # noqa: E402

RING = 3  # input frames of 50.3 MB: 151 MB, three times the H100's 50 MB L2


def stereo_rig(t360, iw, ih):
    rig = t360.T360LensRig(2, iw, ih)
    f = (iw / 4) / (95 * 3.141592653589793 / 180)  # the 190-degree circle fills its half's height
    for i in range(2):
        rig.lens[i] = t360.T360Lens(f, f, iw / 4 - 0.5 + i * iw / 2, ih / 2 - 0.5, (0.0, 0.0, 0.0, 0.0), 0.6 * i, -0.8 * i, 0.3 * i, 95.0)
    return rig


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100, help="frames per timed window")
    ap.add_argument("--windows", type=int, default=3, help="timed windows per arm")
    ap.add_argument("--out", help="append the JSON line to this file")
    args = ap.parse_args()
    import numpy as np
    import torch
    import transform360_b200 as t360
    from oracle import c_oracle as co

    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    info = gpu_info()
    iw, ih, ow, oh = 8192, 4096, 7680, 3840
    rig = stereo_rig(t360, iw, ih)
    identity, ph = photometries(t360)
    rng = np.random.default_rng(1)
    drift = np.cumsum(rng.normal(0, [0.3, 0.2, 0.1], (args.frames, 3)), 0)
    poses = [(a, b, c, 180.0, 180.0) for a, b, c in drift]
    cam = (t360.T360_CAMERA_EQUIRECT, 0.0)
    pitch = lambda w: (w + 255) // 256 * 256
    in_dims = [(iw, ih), (iw // 2, ih // 2), (iw // 2, ih // 2)]
    dims = [(*in_dims[0], ow, oh), (*in_dims[1], ow // 2, oh // 2), (*in_dims[2], ow // 2, oh // 2)]
    ring = []
    for f in range(RING):
        frame = []
        for p, (w, h) in enumerate(in_dims):
            t = torch.zeros((h, pitch(w)), dtype=torch.uint8, device="cuda")
            t[:, :w] = torch.from_numpy(co.noise_plane(w, h, plane=p, frame=f)).cuda()
            frame.append(t)
        ring.append(frame)
    in_planes = [[(t.data_ptr(), t.stride(0)) for t in frame] for frame in ring]
    outs = [torch.zeros((d[3], pitch(d[2])), dtype=torch.uint8, device="cuda") for d in dims]
    out_planes = [(t.data_ptr(), t.stride(0)) for t in outs]
    stats = torch.zeros((3, 6), dtype=torch.int64, device="cuda")
    sp = stats.data_ptr()
    ctx = t360.make_context(interpolation_alg=CUBIC, enable_low_pass_filter=0, output_stereo_format=t360.STEREO_FORMAT_LR)
    vft = t360.VideoFrameTransform(ctx)
    calls = [vft.make_stereo_camera_frame_call(in_planes[f], out_planes, dims) for f in range(RING)]
    st = torch.cuda.Stream()
    s = st.cuda_stream
    arms = {"identity_ms": lambda i: calls[i % RING](rig, identity, poses[i], cam, None, s),
            "photo_ms": lambda i: calls[i % RING](rig, ph, poses[i], cam, None, s),
            "photo_stats_ms": lambda i: calls[i % RING](rig, ph, poses[i], cam, None, s, sp),
            "mip_ms": lambda i: calls[i % RING](rig, ph, poses[i], cam, (3, 0.0), s)}
    for call in arms.values():  # warm-up: first launches, weight tables, pyramid scratch
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
    vft.close()
    result = dict(info, frames=args.frames, windows=args.windows, input=[iw, ih], output=[ow, oh], ring_frames=RING, interp=CUBIC,
                  camera="equirect 180 x 180 per eye, LR", **times)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
