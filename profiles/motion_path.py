"""What a rig motion over the readout costs on the GPU machine: the lens-motion call against the lens-photo call on
profiles/lens_photo_path.py's frame, and the camera-motion call against the camera-photo call at
profiles/camera_photo_path.py's views, a new orientation or pose and a new motion every frame.  Needs a GPU.

    python profiles/motion_path.py [--frames 100] [--windows 3] [--out FILE]

Workload: a 5760x2880 yuv420p dual-fisheye frame from back-to-back 190-degree lenses (profiles/lens_path.py), bicubic,
inputs from a ring of frames larger than the L2 cache, the non-identity photometry of lens_photo_path.py.  Sphere outputs:
EQUIRECT 5760x2880 and CUBEMAP_32 3840x2560, the hard seam and a 4-degree belt.  Camera views: a 1920x1080 pinhole and a
1024x1024 180-degree equidistant dome with maxLevel 4, across the seam.  The motion: 9 samples of a gyro-like turn of
about 2 degrees across a top-to-bottom readout of each lens.  Arms, each the CUDA-event GPU time per frame of `--frames`
frames enqueued back to back on one stream after a warm-up, `--windows` windows per arm, the arms alternated window by
window: photo*_ms the photometric call, motion*_ms the motion call with the same arguments.  identical: whether the motion
call with all-zero deltas gives the photometric call's frame, byte for byte.  Prints one JSON line (also appended to
--out) with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from profiles.lens_path import CUBEMAP_32, CUBIC, EQUIRECT, RING, dual_fisheye_rig, gpu_info  # noqa: E402
from profiles.lens_photo_path import photometries  # noqa: E402


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
    rig = dual_fisheye_rig()
    _, ph = photometries(t360)
    rng = np.random.default_rng(1)
    path = [tuple(float(v) for v in o) for o in np.cumsum(rng.normal(0, [3.0, 1.0, 1.0], (args.frames, 3)), 0) + (35.0, -10.0, 5.0)]
    readouts = ((0.0, 1.0, 0.0), (0.0, 1.0, 0.0))
    motions = [t360.rig_motion([tuple(d) for d in np.cumsum(rng.normal(0, 0.25, (9, 3)), 0) - 1.0], readouts) for _ in range(args.frames)]
    still = t360.rig_motion([(0.0, 0.0, 0.0)] * 9, readouts)
    iw, ih = 5760, 2880
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
    result = dict(info, frames=args.frames, windows=args.windows, input=[iw, ih], ring_frames=RING, interp=CUBIC, motion_samples=9, cases={})

    def measure(arms, st):
        for call in arms.values():  # warm-up: first launches, weight tables, the table uploads
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
        return times

    def same(outs, dims):
        return all(bool(torch.equal(a[:, :d[2]], b[:, :d[2]])) for a, b, d in zip(outs["photo"], outs["motion"], dims))

    targets = {"equirect_5760x2880": (EQUIRECT, 5760, 2880), "cubemap_32_3840x2560": (CUBEMAP_32, 3840, 2560)}
    for name, (layout, ow, oh) in targets.items():
        ctx = t360.make_context(output_layout=layout, interpolation_alg=CUBIC, enable_low_pass_filter=0)
        dims = [(*in_dims[0], ow, oh), (*in_dims[1], ow // 2, oh // 2), (*in_dims[2], ow // 2, oh // 2)]
        vft = t360.VideoFrameTransform(ctx)
        outs = {k: [torch.zeros((d[3], pitch(d[2])), dtype=torch.uint8, device="cuda") for d in dims] for k in ("photo", "motion")}
        out_planes = {k: [(t.data_ptr(), t.stride(0)) for t in v] for k, v in outs.items()}
        photo = [vft.make_lens_photo_frame_call(in_planes[f], out_planes["photo"], dims) for f in range(RING)]
        moving = [vft.make_lens_motion_frame_call(in_planes[f], out_planes["motion"], dims) for f in range(RING)]
        st = torch.cuda.Stream()
        s = st.cuda_stream
        identical = {}
        for seam in (0.0, 4.0):
            torch.cuda.synchronize()
            assert photo[0](rig, ph, seam, path[0], s) and moving[0](rig, ph, seam, path[0], still, s)
            st.synchronize()
            identical[f"{seam:g}"] = same(outs, dims)
        arms = {}
        for seam in (0.0, 4.0):
            arms[f"photo{seam:g}_ms"] = lambda i, seam=seam: photo[i % RING](rig, ph, seam, path[i], s)
            arms[f"motion{seam:g}_ms"] = lambda i, seam=seam: moving[i % RING](rig, ph, seam, path[i], motions[i], s)
        result["cases"][name] = dict(layout=layout, output=[ow, oh], **measure(arms, st), identical=identical)
        vft.close()
        del outs
        torch.cuda.empty_cache()
    drift = np.cumsum(rng.normal(0, [1.0, 0.5, 0.5], (args.frames, 3)), 0)
    views = {"pinhole_1920x1080": (t360.T360_CAMERA_PINHOLE, 1920, 1080, 90.0, 50.625, None),
             "dome_1024x1024": (t360.T360_CAMERA_EQUIDISTANT, 1024, 1024, 180.0, 180.0, (4, 0.0))}
    ctx = t360.make_context(interpolation_alg=CUBIC, enable_low_pass_filter=0)
    for name, (model, ow, oh, hfov, vfov, minify) in views.items():
        cam = (model, 0.0)
        poses = [(90.0 + a, b, c, hfov, vfov) for a, b, c in drift]
        dims = [(*in_dims[0], ow, oh), (*in_dims[1], ow // 2, oh // 2), (*in_dims[2], ow // 2, oh // 2)]
        vft = t360.VideoFrameTransform(ctx)
        outs = {k: [torch.zeros((d[3], pitch(d[2])), dtype=torch.uint8, device="cuda") for d in dims] for k in ("photo", "motion")}
        out_planes = {k: [(t.data_ptr(), t.stride(0)) for t in v] for k, v in outs.items()}
        photo = [vft.make_camera_photo_frame_call(in_planes[f], out_planes["photo"], dims) for f in range(RING)]
        moving = [vft.make_camera_motion_frame_call(in_planes[f], out_planes["motion"], dims) for f in range(RING)]
        st = torch.cuda.Stream()
        s = st.cuda_stream
        torch.cuda.synchronize()
        assert photo[0](rig, ph, 4.0, poses[0], cam, minify, s) and moving[0](rig, ph, 4.0, poses[0], cam, minify, still, s)
        st.synchronize()
        identical = same(outs, dims)
        arms = {}
        for seam in (0.0, 4.0):
            arms[f"photo{seam:g}_ms"] = lambda i, seam=seam: photo[i % RING](rig, ph, seam, poses[i], cam, minify, s)
            arms[f"motion{seam:g}_ms"] = lambda i, seam=seam: moving[i % RING](rig, ph, seam, poses[i], cam, minify, motions[i], s)
        result["cases"][name] = dict(model=model, output=[ow, oh], fov=[hfov, vfov], minify=minify, **measure(arms, st), identical=identical)
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
