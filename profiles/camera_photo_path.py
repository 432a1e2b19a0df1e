"""What photometry costs in a camera view of a lens rig on the GPU machine: T360B200_transformFrameCameraPhotoAsync against
the camera call (no pyramid) and the camera-mip call (a pyramid) it extends, a new pose every frame.  Needs a GPU.

    python profiles/camera_photo_path.py [--frames 100] [--windows 3] [--out FILE]

Workload: profiles/lens_path.py's, a 5760x2880 yuv420p dual-fisheye frame from back-to-back 190-degree lenses, bicubic,
inputs from a ring of frames larger than the L2 cache.  Two views: a 1920x1080 pinhole (90 x 50.6 degrees) looking across
the seam (yaw about 90), and a 1024x1024 180-degree equidistant dome with maxLevel 4, also across the seam.  Arms, each
the CUDA-event GPU time per frame of `--frames` frames enqueued back to back on one stream after a warm-up, `--windows`
windows per arm, the arms alternated window by window:
- base_ms: the camera call (pinhole) or the camera-mip call (dome);
- photo_id_ms: this call with the identity photometry and seamWidth 0;
- photo{0,4}_ms / photo{0,4}_stats_ms: this call with a non-identity photometry (falloff, unequal gains, offsets), the
  hard seam and a 4-degree belt, without and with statistics.
identical: whether the identity frame equals the base call's byte for byte.  Prints one JSON line (also appended to --out)
with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from profiles.lens_path import CUBIC, RING, dual_fisheye_rig, gpu_info  # noqa: E402
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
    identity, ph = photometries(t360)
    rng = np.random.default_rng(1)
    drift = np.cumsum(rng.normal(0, [1.0, 0.5, 0.5], (args.frames, 3)), 0)
    iw, ih = 5760, 2880
    views = {"pinhole_1920x1080": (t360.T360_CAMERA_PINHOLE, 1920, 1080, 90.0, 50.625, None),
             "dome_1024x1024": (t360.T360_CAMERA_EQUIDISTANT, 1024, 1024, 180.0, 180.0, (4, 0.0))}
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
    stats = torch.zeros((3, 6), dtype=torch.int64, device="cuda")
    sp = stats.data_ptr()
    ctx = t360.make_context(interpolation_alg=CUBIC, enable_low_pass_filter=0)
    result = dict(info, frames=args.frames, windows=args.windows, input=[iw, ih], ring_frames=RING, interp=CUBIC, cases={})
    for name, (model, ow, oh, hfov, vfov, minify) in views.items():
        cam = (model, 0.0)
        poses = [(90.0 + a, b, c, hfov, vfov) for a, b, c in drift]
        dims = [(*in_dims[0], ow, oh), (*in_dims[1], ow // 2, oh // 2), (*in_dims[2], ow // 2, oh // 2)]
        vft = t360.VideoFrameTransform(ctx)
        outs = {k: [torch.zeros((d[3], pitch(d[2])), dtype=torch.uint8, device="cuda") for d in dims] for k in ("base", "photo")}
        out_planes = {k: [(t.data_ptr(), t.stride(0)) for t in v] for k, v in outs.items()}
        if minify is None:
            base = [vft.make_camera_frame_call(in_planes[f], out_planes["base"], dims) for f in range(RING)]
            base_call = lambda i: base[i % RING](poses[i], cam, s, rig)
        else:
            base = [vft.make_camera_mip_frame_call(in_planes[f], out_planes["base"], dims) for f in range(RING)]
            base_call = lambda i: base[i % RING](poses[i], cam, minify, s, rig)
        photo = [vft.make_camera_photo_frame_call(in_planes[f], out_planes["photo"], dims) for f in range(RING)]
        st = torch.cuda.Stream()
        s = st.cuda_stream
        for v in outs.values():
            for t in v:
                t.fill_(7)
        torch.cuda.synchronize()
        assert base_call(0) and photo[0](rig, identity, 0.0, poses[0], cam, minify, s, sp)
        st.synchronize()
        identical = all(bool(torch.equal(a[:, :d[2]], b[:, :d[2]])) for a, b, d in zip(outs["base"], outs["photo"], dims))
        arms = {"base_ms": base_call, "photo_id_ms": lambda i: photo[i % RING](rig, identity, 0.0, poses[i], cam, minify, s)}
        for seam in (0.0, 4.0):
            arms[f"photo{seam:g}_ms"] = lambda i, seam=seam: photo[i % RING](rig, ph, seam, poses[i], cam, minify, s)
            arms[f"photo{seam:g}_stats_ms"] = lambda i, seam=seam: photo[i % RING](rig, ph, seam, poses[i], cam, minify, s, sp)
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
        result["cases"][name] = dict(model=model, output=[ow, oh], fov=[hfov, vfov], minify=minify, **times, identical=identical)
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
