"""What lens photometry costs on the GPU machine: the photometric call (T360B200_transformFrameLensPhotoAsync) against the
lens call (hard seam) and the blend call (feathered seam) it extends, a new orientation every frame.  Needs a GPU.

    python profiles/lens_photo_path.py [--frames 100] [--windows 3] [--out FILE]

Workload: profiles/lens_path.py's, a 5760x2880 yuv420p dual-fisheye frame from back-to-back 190-degree lenses, bicubic,
to EQUIRECT 5760x2880 and to CUBEMAP_32 3840x2560, inputs from a ring of frames larger than the L2 cache.  Arms, each
the CUDA-event GPU time per frame of `--frames` frames enqueued back to back on one stream after a warm-up, `--windows`
windows per arm, the arms alternated window by window:
- lens_ms: the lens call; photo_hard_id_ms / photo_hard_ms: the photometric call with seamWidth 0 and the identity / a
  non-identity photometry (falloff, unequal gains, offsets); photo_hard_stats_ms: the latter with statistics;
- blend4_ms / blend10_ms: the blend call with belts of 4 and 10 degrees; photo4_ms / photo10_ms, photo4_stats_ms /
  photo10_stats_ms: the photometric call with the non-identity photometry and those belts, without and with statistics.
identical: whether the identity photometry's frame equals the lens call's and the blend call's (4 degrees), byte for
byte.  Prints one JSON line (also appended to --out) with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from profiles.lens_path import CUBEMAP_32, CUBIC, EQUIRECT, RING, dual_fisheye_rig, gpu_info  # noqa: E402


def photometries(t360):
    identity = t360.T360RigPhotometry(16)
    ph = t360.T360RigPhotometry(16)
    for i in range(2):
        identity.lens[i].gain[:] = [1.0, 1.0, 1.0]
        ph.lens[i].vignetting[:] = [-0.06 - 0.02 * i, 0.004, 0.0]
        ph.lens[i].gain[:] = [1.0 + 0.1 * i, 0.97, 1.02]
        ph.lens[i].offset[:] = [1.5 - 3 * i, -0.5, 0.25]
    return identity, ph


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
    path = [tuple(float(v) for v in o) for o in np.cumsum(rng.normal(0, [3.0, 1.0, 1.0], (args.frames, 3)), 0) + (35.0, -10.0, 5.0)]
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
    stats = torch.zeros((3, 6), dtype=torch.int64, device="cuda")
    sp = stats.data_ptr()
    result = dict(info, frames=args.frames, windows=args.windows, input=[iw, ih], ring_frames=RING, interp=CUBIC, cases={})
    for name, (layout, ow, oh) in targets.items():
        ctx = t360.make_context(output_layout=layout, interpolation_alg=CUBIC, enable_low_pass_filter=0)
        dims = [(*in_dims[0], ow, oh), (*in_dims[1], ow // 2, oh // 2), (*in_dims[2], ow // 2, oh // 2)]
        vft = t360.VideoFrameTransform(ctx)
        outs = {k: [torch.zeros((d[3], pitch(d[2])), dtype=torch.uint8, device="cuda") for d in dims] for k in ("base", "photo")}
        out_planes = {k: [(t.data_ptr(), t.stride(0)) for t in v] for k, v in outs.items()}
        lens = [vft.make_lens_frame_call(in_planes[f], out_planes["base"], dims) for f in range(RING)]
        blend = [vft.make_lens_blend_frame_call(in_planes[f], out_planes["base"], dims) for f in range(RING)]
        photo = [vft.make_lens_photo_frame_call(in_planes[f], out_planes["photo"], dims) for f in range(RING)]
        st = torch.cuda.Stream()
        s = st.cuda_stream
        identical = {}
        for seam, base in ((0.0, lambda: lens[0](rig, path[0], s)), (4.0, lambda: blend[0](rig, 4.0, path[0], s))):
            for v in outs.values():
                for t in v:
                    t.fill_(7)
            torch.cuda.synchronize()
            assert base() and photo[0](rig, identity, seam, path[0], s, sp)
            st.synchronize()
            identical[f"{seam:g}"] = all(bool(torch.equal(a[:, :d[2]], b[:, :d[2]])) for a, b, d in zip(outs["base"], outs["photo"], dims))
        arms = {
            "lens_ms": lambda i: lens[i % RING](rig, path[i], s),
            "photo_hard_id_ms": lambda i: photo[i % RING](rig, identity, 0.0, path[i], s),
            "photo_hard_ms": lambda i: photo[i % RING](rig, ph, 0.0, path[i], s),
            "photo_hard_stats_ms": lambda i: photo[i % RING](rig, ph, 0.0, path[i], s, sp),
        }
        for seam in (4.0, 10.0):
            arms[f"blend{seam:g}_ms"] = lambda i, seam=seam: blend[i % RING](rig, seam, path[i], s)
            arms[f"photo{seam:g}_ms"] = lambda i, seam=seam: photo[i % RING](rig, ph, seam, path[i], s)
            arms[f"photo{seam:g}_stats_ms"] = lambda i, seam=seam: photo[i % RING](rig, ph, seam, path[i], s, sp)
        for call in arms.values():  # warm-up: first launches, weight tables, the table upload
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
        result["cases"][name] = dict(layout=layout, output=[ow, oh], **times, identical=identical)
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
