"""What a rectilinear view costs on the GPU machine: the per-frame call (T360B200_transformFrameRectilinearAsync, a new
pose every frame) against the planned path for one pose (T360B200_rectilinearMap -> T360B200_generateMapFromWarp ->
T360B200_transformFrameAsync) and against the FLAT_FIXED per-view call (T360B200_transformFrameViewAsync, a new view
every frame) at the same output size; and a dual-fisheye frame through a rig.  Needs a GPU.

    python profiles/rectilinear_path.py [--frames 100] [--windows 3] [--out FILE]

Workloads, yuv420p, to a 1920x1080 view (chroma 960x540), without low-pass:
- equirect_cubic / equirect_lanczos4: a 7680x3840 equirect input, bicubic and Lanczos4;
- dual_fisheye_cubic: a 7680x3840 frame of two back-to-back 190-degree lenses side by side (seeded small k1..k4), bicubic.
Inputs come from a ring of frames larger than the L2 cache.  Per workload:
- map_ms / generate_ms: host wall time of rectilinearMap and of generateMapFromWarp, per plan index;
- rect_ms / planned_ms / view_ms: CUDA-event GPU time per frame of `--frames` frames enqueued back to back on one stream
  after a warm-up, `--windows` windows per arm, the arms alternated window by window (the rectilinear and view calls with a
  new pose every frame, the planned path with the fixed pose its maps were made for; no view arm for the rig);
- identical: whether the per-frame call and the planned path give the same bytes for the fixed pose, plane by plane.
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

CUBIC, LANCZOS4, EQUIRECT, FLAT_FIXED = 2, 4, 3, 2
RING = 3  # input frames of 44.2 MB: 133 MB, more than twice the H100's 50 MB L2
IN_W, IN_H, OUT_W, OUT_H = 7680, 3840, 1920, 1080


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().split(", ")
    return {"gpu": q[0], "power_limit_w": float(q[1])} if len(q) == 2 else {"gpu": None, "power_limit_w": None}


def dual_fisheye_rig(seed=0):
    import numpy as np
    import transform360_b200 as t360
    from tests.test_lens import _lens
    rng = np.random.default_rng(seed)
    rig = t360.T360LensRig(2, IN_W, IN_H)
    rig.lens[0] = _lens(rng, IN_H / 2, IN_W / 4 - 0.5, IN_H / 2 - 0.5, 0, 0, 0, 95)
    rig.lens[1] = _lens(rng, IN_H / 2, 3 * IN_W / 4 - 0.5, IN_H / 2 - 0.5, 180, 0, 0, 95)
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
    rig = dual_fisheye_rig()
    hfov = 90.0
    vfov = t360.square_pixel_vfov(hfov, OUT_W, OUT_H)
    fixed = (35.0, -10.0, 5.0, hfov, vfov)
    rng = np.random.default_rng(1)
    steps = np.cumsum(rng.normal(0, [3.0, 1.0, 1.0, 1.0], (args.frames, 4)), 0)
    path = [(35.0 + a, float(np.clip(-10.0 + b, -80, 80)), 5.0 + c, float(np.clip(hfov + d, 30, 150)), vfov) for a, b, c, d in steps]
    pitch = lambda w: (w + 255) // 256 * 256
    in_dims = [(IN_W, IN_H), (IN_W // 2, IN_H // 2), (IN_W // 2, IN_H // 2)]
    dims = [(*in_dims[0], OUT_W, OUT_H), (*in_dims[1], OUT_W // 2, OUT_H // 2), (*in_dims[2], OUT_W // 2, OUT_H // 2)]
    ring = []
    for f in range(RING):
        frame = []
        for p, (w, h) in enumerate(in_dims):
            t = torch.zeros((h, pitch(w)), dtype=torch.uint8, device="cuda")
            t[:, :w] = torch.from_numpy(co.noise_plane(w, h, plane=p, frame=f)).cuda()
            frame.append(t)
        ring.append(frame)
    in_planes = [[(t.data_ptr(), t.stride(0)) for t in frame] for frame in ring]
    result = dict(info, frames=args.frames, windows=args.windows, input=[IN_W, IN_H], output=[OUT_W, OUT_H], ring_frames=RING, cases={})
    workloads = {"equirect_cubic": (CUBIC, None), "equirect_lanczos4": (LANCZOS4, None), "dual_fisheye_cubic": (CUBIC, rig)}
    for name, (interp, r) in workloads.items():
        ctx = t360.make_context(interpolation_alg=interp, enable_low_pass_filter=0)
        border = t360.BORDER_TRANSPARENT if r is not None else t360.BORDER_WRAP
        vft = t360.VideoFrameTransform(ctx)
        map_ms, generate_ms = [], []
        for idx in (0, 1):
            t0 = time.perf_counter()
            m = t360.rectilinear_map(ctx, fixed, *dims[idx], r)
            map_ms.append(round((time.perf_counter() - t0) * 1e3, 1))
            t0 = time.perf_counter()
            assert vft.generate_map_from_warp(m, *dims[idx][:2], idx, border)
            generate_ms.append(round((time.perf_counter() - t0) * 1e3, 1))
        outs = {k: [torch.zeros((d[3], pitch(d[2])), dtype=torch.uint8, device="cuda") for d in dims] for k in ("rect", "planned", "view")}
        out_planes = {k: [(t.data_ptr(), t.stride(0)) for t in v] for k, v in outs.items()}
        rect = [vft.make_rectilinear_frame_call(in_planes[f], out_planes["rect"], dims) for f in range(RING)]
        planned = [vft.make_frame_call(in_planes[f], out_planes["planned"], dims) for f in range(RING)]
        st = torch.cuda.Stream()
        s = st.cuda_stream
        for v in outs.values():
            for t in v:
                t.fill_(7)
        torch.cuda.synchronize()
        assert rect[0](fixed, s, r) and planned[0](s)
        st.synchronize()
        identical = [bool(torch.equal(a[:, :d[2]], b[:, :d[2]])) for a, b, d in zip(outs["rect"], outs["planned"], dims)]
        arms = {"rect_ms": lambda i: rect[i % RING](path[i], s, r), "planned_ms": lambda i: planned[i % RING](s)}
        view_vft = None
        if r is None:  # the FLAT_FIXED latitude / longitude window at the same output size, a new view every frame
            view_vft = t360.VideoFrameTransform(t360.make_context(interpolation_alg=interp, enable_low_pass_filter=0, output_layout=FLAT_FIXED,
                                                                  fixed_hfov=hfov, fixed_vfov=vfov))
            for idx in (0, 1):
                assert view_vft.generateMapForPlane(*dims[idx], idx)
            view = [view_vft.make_view_frame_call(in_planes[f], out_planes["view"], dims) for f in range(RING)]
            arms["view_ms"] = lambda i: view[i % RING]((path[i][0], path[i][1], path[i][3], path[i][4]), s)
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
        result["cases"][name] = dict(interp=interp, rig=r is not None, map_ms=map_ms, generate_ms=generate_ms, **times, identical=identical)
        vft.close()
        if view_vft:
            view_vft.close()
        del outs
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
