"""Per-frame poses for barrel outputs on the GPU machine: the frame time of the planned whole-frame entry point against the
per-frame pose entry point (T360B200_transformFramePoseAsync) at the same pose, and of the latter with a new pose every
frame.  Needs a GPU.

    python profiles/pose_path.py [--frames 200] [--rounds 5] [--out FILE]

Cases (yuv420p frames): MONO 7680x3840 equirect -> BARREL 5760x2304 (square end caps: 0.2 w = h / 2), bicubic, without and
with low-pass (32 x 15 segments, adjust_kernel), and MONO 3840x1920 equirect -> BARREL_SPLIT 2880x1920, Lanczos4, without
low-pass.  Variants, alternated `--rounds` times in one process:
  planned  T360B200_transformFrameAsync of a transform planned for the fixed pose
  fixed    T360B200_transformFramePoseAsync with that same pose every frame
  moving   T360B200_transformFramePoseAsync with a new pose every frame: a seeded path that sweeps yaw over 720 degrees,
           crosses a pole and rolls
  repeated T360B200_transformFramePoseAsync with the poses of `moving`, each twice in a row
Per variant and round (timing without the profiler): wall_us = CUDA-event time of the window over its frames (frames
enqueued back to back, no synchronisation: if the host enqueues more slowly than the GPU runs, this is the host's rate);
host_us = the median host time of one enqueue call.  Then one window per variant under torch.profiler: gpu_us = the device
time of all its kernels, copies and memsets over its frames (what the GPU spends on a frame, whether or not it waits for
the host in between).  outputs_identical: the pose entry point's frames at the fixed pose equal the planned frames, and
three frames of the path equal fresh transforms planned for their poses.  Prints one JSON line (also
appended to --out) with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

FIXED = dict(fixed_yaw=35.0, fixed_pitch=-10.0, fixed_roll=5.0)
LOW_PASS = dict(enable_low_pass_filter=1, num_horizontal_segments=32, num_vertical_segments=15, adjust_kernel=1)
CASES = {  # name: (context overrides, (in w, in h, out w, out h))
    "barrel": (dict(FIXED, output_layout=4, interpolation_alg=2, enable_low_pass_filter=0), (7680, 3840, 5760, 2304)),
    "barrel_low_pass": (dict(FIXED, output_layout=4, interpolation_alg=2, **LOW_PASS), (7680, 3840, 5760, 2304)),
    "barrel_split_lanczos4": (dict(FIXED, output_layout=5, interpolation_alg=4, enable_low_pass_filter=0), (3840, 1920, 2880, 1920)),
}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().split(", ")
    return {"gpu": q[0], "power_limit_w": float(q[1])} if len(q) == 2 else {"gpu": None, "power_limit_w": None}


def pose_path(n, seed=360):
    rng = np.random.default_rng(seed)
    t = np.linspace(0.0, 1.0, n)
    yaw = -360.0 + 720.0 * t + rng.uniform(-2, 2, n)
    pitch = 105.0 * np.sin(2 * np.pi * t) + rng.uniform(-2, 2, n)  # beyond +-90: over a pole
    roll = 30.0 * np.sin(6 * np.pi * t) + rng.uniform(-2, 2, n)
    return [tuple(float(np.float32(v)) for v in row) + (120.0, 110.0) for row in zip(yaw, pitch, roll)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200, help="frames per timed window")
    ap.add_argument("--rounds", type=int, default=5, help="alternated windows per variant")
    ap.add_argument("--out", help="append the JSON line to this file")
    args = ap.parse_args()
    import torch
    import transform360_b200 as t360
    from oracle import c_oracle as co
    from transform360_b200.stream import FrameTransformer, StreamSpec

    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    info = gpu_info()
    pitch = lambda w: (w + 255) // 256 * 256  # noqa: E731
    st = torch.cuda.Stream()

    def planes(shape_of):
        out = []
        for p in range(3):
            w, h = shape_of(p)
            out.append(torch.zeros((h, pitch(w)), dtype=torch.uint8, device="cuda"))
        return out

    path = pose_path(args.frames)
    fixed = tuple(float(np.float32(FIXED[k])) for k in ("fixed_yaw", "fixed_pitch", "fixed_roll")) + (120.0, 110.0)
    result = dict(info, frames=args.frames, rounds=args.rounds, cases={})
    for name, (ov, size) in CASES.items():
        spec = StreamSpec(*size)
        d_in = planes(lambda p: spec.plane_dims(p)[:2])
        for p, t in enumerate(d_in):
            w, h = spec.plane_dims(p)[:2]
            t[:, :w] = torch.from_numpy(co.noise_plane(w, h, plane=p, frame=0)).cuda()
        ptrs = lambda ts: [(t.data_ptr(), t.stride(0)) for t in ts]  # noqa: E731
        host = lambda ts: [t[:, :spec.plane_dims(p)[2]].cpu().numpy() for p, t in enumerate(ts)]  # noqa: E731
        ft = FrameTransformer(t360.make_context(**ov), spec)
        out_planned, out_view = planes(lambda p: spec.plane_dims(p)[2:4]), planes(lambda p: spec.plane_dims(p)[2:4])
        planned = ft.frame_call(ptrs(d_in), ptrs(out_planned))
        view = ft.pose_frame_call(ptrs(d_in), ptrs(out_view))
        variants = {
            "planned": lambda f: planned(st.cuda_stream),
            "fixed": lambda f: view(fixed, st.cuda_stream),
            "moving": lambda f: view(path[f], st.cuda_stream),
            "repeated": lambda f: view(path[f // 2], st.cuda_stream),
        }
        frames = {k: args.frames * 2 if k == "repeated" else args.frames for k in variants}
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = {k: dict(wall_us=[], host_us=[]) for k in variants}
        for k, fn in variants.items():  # warm-up: every scratch plane, table and ring entry
            for f in range(frames[k]):
                assert fn(f), (name, k)
        st.synchronize()
        for _ in range(args.rounds):
            for k, fn in variants.items():
                host_s = []
                st.synchronize()
                a.record(st)
                for f in range(frames[k]):
                    t0 = time.perf_counter()
                    assert fn(f)
                    host_s.append(time.perf_counter() - t0)
                b.record(st)
                st.synchronize()
                times[k]["wall_us"].append(round(a.elapsed_time(b) * 1e3 / frames[k], 2))
                times[k]["host_us"].append(round(statistics.median(host_s) * 1e6, 1))
        for k, fn in variants.items():
            st.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for f in range(frames[k]):
                    assert fn(f)
                st.synchronize()
            device_us = sum(getattr(e, "self_device_time_total", 0) for e in prof.key_averages())
            times[k]["gpu_us"] = [round(device_us / frames[k], 2)]
        # outputs: the fixed pose through both entry points, and three poses of the path against fresh plans
        assert planned(st.cuda_stream) and view(fixed, st.cuda_stream)
        st.synchronize()
        identical = all(np.array_equal(a, b) for a, b in zip(host(out_planned), host(out_view)))
        for f in (0, args.frames // 3, args.frames - 1):
            assert view(path[f], st.cuda_stream)
            st.synchronize()
            got = host(out_view)
            fresh = FrameTransformer(t360.make_context(**dict(ov, fixed_yaw=path[f][0], fixed_pitch=path[f][1], fixed_roll=path[f][2])),
                                     spec)
            assert fresh.frame_call(ptrs(d_in), ptrs(out_planned))(st.cuda_stream)
            st.synchronize()
            identical = identical and all(np.array_equal(a, b) for a, b in zip(got, host(out_planned)))
            fresh.close()
        ft.close()
        summary = {k: {m: statistics.median(v) for m, v in t.items()} for k, t in times.items()}
        summary["spread_wall_us"] = {k: [min(t["wall_us"]), max(t["wall_us"])] for k, t in times.items()}
        result["cases"][name] = dict(size=list(size), median=summary, rounds=times, outputs_identical=identical)
        print(name, json.dumps(summary), "identical" if identical else "DIFFERENT", flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "a") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
