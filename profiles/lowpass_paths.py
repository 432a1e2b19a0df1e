"""The per-plane low-pass paths on the GPU machine: T360B200_lowPassPlaneAsync on cfg3's luma and chroma planes, and the
per-plane entry point T360B200_transformFramePlaneAsync (low-pass, then the gather) on the same planes.  Neither bench.py
nor profiles/view_path.py times them: bench.py runs whole frames, whose low-pass is one merged launch per vertical
half-size.  Needs a GPU.

    python profiles/lowpass_paths.py [--calls 200] [--rounds 5] [--label NAME] [--out FILE]

Per case and round: us = CUDA-event time of a window of `calls` calls enqueued back to back on one stream, per call.
out_sha: a digest of the case's output plane (to compare two builds).  To compare two builds, run the script from each
tree in turn, alternating, and compare the medians against the spread of each build's rounds.  Prints one JSON line (also
appended to --out) with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

CFG3 = dict(interpolation_alg=2, enable_low_pass_filter=1, num_horizontal_segments=32, num_vertical_segments=15, adjust_kernel=1)
SIZE = (7680, 3840, 3840, 2560)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().split(", ")
    return {"gpu": q[0], "power_limit_w": float(q[1])} if len(q) == 2 else {"gpu": None, "power_limit_w": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200, help="calls per timed window")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--label", default="")
    ap.add_argument("--out", help="append the JSON line to this file")
    args = ap.parse_args()
    import torch
    import transform360_b200 as t360
    from oracle import c_oracle as co
    from transform360_b200.stream import StreamSpec

    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    spec = StreamSpec(*SIZE)
    pitch = lambda w: (w + 255) // 256 * 256  # noqa: E731
    st = torch.cuda.Stream()
    vft = t360.VideoFrameTransform(t360.make_context(**CFG3))
    cases = {}
    for plane, name in ((0, "luma"), (1, "chroma")):
        iw, ih, ow, oh, idx = spec.plane_dims(plane)
        assert vft.generateMapForPlane(iw, ih, ow, oh, idx)
        src = torch.zeros((ih, pitch(iw)), dtype=torch.uint8, device="cuda")
        src[:, :iw] = torch.from_numpy(co.noise_plane(iw, ih, plane=plane, frame=0)).cuda()
        blurred = torch.zeros((ih, pitch(iw)), dtype=torch.uint8, device="cuda")
        out = torch.zeros((oh, pitch(ow)), dtype=torch.uint8, device="cuda")
        cases[f"low_pass_{name}"] = (lambda iw=iw, ih=ih, idx=idx, src=src, dst=blurred: vft.low_pass_async(
            src.data_ptr(), dst.data_ptr(), iw, ih, src.stride(0), dst.stride(0), idx, st.cuda_stream), blurred, iw)
        cases[f"plane_{name}"] = (lambda iw=iw, ih=ih, ow=ow, oh=oh, idx=idx, src=src, dst=out: vft.transform_plane_async(
            src.data_ptr(), dst.data_ptr(), iw, ih, src.stride(0), ow, oh, dst.stride(0), idx, st.cuda_stream), out, ow)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {k: [] for k in cases}
    for fn, _, _ in cases.values():  # warm-up: scratch planes, tensor maps, modules
        for _ in range(20):
            assert fn()
    st.synchronize()
    for _ in range(args.rounds):
        for k, (fn, _, _) in cases.items():
            st.synchronize()
            a.record(st)
            for _ in range(args.calls):
                assert fn()
            b.record(st)
            st.synchronize()
            times[k].append(round(a.elapsed_time(b) * 1e3 / args.calls, 2))
    result = dict(gpu_info(), label=args.label, calls=args.calls, rounds=args.rounds, cases={})
    for k, (_, dst, w) in cases.items():
        sha = hashlib.sha256(dst[:, :w].cpu().numpy().tobytes()).hexdigest()[:16]
        result["cases"][k] = dict(median_us=statistics.median(times[k]), spread_us=[min(times[k]), max(times[k])], rounds_us=times[k], out_sha=sha)
    vft.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "a") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
