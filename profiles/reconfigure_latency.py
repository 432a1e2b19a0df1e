"""What a view change costs on the GPU machine: the wall time of T360B200_reconfigure, and the frame time of the
transform before and after the call against a fresh transform made with the new context.  Needs a GPU.

    python profiles/reconfigure_latency.py [--calls 7] [--frames 300] [--rounds 3] [--out FILE]

Cases: cfg2 (7680x3840 -> 3840x2560 cube map, luma and chroma plan) with a yaw/pitch/roll change, and a FLAT_FIXED
1920x1080 viewport from 7680x3840 (both plan indices) with a yaw/hfov change.  The reconfigure time is taken with the
device idle (host planning of both indices, upload, swap); the frame times are CUDA-event medians of `--frames` frames
through the whole-frame entry point, alternating the reconfigured and the fresh transform `--rounds` times.  Prints one
JSON line (also appended to --out) with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

CUBIC = dict(interpolation_alg=2, enable_low_pass_filter=0)
CASES = {
    "cfg2": (dict(CUBIC), dict(CUBIC, fixed_yaw=30.0, fixed_pitch=-10.0, fixed_roll=5.0), (7680, 3840, 3840, 2560)),
    "flat_fixed_1920x1080": (dict(CUBIC, output_layout=2, fixed_hfov=120.0, fixed_vfov=70.0),
                             dict(CUBIC, output_layout=2, fixed_yaw=40.0, fixed_pitch=-15.0, fixed_hfov=90.0, fixed_vfov=55.0),
                             (7680, 3840, 1920, 1080)),
}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().split(", ")
    return {"gpu": q[0], "power_limit_w": float(q[1])} if len(q) == 2 else {"gpu": None, "power_limit_w": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=7, help="reconfigure calls per case (alternating, the last one to the new view)")
    ap.add_argument("--frames", type=int, default=300, help="frames per timed window")
    ap.add_argument("--rounds", type=int, default=3, help="alternated windows of the reconfigured and the fresh transform")
    ap.add_argument("--out", help="append the JSON line to this file")
    args = ap.parse_args()
    import torch
    import transform360_b200 as t360
    from transform360_b200.stream import FrameTransformer, StreamSpec

    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    info = gpu_info()
    st = torch.cuda.Stream()
    pitch = lambda w: (w + 255) // 256 * 256  # noqa: E731

    def frame_ms(call, n):
        for _ in range(10):
            assert call(st.cuda_stream)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st)
        for _ in range(n):
            assert call(st.cuda_stream)
        b.record(st)
        b.synchronize()
        return a.elapsed_time(b) / n

    result = dict(info, frames=args.frames, calls=args.calls, cases={})
    for name, (a, b, dims) in CASES.items():
        spec = StreamSpec(*dims)
        g = torch.Generator(device="cuda").manual_seed(1)
        d_in = [torch.randint(0, 256, (spec.plane_dims(p)[1], pitch(spec.plane_dims(p)[0])), dtype=torch.uint8, device="cuda", generator=g)
                for p in range(3)]
        outs = [[torch.zeros((spec.plane_dims(p)[3], pitch(spec.plane_dims(p)[2])), dtype=torch.uint8, device="cuda") for p in range(3)]
                for _ in range(2)]
        ins = [(t.data_ptr(), t.stride(0)) for t in d_in]
        ft = FrameTransformer(t360.make_context(**a), spec)
        call = ft.frame_call(ins, [(t.data_ptr(), t.stride(0)) for t in outs[0]])
        before = frame_ms(call, args.frames)
        walls = []
        for k in range(args.calls):  # ... A -> B -> A -> B: the last call leaves the new view in place
            ctx = t360.make_context(**(b if (args.calls - k) % 2 else a))
            st.synchronize()
            t0 = time.perf_counter()
            ft.vft.reconfigure(ctx)
            walls.append((time.perf_counter() - t0) * 1e3)
        fresh = FrameTransformer(t360.make_context(**b), spec)
        fresh_call = fresh.frame_call(ins, [(t.data_ptr(), t.stride(0)) for t in outs[1]])
        after, new = [], []
        for _ in range(args.rounds):
            after.append(frame_ms(call, args.frames))
            new.append(frame_ms(fresh_call, args.frames))
        st.synchronize()
        identical = all(torch.equal(x, y) for x, y in zip(outs[0], outs[1]))
        result["cases"][name] = {
            "size": list(dims), "reconfigure_ms_median": round(statistics.median(walls), 2), "reconfigure_ms": [round(w, 2) for w in walls],
            "frame_ms_before": round(before, 4), "frame_ms_after": [round(x, 4) for x in after],
            "frame_ms_fresh": [round(x, 4) for x in new], "outputs_identical": identical,
            "plan_device_bytes": [ft.vft.plan_device_bytes(i) for i in (0, 1)]}
        ft.close()
        fresh.close()
        del d_in, outs
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
