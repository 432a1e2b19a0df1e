"""What a context change costs with T360B200_reconfigureAsync on the GPU machine: the host time of the call, the frame time
while the new plan is pending (per-frame kernels) and after the swap (planned frame kernel), the time from the call to the
swap, and the longest enqueue call in a window of back-to-back frames that spans the swap.  Needs a GPU.

    python profiles/reconfigure_async.py [--calls 7] [--frames 50] [--out FILE]

Cases, as in reconfigure_latency.py: cfg2 (7680x3840 -> 3840x2560 cube map, luma and chroma plan) and a FLAT_FIXED 1920x1080
viewport from 7680x3840, each with a change that needs a re-plan (interpolation cubic -> Lanczos4 with a new view).
- call_us: wall time of each reconfigureAsync call, the device idle; the calls alternate B and A, each followed by
  reconfigure_wait(True), so every call starts with nothing pending.
- frame_ms_pending / frame_ms_planned: CUDA-event time of `--frames` frames through the whole-frame entry point right after
  the call (checked to be still pending at the end of the window) and after the wait.
- swap_ms: from the call to reconfigure_wait(False) == 1, polled every millisecond while frames are enqueued (settle interval
  included).
- enqueue_ms_max / _p99: host time of each T360B200_transformFrameAsync call over a window of back-to-back frames (the
  stream drained after each, as a filter does) that starts at the call and ends 20 frames after the swap.
Prints one JSON line (also appended to --out) with the card's name and power limit read in the same run.
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
LANCZOS4 = 4
CASES = {
    "cfg2": (dict(CUBIC), dict(CUBIC, interpolation_alg=LANCZOS4, fixed_yaw=30.0, fixed_pitch=-10.0, fixed_roll=5.0), (7680, 3840, 3840, 2560)),
    "flat_fixed_1920x1080": (dict(CUBIC, output_layout=2, fixed_hfov=120.0, fixed_vfov=70.0),
                             dict(CUBIC, output_layout=2, interpolation_alg=LANCZOS4, fixed_yaw=40.0, fixed_pitch=-15.0, fixed_hfov=90.0,
                                  fixed_vfov=55.0), (7680, 3840, 1920, 1080)),
}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().split(", ")
    return {"gpu": q[0], "power_limit_w": float(q[1])} if len(q) == 2 else {"gpu": None, "power_limit_w": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=7, help="reconfigureAsync calls timed per case")
    ap.add_argument("--frames", type=int, default=50, help="frames per timed window")
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
                for _ in range(3)]
        ins = [(t.data_ptr(), t.stride(0)) for t in d_in]
        ctx_a, ctx_b = t360.make_context(**a), t360.make_context(**b)
        ft = FrameTransformer(ctx_a, spec)
        vft = ft.vft
        call = ft.frame_call(ins, [(t.data_ptr(), t.stride(0)) for t in outs[0]])
        for _ in range(10):
            assert call(st.cuda_stream)
        st.synchronize()

        calls = []  # host time of the call, nothing pending before it
        for k in range(args.calls):
            t0 = time.perf_counter()
            vft.reconfigure_async(ctx_b if k % 2 == 0 else ctx_a)
            calls.append((time.perf_counter() - t0) * 1e6)
            assert call(st.cuda_stream)
            assert vft.reconfigure_wait(True) == 1
            st.synchronize()
        vft.reconfigure_async(ctx_a)
        assert vft.reconfigure_wait(True) == 1

        pending, planned, swaps, still_pending = [], [], [], True
        for _ in range(3):  # A -> B: frames while pending, then after the swap; back to A (waited for, untimed)
            st.synchronize()
            vft.reconfigure_async(ctx_b)
            for _ in range(3):  # (first use of the per-frame path's tables and scratch in this window)
                assert call(st.cuda_stream)
            pending.append(frame_ms(call, args.frames))
            still_pending = still_pending and vft.reconfigure_wait(False) == 0
            assert vft.reconfigure_wait(True) == 1
            planned.append(frame_ms(call, args.frames))
            vft.reconfigure_async(ctx_a)
            assert vft.reconfigure_wait(True) == 1
        for _ in range(3):  # call -> swap, with frames flowing
            st.synchronize()
            t0 = time.perf_counter()
            vft.reconfigure_async(ctx_b)
            while vft.reconfigure_wait(False) == 0:
                assert call(st.cuda_stream)
                st.synchronize()
                time.sleep(0.001)
            swaps.append((time.perf_counter() - t0) * 1e3)
            vft.reconfigure_async(ctx_a)
            assert vft.reconfigure_wait(True) == 1

        st.synchronize()
        enqueue, after = [], 0  # back-to-back frames across the swap
        vft.reconfigure_async(ctx_b)
        while after < 20:
            done = vft.reconfigure_wait(False) == 1
            t0 = time.perf_counter()
            assert call(st.cuda_stream)
            enqueue.append((time.perf_counter() - t0) * 1e3)
            st.synchronize()
            after += done
        frames_in_window = len(enqueue)
        enqueue.sort()

        fresh = FrameTransformer(ctx_b, spec)
        assert fresh.frame_call(ins, [(t.data_ptr(), t.stride(0)) for t in outs[1]])(st.cuda_stream)
        st.synchronize()
        identical = all(torch.equal(x, y) for x, y in zip(outs[0], outs[1]))
        result["cases"][name] = {
            "size": list(dims), "call_us_median": round(statistics.median(calls), 1), "call_us": [round(c, 1) for c in calls],
            "frame_ms_pending": [round(x, 4) for x in pending], "frame_ms_planned": [round(x, 4) for x in planned],
            "window_still_pending": still_pending, "swap_ms": [round(x, 1) for x in swaps],
            "enqueue_ms_max": round(enqueue[-1], 3), "enqueue_ms_p99": round(enqueue[int(0.99 * (len(enqueue) - 1))], 3),
            "enqueue_ms_median": round(statistics.median(enqueue), 3), "frames_in_window": frames_in_window,
            "outputs_identical": identical, "plan_device_bytes": [vft.plan_device_bytes(i) for i in (0, 1)]}
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
