#!/usr/bin/env python
"""Timeline of one frame gather (tuning aid; needs a GPU): runs cfg2 frames device-resident with the library's debug
trace on and prints, per job kind, how long the consumer groups wait for a job's data and how long they compute,
plus the spread of the groups' finishing times.

    python profiles/trace_frame.py [cfg2|cfg3|cfg4] [out.npy]
"""
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import transform360_b200 as t360  # noqa: E402
from bench import CONFIGS  # noqa: E402
from transform360_b200 import synth  # noqa: E402
from transform360_b200.stream import FrameTransformer, StreamSpec  # noqa: E402

KINDS = {0: "class0", 1: "class1", 3: "share-stay", 4: "share", 5: "nop", 7: "seam", 8: "pole-cap", 9: "border"}


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
    cfg = CONFIGS[name]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    ctx = t360.make_context(**dict(cfg["ov"], enable_low_pass_filter=0))
    spec = StreamSpec(cfg["inp"][0], cfg["inp"][1], cfg["out"][0], cfg["out"][1])
    ft = FrameTransformer(ctx, spec)
    pitch = lambda w: (w + 255) // 256 * 256
    ring = 5
    d_in = [[synth.noise_plane_torch(*spec.plane_dims(p)[:2], plane=p, frame=f, device=dev, pitch=pitch(spec.plane_dims(p)[0])) for p in range(3)]
            for f in range(ring)]
    d_out = [torch.zeros((spec.plane_dims(p)[3], pitch(spec.plane_dims(p)[2])), dtype=torch.uint8, device=dev) for p in range(3)]
    calls = [ft.frame_call([(t.data_ptr(), t.stride(0)) for t in fr], [(t.data_ptr(), t.stride(0)) for t in d_out]) for fr in d_in]
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    for i in range(6):
        calls[i % ring](stream.cuda_stream)
    torch.cuda.synchronize()
    ft.vft.debug_trace(True)
    calls[1](stream.cuda_stream)   # one isolated frame
    torch.cuda.synchronize()
    tr = ft.vft.read_trace().astype(np.int64)
    ft.vft.debug_trace(False)
    if len(sys.argv) > 2:
        np.save(sys.argv[2], tr)
    used = tr[..., 2] > 0
    t_start = tr[..., 0][used].min()
    end = np.where(used, tr[..., 2], 0).max(axis=1) - t_start
    begin = np.where(used, tr[..., 0], 1 << 62).min(axis=1) - t_start
    print(f"groups {tr.shape[0]}, jobs traced {int(used.sum())}, frame {end.max() / 1e3:.1f} us; groups finish at "
          f"min {end.min() / 1e3:.1f} / median {np.median(end) / 1e3:.1f} / max {end.max() / 1e3:.1f} us, start at median {np.median(begin) / 1e3:.1f} us")
    wait, comp, kind = (tr[..., 1] - tr[..., 0])[used], (tr[..., 2] - tr[..., 1])[used], tr[..., 3][used]
    print(f"all jobs: waiting {wait.sum() / 1e3:.0f} group-us, computing {comp.sum() / 1e3:.0f} group-us "
          f"({100 * wait.sum() / (wait.sum() + comp.sum()):.0f} % waiting)")
    for k in sorted(set(kind.tolist())):
        m = kind == k
        print(f"  {KINDS.get(k, k):10s} n={int(m.sum()):5d}  wait mean {wait[m].mean():7.0f} ns (p90 {np.percentile(wait[m], 90):6.0f})  "
              f"compute mean {comp[m].mean():7.0f} ns (p10 {np.percentile(comp[m], 10):6.0f} p90 {np.percentile(comp[m], 90):6.0f})")
    # the first job of every group waits for the prologue (weights, first box)
    first = tr[:, 0, :]
    print(f"first job of a group: wait {np.mean(first[:, 1] - first[:, 0]) / 1e3:.2f} us")


if __name__ == "__main__":
    main()
