#!/usr/bin/env python
"""Offline bank model of the 128-bit weight loads of the staged gather, from the plan's own compact records (no GPU):

    python profiles/weight_sim.py [cfg2]

Decodes the share-job and tile-job records of a BASELINE config exactly like gather_frame.cu does (slot field = byte
offset of a pixel's first weight vector in the shared-memory image), and counts per warp step the wavefronts of one weight
load: a quarter-warp of 8 lanes per pass, a pass costs as many wavefronts as its fullest 16-byte bank group holds distinct
addresses.  With GroupMatcher::balance + PassDealer (csrc/gather_plan.cpp) the model gives 4.42 / 4.49 (share / tile)
wavefronts per load at cfg2.  Also prints the lower bound the chosen table copies allow (max(4, fullest bank group)), i.e.
what is left to a better deal."""
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import transform360_b200 as t360  # noqa: E402
from tests.golden.cases import FULL, plane_dims  # noqa: E402

KIND_SHIFT, SKIP, SLOT_MASK = 24, 0x8000, 0x7FF0
CLASS0, SHARE_STAY, SHARE, SEAM = 0, 3, 4, 7


def wavefronts(field, live):
    """field, live: [n][32] -> (modelled wavefronts, lower bound given the copies) per row"""
    a = np.where(live, field >> 4, -1)
    n = a.shape[0]

    def fullest(x):
        mx = np.zeros(n, np.int64)
        for g in range(8):
            s = np.sort(np.where((x >= 0) & ((x & 7) == g), x, -1), axis=1)
            mx = np.maximum(mx, ((s[:, 1:] != s[:, :-1]) & (s[:, 1:] >= 0)).sum(axis=1) + (s[:, 0] >= 0))
        return mx

    cost = sum(np.where(live[:, q * 8:q * 8 + 8].any(axis=1), np.maximum(fullest(a[:, q * 8:q * 8 + 8]), 1), 0) for q in range(4))
    return cost, np.maximum(fullest(a), 4)


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
    case = FULL[name]
    for plane in (0, 1):
        ctx = t360.make_context(**case["ov"])
        iw, ih, ow, oh, _ = plane_dims(case, plane)
        g = t360.HostPlan(ctx, iw, ih, ow, oh).gather_plan()
        jobs, compact = g["jobs"], g["compact"]
        kinds = (jobs[:, 1] >> KIND_SHIFT) & 15
        share = jobs[np.isin(kinds, (SHARE, SHARE_STAY))]
        if len(share):
            recs = np.stack([compact[j[3] * 4:j[3] * 4 + 8 * 160] for j in share]).reshape(len(share), 8, 160)
            words = recs[:, :, :128].reshape(len(share), 8, 32, 4).astype(np.int64)
            cost = bound = rows = 0
            for j in range(8):
                w = words[..., (j >> 1) & 3]
                f = (((w >> 16) if j & 1 else w) & SLOT_MASK).reshape(-1, 32)
                c, b = wavefronts(f, np.ones_like(f, bool))
                cost, bound, rows = cost + c.sum(), bound + b.sum(), rows + len(c)
            print(f"{name} plane {plane}: share jobs {len(share):5d}: {cost / rows:.3f} wavefronts per weight load (bound of the chosen copies {bound / rows:.3f})")
        tiles = jobs[np.isin(kinds, (CLASS0, SEAM)) & ((jobs[:, 0] & 7) == 0)]
        if len(tiles):
            words = np.stack([compact[j[3] * 4:j[3] * 4 + 1024] for j in tiles]).reshape(-1, 32, 4).astype(np.int64)
            cost = bound = rows = 0
            for j in range(4):
                w = words[..., j]
                live = (w & SKIP) == 0
                keep = live.any(axis=1)
                c, b = wavefronts(((w >> 17) & SLOT_MASK)[keep], live[keep])
                cost, bound, rows = cost + c.sum(), bound + b.sum(), rows + len(c)
            print(f"{name} plane {plane}: tile jobs  {len(tiles):5d}: {cost / rows:.3f} wavefronts per weight load (bound of the chosen copies {bound / rows:.3f})")


if __name__ == "__main__":
    main()
