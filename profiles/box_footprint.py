#!/usr/bin/env python
"""Source-box footprint of the class-0 box jobs of a frame (no GPU needed).

Works from the plan the host builds (T360B200_hostPlanGather / T360B200_hostPlanPoleCaps), decoding the compact records
the way tests/test_gather_plan.py does.  For every class-0 tile and quadrant job, seam job and pole-cap job it takes the
true span of its windows -- bytes from the box's first column to the end of the rightmost window, and rows from the
box's first row to the end of the lowest window -- and prints their distribution, then the box bytes one frame moves
from L2 into shared memory with 208-byte class-0 boxes only and with the widths of kernels.cuh (class0BoxW, "used"),
plus other sets of widths for comparison, and the bank model of the tile jobs' window loads at either pitch.  Share and
class-1 boxes are left as they are; seam and pole-cap jobs keep 208 bytes.

    python profiles/box_footprint.py [cfg2|cfg4 ...]
"""
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import transform360_b200 as t360  # noqa: E402
from tests.golden.cases import FULL, plane_dims  # noqa: E402

KIND_SHIFT, SKIP, PITCH = 24, 0x8000, 208
CLASS0, SHARE_STAY, SHARE, SEAM, CAP = 0, 3, 4, 7, 8
SHARE_W = 192
# box widths that are 4 * odd words (the bank argument for 208 B, kernels.cuh), as sets to compare; "used" is class0BoxW
WIDTH_SETS = {"today": (208,), "2 widths": (112, 208), "3 widths": (80, 144, 208), "used": (80, 112, 144, 208),
              "5 widths": (80, 112, 144, 176, 208)}
USED = WIDTH_SETS["used"]


def box_h(k, share):
    return (80 if share else 72) if k == 8 else (72 if share else 64)


def variant_rows(k, share, rows):
    """the height of the lowest box variant that holds `rows` rows (kernels.cuh boxVariantRows / boxVariantFor)"""
    h = box_h(k, share)
    heights = (h, h - 8, h - 16) if share else (h, h - 16, h - 24)
    return min(v for v in heights if v >= rows)


def plane_jobs(hp):
    """[(kind, span bytes, span rows)] of the class-0 box jobs of one plane, and the share-job box bytes"""
    k = hp.kernel_size
    g, pc = hp.gather_plan(), hp.pole_caps()
    out, share_bytes = [], 0
    if g["jobs"] is None:
        return out, 0
    compact = g["compact"]
    for ox, oy, boxxy, rec in g["jobs"]:
        kind = (int(oy) >> KIND_SHIFT) & 15
        if kind in (SHARE, SHARE_STAY):
            share_bytes += SHARE_W * (box_h(k, True) - 8 * (int(boxxy) & 15))
            continue
        if kind not in (CLASS0, SEAM):
            continue
        quad = (int(ox) & 7) - 1
        n = 8 * 128 if quad < 0 else 4 * 64
        words = compact[int(rec) * 4:int(rec) * 4 + n].astype(np.int64)
        off = words[(words & SKIP) == 0] & 0x7FFF
        name = "seam" if kind == SEAM else ("quad" if quad >= 0 else "tile")
        out.append((name, int((off % PITCH).max()) + k, int((off // PITCH).max()) + k))
    base = 0 if compact is None else compact.size // 4
    for n, oy, boxxy, rec in pc["jobs"]:
        if (int(oy) >> KIND_SHIFT) & 15 != CAP:
            continue
        w = pc["records"][(int(rec) - base) * 4:(int(rec) - base) * 4 + int(n) * 64].reshape(-1, 2)[:, 0].astype(np.int64)
        off = w[(w & SKIP) == 0] & 0x7FFF
        out.append(("cap", int((off % PITCH).max()) + k, int((off // PITCH).max()) + k))
    return out, share_bytes


def window_wavefronts(hp, widths):
    """bank model (profiles/bank_sim.py) of the 32-bit window loads of the class-0 tiles and quadrants of one plane, with
    their window offsets at the box's pitch (gather_plan.h deviceRecords): mean wavefronts per load at 208 B and at the
    narrowest width of `widths` that holds each job"""
    from bank_sim import max_distinct_per_bank
    k, g = hp.kernel_size, hp.gather_plan()
    tot = {"208": 0, "narrow": 0}
    n = 0
    for ox, oy, boxxy, rec in g["jobs"][::97]:
        if (int(oy) >> KIND_SHIFT) & 15 != CLASS0:
            continue
        quad = (int(ox) & 7) - 1
        words = g["compact"][int(rec) * 4:int(rec) * 4 + (8 * 128 if quad < 0 else 4 * 64)].astype(np.int64)
        words = words.reshape(8, 32, 4).transpose(0, 2, 1).reshape(-1, 32) if quad < 0 else words.reshape(4, 32, 2).transpose(0, 2, 1).reshape(-1, 32)
        off = words & 0x7FFF
        live = (words & SKIP) == 0
        span = int((off[live] % PITCH).max()) + k
        pitch = min(w for w in widths if w >= span)
        for label, p in (("208", PITCH), ("narrow", pitch)):
            moved = off - off // PITCH * (PITCH - p)
            for step, ok in zip(moved, live):
                if not ok.any():
                    continue
                for r in range(k):
                    a = ((step[ok] & ~3) + r * p) // 4
                    for extra in range(3 if k == 8 else 2):
                        tot[label] += int(max_distinct_per_bank((a + extra)[None, :], 32)[0])
                        n += label == "208"
    return tot["208"] / max(n, 1), tot["narrow"] / max(n, 1)


def box_bytes(jobs, k, widths, kinds=("tile", "quad")):
    """box bytes of the jobs: for the `kinds` the narrowest width of `widths` that holds the span, for the others 208
    bytes (seam jobs: two boxes), as the kernel loads them"""
    total = 0
    for name, span, rows in jobs:
        h = variant_rows(k, False, rows)
        if name == "seam":
            total += 2 * PITCH * h
        elif name in kinds:
            total += min(w for w in widths if w >= span) * h
        else:
            total += PITCH * h
    return total


def main():
    for name in sys.argv[1:] or ["cfg2", "cfg4"]:
        case = FULL[name]
        ctx = t360.make_context(**case["ov"])
        frame, share = [], 0
        for plane, copies in ((0, 1), (1, 2)):  # yuv420p: the chroma plan serves U and V
            iw, ih, ow, oh, _ = plane_dims(case, plane)
            hp = t360.HostPlan(ctx, iw, ih, ow, oh)
            k = hp.kernel_size
            jobs, sb = plane_jobs(hp)
            frame += jobs * copies
            share += sb * copies
            if plane == 0:
                bank = window_wavefronts(hp, USED)
            hp.close()
        print(f"{name}: kernel size {k}, {len(frame)} class-0 box jobs per frame (Y + U + V)")
        for kind in ("tile", "quad", "cap", "seam"):
            span = np.array([s for n, s, _ in frame if n == kind])
            rows = np.array([r for n, _, r in frame if n == kind])
            if not span.size:
                continue
            q = np.percentile(span, [10, 50, 90, 100]).astype(int)
            hist = np.bincount(np.minimum(span, 208) // 16, minlength=14)[1:14]
            print(f"  {kind:4s} {span.size:5d} jobs  span bytes p10/p50/p90/max {q[0]}/{q[1]}/{q[2]}/{q[3]}  rows p50/max "
                  f"{int(np.median(rows))}/{rows.max()}")
            print(f"       span bytes in 16-byte steps (16 .. 208): {' '.join(str(int(v)) for v in hist)}")
        polar = [j for j in frame if j[0] in ("tile", "quad")]
        used = np.array([min(w for w in USED if w >= s) for n, s, _ in polar])
        print("  tiles and quadrants per width of " + str(USED) + ": " +
              " / ".join(f"{100 * (used == w).mean():.0f} %" for w in USED))
        print(f"  window loads of the luma tiles and quadrants (bank model, wavefronts per 32-bit load): "
              f"{bank[0]:.2f} at 208 B, {bank[1]:.2f} in the narrow boxes")
        today = box_bytes(frame, k, (208,))
        print(f"  share-job boxes {share / 1e6:.2f} MB per frame; class-0 box jobs:")
        for label, widths in WIDTH_SETS.items():
            b = box_bytes(frame, k, widths)
            p0, p1 = box_bytes(polar, k, (208,)), box_bytes(polar, k, widths)
            print(f"    {label:6s} {str(widths):22s} {b / 1e6:6.2f} MB per frame ({100 * (1 - b / today):4.1f} % less; "
                  f"the tiles and quadrants alone {p0 / 1e6:.2f} -> {p1 / 1e6:.2f} MB, {100 * (1 - p1 / p0):4.1f} % less)")


if __name__ == "__main__":
    main()
