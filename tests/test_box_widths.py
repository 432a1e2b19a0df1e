"""CPU checks of the narrow class-0 source boxes (csrc/kernels.cuh: class0BoxW) and of the job list and record buffer
the frame kernel reads (csrc/gather_plan.h: deviceJobs, deviceRecords; T360B200_hostPlanDeviceLists).

A class-0 tile or quadrant job loads the narrowest of four box widths (Lanczos4: the whole width only) that holds the
columns its windows span.  The device's job list is the plan's launch list with that width in the top bits of the record
offset; the device's record buffer is the plan's records with the window offsets of a narrow job at its box's pitch.
Decoded here the way gather_frame.cu decodes them and compared with the plan's records (which tests/test_gather_plan.py
and tests/test_pole_cap_plan.py check against the sampling records): every window lies inside the narrow box, the job
names the narrowest width that holds it, every other job and word is unchanged, and the GPU frames of
tests/test_frame_coverage.py reach every (kernel size, width) instantiation of the tile compute.
"""
import functools

import numpy as np
import pytest

import transform360_b200 as t360
from tests.golden.cases import FULL, SMALL
from tests.test_frame_coverage import BOUNDARY, boundary_case, boundary_size, boundary_targets, case_spec, page_layout, staged, sweep_cases
from tests.test_gather_plan import CASES, CLASS0, KIND_SHIFT, SKIP, _plan, box_variant_rows

WIDTHS = (208, 144, 112, 80)  # kernels.cuh class0BoxW
WIDTH_SHIFT, RECORD_MASK = 28, (1 << 28) - 1


def class0_widths(k):
    """kernels.cuh class0Widths: Lanczos4 keeps the whole width"""
    return 1 if k == 8 else len(WIDTHS)


def _device_widths(hp):
    """(launch list, device job list, width index per job)"""
    launch, dev = hp.pole_caps()["launch"], hp.device_lists()["jobs"]
    return launch, dev, (dev[:, 3].astype(np.int64) >> WIDTH_SHIFT) & 15


@pytest.mark.parametrize("group,name,plane", CASES)
def test_device_lists_and_narrow_boxes(group, name, plane):
    case = (SMALL if group == "small" else FULL)[name]
    _, hp, _, _ = _plan(case, plane)
    k = hp.kernel_size
    g, pc, dl = hp.gather_plan(), hp.pole_caps(), hp.device_lists()
    launch, dev, recs = pc["launch"], dl["jobs"], dl["records"]
    plan_recs = np.concatenate([g["compact"] if g["compact"] is not None else np.zeros(0, np.uint32), pc["records"]])
    assert len(dev) == len(launch) and recs.size == plan_recs.size
    if not len(launch):
        return
    widths = (dev[:, 3].astype(np.int64) >> WIDTH_SHIFT) & 15
    assert (dev[:, :3] == launch[:, :3]).all() and (dev[:, 3] & RECORD_MASK == launch[:, 3]).all(), "the launch list, widths aside"
    kinds = (launch[:, 1] >> KIND_SHIFT) & 15
    assert (widths[kinds != CLASS0] == 0).all(), "only class-0 tile and quadrant jobs load a narrow box"
    assert (widths < class0_widths(k)).all()
    changed = np.zeros(recs.size, bool)
    for job, w in zip(launch[kinds == CLASS0], widths[kinds == CLASS0]):
        n = 8 * 128 if (int(job[0]) & 7) == 0 else 4 * 64
        at = slice(int(job[3]) * 4, int(job[3]) * 4 + n)
        planned, got = plan_recs[at].astype(np.int64), recs[at].astype(np.int64)
        live = (planned & SKIP) == 0
        assert ((got & ~0x7FFF) == (planned & ~0x7FFF)).all() and (got[~live] == planned[~live]).all()
        off208, off = planned[live] & 0x7FFF, got[live] & 0x7FFF
        pitch, rows = WIDTHS[w], box_variant_rows(k, CLASS0, int(job[2]) & 15)
        cols = int((off208 % 208).max()) + k  # bytes from the box's first column to the end of the last window
        assert cols <= pitch, "every window lies inside the narrow box"
        assert w == class0_widths(k) - 1 or cols > WIDTHS[w + 1], "the job names the narrowest width that holds its windows"
        assert (off // pitch == off208 // 208).all() and (off % pitch == off208 % 208).all(), "the same window at the box's pitch"
        assert (off // pitch + k <= rows).all()
        changed[at] = True
    assert (recs[~changed] == plan_recs[~changed]).all(), "the records of every other job are the plan's"


def test_narrow_boxes_of_the_headline_plan():
    """cfg2 (profiles/box_footprint.py): most polar tiles and quadrants load a box of 112 bytes or less."""
    counts = np.zeros(len(WIDTHS), np.int64)
    for plane in (0, 1):
        _, hp, _, _ = _plan(FULL["cfg2"], plane)
        launch, _, widths = _device_widths(hp)
        counts += np.bincount(widths[((launch[:, 1] >> KIND_SHIFT) & 15) == CLASS0], minlength=len(WIDTHS))
    assert counts[0] < counts[1:].sum() and counts[2] + counts[3] > counts.sum() / 2, counts


@functools.lru_cache(maxsize=None)
def _plane_widths(ov_items, iw, ih, ow, oh):
    """(kernel size, {widths of the plane's class-0 jobs})"""
    hp = t360.HostPlan(t360.make_context(**dict(ov_items)), iw, ih, ow, oh)
    launch, _, widths = _device_widths(hp)
    out = (hp.kernel_size, frozenset(int(w) for w in widths[((launch[:, 1] >> KIND_SHIFT) & 15) == CLASS0]))
    hp.close()
    return out


def test_gpu_frames_reach_every_box_width():
    """The frames of tests/test_frame_coverage.py's GPU tests run a class-0 job of every width each kernel size uses: every
    instantiation of the tile compute (one per box pitch) is checked against the oracle on the device."""
    cases = list(sweep_cases())
    for k, planes, i in BOUNDARY:
        size = boundary_size(k, planes, boundary_targets(k, planes, 132)[i])
        if size:
            case = boundary_case(k, planes, *size)
            cases.append(dict(case, layout=page_layout(case)))
    seen = set()
    for case in cases:
        for p in range(case["planes"]):
            if staged(case, p):
                iw, ih, ow, oh, _ = case_spec(case).plane_dims(p)
                k, widths = _plane_widths(tuple(sorted(case["ov"].items())), iw, ih, ow, oh)
                seen.update((k, w) for w in widths)
    missing = sorted({(k, w) for k in (2, 4, 8) for w in range(class0_widths(k))} - seen)
    assert not missing, f"no GPU frame runs a class-0 job of (K, width index) {missing}"
