"""CPU checks of the pole-cap and border jobs (csrc/gather_plan.cpp: coverPoleCaps) and of the launch list the frame
kernel claims from.

The general entries of the tile list (tests/test_gather_plan.py) are the 32 x 32 tiles whose windows fit no box: the
pole caps.  The kernel runs their pixels as pole-cap jobs -- grouped by SOURCE position, one class-0 box each, per
pixel a window offset, a slot field and an output position -- and, where a window leaves the plane, as border jobs
that read their taps through L1.  Everything the kernel trusts about those records is checked here the way
gather_frame.cu decodes them: every window inside its box and the plane, the slot field addressing the pixel's weights,
every pixel of a general tile produced exactly once; and the launch list holds every staged tile and every pole-cap job
once, in launch order, and no general tile.
"""
import numpy as np
import pytest

from tests.golden.cases import FULL, SMALL
from tests.test_gather_plan import (CASES, CLASS0, CLASS1, GENERAL, KIND_SHIFT, ROW_MASK, SEAM, SHARE, SHARE_STAY, SKIP,
                                    SLOT_MASK, WeightImage, _plan, box_variant_rows, box_w)

CAP, BORDER = 8, 9
RANK = {BORDER: 0, SEAM: 1, CLASS1: 2, CAP: 3, SHARE_STAY: 4, SHARE: 5}  # class 0: 6, quadrants 7 (gather_plan.h)


def _rank(job):
    kind = (int(job[1]) >> KIND_SHIFT) & 15
    return RANK[kind] if kind in RANK else (7 if job[0] & 7 else 6)


def _check_pixel_job(kind, n, boxxy, words, s, k, iw, ih, wimg, produced):
    """One pole-cap job (n warp steps of 32 x {window offset | slot field << 17, outX | outY << 16} in a class-0 box) or
    border job (n x {col0, row0 << 10 | phase, outX | outY << 16, 0}).  Returns its record size in 16-byte units."""
    mh, mw = s.shape[:2]
    if kind == BORDER:
        assert boxxy == 0 and 1 <= n <= 320
        rec = words[:n * 4].view(np.int32).reshape(n, 4).astype(np.int64)
        xs, ys = rec[:, 2] & 0xFFFF, rec[:, 2] >> 16
        assert (xs < mw).all() and (ys < mh).all() and (rec[:, 3] == 0).all()
        want = s[ys, xs]
        assert (rec[:, 0] == want[:, 0]).all() and (rec[:, 1] == want[:, 1]).all()
        col0, row0 = rec[:, 0], rec[:, 1] >> 10
        assert ((col0 < 0) | (row0 < 0) | (col0 + k > iw) | (row0 + k > ih)).all(), "a border job holds windows that leave the plane only"
        np.add.at(produced, (ys, xs), 1)
        return n
    bx, by, variant = boxxy & 0xFFF0, boxxy >> 16, boxxy & 15
    pitch, bh = box_w(CLASS0), box_variant_rows(k, CLASS0, variant)
    lower = box_variant_rows(k, CLASS0, variant + 1) if variant < 2 else 0
    assert variant < 3 and 1 <= n <= 20, "a job's records fit a stage's record buffer"
    rec = words[:n * 64].reshape(n, 32, 2).astype(np.int64)  # [step][lane][word]
    w0, pos = rec[..., 0], rec[..., 1]
    skip = (w0 & SKIP) != 0
    assert (w0[skip] == SKIP).all() and (pos[skip] == 0).all()
    assert not skip[:-1].any() and not skip[-1].all(), "only the last step has empty lanes"
    w0, pos = w0[~skip], pos[~skip]
    assert (w0 & (3 << 15) == 0).all()
    off, field = w0 & 0x7FFF, (w0 >> 17) & SLOT_MASK
    xs, ys = pos & 0xFFFF, pos >> 16
    assert (xs < mw).all() and (ys < mh).all()
    want = s[ys, xs]
    row0, col0 = by + off // pitch, bx + off % pitch
    assert (row0 == want[:, 1] >> 10).all() and (col0 == want[:, 0]).all()
    wimg.check(field, want[:, 1] & 1023)
    assert (off % pitch + k <= pitch).all() and (off // pitch + k <= bh).all(), "every window lies inside the job's box"
    assert (col0 >= 0).all() and (col0 + k <= iw).all() and (row0 >= 0).all() and (row0 + k <= ih).all(), "... and the plane"
    assert int((off // pitch).max()) + k > lower, "the job names the lowest box that holds its windows"
    np.add.at(produced, (ys, xs), 1)
    return n * 16


@pytest.mark.parametrize("group,name,plane", CASES)
def test_pole_cap_jobs_and_launch_list(group, name, plane):
    case = (SMALL if group == "small" else FULL)[name]
    _, hp, iw, ih = _plan(case, plane)
    k = hp.kernel_size
    g, pc = hp.gather_plan(), hp.pole_caps()
    jobs, cap_jobs, launch = g["jobs"], pc["jobs"], pc["launch"]
    if jobs is None:
        assert len(cap_jobs) == 0 and len(launch) == 0
        return
    s = hp.samples.astype(np.int64)
    mh, mw = s.shape[:2]
    kinds = (cap_jobs[:, 1] >> KIND_SHIFT) & 15
    assert ((kinds == CAP) | (kinds == BORDER)).all()
    assert [(kinds == CAP).sum(), (kinds == BORDER).sum()] == [pc["counts"]["cap"], pc["counts"]["border"]]
    # the pixels of the general tiles, and no other, each produced once
    want = np.zeros((mh, mw), np.int32)
    for ox, oy, _, _ in jobs[((jobs[:, 1] >> KIND_SHIFT) & 15) == GENERAL]:
        want[oy & ROW_MASK:(oy & ROW_MASK) + 32, ox:ox + 32] = 1
    produced = np.zeros((mh, mw), np.int32)
    base = 0 if g["compact"] is None else g["compact"].size // 4  # records count on after the tiles' (16-byte units)
    next_offset, wimg = base, WeightImage(k)
    for (n, oy, boxxy, rec_off), kind in zip(cap_jobs, kinds):
        assert oy & ROW_MASK == 0 and (oy >> 28) == 0 and rec_off == next_offset
        next_offset += _check_pixel_job(kind, int(n), int(boxxy), pc["records"][(rec_off - base) * 4:], s, k, iw, ih, wimg, produced)
    assert (next_offset - base) * 4 == pc["records"].size
    assert (produced == want).all(), "every pixel of a general tile belongs to exactly one pole-cap or border job"
    # the launch list: the staged tiles and the pole-cap / border jobs, each once, in launch order
    staged = jobs[((jobs[:, 1] >> KIND_SHIFT) & 15) != GENERAL]
    assert ((launch[:, 1] >> KIND_SHIFT) & 15 != GENERAL).all(), "no general tile is launched"
    ranks = [_rank(j) for j in launch]
    assert ranks == sorted(ranks)
    key = lambda a: sorted(map(tuple, a.tolist()))
    assert key(launch) == key(np.concatenate([staged, cap_jobs]))


def test_pole_cap_counts_of_the_headline_plan():
    """cfg2: the 120 luma / 32 chroma general tiles run as 392 / 116 pole-cap jobs, and the 24 pixels of a frame whose
    window wraps as 8 border jobs per plane (one per tile that has such pixels)."""
    for plane, want in ((0, dict(cap=392, border=8)), (1, dict(cap=116, border=8))):
        _, hp, _, _ = _plan(FULL["cfg2"], plane)
        assert hp.pole_caps()["counts"] == want


@pytest.mark.parametrize("name,plane", [("cfg2", 0), ("cfg2", 1), ("cfg4", 0), ("cfg4", 1)])
def test_headline_launch_lists_have_no_general_tile(name, plane):
    _, hp, _, _ = _plan(FULL[name], plane)
    launch = hp.pole_caps()["launch"]
    kinds = (launch[:, 1] >> KIND_SHIFT) & 15
    assert len(launch) and not (kinds == GENERAL).any() and (kinds == CAP).any()


def test_pole_cap_jobs_on_random_contexts():
    """The same checks over the random contexts of the tile-list sweep."""
    from tests.test_host_plan import _random_context
    rng = np.random.default_rng(500)
    checked = 0
    for _ in range(30):
        ov = _random_context(rng)
        iw, ih = int(rng.integers(200, 700)) * 2, int(rng.integers(100, 300)) * 2
        ow, oh = int(rng.integers(40, 200)) * 2 + int(rng.random() < 0.3), int(rng.integers(30, 150)) * 2 + int(rng.random() < 0.3)
        if rng.random() < 0.5:
            iw = (iw + 15) // 16 * 16
        SMALL["__random_caps"] = dict(ov=ov, inp=(iw, ih), out=(ow, oh))
        try:
            test_pole_cap_jobs_and_launch_list("small", "__random_caps", int(rng.integers(0, 2)))
            checked += 1
        except ValueError:  # the planner refuses what the reference refuses
            pass
        finally:
            SMALL.pop("__random_caps", None)
    assert checked >= 25
