"""What the reference's own object code (oracle/_ref: unmodified reference sources + cv2) returns in the tests that
compare against it, kept as digests in live_reference.json so that those tests also run where oracle/_ref cannot be
built (the reference sources are not part of this repository).

Where oracle/_ref is built, ``recorded(key, compute)`` runs ``compute()`` against the live reference and checks it
against the record (a tripwire, like golden.json: the digests depend on the host's libm); elsewhere it returns the
record.  With T360_RECORD_LIVE_REFERENCE=1 and oracle/_ref built, the tests rewrite the records they reach instead:

    T360_RECORD_LIVE_REFERENCE=1 python -m pytest tests -m "not gpu"
"""
from __future__ import annotations

import atexit
import json
import os
from pathlib import Path

import numpy as np

from oracle import ref_harness as rh

PATH = Path(__file__).with_name("live_reference.json")
_RECORD = os.environ.get("T360_RECORD_LIVE_REFERENCE") == "1"
_data = json.loads(PATH.read_text()) if PATH.exists() else {}


def recorded(key: str, compute, live: bool | None = None):
    """The reference's result for `key`: computed live when `live` (default: oracle/_ref is built), else the record."""
    if live is None:
        live = rh.ref_available()
    if live:
        got = json.loads(json.dumps(compute()))
        if _RECORD:
            _data[key] = got
        else:
            assert _data.get(key) == got, f"the live reference no longer gives its recorded result for {key}"
        return got
    assert key in _data, f"no recorded reference result for {key}"
    return _data[key]


def map_digest(m: np.ndarray) -> str:
    return rh.fnv1a64(np.ascontiguousarray(m).view(np.uint32))


def segs_digest(segs) -> str:
    """(left, top, width, height, kx, ky) segments -> their count, FNV of the rectangles, FNV of every kernel's length and
    tap bits, in order."""
    rects = np.array([[int(v) for v in s[:4]] for s in segs], np.int32).reshape(-1, 4)
    taps = [np.concatenate([[len(s[4]), len(s[5])], np.asarray(s[4], np.float32).view(np.uint32),
                            np.asarray(s[5], np.float32).view(np.uint32)]).astype(np.uint32) for s in segs]
    return f"{len(segs)}:{rh.fnv1a64(rects)}:{rh.fnv1a64(np.concatenate(taps) if taps else np.zeros(0, np.uint32))}"


def plan_digest(ref: "rh.RefTransform", idx: int) -> dict:
    m = ref.map(idx)
    return {"shape": list(m.shape), "map": map_digest(m), "segs": segs_digest(ref.segments(idx))}


def _save():
    PATH.write_text("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v, sort_keys=True)}" for k, v in sorted(_data.items())) + "\n}\n")


if _RECORD:
    atexit.register(_save)
