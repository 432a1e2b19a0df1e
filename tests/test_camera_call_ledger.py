"""The host behaviour of the 16 rig and camera entry points, pinned exactly: which message each refusal prints, and the
bytes each host twin computes.

  - Refusals.  For every twin (lensMap, lensBlendMaps, lensPhotoMaps, cameraMap, rectilinearMap, cameraMipMaps,
    cameraPhotoMaps, stereoCameraMaps) and every frame call (transformFrame{Lens, LensBlend, LensPhoto, Camera, Rectilinear,
    CameraMip, CameraPhoto, StereoCamera}Async): each single fault of the refusal tests' _bad_* helpers plus the call's own
    argument, size, array and frame faults, and pairs of faults in different arguments (the first and the last fault of
    each argument against each other's), so the ledger says which check wins.  Each case records the return value and
    the exact stdout.  Frame calls get bogus device pointers that are never dereferenced: no CUDA call happens.
  - Twin outputs.  The SHA-256 of every output array of the 8 twins over seeded valid configurations: every camera
    model, with and without a rig, minify None / (0, 0) / (4, +-1), seams 0 and 4 degrees, MONO / LR / TB stereo, planes
    0-2 and lenses 0-1.

tests/golden/camera_call_ledger.json holds what the library gave; `python -m tests.test_camera_call_ledger` rewrites it
(run it only where the library's behaviour is the one to pin)."""
import ctypes as C
import hashlib
import json
import os
import sys
import tempfile
from pathlib import Path

import numpy as np

import transform360_b200 as t360
from tests.test_camera_mip import _bad_minify
from tests.test_camera_models import EQUIDISTANT, PANNINI, PINHOLE, STEREOGRAPHIC
from tests.test_camera_models import _bad_calls as _bad_camera_calls
from tests.test_lens import _bad_rigs, make_rig
from tests.test_lens_blend import _bad_blend_calls
from tests.test_lens_photo import IDENTITY, _bad_photo_calls, rig_photos
from tests.test_rectilinear import _bad_calls as _bad_rect_calls
from tests.test_stereo_camera import EQUIRECT, LR, MONO, TB, _bad_stereo_calls, stereo_rig

GOLDEN = Path(__file__).parent / "golden" / "camera_call_ledger.json"
STATS_PTR, PLANE_PTR = 0x40000, 0x20000


# ---- running a call -------------------------------------------------------------------------------------------------
def _captured(fn):
    """(fn(), what it printed on fd 1): the library prints with printf."""
    libc = C.CDLL(None)
    sys.stdout.flush()
    libc.fflush(None)
    saved = os.dup(1)
    with tempfile.TemporaryFile() as tmp:
        os.dup2(tmp.fileno(), 1)
        try:
            ret = fn()
            libc.fflush(None)
        finally:
            os.dup2(saved, 1)
            os.close(saved)
        tmp.seek(0)
        return ret, tmp.read().decode()


def _ref(s):
    return C.byref(s) if s is not None else None


def _frame(n=1, planes=(PLANE_PTR,), dims=(64, 32, 8, 8), pitch=(64, 8), null=None):
    """The frame arguments (numPlanes .. stream) of a whole-frame call; null: the index of an array passed as NULL."""
    P, I = C.c_void_p * 3, C.c_int * 3
    arr = lambda v: I(*([v] * 3))
    args = [n, P(*(list(planes) * 3)[:3]), P(*(list(planes) * 3)[:3]), arr(dims[0]), arr(dims[1]), arr(pitch[0]), arr(dims[2]),
            arr(dims[3]), arr(pitch[1])]
    if null is not None:
        args[1 + null] = None
    return args + [None]


def _structs(a):
    """The C arguments of case a."""
    return dict(rig=_ref(a["rig"]), ph=_ref(a["photometry"]), o=_ref(t360.T360Orientation(*a["orientation"]) if a["orientation"] else None),
                pose=_ref(t360.T360Pose(*a["pose"]) if a["pose"] else None), cam=_ref(t360.T360Camera(*a["camera"]) if a["camera"] else None),
                minify=_ref(t360.T360Minify(*a["minify"]) if a["minify"] else None))


def _twin_call(L, name, a):
    s = _structs(a)
    ctx = t360.make_context(**{**a["base"], **a["ctx"]}) if a["ctx"] is not None else None
    bufs = [np.zeros((8, 8, 2), np.float32) for _ in range(6)]
    arrays = [b.ctypes.data if present else None for b, present in zip(bufs, a["arrays"])]
    sizes = a["sizes"]
    args = {
        "lensMap": (s["rig"], s["o"], *sizes, *arrays[:1]),
        "lensBlendMaps": (s["rig"], a["seam"], s["o"], *sizes, *arrays[:3]),
        "lensPhotoMaps": (s["rig"], s["ph"], a["seam"], s["o"], a["plane"], *sizes, *arrays[:5]),
        "cameraMap": (s["rig"], s["pose"], s["cam"], *sizes, *arrays[:1]),
        "rectilinearMap": (s["rig"], s["pose"], *sizes, *arrays[:1]),
        "cameraMipMaps": (s["rig"], s["pose"], s["cam"], s["minify"], *sizes, *arrays[:4]),
        "cameraPhotoMaps": (s["rig"], s["ph"], a["seam"], s["pose"], s["cam"], s["minify"], a["lens"], a["plane"], *sizes, *arrays),
        "stereoCameraMaps": (s["rig"], s["ph"], s["pose"], s["cam"], s["minify"], a["lens"], a["plane"], *sizes, *arrays),
    }[name]
    return _captured(lambda: getattr(L, "T360B200_" + name)(_ref(ctx), *args))


def _frame_call(L, name, a, transforms):
    s = _structs(a)
    if a["ctx"] is None:
        h = None
    else:
        key = json.dumps(a["ctx"], sort_keys=True)
        if key not in transforms:
            transforms[key] = t360.VideoFrameTransform(t360.make_context(**{**a["base"], **a["ctx"]}))
        h = transforms[key]._h
    frame = _frame(**a["frame"])
    args = {
        "Lens": (s["rig"], s["o"]),
        "LensBlend": (s["rig"], a["seam"], s["o"]),
        "LensPhoto": (s["rig"], s["ph"], a["seam"], s["o"], STATS_PTR),
        "Camera": (s["rig"], s["pose"], s["cam"]),
        "Rectilinear": (s["rig"], s["pose"]),
        "CameraMip": (s["rig"], s["pose"], s["cam"], s["minify"]),
        "CameraPhoto": (s["rig"], s["ph"], a["seam"], s["pose"], s["cam"], s["minify"], STATS_PTR),
        "StereoCamera": (s["rig"], s["ph"], s["pose"], s["cam"], s["minify"], STATS_PTR),
    }[name]
    return _captured(lambda: getattr(L, f"T360B200_transformFrame{name}Async")(h, *args, *frame))


# ---- the cases ------------------------------------------------------------------------------------------------------
def _same(x, y):
    if isinstance(x, C.Structure) or isinstance(y, C.Structure):
        return x is not None and y is not None and bytes(x) == bytes(y)
    if isinstance(x, tuple) and isinstance(y, tuple):  # (orientations, poses and cameras given as ints or floats)
        return repr(tuple(map(float, x))) == repr(tuple(map(float, y)))
    return repr(x) == repr(y)


# The calls' arguments, each with its valid value; the family picks the call's base context and the helpers' faults
LENS_GOOD = dict(ctx={}, rig=make_rig("pair_190"), orientation=(0.0, 0.0, 0.0))
CAMERA_GOOD = dict(ctx={}, rig=None, pose=(10.0, 5.0, 0.0, 90.0, 60.0), camera=(PINHOLE, 0.0))
PHOTO_GOOD = dict(ctx={}, rig=make_rig("pair_190"), photometry=IDENTITY, seam=0.0, pose=(80.0, 5.0, 0.0, 90.0, 60.0),
                  camera=(EQUIDISTANT, 0.0), minify=(4, 0.0))
STEREO_GOOD = dict(ctx={}, rig=stereo_rig(), photometry=IDENTITY, pose=(0.0, 5.0, 0.0, 180.0, 180.0), camera=(EQUIRECT, 0.0), minify=(4, 0.0))

# family: (base context, valid arguments, twin, frame call, the helpers' faults as (what, {argument: value}))
def _families():
    lens = [(w, dict(rig=r, orientation=o, ctx=ov)) for w, r, o, ov in _bad_rigs()]
    blend = [(w, dict(rig=r, seam=s, orientation=o, ctx=ov)) for w, r, s, o, ov in _bad_blend_calls()]
    photo = [(w, dict(rig=r, photometry=ph, seam=s, orientation=o, ctx=ov)) for w, r, ph, s, o, ov in _bad_photo_calls()]
    rect = [(w, dict(rig=r, pose=p, ctx=ov)) for w, r, p, ov in _bad_rect_calls()]
    camera = [(w, dict(rig=r, pose=p, camera=c, ctx=ov)) for w, r, p, c, ov in _bad_camera_calls()] + rect
    minify = [(w, dict(minify=m)) for w, m in _bad_minify()]
    pair = PHOTO_GOOD["rig"]
    camera_photo = [("NULL rig", dict(rig=None))]
    camera_photo += [(w, dict(rig=r or pair, pose=p, camera=c, ctx=ov)) for w, r, p, c, ov in _bad_camera_calls()]
    camera_photo += [(w, dict(rig=r, photometry=ph, seam=s, ctx=ov)) for w, r, ph, s, o, ov in _bad_photo_calls()
                     if r is not None and o is not None and not w.startswith("orientation") and "output_layout" not in ov]
    camera_photo += [(w, dict(minify=m)) for w, m in _bad_minify() if m is not None]
    stereo = [(w, dict(rig=r, photometry=ph, pose=p, camera=c, minify=m or STEREO_GOOD["minify"], ctx=ov))
              for w, r, ph, p, c, m, ov in _bad_stereo_calls()]
    rect_good = {k: v for k, v in CAMERA_GOOD.items() if k != "camera"}
    return {
        "lens": ({}, LENS_GOOD, "lensMap", "Lens", lens),
        "lens_blend": ({}, {**LENS_GOOD, "seam": 10.0}, "lensBlendMaps", "LensBlend", blend),
        "lens_photo": ({}, {**LENS_GOOD, "photometry": IDENTITY, "seam": 0.0}, "lensPhotoMaps", "LensPhoto", photo),
        "camera": ({}, CAMERA_GOOD, "cameraMap", "Camera", camera),
        "rectilinear": ({}, rect_good, "rectilinearMap", "Rectilinear", rect),
        "camera_mip": ({}, {**CAMERA_GOOD, "minify": (4, 0.0)}, "cameraMipMaps", "CameraMip", camera + minify),
        "camera_photo": ({}, PHOTO_GOOD, "cameraPhotoMaps", "CameraPhoto", camera_photo),
        "stereo_camera": (dict(output_stereo_format=LR), STEREO_GOOD, "stereoCameraMaps", "StereoCamera", stereo),
    }


TWIN_ARRAYS = dict(lensMap=1, lensBlendMaps=3, lensPhotoMaps=5, cameraMap=1, rectilinearMap=1, cameraMipMaps=4, cameraPhotoMaps=6, stereoCameraMaps=6)
TWIN_FAULTS = [("NULL context", dict(ctx=None))] + \
    [(f"sizes {s}", dict(sizes=s)) for s in ((0, 32, 8, 8), (64, -1, 8, 8), (64, 32, 0, 8), (64, 32, 8, 0))]
INDEX_FAULTS = [(f"lens {v}", dict(lens=v)) for v in (-1, 2)] + [(f"plane {v}", dict(plane=v)) for v in (-1, 3)]
FRAME_FAULTS = [("NULL transform", dict(ctx=None))] + \
    [(f"frame {kw}", dict(frame=kw)) for kw in (dict(n=0), dict(n=4), dict(planes=(None,)), dict(dims=(0, 32, 8, 8)), dict(pitch=(63, 8)),
                                               dict(null=0), dict(null=4))]
# a pyramid over a plane side above 131070 (refused by the photometric and stereo frame calls when maxLevel > 0)
BIG_PLANE = ("frame 131071 wide", dict(frame=dict(dims=(131071, 32, 8, 8), pitch=(131072, 8))))


def _cases(good, faults):
    """Each fault alone, then each pair of faults in disjoint arguments among the first and last fault of each argument
    set: [(what, arguments)]."""
    singles = []
    for what, f in faults:
        diff = {k: v for k, v in f.items() if not _same(v, good[k])}
        assert diff, what
        singles.append((what, diff))
    groups = {}
    for what, diff in singles:
        groups.setdefault(tuple(sorted(diff)), []).append((what, diff))
    reps = [(key, c) for key, g in groups.items() for c in ([g[0], g[-1]] if len(g) > 1 else g)]
    cases = [(what, {**good, **diff}) for what, diff in singles]
    for i, (ka, (wa, da)) in enumerate(reps):
        for kb, (wb, db) in reps[i + 1:]:
            if not set(ka) & set(kb):
                cases.append((f"{wa} & {wb}", {**good, **da, **db}))
    return cases


def ledger():
    """({'refusals': {call: [[return, message index]...]}, 'messages': [...], 'case_digest': {call: sha256 of the case
    names}, 'twins': {config: {twin: [sha256 of each array]}}}, {call: [case name]})"""
    L = t360.load()
    n0 = t360.kernel_launch_count()
    messages, index, refusals, digests, case_names = [], {}, {}, {}, {}
    transforms = {}
    common = dict(photometry=None, seam=0.0, orientation=None, pose=None, camera=None, minify=None, lens=0, plane=0, sizes=(64, 32, 8, 8),
                  arrays=(True,) * 6, frame={})
    try:
        for family, (base, good, twin, frame, faults) in _families().items():
            good = {**common, **good, "base": {"enable_low_pass_filter": 0, **base}}
            twin_faults = faults + TWIN_FAULTS + [(f"array {k} NULL", dict(arrays=tuple(i != k for i in range(6)))) for k in range(TWIN_ARRAYS[twin])] + (INDEX_FAULTS if twin in ("cameraPhotoMaps", "stereoCameraMaps") else []) + \
                ([(f"plane {v}", dict(plane=v)) for v in (-1, 3)] if twin == "lensPhotoMaps" else [])
            frame_faults = faults + FRAME_FAULTS + ([BIG_PLANE] if frame in ("CameraPhoto", "StereoCamera") else [])
            for call, fs, run in ((twin, twin_faults, lambda n, a: _twin_call(L, n, a)),
                                  (f"transformFrame{frame}Async", frame_faults, lambda n, a: _frame_call(L, frame, a, transforms))):
                rows, names = [], []
                for what, a in _cases(good, fs):
                    ret, out = run(call, a)
                    assert ret == 0 and out.strip() and "CUDA" not in out, (call, what, ret, out)
                    if out not in index:
                        index[out] = len(messages)
                        messages.append(out)
                    rows.append([int(ret), index[out]])
                    names.append(what)
                refusals[call], case_names[call] = rows, names
                digests[call] = hashlib.sha256("\n".join(names).encode()).hexdigest()
    finally:
        for vft in transforms.values():
            vft.close()
    assert t360.kernel_launch_count() == n0
    return dict(refusals=refusals, messages=messages, case_digest=digests, twins=twin_hashes()), case_names


# ---- twin outputs ---------------------------------------------------------------------------------------------------
def _pose(model, rng):
    ang = (float(rng.uniform(-30, 30)), float(rng.uniform(-20, 20)), float(rng.uniform(-10, 10)))
    fov = {PINHOLE: (100.0, 70.0), EQUIDISTANT: (200.0, 150.0), STEREOGRAPHIC: (170.0, 120.0), PANNINI: (150.0, 90.0),
           EQUIRECT: (180.0, 180.0)}[model]
    return (*ang, *fov), (model, 0.6 if model == PANNINI else 0.0)


# (rig or None, camera model, minify, seamWidth, output_stereo_format, plane, lens); the seed is the row's index
TWIN_CONFIGS = [
    (None, PINHOLE, None, 0.0, MONO, 0, 0), (None, EQUIDISTANT, (0, 0.0), 0.0, MONO, 1, 0), (None, STEREOGRAPHIC, (4, 1.0), 0.0, MONO, 2, 0),
    (None, PANNINI, (4, -1.0), 0.0, MONO, 0, 0), (None, EQUIRECT, (4, 1.0), 0.0, MONO, 1, 0),
    ("pair_190", PINHOLE, None, 0.0, MONO, 0, 0), ("pair_190", PINHOLE, (4, 1.0), 4.0, MONO, 1, 1), ("pair_190", EQUIDISTANT, (0, 0.0), 4.0, MONO, 2, 0),
    ("pair_190", STEREOGRAPHIC, (4, -1.0), 0.0, MONO, 0, 1), ("pair_190", PANNINI, None, 4.0, MONO, 1, 0), ("pair_190", EQUIRECT, (4, 1.0), 4.0, MONO, 2, 1),
    ("single_200", PINHOLE, (4, 1.0), 0.0, MONO, 0, 0), ("single_200", EQUIDISTANT, None, 0.0, MONO, 1, 1), ("tilted", STEREOGRAPHIC, (4, 1.0), 4.0, MONO, 2, 1),
    ("stereo", EQUIRECT, None, 0.0, MONO, 0, 0), ("stereo", EQUIRECT, (4, 1.0), 0.0, LR, 1, 1), ("stereo", PINHOLE, (0, 0.0), 0.0, TB, 2, 0),
    ("stereo", EQUIDISTANT, (4, -1.0), 0.0, LR, 0, 1), ("stereo", PANNINI, None, 0.0, TB, 1, 1), ("stereo", STEREOGRAPHIC, (4, 1.0), 0.0, MONO, 2, 1),
]
LENS_LAYOUTS = [t360.LAYOUT_CUBEMAP_32, t360.LAYOUT_EQUIRECT, t360.LAYOUT_BARREL]
IN_W, IN_H, OUT_W, OUT_H = 512, 256, 40, 24


def twin_hashes():
    def digest(arrays):
        return [hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest() for a in arrays]
    out = {}
    for seed, (rig_name, model, minify, seam, sf, plane, lens) in enumerate(TWIN_CONFIGS):
        rng = np.random.default_rng(1000 + seed)
        pose, cam = _pose(model, rng)
        rig = None if rig_name is None else stereo_rig(seed=seed) if rig_name == "stereo" else make_rig(rig_name, seed)
        ctx = t360.make_context(enable_low_pass_filter=0, output_stereo_format=sf, interpolation_alg=[t360.LINEAR, t360.CUBIC, t360.LANCZOS4][seed % 3])
        name = f"{seed}:{rig_name}/{model}/{minify}/{seam}/{sf}/{plane}/{lens}"
        r = {"camera_map": digest([t360.camera_map(ctx, pose, cam, IN_W, IN_H, OUT_W, OUT_H, rig)])}
        if model == PINHOLE:
            r["rectilinear_map"] = digest([t360.rectilinear_map(ctx, pose, IN_W, IN_H, OUT_W, OUT_H, rig)])
        if minify is not None:
            r["camera_mip_maps"] = digest(t360.camera_mip_maps(ctx, pose, cam, minify, IN_W, IN_H, OUT_W, OUT_H, rig))
        if rig is not None:
            ph = rig_photos(rig)["falloff"]
            if rig_name == "stereo":
                r["stereo_camera_maps"] = digest(t360.stereo_camera_maps(ctx, rig, ph, pose, cam, minify, lens, plane, IN_W, IN_H, OUT_W, OUT_H))
            else:
                r["camera_photo_maps"] = digest(t360.camera_photo_maps(ctx, rig, ph, seam if rig.numLenses == 2 else 0.0, pose, cam, minify, lens,
                                                                       plane, IN_W, IN_H, OUT_W, OUT_H))
                lctx = t360.make_context(enable_low_pass_filter=0, output_layout=LENS_LAYOUTS[seed % 3])
                o = pose[:3]
                r["lens_map"] = digest([t360.lens_map(lctx, rig, o, IN_W, IN_H, OUT_W, OUT_H)])
                if rig.numLenses == 2:
                    r["lens_blend_maps"] = digest(t360.lens_blend_maps(lctx, rig, seam or 4.0, o, IN_W, IN_H, OUT_W, OUT_H))
                r["lens_photo_maps"] = digest(t360.lens_photo_maps(lctx, rig, ph, seam if rig.numLenses == 2 else 0.0, o, plane, IN_W, IN_H,
                                                                   OUT_W, OUT_H))
        out[name] = r
    return out


# ---- the test -------------------------------------------------------------------------------------------------------
def test_the_rig_and_camera_calls_keep_their_ledger():
    """Every refusal prints the message it printed when the ledger was written, and every twin array has the same bytes;
    no CUDA call happens."""
    want = json.loads(GOLDEN.read_text())
    got, names = ledger()
    assert got["case_digest"] == want["case_digest"], "the cases changed: regenerate the ledger where its behaviour is pinned"
    assert got["refusals"].keys() == want["refusals"].keys()
    for call, rows in want["refusals"].items():
        assert len(rows) == len(got["refusals"][call]), call
        for what, w, g in zip(names[call], rows, got["refusals"][call]):
            assert g == w or (g[0] == w[0] and got["messages"][g[1]] == want["messages"][w[1]]), \
                f"{call}, {what}: printed {got['messages'][g[1]]!r} (returned {g[0]}), the ledger has {want['messages'][w[1]]!r} (returned {w[0]})"
    assert got["twins"] == want["twins"]


if __name__ == "__main__":
    GOLDEN.write_text(json.dumps(ledger()[0], separators=(",", ":")) + "\n")
    print(f"wrote {GOLDEN}")
