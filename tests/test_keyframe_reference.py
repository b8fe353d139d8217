"""CPU checks of the keyframe-decision restatement tests/keyframe_reference.py: against OpenCV directly (when cv2 is
installed) and through tests/golden/keyframe_opencv.npz (always): identical hull vertex sequences, bit-identical areas,
identical pointPolygonTest signs, per-camera integers and decisions.  Also: the device's extreme-point pre-filter
changes no hull, and the okb_keyframe_* structs of okvis_b200/abi.py match include/okvis_b200.h."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import keyframe_reference as ref
import keyframe_scene as S
from okvis_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "keyframe_opencv.npz")


def _golden_images():
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_golden_keyframe as mk
    return mk


def _bits(v):
    return np.float64(v).tobytes()


def _check_camera(kp, matched, g):
    """The restatement against one camera's OpenCV results g (dict-like of make_golden_keyframe's fields)."""
    r = ref.camera_overlap(kp, matched)
    for k in ("n_points", "n_matched", "inside", "skipped"):
        assert int(r[k]) == int(g[k]), k
    for k in ("area_all", "area_matched", "overlap", "ratio"):
        assert _bits(r[k]) == _bits(g[k]), (k, r[k], float(g[k]))
    if not r["skipped"]:
        p = np.asarray(kp, np.float32).reshape(-1, 2)
        m = p[np.asarray(matched, bool)]
        assert np.array_equal(p[ref.convex_hull(p)], np.asarray(g["hull_all"])), "hull of all points"
        assert np.array_equal(m[ref.convex_hull(m)], np.asarray(g["hull_matched"])), "hull of the matched points"
        assert r["hull_all"] == len(g["hull_all"]) and r["hull_matched"] == len(g["hull_matched"])
        assert np.array_equal(ref.point_polygon(m[ref.convex_hull(m)], p), np.asarray(g["signs"]))


def test_restatement_vs_golden():
    mk = _golden_images()
    g = np.load(GOLDEN)
    names = [str(x) for x in g["images"]]
    imgs = {name: (kp, lm) for name, kp, lm in mk.images()}
    assert sorted(names) == sorted(imgs)
    for name in names:
        kp, lm = imgs[name]
        fields = {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}
        _check_camera(kp, lm >= 0, fields)
    sess = mk.sessions()
    assert int(g["n_sessions"]) == len(sess)
    for s, v in enumerate(sess):
        need, overlap, ratio = g["session%d/decision" % s]
        assert v["need_keyframe"] == bool(need) and _bits(v["overlap"]) == _bits(overlap) and _bits(v["ratio"]) == _bits(ratio)
    assert {v["need_keyframe"] for v in sess} == {True, False}


def test_golden_covers_the_quirks():
    g = np.load(GOLDEN)
    assert np.isnan(g["all_equal/overlap"]) and np.isnan(g["all_collinear/overlap"])
    assert len(g["all_equal/hull_all"]) == 1 and len(g["all_collinear/hull_all"]) == 2
    assert np.isinf(g["matched_on_own_hull/ratio"]) and int(g["matched_on_own_hull/inside"]) == 0
    assert int(g["none_matched/skipped"]) == 1 and int(g["points_2/skipped"]) == 1 and int(g["points_3/skipped"]) == 0
    s = g["on_edges/signs"]
    assert (s[:10] == 0).all() and (s > 0).any() and (s < 0).any()     # vertices and edges give 0
    assert len(g["circle/hull_all"]) == 64


def _cv2_sets():
    """Point sets for the direct comparison: random, integer grids with duplicates, circles in both orders, exact
    lines, clusters of duplicates."""
    for s in range(240):
        rng = np.random.default_rng(1000 + s)
        n = int(rng.integers(3, 80)) if s % 2 else 400
        kind = s % 6
        if kind == 0:
            p = rng.uniform(0, 752, (n, 2))
        elif kind == 1:
            p = np.round(rng.uniform(0, 20, (n, 2)))
        elif kind == 2:
            t = np.sort(rng.uniform(0, 2 * np.pi, n))
            p = np.stack([320 + 100 * np.cos(t), 240 + 100 * np.sin(t)], 1)[::(1 if s % 4 else -1)]
        elif kind == 3:
            t = np.round(rng.uniform(0, 64, n))
            p = np.stack([10 + t, 3 + 0.5 * t], 1)
        elif kind == 4:
            p = np.repeat(rng.uniform(0, 10, (max(n // 3, 1), 2)), 3, 0)
            rng.shuffle(p)
        else:
            p = np.round(rng.uniform(0, 4, (n, 2)))
        yield rng, p.astype(np.float32)


def test_restatement_vs_cv2():
    cv2 = pytest.importorskip("cv2")
    for rng, p in _cv2_sets():
        h = cv2.convexHull(p, clockwise=False).reshape(-1, 2)
        mine = ref.convex_hull(p)
        assert np.array_equal(p[mine], h)
        assert ref.contour_area(p[mine]) == cv2.contourArea(h)
        q = np.concatenate([p, h, (h + np.roll(h, 1, 0)) / 2, rng.uniform(-10, 760, (20, 2))]).astype(np.float32)
        want = np.array([np.sign(cv2.pointPolygonTest(h, (float(a), float(b)), False)) for a, b in q], np.int8)
        assert np.array_equal(ref.point_polygon(h, q), want)


def test_prefilter_changes_no_hull():
    sets = [p for _, p in _cv2_sets()]
    sets += [kp for kp, _ in S.CASES.values()]
    rng = np.random.default_rng(5)
    sets += [S.random_image(rng, 3000)[0]]
    for p in sets:
        p = np.asarray(p, np.float32).reshape(-1, 2)
        assert np.array_equal(ref.convex_hull(p), ref.convex_hull(p, prefilter=True))
    # the filter does its job on the common shape
    kp, _ = S.random_image(np.random.default_rng(1))
    assert ref.extreme_filter(kp).sum() < len(kp) // 4


def test_std_max_nan_semantics():
    nan = float("nan")
    assert np.isnan(ref.std_max(nan, 0.5))          # a NaN value wins
    assert ref.std_max(0.5, nan) == 0.5             # a NaN running maximum is replaced
    assert ref.keyframe_decision([dict(skipped=0, overlap=nan, ratio=1.0), dict(skipped=0, overlap=0.9, ratio=1.0)])[1] == 0.9
    assert np.isnan(ref.keyframe_decision([dict(skipped=0, overlap=0.9, ratio=1.0), dict(skipped=0, overlap=nan, ratio=1.0)])[1])
    assert ref.keyframe_decision([]) == (True, 0.0, 0.0)


def _header_struct(name):
    txt = open(os.path.join(ROOT, "include", "okvis_b200.h")).read()
    m = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), txt, re.S)
    assert m, name
    body = re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        typ, names = re.match(r"([\w\s\*]+?\*?)\s*((?:\*?\w+\s*,\s*)*\*?\w+)$", decl).groups()
        for nm in names.split(","):
            nm = nm.strip()
            fields.append((nm.lstrip("*"), "*" in typ or nm.startswith("*"), typ.replace("*", "").strip()))
    return fields


_CT = {"int32_t": C.c_int32, "float": C.c_float, "double": C.c_double}


@pytest.mark.parametrize("cname,py", [("okb_keyframe_cam", abi.KeyframeCam), ("okb_keyframe_result", abi.KeyframeResult),
                                      ("okb_keyframe_job", abi.KeyframeJob)])
def test_abi_layout_matches_header(cname, py):
    """Field names and order as the header declares them; offsets and size as a C compiler lays them out (recomputed
    here from the header's types with the natural alignment of x86-64 / aarch64)."""
    fields = _header_struct(cname)
    assert [f for f, _, _ in fields] == [f for f, _ in py._fields_]
    off = 0
    align = 1
    for (nm, is_ptr, typ), (pnm, ptyp) in zip(fields, py._fields_):
        ct = C.c_void_p if is_ptr else _CT[typ]
        a = C.alignment(ct)
        off = (off + a - 1) // a * a
        assert getattr(py, pnm).offset == off, nm
        assert C.sizeof(ptyp) == C.sizeof(ct), nm
        off += C.sizeof(ct)
        align = max(align, a)
    assert C.sizeof(py) == (off + align - 1) // align * align
