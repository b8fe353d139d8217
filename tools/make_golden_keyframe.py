"""Writes tests/golden/keyframe_opencv.npz: what OpenCV (cv2) computes for the images of tests/keyframe_scene.py --
cv::convexHull of all points and of the matched points (vertex sequences), cv::contourArea of both, the sign of
cv::pointPolygonTest(matchesHull, p, false) for every point, the per-camera values of Frontend::doWeNeedANewKeyframe and
the decisions of seeded sessions -- so that the tests pin the NumPy restatement against OpenCV without needing cv2.
--check regenerates everything in memory and compares it with the file."""
import argparse
import io
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "keyframe_opencv.npz")

import keyframe_reference as ref  # noqa: E402
import keyframe_scene as S  # noqa: E402


def images():
    out = [(name, kp, lm) for name, (kp, lm) in sorted(S.CASES.items())]
    rng = np.random.default_rng(31)
    out += [("random_%d" % i, *S.random_image(rng)) for i in range(6)]
    out.append(("big", *S.big_image()))
    return out


def sessions():
    return S.make_sessions(41, 6)


def cv_camera(cv2, kp, matched):
    """doWeNeedANewKeyframe's body for one camera, through cv2 (returns the hulls and signs as well)."""
    pts = np.asarray(kp, np.float32).reshape(-1, 2)
    m = pts[matched]
    r = dict(n_points=len(pts), n_matched=len(m), hull_all=np.zeros((0, 2), np.float32), hull_matched=np.zeros((0, 2), np.float32),
             area_all=0.0, area_matched=0.0, signs=np.zeros(0, np.int8), inside=0, skipped=1, overlap=0.0, ratio=0.0)
    if len(pts) < 3 or len(m) < 3:
        return r
    ha = cv2.convexHull(pts, clockwise=False).reshape(-1, 2)
    hm = cv2.convexHull(m, clockwise=False).reshape(-1, 2)
    aa, am = cv2.contourArea(ha), cv2.contourArea(hm)
    signs = np.array([np.sign(cv2.pointPolygonTest(hm, (float(x), float(y)), False)) for x, y in pts], np.int8)
    inside = int((signs > 0).sum()) if len(hm) > 2 else 0
    with np.errstate(divide="ignore", invalid="ignore"):
        overlap = float(np.float64(am) / np.float64(aa))
        ratio = float(np.float64(len(m)) / np.float64(inside))
    r.update(hull_all=ha, hull_matched=hm, area_all=aa, area_matched=am, signs=signs, inside=inside, skipped=0,
             overlap=overlap, ratio=ratio)
    return r


def generate():
    import cv2
    d = {"cv2_version": np.array(cv2.__version__)}
    names = []
    for name, kp, lm in images():
        names.append(name)
        r = cv_camera(cv2, kp, lm >= 0)
        for k, v in r.items():
            d["%s/%s" % (name, k)] = np.asarray(v)
    d["images"] = np.array(names)
    for s, sess in enumerate(sessions()):
        cams = [cv_camera(cv2, kp, lm >= 0) for kp, lm in sess["images"]]
        need, overlap, ratio = ref.keyframe_decision(cams, S.THR_O, S.THR_R)
        d["session%d/n_cams" % s] = np.array(len(cams))
        d["session%d/decision" % s] = np.array([float(need), overlap, ratio])
    d["n_sessions"] = np.array(len(sessions()))
    return d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true", help="regenerate and compare with the committed file")
    args = ap.parse_args()
    d = generate()
    if args.check:
        g = np.load(OUT)
        assert sorted(g.files) == sorted(d), "keys differ"
        for k in d:
            a, b = np.asarray(d[k]), g[k]
            same = a.shape == b.shape and (a.tobytes() == b.tobytes() if a.dtype.kind != "U" else bool(np.all(a == b)))
            assert same, k
        print("keyframe_opencv.npz: %d arrays match (cv2 %s)" % (len(d), d["cv2_version"]))
        return
    buf = io.BytesIO()
    np.savez_compressed(buf, **d)
    with open(OUT, "wb") as f:
        f.write(buf.getvalue())
    print("wrote %s (%d bytes, cv2 %s)" % (OUT, len(buf.getvalue()), d["cv2_version"]))


if __name__ == "__main__":
    main()
