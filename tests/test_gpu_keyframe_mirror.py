"""The keyframe decision through the C++ mirror (include/okvis_b200_frontend.hpp Frontend::doWeNeedANewKeyframe and
Frontend::dataAssociationAndInitialization, with their EstimatorGroup forms): tests/shim/keyframe_test.cpp slides three
stereo sessions and one monocular session with keyframes chosen by the decision, standalone and as one group, and
dumps every device decision with the keypoints and matched flags it saw; each dump is checked here against the
restatement tests/keyframe_reference.py.  A RANSAC hook that rejects keypoints through setFrameLandmarkId changes the
frame's matched count."""
import glob
import json
import os
import struct
import subprocess

import pytest

import keyframe_reference as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "shim", "keyframe_test.bin")


def run(*args, timeout=900):
    import __graft_entry__ as g
    g.build()
    out = subprocess.run([BIN, *args], capture_output=True, text=True, timeout=timeout)
    assert out.returncode == 0, out.stderr + out.stdout
    r = json.loads(out.stdout.strip().splitlines()[-1])
    assert "error" not in r, r
    return r


def _d(h):
    return struct.unpack("<d", struct.pack("<Q", int(h, 16)))[0]


def _bits(v):
    return struct.pack("<d", v)


def test_keyframe_driver_compiles_and_fails_loudly_without_gpu():
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a GPU is present")
    except ImportError:
        pass
    assert run("--no-gpu")["threw"] is True


@pytest.mark.gpu
def test_sliding_sessions_choose_their_keyframes(tmp_path):
    r = run("--slide", str(tmp_path))
    assert r["group_equals_single"] == 1, r
    # sparse at rest, dense under motion
    assert r["rest_keyframes"] <= r["sessions"], r
    assert r["motion_keyframes"] >= 2 * r["sessions"], r
    assert r["motion_keyframes"] / (r["motion_frames"] * r["sessions"]) > 2 * r["rest_keyframes"] / ((r["rest_frames"] - 1) * r["sessions"]), r
    files = sorted(glob.glob(os.path.join(str(tmp_path), "*.txt")))
    assert len(files) == r["device_decisions"] and len(files) > 40, r
    decisions = set()
    for path in files:
        lines = open(path).read().split("\n")
        need, overlap, ratio, n_cams = lines[0].split()
        pos = 1
        cams = []
        for _ in range(int(n_cams)):
            v = lines[pos].split()
            pos += 1
            n = int(v[0])
            pts = [lines[pos + k].split() for k in range(n)]
            pos += n
            kp = [(float.fromhex(a), float.fromhex(b)) for a, b, _ in pts]
            matched = [m == "1" for _, _, m in pts]
            want = ref.camera_overlap(kp, matched)
            got = dict(zip(("n_points", "n_matched", "hull_all", "hull_matched", "inside", "skipped"), map(int, v[:6])))
            got.update(zip(("area_all", "area_matched", "overlap", "ratio"), map(_d, v[6:10])))
            for k in got:
                if isinstance(want[k], float):
                    assert _bits(got[k]) == _bits(want[k]), (path, k, got[k], want[k])
                else:
                    assert got[k] == want[k], (path, k, got[k], want[k])
            cams.append(want)
        w_need, w_overlap, w_ratio = ref.keyframe_decision(cams, 0.6, 0.2)
        assert bool(int(need)) == w_need and _bits(_d(overlap)) == _bits(w_overlap) and _bits(_d(ratio)) == _bits(w_ratio), path
        decisions.add(w_need)
    assert decisions == {True, False}


@pytest.mark.gpu
def test_a_rejecting_hook_changes_the_matched_count():
    r = run("--reject")
    assert r["rejected"] == 5 and r["matched"] > 20, r
    assert r["matched_remove_only"] == r["matched"], r          # removeObservation keeps the store slot
    assert r["matched_set_id"] == r["matched"] - 5, r           # setFrameLandmarkId(..., 0) clears it
