"""The device 3D-2D RANSAC through the C++ mirror (include/okvis_b200_frontend.hpp Frontend::runRansac3d2d, its
EstimatorGroup form and RansacHooks::device3d2d in Frontend::dataAssociationAndInitialization): tests/shim/ransac_test.cpp
slides three stereo sessions through 24 frames with injected wrong associations (look-alike keypoints), standalone and
as one group, with and without device3d2d, and calls runRansac3d2d on its own to check every outlier's end state."""
import json
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "shim", "ransac_test.bin")


def run(*args, timeout=900):
    import __graft_entry__ as g
    g.build()
    out = subprocess.run([BIN, *args], capture_output=True, text=True, timeout=timeout)
    assert out.returncode == 0, out.stderr + out.stdout
    r = json.loads(out.stdout.strip().splitlines()[-1])
    assert "error" not in r, r
    return r


def test_ransac_driver_compiles_and_fails_loudly_without_gpu():
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a GPU is present")
    except ImportError:
        pass
    assert run("--no-gpu")["threw"] is True


@pytest.mark.gpu
def test_sliding_sessions_reject_injected_associations():
    r = run("--slide")
    assert r["group_equals_single"] == 1, r
    assert r["lookalikes"] > 300 and r["decisions"] > 20, r
    # without the device RANSAC the wrong associations survive; with it they are gone after every frame's association,
    # and none is seen matched by the keyframe decision
    assert r["wrong_after_no_ransac"] > 50, r
    assert r["wrong_after"] <= r["wrong_after_no_ransac"] // 20, r
    assert r["wrong_at_decision"] <= r["wrong_at_decision_no_ransac"] // 10, r
    # true associations are kept, and the stereo trajectories stay within a few centimetres
    assert r["true_obs"] >= 0.95 * r["true_obs_no_ransac"], r
    assert r["max_pos_err"] < 0.05, r


@pytest.mark.gpu
def test_outliers_reach_the_reference_end_state():
    r = run("--direct")
    assert r["calls"] >= 10 and r["ret_fails"] == 0 and r["first_frame_ret"] == 1 and r["decisions"] >= 10, r
    assert r["removed"] > 0 and r["lookalikes_removed"] > 0, r
    assert r["end_state_fails"] == 0 and r["store_fails"] == 0, r
