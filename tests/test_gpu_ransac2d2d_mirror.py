"""The device 2D-2D RANSAC and pose initialisation through the C++ mirror (include/okvis_b200_frontend.hpp
Frontend::runRansac2d2d, its EstimatorGroup form and RansacHooks::device2d2d in Frontend::dataAssociationAndInitialization):
tests/shim/ransac2d2d_test.cpp runs two stereo sessions and a monocular one that start at rest and then accelerate
sideways, with injected wrong associations (look-alike keypoints), standalone and as one group, and calls
runRansac2d2d on its own to check every outlier's end state and the initialised pose."""
import json
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "shim", "ransac2d2d_test.bin")


def run(*args, timeout=900):
    import __graft_entry__ as g
    g.build()
    out = subprocess.run([BIN, *args], capture_output=True, text=True, timeout=timeout)
    assert out.returncode == 0, out.stderr + out.stdout
    r = json.loads(out.stdout.strip().splitlines()[-1])
    assert "error" not in r, r
    return r


def test_ransac2d2d_driver_compiles_and_fails_loudly_without_gpu():
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a GPU is present")
    except ImportError:
        pass
    assert run("--no-gpu")["threw"] is True


@pytest.mark.gpu
def test_sessions_initialise_once_there_is_parallax():
    r = run("--slide")
    assert r["group_equals_single"] == 1, r
    # uninitialised through the rest frames (the rotation-only model wins), initialised once the rig moves
    for f in r["first_initialized"]:
        assert r["rest"] <= f < r["frames"], r
    # sessions initialised from the start: device2d2d changes nothing
    assert r["initialized_unchanged"] == 1, r


@pytest.mark.gpu
@pytest.mark.parametrize("cams", [1, 2])
def test_outliers_reach_the_end_state_and_the_pose_points_the_right_way(cams):
    r = run("--direct", str(cams))
    assert r["calls"] >= 3 and r["rotation_only_calls"] >= 1 and r["initialized"] == 1, r
    assert r["ret_rot_mismatch"] == 0, r
    # the winner is an unrefined minimal-sample model, as in the reference, chosen as soon as its inlier ratio beats the
    # rotation-only model's: here at a baseline of about 12 cm, where it points within 10-20 degrees of the truth
    # (tests/test_ransac2d2d_reference.py::test_scene_outcomes holds it to 5 degrees at 30 cm)
    assert r["pose_sets"] >= 1 and r["max_translation_angle_deg"] < 30.0, r
    assert r["removed"] > 0 and r["lookalikes_removed"] > 0, r
    assert r["end_state_fails"] == 0 and r["store_fails"] == 0, r
