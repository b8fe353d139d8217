"""Detection straight into the feature store through the C++ mirror (include/okvis_b200_frontend.hpp
Frontend::detectAndDescribe(Estimator&, frameId, images) and its EstimatorGroup form): tests/shim/detect_store_test.cpp
slides three stereo sessions over a textured plane for 14 frames -- addStates, detectAndDescribe, the frame's association,
optimize, marginalisation -- against twins fed by the single-image detectAndDescribe + Estimator::setFrameFeatures, and
checks the store form's refusals."""
import json
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "shim", "detect_store_test.bin")


def run(*args, timeout=900):
    import __graft_entry__ as g
    g.build()
    out = subprocess.run([BIN, *args], capture_output=True, text=True, timeout=timeout)
    assert out.returncode == 0, out.stderr + out.stdout
    r = json.loads(out.stdout.strip().splitlines()[-1])
    assert "error" not in r, r
    return r


def test_detect_store_driver_compiles_and_fails_loudly_without_gpu():
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a GPU is present")
    except ImportError:
        pass
    assert run("--no-gpu")["threw"] is True


@pytest.mark.gpu
def test_sliding_sessions_equal_their_twins():
    r = run("--slide")
    # keypoints, landmark ids, keyframe decision values, observations and estimates bit-identical, frame by frame
    assert r["store_vs_twin_first_diff"] == -1, r
    assert r["group_vs_single_first_diff"] == -1, r
    # real images reach the association: tracking and the 2D-2D rounds find matches, landmarks persist across frames
    assert r["keypoints"] > 3 * 14 * 2 * 60, r
    assert r["num3d"] > 500 and r["decisions"] > 20 and r["tracked_landmarks"] > 500, r
    assert r["max_pos_err"] < 0.05, r


@pytest.mark.gpu
def test_store_form_refusals():
    r = run("--refusals")
    assert r["cases"] == 4 and r["thrown"] == 4, r
    assert r["untouched"] == 1 and r["valid_after"] == 1 and r["keypoints"] > 50, r
