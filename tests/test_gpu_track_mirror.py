"""Device-side 3D-2D tracking through the C++ mirror (include/okvis_b200_estimator.hpp Estimator::setFrameFeatures,
include/okvis_b200_frontend.hpp Frontend::matchToKeyframes3D2D / matchToLastFrame3D2D and their EstimatorGroup forms):
tests/shim/track_test.cpp slides three sessions over 24 frames (tracking, new stereo landmarks, optimize,
applyMarginalizationStrategy(5, 3)), standalone and as one group."""
import json
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "shim", "track_test.bin")


def run(*args, timeout=900):
    import __graft_entry__ as g
    g.build()
    out = subprocess.run([BIN, *args], capture_output=True, text=True, timeout=timeout)
    assert out.returncode == 0, out.stderr + out.stdout
    r = json.loads(out.stdout.strip().splitlines()[-1])
    assert "error" not in r, r
    return r


def test_track_driver_compiles_and_fails_loudly_without_gpu():
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a GPU is present")
    except ImportError:
        pass
    assert run("--no-gpu")["threw"] is True


@pytest.mark.gpu
def test_sliding_sessions_track_their_landmarks():
    r = run("--slide")
    # every association names the landmark the keypoint sees; distractors (40 per image) are never taken
    assert r["wrong"] == 0 and r["group_wrong"] == 0
    # the window keeps tracking while frames leave it (feature slots are freed and reused, landmarks marginalised);
    # min_matches is over the frames after start-up (frame 4 on)
    assert r["frames_tracked"] == (r["frames"] - 1) * r["sessions"] and r["min_matches"] >= 20
    assert r["assoc"] > 2000 and r["assoc"] == r["group_assoc"]
    # one okb_track_3d2d_batch per group call gives what the single calls give, frame by frame
    assert r["group_equals_single"] == 1
