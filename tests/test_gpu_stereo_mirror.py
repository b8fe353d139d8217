"""Stereo landmark initialisation through the C++ mirror (include/okvis_b200_frontend.hpp Frontend::matchStereo and its
EstimatorGroup form): tests/shim/stereo_test.cpp slides three sessions over 24 frames (3D-2D tracking, matchStereo,
optimize, applyMarginalizationStrategy(5, 3)) with no landmark taken from the scene's truth, standalone and as one group."""
import json
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "shim", "stereo_test.bin")


def run(*args, timeout=900):
    import __graft_entry__ as g
    g.build()
    out = subprocess.run([BIN, *args], capture_output=True, text=True, timeout=timeout)
    assert out.returncode == 0, out.stderr + out.stdout
    r = json.loads(out.stdout.strip().splitlines()[-1])
    assert "error" not in r, r
    return r


def test_stereo_driver_compiles_and_fails_loudly_without_gpu():
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a GPU is present")
    except ImportError:
        pass
    assert run("--no-gpu")["threw"] is True


@pytest.mark.gpu
def test_sliding_sessions_initialise_and_track_their_landmarks():
    r = run("--slide")
    # every landmark matchStereo made (and tracking extended) sees one true point, never a distractor
    assert r["landmarks"] > 300 and r["mixed"] == 0 and r["group_mixed"] == 0 and r["distractor_obs"] == 0
    # initialised landmarks with three or more observations lie near their point after optimize
    assert r["init_checked"] > 100 and r["mean_rel"] < 0.01 and r["max_rel"] < 0.1
    # tracking holds on the landmarks stereo initialisation made (frame 4 on)
    assert r["frames_tracked"] == (r["frames"] - 1) * r["sessions"] and r["min_matches"] >= 20
    # one call per camera pair for the group gives what the single calls give, ids included, frame by frame
    assert r["group_equals_single"] == 1
