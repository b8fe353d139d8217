"""okvis_b200::EstimatorGroup (include/okvis_b200_estimator.hpp): many okvis::Estimator sessions in one context, each
per-frame step of the ThreadedKFVio cycle one batched device call for a list of them.  tests/shim/group_test.cpp drives
eight sessions over 30 frames (staggered joins, one session leaving at frame 12 and a newcomer taking its slot, and
every fourth frame some sessions left out, so lists are scattered and out of slot order)."""
import json
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "shim", "group_test.bin")


def build_driver():
    import __graft_entry__ as g
    g.build()
    assert os.path.exists(BIN)


def run(*args, timeout=900):
    out = subprocess.run([BIN, *args], capture_output=True, text=True, timeout=timeout)
    assert out.returncode == 0, out.stderr + out.stdout
    r = json.loads(out.stdout.strip().splitlines()[-1])
    assert "error" not in r, r
    return r


def test_group_driver_compiles_and_fails_loudly_without_gpu():
    build_driver()
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a GPU is present")
    except ImportError:
        pass
    out = subprocess.run([BIN, "--no-gpu"], capture_output=True, text=True, timeout=60).stdout
    r = json.loads(out.strip().splitlines()[-1])
    assert r["created"] is False and "no CUDA device" in r["error"]


@pytest.fixture(scope="module")
def arms():
    build_driver()
    return run("--arms")


@pytest.mark.gpu
def test_group_equals_one_session_per_call_bit_for_bit(arms):
    """Arm A (batched lists) against arm B (a group of the same size and slots, every call listing one session): every
    session's poses, speed/bias, landmarks, quality, summaries, removed landmarks and frame / IMU-window pattern after
    every frame, bit for bit."""
    r = arms
    assert r["same_slots"] == 1 and r["records"] > 150
    assert r["group_equals_one_by_one"] == 1, r
    assert r["final_frames"] == 8                   # numKeyframes + numImuFrames once the window has filled


@pytest.mark.gpu
def test_group_agrees_with_standalone_estimators(arms):
    """Against a standalone Estimator per session (own one-window context, a larger landmark chunk cap): identical
    bookkeeping, estimates equal to rounding (bit for bit at this scene's 600 landmarks, below the chunk cap)."""
    r = arms
    print("group vs standalone: max |dpose| %.3e, max |dsb| %.3e, max |dlandmark| %.3e, max rel dcost %.3e, "
          "iteration differences %d" % (r["max_dpose"], r["max_dsb"], r["max_dlandmark"], r["max_rel_dcost"],
                                        r["iteration_diffs"]))
    assert r["bookkeeping_equals_standalone"] == 1
    assert r["max_dpose"] < 1e-8 and r["max_dsb"] < 1e-8
    assert r["max_rel_dcost"] < 1e-9


@pytest.mark.gpu
def test_reused_slot_starts_clean(arms):
    """The newcomer takes the slot the leaver freed (with the leaver's last frame still pending there) and gives what it
    gives alone in a fresh group: no prior, IMU cache, landmark slot or pending command of the previous occupant."""
    r = arms
    assert r["newcomer_slot"] == r["leaver_slot"] >= 0
    assert r["newcomer_frames"] > 10
    assert r["reuse_equals_fresh"] == 1


@pytest.fixture(scope="module")
def rules():
    build_driver()
    return run("--rules")


@pytest.mark.gpu
def test_unlisted_session_is_untouched(rules):
    """A session with a pending addStates that a group optimize does not list keeps its lastUploadBytes (nothing was
    committed) and its estimates."""
    assert rules["unlisted_untouched"] == 1 and rules["pending_bytes"] > 0


@pytest.mark.gpu
def test_group_optimize_launches_as_one_session(rules):
    assert rules["launches_all"] == rules["launches_one"] > 0, rules


@pytest.mark.gpu
def test_list_errors_throw_and_change_nothing(rules):
    """A duplicate, a session of another group, a standalone session (optimize, applyMarginalizationStrategy and
    addStates), and a session joining a full group: each throws before anything changes."""
    assert rules["errors_thrown"] == 7, rules["messages"]
    assert rules["full_group_throws"] == 1
    assert rules["errors_change_nothing"] == 1
    assert rules["still_works"] == 1
    for phrase in ("twice", "another group", "standalone"):
        assert phrase in rules["messages"]
