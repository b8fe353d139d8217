"""k_schur's packed column layout: the window's 6K pose columns lie densely in 8-column blocks, so a frame whose columns
straddle two blocks shares them with its neighbours.  Covers the launch shapes the library picks as K grows (256-thread
CTAs, 512-thread CTAs with shared-memory accumulators, accumulators in the global partial), read from the library's own
plan, and single-frame tiles on a straddling frame right after a wide-range tile in the same chunk (stale edge columns,
the mirrored diagonal entries of the straddling frame).  Every solve must equal the CPU oracle's within
test_gpu_solver's tolerances; reruns must be bit-identical."""
import dataclasses

import numpy as np
import pytest

from okvis_b200 import synthetic
from test_gpu_schur import run, tile_ranges

pytestmark = pytest.mark.gpu


def frames_window(K, n_landmarks, seed_idx):
    cfg = dataclasses.replace(synthetic.CONFIGS[2], n_frames=K, n_landmarks=n_landmarks)
    w = synthetic.make_window(2, seed_idx, cfg=cfg)
    assert len(w.poses) == K
    return w


def straddle_window():
    """cfg-2 frames and cameras, 400 landmarks; 64 landmarks first seen in both cameras of frame 1 keep only those two
    observations.  Frame 1 is pose columns 6-11: the last two columns of block 0 and the first four of block 1."""
    cfg = dataclasses.replace(synthetic.CONFIGS[2], n_landmarks=400)
    w = synthetic.make_window(2, 5, cfg=cfg)
    obs = w.obs
    lm, pose = obs["lm_idx"].astype(np.int64), obs["pose_idx"].astype(np.int64)
    first = np.full(len(w.landmarks), 1 << 30)
    np.minimum.at(first, lm, pose)
    n1 = np.bincount(lm[pose == 1], minlength=len(w.landmarks))
    pick = np.flatnonzero((first == 1) & (n1 == 2))[:64]
    assert len(pick) == 64
    keep = ~(np.isin(lm, pick) & (pose != 1))
    w.obs = obs[keep]
    return w


def rerun_identical(ctx, windows, first_run):
    s1, g1 = first_run
    for i, w in enumerate(windows):
        ctx.upload(i, w)
    s2 = ctx.optimize(0, len(windows), max_iterations=10)
    for i in range(len(windows)):
        g2 = ctx.download(i)
        assert s1[i]["final_cost"] == s2[i]["final_cost"]
        for k in ("poses", "speed_bias", "landmarks"):
            assert np.array_equal(g1[i][k], g2[k]), k


@pytest.fixture(scope="module")
def ctx(okb):
    c = okb.Context(0, 2)
    yield c
    c.close()


@pytest.fixture(scope="module")
def ctx_one_chunk(okb):
    """As many slots as the GPU has two SMs for: every window is one chunk, so all its tiles run in order in one CTA."""
    c = okb.Context(0, 264)
    yield c
    c.close()


def test_twelve_and_twenty_frames_accumulate_in_shared_memory(ctx):
    for K, n in ((12, 400), (20, 500)):
        ctx.upload(0, frames_window(K, n, 4))
        assert ctx.debug_schur_plan(0, 1)["acc_smem"], K


def test_wide_ctas_with_shared_memory_accumulators(ctx, oracle):
    w = frames_window(16, 500, 1)
    ctx.upload(0, w)
    plan = ctx.debug_schur_plan(0, 1)
    assert plan["threads"] == 512 and plan["acc_smem"], plan
    ctx.upload(0, frames_window(10, 400, 1))
    assert ctx.debug_schur_plan(0, 1)["threads"] == 256
    run(ctx, oracle, [w])


def test_global_partial_accumulators(ctx, oracle):
    w = frames_window(24, 600, 2)
    ctx.upload(0, w)
    plan = ctx.debug_schur_plan(0, 1)
    assert plan["threads"] == 512 and not plan["acc_smem"], plan
    first = run(ctx, oracle, [w])
    rerun_identical(ctx, [w], first)


def test_single_frame_tiles_on_a_straddling_frame(ctx_one_chunk, oracle):
    w = straddle_window()
    K = len(w.poses)
    ranges = tile_ranges(w)
    at = ranges.index((1, 1))
    fa, fb = ranges[at - 1]
    assert fa == 0 and fb >= 2, ranges          # the tile before covers frames 0 and 2: blocks 0 and 1 in full
    assert (6 * 1) % 8 == 6 and K == 10
    first = run(ctx_one_chunk, oracle, [w])
    rerun_identical(ctx_one_chunk, [w], first)
