"""k_schur on windows that stress its frame-pair layout: tiles whose frame range is a single frame or all K frames,
L not a multiple of 32, K = 12 (one 512-thread CTA per SM) and K = 20 (frame-pair accumulators in global
memory), and a batch whose windows are split
into different chunk counts.  The solve outcome must equal the CPU oracle's within test_gpu_solver's tolerances,
and two runs must be bit-identical (fixed accumulation order)."""
import dataclasses

import numpy as np
import pytest

from okvis_b200 import synthetic

pytestmark = pytest.mark.gpu


def rot_angle(qa, qb):
    Ra, Rb = synthetic.R_from_quat(qa), synthetic.R_from_quat(qb)
    return float(np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1) / 2, -1, 1)))


def tile_ranges(w):
    """(first, last) observing frame of every 32-landmark tile, in the library's internal landmark order."""
    L = len(w.landmarks)
    vis = np.zeros(L, dtype=np.int64)
    np.bitwise_or.at(vis, w.obs["lm_idx"].astype(np.int64), np.left_shift(1, w.obs["pose_idx"].astype(np.int64)))
    seen = vis != 0
    first = np.where(seen, np.array([int(v & -v).bit_length() - 1 for v in vis]), 32)
    last = np.where(seen, np.array([int(v).bit_length() - 1 for v in vis]), 32)
    order = np.argsort(first * 32 + last, kind="stable")
    out = []
    for t in range(0, L, 32):
        idx = [j for j in order[t:t + 32] if seen[j]]
        if idx:
            out.append((int(first[idx].min()), int(last[idx].max())))
    return out


def single_frame_window():
    """cfg-2 frames and cameras, 300 landmarks; 64 landmarks first seen in both cameras of frame 0 keep only those two
    observations, so the first two tiles span one frame, and the tile that ends the frame-0 group spans all K."""
    cfg = dataclasses.replace(synthetic.CONFIGS[2], n_landmarks=300)
    w = synthetic.make_window(2, 3, cfg=cfg)
    obs = w.obs
    lm, pose = obs["lm_idx"].astype(np.int64), obs["pose_idx"].astype(np.int64)
    first = np.full(len(w.landmarks), 1 << 30)
    np.minimum.at(first, lm, pose)
    n0 = np.bincount(lm[pose == 0], minlength=len(w.landmarks))
    pick = np.flatnonzero((first == 0) & (n0 == 2))[:64]
    assert len(pick) == 64
    keep = ~(np.isin(lm, pick) & (pose != 0))
    w.obs = obs[keep]
    return w


def run(ctx, oracle, windows, max_iterations=10):
    for i, w in enumerate(windows):
        ctx.upload(i, w)
    summaries = ctx.optimize(0, len(windows), max_iterations=max_iterations)
    got = [ctx.download(i) for i in range(len(windows))]
    for sg, g, w in zip(summaries, got, windows):
        ref = oracle.OracleProblem(w)
        so = ref.solve(max_iterations, 2)
        rst = ref.state()
        assert sg["iterations"] == so["iterations"]
        assert sg["num_successful_steps"] == so["num_successful_steps"]
        assert sg["termination"] == so["termination"]
        assert sg["imu_redo_count"] == so["imu_redo_count"]
        assert abs(sg["initial_cost"] - so["initial_cost"]) < 1e-9 * so["initial_cost"]
        assert abs(sg["final_cost"] - so["final_cost"]) < 1e-7 * so["final_cost"]
        assert abs(sg["final_radius"] - so["final_radius"]) < 1e-6 * so["final_radius"]
        dt = np.abs(g["poses"][:, :3] - rst["poses"][:, :3]).max()
        dr = max(rot_angle(a[3:], b[3:]) for a, b in zip(g["poses"], rst["poses"]))
        assert dt < 1e-7 and dr < 1e-7, (dt, dr)
        assert np.abs(g["speed_bias"] - rst["speed_bias"]).max() < 1e-7
        q = rst["quality"]
        good = q > 0.01
        pg = g["landmarks"][good, :3] / g["landmarks"][good, 3:4]
        po = rst["landmarks"][good, :3] / rst["landmarks"][good, 3:4]
        assert np.abs(pg - po).max() < 1e-5
        assert np.abs(g["quality"] - q).max() < 1e-7
    return summaries, got


@pytest.fixture(scope="module")
def ctx(okb):
    c = okb.Context(0, 2)
    yield c
    c.close()


def test_single_frame_and_full_range_tiles(ctx, oracle):
    w = single_frame_window()
    K = len(w.poses)
    ranges = tile_ranges(w)
    assert len(w.landmarks) % 32 != 0
    assert any(a == b for a, b in ranges) and (0, K - 1) in ranges
    run(ctx, oracle, [w])


def test_twelve_frames(ctx, oracle):
    """Accumulators in shared memory with one 512-thread CTA per SM."""
    cfg = dataclasses.replace(synthetic.CONFIGS[2], n_frames=12, n_landmarks=400)
    w = synthetic.make_window(2, 4, cfg=cfg)
    assert len(w.poses) == 12
    run(ctx, oracle, [w])


def test_twenty_frames(ctx, oracle):
    """Accumulators in the chunk's global partial."""
    cfg = dataclasses.replace(synthetic.CONFIGS[5], n_landmarks=500)
    w = synthetic.make_window(5, 0, cfg=cfg)
    assert len(w.poses) == 20
    run(ctx, oracle, [w])


def test_batch_with_different_chunk_counts_is_deterministic(ctx, oracle):
    windows = [synthetic.make_window(1, 2), synthetic.make_window(2, 1)]     # L = 300 and 2000: 4 and 31 chunks
    s1, g1 = run(ctx, oracle, windows)
    for i, w in enumerate(windows):
        ctx.upload(i, w)
    s2 = ctx.optimize(0, 2, max_iterations=10)
    for i in range(2):
        g2 = ctx.download(i)
        assert s1[i]["final_cost"] == s2[i]["final_cost"]
        for k in ("poses", "speed_bias", "landmarks"):
            assert np.array_equal(g1[i][k], g2[k]), k
