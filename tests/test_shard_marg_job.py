"""Host side of marginalising a landmark-sharded window (no device needed): the rank's job from sharding.shard_marg_job,
the routing of resident edits by slot owner, and the job fingerprint the ranks compare before summing."""
import numpy as np
import pytest

from okvis_b200 import abi, capi, sharding, synthetic

P, SB = abi.BLOCK_POSE, abi.BLOCK_SPEED_BIAS
DENSE = dict(block_kind=[P, SB, P, SB, P], block_idx=[0, 0, 1, 1, 2], block_prev=[-1, 2, 0, -1, 1], block_marginalize=[1, 1, 0, 0, 0],
             imu_terms=[0], sb_priors=[0])


def _lms(job):
    return np.ctypeslib.as_array(job.landmarks, (job.n_landmarks,)).copy() if job.n_landmarks else np.zeros(0, np.uint32)


def _dense(job):
    n = job.n_blocks
    return (np.ctypeslib.as_array(job.block_kind, (n,)).tobytes(), np.ctypeslib.as_array(job.block_idx, (n,)).tobytes(),
            np.ctypeslib.as_array(job.block_prev, (n,)).tobytes(), np.ctypeslib.as_array(job.block_marginalize, (n,)).tobytes(),
            np.ctypeslib.as_array(job.imu_terms, (job.n_imu_terms,)).tobytes(), np.ctypeslib.as_array(job.sb_priors, (job.n_sb_priors,)).tobytes())


@pytest.mark.parametrize("world", [2, 3, 4])
def test_shard_marg_job_partitions_landmarks_and_keeps_the_dense_part(world):
    rng = np.random.default_rng(world)
    lms = np.sort(rng.choice(5000, 700, replace=False)).astype(np.uint32)
    jobs = [sharding.shard_marg_job(r, world, landmarks=lms, **DENSE) for r in range(world)]
    back = np.concatenate([sharding.global_slots(_lms(j), r, world) for r, j in enumerate(jobs)])
    assert len(back) == len(lms) and np.array_equal(np.sort(back), lms.astype(np.int64))      # each landmark exactly once
    for r, j in enumerate(jobs):
        assert np.all(sharding.global_slots(_lms(j), r, world) % world == r)
        assert _dense(j) == _dense(jobs[0])
        assert capi.marg_job_fingerprint(j) == capi.marg_job_fingerprint(jobs[0])


def test_a_rank_may_own_none_of_the_landmarks():
    jobs = [sharding.shard_marg_job(r, 2, landmarks=[4, 8, 10], **DENSE) for r in range(2)]
    assert jobs[0].n_landmarks == 3 and jobs[1].n_landmarks == 0
    assert np.array_equal(_lms(jobs[0]), [2, 4, 5])


def test_local_slots_follow_shard_window():
    """shard_window deals landmark g to rank g % world at local position g // world: the routing rule agrees with it."""
    w = synthetic.make_window(1, 0)
    L = len(w.landmarks)
    for world in (2, 3):
        for r in range(world):
            sw, mine = sharding.shard_window(w, r, world)
            pos, local = sharding.owned_slots(np.arange(L), r, world)
            assert np.array_equal(pos, mine) and np.array_equal(local, np.arange(len(mine)))
            assert np.array_equal(sw.landmarks[local], w.landmarks[mine])


@pytest.mark.parametrize("field", ["block_kind", "block_idx", "block_prev", "block_marginalize", "imu_terms", "sb_priors"])
def test_fingerprint_changes_with_every_replicated_field(field):
    base = capi.marg_job_fingerprint(abi.make_marg_job(landmarks=[1, 2, 3], **DENSE))
    changed = dict(DENSE)
    v = list(changed[field])
    if field == "block_kind":
        v[4] = SB
    elif field == "block_marginalize":
        v[2] = 1
    else:
        v[0] = v[0] + 1
    changed[field] = v
    assert capi.marg_job_fingerprint(abi.make_marg_job(landmarks=[1, 2, 3], **changed)) != base
    # a list that only moves an entry between the IMU and the prior list changes it too
    moved = dict(DENSE, imu_terms=[0, 0], sb_priors=[])
    assert capi.marg_job_fingerprint(abi.make_marg_job(**moved)) != capi.marg_job_fingerprint(abi.make_marg_job(**dict(DENSE, imu_terms=[0], sb_priors=[0])))


def test_fingerprint_ignores_the_landmarks():
    a = capi.marg_job_fingerprint(abi.make_marg_job(landmarks=[1, 2, 3], **DENSE))
    assert a == capi.marg_job_fingerprint(abi.make_marg_job(landmarks=[], **DENSE))


def test_route_edit_sends_landmark_edits_to_their_owner_and_the_rest_everywhere():
    world = 3
    idx = np.array([3, 4, 7, 11, 12], np.uint32)
    xyzw = np.arange(20, dtype=np.float64).reshape(5, 4)
    obs = np.zeros(6, abi.observation_dtype)
    obs["lm_idx"] = [3, 4, 4, 7, 11, 12]
    obs["pose_idx"] = np.arange(6)
    seen_lm, seen_obs = [], []
    for r in range(world):
        s = sharding.route_edit("set_landmarks", r, world, idx, xyzw)
        rm = sharding.route_edit("remove_landmarks", r, world, idx)
        ob = sharding.route_edit("add_observations", r, world, obs)
        if s is None:
            assert rm is None and ob is None
            continue
        g = sharding.global_slots(s[0], r, world)
        assert np.all(g % world == r) and np.array_equal(sharding.global_slots(rm[0], r, world), g)
        assert np.array_equal(s[1], xyzw[np.isin(idx, g)])
        seen_lm.extend(g.tolist())
        assert np.array_equal(sharding.global_slots(ob[0]["lm_idx"], r, world), obs["lm_idx"][obs["lm_idx"] % world == r])
        seen_obs.extend(ob[0]["pose_idx"].tolist())
    assert sorted(seen_lm) == sorted(idx.tolist()) and sorted(seen_obs) == list(range(6))
    pose = np.zeros(7)
    for r in range(world):
        assert sharding.route_edit("remove_frame", r, world, 0, 0) == (0, 0)
        assert sharding.route_edit("add_frame", r, world, pose)[0] is pose


def test_route_edit_sends_observation_removals_to_their_owner():
    world = 2
    keys = np.array([[1, 3, 0], [2, 4, 1], [0, 5, 1], [3, 6, 0]])       # (pose_idx, global lm_idx, cam_idx)
    got = {}
    for r in range(world):
        a = sharding.route_edit("remove_observations", r, world, keys)
        got[r] = a[0]
        assert np.array_equal(sharding.global_slots(a[0][:, 1], r, world), keys[keys[:, 1] % world == r, 1])
        assert np.array_equal(a[0][:, [0, 2]], keys[keys[:, 1] % world == r][:, [0, 2]])
    assert sum(len(v) for v in got.values()) == len(keys)
    assert sharding.route_edit("remove_observations", 1, 4, keys[:1]) is None     # slot 3 lives on rank 3


def test_route_edit_refuses_ops_it_does_not_know():
    with pytest.raises(ValueError):
        sharding.route_edit("eval_reprojection", 0, 2, 1, 2)
    with pytest.raises(ValueError):
        sharding.route_edit("upload", 0, 2, None)
