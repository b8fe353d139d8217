"""Host side of the frontend calls on a landmark-sharded window (no device needed): the feature store's edits are
replicated to every rank, a landmark's initialised flag goes to its owner, and the landmark replica's place and size in
each window's mailbox agree with the stated byte counts."""
import numpy as np
import pytest

from okvis_b200 import capi, sharding


@pytest.mark.parametrize("world", [2, 3, 4])
def test_store_edits_are_replicated_unchanged(world):
    kp = np.arange(30, dtype=np.float64).reshape(10, 3)
    desc = np.arange(480, dtype=np.uint8).reshape(10, 48)
    lm = np.array([-1, 0, 1, 2, 3, 4, 5, 6, 7, 1999], np.int32)
    ob = np.ones(10, np.uint8)
    calls = [("reserve_features", (11, 4, 400, 48)), ("set_features", (3, 1, kp, desc, lm, ob)),
             ("set_feature_landmarks", (3, 1, np.arange(4), np.array([5, 6, 7, 8], np.int32), np.ones(4, np.uint8))),
             ("clear_features", (3,))]
    for op, args in calls:
        for r in range(world):
            got = sharding.route_edit(op, r, world, *args)
            assert len(got) == len(args) and all(x is y for x, y in zip(got, args)), op     # every rank, the same global slots


@pytest.mark.parametrize("world", [2, 3, 4])
def test_initialised_flags_go_to_their_owner(world):
    idx = np.array([0, 5, 6, 7, 1234, 1999], np.uint32)
    flags = np.array([1, 0, 1, 1, 0, 1], np.uint8)
    seen = []
    for r in range(world):
        a = sharding.route_edit("set_landmark_initialized", r, world, idx, flags)
        mine = idx[idx % world == r]
        if not len(mine):
            assert a is None
            continue
        local, f = a
        assert np.array_equal(sharding.global_slots(local, r, world), mine.astype(np.int64))
        assert np.array_equal(f, flags[idx % world == r])
        seen += list(sharding.global_slots(local, r, world))
    assert sorted(seen) == sorted(idx.tolist())


def test_other_ops_are_still_refused():
    with pytest.raises(ValueError):
        sharding.route_edit("reserve", 0, 2, 1, 2, 3)


@pytest.mark.parametrize("world,max_frames", [(2, 20), (3, 8), (4, 20), (8, 32)])
def test_replica_layout_matches_the_stated_bytes(world, max_frames):
    """Replica offset = 4096-byte header + [2][world] solver boxes + [2][world] marginalisation boxes (doubles, DESIGN §7),
    256-byte aligned; replica = two halves of 40 bytes per global landmark slot, each 256-byte aligned; the slot's mailbox
    is the sum."""
    P = 6 * max_frames
    dcp = 4 * ((6 * max_frames + 1 + 3) // 4)
    box = dcp * dcp + max_frames * 32 + 8
    marg = 4 + P * P + P
    off0, rep0, win0 = capi.Context.shard_mailbox_layout(world, max_frames, 0)
    a256 = lambda n: (n + 255) // 256 * 256       # noqa: E731
    assert off0 == a256(4096 + 2 * world * (box + marg) * 8) and rep0 == 0 and win0 == off0
    for L in (1, 2000, 2001, 8000):
        off, rep, win = capi.Context.shard_mailbox_layout(world, max_frames, L)
        assert off == off0 and rep == 2 * a256(40 * L) and win == off + rep
    # cfg-5 (20 keyframes, 8 000 landmarks): 640 000 bytes of replica per window on every rank
    assert capi.Context.shard_mailbox_layout(world, 20, 8000)[1] == 640000


def test_layout_refuses_bad_arguments():
    for args in ((1, 20, 10), (9, 20, 10), (2, 0, 10), (2, 33, 10), (2, 20, -1)):
        with pytest.raises(capi.OkbError):
            capi.Context.shard_mailbox_layout(*args)
