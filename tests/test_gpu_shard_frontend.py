"""The frontend calls on the feature store of a landmark-sharded window.  Every rank makes the same call with the same
arguments (concurrently, one host thread per rank) and must return, byte for byte, what an unsharded context holding
the whole window returns; afterwards every rank's replicated store equals the unsharded store, and the rank's landmark
shard, mapped back to global slots, equals the unsharded window's landmarks.  All rank contexts live in this process on
device 0 (okb_shard_connect_local)."""
import dataclasses
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import track_scene
from okvis_b200 import abi, capi, images, sharding, synthetic

pytestmark = pytest.mark.gpu

MAX_LM = 2048


class Group:
    """`world` rank contexts connected as one landmark-sharded group with MAX_LM global landmark slots, and an unsharded
    context that receives the same edits and calls."""

    def __init__(self, world, max_frames, max_landmarks=MAX_LM, slots=1):
        self.world = world
        self.ctxs = [capi.Context(0, slots) for _ in range(world)]
        capi.Context.shard_connect_local(self.ctxs, max_frames=max_frames, max_landmarks=max_landmarks)
        self.un = capi.Context(0, slots)
        self.pool = ThreadPoolExecutor(world)
        self.n_local = {}

    def close(self):
        self.pool.shutdown()
        for c in self.ctxs + [self.un]:
            c.close()

    def each(self, fn):
        """fn(rank, ctx) on every rank at once (each rank's call waits for its peers at the landmark exchange)."""
        futs = [self.pool.submit(fn, r, c) for r, c in enumerate(self.ctxs)]
        return [f.result() for f in futs]

    def call(self, name, jobs, **kw):
        got = self.each(lambda r, c: getattr(c, name)(jobs, **kw))
        return got, getattr(self.un, name)(jobs, **kw)

    def edit(self, win, op, *args):
        getattr(self.un, op)(win, *args)
        for r, c in enumerate(self.ctxs):
            a = sharding.route_edit(op, r, self.world, *args)
            if a is not None:
                getattr(c, op)(win, *a)

    def upload(self, win, w, F, n_cams, n_kp, desc_bytes):
        self.un.reserve(win, len(w.poses), len(w.landmarks), len(w.obs), len(w.imu_samples))
        self.un.reserve_features(win, F, n_cams, n_kp, desc_bytes)
        self.un.upload(win, w)
        for r, c in enumerate(self.ctxs):
            sw, _ = sharding.shard_window(w, r, self.world)
            self.n_local[win, r] = len(sw.landmarks)
            c.reserve(win, len(w.poses), len(sw.landmarks), len(sw.obs), len(w.imu_samples))
            c.reserve_features(win, F, n_cams, n_kp, desc_bytes)
            c.upload(win, sw)

    def commit(self, win):
        for c in self.ctxs + [self.un]:
            c.commit(win, 1)

    def check_store(self, win, F, n_cams):
        for f in range(F):
            for cam in range(n_cams):
                want = self.un.debug_features(win, f, cam)
                for c in self.ctxs:
                    got = c.debug_features(win, f, cam)
                    assert got["n"] == want["n"], (f, cam)
                    for k in ("kp", "size", "desc", "lm_slot", "observed"):
                        assert got[k].tobytes() == want[k].tobytes(), (f, cam, k)

    def check_landmarks(self, win, w):
        K, NSB, L = len(w.poses), len(w.speed_bias), len(w.landmarks)
        want = self.un.download(win, with_quality=False, dims=(K, NSB, L))
        for r, c in enumerate(self.ctxs):
            d = c.download(win, with_quality=False, dims=(K, NSB, self.n_local[win, r]))
            assert d["poses"].tobytes() == want["poses"].tobytes()
            assert d["landmarks"].tobytes() == want["landmarks"][r::self.world].tobytes()


def same(a, b, where="result"):
    """Byte equality of two call results (dicts, lists, numpy arrays and scalars)."""
    if isinstance(a, dict):
        assert a.keys() == b.keys(), where
        for k in a:
            same(a[k], b[k], "%s.%s" % (where, k))
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            same(x, y, "%s[%d]" % (where, i))
    elif isinstance(a, np.ndarray) or a is None:
        assert (a is None) == (b is None), where
        if a is not None:
            assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), where
    else:
        assert np.asarray(a).tobytes() == np.asarray(b).tobytes(), (where, a, b)


def call_same(g, name, jobs, **kw):
    got, want = g.call(name, jobs, **kw)
    for r, x in enumerate(got):
        same(x, want, "%s rank %d" % (name, r))
    return want


# ---------------------------------------------------------------- the tracking scene (2 cameras, 2 000 landmarks)
_SCENES = {}


def tscene(i):
    if i not in _SCENES:
        _SCENES[i] = track_scene.make_track_scene(i, n_landmarks=2000, distortion=[abi.DIST_RADTAN, abi.DIST_EQUIDISTANT][i % 2])
    return _SCENES[i]


def load_tscene(g, win, sc):
    w = sc["window"]
    g.upload(win, w, sc["F"], sc["n_cams"], sc["n_kp"], sc["desc_bytes"])
    for (f, c), e in sorted(sc["store"].items()):
        g.edit(win, "set_features", f, c, np.stack([e["kp"][:, 0], e["kp"][:, 1], e["size"]], 1), e["desc"], e["lm"], e["observed"])
        g.commit(win)
    g.edit(win, "set_landmark_initialized", np.arange(len(w.landmarks)), sc["lm_init"])


def tjobs(sc, win):
    B, kf, fb = sc["pose_b"], sc["rounds"]["last_frame"][0][0], sc["feat_b"]
    return dict(
        track=[dict(win=win, pose_b=B, sb_b=sc["sb_b"], feat_slot_b=fb, rounds=sc["rounds"]["keyframes"] + sc["rounds"]["stereo"])],
        match2d2d=[dict(win=win, pose_a=B - 1, feat_slot_a=kf, cam_a=c, pose_b=B, feat_slot_b=fb, cam_b=c, sb_current=sc["sb_b"])
                   for c in range(sc["n_cams"])][:1],
        stereo=[dict(win=win, pose=B, feat_slot=fb, cam_a=0, cam_b=1)],
        ransac=[dict(win=win, feat_slot=fb, n_cams=sc["n_cams"], seed=11)],
        keyframe=[dict(win=win, feat_slot=fb, n_cams=sc["n_cams"])])


@pytest.mark.parametrize("world", [2, 3, 4])
def test_every_call_equals_the_unsharded_window(world):
    sc = tscene(world)
    w = sc["window"]
    g = Group(world, len(w.poses))
    try:
        load_tscene(g, 0, sc)
        J = tjobs(sc, 0)
        t1 = call_same(g, "track_3d2d_batch", J["track"])
        assert len(t1[0]["assoc"]) > 50 and len(t1[0]["uninit"]) > 0
        g.check_store(0, sc["F"], sc["n_cams"])
        # the flags track cleared came back through their owners: a second track sees them cleared on every rank
        t2 = call_same(g, "track_3d2d_batch", J["track"])
        assert len(t2[0]["uninit"]) < len(t1[0]["uninit"])
        g.check_store(0, sc["F"], sc["n_cams"])
        r = call_same(g, "ransac_3d2d_batch", J["ransac"])
        assert r[0]["ret"] == r[0]["n_inliers"] > 10
        m = call_same(g, "match2d2d_batch", J["match2d2d"])
        s = call_same(g, "stereo_init_batch", J["stereo"])
        assert len(m[0]) + len(s[0]) > 0
        call_same(g, "keyframe_overlap_batch", J["keyframe"])
        g.check_store(0, sc["F"], sc["n_cams"])
        g.check_landmarks(0, w)
    finally:
        g.close()


def test_removed_landmarks_are_forgotten_on_every_rank():
    """A removal reaches only the slot's owner; every rank's store forgets the slot's references at the next exchange,
    as the unsharded store does at the removal, also when the slot is taken by a new landmark before the call."""
    sc = tscene(5)
    w = sc["window"]
    g = Group(2, len(w.poses))
    try:
        load_tscene(g, 0, sc)
        J = tjobs(sc, 0)
        A = sc["store"][sc["rounds"]["keyframes"][0][:2]]
        live = np.any(w.landmarks != 0, axis=1)
        used = [int(l) for l in A["lm"] if l >= 0 and live[l] and sc["lm_init"][l]]
        gone = used[10:40]
        g.edit(0, "remove_landmarks", np.array(gone, np.uint32))
        reuse = gone[0]
        g.edit(0, "set_landmarks", np.array([reuse], np.uint32), w.landmarks[used[0]:used[0] + 1])
        g.edit(0, "set_landmark_initialized", np.array([reuse], np.uint32), np.ones(1, np.uint8))
        t = call_same(g, "track_3d2d_batch", J["track"])
        assert not np.isin(t[0]["assoc"]["lm_slot"], gone).any()
        g.check_store(0, sc["F"], sc["n_cams"])
        call_same(g, "ransac_3d2d_batch", J["ransac"])
        call_same(g, "keyframe_overlap_batch", J["keyframe"])
    finally:
        g.close()


# ---------------------------------------------------------------- detection into the store (4 cameras, cfg-5 shaped)
PRM = dict(uniformity_radius=40.0, max_keypoints=400, desc_bytes=48)
R_LIST = [np.eye(3), np.array([[0.9950, 0.0, -0.0998], [0.0198, 0.9801, 0.1977], [0.0978, -0.1987, 0.9752]])]


def frame(seed, cams, shift=0):
    out = []
    for c in range(len(cams)):
        left, right = images.stereo_pair(seed=seed + c // 2)
        out.append(np.roll(left if c % 2 == 0 else right, shift, axis=1))
    return dict(imgs=out, cams=list(cams), R_CWs=[R_LIST[c % 2] for c in range(len(cams))])


@pytest.mark.parametrize("world", [2, 4])
def test_detect_into_the_store_and_the_calls_on_it(world):
    cfg = synthetic.WindowConfig(n_frames=8, n_cams=4, n_landmarks=2000, frame_dt=0.25)
    w = synthetic.make_window(cfg=cfg, seed=0x5F00 + world)
    n_cams, F = 4, 3
    g = Group(world, len(w.poses))
    try:
        g.upload(0, w, F, n_cams, PRM["max_keypoints"], PRM["desc_bytes"])
        for f, shift in ((0, 0), (2, 9)):
            call_same(g, "detect_describe_store_batch", [dict(frame(0x0B200 + 77, w.cameras, shift), win=0, feat_slot=f)], **PRM)
        g.check_store(0, F, n_cams)
        # global slots from every rank's share name keypoints of frame 0 (edits replicated), flags set on the owners
        slots = np.arange(3, 3 + 5 * 60, 5).astype(np.int32)
        for cam in range(n_cams):
            g.edit(0, "set_feature_landmarks", 0, cam, np.arange(0, 120, 2), slots + cam, np.ones(60, np.uint8))
        g.edit(0, "set_landmark_initialized", np.arange(0, 400, dtype=np.uint32), (np.arange(400) % 7 != 0).astype(np.uint8))
        K = len(w.poses)
        call_same(g, "track_3d2d_batch", [dict(win=0, pose_b=K - 1, sb_b=K - 1, feat_slot_b=2, rounds=[(0, c, c) for c in range(n_cams)])])
        call_same(g, "match2d2d_batch", [dict(win=0, pose_a=K - 2, feat_slot_a=0, cam_a=c, pose_b=K - 1, feat_slot_b=2, cam_b=c)
                                         for c in range(1)])
        call_same(g, "stereo_init_batch", [dict(win=0, pose=K - 1, feat_slot=2, cam_a=0, cam_b=1)])
        call_same(g, "ransac_3d2d_batch", [dict(win=0, feat_slot=2, n_cams=n_cams, seed=5)])
        kf = call_same(g, "keyframe_overlap_batch", [dict(win=0, feat_slot=f, n_cams=n_cams) for f in (0,)])
        assert kf[0]["cams"][0]["n_matched"] > 0
        g.check_store(0, F, n_cams)
        g.check_landmarks(0, w)
    finally:
        g.close()


# ---------------------------------------------------------------- refusals
def test_refusals():
    sc = tscene(6)
    w = sc["window"]
    g = Group(2, len(w.poses))
    try:
        load_tscene(g, 0, sc)
        c0, c1 = g.ctxs
        f0, cam0 = sorted(sc["store"])[0]
        # a store edit with a slot beyond the global landmark slots, and an initialised flag sent to a rank unrouted
        with pytest.raises(capi.OkbError) as e:
            c0.set_feature_landmarks(0, f0, cam0, [0], [MAX_LM], [1])
        assert e.value.code == abi.OKB_ERR_INVALID_ARG
        with pytest.raises(capi.OkbError) as e:
            c1.set_landmark_initialized(0, [1999], [1])
        assert e.value.code == abi.OKB_ERR_CAPACITY
        # a rank that skips the call: its peer reports the time-out (status 7) and returns
        J = tjobs(sc, 0)
        with pytest.raises(capi.OkbError) as e:
            c0.track_3d2d_batch(J["track"])
        assert e.value.code == abi.OKB_ERR_SHARD_TIMEOUT and "status 7" in str(e.value)
    finally:
        g.close()
    # a group whose global landmark slots do not cover a shard
    g = Group(2, len(w.poses), max_landmarks=1000)
    try:
        g.upload(0, w, sc["F"], sc["n_cams"], sc["n_kp"], sc["desc_bytes"])
        for cam in range(sc["n_cams"]):
            e = sc["store"][sc["feat_b"], cam]
            g.edit(0, "set_features", sc["feat_b"], cam, np.stack([e["kp"][:, 0], e["kp"][:, 1], e["size"]], 1), e["desc"])
        with pytest.raises(capi.OkbError) as e:
            g.ctxs[0].ransac_3d2d_batch(tjobs(sc, 0)["ransac"])
        assert e.value.code == abi.OKB_ERR_CAPACITY
    finally:
        g.close()


# ---------------------------------------------------------------- a sliding cfg-5 shaped window (20 frames, 4 cameras)
def _tools():
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import bench_shard_frontend
    import shard_slide_worker
    return shard_slide_worker, bench_shard_frontend.frame_features


def agree(got, ref, exact, where="result"):
    """got (any rank) against the unsharded result: byte-equal, or, once the solver has run (the sharded solve sums
    the ranks' Schur terms in another order), equal in every integer and close in every floating-point field."""
    if exact:
        same(got, ref, where)
    elif isinstance(ref, dict):
        for k in ref:
            agree(got[k], ref[k], exact, "%s.%s" % (where, k))
    elif isinstance(ref, (list, tuple)):
        assert len(got) == len(ref), where
        for i, (x, y) in enumerate(zip(got, ref)):
            agree(x, y, exact, "%s[%d]" % (where, i))
    elif isinstance(ref, np.ndarray) and ref.dtype.names:
        assert got.shape == ref.shape, where
        for f in ref.dtype.names:
            agree(got[f], ref[f], exact, "%s.%s" % (where, f))
    elif isinstance(ref, (np.ndarray, float, np.floating)) and np.asarray(ref).dtype.kind == "f":
        assert np.allclose(got, ref, rtol=1e-6, atol=1e-9), where
    else:
        same(got, ref, where)


@pytest.mark.parametrize("world", [2, 4])
def test_sliding_sequence_equals_the_unsharded_window(world):
    """Per frame (tools/bench_shard_frontend.py's feature store on tools/shard_slide_worker.py's window): detect into the store, the 3D-2D rounds, a 2D-2D round, RANSAC 3D-2D and its outliers removed, the
    keyframe decision, stereo initialisation, optimize(6) and marginalisation of the oldest frame, with every edit routed
    by route_edit; the ranks agree byte for byte after every call and with an unsharded context driven alike."""
    import marg_reference as mr
    from test_gpu_shard_marginalization import assert_identical, compare_sliding
    T, frame_features = _tools()
    steps = 3
    full, w0, first_seen = T.slide_problem(2000, extra=steps)
    K, L, C, N, D = len(w0.poses), len(w0.landmarks), len(w0.cameras), 384, 48
    F = K + steps + 1
    det_slot = F - 1
    ctxs = [capi.Context(0, 1) for _ in range(world)]
    uctx = capi.Context(0, 1)
    pool = ThreadPoolExecutor(world)
    try:
        capi.Context.shard_connect_local(ctxs, max_frames=K, max_landmarks=L)
        sh = T.Slide(list(enumerate(ctxs)), world, full, w0, first_seen, features=(F, C, N, D))
        un = T.Slide([(0, uctx)], 1, full, w0, first_seen, features=(F, C, N, D))
        base = np.random.default_rng(7).integers(0, 256, (L, D), dtype=np.uint8)

        def edit(op, *args):
            sh.edit(op, *args)
            un.edit(op, *args)

        def call(name, jobs, exact, **kw):
            got = [f.result() for f in [pool.submit(lambda c=c: getattr(c, name)(jobs, **kw)) for c in ctxs]]
            ref = getattr(uctx, name)(jobs, **kw)
            for x in got[1:]:
                same(x, got[0], name + " ranks")
            agree(got[0], ref, exact, name)
            return ref

        def check_store():
            for f in range(F):
                for cam in range(C):
                    want = uctx.debug_features(0, f, cam)
                    for c in ctxs:
                        got = c.debug_features(0, f, cam)
                        assert got["n"] == want["n"]
                        for k in ("kp", "size", "desc", "lm_slot", "observed"):
                            assert got[k].tobytes() == want[k].tobytes(), (f, cam, k)

        for k in range(K):
            for cam in range(C):
                edit("set_features", k, cam, *frame_features(full, k, cam, base, N, tracked=k < K - 1))
            for c in ctxs + [uctx]:
                c.commit(0, 1)
        edit("set_landmark_initialized", np.arange(L), np.any(w0.landmarks != 0, axis=1).astype(np.uint8))
        for step in range(steps):
            exact = step == 0
            B, sB = K - 1, K - 1 + step
            slot = lambda p: p + step        # noqa: E731  feature slot of window position p (generated frame p + step)
            fr = frame(0x0B200 + 500 + step, w0.cameras)
            call("detect_describe_store_batch", [dict(fr, win=0, feat_slot=det_slot)], True, uniformity_radius=40.0, max_keypoints=N,
                 desc_bytes=D)
            tr = call("track_3d2d_batch", [dict(win=0, pose_b=B, sb_b=B, feat_slot_b=sB,
                                                rounds=[(slot(B - a), cam, cam) for a in (1, 2, 3) for cam in range(C)] + [(sB, 0, 1), (sB, 1, 0)])], exact)
            assert len(tr[0]["assoc"]) > 50
            call("match2d2d_batch", [dict(win=0, pose_a=B - 1, feat_slot_a=slot(B - 1), cam_a=0, pose_b=B, feat_slot_b=sB, cam_b=0,
                                          sb_current=B)], exact)
            rs = call("ransac_3d2d_batch", [dict(win=0, feat_slot=sB, n_cams=C, seed=100 + step)], exact)[0]
            call("keyframe_overlap_batch", [dict(win=0, feat_slot=sB, n_cams=C)], exact)
            call("stereo_init_batch", [dict(win=0, pose=B, feat_slot=sB, cam_a=0, cam_b=1)], exact)
            check_store()
            # the RANSAC outliers, applied as the mirror does: the observation leaves the window (routed to the landmark's
            # owner) and the keypoint its landmark (replicated)
            out = rs["outliers"]
            if len(out):
                keys = np.stack([np.full(len(out), B), out["lm_slot"], out["cam"]], 1).astype(np.int64)
                o = un.w.obs
                have = {(int(p), int(l), int(c)) for p, l, c in zip(o["pose_idx"], o["lm_idx"], o["cam_idx"])}
                keys = keys[[tuple(k) in have for k in keys.tolist()]]
                if len(keys):
                    edit("remove_observations", keys)
                    code = lambda p, l, c: (np.asarray(p, np.int64) << 40) + (np.asarray(l, np.int64) << 4) + np.asarray(c, np.int64)  # noqa: E731
                    drop = np.isin(code(o["pose_idx"], o["lm_idx"], o["cam_idx"]), code(keys[:, 0], keys[:, 1], keys[:, 2]))
                    for s in (sh, un):
                        s.w = dataclasses.replace(s.w, obs=np.ascontiguousarray(o[~drop]))
                for cam in range(C):
                    m = out["cam"] == cam
                    if m.any():
                        edit("set_feature_landmarks", sB, cam, out["kp"][m], -np.ones(int(m.sum()), np.int32), np.zeros(int(m.sum()), np.uint8))
            # the solver and marginalisation, as test_gpu_shard_marginalization checks them
            ss, su = sh.optimize(6), un.optimize(6)[0]
            for s in ss:
                assert s["iterations"] == su["iterations"] and s["termination"] == su["termination"] != 6, (step, s, su)
                assert abs(s["final_cost"] - su["final_cost"]) <= 1e-7 * su["final_cost"]
            parts = sh.parts()
            eg = sharding.merge_shard_results(sh.L, parts)
            eu = sharding.merge_shard_results(un.L, un.parts())
            assert np.abs(eg["poses"] - eu["poses"]).max() < 1e-7
            kw, cand = un.job(eu, select=mr.well_conditioned)
            sh.marginalize(kw)
            un.marginalize(kw)
            gs, u = sh.priors(), un.priors()[0]
            assert_identical(gs)
            assert u["status"][0] == 0
            compare_sliding(gs[0], u)
            sh.advance(cand, eg["poses"][1])
            un.advance(cand, eu["poses"][1])
            # the store follows: the oldest frame's slot is cleared, the arriving frame's keypoints come untracked
            edit("clear_features", step)
            kN = K + step
            for cam in range(C):
                edit("set_features", kN, cam, *frame_features(full, kN, cam, base, N, tracked=False))
            new = np.nonzero(first_seen == kN)[0].astype(np.uint32)
            if len(new):
                edit("set_landmark_initialized", new, np.ones(len(new), np.uint8))
    finally:
        pool.shutdown()
        for c in ctxs + [uctx]:
            c.close()
