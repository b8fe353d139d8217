"""GPU checks of okb_detect_describe_store_batch (Frontend::detectAndDescribe straight into the windows' feature stores):
outputs bit-identical to okb_detect_describe_batch; store entries, read back through okb_debug_features, bit-identical
to a twin window fed by the batch call + okb_window_set_features + commit, and so are the tracking, 2D-2D, stereo and
keyframe calls on them; pending edits honoured in both directions; every refusal before device work, leaving the store
as it was; the over-capacity image; n_jobs = 0 and out_desc = NULL."""
import ctypes as C

import numpy as np
import pytest

from okvis_b200 import abi, capi, images, synthetic

pytestmark = pytest.mark.gpu

PARAMS = {"cfg3": dict(uniformity_radius=15.0, max_keypoints=1000), "shipped": dict(uniformity_radius=40.0, max_keypoints=400)}
R_LIST = [np.eye(3), np.array([[0.9950, 0.0, -0.0998], [0.0198, 0.9801, 0.1977], [0.0978, -0.1987, 0.9752]])]
N_FEAT = 3


def window(n_cams, i):
    return synthetic.make_window(2 if n_cams == 2 else 5, i)


def setup(ctx, win, w, n_keypoints, desc_bytes):
    ctx.reserve(win, len(w.poses), len(w.landmarks), len(w.obs), len(w.imu_samples))
    ctx.reserve_features(win, N_FEAT, len(w.cameras), n_keypoints, desc_bytes)
    ctx.upload(win, w)


def frame_images(seed, n_cams, cams, shift=0):
    """n_cams seeded textured views (the stereo pair's two images, then further seeds), rolled by `shift` columns."""
    out = []
    for c in range(n_cams):
        left, right = images.stereo_pair(seed=seed + c // 2)
        out.append(np.roll(left if c % 2 == 0 else right, shift, axis=1))
    return dict(imgs=out, cams=[cams[c] for c in range(n_cams)], R_CWs=[R_LIST[c % 2] for c in range(n_cams)])


def entries(ctx, win, n_cams):
    return [[ctx.debug_features(win, f, c) for c in range(n_cams)] for f in range(N_FEAT)]


def assert_entry_equal(a, b):
    assert a["n"] == b["n"]
    for k in ("kp", "size", "desc", "lm_slot", "observed"):
        assert a[k].tobytes() == b[k].tobytes(), k


def assert_det_equal(a, b):
    (ka, da), (kb, db) = a, b
    assert ka.tobytes() == kb.tobytes()
    if da is not None and db is not None:
        assert da.tobytes() == db.tobytes()


def feed_twin(ctx, win, feat_slot, frame, prm):
    """The path the store call replaces: okb_detect_describe_batch, okb_window_set_features per image, a commit."""
    got = ctx.detect_describe_batch(frame["imgs"], frame["cams"], frame["R_CWs"], **prm)
    for c, (kp, desc) in enumerate(got):
        ctx.set_features(win, feat_slot, c, kp, desc)
    ctx.commit(win, 1)
    return got


@pytest.mark.parametrize("pname,desc_bytes,n_cams", [("shipped", 48, 2), ("cfg3", 64, 2), ("shipped", 64, 4), ("cfg3", 48, 4)])
def test_store_equals_batch_and_set_features(pname, desc_bytes, n_cams):
    prm = dict(PARAMS[pname], desc_bytes=desc_bytes)
    n_sessions = 3
    ctx = capi.Context(0, 2 * n_sessions)
    ws = [window(n_cams, s) for s in range(n_sessions)]
    for s in range(n_sessions):
        for win in (s, n_sessions + s):           # the store window and its twin
            setup(ctx, win, ws[s], prm["max_keypoints"], desc_bytes)
    # two frames per session: feature slots 0 and 2 (slot 1 stays empty)
    for f, shift in ((0, 0), (2, 9)):
        frames = [frame_images(0x0B200 + 3000 + 10 * s, n_cams, ws[s].cameras, shift) for s in range(n_sessions)]
        got = ctx.detect_describe_store_batch([dict(fr, win=s, feat_slot=f) for s, fr in enumerate(frames)], host_threads=2, **prm)
        for s, fr in enumerate(frames):
            ref = feed_twin(ctx, n_sessions + s, f, fr, prm)
            assert len(got[s]) == n_cams
            for c in range(n_cams):
                assert_det_equal(got[s][c], ref[c])
                assert len(ref[c][0]) > 50
    for s in range(n_sessions):
        a, b = entries(ctx, s, n_cams), entries(ctx, n_sessions + s, n_cams)
        for ea, eb in zip(a, b):
            for x, y in zip(ea, eb):
                assert_entry_equal(x, y)
        assert all(e["n"] == -1 for e in a[1])
        e = a[2][1]
        assert e["n"] > 50 and np.all(e["lm_slot"] == -1) and np.all(e["observed"] == 0)
    # the calls that read the store give the same answers on the two twins, also after the same landmark edits
    for s in range(n_sessions):
        for win in (s, n_sessions + s):
            ctx.set_feature_landmarks(win, 0, 0, np.arange(0, 40, 2), np.arange(20), np.ones(20, np.uint8))
            ctx.set_landmark_initialized(win, np.arange(20), np.ones(20, np.uint8))
    res = {}
    for win0 in (0, n_sessions):
        wins = range(win0, win0 + n_sessions)
        res[win0] = (
            ctx.track_3d2d_batch([dict(win=w, pose_b=2, feat_slot_b=2, rounds=[(0, c, c) for c in range(n_cams)]) for w in wins]),
            ctx.match2d2d_batch([dict(win=w, pose_a=1, feat_slot_a=0, cam_a=1, pose_b=2, feat_slot_b=2, cam_b=1) for w in wins]),
            ctx.stereo_init_batch([dict(win=w, pose=2, feat_slot=2, cam_a=0, cam_b=1) for w in wins]),
            ctx.keyframe_overlap_batch([dict(win=w, feat_slot=f, n_cams=n_cams) for w in wins for f in (0,)]))
    track, m2, st, kf = res[0]
    track_t, m2_t, st_t, kf_t = res[n_sessions]
    for s in range(n_sessions):
        for k in ("assoc", "num_matches", "num_uncertain", "uninit"):
            assert track[s][k].tobytes() == track_t[s][k].tobytes(), k
        assert m2[s].tobytes() == m2_t[s].tobytes()
        assert st[s].tobytes() == st_t[s].tobytes()
        assert kf[s] == kf_t[s]
    assert any(kf[s]["cams"][0]["n_matched"] == 20 for s in range(n_sessions))
    ctx.close()


def test_pending_edits_in_both_directions():
    prm = dict(PARAMS["shipped"], desc_bytes=48)
    ctx = capi.Context(0, 1)
    w = window(2, 0)
    setup(ctx, 0, w, 400, 48)
    old = np.zeros((30, 3))
    old[:, 0], old[:, 1], old[:, 2] = np.arange(30), 5.0, 7.0
    for c in range(2):
        ctx.set_features(0, 1, c, old, np.full((30, 48), 3, np.uint8))
    ctx.commit(0, 1)
    fr = frame_images(77, 2, w.cameras)
    # a clear of the slot queued before the call is committed first: it does not erase the new features
    ctx.clear_features(0, 1)
    got = ctx.detect_describe_store_batch([dict(fr, win=0, feat_slot=1)], **prm)[0]
    for c in range(2):
        e = ctx.debug_features(0, 1, c)
        assert e["n"] == len(got[c][0]) > 50
        assert e["kp"].tobytes() == np.stack([got[c][0]["x"], got[c][0]["y"]], 1).astype(np.float64).tobytes()
        assert e["desc"].tobytes() == got[c][1].tobytes()
    # the host's counts follow: an edit of the last new keypoint is accepted, one past it refused
    n0 = len(got[0][0])
    ctx.set_feature_landmarks(0, 1, 0, [n0 - 1], [3], [1])
    with pytest.raises(capi.OkbError):
        ctx.set_feature_landmarks(0, 1, 0, [n0], [3], [1])
    ctx.commit(0, 1)
    e = ctx.debug_features(0, 1, 0)
    assert e["lm_slot"][n0 - 1] == 3 and e["observed"][n0 - 1] == 1 and np.all(e["lm_slot"][:n0 - 1] == -1)
    # one queued after it does
    ctx.clear_features(0, 1)
    ctx.commit(0, 1)
    assert ctx.debug_features(0, 1, 0)["n"] == -1 and ctx.debug_features(0, 1, 1)["n"] == -1
    # other cameras of the slot are left as they are
    ctx.set_features(0, 2, 1, old, np.full((30, 48), 3, np.uint8))
    ctx.commit(0, 1)
    before = ctx.debug_features(0, 2, 1)
    ctx.detect_describe_store_batch([dict(imgs=fr["imgs"][:1], cams=fr["cams"][:1], R_CWs=fr["R_CWs"][:1], win=0, feat_slot=2)], **prm)
    assert ctx.debug_features(0, 2, 0)["n"] > 50
    assert_entry_equal(ctx.debug_features(0, 2, 1), before)
    ctx.close()


def _raw_job(fr, win, feat_slot, n_cams=None, out=True):
    """An okb_detect_store_job over numpy arrays (kept on the returned tuple)."""
    n = len(fr["imgs"]) if n_cams is None else n_cams
    descs, keep = capi.Context._image_descs(fr["imgs"], fr["cams"], fr["R_CWs"])
    kp = np.zeros((max(len(fr["imgs"]), 1), 1000), abi.keypoint_dtype)
    cnt = np.zeros(max(len(fr["imgs"]), 1), np.int32)
    j = abi.DetectStoreJob()
    j.win, j.feat_slot, j.n_cams = win, feat_slot, n
    j.images = C.cast(descs, C.POINTER(abi.ImageDesc))
    j.out_kp = kp.ctypes.data if out else None
    j.n_out = cnt.ctypes.data_as(C.POINTER(C.c_int32)) if out else None
    return j, (descs, keep, kp, cnt)


def test_refusals_leave_the_store_untouched():
    lib = capi.lib()
    ctx = capi.Context(0, 3)
    w = window(2, 0)
    setup(ctx, 0, w, 400, 48)
    setup(ctx, 1, w, 400, 48)
    ctx.upload(2, w)                              # uploaded, no store
    old = np.zeros((30, 3))
    old[:, 0], old[:, 1], old[:, 2] = np.arange(30), 5.0, 7.0
    for win in (0, 1):
        for f in range(N_FEAT):
            for c in range(2):
                ctx.set_features(win, f, c, old, np.full((30, 48), f + 1, np.uint8))
    ctx.commit(0, 2)
    before = [entries(ctx, win, 2) for win in (0, 1)]
    fr = frame_images(5, 2, w.cameras)
    prm = abi.DetectParams()
    prm.uniformity_radius, prm.absolute_threshold, prm.max_keypoints, prm.desc_bytes, prm.rotation_invariance = 40.0, 800.0, 400, 48, 1

    def call(jobs, p=prm, max_out=400):
        arr = (abi.DetectStoreJob * max(len(jobs), 1))(*[j for j, _ in jobs])
        return lib.okb_detect_describe_store_batch(ctx._h, len(jobs), arr, C.byref(p) if p is not None else None, max_out, 0)

    good = _raw_job(fr, 0, 1)
    bad_img = dict(fr, imgs=[fr["imgs"][0], fr["imgs"][1][:, :32]])
    p64 = abi.DetectParams()
    C.pointer(p64)[0] = prm
    p64.desc_bytes = 64
    p1000 = abi.DetectParams()
    C.pointer(p1000)[0] = prm
    p1000.max_keypoints = 1000
    cases = [([good, _raw_job(fr, 2, 1)], prm, 400, "no feature store"),
             ([good, _raw_job(fr, 1, N_FEAT)], prm, 400, "feat_slot out of range"),
             ([good, _raw_job(fr, 1, -1)], prm, 400, "feat_slot out of range"),
             ([good, _raw_job(fr, 1, 1, n_cams=0)], prm, 400, "n_cams out of range"),
             ([good, _raw_job(dict(imgs=fr["imgs"] * 2, cams=list(fr["cams"]) * 2, R_CWs=fr["R_CWs"] * 2), 1, 1)], prm, 400, "n_cams out of range"),
             ([good], p64, 400, "descriptor length"),
             ([good], p1000, 1000, "fewer keypoints"),
             ([good, _raw_job(fr, 1, 1, out=False)], prm, 400, "missing"),
             ([good, _raw_job(bad_img, 1, 1)], prm, 400, "images[1]"),
             ([good, _raw_job(fr, 0, 2)], prm, 400, "listed twice"),
             ([good], None, 400, "params"),
             ([good], prm, 0, "params")]
    for jobs, p, max_out, why in cases:
        assert call(jobs, p, max_out) == abi.OKB_ERR_INVALID_ARG, why
        msg = lib.okb_last_error(ctx._h).decode()
        assert why in msg, (why, msg)
        if why not in ("params", "descriptor length", "fewer keypoints"):
            assert "jobs[1]" in msg, msg
    assert lib.okb_detect_describe_store_batch(ctx._h, -1, None, C.byref(prm), 400, 0) == abi.OKB_ERR_INVALID_ARG
    assert lib.okb_detect_describe_store_batch(ctx._h, 1, None, C.byref(prm), 400, 0) == abi.OKB_ERR_INVALID_ARG
    for win in (0, 1):
        for ea, eb in zip(entries(ctx, win, 2), before[win]):
            for x, y in zip(ea, eb):
                assert_entry_equal(x, y)
    # with the 1000-keypoint parameters, max_out = 400 fits the store
    assert call([good], p1000, 400) == abi.OKB_OK
    assert ctx.debug_features(0, 1, 0)["n"] == good[1][3][0] > 50
    ctx.close()
    # a landmark-sharded context
    c0, c1 = capi.Context(0, 1), capi.Context(0, 1)
    capi.Context.shard_connect_local([c0, c1])
    with pytest.raises(capi.OkbError) as e:
        c0.detect_describe_store_batch([dict(fr, win=0, feat_slot=0)])
    assert e.value.code == abi.OKB_ERR_UNSUPPORTED
    c0.close()
    c1.close()


def test_more_than_65535_images_refused():
    # 517 windows whose stores hold 127 one-keypoint cameras: 516 jobs fit (65 532 images), the 517th does not
    n = 517
    ctx = capi.Context(0, n)
    w = synthetic.make_window(1, 0)
    for win in range(n):
        ctx.reserve(win, len(w.poses), len(w.landmarks), len(w.obs), len(w.imu_samples))
        ctx.reserve_features(win, 1, 127, 1, 48)
        ctx.upload(win, w)
    img = images.textured_image(seed=3, width=64, height=64, n_shapes=10)
    fr = dict(imgs=[img] * 127, cams=[w.cameras[0]] * 127, R_CWs=[np.eye(3)] * 127)
    with pytest.raises(capi.OkbError) as e:
        ctx.detect_describe_store_batch([dict(fr, win=win, feat_slot=0) for win in range(n)], max_keypoints=1)
    assert e.value.code == abi.OKB_ERR_INVALID_ARG and "jobs[516]" in str(e.value) and "65535" in str(e.value)
    assert all(ctx.debug_features(win, 0, 0)["n"] == -1 for win in (0, 515, 516))
    ctx.close()


def test_over_capacity_image_keeps_its_entry():
    big = np.random.default_rng(9).integers(0, 256, (4096, 4096), dtype=np.uint8)   # far more NMS candidates than the detector holds
    cam_big = abi.make_camera(abi.DIST_RADTAN, 4096, 4096, 2000.0, 2000.0, 2048.0, 2048.0)
    prm = dict(absolute_threshold=1.0, uniformity_radius=15.0, max_keypoints=1000, desc_bytes=48)
    ctx = capi.Context(0, 2)
    w = window(2, 0)
    for win in (0, 1):
        setup(ctx, win, w, 1000, 48)
    left, right = images.stereo_pair()
    old = np.zeros((30, 3))
    old[:, 0], old[:, 1], old[:, 2] = np.arange(30), 5.0, 7.0
    ctx.set_features(0, 0, 1, old, np.full((30, 48), 9, np.uint8))
    ctx.commit(0, 1)
    before = ctx.debug_features(0, 0, 1)
    jobs = [dict(imgs=[left, big], cams=[w.cameras[0], cam_big], R_CWs=[np.eye(3)] * 2, win=0, feat_slot=0),
            dict(imgs=[right, left], cams=[w.cameras[0], w.cameras[1]], R_CWs=[np.eye(3)] * 2, win=1, feat_slot=0)]
    got, rc = ctx.detect_describe_store_batch(jobs, return_status=True, **prm)
    assert rc == abi.OKB_ERR_CAPACITY
    assert got[0][1] is None
    ref, rc_ref = ctx.detect_describe_batch([left, big, right, left], [w.cameras[0], cam_big, w.cameras[0], w.cameras[1]],
                                            [np.eye(3)] * 4, return_status=True, **prm)
    assert rc_ref == abi.OKB_ERR_CAPACITY and ref[1] is None
    for got_i, ref_i in ((got[0][0], ref[0]), (got[1][0], ref[2]), (got[1][1], ref[3])):
        assert_det_equal(got_i, ref_i)
    assert_entry_equal(ctx.debug_features(0, 0, 1), before)
    assert ctx.debug_features(0, 0, 0)["n"] == len(ref[0][0])
    assert ctx.debug_features(1, 0, 1)["desc"].tobytes() == ref[3][1].tobytes()
    ctx.set_features(0, 0, 1, old[:29], np.zeros((29, 48), np.uint8))   # the host count of the kept entry is still 30
    ctx.set_feature_landmarks(0, 0, 0, [len(ref[0][0]) - 1], [0], [0])
    ctx.close()


def test_no_jobs_and_no_descriptors():
    lib = capi.lib()
    prm = dict(PARAMS["cfg3"], desc_bytes=64)
    ctx = capi.Context(0, 2)
    w = window(2, 0)
    for win in (0, 1):
        setup(ctx, win, w, 1000, 64)
    p = abi.DetectParams()
    assert lib.okb_detect_describe_store_batch(ctx._h, 0, None, C.byref(p), 0, 0) == abi.OKB_OK    # nothing is checked
    assert ctx.detect_describe_store_batch([], **prm) == []
    fr = frame_images(123, 2, w.cameras)
    got = ctx.detect_describe_store_batch([dict(fr, win=0, feat_slot=1, want_desc=False)], **prm)[0]
    ref = feed_twin(ctx, 1, 1, fr, prm)
    for c in range(2):
        assert got[c][1] is None
        assert got[c][0].tobytes() == ref[c][0].tobytes()
        assert_entry_equal(ctx.debug_features(0, 1, c), ctx.debug_features(1, 1, c))
    ctx.close()
