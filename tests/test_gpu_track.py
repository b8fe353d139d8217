"""GPU checks of okb_track_3d2d_batch (3D-2D tracking of a new frame against its resident window) against the CPU
reference tests/track_reference.py: bit-exact associations, per-round counts and cleared flags; batch against single
calls; no effect on the solver; the feature store's life cycle; host-side errors."""
import numpy as np
import pytest

import track_reference as tr
from okvis_b200 import abi, capi
from track_scene import load, make_track_scene

pytestmark = pytest.mark.gpu

_SCENES = {}


def scene(i, desc_bytes=48):
    key = (i, desc_bytes)
    if key not in _SCENES:
        _SCENES[key] = make_track_scene(i, desc_bytes=desc_bytes,
                                        distortion=[abi.DIST_RADTAN, abi.DIST_EQUIDISTANT, abi.DIST_NONE, abi.DIST_RADTAN8][i % 4])
    return _SCENES[key]


def rounds_of(sc, kind):
    return {0: sc["rounds"]["keyframes"], 1: sc["rounds"]["last_frame"], 2: sc["rounds"]["keyframes"] + sc["rounds"]["stereo"]}[kind]


def job(sc, win, kind):
    return dict(win=win, pose_b=sc["pose_b"], sb_b=sc["sb_b"], feat_slot_b=sc["feat_b"], rounds=rounds_of(sc, kind))


def reference(oracle, sc, kind, state=None):
    st = state or tr.TrackState(sc["window"], sc["store"], sc["lm_init"])
    return tr.track(oracle, st, sc["pose_b"], sc["sb_b"], sc["feat_b"], rounds_of(sc, kind)), st


def rows(res):
    """A result as plain lists: the device's arrays or the reference's tuples."""
    a = res["assoc"]
    if isinstance(a, np.ndarray):
        a = [(r["round"], r["cam_b"], r["kp_b"], r["lm_slot"], r["uncertain"]) for r in a]
    return ([tuple(int(x) for x in t) for t in a], [int(x) for x in res["num_matches"]], [int(x) for x in res["num_uncertain"]],
            [int(x) for x in res["uninit"]])


def assert_same(got, ref):
    g, r = rows(got), rows(ref)
    assert g[0] == r[0]
    assert g[1:] == r[1:]


@pytest.mark.parametrize("desc_bytes", [48, 64])
@pytest.mark.parametrize("n_sessions", [1, 8, 132])
def test_bit_exact_vs_reference(oracle, n_sessions, desc_bytes):
    ctx = capi.Context(0, n_sessions)
    n_scenes = min(n_sessions, 8)
    for s in range(n_sessions):
        load(ctx, s, scene(s % n_scenes, desc_bytes))
    jobs = [job(scene(s % n_scenes, desc_bytes), s, s % 3) for s in range(n_sessions)]
    got = ctx.track_3d2d_batch(jobs)
    refs = {}
    for s in range(n_sessions):
        key = (s % n_scenes, s % 3)
        if key not in refs:
            refs[key] = reference(oracle, scene(key[0], desc_bytes), key[1])[0]
        assert_same(got[s], refs[key])
    assert sum(int(g["num_matches"].sum()) for g in got) > 50 * n_sessions
    if n_sessions > 1:      # the larger batches also exercise cleared flags and uncertain matches
        assert any(g["uninit"].size for g in got) and any(int(g["num_uncertain"].sum()) for g in got)
    ctx.close()


def test_batch_equals_single_calls_and_leaves_other_windows(oracle):
    n = 8
    a, b = capi.Context(0, n), capi.Context(0, n)
    for s in range(n):
        load(a, s, scene(s))
        load(b, s, scene(s))
    listed = list(range(0, n, 2))[::-1]               # every other window, in another order
    batch = a.track_3d2d_batch([job(scene(s), s, 2) for s in listed])
    for s, g in zip(listed, batch):
        assert_same(g, b.track_3d2d_batch([job(scene(s), s, 2)])[0])
    for s in range(1, n, 2):                           # windows not listed still track as fresh ones
        assert_same(a.track_3d2d_batch([job(scene(s), s, 0)])[0], reference(oracle, scene(s), 0)[0])
    a.close(); b.close()


def test_no_solver_change():
    sc = scene(0)
    a, b = capi.Context(0, 1), capi.Context(0, 1)
    load(a, 0, sc); load(b, 0, sc)
    b.track_3d2d_batch([job(sc, 0, 2)])
    sa, sb = a.optimize(0, 1, max_iterations=10)[0], b.optimize(0, 1, max_iterations=10)[0]
    assert sa["final_cost"] == sb["final_cost"] and sa["iterations"] == sb["iterations"]
    da, db = a.download(0), b.download(0)
    for k in da:
        if da[k] is not None:
            assert np.array_equal(da[k], db[k]), k
    a.close(); b.close()


def test_store_lifecycle(oracle):
    sc = scene(1)
    ctx = capi.Context(0, 1)
    load(ctx, 0, sc)
    st = tr.TrackState(sc["window"], sc["store"], sc["lm_init"])
    # survives a full upload and a reset (a full upload drops edits still pending: commit them first)
    ctx.commit(0, 1)
    ctx.upload(0, sc["window"])
    ctx.reset(0, 1)
    # pending edits are seen without a commit: flags cleared, landmarks removed (and their references with them), one
    # removed slot reused at once by a new landmark that no keypoint names
    A = st.store[rounds_of(sc, 0)[0][:2]]
    used = [int(l) for l in A["lm"] if l >= 0 and st.live(int(l)) and st.lm_init[l]]
    clear, gone = used[:10], used[10:30]
    ctx.set_landmark_initialized(0, clear, np.zeros(len(clear)))
    st.lm_init[clear] = 0
    ctx.remove_landmarks(0, gone)
    for e in st.store.values():
        m = np.isin(e["lm"], gone)
        e["lm"][m], e["observed"][m] = -1, 0
    st.lm_init[gone] = 0
    st.lm[gone] = 0.0
    reuse = gone[0]
    st.lm[reuse] = st.lm[used[0]]
    ctx.set_landmarks(0, [reuse], st.lm[reuse:reuse + 1])
    ctx.set_landmark_initialized(0, [reuse], [1])
    st.lm_init[reuse] = 1
    got = ctx.track_3d2d_batch([job(sc, 0, 0)])[0]
    ref = reference(oracle, sc, 0, st)[0]
    assert_same(got, ref)
    assert reuse not in got["assoc"]["lm_slot"].tolist()
    ctx.close()


def test_remove_frame_keeps_feature_slots(oracle):
    sc = scene(2)
    ctx = capi.Context(0, 1)
    load(ctx, 0, sc)
    ctx.remove_frame(0, 0, 0)
    w = sc["window"]
    st = tr.TrackState(w, sc["store"], sc["lm_init"])
    st.counts = np.bincount(w.obs["lm_idx"][w.obs["pose_idx"] != 0].astype(np.int64), minlength=len(w.landmarks))
    rounds = rounds_of(sc, 0)
    got = ctx.track_3d2d_batch([dict(win=0, pose_b=sc["pose_b"] - 1, sb_b=sc["sb_b"] - 1, feat_slot_b=sc["feat_b"], rounds=rounds)])[0]
    st.w = type("W", (), dict(poses=w.poses[1:], speed_bias=w.speed_bias[1:], extrinsics=w.extrinsics, cameras=w.cameras))
    ref = tr.track(oracle, st, sc["pose_b"] - 1, sc["sb_b"] - 1, sc["feat_b"], rounds)
    assert_same(got, ref)
    ctx.close()


def test_errors_before_device_work(oracle):
    sc = scene(3)
    ctx = capi.Context(0, 2)
    load(ctx, 0, sc)
    ctx.upload(1, sc["window"])                     # uploaded, no store
    good = job(sc, 0, 0)
    bad = [dict(good, win=1), dict(good, win=5), dict(good, pose_b=99), dict(good, sb_b=99), dict(good, feat_slot_b=99),
           dict(good, num_best=9), dict(good, rounds=[(99, 0, 0)]), dict(good, rounds=[(0, 0, 7)]),
           dict(good, rounds=[(min(set(range(sc["F"])) - {f for f, _ in sc["store"]}), 0, 0)])]     # a slot with no keypoints
    assert all(0 <= f < sc["F"] for f, _ in sc["store"]) and len({f for f, _ in sc["store"]}) < sc["F"]
    for b in bad:
        with pytest.raises(capi.OkbError) as e:
            ctx.track_3d2d_batch([good, b] if b["win"] != 0 else [b])
        assert e.value.code == abi.OKB_ERR_INVALID_ARG
    with pytest.raises(capi.OkbError) as e:
        ctx.track_3d2d_batch([good, good])              # a window listed twice
    assert e.value.code == abi.OKB_ERR_INVALID_ARG
    fb = sc["feat_b"]
    for b in (dict(good, rounds=[(0, 5, 0)]),                                     # cam_a out of range
              dict(good, rounds=[(fb, 0, 0)]),                                    # frame B against itself in one camera
              dict(good, rounds=[sc["rounds"]["keyframes"][0]] * 256)):           # more than 255 rounds
        with pytest.raises(capi.OkbError) as e:
            ctx.track_3d2d_batch([b])
        assert e.value.code == abi.OKB_ERR_INVALID_ARG
    # output capacities and pointers, through the raw call
    import ctypes as C
    lib = capi.lib()
    rounds = (abi.TrackRound * 1)()
    rounds[0].feat_slot_a, rounds[0].cam_a, rounds[0].cam_b = sc["rounds"]["keyframes"][0]
    nA, nB = len(sc["store"][sc["rounds"]["keyframes"][0][:2]]["lm"]), len(sc["store"][(fb, 0)]["lm"])
    assoc = np.zeros(nB, abi.track_assoc_dtype)
    un = np.zeros(nA, np.uint32)
    nm, nu = np.zeros(1, np.int32), np.zeros(1, np.int32)
    na, nun = C.c_int32(0), C.c_int32(0)

    def raw(**kw):
        t = abi.TrackJob()
        t.win, t.pose_b, t.sb_b, t.feat_slot_b, t.threshold, t.num_best, t.n_rounds = 0, sc["pose_b"], sc["sb_b"], fb, 60.0, 4, 1
        t.rounds = C.cast(rounds, C.POINTER(abi.TrackRound))
        t.assoc, t.assoc_cap, t.n_assoc = assoc.ctypes.data, nB, C.pointer(na)
        t.num_matches = nm.ctypes.data_as(C.POINTER(C.c_int32)); t.num_uncertain = nu.ctypes.data_as(C.POINTER(C.c_int32))
        t.uninit, t.uninit_cap, t.n_uninit = un.ctypes.data_as(C.POINTER(C.c_uint32)), nA, C.pointer(nun)
        for k, v in kw.items():
            setattr(t, k, v)
        return lib.okb_track_3d2d_batch(ctx._h, 1, C.byref(t))
    for kw in (dict(assoc_cap=nB - 1), dict(uninit_cap=nA - 1), dict(assoc=None), dict(uninit=None), dict(n_assoc=None),
               dict(n_uninit=None), dict(num_matches=None), dict(num_uncertain=None), dict(rounds=None)):
        assert raw(**kw) == abi.OKB_ERR_INVALID_ARG, kw
    assert raw() == abi.OKB_OK
    ctx.close()
    # a descriptor length that differs across the jobs of a call
    ctx = capi.Context(0, 2)
    load(ctx, 0, sc)
    load(ctx, 1, scene(3, 64))
    with pytest.raises(capi.OkbError) as e:
        ctx.track_3d2d_batch([good, job(scene(3, 64), 1, 0)])
    assert e.value.code == abi.OKB_ERR_INVALID_ARG
    ctx.close()
    ctx = capi.Context(0, 1)
    load(ctx, 0, sc)
    assert_same(ctx.track_3d2d_batch([good])[0], reference(oracle, sc, 0)[0])   # nothing changed on the device
    ctx.close()
    c0, c1 = capi.Context(0, 1), capi.Context(0, 1)
    capi.Context.shard_connect_local([c0, c1])
    with pytest.raises(capi.OkbError) as e:
        c0.track_3d2d_batch([good])
    assert e.value.code == abi.OKB_ERR_UNSUPPORTED
    c0.close(); c1.close()
