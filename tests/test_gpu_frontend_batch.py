"""Batched frontend (okb_detect_describe_batch, okb_hamming_match_batch): every image and every match job of a batch
gives exactly what the single call gives on it, and the oracle's answer where the oracle is run."""
import ctypes as C

import numpy as np
import pytest

from okvis_b200 import abi, images, synthetic
from gate_scene import gates, make_scene
from test_oracle_frontend import CAM

gpu = pytest.mark.gpu

CAM_EQUI = abi.make_camera(abi.DIST_EQUIDISTANT, 752, 480, 461.1, 460.3, 366.2, 249.1, (-0.0027, 0.0171, -0.0201, 0.0095))
R_LIST = [np.eye(3),
          np.array([[0.9950, 0.0, -0.0998], [0.0198, 0.9801, 0.1977], [0.0978, -0.1987, 0.9752]]),
          np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])]


@pytest.fixture(scope="module")
def ctx(okb):
    c = okb.Context(0, 4)
    yield c
    c.close()


def strided(img, pad=13):
    """The same pixels in a buffer whose rows are `pad` bytes longer than the image."""
    buf = np.full((img.shape[0], img.shape[1] + pad), 77, np.uint8)
    buf[:, :img.shape[1]] = img
    return buf[:, :img.shape[1]]


def noise(seed, h, w):
    return np.random.default_rng(seed).integers(0, 256, (h, w), dtype=np.uint8)


def assert_same(a, b):
    (ka, da), (kb, db) = a, b
    assert len(ka) == len(kb)
    for f in ka.dtype.names:
        assert np.array_equal(ka[f], kb[f]), f
    assert np.array_equal(da, db)


def mixed_images():
    """stereo pairs at several seeds, two image sizes, strided rows, radtan and equidistant cameras, several R_CW,
    a flat image (no keypoints) and a noise image (too many NMS candidates for the shared-memory uniformity kernel)."""
    imgs, cams, Rs = [], [], []
    for k, seed in enumerate((0x0B200 + 3000, 11, 12)):
        left, right = images.stereo_pair(seed=seed)
        for j, img in enumerate((left, right)):
            imgs.append(strided(img) if (k + j) % 2 else img)
            cams.append(CAM if j == 0 else CAM_EQUI)
            Rs.append(R_LIST[(k + j) % 3])
    small = images.textured_image(seed=21, width=320, height=240, n_shapes=200)
    cam_small = abi.make_camera(abi.DIST_RADTAN, 320, 240, 250.0, 250.0, 160.0, 120.0, (-0.28, 0.07, 1e-4, 2e-5))
    imgs += [small, strided(small, 5), np.full((480, 752), 128, np.uint8), noise(5, 480, 752)]
    cams += [cam_small, cam_small, CAM, CAM]
    Rs += [R_LIST[1], R_LIST[2], R_LIST[0], R_LIST[1]]
    return imgs, cams, Rs


@gpu
@pytest.mark.parametrize("radius,maxk,nbytes", [(15.0, 1000, 48), (40.0, 400, 48), (15.0, 1000, 64), (40.0, 400, 64)])
def test_mixed_image_batch_equals_single_calls_and_oracle(ctx, oracle, radius, maxk, nbytes):
    imgs, cams, Rs = mixed_images()
    prm = dict(uniformity_radius=radius, max_keypoints=maxk, desc_bytes=nbytes)
    got = ctx.detect_describe_batch(imgs, cams, Rs, host_threads=3, **prm)
    assert len(got) == len(imgs)
    for i, (img, cam, R) in enumerate(zip(imgs, cams, Rs)):
        assert_same(got[i], ctx.detect_describe(img, cam, R, cam_slot=i % 8, **prm))
    assert len(got[-2][0]) == 0                       # flat image
    assert len(got[-1][0]) > 100                      # noise image (global-memory uniformity kernel)
    for i in (0, 1, 6, len(imgs) - 1):                # oracle on a subset (radtan cameras)
        if cams[i]["model"] != abi.DIST_RADTAN:
            continue
        ko, do = oracle.detect_describe(np.ascontiguousarray(imgs[i]), cams[i], Rs[i], **prm)
        kg, dg = got[i]
        for f in ("x", "y", "size", "response", "octave"):
            assert np.array_equal(kg[f], ko[f]), f
        assert np.abs(kg["angle"] - ko["angle"]).max() < 1e-3
        assert np.array_equal(dg, do)


@gpu
def test_batch_of_one_equals_single_call(ctx):
    left, _ = images.stereo_pair()
    one = ctx.detect_describe_batch([left], [CAM], [R_LIST[1]])
    assert_same(one[0], ctx.detect_describe(left, CAM, R_LIST[1]))


@gpu
def test_large_batch_sampled(ctx):
    pairs = [images.stereo_pair(seed=100 + s) for s in range(4)]
    imgs = [pairs[i % 4][(i // 4) % 2] for i in range(264)]
    Rs = [R_LIST[i % 3] for i in range(264)]
    cams = [CAM] * 264
    got = ctx.detect_describe_batch(imgs, cams, Rs, uniformity_radius=15.0, max_keypoints=1000)
    for i in (0, 1, 5, 131, 132, 200, 263):
        assert_same(got[i], ctx.detect_describe(imgs[i], cams[i], Rs[i], uniformity_radius=15.0, max_keypoints=1000))


@gpu
def test_candidate_overflow_marks_only_that_image(ctx, okb):
    big = noise(9, 4096, 4096)           # far more 3x3 maxima of the Harris score than kMaxCand (131 072)
    cam_big = abi.make_camera(abi.DIST_RADTAN, 4096, 4096, 2000.0, 2000.0, 2048.0, 2048.0)
    prm = dict(absolute_threshold=1.0, uniformity_radius=15.0, max_keypoints=1000)
    with pytest.raises(okb.OkbError) as e:
        ctx.detect_describe(big, cam_big, np.eye(3), **prm)
    assert e.value.code == abi.OKB_ERR_CAPACITY
    left, right = images.stereo_pair()
    imgs, cams = [left, big, right], [CAM, cam_big, CAM]
    out, rc = ctx.detect_describe_batch(imgs, cams, [np.eye(3)] * 3, return_status=True, **prm)
    assert rc == abi.OKB_ERR_CAPACITY
    assert out[1] is None
    for i in (0, 2):
        assert_same(out[i], ctx.detect_describe(imgs[i], cams[i], np.eye(3), **prm))


def unary(values, nbytes=48):
    out = np.zeros((len(values), nbytes * 8), np.uint8)
    for i, v in enumerate(values):
        out[i, :int(v)] = 1
    return np.packbits(out, axis=1, bitorder="little")


def match_jobs(nbytes):
    """Keyword arguments of one match per job: plain and ratio lists, 3D-2D and 2D-2D gated, skip masks, num_best 1/2/4/8,
    empty A or B, and the testMatcher.cpp known answers."""
    jobs = []
    rng = np.random.default_rng(3)
    for seed in (0, 1):
        sc = make_scene(seed, nbytes=nbytes)
        g3, g2 = gates(sc)
        skipA = (rng.random(len(sc["A"])) < 0.05).astype(np.uint8)
        skipB = (rng.random(len(sc["B"])) < 0.05).astype(np.uint8)
        for k, nb in enumerate((1, 2, 4, 8)):
            jobs.append(dict(A=sc["A"], B=sc["B"], skipA=skipA if k % 2 else None, skipB=skipB, num_best=nb, use_ratio=bool(k % 2)))
        jobs.append(dict(A=sc["A"], B=sc["B"], skipA=skipA, skipB=skipB, gate=g3, num_best=4))
        jobs.append(dict(A=sc["A"], B=sc["B"], skipA=skipA, gate=g2, num_best=2, use_ratio=True))
        jobs.append(dict(A=sc["A"], B=sc["B"], gate=g2, num_best=8))
    base = rng.integers(0, 256, (700, nbytes), dtype=np.uint8)
    B = base[rng.permutation(700)[:650]].copy()
    jobs.append(dict(A=base, B=B, threshold=60.0, num_best=4))
    jobs.append(dict(A=base[:0], B=B, threshold=60.0, num_best=4))
    jobs.append(dict(A=base[:10], B=B[:0], threshold=50.0, num_best=2))
    if nbytes == 48:
        jobs.append(dict(A=unary([10, 30, 20, 9]), B=unary([180, 21, 40, 10]), skipA=np.array([1, 0, 0, 0], np.uint8),
                         threshold=40.0, num_best=4))
        jobs.append(dict(A=unary([80, 10, 30, 20, 9]), B=unary([180, 21, 40, 10, 70]), skipA=np.array([1, 0, 0, 0, 0], np.uint8),
                         threshold=40.0, num_best=4, use_ratio=True))
    return jobs


def single_match(ctx, j):
    kw = {k: v for k, v in j.items() if k not in ("A", "B", "gate")}
    if j.get("gate") is not None:
        return ctx.hamming_match_gated(j["A"], j["B"], j["gate"], **kw)
    return ctx.hamming_match(j["A"], j["B"], **kw)


def oracle_match(oracle, j):
    kw = {k: v for k, v in j.items() if k not in ("A", "B", "gate")}
    if j.get("gate") is not None:
        return oracle.match_hamming_gated(j["A"], j["B"], j["gate"], **kw)
    return oracle.match_hamming(j["A"], j["B"], **kw)


def assert_match_equal(a, b):
    for k in ("topk", "pairs"):
        assert np.array_equal(a[k]["index_a"], b[k]["index_a"]), k
        assert np.array_equal(a[k]["distance"], b[k]["distance"]), k


@gpu
@pytest.mark.parametrize("nbytes", [48, 64])
def test_mixed_match_batch_equals_single_calls_and_oracle(ctx, okb, oracle, nbytes):
    jobs = match_jobs(nbytes)
    got = ctx.hamming_match_batch(jobs, nbytes)
    for j, g in zip(jobs, got):
        assert_match_equal(g, single_match(ctx, j))
        if len(j["A"]) and len(j["B"]):
            assert_match_equal(g, oracle_match(oracle, j))
    if nbytes == 48:
        ka, ratio = got[-2], got[-1]
        assert {(a, b) for a, b, _ in okb.matches_from_pairs(ka["pairs"], ka["topk"], 40.0)} == {(1, 2), (2, 1), (3, 3)}
        assert {(a, b) for a, b, _ in okb.matches_from_pairs(ratio["pairs"], ratio["topk"], 40.0, True, 3.0)} == {(1, 3), (3, 1)}
    empty_a, empty_b = got[-4:-2] if nbytes == 48 else got[-2:]
    assert np.all(empty_a["pairs"]["index_a"] == -1) and np.all(empty_a["pairs"]["distance"] == 60.0)
    assert np.all(empty_b["topk"]["index_a"] == -1) and np.all(empty_b["topk"]["distance"] == 50.0)


@gpu
def test_batches_beside_an_optimize_in_flight(okb):
    c = okb.Context(0, 4)
    try:
        ws = [synthetic.make_window(1, i) for i in range(4)]
        c.upload_batch(0, ws)
        ref = c.optimize(0, 4, max_iterations=6)
        ref_states = c.download_batch(0, 4)
        left, right = images.stereo_pair()
        imgs, cams, Rs = [left, right] * 4, [CAM, CAM_EQUI] * 4, R_LIST[:2] * 4
        det_ref = [c.detect_describe(i, cm, R) for i, cm, R in zip(imgs, cams, Rs)]
        jobs = match_jobs(48)
        match_ref = [single_match(c, j) for j in jobs]
        c.detect_describe_batch(imgs, cams, Rs)        # sizes the batch buffers, so the calls below allocate nothing
        c.hamming_match_batch(jobs, 48)
        c.upload_batch(0, ws)
        c.optimize_async(0, 4, max_iterations=6)
        det = c.detect_describe_batch(imgs, cams, Rs)
        got = c.hamming_match_batch(jobs, 48)
        summ = c.optimize_finish(0, 4)
        states = c.download_batch(0, 4)
        for a, b in zip(det, det_ref):
            assert_same(a, b)
        for a, b in zip(got, match_ref):
            assert_match_equal(a, b)
        for a, b in zip(summ, ref):
            assert {k: v for k, v in a.items() if k != "solve_time_s"} == {k: v for k, v in b.items() if k != "solve_time_s"}
        for a, b in zip(states, ref_states):
            for k in ("poses", "speed_bias", "landmarks", "quality"):
                assert np.array_equal(a[k], b[k]), k
    finally:
        c.close()


@gpu
def test_batch_argument_checks(ctx, okb):
    L = okb.lib()
    h = ctx._h
    left, _ = images.stereo_pair()
    prm = abi.DetectParams()
    prm.uniformity_radius, prm.absolute_threshold, prm.max_keypoints, prm.desc_bytes, prm.rotation_invariance = 40.0, 800.0, 400, 48, 1
    kps = np.zeros((2, 400), abi.keypoint_dtype)
    desc = np.zeros((2, 400, 48), np.uint8)
    n_out = np.full(2, 7, np.int32)

    def descs(**override):
        arr = (abi.ImageDesc * 2)()
        for d in arr:
            d.img, d.width, d.height, d.stride = left.ctypes.data, 752, 480, 752
            C.memmove(C.addressof(d.cam), np.array([CAM], abi.camera_dtype).ctypes.data, C.sizeof(abi.Camera))
        for k, v in override.items():
            setattr(arr[1], k, v)
        return arr

    def call(arr, n=2, p=prm, out=kps):
        return L.okb_detect_describe_batch(h, n, arr, C.byref(p) if p is not None else None,
                                           C.c_void_p(out.ctypes.data) if out is not None else None, C.c_void_p(desc.ctypes.data), 400,
                                           C.c_void_p(n_out.ctypes.data), 0)

    assert call(descs()) == 0
    assert call(descs(), n=0) == 0
    for bad in (dict(img=None), dict(stride=700), dict(width=32), dict(height=-1)):
        assert call(descs(**bad)) == abi.OKB_ERR_INVALID_ARG, bad
    assert call(descs(), n=-1) == abi.OKB_ERR_INVALID_ARG
    assert call(None) == abi.OKB_ERR_INVALID_ARG
    assert call(descs(), p=None) == abi.OKB_ERR_INVALID_ARG
    assert call(descs(), out=None) == abi.OKB_ERR_INVALID_ARG
    A = np.zeros((4, 48), np.uint8)
    good = ctx.make_match_job(A, A)
    for field, value in (("nA", -1), ("nB", -2), ("num_best", 0), ("num_best", 9), ("A", None), ("out_pairs", None)):
        bad = ctx.make_match_job(A, A)
        setattr(bad, field, value)
        arr = (abi.MatchJob * 2)(good, bad)
        assert L.okb_hamming_match_batch(h, 2, arr, 48) == abi.OKB_ERR_INVALID_ARG, field
    assert L.okb_hamming_match_batch(h, -1, None, 48) == abi.OKB_ERR_INVALID_ARG
    assert L.okb_hamming_match_batch(h, 0, None, 48) == 0
    assert L.okb_hamming_match_batch(h, 1, None, 48) == abi.OKB_ERR_INVALID_ARG


def test_batch_struct_layouts():
    assert C.sizeof(abi.ImageDesc) == 8 + 4 * 4 + 112 + 9 * 8
    assert abi.ImageDesc.cam.offset == 24 and abi.ImageDesc.R_CW.offset == 136
    assert C.sizeof(abi.MatchJob) == 4 * 8 + 6 * 4 + 3 * 8
    assert abi.MatchJob.nA.offset == 32 and abi.MatchJob.gate.offset == 56 and abi.MatchJob.out_pairs.offset == 72
