"""CPU: the oracle's restatement of DenseMatcher::match against the REAL reference matcher -- okvis_matcher's own sources
compiled unmodified (oracle/Makefile.ref -> oracle/_ref/libokvis_matcher_ref.so; the one part of the reference that builds
without Eigen / Ceres / OpenCV).  What the reference returned on every input below is stored in
tests/golden/matcher_reference_cases.npz (tools/make_golden_matcher_cases.py), so the comparison needs no reference tree.
Bit-exact match sets on tie-heavy random inputs, with skips, all numBest values, absolute and ratio thresholds, and
through the Hamming distance.  The inputs are regenerated here from their seeds; a checksum per input guards against a
generator that no longer reproduces what the reference was run on."""
import os
import zlib

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = os.path.join(ROOT, "tests", "golden", "matcher_reference_cases.npz")


def _dist(va, vb):
    return np.abs(np.subtract.outer(np.array(va, float), np.array(vb, float))).astype(np.float32)


def known_answer_calls():
    """testMatcher.cpp:69-155."""
    yield "known0", dict(D=_dist([1, 3, 2, 0.9], [18, 2.1, 4, 1]), skipA=[1, 0, 0, 0], threshold=4.0)
    yield "known1", dict(D=_dist([8, 1, 3, 2, 0.9], [18, 2.1, 4, 1, 7]), skipA=[1, 0, 0, 0, 0], threshold=4.0, use_ratio=True,
                         ratio_threshold=3.0)


def tie_heavy_calls(num_best, use_ratio):
    rng = np.random.default_rng(100 + num_best + 10 * use_ratio)
    for trial in range(60):
        nA, nB = int(rng.integers(1, 60)), int(rng.integers(1, 60))
        levels = int(rng.integers(2, 12))                                  # few distinct distances: ties everywhere
        D = rng.integers(0, levels, (nA, nB)).astype(np.float32)
        skipA = (rng.random(nA) < 0.1).astype(np.uint8)
        skipB = (rng.random(nB) < 0.1).astype(np.uint8)
        thr = float(rng.integers(1, levels + 1))
        ratio = float(rng.choice([1.0, 1.5, 3.0]))
        yield "tie_nb%d_r%d_%d" % (num_best, use_ratio, trial), dict(D=D, skipA=skipA, skipB=skipB, threshold=thr, num_best=num_best,
                                                                      use_ratio=use_ratio, ratio_threshold=ratio)


def hamming_inputs():
    rng = np.random.default_rng(7)
    for nA, nB, flips in ((300, 280, 30), (64, 512, 60), (500, 37, 12)):
        base = rng.integers(0, 256, (max(nA, nB), 48), dtype=np.uint8)
        A = base[:nA].copy()
        B = base[rng.permutation(max(nA, nB))[:nB]].copy()
        for row in B:
            for i in rng.integers(0, 384, rng.integers(0, flips)):
                row[i >> 3] ^= np.uint8(1 << (i & 7))
        yield "%dx%d" % (nA, nB), A, B


def hamming_calls():
    for tag, A, B in hamming_inputs():
        D = np.unpackbits(A[:, None, :] ^ B[None, :, :], axis=2).sum(2).astype(np.float32)
        for use_ratio in (False, True):
            yield "hamming_%s_r%d" % (tag, use_ratio), dict(D=D, threshold=60.0, num_best=4, use_ratio=use_ratio, ratio_threshold=3.0)


def thread_calls():
    rng = np.random.default_rng(11)
    D = rng.random((200, 180)).astype(np.float32) * 100.0                  # continuous distances: no ties
    for threads in (1, 4):
        yield "threads%d" % threads, dict(D=D, threshold=30.0, threads=threads)


def all_calls():
    yield from known_answer_calls()
    for num_best in (1, 2, 4, 8):
        for use_ratio in (False, True):
            yield from tie_heavy_calls(num_best, use_ratio)
    yield from hamming_calls()
    yield from thread_calls()


def input_checksum(kw):
    """crc32 over the call's inputs: distance matrix, skip flags and parameters."""
    c = zlib.crc32(np.ascontiguousarray(kw["D"], np.float32).tobytes())
    for k in ("skipA", "skipB"):
        if kw.get(k) is not None:
            c = zlib.crc32(np.ascontiguousarray(kw[k], np.uint8).tobytes(), c)
    p = [kw.get("threshold", 4.0), kw.get("num_best", 4), float(kw.get("use_ratio", False)), kw.get("ratio_threshold", 3.0),
         kw.get("threads", 1)]
    return zlib.crc32(np.array(p, np.float64).tobytes(), c)


@pytest.fixture(scope="module")
def ref():
    """ref(key, **inputs) -> (sorted [(a, b, distance)], number of matches) as the reference matcher returned them."""
    z = np.load(FIX)
    row = {k: i for i, k in enumerate(z["keys"].tolist())}
    offsets, matches = z["offsets"], z["matches"]

    def match(key, **kw):
        i = row[key]
        assert int(z["crc"][i]) == input_checksum(kw), "inputs of %s are not those the reference was run on" % key
        return sorted((int(a), int(b), float(d)) for a, b, d in matches[offsets[i]:offsets[i + 1]]), int(z["n"][i])
    return match


def oracle_set(o):
    return sorted((int(a), int(b), float(d)) for (a, b), d in zip(o["matches"], o["distances"]))


def test_reference_known_answers_on_the_reference_itself(ref):
    """testMatcher.cpp:69-155 on the compiled reference: the fixture the oracle is pinned with really is what the
    reference computes."""
    (k0, c0), (k1, c1) = known_answer_calls()
    got, _ = ref(k0, **c0)
    assert {(a, b) for a, b, _ in got} == {(1, 2), (2, 1), (3, 3)}
    got, _ = ref(k1, **c1)
    assert {(a, b) for a, b, _ in got} == {(1, 3), (3, 1)}


@pytest.mark.parametrize("num_best", [1, 2, 4, 8])
@pytest.mark.parametrize("use_ratio", [False, True])
def test_oracle_equals_reference_on_tie_heavy_matrices(ref, oracle, num_best, use_ratio):
    for trial, (key, kw) in enumerate(tie_heavy_calls(num_best, use_ratio)):
        r, n = ref(key, **kw)
        o = oracle.match_matrix(kw["D"], kw["skipA"], kw["skipB"], kw["threshold"], num_best, use_ratio, kw["ratio_threshold"])
        assert oracle_set(o) == r, (trial, kw["D"].shape, kw["threshold"])
        assert n == len(r)


def test_oracle_hamming_equals_reference_on_descriptor_distances(ref, oracle):
    calls = dict(hamming_calls())
    for tag, A, B in hamming_inputs():
        for use_ratio in (False, True):
            key = "hamming_%s_r%d" % (tag, use_ratio)
            r, _ = ref(key, **calls[key])
            o = oracle.match_hamming(A, B, None, None, threshold=60.0, num_best=4, use_ratio=use_ratio, ratio_threshold=3.0)
            assert oracle_set(o) == r


def test_four_reference_threads_agree_with_the_sequential_order_on_these_inputs(ref):
    """The reference runs four matcher threads (Frontend.cpp:80) and its result can depend on their interleaving; the
    project's contract is the sequential order.  On inputs without contested ties the two coincide -- a sanity check that the
    threaded reference is the same algorithm, not a parity requirement."""
    (k1, c1), (k4, c4) = thread_calls()
    r1, _ = ref(k1, **c1)
    r4, _ = ref(k4, **c4)
    assert r1 == r4
