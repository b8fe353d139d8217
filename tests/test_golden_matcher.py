"""Golden vectors made by the reference's own matcher (tools/make_golden_matcher.py: okvis_matcher compiled unmodified,
tests/golden/matcher_reference.npz).  CPU: the oracle reproduces them bit-exactly.  GPU: the CUDA matcher, through the
C-ABI, reproduces them bit-exactly -- parity of row a-U against outputs of the reference itself, without the reference
tree."""
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = os.path.join(ROOT, "tests", "golden", "matcher_reference.npz")


def cases():
    z = np.load(FIX)
    for i in range(int(z["n_cases"])):
        thr, nb, use_ratio, ratio = z["params%d" % i]
        yield i, z["A%d" % i], z["B%d" % i], z["skipA%d" % i], z["skipB%d" % i], float(thr), int(nb), bool(use_ratio), float(ratio), z["matches%d" % i]


def check(run_match, epilogue):
    """run_match(A, B, skipA, skipB, threshold, num_best, use_ratio, ratio) -> dict(pairs, topk); epilogue = the host-side
    setBestMatch loop (capi.matches_from_pairs)."""
    n = 0
    for i, A, B, sA, sB, thr, nb, use_ratio, ratio, want in cases():
        r = run_match(A, B, sA, sB, thr, nb, use_ratio, ratio)
        got = np.array(epilogue(r["pairs"], r["topk"], thr, use_ratio, ratio), np.float64).reshape(-1, 3)
        assert got.shape == want.shape, (i, got.shape, want.shape)
        assert np.array_equal(got, want), i
        n += len(want)
    assert n > 1000


def test_fixture_present():
    z = np.load(FIX)
    assert int(z["n_cases"]) == 10 and "unmodified reference sources" in str(z["source"])


def test_oracle_reproduces_the_reference_vectors(oracle, okb):
    check(lambda A, B, sA, sB, thr, nb, ur, ratio: oracle.match_hamming(A, B, sA, sB, threshold=thr, num_best=nb, use_ratio=ur, ratio_threshold=ratio),
          okb.matches_from_pairs)


@pytest.mark.gpu
def test_cuda_matcher_reproduces_the_reference_vectors(okb):
    ctx = okb.Context(0, 1)
    try:
        check(lambda A, B, sA, sB, thr, nb, ur, ratio: ctx.hamming_match(A, B, sA, sB, threshold=thr, num_best=nb, use_ratio=ur, ratio_threshold=ratio),
              okb.matches_from_pairs)
    finally:
        ctx.close()
