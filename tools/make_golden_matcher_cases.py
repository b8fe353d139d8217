#!/usr/bin/env python
"""Runs the REFERENCE's own matcher (okvis_matcher compiled unmodified: oracle/Makefile.ref ->
oracle/_ref/libokvis_matcher_ref.so) on every input of tests/test_oracle_vs_reference_matcher.py and stores what it
returned in tests/golden/matcher_reference_cases.npz: per call the (A, B, distance) matches, their number and a checksum
of the inputs.  Needs a checkout of the reference (REF=<path> for oracle/Makefile.ref).
Usage: python tools/make_golden_matcher_cases.py [--check]"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "matcher_reference_cases.npz")
SO = os.path.join(ROOT, "oracle", "_ref", "libokvis_matcher_ref.so")
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_oracle_vs_reference_matcher as cases  # noqa: E402


def reference_match(lib, D, skipA=None, skipB=None, threshold=4.0, num_best=4, use_ratio=False, ratio_threshold=3.0, threads=1):
    D = np.ascontiguousarray(D, np.float32)
    nA, nB = D.shape
    a, d = np.zeros(nB, np.int32), np.zeros(nB, np.float32)
    sa = np.ascontiguousarray(skipA, np.uint8) if skipA is not None else None
    sb = np.ascontiguousarray(skipB, np.uint8) if skipB is not None else None
    n = lib.okr_match(C.c_void_p(D.ctypes.data), nA, nB, C.c_void_p(sa.ctypes.data) if sa is not None else None,
                      C.c_void_p(sb.ctypes.data) if sb is not None else None, C.c_float(threshold), num_best, int(use_ratio),
                      C.c_float(ratio_threshold), threads, C.c_void_p(a.ctypes.data), C.c_void_p(d.ctypes.data))
    m = np.array([(int(a[b]), b, float(d[b])) for b in range(nB) if a[b] >= 0], np.float64).reshape(-1, 3)
    return m, n


def generate():
    """One packed record for all calls: call i returned matches[offsets[i]:offsets[i + 1]] (rows A, B, distance)."""
    subprocess.run(["make", "-s", "-f", "Makefile.ref"], cwd=os.path.join(ROOT, "oracle"), check=True)
    lib = C.CDLL(SO)
    lib.okr_match.restype = C.c_int
    keys, ms, ns, crcs = [], [], [], []
    for key, kw in cases.all_calls():
        m, n = reference_match(lib, **kw)
        keys.append(key)
        ms.append(m)
        ns.append(n)
        crcs.append(cases.input_checksum(kw))
    return {"source": np.array("okvis_matcher (unmodified reference sources) via oracle/Makefile.ref"), "keys": np.array(keys),
            "offsets": np.cumsum([0] + [len(m) for m in ms]), "matches": np.concatenate(ms), "n": np.array(ns, np.int32),
            "crc": np.array(crcs, np.int64)}


def main():
    out = generate()
    if "--check" in sys.argv:
        old = np.load(OUT)
        for k in out:
            if k != "source":
                assert np.array_equal(out[k], old[k]), k
        print("fixture reproduced")
        return
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes,", len(out["keys"]), "calls")


if __name__ == "__main__":
    main()
