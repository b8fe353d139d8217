"""The IMU term against its extended-precision reference (tests/imu_reference.py) at the edges of the sample recursion
(tests/imu_cases.py), without a GPU: the oracle and the host build of the device templates (okb_imu.cuh with one lane,
tests/hostcheck) must both land within the measured bound at every case, for propagation, for a fresh term (redo path)
and for a term preintegrated at an earlier bias (first-order correction or redo).  Faults planted in a copy of the
reference's float64 run must each be rejected by the same comparator somewhere."""
import ctypes as C

import numpy as np
import pytest

import imu_cases as ic
import imu_reference as ir
from test_hostcheck import _hc_imu_eval, hc  # noqa: F401  (hc is a fixture)

CASES = ic.cases()
IDS = ic.case_ids()
PATHS = ("prop", "eval", "corr")


@pytest.fixture(scope="module")
def refs():
    """(case index, path) -> (reference quantities, bounds), computed once per module."""
    memo = {}

    def get(i, path):
        if (i, path) not in memo:
            memo[(i, path)] = ir.reference_and_bounds(CASES[i], path)
        return memo[(i, path)]
    return get


def test_long_double_is_extended():
    ir.require_long_double()
    assert np.finfo(np.longdouble).nmant >= 63


def _p(a):
    return C.c_void_p(a.ctypes.data)


def hc_propagate(hc, c):
    pose, sb = np.array(c["pose0"], np.float64), np.array(c["sb0"], np.float64)
    P, F = np.zeros((15, 15)), np.zeros((15, 15))
    hc.hc_imu_propagate.restype = C.c_int
    n = hc.hc_imu_propagate(C.byref(c["prm"]), _p(c["samples"]), C.c_int(len(c["samples"])), C.c_int64(c["t0"]),
                            C.c_int64(c["t1"]), _p(pose), _p(sb), _p(P), _p(F))
    return n, pose, sb, P, F


def eval_args(c):
    return (c["prm"], c["samples"], c["t0"], c["t1"], c["pose0"], c["sb0"], c["pose1"], c["sb1"])


@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_oracle_and_host_build_match_reference(i, refs, oracle, hc):  # noqa: F811
    c = CASES[i]
    for path in PATHS:
        ref, bounds = refs(i, path)
        if path == "prop":
            got = {"oracle": ir.prop_quantities(*oracle.imu_propagate(c["prm"], c["samples"], c["t0"], c["t1"], c["pose0"], c["sb0"])),
                   "host": ir.prop_quantities(*hc_propagate(hc, c))}
        else:
            sb_ref = c["sb_ref"] if path == "corr" else None
            r0, J0, S0, redo0 = oracle.eval_imu(*eval_args(c), sb_ref=sb_ref)
            r1, J1, S1, redo1 = _hc_imu_eval(hc, *eval_args(c), sb_ref=sb_ref)
            got = {"oracle": ir.eval_quantities(redo0, r0, np.hstack(J0), S0),
                   "host": ir.eval_quantities(redo1, r1, np.hstack(J1), S1)}
        for who, g in got.items():
            ratio, where = ir.compare(g, ref, bounds)
            assert ratio <= 1.0, (who, path, where, ratio)


def test_case_list_reaches_its_edges():
    """The cases do what their names say: the last integrated interval at every batch position, t1 on and between
    samples, the redo predicate on both sides, saturation exactly at the limit and one ulp above."""
    last_pos = set()
    for c in CASES:
        ts = c["samples"]["t_ns"]
        st = ir.integrate(c["samples"], c["prm"], c["t0"], c["t1"], c["sb0"], np.float64, True, False)
        assert st is not None and st["steps"] >= 1, c["name"]
        if c["group"] == "batch_end":
            last_pos.add((int(np.searchsorted(ts, c["t1"], side="left")) - 1) % 8)
    assert last_pos == set(range(8))
    by = {c["name"]: c for c in CASES}
    for name, redo in (("bg_0.9", 0), ("bg_1.1", 1), ("ba_only", 0)):
        c = by[name]
        assert ir.run_eval(c, np.float64, True)["redo"] == redo, name
    assert by["gyro_at"]["samples"]["gyro"][9, 1] == -ic.PRM_A.g_max
    assert by["gyro_ulp"]["samples"]["gyro"][9, 1] == -np.nextafter(ic.PRM_A.g_max, np.inf)


# ---------------------------------------------------------------------------------------------------- planted faults
def _drop_at_batch_boundary(c):
    """One sample dropped at a batch boundary: record 8, where the samples still cover [t0, t1]."""
    n = len(c["samples"])
    if n < 11 or not (c["samples"]["t_ns"][0] <= c["t0"] and c["samples"]["t_ns"][9] < c["t1"]):
        return None
    return dict(c, samples=np.delete(c["samples"], 8))


def _faulty_run(fault, i, path):
    """The float64 reference with `fault` planted, or None where the fault does not apply to the case."""
    c = CASES[i]
    if fault == "drop_sample":
        c = _drop_at_batch_boundary(c)
        if c is None:
            return None
        faults = ()
    elif fault == "neighbour_cache":
        if path == "prop":
            return None
        return ir.ref_eval_quantities(ir.run_eval(c, np.float64, path == "corr", cache_from=CASES[(i + 1) % len(CASES)]))
    elif fault == "nan_in_J":          # one NaN in one Jacobian column: 30 NaN in H30, 1 in g30, cost and info finite
        res = ir.run_eval(c, np.float64, path == "corr") if path != "prop" else None
        if res is None:
            return None
        res["J"][0, 29] = np.nan
        return ir.ref_eval_quantities(res)
    elif fault == "nan_in_P":          # one NaN in the propagated covariance, everything else exact
        if path != "prop":
            return None
        res = ir.run_prop(c, np.float64)
        res["P"][0, 0] = np.nan
        return ir.ref_prop_quantities(res)
    else:
        faults = (fault,)
    if path == "prop":
        return ir.ref_prop_quantities(ir.run_prop(c, np.float64, faults))
    return ir.ref_eval_quantities(ir.run_eval(c, np.float64, path == "corr", faults))


@pytest.mark.parametrize("fault", ir.FAULTS + ("drop_sample", "neighbour_cache", "nan_in_J", "nan_in_P"))
def test_planted_fault_is_rejected(fault, refs):
    """Each fault makes the comparator fail in at least one case (cheapest cases first)."""
    order = sorted(range(len(CASES)), key=lambda i: len(CASES[i]["samples"]))
    for i in order:
        for path in PATHS:
            got = _faulty_run(fault, i, path)
            if got is None:
                continue
            ratio, _ = ir.compare(got, *refs(i, path))
            if ratio > 1.0:
                return
    pytest.fail("planted fault %s passed every case" % fault)


@pytest.mark.parametrize("fault", ["nan_in_J", "nan_in_P"])
def test_non_finite_output_is_rejected_at_every_case(fault, refs):
    """A single NaN anywhere fails the comparator outright, whatever the case (not only somewhere)."""
    for i in range(len(CASES)):
        for path in PATHS:
            got = _faulty_run(fault, i, path)
            if got is not None:
                assert ir.compare(got, *refs(i, path))[0] == np.inf, (CASES[i]["name"], path)
