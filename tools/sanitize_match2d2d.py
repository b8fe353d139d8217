#!/usr/bin/env python
"""Small run of okb_match2d2d_batch for compute-sanitizer (memcheck / racecheck), in the style of tools/sanitize_run.py:
two sessions of tests/temporal_scene.py at 160 keypoints per image, a call with the temporal jobs of both cameras (A and
B in different feature slots and poses), a mixed call (one temporal job, one stereo-shaped job with A = B) and the
stereo call.  Records are checked against the CPU restatement so that a run that completes also computed the right
thing.

    compute-sanitizer --tool memcheck python tools/sanitize_match2d2d.py
    compute-sanitizer --tool racecheck python tools/sanitize_match2d2d.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from okvis_b200 import abi, capi  # noqa: E402
from oracle import oracle_py  # noqa: E402
from temporal_scene import jobs, load, make_temporal_scene, stereo_jobs  # noqa: E402


def main():
    scs = [make_temporal_scene(i, m, n_kp=160, oracle=oracle_py) for i, m in enumerate([abi.DIST_RADTAN, abi.DIST_EQUIDISTANT])]
    ctx = capi.Context(0, 2)
    for s, sc in enumerate(scs):
        load(ctx, s, sc)
    n = 0
    for c in (0, 1):
        got = ctx.match2d2d_batch([dict(jobs(sc)[c], win=s) for s, sc in enumerate(scs)])
        for s, sc in enumerate(scs):
            ref = sc["records"][c]
            assert [tuple(int(g[k]) for k in ("kp_a", "kp_b", "lm_slot_a", "lm_slot_b", "can_be_initialized")) for g in got[s]] == \
                   [r[:5] for r in ref]
            n += len(got[s])
    mixed = ctx.match2d2d_batch([dict(jobs(scs[0])[0], win=0), dict(stereo_jobs(scs[1])[1], win=1)])
    st = ctx.stereo_init_batch([dict(stereo_jobs(scs[1])[0], win=1)])
    assert mixed[1].tobytes() == st[0].tobytes()
    ctx.close()
    print("match2d2d: %d temporal records, mixed %d + %d, stereo %d" % (n, len(mixed[0]), len(mixed[1]), len(st[0])))


if __name__ == "__main__":
    main()
