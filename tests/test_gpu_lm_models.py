"""k_landmarks is instantiated per distortion model: one model shared by every camera of a launch selects that
model's instantiation, a launch that mixes models runs the run-time switch.  Every model goes through the solver
against the CPU oracle, and a mixed-model batch must give each window the result it gets alone."""
import dataclasses

import numpy as np
import pytest

from okvis_b200 import abi, synthetic
from test_gpu_solver import compare

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(okb):
    c = okb.Context(0, 8)
    yield c
    c.close()


def radtan8_window():
    """A radtan window whose cameras use the rational 8-coefficient model (small rational terms)."""
    w = synthetic.make_window(1, 9, cfg=dataclasses.replace(synthetic.CONFIGS[1], n_cams=2, n_landmarks=200))
    cams = w.cameras.copy()
    cams["model"] = abi.DIST_RADTAN8
    cams["dist"][:, 4:8] = (0.002, 0.001, 0.0005, 0.0002)
    return dataclasses.replace(w, cameras=cams)


def test_radtan8_model(ctx, oracle):
    compare(ctx, oracle, radtan8_window())


def test_mixed_model_batch_equals_single(ctx):
    """The batch mixes radtan and equidistant cameras, so it runs the run-time switch; alone, each window runs its
    model's instantiation.  The two compile the same formulas into differently fused multiply-adds, so the results
    agree to rounding (amplified over the iterations), not bit for bit; the solver decisions are identical."""
    equi = dataclasses.replace(synthetic.CONFIGS[1], distortion=abi.DIST_EQUIDISTANT, n_cams=2, n_landmarks=200)
    ws = [synthetic.make_window(1, i) for i in range(3)] + [synthetic.make_window(2, 1), synthetic.make_window(1, 7, cfg=equi)]
    for i, w in enumerate(ws):
        ctx.upload(i, w)
    batch = ctx.optimize(0, len(ws), max_iterations=8)
    states = [ctx.download(i) for i in range(len(ws))]
    for i, w in enumerate(ws):
        ctx.upload(7, w)
        single = ctx.optimize(7, 1, max_iterations=8)[0]
        st = ctx.download(7)
        assert batch[i]["iterations"] == single["iterations"]
        assert batch[i]["num_successful_steps"] == single["num_successful_steps"]
        assert batch[i]["termination"] == single["termination"]
        assert abs(batch[i]["final_cost"] - single["final_cost"]) < 1e-9 * single["final_cost"]
        assert np.abs(states[i]["poses"] - st["poses"]).max() < 1e-8
