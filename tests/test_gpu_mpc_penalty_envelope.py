"""The MPC solve where its soft constraints act, against the float64 CPU oracle: joint position and velocity limits, normal-force bounds and
friction cones in every region of the relaxed barrier (interior just above delta, the quadratic band 0 < h <= delta, violation h <= 0), on
both sides of every bound, in stance, both single supports and flight (penalty_ref.make_cases). The node LQ kernel evaluates the
penalties' value, gradient and curvature in one lane pass from its per-lane limit table; the line search evaluates their values again with
one logarithm per group of arguments above delta (BarrierSum) from the model constants. merit0 checks the first, merit1, alpha and the
trial count the second, and the iterates both. Tolerances are the suite's (test_gpu_horizon_envelope): alpha and trial counts equal, merit0
and merit1 within 1e-8, x within 1e-7 and u within 1e-6 relative to max(1, |ref|)."""
import os

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
import penalty_ref as P
from test_gpu_horizon_envelope import _assert_iteration

pytestmark = pytest.mark.gpu

THREADS = min(8, os.cpu_count() or 1)
FAMILIES = ("base", "pos", "vel", "force", "cone", "mixed")


@pytest.fixture(scope="module")
def solved(oracle):
    """Every case in one batch: two SQP iterations on the device (the second from the first's result) and on the oracle."""
    cases = P.make_cases(oracle)
    x0, xr, sw, md, xt, ut = P.stack(cases)
    ctx = hb.Context(horizon_N=P.N, dt=P.DT, max_batch=len(cases), device=0)
    try:
        dev1 = ctx.mpc_solve(x0, xr, sw, md, xt, ut)
        dev2 = ctx.mpc_solve(x0, xr, sw, md, dev1[0], dev1[1])
        alone = {j: ctx.mpc_solve(*(a[j:j + 1] for a in (x0, xr, sw, md, xt, ut))) for j in _probe_indices(cases)}
    finally:
        ctx.close()
    orc1 = oracle.mpc_iteration_batch(P.N, P.DT, x0, xr, sw, md, xt, ut, threads=THREADS)
    orc2 = oracle.mpc_iteration_batch(P.N, P.DT, x0, xr, sw, md, orc1[0], orc1[1], threads=THREADS)
    return cases, ((dev1, orc1), (dev2, orc2)), dev1, alone


def _probe_indices(cases):
    """A few instances for the batch-shape check: the first and last case, and one band case of each family."""
    pick = [0, len(cases) - 1]
    for fam in ("pos", "vel", "force", "cone"):
        pick.append(next(i for i, c in enumerate(cases) if P.family(c) == fam and "band" in c["targets"].values()))
    return pick


def _rel(a, b):
    return abs(a - b) / max(1.0, abs(b))


@pytest.mark.parametrize("fam", FAMILIES)
def test_sqp_iterations_in_every_penalty_region_vs_oracle(fam, solved):
    """Two iterations of every case of one penalty family: status, alpha, trial count, merit0, merit1, viol1 and the iterates."""
    cases, its, _, _ = solved
    idx = [i for i, c in enumerate(cases) if P.family(c) == fam]
    assert idx
    worst = np.zeros(4)
    for it, (dev, orc) in enumerate(its):
        for i in idx:
            what = (cases[i]["name"], it)
            io = orc[2][i]
            assert io["status"] == 0, what
            ex, eu = _assert_iteration(dev, orc, i, what)
            em, ev = _rel(dev[2]["merit1"][i], io["merit1"]), _rel(dev[2]["viol1"][i], io["viol1"])
            assert em < 1e-8 and ev < 1e-8, (what, io, dev[2][i])
            worst = np.maximum(worst, (ex, eu, _rel(dev[2]["merit0"][i], io["merit0"]), em))
    back = sum(its[0][1][2][i]["alpha"] < 1.0 for i in idx)
    print("%s: %d cases, %d back-track; max relative deviation from the oracle x %.2e u %.2e merit0 %.2e merit1 %.2e"
          % (fam, len(idx), back, *worst))


def test_batch_shape_leaves_penalty_cases_bitwise_unchanged(solved):
    """A case solved alone (B = 1) equals its copy in the full batch, bit for bit."""
    cases, _, full, alone = solved
    for j, one in alone.items():
        assert np.array_equal(one[0][0], full[0][j]) and np.array_equal(one[1][0], full[1][j]), cases[j]["name"]
        assert one[2][0].tobytes() == full[2][j].tobytes(), cases[j]["name"]
