"""The MPC's filter line search (step S6 of forward_linesearch2_kernel) decision by decision against the oracle: every case of
linesearch_ref in one batch per grid, at trial caps from 1 to past the 14 that alpha_min allows, with non-finite inputs, and through the
control step. Trial counts, step lengths and status are equal; merits, violations and the descent metric armijo agree within 1e-8, x
within 1e-7 and u within 1e-6, relative to max(1, |oracle|)."""
import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc

import linesearch_ref as L

pytestmark = pytest.mark.gpu

CAPS = (1, 2, 13, 14, 20)
FIELDS = ("merit0", "merit1", "viol0", "viol1", "armijo")


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


@pytest.fixture(scope="module")
def cases(oracle):
    return {g: L.make_cases(oracle, g) for g in L.GRIDS}


def _context(grid, B, cap=L.MAX_TRIALS):
    N, dt = L.GRIDS[grid]
    if np.ndim(dt) == 0:
        return hb.Context(horizon_N=N, dt=dt, max_batch=B, device=0, line_search_max_trials=cap)
    return hb.Context(horizon_N=N, dt=float(np.max(dt)), max_batch=B, device=0, line_search_max_trials=cap, time_horizon=float(np.sum(dt)),
                      event_nodes=True)


def _solve(ctx, grid, x0, xr, sw, md, xt, ut):
    """hb_mpc_solve_batch on the uniform grids, hb_mpc_solve_grid_batch with the grid's node times on the event grid."""
    N, dt = L.GRIDS[grid]
    if np.ndim(dt) == 0:
        return ctx.mpc_solve(x0, xr, sw, md, xt, ut)
    B = x0.shape[0]
    tk = np.tile(L.EVENT_TIMES, (B, 1))
    return ctx.mpc_solve_grid(x0, tk, np.full(B, N, dtype=np.int32), xr, sw, md, xt, ut)


def _compare(dev, cases, oracle, cap, what):
    """Instance by instance against the capped oracle; returns the largest deviation of each compared field."""
    dev_max = dict.fromkeys(FIELDS + ("x", "u"), 0.0)
    for i, (name, N, dt, *c, expected) in enumerate(cases):
        xo, uo, io = oracle.mpc_iteration(N, dt, *c, max_trials=cap)
        d = dev[2][i]
        tag = (what, cap, name)
        assert (d["alpha"], d["n_trials"], d["status"]) == (io["alpha"], io["n_trials"], io["status"]), (tag, io, d)
        for f in FIELDS:
            e = abs(d[f] - io[f]) / max(1.0, abs(io[f]))
            assert e < L.TOL, (tag, f, d[f], io[f])
            dev_max[f] = max(dev_max[f], e)
        ex, eu = _rel(dev[0][i], xo), _rel(dev[1][i], uo)
        assert ex < 1e-7 and eu < 1e-6, (tag, ex, eu)
        dev_max["x"], dev_max["u"] = max(dev_max["x"], ex), max(dev_max["u"], eu)
        if io["alpha"] == 0.0:
            # rejected: the warm start comes back as it went in, but for node 0, which the kernel pins to x0 before the search
            x0, xt, ut = c[0], c[4], c[5]
            assert dev[1][i].tobytes() == ut.tobytes(), tag
            assert dev[0][i, 1:].tobytes() == xt[1:].tobytes() and dev[0][i, 0].tobytes() == x0.tobytes(), tag
            assert d["merit1"] == d["merit0"] and d["viol1"] == d["viol0"], tag
    return dev_max


@pytest.mark.parametrize("grid", tuple(L.GRIDS))
def test_every_line_search_case_vs_oracle(grid, cases, oracle):
    """All cases of the grid in one batch, each trial's decision the oracle's."""
    cs = cases[grid]
    ctx = _context(grid, len(cs))
    try:
        dev = _solve(ctx, grid, *L.stack(cs))
    finally:
        ctx.close()
    dev_max = _compare(dev, cs, oracle, L.MAX_TRIALS, grid)
    assert sum(dev[2]["alpha"] == 0.0) >= 1
    print("%s: largest deviation from the oracle %s" % (grid, {k: "%.1e" % v for k, v in dev_max.items()}))


@pytest.mark.parametrize("cap", CAPS)
def test_trial_caps_vs_capped_oracle(cap, cases, oracle):
    """One context per cap on every grid's cases: the kernel stops where the capped oracle does; caps above 14 act as 14, since
    alpha_min ends the search first."""
    for grid, cs in cases.items():
        ctx = _context(grid, len(cs), cap)
        try:
            dev = _solve(ctx, grid, *L.stack(cs))
        finally:
            ctx.close()
        _compare(dev, cs, oracle, cap, grid)
        if cap >= L.MAX_TRIALS:
            assert dev[2]["n_trials"].max() == L.MAX_TRIALS


def test_non_finite_inputs_keep_the_iterate_and_leave_the_batch_alone(cases, oracle):
    """A NaN in one node of x_ref and a NaN in the warm-start input: status 3, no trial, alpha 0, the iterate kept but for node 0; every
    other instance of the batch is the same bit for bit as in a batch without the poisoned ones."""
    grid = "baseline"
    cs = [c for c in cases[grid] if c[0] in ("filter/alpha1/merit-only", "armijo/alpha1/squeeze", "trials/03/move-x", "rejected/move-x")]
    x0, xr, sw, md, xt, ut = L.stack(cs)
    B = len(cs)
    bad = tuple(a.copy() for a in (x0, xr, sw, md, xt, ut))
    bad = tuple(np.concatenate([a, a[:2]]) for a in bad)
    bad[1][B, 37, 7] = np.nan                 # x_ref of instance B at node 37
    bad[5][B + 1, 12, 14] = np.nan            # warm-start input of instance B + 1 at node 12
    ctx = _context(grid, B + 2)
    try:
        clean = _solve(ctx, grid, x0, xr, sw, md, xt, ut)
        dev = _solve(ctx, grid, *bad)
    finally:
        ctx.close()
    for j in (B, B + 1):
        d = dev[2][j]
        assert (d["status"], d["n_trials"], d["alpha"]) == (3, 0, 0.0), j
        assert dev[1][j].tobytes() == bad[5][j].tobytes(), j
        assert dev[0][j, 1:].tobytes() == bad[4][j, 1:].tobytes() and dev[0][j, 0].tobytes() == bad[0][j].tobytes(), j
        io = oracle.mpc_iteration(L.GRIDS[grid][0], L.GRIDS[grid][1], *(a[j] for a in bad))[2]
        assert (io["status"], io["n_trials"], io["alpha"]) == (3, 0, 0.0), j
    for k in range(3):
        assert dev[k][:B].tobytes() == clean[k].tobytes(), k


def test_control_step_reports_the_solve_info(cases):
    """hb_control_step_batch runs the same line search: its info equals hb_mpc_solve_batch's on cases of every branch."""
    grid = "baseline"
    names = ("violation/alpha1/cold-start", "violation/backtracked/single-support-cold-start", "filter/alpha1/merit-only",
             "filter/alpha1/violation-only", "armijo/alpha1/squeeze", "armijo/backtracked/unloaded-heels", "armijo/alpha1/between-factors",
             "trials/05/move-x",
             "rejected/move-x")
    cs = [c for c in cases[grid] if c[0] in names]
    assert len(cs) == len(names)
    x0, xr, sw, md, xt, ut = L.stack(cs)
    ctx = _context(grid, len(cs))
    try:
        solve = ctx.mpc_solve(x0, xr, sw, md, xt, ut)
        step = ctx.control_step(0.002, x0, xr, sw, md, sc.consistent_rbd(x0), xt, ut)
    finally:
        ctx.close()
    assert step[2].tobytes() == solve[2].tobytes()
    assert _rel(step[0], solve[0]) < 1e-12 and _rel(step[1], solve[1]) < 1e-12
