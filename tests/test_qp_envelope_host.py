"""The known-optimum QPs of tests/qp_ref.py against the float64 CPU interior point (oracle.hbo.qp_solve: no row capacity, termination
at relative residuals 1e-11 and complementarity 1e-13). This pins the generator independently of the CUDA solver, at every problem the GPU
envelope test (test_gpu_qp_envelope.py) solves."""
import numpy as np
import pytest

import qp_ref as Q

RHO = 1e-8          # Context's default wbc_rho, the weight the GPU test solves with
ORACLE_RTOL = 1e-9


def _solve_all(oracle, qps, what):
    worst = 0.0
    for i, q in enumerate(qps):
        x, st, it = oracle.qp_solve(q.H, q.g, q.A, q.lb, q.ub, RHO)
        assert st == 0, "%s[%d]: oracle status %d after %d iterations" % (what, i, st, it)
        worst = max(worst, Q.check_solution(x, q, "%s[%d]" % (what, i)))
    assert worst <= ORACLE_RTOL, "%s: |x - x*| = %.3g (relative)" % (what, worst)
    return worst


def test_generator_is_exact():
    """x* satisfies the KKT conditions of the generated problem: stationarity with the multipliers implied by the active set, and feasibility."""
    rng = np.random.default_rng(7)
    for n in (3, 38):
        for singular_h in (False, True):
            me, rows = Q.mix(rng, n, "ineq")
            q = Q.make_qp(n, me, rows, rng, RHO, singular_h)
            assert np.array_equal(q.H, q.H.T)
            act = ~np.isnan(q.bound)
            # g + (H + rho I) x* lies in the span of the active normals, and the rest of x* is feasible with the stated gaps
            r = q.g + q.H @ q.x + RHO * q.x
            lam, *_ = np.linalg.lstsq(q.A[act].T, -r, rcond=None)
            assert np.abs(q.A[act].T @ lam + r).max() < 1e-12 * max(1.0, np.abs(r).max())
            assert max(Q.solution_error(q.x, q)) < 1e-15
            ax = q.A @ q.x
            ina = ~act & (np.abs(q.A).max(axis=1) > 0)
            gap = np.minimum(np.where(q.ub[ina] < 1e19, q.ub[ina] - ax[ina], np.inf), np.where(q.lb[ina] > -1e19, ax[ina] - q.lb[ina], np.inf))
            assert (gap >= 0.5 - 1e-12).all()
            if singular_h and act.sum() > 1:
                assert np.linalg.matrix_rank(q.H) < n


def test_case_shapes():
    """The boundary and capacity problems sit where their names say, counted the way the solver classifies rows."""
    b = Q.boundary_cases(RHO)
    shape = {k: {Q.classify(q) + (q.n,) for q in v} for k, v in b.items()}
    assert shape["n32_narrow32"] == {(2, 32, 32, 32, 32)}
    assert shape["n32_narrow33"] == {(2, 33, 33, 33, 32)}
    assert shape["n33_narrow32"] == {(2, 32, 32, 32, 33)}
    for n in (20, 38):
        for w in (8, 9):
            for q in b["n%d_span%d" % (n, w)]:
                act = ~np.isnan(q.bound) & (q.lb != q.ub)
                spans = [np.flatnonzero(a)[-1] + 1 - np.flatnonzero(a)[0] for a in q.A[act]]
                assert len(spans) == 6 and set(spans) == {w}
    for n in (20, 40):
        for q in b["n%d_two_sided_lower" % n]:
            act = ~np.isnan(q.bound) & (q.lb != q.ub)
            assert act.sum() == 6 and (q.bound[act] == q.lb[act]).all() and (q.ub[act] < 1e19).all()
    for name in ("n28_wide24", "n64_wide24"):
        for q in b[name]:
            me, entries, ordered, narrow = Q.classify(q)
            wide_active = sum(np.ptp(np.flatnonzero(a)) >= 8 for a in q.A[~np.isnan(q.bound) & (q.lb != q.ub)])
            assert ordered - narrow == 24 and wide_active > 10
    c = Q.capacity_cases(RHO)
    counts = {k: {Q.classify(q)[:2] + (q.m,) for q in v[0]} for k, v in c.items()}
    assert counts == {"eq32": {(32, 2, 34)}, "in96": {(0, 96, 96)}, "two48": {(0, 96, 48)}, "m160": {(32, 96, 160)},
                      "eq33": {(33, 2, 35)}, "in97": {(0, 97, 97)}, "two48_in1": {(0, 97, 49)}}


@pytest.mark.parametrize("n", Q.NS)
def test_envelope_oracle(oracle, n):
    for mix in Q.MIXES:
        for singular_h in (False, True):
            _solve_all(oracle, Q.envelope_cell(n, mix, singular_h, RHO), "n=%d %s singular_h=%s" % (n, mix, singular_h))


def test_boundary_oracle(oracle):
    for name, qps in Q.boundary_cases(RHO).items():
        _solve_all(oracle, qps, name)


def test_capacity_oracle(oracle):
    """Every capacity problem is feasible with a known optimum, including those beyond the CUDA solver's row capacity."""
    for name, (qps, _) in Q.capacity_cases(RHO).items():
        _solve_all(oracle, qps, name)
