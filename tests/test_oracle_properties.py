"""Property tests of the oracle over random states (hypothesis): structural facts that hold for every configuration."""
import numpy as np
from hypothesis import given, settings, strategies as st

X0 = np.array([0, 0, 0, 0, 0, 0, 0, 0, 0.63, 0, 0, 0, .1, 0, .4, .93, .53, -.1, 0, -.4, .93, -.53])
LO = np.array([-0.2, -0.5, -0.8, 0.0, -1.1, -0.5, -1.0, -1.2, 0.0, -1.1])
HI = np.array([0.5, 1.0, 1.2, 1.5, 1.1, 0.2, 0.5, 0.8, 1.5, 1.1])


@settings(max_examples=25, deadline=None)
@given(st.integers(0, 10**6))
def test_rigid_body_structure(oracle, seed):
    rng = np.random.default_rng(seed)
    q = np.r_[rng.uniform(-1, 1, 3), rng.uniform(-np.pi, np.pi), rng.uniform(-0.6, 0.6, 2), rng.uniform(LO, HI)]
    v = rng.uniform(-2, 2, 16)
    r = oracle.rbd(q, v)
    M = r["M"]
    assert np.abs(M - M.T).max() < 1e-11 and np.linalg.eigvalsh(M).min() > 1e-6
    # translation block of M is m I; linear momentum rows of A equal the translation rows of M
    assert np.allclose(M[:3, :3], 12.586944 * np.eye(3), atol=1e-10)
    assert np.allclose(r["A"][:3], M[:3], atol=1e-10)
    assert np.abs(r["A"] @ v - r["h"]).max() < 1e-11
    # translating the base moves contacts and CoM rigidly and leaves M, A unchanged
    d = rng.uniform(-1, 1, 3)
    q2 = q.copy(); q2[:3] += d
    r2 = oracle.rbd(q2, v)
    assert np.abs(r2["M"] - M).max() < 1e-11 and np.abs(r2["A"] - r["A"]).max() < 1e-11
    assert np.abs(r2["cpos"].reshape(4, 3) - r["cpos"].reshape(4, 3) - d).max() < 1e-12
    # kinetic energy identity 1/2 v'Mv >= 1/2 |h_lin|^2 / m (Koenig)
    assert 0.5 * v @ M @ v >= 0.5 * (r["h"][:3] @ r["h"][:3]) / 12.586944 - 1e-9


@settings(max_examples=10, deadline=None)
@given(st.integers(0, 10**6), st.sampled_from([0, 1, 2, 3]))
def test_wbc_solution_satisfies_reference_constraints(oracle, seed, mode):
    rng = np.random.default_rng(seed)
    x = X0 + rng.uniform(-.05, .05, 22)
    u = np.zeros(22)
    fl = [mode in (2, 3), mode in (1, 3), mode in (2, 3), mode in (1, 3)]
    for c in range(4):
        if fl[c]:
            u[3 * c + 2] = 12.586944 * 9.81 / sum(fl)
    q = x[6:] + rng.uniform(-.02, .02, 16)
    rbd = np.r_[q[3:6], q[0:3], q[6:], rng.uniform(-.3, .3, 16)]
    H, g, A, lb, ub = oracle.wbc_assemble(x, u, rbd, mode, False)
    sol, stt, _ = oracle.qp_solve(H, g, A, lb, ub, 1e-8)
    assert stt == 0
    Ax = A @ sol
    assert (Ax <= ub + 1e-7 * (1 + np.abs(ub))).all() and (Ax >= lb - 1e-7 * (1 + np.abs(lb))).all()
    for c in range(4):
        if not fl[c]:
            assert np.abs(sol[16 + 3 * c:19 + 3 * c]).max() < 1e-8


def test_foot_wrench_matrix_loses_rank_inside_the_knee_limits(oracle):
    """The premise of the observer's near-singular sweep (test_gpu_estimator_envelope.py): each leg's S J_foot' (5 x 6) loses rank at one
    knee angle k* strictly inside the knee's limits (the 5 mm forward offset of the ankle origin puts the hip-pitch, knee and ankle
    origins in line there), and k* does not depend on the hip pitch or the ankle."""
    from oracle import refs as R
    q0 = np.r_[X0[6:9], X0[9:12], X0[12:]]
    for leg in (0, 1):
        ks = []
        for hp, ank in ((X0[12 + 5 * leg + 2], X0[12 + 5 * leg + 4]), (-0.4, 0.6), (0.3, -0.5), (0.9, 0.0)):
            q = q0.copy(); q[6 + 5 * leg + 2] = hp; q[6 + 5 * leg + 4] = ank
            k = R.singular_knee(leg, q)
            q[6 + 5 * leg + 3] = k
            s = np.linalg.svd(R.foot_wrench_matrix(q, leg), compute_uv=False)
            assert s[-1] / s[0] < 1e-10, (leg, hp, ank, s)
            ks.append(k)
        assert LO[5 * leg + 3] < min(ks) and max(ks) < HI[5 * leg + 3], ks
        assert max(ks) - min(ks) < 1e-8, ks
        # away from k* the matrix has full rank: cond ~ 20 at the default knee, ~ 880 at knee 0
        q = q0.copy()
        assert np.linalg.cond(R.foot_wrench_matrix(q, leg)) < 100


def test_event_time_grid_restatement_properties():
    """scenarios.event_time_grid is the numpy side of row S1's parity test (ocs2::timeDiscretizationWithEvents with the event node pair collapsed):
    first node t0, last node t0 + T, strictly increasing, no step longer than dt, every mode switch strictly inside the horizon is a node, the grid
    re-anchors at a switch (the step after it is a full dt again), the uniform case is reproduced, and the capacity is respected."""
    from hunter_bipedal_control_b200 import scenarios as sc
    rng = np.random.default_rng(12)
    dt, T = 0.015, 0.8
    for trial in range(200):
        t0 = float(rng.uniform(0.0, 1.0))
        ev = np.sort(rng.uniform(t0 - 0.2, t0 + T + 0.2, rng.integers(0, 9)))
        g = sc.event_time_grid(t0, T, dt, list(ev), 96)
        assert g[0] == t0 and abs(g[-1] - (t0 + T)) < 1e-12
        d = np.diff(g)
        assert (d > 1e-9).all() and (d < dt + 1e-12).all()
        inside = [e for e in ev if t0 + 1e-9 < e < t0 + T - 1e-9]
        for e in inside:
            k = int(np.argmin(np.abs(g - e)))
            assert abs(g[k] - e) < 1e-12
            if k + 1 < len(g) - 1 and not any(abs(g[k + 1] - f) < 1e-12 for f in inside):
                assert abs(g[k + 1] - g[k] - dt) < 1e-12            # re-anchored: a full step follows the event node
        assert len(g) - 1 <= int(np.ceil(T / dt)) + len(inside) + 1
    # no events: the uniform grid (0.8 / 0.015 is not an integer: the last interval is the remainder)
    g = sc.event_time_grid(0.0, T, dt, [], 96)
    assert len(g) == 55 and np.allclose(np.diff(g)[:-1], dt) and abs(g[-1] - T) < 1e-12
    # capacity exhausted: the last interval is stretched to the final time, the node count stays within the capacity
    g = sc.event_time_grid(0.0, T, dt, [0.1003, 0.2007, 0.3001], 40)
    assert len(g) - 1 == 40 and abs(g[-1] - T) < 1e-12 and (np.diff(g) > 0).all()
