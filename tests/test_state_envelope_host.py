"""The float64 oracle across the robot's state envelope (tests/state_envelope_ref.py), on the CPU: the contract the device's MPC solve is
held to there (tests/test_gpu_state_envelope.py).

Jacobians. The oracle's flow_map and ee_kinematics Jacobians are pinned against central differences with one Richardson step on every axis
and the mixed sample. With steps h = 1e-3 for x (shrunk with cos(pitch) / 0.2 near the vertical, where the higher derivatives grow like
1 / cos(pitch)) and 1e-2 for u, the truncation error is O(h^4) and stays below 1e-10 of max(1, |J|); what remains is rounding, about
eps |value| / h for a value of magnitude |value|, and eps |z| |J| / h for an argument z of magnitude |z| (sin(1e3 + h) knows h only to
eps 1e3). So the bound is 1e-9 max(1, |J|) + 16 eps (max(1, |value|) + |z| |J|) / h: 2000 times tighter than the 2e-6 of
test_oracle_rbd's plain differences at nominal states; the rounding term matters only where a coordinate or a contact position is 1e3.
Worst seen: 8e-8 (1.1e-9 of |A| = 75, five times eps |z| |A| / h) on the mixed sample's yaw-rate row at yaw and position near 1e3,
4e-10 on the contact positions at 1e3 m, below 4e-12 of max(1, |J|) on the other axes.

Invariances. Yaw enters the model only through its sine and cosine, and the model is invariant under horizontal translation. One oracle
iteration of every solve case, turned by 2 pi k (k = 1, 10, 159, +-1000) or moved by up to 1e3 m, takes the same alpha after the same
number of trials, and its solution, turned or moved back, is within 1e-10 (x) and 1e-9 (u) of max(1, |ref|) of the original's. Worst seen:
x 6.5e-12, u 4e-11.

Near the vertical. The Euler-rate map is singular at pitch = pi/2, and |A| grows like 100 / cos(pitch): 1.4e3 at pitch 1.5, 4.9e3 at 1.55,
1.3e5 at 1.57, 3.8e9 at 1.5707963 and 1.6e18 at the double nearest pi/2, with f staying near 4.8 and every entry finite. One oracle iteration from the cold
start: at 1.5 it is an ordinary step (alpha 1, status 0); at 1.55 stepping gaits back-track once (alpha 0.5); at 1.57 and 1.5707 the line
search shrinks alpha to 2^-13 or rejects every trial (alpha 0, 14 trials), still with status 0 and a finite iterate; at 1.5707963 the
direction is not finite: status 3, no trial, the iterate kept. The GPU test holds the device to that: status 0 with finite output matching
the oracle, or a non-zero status with the iterate kept."""
import numpy as np
import pytest

import state_envelope_ref as E

N, DT = 20, 0.02
EPS = np.finfo(np.float64).eps
JAC_TOL = 1e-9
YAW_TURNS = (1, 10, 159, 1000, -1000)
SHIFTS = ((1e3, 1e3), (-1e3, 250.0), (0.37, -5e2))
INV_X, INV_U = 1e-10, 1e-9


def _h(x):
    return 1e-3 * min(1.0, abs(np.cos(x[10])) / 0.2)


def _assert_jacobian(num, ana, value, z, h, what):
    err = np.abs(num - ana).max()
    bound = JAC_TOL * max(1.0, np.abs(ana).max()) + 16 * EPS * (max(1.0, np.abs(value).max()) + np.abs(z).max() * np.abs(ana).max()) / h
    assert err <= bound, (what, err, bound)


@pytest.mark.parametrize("axis", E.AXES + ("mixed",))
def test_flow_map_jacobians_vs_extrapolated_differences(axis, oracle):
    for label, x, u in E.all_points()[axis]:
        f, A, B = oracle.flow_map(x, u)
        assert np.isfinite(f).all() and np.isfinite(A).all() and np.isfinite(B).all(), label
        h = _h(x)
        _assert_jacobian(E.richardson_jacobian(lambda z: oracle.flow_map(z, u, False), x, h), A, f, x, h, (label, "A"))
        _assert_jacobian(E.richardson_jacobian(lambda z: oracle.flow_map(x, z, False), u, 1e-2), B, f, u, 1e-2, (label, "B"))


@pytest.mark.parametrize("axis", E.AXES + ("mixed",))
def test_ee_kinematics_jacobians_vs_extrapolated_differences(axis, oracle):
    for label, x, u in E.all_points()[axis]:
        pos, vel, dp, dvx, dvu = oracle.ee_kinematics(x, u)
        h = _h(x)
        _assert_jacobian(E.richardson_jacobian(lambda z: oracle.ee_kinematics(z, u)[0], x, h), dp, pos, x, h, (label, "dpos/dx"))
        _assert_jacobian(E.richardson_jacobian(lambda z: oracle.ee_kinematics(z, u)[1], x, h), dvx, vel, x, h, (label, "dvel/dx"))
        _assert_jacobian(E.richardson_jacobian(lambda z: oracle.ee_kinematics(x, z)[1], u, 1e-2), dvu, vel, u, 1e-2, (label, "dvel/du"))


def test_richardson_step_is_fourth_order():
    """The extrapolated difference of a function with known derivative: error O(h^4), far below plain central differences."""
    fn = lambda z: np.array([np.sin(3 * z[0]) * np.exp(z[1]), z[0] ** 5])
    z = np.array([0.4, -0.2])
    exact = np.array([[3 * np.cos(1.2) * np.exp(-0.2), np.sin(1.2) * np.exp(-0.2)], [5 * 0.4 ** 4, 0.0]])
    e1, e2 = (np.abs(E.richardson_jacobian(fn, z, h) - exact).max() for h in (1e-2, 5e-3))
    assert e1 < 1e-8 and 12 < e1 / e2 < 20                      # halving h divides the error by about 16


def test_axes_reach_their_extremes():
    """Each axis reaches the extremes the module docstring names, well outside random_initial_states' box, and the mixed sample spans
    them all; the solve cases start where their labels say."""
    pts = E.all_points()
    b = {a: E.bounds_of([p[1] for p in pts[a]], [p[2] for p in pts[a]]) for a in pts}
    assert b["attitude"]["pitch"] == 1.4 and b["attitude"]["roll"] == 1.4
    assert b["yaw"]["yaw"] == 1e3 and b["position"]["position"] == 1e3 and b["position"]["height"][1] == 1e3
    assert b["momentum"]["linear"] == 1.0 == b["momentum"]["angular"] == 10 * E.BOX["momentum"]
    lo, hi = b["joints"]["joints"]
    assert np.array_equal(lo, E.LOWER) and np.array_equal(hi, E.UPPER)
    assert b["joint_velocity"]["joint_velocity"] == 40.0 and b["force"]["normal_force"] == 3 * E.WEIGHT
    m = b["mixed"]
    assert m["pitch"] > 1.0 and m["yaw"] > 100 and m["position"] > 100 and m["joint_velocity"] > 5
    labels = {lab for lab, _, _ in E.axis_points("joints")}
    assert {"knees 0", "knees singular", "all joints lower", "all joints upper"} <= labels
    kn = E.singular_knees()
    assert all(0.0 < k < 0.05 for k in kn)
    cases = E.solve_cases(N, DT)
    assert {g for _, _, g, _ in cases} == set(E.GAITS)
    assert {a for a, _, _, _ in cases} == set(E.AXES) | {"mixed"}
    for axis, lab, g, c in cases:
        x0, xr, sw, md, xt, ut = c
        if lab.startswith("pitch"):
            assert x0[10] == float(lab.split()[1])
        if lab.startswith("yaw"):
            assert abs(x0[9]) >= np.pi and xr[0, 9] == x0[9]
        if axis == "position":
            assert np.abs(x0[6:8]).max() == 1e3
        if axis == "joint_velocity":
            assert np.abs(ut[:, 12:]).max() == 40.0
        if axis == "force":
            assert np.abs(ut[:, :12]).max() in (0.0, 3 * E.WEIGHT) or lab == "3mg spread"


def test_iteration_invariant_under_yaw_turns_and_horizontal_shifts(oracle):
    worst = np.zeros(4)
    for axis, lab, g, c in E.solve_cases(N, DT, oracle):
        xa, ua, ia = oracle.mpc_iteration(N, DT, *c)
        assert ia["status"] == 0, lab
        for k in YAW_TURNS:
            xb, ub, ib = oracle.mpc_iteration(N, DT, *E.yaw_turn(c, k))
            assert (ib["alpha"], ib["n_trials"], ib["status"]) == (ia["alpha"], ia["n_trials"], 0), (lab, k)
            ex, eu = E.rel(E.yaw_turn_back(xb, k), xa), E.rel(ub, ua)
            assert ex < INV_X and eu < INV_U, (lab, k, ex, eu)
            worst[:2] = np.maximum(worst[:2], (ex, eu))
        for d in SHIFTS:
            xb, ub, ib = oracle.mpc_iteration(N, DT, *E.shift(c, d))
            assert (ib["alpha"], ib["n_trials"], ib["status"]) == (ia["alpha"], ia["n_trials"], 0), (lab, d)
            ex, eu = E.rel(E.shift_back(xb, d), xa), E.rel(ub, ua)
            assert ex < INV_X and eu < INV_U, (lab, d, ex, eu)
            worst[2:] = np.maximum(worst[2:], (ex, eu))
    print("invariance: yaw turns x %.1e u %.1e, shifts x %.1e u %.1e" % tuple(worst))


def test_transforms_invert_exactly_enough():
    c = E.solve_case(E._x(yaw=0.3), "trot", N, DT)
    t = E.shift(E.yaw_turn(c, 1000), (1e3, -1e3))
    assert t[0][9] > 6000 and t[0][6] == 1e3 + c[0][6] and np.array_equal(t[2][:, 7], c[2][:, 7] - 1e3)
    back = E.shift_back(E.yaw_turn_back(t[4], 1000), (1e3, -1e3))
    assert E.rel(back, c[4]) < 1e-12 and np.array_equal(t[5], c[5]) and np.array_equal(t[3], c[3])


NEAR_VERTICAL = {1.5: (0, 1e3, 2e3), 1.55: (0, 4e3, 6e3), 1.57: (0, 1e5, 2e5), 1.5707: (0, 1e6, 2e6), 1.5707963: (3, 1e9, 1e10)}


@pytest.mark.parametrize("pitch", sorted(NEAR_VERTICAL))
def test_oracle_near_vertical_pitch(pitch, oracle):
    """The behaviour recorded in the module docstring: finite flow map with |A| near 100 / cos(pitch); one iteration either ordinary
    (status 0, finite) or, at the double-precision edge, status 3 with no trial and the iterate kept."""
    status, a_lo, a_hi = NEAR_VERTICAL[pitch]
    x = E._x(pitch=pitch)
    f, A, B = oracle.flow_map(x, E.stance_input())
    assert np.isfinite(f).all() and np.isfinite(A).all() and np.isfinite(B).all()
    assert a_lo < np.abs(A).max() < a_hi and np.abs(f).max() < 5.0
    for g in E.GAITS:
        c = E.solve_case(x, g, N, DT, oracle=oracle)
        x1, u1, info = oracle.mpc_iteration(N, DT, *c)
        assert info["status"] == status, g
        assert np.isfinite(x1).all() and np.isfinite(u1).all()
        if status:
            assert info["n_trials"] == 0 and np.array_equal(x1, c[4]) and np.array_equal(u1, c[5])
        elif pitch <= 1.5 or g == "stance":
            assert info["alpha"] == 1.0 or pitch >= 1.57, g
        if status == 0 and pitch == 1.55 and g != "stance":
            assert info["alpha"] == 0.5 and info["n_trials"] == 2, g
        if pitch >= 1.57:
            assert info["alpha"] < 0.02, g
