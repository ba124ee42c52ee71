"""The time axis restated from OCS2 (tests/time_axis_ref.py) against the grid the repository documents (scenarios.event_time_grid, the
rule time_grid_kernel runs): bit for bit on the edge cases where a grid goes wrong and on random schedules, the grid's properties, and
the places where the repository departs from OCS2 on purpose."""
import numpy as np
import pytest

from hunter_bipedal_control_b200 import scenarios as sc
import time_axis_ref as TA

DT, T = 0.015, 0.8


def _steps(t0, dt, n):
    """The first n node times t0 + dt + dt ... as the grid computes them (one addition per step)."""
    out, t = [], t0
    for _ in range(n):
        t = t + dt
        out.append(t)
    return out


def edge_cases():
    """(name, t0, T, dt, events, capacity): events on, near and between the steps, at and around t0 and tf, many events, short horizons,
    the capacity reached and exceeded."""
    t0 = 0.35
    s = _steps(t0, DT, 60)
    tf = t0 + T
    cases = []
    for k in (3, 17):
        for d in (0.0, 1e-12, -1e-12, 1e-9, -1e-9, 2e-9, -2e-9):
            cases.append(("step%d%+g" % (k, d), t0, T, DT, [s[k] + d], 64))
    cases += [
        ("two_in_one_dt", t0, T, DT, [s[4] + 0.003, s[4] + 0.011], 64),
        ("three_in_one_dt", t0, T, DT, [s[4] + 0.002, s[4] + 0.006, s[4] + 0.013], 64),
        ("coincident", t0, T, DT, [s[6] + 0.004, s[6] + 0.004, s[9]], 64),
        ("closer_than_dt_min", t0, T, DT, [s[6] + 0.004, s[6] + 0.004 + 5e-10, s[9] + 0.001, s[9] + 0.001 + 1e-9], 64),
        ("at_t0", t0, T, DT, [t0, s[5] + 0.001], 64),
        ("t0_plus_1e-12", t0, T, DT, [t0 + 1e-12], 64),
        ("t0_plus_1e-9", t0, T, DT, [t0 + 1e-9], 64),
        ("t0_plus_2e-9", t0, T, DT, [t0 + 2e-9], 64),
        ("before_t0", t0, T, DT, [t0 - 0.2, t0 - 1e-9, s[2] + 0.005], 64),
        ("at_tf", t0, T, DT, [s[10] + 0.002, tf], 64),
        ("tf_minus_1e-9", t0, T, DT, [tf - 1e-9], 64),
        ("after_tf", t0, T, DT, [s[10] + 0.002, tf + 1e-12, tf + 0.01], 64),
        ("max_events", t0, T, DT, list(t0 + 0.003 + 0.0245 * np.arange(32)), 96),
        ("T_not_multiple", t0, 0.1234, DT, [s[2] + 0.004], 16),
        ("T_below_dt", t0, 0.01, DT, [t0 + 0.004], 4),
        ("T_below_dt_min", t0, 5e-10, DT, [], 4),
        ("N1", t0, 0.01, DT, [t0 + 0.004], 1),
        ("N2", t0, 0.01, DT, [t0 + 0.004], 2),
    ]
    ev = [s[2] + 0.004, s[20] + 0.001, s[33] + 0.009]
    n_full = len(sc.event_time_grid(t0, T, DT, ev, 512)) - 1
    cases += [("capacity_exact", t0, T, DT, ev, n_full), ("capacity_plus_one", t0, T, DT, ev, n_full - 1),
              ("capacity_33", t0, T, DT, ev, 33), ("capacity_512", t0, 2.5, 0.005, ev + [t0 + 1.3, t0 + 2.2], 512)]
    return cases


CASES = edge_cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_restated_grid_equals_the_documented_grid_on_edge_cases(case):
    _, t0, T_, dt, events, cap = case
    g, st = TA.event_node_grid(t0, T_, dt, sorted(events), cap)
    ref = sc.event_time_grid(t0, T_, dt, sorted(events), cap)
    assert np.array_equal(g, ref), (g, ref)
    _assert_properties(g, st, t0, T_, dt, sorted(events), cap)


def _assert_properties(g, st, t0, T_, dt, events, cap):
    tf = t0 + T_
    d = np.diff(g)
    assert g[0] == t0 and g[-1] == tf and 1 <= len(g) - 1 <= cap
    if st == 0:
        # at most dt, plus up to dt_min for each switch a node moved forward onto when merged, plus rounding of the differences
        assert (d <= dt + (len(events) + 1) * TA.DT_MIN + 1e-12).all() and ((d > TA.DT_MIN).all() or T_ <= TA.DT_MIN), d
        for e in events:   # every switch strictly inside the horizon is a node, or merged into one at most dt_min per later switch away
            if t0 + TA.DT_MIN < e < tf:
                assert e in g or np.any((g > e) & (g - e <= 1.000001 * len(events) * TA.DT_MIN)), e
    else:                                                   # capacity exhausted: every interval but the stretched last one as usual
        assert len(g) - 1 == cap and (d[:-1] <= dt + (len(events) + 1) * TA.DT_MIN + 1e-12).all() and (d[:-1] > TA.DT_MIN).all() and d[-1] > 0.0


def test_capacity_rule():
    by_name = {c[0]: c for c in CASES}
    for name, status in (("capacity_exact", 0), ("capacity_plus_one", 1), ("N1", 1), ("N2", 0)):
        _, t0, T_, dt, events, cap = by_name[name]
        g, st = TA.event_node_grid(t0, T_, dt, events, cap)
        assert st == status and len(g) - 1 == cap and g[-1] == t0 + T_, name


def test_restated_grid_equals_the_documented_grid_on_random_schedules():
    rng = np.random.default_rng(2024)
    for it in range(2000):
        t0 = float(rng.uniform(0.0, 3.0))
        dt = float(rng.choice([0.005, 0.01, 0.015, rng.uniform(0.002, 0.03)]))
        T_ = float(rng.choice([0.8, rng.uniform(0.0005, 1.2)]))
        cap = int(rng.integers(1, 200))
        ne = int(rng.integers(0, 33))
        ev = np.sort(rng.uniform(t0 - 0.3, t0 + T_ + 0.3, ne))
        # some events exactly on steps, on t0, on tf, or near one another
        steps = _steps(t0, dt, 8)
        for j in range(ne):
            r = rng.integers(0, 8)
            if r == 0:
                ev[j] = steps[rng.integers(0, 8)] + rng.choice([0.0, 1e-12, -1e-12, 1e-9, 2e-9, -2e-9])
            elif r == 1:
                ev[j] = t0 + rng.choice([0.0, 1e-12, 1e-9, 2e-9])
            elif r == 2:
                ev[j] = t0 + T_ + rng.choice([0.0, -1e-9, 1e-12])
            elif r == 3 and j > 0:
                ev[j] = ev[j - 1] + rng.choice([0.0, 5e-10, 1e-9, 3e-9])
        ev = sorted(ev.tolist())
        g, st = TA.event_node_grid(t0, T_, dt, ev, cap)
        assert np.array_equal(g, sc.event_time_grid(t0, T_, dt, ev, cap)), (it, t0, T_, dt, ev, cap)
        _assert_properties(g, st, t0, T_, dt, ev, cap)


def test_ocs2_discretisation_and_the_repository_rules():
    """Where the repository departs from OCS2's grid on purpose, and nowhere else: with no switch within dt_min after t0, a horizon
    longer than dt_min and enough capacity, the collapsed OCS2 grid is the repository's grid."""
    t0 = 0.35
    s = _steps(t0, DT, 60)
    ann = TA.time_discretization_with_events(t0, t0 + T, DT, [s[3], s[7] + 0.004])
    assert [e for _, e in ann].count(TA.PRE_EVENT) == 2 and [e for _, e in ann].count(TA.POST_EVENT) == 2
    assert np.array_equal(TA.collapse_event_pairs(ann), TA.event_node_grid(t0, T, DT, [s[3], s[7] + 0.004], 64)[0])
    # rule 1: a switch at t0 is the same in both; one within dt_min after t0 moves OCS2's node 0, not the repository's
    assert np.array_equal(TA.collapse_event_pairs(TA.time_discretization_with_events(t0, t0 + T, DT, [t0])), TA.event_node_grid(t0, T, DT, [t0], 64)[0])
    moved = TA.collapse_event_pairs(TA.time_discretization_with_events(t0, t0 + T, DT, [t0 + 5e-10]))
    kept = TA.event_node_grid(t0, T, DT, [t0 + 5e-10], 64)[0]
    assert moved[0] == t0 + 5e-10 and kept[0] == t0 and len(moved) == len(kept)
    # and the switch is in force on the first interval either way
    assert TA.interval_mode([t0 + 5e-10], [3, 1], kept[0]) == 1
    # rule 2: a horizon within dt_min
    assert len(TA.collapse_event_pairs(TA.time_discretization_with_events(t0, t0 + 5e-10, DT, []))) == 1
    assert np.array_equal(TA.event_node_grid(t0, 5e-10, DT, [], 4)[0], [t0, t0 + 5e-10])


def test_policy_and_warm_start_restatements_on_known_answers():
    times = np.array([1.0, 1.01, 1.015, 1.03])
    x = np.arange(4.0)[:, None] * np.ones((1, 22))
    u = 10.0 + np.arange(3.0)[:, None] * np.ones((1, 22))
    md = np.array([3, 2, 1, 1])
    # inside an interval, on an interior node (the interval ending there), before t0 and past the end (clamped)
    for t, xe, ue, me in ((1.005, 0.5, 10.5, 3), (1.01, 1.0, 11.0, 3), (1.0125, 1.5, 11.5, 2), (0.9, 0.0, 10.0, 3), (1.2, 3.0, 12.0, 1),
                          (1.03, 3.0, 12.0, 1)):
        xs, us, m = TA.evaluate_policy(times, x, u, md, t)
        assert np.allclose(xs, xe, rtol=0, atol=1e-13) and np.allclose(us, ue, rtol=0, atol=1e-13) and m == me, t
    assert TA.mode_at_time([1.01, 1.015], [3, 2, 1], 1.01) == 3 and TA.mode_at_time([1.01, 1.015], [3, 2, 1], 1.0100001) == 2
    # warm start: the same grid gives back the previous solution (x[0] measured); a shift past the end gives the initializer everywhere
    x0 = np.full(22, 7.0)
    xw, uw = TA.warm_start(times, x, u, times, x0, md, 12.586944)
    assert np.array_equal(xw[0], x0) and np.allclose(xw[1:], x[1:], atol=1e-15) and np.allclose(uw, u, atol=1e-14)
    xw, uw = TA.warm_start(times, x, u, times + 0.04, x0, md, 12.586944)
    assert (xw == 7.0).all() and uw[0, 2] == uw[0, 8] == 12.586944 * 9.81 / 4 and uw[1, 2] == 12.586944 * 9.81 / 2 and uw[1, 5] == 0.0
    # the 1e-9 guard: a new node within 1e-9 past the previous end still interpolates (the end, clamped), one 2e-9 past it does not
    xw, _ = TA.warm_start(times, x, u, np.array([1.0, 1.03 + 1e-9]), x0, md, 1.0)
    assert np.array_equal(xw[1], x[3])
    xw, _ = TA.warm_start(times, x, u, np.array([1.0, 1.03 + 2e-9]), x0, md, 1.0)
    assert np.array_equal(xw[1], x0)
