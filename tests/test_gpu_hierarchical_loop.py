"""HierarchicalWbc in the closed loop: the per-context WBC choice (hb_wbc_set_formulation) and the fused cascade kernel behind
hb_hierarchical_wbc_solve_batch. The fused kernel is checked against the composition it replaced (hb_hierarchical_wbc_tasks_batch +
hb_hoqp_solve_batch) and against the oracle; the entry points that run the controller's WBC are checked bit for bit against the stepwise
loop of existing calls under the hierarchical formulation."""
import ctypes as C
import os

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from episode_ref import (GAITS, assert_continues, assert_episode_equal, cmd_vels, context, device, est_params, launch_coefficients, params,
                         start_states, stepwise)

pytestmark = pytest.mark.gpu

N, DT = 40, 0.02


def _wbc_cases(B, seed):
    """States perturbed as in test_gpu_hoqp: all four modes, forces sharing the weight over the stance contacts."""
    rng = np.random.default_rng(seed)
    mode = np.array([3, 2, 1, 0] * ((B + 3) // 4), dtype=np.int32)[:B]
    x = np.tile(sc.INITIAL_STATE, (B, 1)) + rng.uniform(-.04, .04, (B, 22))
    u = np.zeros((B, 22))
    for i in range(B):
        fl = sc.mode_flags(int(mode[i]))
        for c in range(4):
            if fl[c]:
                u[i, 3 * c + 2] = sc.TOTAL_MASS * 9.81 / max(1, sum(fl))
        u[i, 12:] = rng.uniform(-.3, .3, 10)
    rbd = sc.consistent_rbd(x, rng, 0.01)
    return x, u, rbd, mode


def _settings(ctx, **kw):
    s = ctx.wbc_settings()
    for k, v in kw.items():
        if k == "torque_limits":
            for j in range(5):
                s.torque_limits[j] = v[j]
        else:
            setattr(s, k, v)
    ctx.set_wbc_settings(s)
    return s


NON_DEFAULT = dict(friction_coefficient=0.5, swing_kp=250.0, swing_kd=30.0, base_height_kp=80.0, base_angular_kp=60.0,
                   torque_limits=(40.0, 50.0, 45.0, 60.0, 20.0))


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


def _check_levels(s, tasks, levels_sol=None):
    """The criteria of test_hierarchical_wbc_tasks_and_solution_vs_oracle for one solution s against reference tasks (device or oracle)
    and a reference solution per level."""
    (a0, b0, d0, f0), (a1, b1, _, _), (a2, b2, _, _) = tasks
    r0, r1, r2 = levels_sol
    assert np.abs(a0 @ s - a0 @ r0).max() < 1e-5 * max(1.0, np.abs(b0).max())
    assert np.abs(a0[:16] @ s - b0[:16]).max() < 1e-4
    assert np.all(d0 @ s <= f0 + 1e-4)
    assert np.abs(a1 @ s - a1 @ r1).max() < 1e-5
    assert np.abs(a2 @ s - a2 @ r2).max() < 1e-4 * max(1.0, np.abs(a2 @ r2).max())
    assert _rel(s[28:], r2[28:]) < 1e-4


@pytest.mark.parametrize("settings", ["default", "non_default"])
def test_fused_equals_composition_and_oracle(oracle, settings):
    from oracle.hoqp import hierarchical_wbc
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=16, device=0)
    if settings == "non_default":
        _settings(ctx, **NON_DEFAULT)
    B = 16
    x, u, rbd, mode = _wbc_cases(B, 5)
    sol, st = ctx.hierarchical_wbc_solve(x, u, rbd, mode)
    pbs = ctx.hierarchical_wbc_tasks(x, u, rbd, mode)
    xc, _, stc = ctx.hoqp_solve(pbs)
    assert (st == 0).all() and (stc == 0).all(), (st, stc)
    worst = 0.0
    for i in range(B):
        tasks = hb.hoqp_tasks(pbs[i])
        _check_levels(sol[i], tasks, (xc[i], xc[i], xc[i]))
        worst = max(worst, _rel(sol[i], xc[i]))
        if settings == "default":
            so, levels, otasks = hierarchical_wbc(x[i], u[i], rbd[i], int(mode[i]))
            ot = [(t.a, t.b, t.d, t.f) for t in otasks]
            _check_levels(sol[i], ot, (levels[0].solution(), levels[1].solution(), so))
    print("largest fused-versus-composition difference (relative, whole solution): %.3e" % worst)
    ctx.close()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def test_task_weights_do_not_change_the_hierarchical_solution():
    """HierarchicalWbc has no task weights: its tasks are the unweighted rows, so the weighted formulation's weights leave its problems
    and its solution bit for bit unchanged."""
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=8, device=0)
    x, u, rbd, mode = _wbc_cases(8, 6)
    s0, st0 = ctx.hierarchical_wbc_solve(x, u, rbd, mode)
    t0 = [hb.hoqp_tasks(p) for p in ctx.hierarchical_wbc_tasks(x, u, rbd, mode)]
    _settings(ctx, weight_swing_leg=ctx.wbc_settings().weight_swing_leg * 7.0, weight_base_accel=ctx.wbc_settings().weight_base_accel * 0.3)
    s1, st1 = ctx.hierarchical_wbc_solve(x, u, rbd, mode)
    t1 = [hb.hoqp_tasks(p) for p in ctx.hierarchical_wbc_tasks(x, u, rbd, mode)]
    assert (st0 == 0).all() and (st1 == 0).all()
    assert np.array_equal(_bits(s1), _bits(s0)) and np.array_equal(st1, st0)
    for i in range(8):
        for lvl in range(3):
            for k in range(4):
                assert np.array_equal(_bits(t1[i][lvl][k]), _bits(t0[i][lvl][k])), (i, lvl, k)
    ctx.close()


@pytest.mark.parametrize("settings", ["default", "non_default"])
def test_weighted_constraints_are_the_hierarchical_task0_rows(settings):
    """WeightedWbc's constraints and HierarchicalWbc's task0 come from the same task functions: the equality rows of
    hb_wbc_assemble_batch (EoM, zero swing forces) and its inequality rows (torque limits, friction pyramid) equal, bit for bit and in
    order, the first 16 + 3 nsw equalities and all the inequalities of task0 of hb_hierarchical_wbc_tasks_batch, in every mode, with and
    without stance mode."""
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=8, device=0)
    if settings == "non_default":
        _settings(ctx, **NON_DEFAULT)
    x, u, rbd, mode = _wbc_cases(8, 9)
    _, _, A, lb, ub, m = ctx.wbc_assemble(x, u, rbd, mode, stance_mode=(np.arange(8) // 4) % 2)
    pbs = ctx.hierarchical_wbc_tasks(x, u, rbd, mode)
    for i in range(8):
        a0, b0, d0, f0 = hb.hoqp_tasks(pbs[i])[0]
        nsw = 4 - sum(sc.mode_flags(int(mode[i])))
        eq, md0 = 16 + 3 * nsw, d0.shape[0]
        assert m[i] == eq + md0 + 3 * nsw, i
        assert np.array_equal(_bits(A[i, :eq]), _bits(a0[:eq])), i
        assert np.array_equal(_bits(lb[i, :eq]), _bits(b0[:eq])) and np.array_equal(_bits(ub[i, :eq]), _bits(b0[:eq])), i
        assert np.array_equal(_bits(A[i, eq:eq + md0]), _bits(d0)), i
        assert np.array_equal(_bits(ub[i, eq:eq + md0]), _bits(f0)) and (lb[i, eq:eq + md0] == -1e20).all(), i
    ctx.close()


def test_instance_alone_equals_its_copy_in_a_large_batch():
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=1025, device=0)
    x, u, rbd, mode = _wbc_cases(1025, 7)
    big, stb = ctx.hierarchical_wbc_solve(x, u, rbd, mode)
    for k in (1000, 1003):
        one, st1 = ctx.hierarchical_wbc_solve(x[k:k + 1], u[k:k + 1], rbd[k:k + 1], mode[k:k + 1])
        assert np.array_equal(one[0], big[k]) and st1[0] == stb[k]
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- the setting
def _resident_setup(B, seed=41):
    x0 = sc.random_initial_states(B, seed=seed)
    gaits = [["trot", "standing_trot", "flying_trot", "stance"][i % 4] for i in range(B)]
    compacts = [sc.make_reference(x0[i], (0.3, 0.0, 0.0, 0.1), gaits[i], N, DT, phase=0.03 * i)[3] for i in range(B)]
    return x0, sc.pack_references(compacts, 2 * N * DT), sc.consistent_rbd(x0)


def _resident_run(ctx, B=8):
    x0, refs, rbd = _resident_setup(B)
    t0 = np.zeros(B)
    cyc0 = ctx.resident_cycle(True, 0.002, t0, x0, refs, rbd)
    cyc1 = ctx.resident_cycle(False, 0.002, t0 + DT, x0 + 1e-3, refs, rbd)
    tick = ctx.resident_wbc(t0 + DT + 0.004, rbd)
    return cyc0 + cyc1 + tick


def test_formulation_setting():
    ctx = hb.Context(horizon_N=N, dt=DT, max_batch=8, device=0)
    lib = hb.load_library()
    assert ctx.wbc_formulation() == "weighted"
    f = C.c_int32(-7)
    assert lib.hb_wbc_get_formulation(ctx._h, C.byref(f)) == 0 and f.value == hb.api.HB_WBC_WEIGHTED
    for bad in (-1, 2, 7):
        assert lib.hb_wbc_set_formulation(ctx._h, C.c_int32(bad)) == -1
        assert ctx.wbc_formulation() == "weighted"
    ctx.set_wbc_formulation("hierarchical")
    assert lib.hb_wbc_set_formulation(ctx._h, C.c_int32(5)) == -1 and ctx.wbc_formulation() == "hierarchical"
    # settings, gains and task.info leave the choice as it is
    _settings(ctx, swing_kp=300.0)
    ctx.set_kp_kd(350.0, 37.0)
    ctx.load_task_info(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "task_wbc_variant.info"))
    assert ctx.wbc_formulation() == "hierarchical"
    with pytest.raises(ValueError):
        ctx.set_wbc_formulation("weighed")
    assert lib.hb_wbc_set_formulation(None, C.c_int32(0)) == -1 and lib.hb_wbc_get_formulation(ctx._h, None) == -1
    ctx.close()


def test_switching_back_to_weighted_is_bitwise_a_context_never_switched():
    a = hb.Context(horizon_N=N, dt=DT, max_batch=8, device=0)
    b = hb.Context(horizon_N=N, dt=DT, max_batch=8, device=0)
    b.set_wbc_formulation("hierarchical")
    b.set_wbc_formulation("weighted")
    for x, y in zip(_resident_run(a), _resident_run(b)):
        x, y = np.asarray(x), np.asarray(y)
        if x.dtype.names:
            for k in x.dtype.names:
                assert np.array_equal(x[k], y[k]), k
        else:
            assert np.array_equal(x, y)
    a.close(); b.close()
    ea, eb = context(), context()
    eb.set_wbc_formulation("hierarchical"); eb.set_wbc_formulation("weighted")
    rbd0 = start_states(ea, 4, seed=21)
    prm = params(5)
    assert_episode_equal(device(ea, rbd0, GAITS[:4], cmd_vels(4), 40, prm, 5), device(eb, rbd0, GAITS[:4], cmd_vels(4), 40, prm, 5))
    ea.close(); eb.close()


# ---------------------------------------------------------------------------------------------------------------- the resident tick
def test_resident_tick_under_hierarchical():
    B = 8
    w = hb.Context(horizon_N=N, dt=DT, max_batch=B, device=0)
    h = hb.Context(horizon_N=N, dt=DT, max_batch=B, device=0)
    h.set_wbc_formulation("hierarchical")
    x0, refs, rbd = _resident_setup(B)
    t0 = np.zeros(B)
    _, sol_w0, _, _ = w.resident_cycle(True, 0.002, t0, x0, refs, rbd)
    info, sol_h0, tau_h0, st_h0 = h.resident_cycle(True, 0.002, t0, x0, refs, rbd)
    assert (st_h0 == 0).all(), st_h0
    assert np.array_equal(tau_h0, sol_h0[:, 28:]) and not np.array_equal(sol_w0, sol_h0)
    t = t0 + 0.006
    xw, uw, mw, _, _, _ = w.resident_wbc(t, rbd)
    xh, uh, mh, sol, tau, st = h.resident_wbc(t, rbd)
    assert np.array_equal(xw, xh) and np.array_equal(uw, uh) and np.array_equal(mw, mh)
    ref, st_ref = h.hierarchical_wbc_solve(xh, uh, rbd, mh)
    assert (st == 0).all() and np.array_equal(st, st_ref)
    assert np.array_equal(sol, ref) and np.array_equal(tau, sol[:, 28:])
    for sm in (np.zeros(B, np.uint8), np.ones(B, np.uint8)):
        o = h.resident_wbc(t, rbd, stance_mode=sm)
        for p, q in zip(o, (xh, uh, mh, sol, tau, st)):
            assert np.array_equal(p, q)
    w.close(); h.close()


def test_resident_fallback_under_hierarchical():
    """An iteration cap of one (two interior-point iterations per level) fails every cascade. After a cold start the cycle returns the
    unsolved iterate (no previous solution); every later tick returns the previous solution and its torques."""
    B = 4
    h = hb.Context(horizon_N=N, dt=DT, max_batch=B, device=0, qp_max_iter=1)
    h.set_wbc_formulation("hierarchical")
    x0, refs, rbd = _resident_setup(B)
    t0 = np.zeros(B)
    _, sol0, tau0, st0 = h.resident_cycle(True, 0.002, t0, x0, refs, rbd)
    assert (st0 != 0).all(), st0
    xd, ud, md, sol_same, _, _ = h.resident_wbc(t0 + 0.002, rbd)
    raw, st_raw = h.hierarchical_wbc_solve(xd, ud, rbd, md)
    assert (st_raw != 0).all() and np.array_equal(sol0, raw)              # cold start: the iterate itself
    xd, ud, md, sol1, tau1, st1 = h.resident_wbc(t0 + 0.006, rbd)
    raw1, _ = h.hierarchical_wbc_solve(xd, ud, rbd, md)
    assert (st1 != 0).all() and not np.array_equal(raw1, sol0)
    assert np.array_equal(sol1, sol0) and np.array_equal(tau1, sol0[:, 28:])
    h.close()


# ---------------------------------------------------------------------------------------------------------------- episodes
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
@pytest.mark.parametrize("estimator", [False, True], ids=["truth", "estimator"])
def test_hierarchical_episode_equals_the_stepwise_loop_bitwise(event_nodes, estimator):
    ctx = context(event_nodes)
    ctx.set_wbc_formulation("hierarchical")
    B, n_ticks, log_every = 6, 100, 10
    rbd0 = start_states(ctx, B, seed=11)
    vels = cmd_vels(B)
    prm = params(log_every)
    ep = est_params(seed=2024) if estimator else None
    est = (lambda: hb.estimation_states(B, 40)) if estimator else (lambda: None)
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, est())
    r = stepwise(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, est())
    assert_episode_equal(d, r)
    assert np.isfinite(r[0]).all()
    ctx.close()


def test_hierarchical_pushed_episode_equals_the_stepwise_loop_bitwise():
    ctx = context()
    ctx.set_wbc_formulation("hierarchical")
    B, n_ticks = 6, 80
    rbd0 = start_states(ctx, B, seed=14)
    vels = cmd_vels(B)
    prm = params(5)
    S = hb.make_push_schedules(B, 0.04, 0.05, [[30.0, -20.0, 0.0]])
    ctx.set_pushes(S)
    assert_episode_equal(device(ctx, rbd0, GAITS, vels, n_ticks, prm, 5), stepwise(ctx, rbd0, GAITS, vels, n_ticks, prm, 5, pushes=S))
    ctx.close()


@pytest.mark.parametrize("estimator", [False, True], ids=["truth", "estimator"])
def test_hierarchical_two_calls_continue_one_call_and_launch_like_weighted(estimator):
    ep = est_params(seed=5) if estimator else None
    counts = {}
    for form in ("weighted", "hierarchical"):
        ctx = context()
        ctx.set_wbc_formulation(form)
        rbd0 = start_states(ctx, 6, seed=12)
        if form == "hierarchical":
            assert_continues(ctx, rbd0, GAITS, cmd_vels(6), 100, 50, params(10), 10, ep)
        counts[form] = launch_coefficients(ctx, rbd0, GAITS, cmd_vels(6), params(), ep)
        ctx.close()
    assert counts["weighted"] == counts["hierarchical"], counts
