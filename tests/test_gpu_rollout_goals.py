"""Goals (hb_rollout_set_goals) and explicit planner targets (hb_plan_set_targets) on the device. The device planner on explicit targets is
checked against the host planner on the same targets; the goal episode bit for bit against the loop of public calls (episode_ref.stepwise:
hb_goal_to_target on the MPC tick a goal comes into force, hb_plan_set_targets, hb_resident_plan_cycle_batch), under both WBC formulations,
truth and estimator, both time grids, together with pushes, plant variations and terrains; then the setting's contract (continuation across a
split between a goal's time and its capture, independence, permutation, instances beyond the setting, re-capture on a new setting, zero-goal
schedules, launch counts, argument checks) and one closed-loop property of trotting robots sent to goals."""
import ctypes as C

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from episode_ref import (FRICTION, GAITS, PUSH, assert_continues, assert_episode_equal, assert_null_settings, assert_rejected_settings,
                         assert_setting_episodes, cmd_vels, context, device, est_params, launch_coefficients, outputs, params, random_goals, start_states,
                         stepwise, use)

pytestmark = pytest.mark.gpu

N, DT = 40, 0.02
T = N * DT


def _plan_cases(n, seed):
    rng = np.random.default_rng(seed)
    x0 = sc.random_initial_states(n, seed=seed)
    gaits = [["trot", "standing_trot", "flying_trot", "stance"][i % 4] for i in range(n)]
    cmd = np.stack([rng.uniform(-0.6, 0.8, n), rng.uniform(-0.2, 0.2, n), np.zeros(n), rng.uniform(-0.5, 0.5, n)], axis=1)
    t0 = rng.uniform(0.0, 3.0, n)
    start = t0 + rng.uniform(-1.3, 0.3, n)
    feet = x0[:, None, 6:9] + rng.normal(0, 0.1, (n, 4, 3))
    feet[:, :, 2] = 0.02
    latest = feet + rng.normal(0, 0.02, feet.shape)
    goal = np.c_[x0[:, 6:8] + rng.uniform(-1.0, 1.0, (n, 2)), x0[:, 9] + rng.uniform(-1.0, 1.0, n)]
    return x0, gaits, cmd, t0, start, feet.reshape(n, 12), latest.reshape(n, 12), goal


def _fields(r):
    ne, nt = r.n_events, r.n_targets
    segs = [[np.array([list(r.segments[c][a][k][:]) for k in range(r.n_segments[c][a])]).reshape(-1, 6) for a in range(3)] for c in range(4)]
    return (ne, nt, np.array(r.event_times[:ne]), np.array(r.modes[:ne + 1]), np.array(r.target_times[:nt]),
            np.array([list(r.target_states[k][:]) for k in range(nt)]), segs)


def _assert_plans_match(rd, rh, exact_targets):
    """The device plan rd against the host plan rh with the tolerances of the planner's device / host parity (the device contracts
    products into fused multiply-adds); the schedule exactly, and the target samples exactly when they are the given ones."""
    for i in range(len(rd)):
        a, b = _fields(rd[i]), _fields(rh[i])
        assert a[0] == b[0] and a[1] == b[1]
        np.testing.assert_array_equal(a[2], b[2])
        np.testing.assert_array_equal(a[3], b[3])
        if exact_targets:
            np.testing.assert_array_equal(a[4], b[4]); np.testing.assert_array_equal(a[5], b[5])
        else:
            np.testing.assert_allclose(a[4], b[4], rtol=0, atol=1e-12)
            np.testing.assert_allclose(a[5], b[5], rtol=0, atol=1e-8)
        for c in range(4):
            for ax in range(3):
                assert a[6][c][ax].shape == b[6][c][ax].shape
                np.testing.assert_allclose(a[6][c][ax], b[6][c][ax], rtol=0, atol=1e-11)


@pytest.mark.parametrize("joint_ik", [False, True], ids=["two_sample", "ik"])
def test_device_planner_on_targets_matches_the_host_planner(joint_ik):
    ctx = hb.Context(horizon_N=N, dt=DT, max_batch=128, device=0)
    n = 96
    x0, gaits, cmd, t0, start, feet, latest, goal = _plan_cases(n, 61)
    tg = hb.goal_to_target(t0, x0, goal)
    ins = hb.make_plan_inputs(t0, T, x0, cmd, feet, gaits, start, joint_ik=joint_ik)
    plain_d, ls_plain, st = ctx.plan_references_gpu(ins, latest)
    ctx.set_plan_targets(tg)
    rd, lsd, st = ctx.plan_references_gpu(ins, latest)
    rh, lsh = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, joint_ik=joint_ik, targets=tg)
    assert (st == 0).all()
    np.testing.assert_allclose(lsd, lsh, rtol=0, atol=1e-14)
    _assert_plans_match(rd, rh, not joint_ik)
    # targets for the first k instances: the others keep their cmd_vel targets, bit for bit; clearing restores every plain plan
    k = 40
    ctx.set_plan_targets((hb.HbTarget * k)(*tg[:k]))
    part, _, _ = ctx.plan_references_gpu(ins, latest)
    assert all(bytes(part[i]) == bytes(rd[i]) for i in range(k)) and all(bytes(part[i]) == bytes(plain_d[i]) for i in range(k, n))
    assert not any(bytes(rd[i]) == bytes(plain_d[i]) for i in range(k))
    ctx.set_plan_targets(None)
    again, _, _ = ctx.plan_references_gpu(ins, latest)
    assert all(bytes(a) == bytes(b) for a, b in zip(again, plain_d))
    ctx.close()


def test_the_cmd_vel_target_given_back_is_the_cmd_vel_plan_on_the_device():
    ctx = hb.Context(horizon_N=N, dt=DT, max_batch=64, device=0)
    n = 48
    x0, gaits, cmd, t0, start, feet, latest, _ = _plan_cases(n, 62)
    two, _, _ = ctx.plan_references_gpu(hb.make_plan_inputs(t0, T, x0, cmd, feet, gaits, start, joint_ik=False), latest)
    ctx.set_plan_targets((hb.HbTarget * n)(*[hb.reference_target(r) for r in two]))
    for ik in (False, True):
        ins = hb.make_plan_inputs(t0, T, x0, cmd, feet, gaits, start, joint_ik=ik)
        given = ctx.plan_references_gpu(ins, latest)
        ctx.set_plan_targets(None)
        plain = ctx.plan_references_gpu(ins, latest)
        ctx.set_plan_targets((hb.HbTarget * n)(*[hb.reference_target(r) for r in two]))
        assert all(bytes(a) == bytes(b) for a, b in zip(given[0], plain[0])) and np.array_equal(given[1], plain[1])
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- the goal episode
@pytest.mark.parametrize("wbc", ["weighted", "hierarchical"])
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_goal_episode_equals_the_stepwise_loop_bitwise(wbc, event_nodes, estimated):
    ctx = context(event_nodes)
    ctx.set_wbc_formulation(wbc)
    B, log_every = 6, 10
    n_ticks = 120 if estimated else 160
    rbd0 = start_states(ctx, B, seed=71)
    vels = cmd_vels(B)
    prm = params(log_every)
    extra = {}
    if wbc == "weighted" and not event_nodes:         # goals with terrains (a 1 cm step), plant variations and pushes
        extra = dict(terrains=hb.make_terrains(B, np.where(np.arange(8)[None, :, None] > 4, 0.03, 0.02) * np.ones((B, 8, 8)), 0.1, rbd0[:, 3:5] - 0.35),
                     plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION), pushes=hb.make_push_schedules(B, 0.15, 0.05, PUSH))
    kw = use(ctx, goals=random_goals(rbd0, B, 71), **extra)
    ep = est_params(seed=2026) if estimated else None
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 40) if estimated else None)
    r = stepwise(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 40) if estimated else None, **kw)
    assert_episode_equal(d, r)
    ctx.set_goals(None)
    u = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 40) if estimated else None)
    moved = [not np.array_equal(a, b) for a, b in zip(d[0].cpu().numpy(), u[0].cpu().numpy())]
    assert moved[:5] == [True] * 5 and not moved[5], moved       # instance 5 has no schedule
    ctx.close()


def _schedules(rbd0, B, t_goal, d=0.3):
    """One goal per robot, d ahead along its start heading, given at t_goal."""
    g = np.c_[rbd0[:B, 3] + d * np.cos(rbd0[:B, 0]), rbd0[:B, 4] + d * np.sin(rbd0[:B, 0]), rbd0[:B, 0] + 0.2]
    return hb.make_goal_schedules(B, t_goal, g[:, None, :])


def test_continuation_independence_permutation_and_instances_beyond_the_setting():
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=72)
    full = _schedules(rbd0, B, 0.19)               # comes into force at t = 0.19, captured on the MPC tick at t = 0.2 (tick 100)
    cont = _schedules(rbd0, B, 0.195)              # given at tick 97.5, captured on tick 100, the first tick of the continuing call
    only0 = hb.make_goal_schedules(B, np.zeros((B, 0)), np.zeros((B, 0, 3)))
    only0[0] = full[0]
    other = _schedules(rbd0[[1, 0, 3, 2, 5, 4]], B, 0.05, 0.2)
    other[3] = full[3]
    padded = hb.make_goal_schedules(B, np.zeros((B, 0)), np.zeros((B, 0, 3)))
    for i in range(3):
        padded[i] = full[i]
    assert_setting_episodes(ctx, "goals", rbd0, params(10), full, only0, other, 3, (hb.HbGoalSchedule * 3)(*[full[i] for i in range(3)]), padded,
                            cont=cont)
    # a split whose second call starts after the goal's time and before its capture tick (t = 0.196 .. 0.2)
    ctx.set_goals(_schedules(rbd0, B, 0.195))
    assert_continues(ctx, rbd0, GAITS, cmd_vels(B), 200, 98, params(1), 1)
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_setting_goals_again_recaptures(estimated):
    """Goals captured in one call are forgotten by a new hb_rollout_set_goals: a continued episode under the same schedules, set again
    between the calls, recaptures every goal in force on its first MPC tick, from that tick's state."""
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=73)
    vels = cmd_vels(B)
    ep = est_params(seed=9) if estimated else None
    first_goals = _schedules(rbd0, B, 0.0)

    def continued(goals):
        """100 ticks under first_goals (goals captured at tick 0), then, with `goals` set if given, 100 more in a second call"""
        ctx.set_goals(first_goals)
        a = device(ctx, rbd0, GAITS, vels, 100, params(10), 10, ep, hb.estimation_states(B, 40) if ep else None)
        if goals is not None:
            ctx.set_goals(goals)
        return outputs(device(ctx, a[0], GAITS, vels, 100, params(10), 10, ep, a[5] if ep else None, tick0=100, act=a[1], estop=a[2], stats=a[3],
                              est_stats=a[6] if ep else None))

    kept = continued(None)
    again = continued(first_goals)                 # the same schedules set again: the goal in force is captured again at t = 0.2
    assert all(not np.array_equal(kept[0][i], again[0][i]) for i in range(B))
    # the same as goals given at the continuation's first tick
    fresh = continued(_schedules(rbd0, B, 0.2))
    assert_episode_equal(again, fresh)
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_zero_goal_schedules_change_nothing_and_goals_add_no_launch(estimated):
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=74)
    vels = cmd_vels(B)
    ep = est_params(seed=5) if estimated else None
    none = hb.make_goal_schedules(B, np.zeros((B, 0)), np.zeros((B, 0, 3)))
    late = _schedules(rbd0, B, 10.0)                # goals that never come into force within the episode
    assert_null_settings(ctx, "goals", lambda: device(ctx, rbd0, GAITS, vels, 100, params(5), 5, ep),
                         (none, (hb.HbGoalSchedule * 3)(*none[:3]), late), _schedules(rbd0, B, 0.0))
    ctx.set_goals(None)
    plain = launch_coefficients(ctx, rbd0, GAITS, vels, params(0), ep)
    ctx.set_goals(_schedules(rbd0, B, 0.03))
    assert launch_coefficients(ctx, rbd0, GAITS, vels, params(0), ep) == plain
    ctx.close()


def test_argument_checks_return_before_any_launch_and_keep_the_setting():
    ctx = context(max_batch=6)
    lib = ctx._lib
    B = 6
    rbd0 = start_states(ctx, B, seed=75)
    vels = cmd_vels(B)
    good = _schedules(rbd0, B, 0.02)
    assert C.sizeof(hb.HbGoalSchedule) == 8 + 8 * 8 * 4
    nan, inf = float("nan"), float("inf")

    def bad(edit):
        W = (hb.HbGoalSchedule * B)(*good)
        edit(W[2])
        return W

    def two(s, t1):
        s.n_goal = 2; s.time[1] = t1

    edits = [lambda s: setattr(s, "n_goal", -1), lambda s: setattr(s, "n_goal", 9), lambda s: s.time.__setitem__(0, nan),
             lambda s: s.time.__setitem__(0, inf), lambda s: s.goal[0].__setitem__(2, nan), lambda s: s.goal[0].__setitem__(0, -inf),
             lambda s: two(s, 0.01)]
    big = (hb.HbGoalSchedule * (B + 1))(*([good[0]] * (B + 1)))
    assert_rejected_settings(ctx, "goals", lambda: device(ctx, rbd0, GAITS, vels, 60, params(10), 10), good, [bad(e) for e in edits], big)
    ok = bad(lambda s: s.goal[5].__setitem__(1, nan))            # entries beyond n_goal are not read
    assert lib.hb_rollout_set_goals(ctx._h, B, ok) == 0
    ok = bad(lambda s: two(s, 0.02))                             # equal times: the later goal is the one in force
    assert lib.hb_rollout_set_goals(ctx._h, B, ok) == 0
    # the planner's targets: the same conventions
    tg = hb.goal_to_target(np.zeros(B), np.tile(sc.INITIAL_STATE, (B, 1)), np.c_[np.full(B, 0.5), np.zeros((B, 2))])
    c0 = ctx.launch_count
    for edit in (lambda r: setattr(r, "n", 0), lambda r: setattr(r, "n", 17), lambda r: r.time.__setitem__(1, 0.0),
                 lambda r: r.state[1].__setitem__(3, nan), lambda r: r.time.__setitem__(0, -inf)):
        W = (hb.HbTarget * B)(*tg)
        edit(W[4])
        assert lib.hb_plan_set_targets(ctx._h, B, W) == -1
    assert lib.hb_plan_set_targets(None, B, tg) == -1 and lib.hb_plan_set_targets(ctx._h, -1, tg) == -1
    assert lib.hb_plan_set_targets(ctx._h, 1, None) == -1
    assert lib.hb_plan_set_targets(ctx._h, B + 1, (hb.HbTarget * (B + 1))(*([tg[0]] * (B + 1)))) == -4
    assert lib.hb_plan_set_targets(ctx._h, B, tg) == 0 and lib.hb_plan_set_targets(ctx._h, 0, None) == 0
    assert ctx.launch_count == c0
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- closed loop
# [m] The robots holding a goal at their start pose drifted at most 0.078 m from it over the 2.5 s in this test on one H100 80GB HBM3
# (700 W power limit); the trot itself sways the base. The bound leaves 28 % above that.
STAY_TOL = 0.1


def test_trotting_robots_hold_a_goal_at_their_start_pose_and_approach_a_goal_ahead():
    """Trotting robots (cmd_vel 0) on the N = 40, dt = 20 ms grid: the first half given their own start pose as a goal from t = 0 (a
    one-sample target) stay within STAY_TOL of it at the start of every tick for 2.5 s; the second half, given a goal 0.5 m ahead at
    t = 0.2 s, end closer to it than they started."""
    ctx = context(max_batch=16)
    B = 16
    rbd0 = start_states(ctx, B, seed=76)
    h = B // 2
    g = np.c_[rbd0[:, 3], rbd0[:, 4], rbd0[:, 0]]
    g[h:, 0] += 0.5 * np.cos(rbd0[h:, 0]); g[h:, 1] += 0.5 * np.sin(rbd0[h:, 0])
    times = np.r_[np.zeros(h), np.full(B - h, 0.2)]
    ctx.set_goals(hb.make_goal_schedules(B, times[:, None], g[:, None, :]))
    assert hb.goal_to_target(0.0, ctx.rbd_to_centroidal(rbd0[:1]), g[0])[0].n == 1
    out = outputs(device(ctx, rbd0, ["trot"] * B, np.zeros((B, 2, 4)), 1250, params(5), 5))
    assert (out[3]["fail_tick"] < 0).all(), out[3]
    drift = np.hypot(out[4][:h, :, 3] - g[:h, 0, None], out[4][:h, :, 4] - g[:h, 1, None])
    end = np.hypot(out[0][h:, 3] - g[h:, 0], out[0][h:, 4] - g[h:, 1])
    print("goal at the start pose: max drift %.4f m; goal 0.5 m ahead: final distance %s" % (drift.max(), np.round(end, 4)))
    assert drift.max() < STAY_TOL
    assert (end < 0.5).all()
    ctx.close()
