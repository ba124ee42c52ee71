"""Teleoperated episodes (hb_rollout_set_teleop, Context.set_teleop) on the GPU: the episode against the stepwise loop of public calls
(teleop_ref.TeleopLoop), a transparent publisher against the unset episode, null settings and launches, the per-robot setting contract
with the entry checks, and episode snapshots with teleop set."""
import ctypes as C

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from episode_ref import (FRICTION, GAITS, PUSH, assert_continues, assert_episode_equal, assert_null_settings, assert_rejected_settings,
                         assert_setting_episodes, cmd_vels, context, device, est_params, launch_coefficients, outputs, params, random_goals,
                         start_states, stepwise, use)
from teleop_ref import TeleopLoop, publish

pytestmark = pytest.mark.gpu

INF, ALWAYS = float("inf"), hb.TELEOP_ALWAYS


def mixed(B):
    """Teleop records of the first B - 1 of B >= 6 robots: the default joystick; 10-tick messages in two windows with a gap; messages from
    tick 50 on; a message on every MPC tick without limits; no window at all; then defaults."""
    r = hb.make_teleop_settings(B - 1)
    r[1] = hb.make_teleop_settings(1, 10, [(0, 40), (80, 130)])[0]
    r[2] = hb.make_teleop_settings(1, 25, [(50, ALWAYS)])[0]
    r[3] = hb.make_teleop_settings(1, 5, change_limit=[INF] * 3)[0]
    r[4] = hb.make_teleop_settings(1, windows=[])[0]
    return r


def transparent(B, mpc_every=5):
    """Records that pass every command through unchanged on every MPC tick: the unset episode for commands the step reproduces exactly."""
    return hb.make_teleop_settings(B, mpc_every, [(0, ALWAYS)], [INF] * 3)


def dyadic_vels(B):
    v = np.zeros((B, 2, 4))
    v[:, 0, 0] = 0.125
    v[:, 1, 0] = np.arange(B) * 0.125 - 0.25; v[:, 1, 3] = 0.25
    return v


# ---------------------------------------------------------------------------------------------------------------- the teleop episode
@pytest.mark.parametrize("wbc", ["weighted", "hierarchical"])
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_teleop_episode_equals_the_stepwise_loop_bitwise(wbc, event_nodes, estimated):
    """Goals arrive inside and outside the windows (tick 30 and, for odd robots, tick 105; robot 2's from tick 0), so messages replace
    goals, a goal and a message fall on one tick (robots 1 and 3), and a robot keeps its last target outside its windows."""
    ctx = context(event_nodes)
    ctx.set_wbc_formulation(wbc)
    B, log_every = 6, 10
    n_ticks = 120 if estimated else 160
    rbd0 = start_states(ctx, B, seed=81)
    vels = cmd_vels(B)
    prm = params(log_every)
    extra = {}
    if wbc == "weighted" and not event_nodes:         # with terrains, plant variations and pushes
        extra = dict(terrains=hb.make_terrains(B, np.where(np.arange(8)[None, :, None] > 4, 0.03, 0.02) * np.ones((B, 8, 8)), 0.1, rbd0[:, 3:5] - 0.35),
                     plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION), pushes=hb.make_push_schedules(B, 0.15, 0.05, PUSH))
    if wbc == "hierarchical" and not event_nodes:     # with MPC latencies and the simulated hardware
        extra = dict(mpc_latencies=[5, 0, 2, 3], hardware=hb.make_hardware_settings(4, actuation_delay=[0.009, 0.004, 0.012, 0.0]))
    goals, teleop = random_goals(rbd0, B, 81), mixed(B)
    kw = use(ctx, **extra)
    ctx.set_goals(goals)
    ctx.set_teleop(teleop)
    ep = est_params(seed=2027) if estimated else None
    fresh = lambda: hb.estimation_states(B, 40) if estimated else None
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, fresh())
    loop = TeleopLoop(ctx, teleop, prm.period, goals)
    r = stepwise(loop, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, fresh(), **kw)
    ctx.set_plan_targets(None)
    assert_episode_equal(d, r)
    assert set(loop.last) == set(range(5)) and loop.last[4].tolist() == [0.0] * 4 and loop.last[3][0] == vels[3, 1, 0]
    ctx.set_teleop(None)
    u = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, fresh())
    moved = [not np.array_equal(a, b) for a, b in zip(d[0].cpu().numpy(), u[0].cpu().numpy())]
    assert moved[:5] == [True] * 5 and not moved[5], moved        # robot 5 has no record
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_a_transparent_publisher_is_the_unset_episode(estimated):
    """period_ticks = mpc_every, one window over the episode, no limits, dyadic commands with vz = 0: every MPC tick captures the target
    the planner would have built from the same command and state, so the episode is the unset one bit for bit."""
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=82)
    vels = dyadic_vels(B)
    ep = est_params(seed=3) if estimated else None
    fresh = lambda: hb.estimation_states(B, 40) if estimated else None
    u = device(ctx, rbd0, GAITS, vels, 200, params(10), 10, ep, fresh())
    ctx.set_teleop(transparent(B))
    t = device(ctx, rbd0, GAITS, vels, 200, params(10), 10, ep, fresh())
    assert_episode_equal(u, t)
    ctx.set_teleop(hb.make_teleop_settings(B))                  # the default publisher ramps the step and moves every robot
    p = outputs(device(ctx, rbd0, GAITS, vels, 200, params(10), 10, ep, fresh()))
    assert all(not np.array_equal(p[0][i], outputs(u)[0][i]) for i in range(B))
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_null_settings_change_nothing_and_teleop_adds_no_launch(estimated):
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=83)
    vels = dyadic_vels(B)
    ep = est_params(seed=5) if estimated else None
    run = lambda: device(ctx, rbd0, GAITS, vels, 100, params(5), 5, ep, hb.estimation_states(B, 40) if estimated else None)
    tr = transparent(B)
    assert_null_settings(ctx, "teleop", run, (tr, (hb.HbTeleopSetting * 3)(*tr[:3])), hb.make_teleop_settings(B))
    ctx.set_teleop(None)
    plain = launch_coefficients(ctx, rbd0, GAITS, vels, params(0), ep)
    ctx.set_teleop(mixed(B))
    assert launch_coefficients(ctx, rbd0, GAITS, vels, params(0), ep) == plain
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- the setting contract
def test_continuation_independence_permutation_and_instances_beyond_the_setting():
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=84)
    full = hb.make_teleop_settings(B, [50, 25, 10, 50, 5, 20], change_limit=[[0.1, 0.05, 0.3]] * 3 + [[0.2, 0.1, 0.5]] * 3)
    one = (hb.HbTeleopSetting * 1)(full[0])
    other = hb.make_teleop_settings(B, 10, [(20, 60)])
    other[3] = full[3]
    part = (hb.HbTeleopSetting * 3)(*full[:3])
    padded = (hb.HbTeleopSetting * B)(*(list(full[:3]) + list(transparent(3))))     # cmd_vels' last three robots pass through exactly
    assert_setting_episodes(ctx, "teleop", rbd0, params(10), full, one, other, 3, part, padded)     # split at tick 100: a message tick
    ctx.set_teleop(full)
    assert_continues(ctx, rbd0, GAITS, cmd_vels(B), 200, 130, params(10), 10)       # between messages of every robot but 4
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_setting_teleop_again_clears_the_publishers(estimated):
    """A continued episode with the same records set again between the calls starts its publishers from last = 0 with no target: the
    robots whose first message then gives another filtered command move differently from the continuation that keeps the publishers."""
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=85)
    vels = cmd_vels(B)
    ep = est_params(seed=9) if estimated else None
    rec = hb.make_teleop_settings(B, 25)

    def continued(again):
        ctx.set_teleop(rec)
        a = device(ctx, rbd0, GAITS, vels, 100, params(10), 10, ep, hb.estimation_states(B, 40) if ep else None)
        if again:
            ctx.set_teleop(rec)
        return outputs(device(ctx, a[0], GAITS, vels, 100, params(10), 10, ep, a[5] if ep else None, tick0=100, act=a[1], estop=a[2], stats=a[3],
                              est_stats=a[6] if ep else None))

    kept, again = continued(False), continued(True)
    # the message of tick 100 from the kept publisher and from a cleared one: where both give the same filtered command, the same target
    # is captured on the same state, and the robot is the same
    seg = lambda i, a: vels[i, 1 if a >= 100 else 0]       # noqa: E731  (CMD_TIMES: the second segment from t = 0.2 s, tick 100)
    cleared = [not np.array_equal(publish(rec[i], [seg(i, a) for a in range(101)], range(101))[1][-1],
                                  publish(rec[i], [seg(i, 100)], [100])[1][-1]) for i in range(B)]
    assert cleared == [True, True, False, True, True, True]
    assert [not np.array_equal(kept[0][i], again[0][i]) for i in range(B)] == cleared
    assert_episode_equal(again, continued(True))
    ctx.close()


def test_entry_checks_return_before_any_launch_and_keep_the_setting():
    ctx = context(max_batch=6)
    lib = ctx._lib
    B = 6
    rbd0 = start_states(ctx, B, seed=86)
    vels = cmd_vels(B)
    run = lambda prm=params(10): device(ctx, rbd0, GAITS, vels, 60, prm, 10)
    good = hb.make_teleop_settings(B, 10, [(0, 40), (55, 200)])

    def bad(**fields):
        W = (hb.HbTeleopSetting * B)(*good)
        for k, v in fields.items():
            if isinstance(v, tuple):
                getattr(W[2], k)[v[0]] = v[1]
            else:
                setattr(W[2], k, v)
        return W

    edits = [dict(period_ticks=0), dict(period_ticks=-5), dict(n_window=5), dict(n_window=-1), dict(on_tick=(0, -5)), dict(off_tick=(0, 0)),
             dict(on_tick=(1, 35)), dict(change_limit=(0, 0.0)), dict(change_limit=(2, float("nan")))]
    big = (hb.HbTeleopSetting * (B + 1))(*([good[0]] * (B + 1)))
    want, launches = assert_rejected_settings(ctx, "teleop", run, good, [bad(**e) for e in edits], big)
    # records the setter accepts and an episode rejects: a period or a window start off the episode's MPC ticks
    for rec in (hb.make_teleop_settings(B, 7), hb.make_teleop_settings(B, 10, [(3, 100)]), hb.make_teleop_settings(2, 10, [(0, 10), (12, 20)])):
        ctx.set_teleop(rec)
        c0 = ctx.launch_count
        with pytest.raises(hb.HunterB200Error, match="-1"):
            run()
        assert ctx.launch_count == c0
    ctx.set_teleop(hb.make_teleop_settings(B, 7))
    p = params(10)
    p.mpc_every = 7                                             # multiples of this call's mpc_every: accepted
    run(p)
    ctx.set_teleop(good)
    assert_episode_equal(want, run())
    assert lib.hb_rollout_set_teleop(ctx._h, 0, None) == 0
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- snapshots
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_snapshots_with_teleop_continue_exactly(estimated):
    """Saved between two messages with a goal captured and replaced, restored in a fresh context with the same settings: one call. A
    context without teleop rejects the rows; its row size is the size without teleop."""
    B, n1, n2 = 6, 115, 85
    ctx = context()
    rbd0 = start_states(ctx, B, seed=87)
    vels = cmd_vels(B)
    ep = est_params(seed=11) if estimated else None
    fresh = lambda: hb.estimation_states(B, 40) if estimated else None
    goals, teleop = random_goals(rbd0, B, 87), mixed(B)
    plain_bytes = ctx.episode_state_bytes
    ctx.set_goals(goals)
    ctx.set_teleop(teleop)
    assert ctx.episode_state_bytes == plain_bytes + 40
    one = device(ctx, rbd0, GAITS, vels, n1 + n2, params(5), 5, ep, fresh())
    first = device(ctx, rbd0, GAITS, vels, n1, params(5), 5, ep, fresh())
    snap = ctx.save_episodes(B, *first[:4], *(first[5:7] if estimated else ()))
    ctx.set_teleop(None)
    assert ctx.episode_state_bytes == plain_bytes
    with pytest.raises(ValueError, match="bytes"):
        ctx.restore_episodes(snap)
    rows = snap.rows.contiguous()
    assert ctx._lib.hb_episode_restore(ctx._h, B, None, B, C.c_void_p(rows.data_ptr())) == -1
    ctx.close()
    ctx2 = context()
    ctx2.set_goals(goals)
    ctx2.set_teleop(teleop)
    r = ctx2.restore_episodes(snap)
    if estimated:
        second = device(ctx2, r[0], GAITS, vels, n2, params(5), 5, ep, r[4], tick0=n1, act=r[1], estop=r[2], stats=r[3], est_stats=r[5])
    else:
        second = device(ctx2, r[0], GAITS, vels, n2, params(5), 5, tick0=n1, act=r[1], estop=r[2], stats=r[3])
    two = outputs(second)
    two[4] = np.concatenate([first[4].cpu().numpy(), two[4]], axis=1)
    if estimated:
        two[7] = np.concatenate([first[7].cpu().numpy(), two[7]], axis=1)
    assert_episode_equal(one, two)
    ctx2.close()


def _schedules(rbd0, B, t_goal, d=0.3):
    """One goal per robot, d ahead along its start heading, given at t_goal."""
    g = np.c_[rbd0[:B, 3] + d * np.cos(rbd0[:B, 0]), rbd0[:B, 4] + d * np.sin(rbd0[:B, 0]), rbd0[:B, 0] + 0.2]
    return hb.make_goal_schedules(B, t_goal, g[:, None, :])


def _continue(ctx, a, vels, n, tick0, ep=None):
    return outputs(device(ctx, a[0], GAITS, vels, n, params(10), 10, ep, a[5] if ep else None, tick0=tick0, act=a[1], estop=a[2], stats=a[3],
                          est_stats=a[6] if ep else None))


# ---------------------------------------------------------------------------------------------------------------- clearing
def test_a_cleared_setting_is_the_unset_path_at_any_mpc_every():
    """Records with period 50, then cleared (Context.set_teleop(None) or a raw B == 0 call): an episode with mpc_every = 3, which does not
    divide 50, is accepted and is the never-set episode bit for bit, with its launches."""
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=89)
    vels = cmd_vels(B)
    p = params(10)
    p.mpc_every = 3
    run = lambda: device(ctx, rbd0, GAITS, vels, 90, p, 10)
    c0 = ctx.launch_count
    never = run()
    launches = ctx.launch_count - c0
    for clear in (lambda: ctx.set_teleop(None), lambda: ctx._lib.hb_rollout_set_teleop(ctx._h, 0, None)):
        ctx.set_teleop(hb.make_teleop_settings(B))
        with pytest.raises(hb.HunterB200Error, match="-1"):
            run()
        clear()
        c0 = ctx.launch_count
        assert_episode_equal(never, run())
        assert ctx.launch_count - c0 == launches
    ctx.close()


def test_clearing_teleop_mid_episode_drops_the_message_targets():
    """Goals set but none in force, teleop cleared between two calls: the continuation plans on the cmd_vel targets, as it does with the
    goals cleared as well, and no robot keeps the target of its last message."""
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=90)
    vels = cmd_vels(B)
    late = _schedules(rbd0, B, 10.0)

    def continued(clear_goals):
        ctx.set_goals(late)
        ctx.set_teleop(mixed(B))
        a = device(ctx, rbd0, GAITS, vels, 100, params(10), 10)
        ctx.set_teleop(None)
        if clear_goals:
            ctx.set_goals(None)
        return _continue(ctx, a, vels, 100, 100)

    assert_episode_equal(continued(False), continued(True))
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_setting_goals_again_recaptures_for_teleoperated_robots(estimated):
    """Teleoperated robots whose last message (tick 40) replaced their goal: goals set again between two calls are captured again on the
    continuation's first MPC tick, as for robots without teleop, the same as goals given at that tick; kept, the message target stays."""
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=91)
    vels = cmd_vels(B)
    ep = est_params(seed=13) if estimated else None
    first = _schedules(rbd0, B, 0.0)

    def continued(goals):
        ctx.set_goals(first)
        ctx.set_teleop(hb.make_teleop_settings(B, 10, [(0, 50)]))
        a = device(ctx, rbd0, GAITS, vels, 100, params(10), 10, ep, hb.estimation_states(B, 40) if ep else None)
        if goals is not None:
            ctx.set_goals(goals)
        return _continue(ctx, a, vels, 100, 100, ep)

    kept, again = continued(None), continued(first)
    assert all(not np.array_equal(kept[0][i], again[0][i]) for i in range(B))
    assert_episode_equal(again, continued(_schedules(rbd0, B, 0.2)))
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- the conversion
def test_a_captured_message_target_is_the_host_conversion():
    """The target an episode captured on its last MPC tick (tick 100, a message of every robot), read from its snapshot row, is
    hb_cmd_vel_to_target of teleop_ref's filtered command on that tick's state, up to the last bits of the device's trigonometry; its
    source is a message (HB_MAX_GOALS)."""
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=88)
    vels = cmd_vels(B)
    rec = hb.make_teleop_settings(B, 5, change_limit=[0.02, 0.01, 0.05])
    ctx.set_teleop(rec)
    out = device(ctx, rbd0, GAITS, vels, 101, params(1), 1)
    snap = ctx.save_episodes(B, *out[:4])
    rows = snap.rows.cpu().numpy()
    N = ctx.N
    at = 32 + 8 + (N + 1) * 22 * 8 + N * 22 * 8 + ((N + 1) * 4 + 7) // 8 * 8 + 38 * 8 + 12 * 8     # the goal index (uniform grid)
    src = rows[:, at:at + 4].copy().view(np.int32)[:, 0]
    assert (src == hb.HB_MAX_GOALS).all(), src
    x0 = ctx.rbd_to_centroidal(out[4].cpu().numpy()[:, 100])                 # the state entering tick 100
    T = ctx.N * ctx.dt
    for i in range(B):
        seg = [vels[i, 1 if a >= 100 else 0] for a in range(101)]
        sent, lasts = publish(rec[i], seg, range(101))
        assert sent[-1] == 100
        got = hb.HbTarget.from_buffer_copy(rows[i, at + 8:at + 8 + C.sizeof(hb.HbTarget)].tobytes())
        host = hb.cmd_vel_to_target(100 * params(1).period, T, x0[i:i + 1], lasts[-1])[0]
        assert got.n == host.n == 2 and list(got.time[:2]) == list(host.time[:2])
        np.testing.assert_allclose(np.array(got.state[:2]), np.array(host.state[:2]), rtol=0, atol=1e-15)
    ctx.close()
