"""Goal poses as planner targets on the host (no GPU): hb_goal_to_target against a numpy restatement of goalToTargetTrajectories,
the planner with explicit targets (hb_plan_references_targets) against the plain cmd_vel plan, and the record checks of the target and
goal setters' host helpers."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import api, scenarios

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_CONSTS = open(os.path.join(ROOT, "include", "hunter_model_constants.h")).read()
COM_HEIGHT = float(re.search(r"#define HB_COM_HEIGHT (\S+)", _CONSTS).group(1))
V_DISP = float(re.search(r"#define HB_TARGET_DISPLACEMENT_VELOCITY (\S+)", _CONSTS).group(1))
V_ROT = float(re.search(r"#define HB_TARGET_ROTATION_VELOCITY (\S+)", _CONSTS).group(1))
DEFAULT_JOINTS = [float(v) for v in re.search(r"HB_DEFAULT_JOINT_STATE\[10\] = \{([^}]*)\}", _CONSTS).group(1).split(",")]
N, DT = 40, 0.02
T = N * DT


def goal_target_ref(t, x, goal):
    """goalToTargetTrajectories + estimateTimeToTarget + targetPoseToTargetTrajectories (TargetTrajectoriesPublisher.cpp:29-100) for one
    observation: (times, states), with the single-sample target where the reaching time is zero."""
    cur = [float(v) for v in x[6:12]]
    dz = COM_HEIGHT - cur[2]
    dz = min(dz, 0.04) if dz > 0 else max(dz, -0.04)
    target = [float(goal[0]), float(goal[1]), cur[2] + dz, float(goal[2]), 0.0, 0.0]
    dx, dy, dyaw = target[0] - cur[0], target[1] - cur[1], target[3] - cur[3]
    reach = max(abs(dyaw) / V_ROT, math.sqrt(dx * dx + dy * dy) / V_DISP)
    start = [cur[0], cur[1], cur[2] + dz, cur[3], 0.0, 0.0]
    row = lambda pose: [0.0] * 6 + pose + DEFAULT_JOINTS
    if reach == 0.0:
        return [t], [row(target)]
    return [t, t + reach], [row(start), row(target)]


def _targets(tg):
    return [(np.array(r.time[:r.n]), np.array([r.state[k][:] for k in range(r.n)])) for r in tg]


def _check_against_ref(t, x, goal):
    got = _targets(hb.goal_to_target(t, x, goal))
    for i in range(len(x)):
        times, states = goal_target_ref(t[i], x[i], goal[i])
        assert np.array_equal(got[i][0], times), (i, got[i][0], times)
        assert np.array_equal(got[i][1], np.array(states)), i
    return got


def test_goal_to_target_matches_the_publisher():
    rng = np.random.default_rng(7)
    B = 64
    x = scenarios.random_initial_states(B, seed=11)
    x[:, 8] = COM_HEIGHT + rng.uniform(-0.1, 0.1, B)            # the z clamp both ways, and inside the limit
    x[:, 10:12] = rng.uniform(-0.2, 0.2, (B, 2))                 # pitch and roll are dropped
    t = rng.uniform(0.0, 5.0, B)
    goal = np.c_[x[:, 6:8] + rng.uniform(-2.0, 2.0, (B, 2)), x[:, 9] + rng.uniform(-3.0, 3.0, B)]
    got = _check_against_ref(t, x, goal)
    reach = np.array([g[0][-1] - g[0][0] for g in got])
    disp = np.hypot(goal[:, 0] - x[:, 6], goal[:, 1] - x[:, 7]) / V_DISP
    rot = np.abs(goal[:, 2] - x[:, 9]) / V_ROT
    assert (disp > rot).any() and (rot > disp).any()             # displacement-bound and rotation-bound reaching times
    assert (x[:, 8] < COM_HEIGHT - 0.04).any() and (x[:, 8] > COM_HEIGHT + 0.04).any()
    np.testing.assert_allclose(reach, np.maximum(disp, rot), rtol=1e-15)


def test_goal_to_target_cases():
    x = np.tile(scenarios.INITIAL_STATE, (6, 1))
    x[:, 6:10] = [0.3, -0.2, COM_HEIGHT, 0.1]
    x[0, 8] = COM_HEIGHT - 0.2                                    # raised by 0.04 only
    x[1, 8] = COM_HEIGHT + 0.2                                    # lowered by 0.04 only
    x[2, 9] = 3.0                                                 # unwrapped: the goal yaw -3 is 6 rad away, not 0.28
    x[4, 9] = 2 * math.pi + 0.1                                   # one turn around: 2 pi to turn back to the goal yaw 0.1
    goal = np.array([[1.3, -0.2, 0.1], [0.3, -0.2, 0.1], [0.3, -0.2, -3.0], [0.3, -0.2, 0.1], [0.3, -0.2, 0.1], [0.3, -0.2, 1.67]])
    got = _check_against_ref(np.full(6, 2.0), x, goal)
    assert got[0][1][0][8] == COM_HEIGHT - 0.2 + 0.04 and got[1][1][0][8] == COM_HEIGHT + 0.2 - 0.04
    assert got[0][0][1] == 2.0 + 1.0 / V_DISP
    assert got[2][0][1] == 2.0 + 6.0 / V_ROT
    assert got[3][0].shape == (1,) and got[3][0][0] == 2.0        # already there: one sample at the goal pose
    assert np.array_equal(got[3][1][0][6:12], [0.3, -0.2, COM_HEIGHT, 0.1, 0.0, 0.0])
    assert got[4][0][1] == 2.0 + 2 * math.pi / V_ROT
    assert got[5][0][1] == 2.0 + 1.0                              # 1.57 rad at 1.57 rad/s


def test_goal_to_target_rejects():
    lib = hb.load_library()
    x = np.tile(scenarios.INITIAL_STATE, (2, 1)); t = np.zeros(2); g = np.zeros((2, 3))
    out = (hb.HbTarget * 2)()
    P = lambda a: C.c_void_p(a.ctypes.data)
    assert lib.hb_goal_to_target(2, P(t), P(x), P(g), out) == 0
    assert lib.hb_goal_to_target(0, None, None, None, None) == -1
    assert lib.hb_goal_to_target(-1, P(t), P(x), P(g), out) == -1
    for a, k in ((t, 1), (x, 22 + 6), (x, 22 + 9), (g, 3), (g, 5)):        # t, the pose x, y, yaw, the goal
        for v in (np.nan, np.inf):
            saved = a.flat[k]
            a.flat[k] = v
            assert lib.hb_goal_to_target(2, P(t), P(x), P(g), out) == -1
            a.flat[k] = saved
    x[1, 0] = np.nan                                             # the momentum part is not read
    assert lib.hb_goal_to_target(2, P(t), P(x), P(g), out) == 0


def _cases(n, seed):
    rng = np.random.default_rng(seed)
    x0 = scenarios.random_initial_states(n, seed=seed)
    gaits = [["trot", "standing_trot", "flying_trot", "stance"][i % 4] for i in range(n)]
    cmd = np.stack([rng.uniform(-0.6, 0.8, n), rng.uniform(-0.2, 0.2, n), np.zeros(n), rng.uniform(-0.5, 0.5, n)], axis=1)
    t0 = rng.uniform(0.0, 3.0, n)
    start = t0 + rng.uniform(-1.3, 0.3, n)
    feet = x0[:, None, 6:9] + rng.normal(0, 0.1, (n, 4, 3))
    feet[:, :, 2] = 0.02
    latest = feet + rng.normal(0, 0.02, feet.shape)
    return x0, gaits, cmd, t0, start, feet.reshape(n, 12), latest.reshape(n, 12)


def _same_refs(a, b):
    return all(bytes(x) == bytes(y) for x, y in zip(a, b))


def test_cmd_vel_target_round_trip_is_the_cmd_vel_plan():
    """The two-sample cmd_vel target a joint_ik = 0 plan writes, fed back as an explicit target, reproduces the plain plan bit for bit,
    with and without IK joint references."""
    n = 48
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, 5)
    plain0, _ = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, joint_ik=False)
    targets = (hb.HbTarget * n)(*[hb.reference_target(r) for r in plain0])
    assert all(t.n == 2 for t in targets)
    for ik in (False, True):
        plain, ls_plain = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, joint_ik=ik)
        given, ls_given = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, joint_ik=ik, targets=targets)
        assert _same_refs(plain, given) and np.array_equal(ls_plain, ls_given)


def test_goal_target_plan():
    """A goal target replaces the cmd_vel target in the plan's target samples; the schedule does not depend on it."""
    n = 16
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, 9)
    goal = np.c_[x0[:, 6:8] + 0.5, x0[:, 9] + 0.3]
    tg = hb.goal_to_target(t0, x0, goal)
    plain, _ = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, joint_ik=False)
    got, _ = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, joint_ik=False, targets=tg)
    for i in range(n):
        assert got[i].n_targets == tg[i].n
        assert np.array_equal(np.array(got[i].target_times[:2]), np.array(tg[i].time[:2]))
        assert bytes(got[i].target_states)[:2 * 22 * 8] == bytes(tg[i].state)[:2 * 22 * 8]
        assert got[i].n_events == plain[i].n_events and bytes(got[i].event_times) == bytes(plain[i].event_times)
    ik, _ = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, targets=tg)
    for i in range(n):
        assert ik[i].n_targets == int(math.floor(T / 0.15)) + 1        # resampled every 0.15 s over the horizon
        np.testing.assert_allclose(ik[i].target_states[ik[i].n_targets - 1][6], goal[i, 0] if tg[i].time[1] <= t0[i] + T else
                                   x0[i, 6] + (goal[i, 0] - x0[i, 6]) * T / (tg[i].time[1] - t0[i]), rtol=0, atol=1e-12)


def test_target_records_are_checked():
    n = 4
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, 2)
    good = hb.goal_to_target(t0, x0, np.c_[x0[:, 6:8] + 0.5, x0[:, 9]])
    hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, targets=good)

    def bad(edit):
        tg = (hb.HbTarget * n)(*good)
        edit(tg[2])
        return tg

    def non_ascending(r):
        r.time[1] = r.time[0]

    def nan_state(r):
        r.state[1][21] = np.nan

    def inf_time(r):
        r.time[0] = -np.inf

    for edit in (lambda r: setattr(r, "n", 0), lambda r: setattr(r, "n", api.HB_MAX_TARGETS + 1), non_ascending, nan_state, inf_time):
        with pytest.raises(hb.HunterB200Error):
            hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, targets=bad(edit))
    ok = bad(lambda r: r.state[5].__setitem__(0, np.nan))            # an unused sample is not read
    hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, targets=ok)
    with pytest.raises(ValueError):
        hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, targets=good[:3])
    with pytest.raises(ValueError):
        hb.make_targets([[0.0, 1.0]], [np.zeros((3, 22))])


def test_make_targets():
    tg = hb.make_targets([[0.5], [0.0, 1.0, 2.0]], [np.ones(22), np.arange(66.0).reshape(3, 22)])
    assert tg[0].n == 1 and tg[0].time[0] == 0.5 and list(tg[0].state[0]) == [1.0] * 22
    assert tg[1].n == 3 and list(tg[1].time[:3]) == [0.0, 1.0, 2.0] and tg[1].state[2][21] == 65.0


def test_make_goal_schedules():
    s = hb.make_goal_schedules(3, [0.0, 1.0], [[1.0, 2.0, 0.5], [0.0, 0.0, -1.0]])
    v = np.ctypeslib.as_array(s)
    assert (v["n_goal"] == 2).all() and np.array_equal(v["time"][:, :2], [[0.0, 1.0]] * 3)
    assert np.array_equal(v["goal"][1, :2], [[1.0, 2.0, 0.5], [0.0, 0.0, -1.0]]) and not v["goal"][:, 2:].any()
    per = hb.make_goal_schedules(2, [[0.2], [0.4]], np.array([[[1.0, 0.0, 0.0]], [[2.0, 0.0, 0.0]]]))
    assert per[1].time[0] == 0.4 and per[1].goal[0][0] == 2.0 and per[0].n_goal == 1
    one = hb.make_goal_schedules(2, 0.3, [0.5, 0.5, 0.0])
    assert one[0].n_goal == 1 and one[1].goal[0][1] == 0.5
    assert (np.ctypeslib.as_array(hb.make_goal_schedules(2, np.zeros((2, 0)), np.zeros((2, 0, 3))))["n_goal"] == 0).all()
    assert C.sizeof(hb.HbGoalSchedule) == 8 + 8 * hb.HB_MAX_GOALS * 4
    for times, goals in (([1.0, 0.0], np.zeros((2, 3))), ([0.0, np.nan], np.zeros((2, 3))), ([0.0, 1.0], [[0.0, np.inf, 0.0], [0.0, 0.0, 0.0]]),
                         (np.zeros(9), np.zeros((9, 3))), ([0.0, 1.0], np.zeros((3, 3)))):
        with pytest.raises(ValueError):
            hb.make_goal_schedules(2, times, goals)
