"""Controller settings in the episodes (hb_rollout_set_controller_settings): each robot's WBC settings and joint PD gains. A record must act
on its robot exactly as the same values set on the context (hb_wbc_set_settings, params.gains) act on an unset episode, under both WBCs,
both time grids, with and without the estimator; then the setting's contract (null settings, launch counts, continuation, independence,
permutation, instances beyond the setting, clearing, argument checks), the precedence over the context's settings, and the calls that
ignore it."""
import ctypes as C
from contextlib import contextmanager

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from episode_ref import (FRICTION, GAITS, PUSH, array_of, assert_episode_equal, assert_null_settings, assert_records_act_as_their_values,
                         assert_rejected_settings, assert_setting_episodes, cmd_vels, context, device, est_params, logged_episode, outputs, params,
                         small_terrains, start_states, stepwise, use)

pytestmark = pytest.mark.gpu

B = 6


def _defaults():
    w = hb.HbWbcSettings()
    assert hb.load_library().hb_default_wbc_settings(C.byref(w)) == 0
    return w


def _records():
    """Three records that between them change the swing task, the base tasks, the torque limits and friction, the weights and the PD gains."""
    w = _defaults()
    return [
        hb.make_controller_settings(1, swing_kp=1.5 * w.swing_kp, swing_kd=1.3 * w.swing_kd, kp_big_stance=45.0, kd_small=2.5)[0],
        hb.make_controller_settings(1, base_height_kp=0.8 * w.base_height_kp, base_height_kd=1.2 * w.base_height_kd,
                                    base_angular_kp=0.7 * w.base_angular_kp, base_angular_kd=1.2 * w.base_angular_kd,
                                    torque_limits=0.9 * np.asarray(w.torque_limits), friction_coefficient=0.5)[0],
        hb.make_controller_settings(1, weight_swing_leg=2.0 * w.weight_swing_leg, weight_base_accel=0.5 * w.weight_base_accel,
                                    weight_contact_force=0.5 * w.weight_contact_force, kp_small_swing=25.0, kp_big_swing=35.0, kd_feet=0.02)[0],
    ]


@contextmanager
def _on_the_context(ctx, rec, prm, ep):
    """The context's WBC settings and a copy of prm carrying rec's values; the previous settings restored on exit."""
    old = ctx.wbc_settings()
    ctx.set_wbc_settings(rec.wbc)
    p = hb.HbRolloutParams.from_buffer_copy(bytes(prm))
    p.gains = rec.gains
    yield p, ep
    ctx.set_wbc_settings(old)


@pytest.mark.parametrize("wbc", ["weighted", "hierarchical"])
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_records_equal_per_context_runs_bitwise(wbc, event_nodes, estimated):
    """Robot i with record k gives bit for bit what robot i gives in the unset episode run with record k's values on the context."""
    ctx = context(event_nodes)
    ctx.set_wbc_formulation(wbc)
    rbd0 = start_states(ctx, B, seed=91)
    if wbc == "weighted" and not event_nodes:       # alongside pushes, variations, a terrain, goals and an MPC latency
        use(ctx, plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION, motor_strength=0.95),
            pushes=hb.make_push_schedules(B, 0.05, 0.05, PUSH), terrains=small_terrains(), goals=hb.make_goal_schedules(B, 0.05, [0.2, 0.0, 0.1]),
            mpc_latencies=[0, 1, 2, 0, 3, 1])
    assert_records_act_as_their_values(ctx, "controller_settings", _records(), _on_the_context, rbd0, params(10),
                                       est_params(seed=2029) if estimated else None)
    ctx.close()


@pytest.mark.parametrize("wbc", ["weighted", "hierarchical"])
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_null_settings(wbc, event_nodes, estimated):
    """Records equal to (the context's settings, params.gains) give the unset episode bit for bit with the same launches."""
    ctx = context(event_nodes)
    ctx.set_wbc_formulation(wbc)
    ctx.set_kp_kd(300.0, 35.0)                        # the records follow the context, whatever it holds
    rbd0 = start_states(ctx, B, seed=92)
    prm = params(5)
    prm.gains.kp_big_stance = 42.0
    ep = est_params(seed=7) if estimated else None
    null = hb.make_controller_settings(B, wbc=ctx.wbc_settings(), gains=prm.gains)
    assert_null_settings(ctx, "controller_settings", lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 60, prm, 5, ep,
                                                                    hb.estimation_states(B, 50) if estimated else None),
                         (null, array_of([null[0]] * 3)), array_of(_records() * 2))
    ctx.close()


def test_setting_contract():
    ctx = context()
    rbd0 = start_states(ctx, B, seed=93)
    r = _records()
    full = array_of([r[0], r[1], r[2], r[1], r[0], r[2]])
    one = hb.make_controller_settings(B)
    one[0] = r[0]
    other = array_of([r[2], r[0], r[1], r[1], r[2], r[0]])       # instance 3 keeps its record
    part = array_of([r[1], r[2]])
    padded = hb.make_controller_settings(B)
    padded[0], padded[1] = r[1], r[2]
    assert_setting_episodes(ctx, "controller_settings", rbd0, params(10), full, one, other, 3, part, padded)
    ctx.close()


def _bad():
    out = []
    for field, value in [("swing_kp", float("nan")), ("kd_big", float("inf")), ("base_angular_kd", -float("inf")),
                         ("friction_coefficient", 0.0), ("weight_swing_leg", 0.0), ("weight_contact_force", -1e-3),
                         ("kp_small_stance", -1.0), ("swing_kd", -1.0)]:
        out.append(hb.make_controller_settings(2, **{field: value}))
    tl = hb.make_controller_settings(2)
    tl[1].wbc.torque_limits[3] = 0.0
    out.append(tl)
    return out


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_rejected_settings(estimated):
    ctx = context()
    rbd0 = start_states(ctx, B, seed=94)
    ep = est_params(seed=8) if estimated else None
    assert_rejected_settings(ctx, "controller_settings",
                             lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 40, params(5), 5, ep, hb.estimation_states(B, 50) if estimated else None),
                             array_of(_records() * 2), _bad(), hb.make_controller_settings(ctx.max_batch + 1))
    ctx.close()


def test_precedence_over_the_context():
    """With records for instances 0..2 of 6, changing hb_wbc_set_settings, hb_wbc_set_kp_kd or params.gains moves none of instances 0..2 and
    some of 3..5."""
    ctx = context()
    rbd0 = start_states(ctx, B, seed=95)
    prm = params(10)
    ctx.set_controller_settings(array_of(_records()))
    base = logged_episode(ctx, rbd0, prm, None)
    w = ctx.wbc_settings()
    changes = []
    s = hb.HbWbcSettings.from_buffer_copy(bytes(w)); s.base_angular_kp *= 0.6
    changes.append(lambda: ctx.set_wbc_settings(s))
    changes.append(lambda: ctx.set_kp_kd(1.4 * w.swing_kp, w.swing_kd))
    for change in changes:
        change()
        moved = logged_episode(ctx, rbd0, prm, None)
        ctx.set_wbc_settings(w)
        assert_episode_equal(moved, base, rows_a=slice(0, 3), rows_b=slice(0, 3))
        assert any(not np.array_equal(moved[0][i], base[0][i]) for i in range(3, B))     # instance 5 stands: no swing task
    p = hb.HbRolloutParams.from_buffer_copy(bytes(prm))
    p.gains.kp_big_stance = 48.0
    moved = logged_episode(ctx, rbd0, p, None)
    assert_episode_equal(moved, base, rows_a=slice(0, 3), rows_b=slice(0, 3))
    assert any(not np.array_equal(moved[0][i], base[0][i]) for i in range(3, B))
    ctx.close()


@pytest.mark.parametrize("wbc", ["weighted", "hierarchical"])
def test_other_calls_ignore_the_setting(wbc):
    """With a setting in force, the episode written as a loop of public calls (resident cycle, resident_wbc, joint_command), the two WBC
    solves and the control step give what they give with none."""
    ctx = context()
    ctx.set_wbc_formulation(wbc)
    rbd0 = start_states(ctx, B, seed=96)
    vels = cmd_vels(B)
    prm = params(10)
    x0 = sc.random_initial_states(B, seed=97)
    refs = [sc.make_reference(x0[i], (0.2, 0.0, 0.0, 0.1), "trot", ctx.N, ctx.dt) for i in range(B)]
    x_ref, swing, cmode = (np.stack([r[j] for r in refs]) for j in range(3))
    rbd_cs = sc.consistent_rbd(x0)
    runs = []
    for setting in (None, array_of(_records() * 2)):
        ctx.set_controller_settings(setting)
        loop = stepwise(ctx, rbd0, GAITS, vels, 30, prm, 10)
        x = np.tile(sc.INITIAL_STATE, (B, 1)); u = np.zeros((B, hb.NU)); u[:, 2:12:3] = 9.81 * 2
        mode = np.array([3, 1, 2, 3, 1, 2], dtype=np.int32)
        w = ctx.wbc_solve(x, u, rbd0, mode)
        h = ctx.hierarchical_wbc_solve(x, u, rbd0, mode)
        xt, ut = ctx.mpc_cold_start(x0, cmode)
        step = ctx.control_step(0.002, x0, x_ref, swing, cmode, rbd_cs, xt, ut)
        runs.append((outputs(loop), w + h + tuple(np.asarray(a) for a in step)))
    (la, ca), (lb, cb) = runs
    assert_episode_equal(la, lb)
    for a, b in zip(ca, cb):
        assert np.array_equal(a, b)
    ctx.close()
