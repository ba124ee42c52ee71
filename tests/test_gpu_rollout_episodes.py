"""Closed-loop episodes on the device (hb_rollout_batch_dev): one call runs, for a batch of robots, the device planner + resident MPC cycle
every mpc_every ticks and the 500 Hz policy + WeightedWbc tick, joint command law, actuation delay, saturation and plant step on every tick.
The call is checked bit for bit against the same loop written with the existing calls (one host round trip per operator), and against
itself: continuation, independence of instances, failure recording and holding, argument checks, launch counts."""
import ctypes as C

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from episode_ref import (GAITS, GROUND, assert_continues, assert_episode_equal, cmd_vels, context, device, launch_coefficients, params,
                         start_states, stepwise)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
def test_episode_equals_the_stepwise_loop_bitwise(event_nodes):
    """200 ticks of B = 6 mixed-gait episodes with a command change at 0.2 s: rbd, actuation state, estop, stats and log equal the loop
    of existing calls bit for bit. This holds because the cycle's own WBC at t_rel = 0 is the tick's WBC at the same time (same policy point,
    same kernel, same fallback state), so the call may skip it."""
    ctx = context(event_nodes)
    B, n_ticks, log_every = 6, 200, 10
    rbd0 = start_states(ctx, B, seed=11)
    vels = cmd_vels(B)
    prm = params(log_every)
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every)
    r = stepwise(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every)
    assert_episode_equal(d, r)
    assert d[4].shape == (B, n_ticks // log_every, 32)
    assert np.isfinite(r[0]).all() and not np.array_equal(r[0], rbd0)
    ctx.close()


def test_two_calls_continue_one_call_bitwise():
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=12)
    vels = cmd_vels(B)
    assert_continues(ctx, rbd0, GAITS, vels, 200, 100, params(10), 10)
    ctx.close()


def test_instances_are_independent():
    ctx = context()
    B, n_ticks, keep = 6, 100, [1, 3, 4]
    rbd0 = start_states(ctx, B, seed=13)
    vels = cmd_vels(B)
    prm = params(5)
    full = device(ctx, rbd0, GAITS, vels, n_ticks, prm, 5)
    part = device(ctx, rbd0[keep], [GAITS[i] for i in keep], vels[keep], n_ticks, prm, 5)
    assert_episode_equal(full, part, rows_a=keep)
    ctx.close()


def test_standing_episode_keeps_the_robots_up():
    """The setup and bounds of test_dynamic_closed_loop_standing_rollout, driven through the planner and one rollout call (stance, zero
    command). The vertical contact force is the plant's spring force at the logged states, averaged over the last 50 ticks."""
    import torch
    B, n_ticks = 4, 200
    ctx = hb.Context(horizon_N=50, dt=0.02, max_batch=B, device=0)
    rbd0 = start_states(ctx, B, seed=2)
    z0 = rbd0[:, 5].copy()
    prm = params(1)
    cmds = hb.make_rollout_commands(["stance"] * B, 0.0, [0.0], [[0.0, 0.0, 0.0, 0.0]])
    rbd, act, estop, st, log = ctx.rollout(torch.from_numpy(rbd0).cuda(), cmds, n_ticks, params=prm, log_every=1)
    rbd, log = rbd.cpu().numpy(), log.cpu().numpy()
    assert (st["fail_tick"] == -1).all() and (estop.cpu().numpy() == 0).all(), st
    assert np.isfinite(log).all() and np.isfinite(rbd).all()
    heights = log[:, -49:, 5].T
    heights = np.vstack([heights, rbd[None, :, 5]])                 # the last 50 states after a plant step
    assert np.abs(heights - z0[None]).max() < 0.03, np.abs(heights - z0[None]).max()
    assert np.abs(rbd[:, 1:3]).max() < 0.1                          # pitch, roll
    assert np.abs(rbd[:, 16:32]).max() < 1.0
    assert (st["max_abs_torque"] <= max(prm.torque_limit[:]) + 1e-12).all()
    states = np.concatenate([log[:, -49:], rbd[:, None]], axis=1).reshape(-1, 32)
    kin = hb.Context(horizon_N=1, dt=0.01, max_batch=len(states), device=0)
    cpos = kin.contact_positions(kin.rbd_to_centroidal(states)).reshape(B, 50, 4, 3)[..., 2]
    kin.close()
    fz = (prm.sim.ground_stiffness * np.maximum(GROUND - cpos, 0.0)).sum(axis=2).mean(axis=1)
    weight = sc.TOTAL_MASS * 9.81
    assert ((fz > 0.8 * weight) & (fz < 1.2 * weight)).all(), fz / weight
    ctx.close()


def test_failures_are_recorded_and_held():
    """A knee beyond its limit + 0.02 raises the emergency stop on the first tick (reason 1), a roll of 1.7 rad fails the orientation check
    of the first state (reason 2); both keep their starting rbd from then on, and the other instances run as if they were not there."""
    B, n_ticks = 6, 60
    ctx = context()
    rbd0 = start_states(ctx, B, seed=2)
    rbd0[2, 6 + 3] = sc.JOINT_UPPER[3] + 0.03
    rbd0[4, 2] = 1.7
    prm = params(1)
    gaits = ["stance"] * B
    vels = np.zeros((B, 2, 4))
    out = device(ctx, rbd0, gaits, vels, n_ticks, prm, 1)
    rbd, st, log = out[0].cpu().numpy(), out[3], out[4].cpu().numpy()
    assert list(st["fail_tick"][[2, 4]]) == [0, 0] and list(st["fail_reason"][[2, 4]]) == [1, 2], st
    for i in (2, 4):
        assert np.array_equal(rbd[i], rbd0[i]) and (log[i] == rbd0[i]).all()
    others = [0, 1, 3, 5]
    assert (st["fail_tick"][others] == -1).all()
    ref = device(ctx, rbd0[others], [gaits[i] for i in others], vels[others], n_ticks, prm, 1)
    assert_episode_equal(out, ref, rows_a=others)
    ctx.close()


def test_argument_checks_return_before_any_launch():
    import torch
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=2, device=0)
    lib = ctx._lib
    rbd = torch.zeros((3, 32), dtype=torch.float64, device="cuda")
    act = torch.zeros(3 * C.sizeof(hb.HbActuationState), dtype=torch.uint8, device="cuda")
    estop = torch.zeros(3, dtype=torch.uint8, device="cuda")
    stats = torch.zeros(3 * hb.ROLLOUT_STATS_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    P = lambda t: C.c_void_p(t.data_ptr())

    def commands():
        return hb.make_rollout_commands(["trot"] * 3, 0.0, [0.0, 0.2], [[0.1, 0, 0, 0], [0.2, 0, 0, 0]])

    def call(B=1, tick0=0, n_ticks=5, prm=None, cmds=None, null=None):
        args = dict(p=C.byref(prm or hb.default_rollout_params()), cmd=cmds or commands(), rbd=P(rbd), act=P(act), estop=P(estop), stats=P(stats))
        if null:
            args[null] = None
        return lib.hb_rollout_batch_dev(ctx._h, B, C.c_int64(tick0), n_ticks, args["p"], args["cmd"], args["rbd"], args["act"], args["estop"],
                                        args["stats"], None)

    c0 = ctx.launch_count
    for name in ("p", "cmd", "rbd", "act", "estop", "stats"):
        assert call(null=name) == -1, name
    assert call(B=-1) == -1 and call(n_ticks=-1) == -1
    for field, value in (("mpc_every", 0), ("period", 0.0), ("period", float("nan")), ("log_every", -1)):
        prm = hb.default_rollout_params()
        setattr(prm, field, value)
        assert call(prm=prm) == -1, field
    for change in ("n_cmd0", "n_cmd9", "unordered", "gait4", "gait-1"):
        cmds = commands()
        c = cmds[1]
        if change == "n_cmd0":
            c.n_cmd = 0
        elif change == "n_cmd9":
            c.n_cmd = hb.api.HB_ROLLOUT_MAX_CMDS + 1
        elif change == "unordered":
            c.cmd_time[1] = -0.1
        else:
            c.gait = int(change[4:])
        assert call(B=2, cmds=cmds) == -1, change
    assert call(tick0=5) == -1                        # no resident solution to continue from
    assert call(B=3) == -4
    assert call(B=0) == 0
    assert ctx.launch_count == c0
    ctx.close()


def test_launches_are_linear_in_cycles_and_ticks():
    """No per-tick host decisions beyond the cadence: a warm call launches a * (MPC cycles) + b * ticks kernels for fixed a, b."""
    ctx = context()
    B = 6
    a, b = launch_coefficients(ctx, start_states(ctx, B, seed=14), GAITS, cmd_vels(B), params())
    assert a > 0 and b > 0
    ctx.close()
