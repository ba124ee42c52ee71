"""Closed-loop episodes on the device (hb_rollout_batch_dev): one call runs, for a batch of robots, the device planner + resident MPC cycle
every mpc_every ticks and the 500 Hz policy + WeightedWbc tick, joint command law, actuation delay, saturation and plant step on every tick.
The call is checked bit for bit against the same loop written with the existing calls (one host round trip per operator), and against
itself: continuation, independence of instances, failure recording and holding, argument checks, launch counts."""
import ctypes as C

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc

pytestmark = pytest.mark.gpu

N, DT = 40, 0.02
GROUND = 0.02                      # the contact frames rest 2 cm above z = 0, as in test_dynamic_closed_loop_standing_rollout
GAITS = ["stance", "trot", "standing_trot", "trot", "standing_trot", "stance"]
GAIT_START = 0.1
CMD_TIMES = [0.0, 0.2]             # the command changes half way through a 200-tick episode


def _torch():
    import torch
    return torch


def _context(event_nodes=False, max_batch=8):
    if event_nodes:
        return hb.Context(horizon_N=N, dt=DT, max_batch=max_batch, device=0, time_horizon=0.6, event_nodes=True)
    return hb.Context(horizon_N=N, dt=DT, max_batch=max_batch, device=0)


def _start_states(ctx, B, seed):
    """Perturbed standing poses with the lowest contact frame 1 mm inside the ground (contact springs loaded from the start)."""
    rng = np.random.default_rng(seed)
    x0 = np.tile(sc.INITIAL_STATE, (B, 1))
    x0[:, 6:8] += rng.uniform(-0.02, 0.02, (B, 2)); x0[:, 9] = rng.uniform(-0.5, 0.5, B)
    x0[:, 12:] += rng.uniform(-0.02, 0.02, (B, 10))
    rbd = sc.consistent_rbd(x0)
    foot_z = ctx.contact_positions(x0).reshape(B, 4, 3)[:, :, 2].min(axis=1)
    rbd[:, 5] -= foot_z - (GROUND - 0.001)
    return rbd


def _cmd_vels(B):
    v = np.zeros((B, 2, 4))
    v[:, 0, 0] = 0.1
    v[:, 1, 0] = np.linspace(-0.2, 0.3, B); v[:, 1, 3] = 0.2
    return v


def _params(log_every=0):
    p = hb.default_rollout_params()
    p.sim.ground_height = GROUND
    p.log_every = log_every
    return p


def _horizon(ctx):
    return ctx.cfg.time_horizon if ctx.cfg.event_nodes else N * DT


def _stepwise(ctx, rbd, gaits, cmd_vels, n_ticks, prm, log_every):
    """The episode as a Python loop over existing calls only, with the checks / holding / stats restated in numpy."""
    B = rbd.shape[0]
    rbd = rbd.copy()
    act = hb.actuation_states(B)
    estop = np.zeros(B, dtype=np.uint8)
    st = hb.rollout_stats(B)
    held = rbd.copy()
    lim = np.array(prm.torque_limit[:])
    times = np.array(CMD_TIMES)
    logs = []
    for a in range(n_ticks):
        t = a * prm.period
        for i in range(B):                               # state entering the tick
            r = rbd[i]
            assert np.isfinite(r).all()
            why = (2 if (r[2] > np.pi / 2 or r[2] < -np.pi / 2) else 0) | (4 if prm.min_base_height != 0 and r[5] < prm.min_base_height else 0)
            if why and st["fail_tick"][i] < 0:
                st["fail_tick"][i] = a; st["fail_reason"][i] = why
            held[i] = r
        if log_every and a % log_every == 0:
            logs.append(rbd.copy())
        mpc = a % prm.mpc_every == 0
        if mpc:
            x0 = ctx.rbd_to_centroidal(rbd)
            cmd = cmd_vels[:, max(np.searchsorted(times, t, side="right") - 1, 0)]      # the last segment that has started
            ins = hb.make_plan_inputs(np.full(B, t), _horizon(ctx), x0, cmd, None, gaits, GAIT_START)
            info, _, _, _, ps = ctx.resident_plan_cycle(a == 0, 0.0, ins, rbd)
        xd, ud, md, sol, _, wst = ctx.resident_wbc(t, rbd)
        jcmd, _, estop = ctx.joint_command(prm.period, xd, ud, sol, md, rbd, estop=estop, gains=prm.gains)
        tau = ctx.actuation(t, act, jcmd, rbd, prm.actuation_delay)
        tau = np.clip(tau, -lim, lim)
        rbd, _, _ = ctx.sim_step(rbd, tau, prm.sim)
        for i in range(B):                               # after the plant step
            if st["fail_tick"][i] < 0:
                if mpc:
                    st["mpc_bad"][i] += info["status"][i] != 0; st["plan_rejects"][i] += ps[i] != 0
                st["wbc_fallbacks"][i] += wst[i] != 0
                m = st["max_abs_torque"][i]
                for v in np.abs(tau[i]):
                    if v > m:
                        m = v
                st["max_abs_torque"][i] = m
                if estop[i]:
                    st["fail_tick"][i] = a; st["fail_reason"][i] = 1
            restore = st["fail_tick"][i] >= 0
            if not restore and not np.isfinite(rbd[i]).all():
                restore = True; st["fail_tick"][i] = a + 1; st["fail_reason"][i] = 8
            if restore:
                rbd[i] = held[i]
    log = np.stack(logs, axis=1) if log_every else None
    return rbd, np.frombuffer(bytes(act), dtype=np.uint8), estop, st, log


def _device(ctx, rbd, gaits, cmd_vels, n_ticks, prm, log_every, tick0=0, act=None, estop=None, stats=None):
    torch = _torch()
    d_rbd = torch.from_numpy(np.ascontiguousarray(rbd)).cuda()
    cmds = hb.make_rollout_commands(gaits, GAIT_START, CMD_TIMES, cmd_vels)
    return ctx.rollout(d_rbd, cmds, n_ticks, tick0=tick0, params=prm, act=act, estop=estop, stats=stats, log_every=log_every)


def _assert_stats_equal(a, b):
    for k in hb.ROLLOUT_STATS_DTYPE.names:
        assert np.array_equal(a[k], b[k]), (k, a[k], b[k])


@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
def test_episode_equals_the_stepwise_loop_bitwise(event_nodes):
    """200 ticks of B = 6 mixed-gait episodes with a command change at 0.2 s: rbd, actuation state, estop, stats and log equal the loop
    of existing calls bit for bit. This holds because the cycle's own WBC at t_rel = 0 is the tick's WBC at the same time (same policy point,
    same kernel, same fallback state), so the call may skip it."""
    ctx = _context(event_nodes)
    B, n_ticks, log_every = 6, 200, 10
    rbd0 = _start_states(ctx, B, seed=11)
    vels = _cmd_vels(B)
    prm = _params(log_every)
    d_rbd, d_act, d_estop, d_st, d_log = _device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every)
    r_rbd, r_act, r_estop, r_st, r_log = _stepwise(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every)
    assert np.array_equal(d_rbd.cpu().numpy(), r_rbd)
    assert np.array_equal(d_act.cpu().numpy(), r_act)
    assert np.array_equal(d_estop.cpu().numpy(), r_estop)
    _assert_stats_equal(d_st, r_st)
    assert np.array_equal(d_log.cpu().numpy(), r_log)
    assert d_log.shape == (B, n_ticks // log_every, 32)
    assert np.isfinite(r_rbd).all() and not np.array_equal(r_rbd, rbd0)
    ctx.close()


def test_two_calls_continue_one_call_bitwise():
    ctx = _context()
    B = 6
    rbd0 = _start_states(ctx, B, seed=12)
    vels = _cmd_vels(B)
    prm = _params(10)
    one = _device(ctx, rbd0, GAITS, vels, 200, prm, 10)
    r1, act, es, st, log1 = _device(ctx, rbd0, GAITS, vels, 100, prm, 10)
    r2, act, es, st, log2 = ctx.rollout(r1, hb.make_rollout_commands(GAITS, GAIT_START, CMD_TIMES, vels), 100, tick0=100, params=prm, act=act,
                                        estop=es, stats=st, log_every=10)
    assert np.array_equal(one[0].cpu().numpy(), r2.cpu().numpy())
    assert np.array_equal(one[1].cpu().numpy(), act.cpu().numpy())
    assert np.array_equal(one[2].cpu().numpy(), es.cpu().numpy())
    _assert_stats_equal(one[3], st)
    assert np.array_equal(one[4].cpu().numpy(), np.concatenate([log1.cpu().numpy(), log2.cpu().numpy()], axis=1))
    ctx.close()


def test_instances_are_independent():
    ctx = _context()
    B, n_ticks, keep = 6, 100, [1, 3, 4]
    rbd0 = _start_states(ctx, B, seed=13)
    vels = _cmd_vels(B)
    prm = _params(5)
    full = _device(ctx, rbd0, GAITS, vels, n_ticks, prm, 5)
    part = _device(ctx, rbd0[keep], [GAITS[i] for i in keep], vels[keep], n_ticks, prm, 5)
    assert np.array_equal(full[0].cpu().numpy()[keep], part[0].cpu().numpy())
    size = C.sizeof(hb.HbActuationState)
    assert np.array_equal(full[1].cpu().numpy().reshape(B, size)[keep], part[1].cpu().numpy().reshape(len(keep), size))
    assert np.array_equal(full[2].cpu().numpy()[keep], part[2].cpu().numpy())
    _assert_stats_equal(full[3][keep], part[3])
    assert np.array_equal(full[4].cpu().numpy()[keep], part[4].cpu().numpy())
    ctx.close()


def test_standing_episode_keeps_the_robots_up():
    """The setup and bounds of test_dynamic_closed_loop_standing_rollout, driven through the planner and one rollout call (stance, zero
    command). The vertical contact force is the plant's spring force at the logged states, averaged over the last 50 ticks."""
    B, n_ticks = 4, 200
    ctx = hb.Context(horizon_N=50, dt=0.02, max_batch=B, device=0)
    rbd0 = _start_states(ctx, B, seed=2)
    z0 = rbd0[:, 5].copy()
    prm = _params(1)
    cmds = hb.make_rollout_commands(["stance"] * B, 0.0, [0.0], [[0.0, 0.0, 0.0, 0.0]])
    torch = _torch()
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
    ctx = _context()
    rbd0 = _start_states(ctx, B, seed=2)
    rbd0[2, 6 + 3] = sc.JOINT_UPPER[3] + 0.03
    rbd0[4, 2] = 1.7
    prm = _params(1)
    gaits = ["stance"] * B
    vels = np.zeros((B, 2, 4))
    rbd, act, estop, st, log = _device(ctx, rbd0, gaits, vels, n_ticks, prm, 1)
    rbd, log = rbd.cpu().numpy(), log.cpu().numpy()
    assert list(st["fail_tick"][[2, 4]]) == [0, 0] and list(st["fail_reason"][[2, 4]]) == [1, 2], st
    for i in (2, 4):
        assert np.array_equal(rbd[i], rbd0[i]) and (log[i] == rbd0[i]).all()
    others = [0, 1, 3, 5]
    assert (st["fail_tick"][others] == -1).all()
    ref = _device(ctx, rbd0[others], [gaits[i] for i in others], vels[others], n_ticks, prm, 1)
    assert np.array_equal(rbd[others], ref[0].cpu().numpy())
    assert np.array_equal(log[others], ref[4].cpu().numpy())
    _assert_stats_equal(st[others], ref[3])
    ctx.close()


def test_argument_checks_return_before_any_launch():
    torch = _torch()
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
    ctx = _context()
    B = 6
    rbd0 = _start_states(ctx, B, seed=14)
    vels = _cmd_vels(B)
    prm = _params()
    r, act, es, st, _ = _device(ctx, rbd0, GAITS, vels, 10, prm, 0)
    cmds = hb.make_rollout_commands(GAITS, GAIT_START, CMD_TIMES, vels)
    rows = []
    tick0 = 10
    for n in (10, 23, 7):
        cycles = sum(1 for a in range(tick0, tick0 + n) if a % prm.mpc_every == 0)
        c0 = ctx.launch_count
        r, act, es, st, _ = ctx.rollout(r, cmds, n, tick0=tick0, params=prm, act=act, estop=es, stats=st)
        rows.append((cycles, n, ctx.launch_count - c0))
        tick0 += n
    M = np.array([[c, n] for c, n, _ in rows[:2]], dtype=float)
    a, b = np.rint(np.linalg.solve(M, [d for _, _, d in rows[:2]])).astype(int)
    assert a > 0 and b > 0
    for c, n, d in rows:
        assert d == a * c + b * n, (rows, a, b)
    ctx.close()
