"""The batched closed-loop episode restated once for its tests (test_gpu_rollout_episodes.py, test_gpu_rollout_estimation.py,
test_gpu_rollout_pushes.py, test_gpu_rollout.py): the shared setup, the plant in numpy, the episode as a loop of public calls, and the
comparisons of episode outputs."""
import ctypes as C
import math

import numpy as np

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from estimation_ref import shortest_angular_distance

N, DT = 40, 0.02
GROUND = 0.02                      # the contact frames rest 2 cm above z = 0 (zero-velocity constraint pulls them there, LeggedInterface.cpp:436-444)
GAITS = ["stance", "trot", "standing_trot", "trot", "standing_trot", "stance"]
GAIT_START = 0.1
CMD_TIMES = [0.0, 0.2]             # the command changes half way through a 200-tick episode
SIGMAS = dict(orientation=0.002, angular_velocity=0.01, linear_acceleration=0.05, joint_position=0.001, joint_velocity=0.01)
OUTPUTS = ("rbd", "act", "estop", "stats", "log", "est", "est_stats", "est_log")      # Context.rollout_estimated's tuple; rollout's: the first 5


# ---------------------------------------------------------------------------------------------------------------- setup
def context(event_nodes=False, max_batch=8):
    if event_nodes:
        return hb.Context(horizon_N=N, dt=DT, max_batch=max_batch, device=0, time_horizon=0.6, event_nodes=True)
    return hb.Context(horizon_N=N, dt=DT, max_batch=max_batch, device=0)


def start_states(ctx, B, seed):
    """Perturbed standing poses with the lowest contact frame 1 mm inside the ground (contact springs loaded from the start)."""
    rng = np.random.default_rng(seed)
    x0 = np.tile(sc.INITIAL_STATE, (B, 1))
    x0[:, 6:8] += rng.uniform(-0.02, 0.02, (B, 2)); x0[:, 9] = rng.uniform(-0.5, 0.5, B)
    x0[:, 12:] += rng.uniform(-0.02, 0.02, (B, 10))
    rbd = sc.consistent_rbd(x0)
    foot_z = ctx.contact_positions(x0).reshape(B, 4, 3)[:, :, 2].min(axis=1)
    rbd[:, 5] -= foot_z - (GROUND - 0.001)
    return rbd


def cmd_vels(B):
    v = np.zeros((B, 2, 4))
    v[:, 0, 0] = 0.1
    v[:, 1, 0] = np.linspace(-0.2, 0.3, B); v[:, 1, 3] = 0.2
    return v


def params(log_every=0):
    p = hb.default_rollout_params()
    p.sim.ground_height = GROUND
    p.log_every = log_every
    return p


def horizon(ctx):
    return ctx.cfg.time_horizon if ctx.cfg.event_nodes else N * DT


def noise(seed, scale=1.0):
    n = hb.HbSensorNoise()
    n.seed = seed
    for k, v in SIGMAS.items():
        setattr(n, k, scale * v)
    return n


def est_params(seed=0, scale=1.0):
    ep = hb.default_estimation_params()
    ep.noise = noise(seed, scale)
    return ep


# ---------------------------------------------------------------------------------------------------------------- the plant
def T(zyx):
    """omega_world = T(zyx) (yaw, pitch, roll rates): the columns are the world axes of the three rotations."""
    sz, cz, sy, cy = np.sin(zyx[0]), np.cos(zyx[0]), np.sin(zyx[1]), np.cos(zyx[1])
    return np.array([[0.0, -sz, cz * cy], [0.0, cz, sz * cy], [1.0, 0.0, -sy]])


def plant_numpy(oracle, rbd, tau, prm, wrench=None):
    """One plant step of one robot: returns (rbd_next, contact forces of the last substep). wrench (6,): an external world force at the base
    origin and a world couple, Q_p = f, Q_zyx = T' tau at each substep's orientation; None adds no generalised force."""
    from oracle import refs
    q = np.concatenate([rbd[3:6], rbd[0:3], rbd[6:16]])
    v = np.concatenate([rbd[19:22], refs.euler_rates_from_global(rbd[0:3], rbd[16:19]), rbd[22:32]])
    h = prm.dt / prm.substeps
    F = np.zeros(12)
    for _ in range(prm.substeps):
        r = oracle.rbd(q, v)
        cvel = r["J"] @ v
        F = np.zeros(12)
        for c in range(4):
            depth = prm.ground_height - r["cpos"][3 * c + 2]
            if depth > 0:
                fz = max(0.0, prm.ground_stiffness * depth - prm.ground_damping * cvel[3 * c + 2])
                ft = -prm.tangential_damping * cvel[3 * c:3 * c + 2]
                n = np.linalg.norm(ft)
                if n > prm.friction_mu * fz:
                    ft = ft * (prm.friction_mu * fz / n if n > 0 else 0.0)
                F[3 * c:3 * c + 3] = [ft[0], ft[1], fz]
        rhs = np.concatenate([np.zeros(6), tau - prm.joint_damping * v[6:]]) + r["J"].T @ F - r["nle"]
        if wrench is not None:
            rhs = rhs + np.concatenate([wrench[:3], T(q[3:6]).T @ wrench[3:], np.zeros(10)])
        qdd = np.linalg.solve(r["M"] + np.diag(np.r_[np.zeros(6), np.full(10, prm.joint_armature)]), rhs)
        v = v + h * qdd
        q = q + h * v
    out = np.zeros(32)
    out[0:3] = q[3:6]; out[3:6] = q[0:3]; out[6:16] = q[6:]
    out[16:19] = refs.global_from_euler_rates(q[3:6], v[3:6]); out[19:22] = v[0:3]; out[22:32] = v[6:]
    return out, F


def wrench_numpy(pushes, t, B):
    """The documented wrench of the tick at time t: zeros, plus every active push in ascending j (B x 6; instances without a schedule: 0)."""
    w = np.zeros((B, 6))
    for i in range(min(B, len(pushes))):
        s = pushes[i]
        for j in range(s.n_push):
            if s.t_start[j] <= t and t < s.t_start[j] + s.duration[j]:
                for c in range(3):
                    w[i, c] += s.force[j][c]; w[i, 3 + c] += s.torque[j][c]
    return w


# ---------------------------------------------------------------------------------------------------------------- the episode
def _mode_at(st, t):
    idx = 0
    while idx < st.n_events and st.event_times[idx] < t:
        idx += 1
    return st.modes[idx]


def stepwise(ctx, rbd0, gaits, cmd_vels, n_ticks, prm, log_every, ep=None, est=None, pushes=None):
    """The episode as a Python loop of public calls from tick 0, with the checks, holding and stats restated in numpy. It is the device
    loop (rollout_impl) tick for tick: with ep and est (fresh estimation states, advanced in place) it is the estimated episode, whose
    controllers read the filter's estimate, and the estimation steps sit where the device loop's estimation branches sit. pushes: the
    schedules set on ctx, applied as each tick's wrench. Returns the tuple of Context.rollout, or of Context.rollout_estimated with ep."""
    B = rbd0.shape[0]
    rbd = rbd0.copy()
    act = hb.actuation_states(B)
    estop = np.zeros(B, dtype=np.uint8)
    st = hb.rollout_stats(B)
    held = rbd.copy()
    lim = np.array(prm.torque_limit[:])
    times = np.array(CMD_TIMES)
    logs = []
    if ep is not None:
        es = hb.estimation_stats(B)
        kf = hb.kf_states(B)
        stance = np.zeros((B, 12))
        est_logs = []
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
        meas = rbd                                       # what the controllers measure: the true state, or the filter's estimate
        if ep is not None:
            # sensors and contact flags at the previous observation's time, filter, observation step (yaw unwrap, estimation stats)
            quat, w, acc, jp, jv = ctx.read_sensors(rbd, est, a, ep.noise, accel_dt=prm.sim.dt)
            flags = np.ones((B, 4), dtype=np.uint8)
            for i in range(B):
                if est[i].has_plan:
                    m = _mode_at(est[i], (a - 1) * prm.period)
                    flags[i] = [1 if (m in (1, 3) if c & 1 else m in (2, 3)) else 0 for c in range(4)]
            meas = ctx.estimator_update(prm.period, kf, quat, w, acc, jp, jv, flags, params=ep.kf)
            for i in range(B):
                est[i].yaw_obs = est[i].yaw_obs + shortest_angular_distance(est[i].yaw_obs, meas[i, 0])
                if st["fail_tick"][i] < 0:
                    d = [float(meas[i, 19 + k] - rbd[i, 19 + k]) for k in range(3)]
                    sq = d[0] * d[0] + d[1] * d[1] + d[2] * d[2]
                    ve, dz = math.sqrt(sq), abs(float(meas[i, 5] - rbd[i, 5]))
                    if ve > es["max_vel_err"][i]:
                        es["max_vel_err"][i] = ve
                    if dz > es["max_height_err"][i]:
                        es["max_height_err"][i] = dz
                    es["sum_sq_vel_err"][i] += sq; es["sum_sq_height_err"][i] += dz * dz; es["count"][i] += 1
            if log_every and a % log_every == 0:
                est_logs.append(meas.copy())
        mpc = a % prm.mpc_every == 0
        if mpc:
            x0 = ctx.rbd_to_centroidal(meas)
            if ep is not None:
                x0[:, 9] = [est[i].yaw_obs for i in range(B)]
            cmd = cmd_vels[:, max(np.searchsorted(times, t, side="right") - 1, 0)]      # the last segment that has started
            ins = hb.make_plan_inputs(np.full(B, t), horizon(ctx), x0, cmd, None, gaits, GAIT_START)
            info, _, _, _, ps = ctx.resident_plan_cycle(a == 0, 0.0, ins, meas)
            if ep is not None:
                # the plan's schedule copied into the estimation state, for the next ticks' contact flags
                refs, stance, _ = ctx.plan_references_gpu(hb.make_plan_inputs(np.full(B, t), horizon(ctx), x0, cmd, ctx.contact_positions(x0), gaits,
                                                                              GAIT_START), stance)
                for i in range(B):
                    n = refs[i].n_events
                    est[i].n_events = n
                    for k in range(n):
                        est[i].event_times[k] = refs[i].event_times[k]
                    for k in range(n + 1):
                        est[i].modes[k] = refs[i].modes[k]
                    est[i].has_plan = 1
        xd, ud, md, sol, _, wst = ctx.resident_wbc(t, meas)
        jcmd, _, estop = ctx.joint_command(prm.period, xd, ud, sol, md, meas, estop=estop, gains=prm.gains)
        tau = ctx.actuation(t, act, jcmd, rbd, prm.actuation_delay)
        tau = np.clip(tau, -lim, lim)
        rbd, _, _ = ctx.sim_step(rbd, tau, prm.sim, wrench=None if pushes is None else wrench_numpy(pushes, t, B))
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
    out = (rbd, np.frombuffer(bytes(act), dtype=np.uint8), estop, st, log)
    if ep is None:
        return out
    for i in range(B):
        est[i].kf = kf[i]
    return out + (est, es, np.stack(est_logs, axis=1) if log_every else None)


def device(ctx, rbd0, gaits, cmd_vels, n_ticks, prm, log_every, ep=None, est=None, tick0=0, act=None, estop=None, stats=None, est_stats=None):
    """Context.rollout, or with ep Context.rollout_estimated, with the commands of gaits, GAIT_START, CMD_TIMES and cmd_vels. rbd0: host
    states or the cuda tensor of a previous call; est: ctypes estimation states, the cuda tensor of a previous call, or None (fresh)."""
    import torch
    d_rbd = rbd0 if hasattr(rbd0, "cpu") else torch.from_numpy(np.ascontiguousarray(rbd0)).cuda()
    cmds = hb.make_rollout_commands(gaits, GAIT_START, CMD_TIMES, cmd_vels)
    if ep is None:
        return ctx.rollout(d_rbd, cmds, n_ticks, tick0=tick0, params=prm, act=act, estop=estop, stats=stats, log_every=log_every)
    if isinstance(est, C.Array):
        est = torch.from_numpy(np.frombuffer(bytes(est), dtype=np.uint8).copy()).cuda()
    return ctx.rollout_estimated(d_rbd, cmds, n_ticks, tick0=tick0, params=prm, est_params=ep, est=est, act=act, estop=estop, stats=stats,
                                 est_stats=est_stats, log_every=log_every)


def _resume(ctx, out, gaits, cmd_vels, n_ticks, tick0, prm, log_every, ep):
    """The call that continues the episode call whose tuple is out, from tick tick0."""
    if ep is None:
        return device(ctx, out[0], gaits, cmd_vels, n_ticks, prm, log_every, tick0=tick0, act=out[1], estop=out[2], stats=out[3])
    return device(ctx, out[0], gaits, cmd_vels, n_ticks, prm, log_every, ep, out[5], tick0=tick0, act=out[1], estop=out[2], stats=out[3],
                  est_stats=out[6])


# ---------------------------------------------------------------------------------------------------------------- comparisons
def outputs(out):
    """An episode tuple (device or stepwise) as numpy arrays with one row per instance: the actuation and estimation states as
    (B, record size) bytes."""
    o = [np.frombuffer(bytes(x), dtype=np.uint8) if isinstance(x, C.Array) else x.cpu().numpy() if hasattr(x, "cpu") else x for x in out]
    B = o[0].shape[0]
    o[1] = o[1].reshape(B, C.sizeof(hb.HbActuationState))
    if len(o) > 5:
        o[5] = o[5].reshape(B, C.sizeof(hb.HbEstimationState))
    return o


def assert_episode_equal(a, b, rows_a=slice(None), rows_b=slice(None)):
    """Every output of two episodes equal bit for bit, instances rows_a of a against instances rows_b of b."""
    a, b = outputs(a), outputs(b)
    assert len(a) == len(b)
    for name, x, y in zip(OUTPUTS, a, b):
        x, y = x[rows_a], y[rows_b]
        if x.dtype.names:
            for k in x.dtype.names:
                assert np.array_equal(x[k], y[k]), (name, k, x[k], y[k])
        elif name == "est" and not np.array_equal(x, y):
            fields = [(f, getattr(hb.HbEstimationState, f)) for f, _ in hb.HbEstimationState._fields_]
            bad = [f for f, d in fields if not np.array_equal(x[:, d.offset:d.offset + d.size], y[:, d.offset:d.offset + d.size])]
            raise AssertionError("estimation state differs in %s" % bad)
        else:
            assert np.array_equal(x, y), name


def assert_continues(ctx, rbd0, gaits, cmd_vels, n_ticks, split, prm, log_every, ep=None):
    """One call of n_ticks equals two calls split at tick `split`, the second continuing the first, bit for bit (the logs joined)."""
    one = device(ctx, rbd0, gaits, cmd_vels, n_ticks, prm, log_every, ep)
    first = device(ctx, rbd0, gaits, cmd_vels, split, prm, log_every, ep)
    two = outputs(_resume(ctx, first, gaits, cmd_vels, n_ticks - split, split, prm, log_every, ep))
    two[4] = np.concatenate([first[4].cpu().numpy(), two[4]], axis=1)
    if ep is not None:
        two[7] = np.concatenate([first[7].cpu().numpy(), two[7]], axis=1)
    assert_episode_equal(one, two)


def launch_coefficients(ctx, rbd0, gaits, cmd_vels, prm, ep=None):
    """Warm calls continuing a 10-tick episode launch a * (MPC cycles) + b * ticks kernels for fixed a, b, asserted over three calls of
    10, 23 and 7 ticks: no per-tick host decisions beyond the cadence. Returns (a, b)."""
    out = device(ctx, rbd0, gaits, cmd_vels, 10, prm, 0, ep)
    rows = []
    tick0 = 10
    for n in (10, 23, 7):
        cycles = sum(1 for a in range(tick0, tick0 + n) if a % prm.mpc_every == 0)
        c0 = ctx.launch_count
        out = _resume(ctx, out, gaits, cmd_vels, n, tick0, prm, 0, ep)
        rows.append((cycles, n, ctx.launch_count - c0))
        tick0 += n
    M = np.array([[c, n] for c, n, _ in rows[:2]], dtype=float)
    a, b = np.rint(np.linalg.solve(M, [d for _, _, d in rows[:2]])).astype(int)
    for c, n, d in rows:
        assert d == a * c + b * n, (rows, a, b)
    return a, b
