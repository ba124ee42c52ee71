"""The batched closed-loop episode restated once for its tests (test_gpu_rollout*.py and the tests of the other per-robot settings): the
shared setup, the plant in numpy, the episode with every per-robot setting as one loop of public calls (stepwise), the comparisons of
episode outputs, and the checks and data shared by the settings."""
import ctypes as C
import math

import numpy as np
import pytest

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
G = 9.81


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
    return ctx.cfg.time_horizon if ctx.cfg.event_nodes else ctx.N * ctx.dt


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


def payload_terms(q, v, variation):
    """The payload of a plant variation in the base coordinates (p, zyx) of q, v: (M_p, nle_p), the 6 x 6 base block it adds to M and the 6
    entries it adds to nle, from the documented formulas: with omega = T zyx_dot, r = R c and I_w = R I_c R', column k of M_p is
    [F; T' n] for F = m (pdd + omega_dot x r), n = I_w omega_dot + r x F at a unit acceleration of coordinate k and v = 0; nle_p is the
    same with omega_dot0 = (omega_1 x a_pitch) dpitch + (omega_2 x a_roll) droll, F = m (omega_dot0 x r + omega x (omega x r)) + m g e_z,
    n = I_w omega_dot0 + omega x I_w omega + r x F."""
    from oracle import refs
    m = variation.payload_mass
    c = np.array(variation.payload_com[:]); Ic = np.array(variation.payload_inertia[:]).reshape(3, 3)
    R, Tm = refs.rot_zyx(q[3:6]), T(q[3:6])
    r, Iw = R @ c, R @ Ic @ R.T
    M = np.zeros((6, 6))
    for k in range(6):
        a = np.zeros(6); a[k] = 1.0
        wd = Tm @ a[3:]
        F = m * (a[:3] + np.cross(wd, r))
        M[:, k] = np.r_[F, Tm.T @ (Iw @ wd + np.cross(r, F))]
    dz = v[3:6]
    w1 = Tm[:, 0] * dz[0]; w2 = w1 + Tm[:, 1] * dz[1]; w = Tm @ dz
    wd0 = np.cross(w1, Tm[:, 1]) * dz[1] + np.cross(w2, Tm[:, 2]) * dz[2]
    F = m * (np.cross(wd0, r) + np.cross(w, np.cross(w, r))) + m * G * np.array([0.0, 0.0, 1.0])
    n = Iw @ wd0 + np.cross(w, Iw @ w) + np.cross(r, F)
    return M, np.r_[F, Tm.T @ n]


def _axis(x, origin, spacing, n):
    """(cell index, fraction, clamped) of world coordinate x along one grid axis; NaN clamps to 0 as the kernel does."""
    u = (x - origin) / spacing
    clamped = False
    if not u >= 0.0:
        u, clamped = 0.0, True
    elif u > n - 1:
        u, clamped = float(n - 1), True
    i = min(int(math.floor(u)), n - 2)
    return i, u - i, clamped


def terrain_height(t, x, y):
    """(h, g_x, g_y) of the HbTerrain t at world (x, y), as hunter_b200.h documents it."""
    i, a, cx = _axis(x, t.origin[0], t.spacing, t.nx)
    j, b, cy = _axis(y, t.origin[1], t.spacing, t.ny)
    h00, h01, h10, h11 = t.height[j][i], t.height[j][i + 1], t.height[j + 1][i], t.height[j + 1][i + 1]
    h0 = h00 + a * (h01 - h00)
    h1 = h10 + a * (h11 - h10)
    d0, d1 = h01 - h00, h11 - h10
    gx = 0.0 if cx else (d0 + b * (d1 - d0)) / t.spacing
    gy = 0.0 if cy else (h1 - h0) / t.spacing
    return h0 + b * (h1 - h0), gx, gy


def contact_numpy(p, v, ground, k, d, ct, mu):
    """(force (3,), normal force) of one contact point at p with velocity v on the ground (h, g_x, g_y) under it, with ground stiffness k,
    damping d, tangential damping ct and friction coefficient mu: the flat path where the gradient is zero, the sloped path elsewhere."""
    h, gx, gy = ground
    if gx == 0.0 and gy == 0.0:
        depth = h - p[2]
        if not depth > 0:
            return np.zeros(3), 0.0
        fz = max(0.0, k * depth - d * v[2])
        ft = -ct * v[:2]
        n = np.linalg.norm(ft)
        if n > mu * fz:
            ft = ft * (mu * fz / n if n > 0 else 0.0)
        return np.array([ft[0], ft[1], fz]), fz
    L = math.sqrt(1.0 + gx * gx + gy * gy)
    n = np.array([-gx, -gy, 1.0]) / L
    depth = (h - p[2]) / L
    if not depth > 0:
        return np.zeros(3), 0.0
    vn = float(v @ n)
    fn = max(0.0, k * depth - d * vn)
    ft = -ct * (v - vn * n)
    tl = np.linalg.norm(ft)
    if tl > mu * fn:
        ft = ft * (mu * fn / tl if tl > 0 else 0.0)
    return fn * n + ft, fn


def plant_numpy(oracle, rbd, tau, prm, wrench=None, variation=None, terrain=None):
    """One plant step of one robot: returns (rbd_next, contact forces of the last substep (12,), contact flags of the last substep (4,)).
    wrench (6,): an external world force at the base origin and a world couple, Q_p = f, Q_zyx = T' tau at each substep's orientation.
    variation (an HbPlantVariation): the ground stiffness, damping and friction scaled, the joint torques scaled by the motor strengths and,
    with a payload, payload_terms added to M and nle. terrain (an HbTerrain): each contact on the ground terrain_height gives under it.
    None is no wrench, the nominal plant, and flat ground at prm.ground_height."""
    from oracle import refs
    q = np.concatenate([rbd[3:6], rbd[0:3], rbd[6:16]])
    v = np.concatenate([rbd[19:22], refs.euler_rates_from_global(rbd[0:3], rbd[16:19]), rbd[22:32]])
    h = prm.dt / prm.substeps
    k_g, d_g, mu = prm.ground_stiffness, prm.ground_damping, prm.friction_mu
    if variation is not None:
        k_g, d_g, mu = k_g * variation.stiffness_scale, d_g * variation.damping_scale, mu * variation.friction_scale
        tau = np.array(variation.motor_strength[:]) * tau
    F, flags = np.zeros(12), np.zeros(4, dtype=bool)
    for _ in range(prm.substeps):
        r = oracle.rbd(q, v)
        M, nle = r["M"].copy(), r["nle"].copy()
        if variation is not None and variation.payload_mass > 0:
            Mp, nlep = payload_terms(q, v, variation)
            M[:6, :6] += Mp; nle[:6] += nlep
        cvel = r["J"] @ v
        F = np.zeros(12)
        for c in range(4):
            p = r["cpos"][3 * c:3 * c + 3]
            ground = (prm.ground_height, 0.0, 0.0) if terrain is None else terrain_height(terrain, p[0], p[1])
            F[3 * c:3 * c + 3], fn = contact_numpy(p, cvel[3 * c:3 * c + 3], ground, k_g, d_g, prm.tangential_damping, mu)
            flags[c] = fn > 0
        rhs = np.concatenate([np.zeros(6), tau - prm.joint_damping * v[6:]]) + r["J"].T @ F - nle
        if wrench is not None:
            rhs = rhs + np.concatenate([wrench[:3], T(q[3:6]).T @ wrench[3:], np.zeros(10)])
        qdd = np.linalg.solve(M + np.diag(np.r_[np.zeros(6), np.full(10, prm.joint_armature)]), rhs)
        v = v + h * qdd
        q = q + h * v
    out = np.zeros(32)
    out[0:3] = q[3:6]; out[3:6] = q[0:3]; out[6:16] = q[6:]
    out[16:19] = refs.global_from_euler_rates(q[3:6], v[3:6]); out[19:22] = v[0:3]; out[22:32] = v[6:]
    return out, F, flags


def flat_terrain(height, center=(0.0, 0.0), spacing=0.5):
    """One flat HbTerrain at `height`: a 2 x 2 grid around `center`."""
    return hb.make_terrains(1, np.full((2, 2), height), spacing, np.asarray(center) - 0.5 * spacing)[0]


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


def latency_due(lat, a, every):
    """The flags of the instances with MPC latencies lat (0 beyond the setting) whose solution comes into force on tick a: the MRT's
    adoption d >= 1 ticks after each cycle."""
    return (lat >= 1) & (a >= lat) & ((a - lat) % every == 0)


def _padded(items, B, default):
    """The B records of a per-robot setting: items, then `default` beyond them."""
    return (type(default) * B)(*[items[i] if i < len(items) else default for i in range(B)])


def stepwise(ctx, rbd0, gaits, cmd_vels, n_ticks, prm, log_every, ep=None, est=None, pushes=None, plant_variations=None, terrains=None,
             goals=None, mpc_latencies=None, odometry=None, hardware=None):
    """The episode as a Python loop of public calls from tick 0, with the checks, holding and stats restated in numpy. It is the device
    loop (rollout_impl) tick for tick, each step in its place there: with ep and est (fresh estimation states, advanced in place) it is the
    estimated episode, whose controllers read the filter's estimate. The per-robot settings are those on ctx, under the names of their
    Context.set_<name>; one not given is unset. Each is restated by the public calls that take it, padded beyond its instances as the
    setting is documented:
    - pushes: each tick's wrench (wrench_numpy).
    - plant_variations, terrains: every plant step, on the default variation and flat ground at prm.sim.ground_height beyond them. The
      height check here is the absolute one, so with terrains this restates the episode only for prm.min_base_height = 0 (params()).
    - goals: on each MPC tick the goal in force is converted by hb_goal_to_target on the tick's x0 when it differs from the captured one,
      and every instance gets its target through hb_plan_set_targets: the captured one, or its cmd_vel target as the device planner
      builds it. The cold tick 0 starts with no goal captured.
    - mpc_latencies: the MRT split. The instances due adopt (hb_policy_update) before the tick's cycle, and on the cold tick every
      instance with a latency adopts after it; the latency-0 instances adopt the resident solution on every tick, then the tick's WBC is
      hb_policy_wbc. The public cycle runs its own WBC on the new solution, which the episodes do not, so the loop equals the episode
      while no WBC falls back.
    - odometry (estimated episodes; the cameras are ctx's): the camera read (hb_sim_read_odometry) after each sensor read, the fusion
      (hb_estimator_fuse_odometry) after each filter update.
    - hardware: the sensor read (hb_sim_read_sensors_hw) and the actuation (hb_actuation_hw) on the records, padded with the call's values
      (call_hardware(prm, ep)), and each robot's torques clipped to its record's limits; unset, the call's delay and prm.torque_limit.
    Controller and planner settings need no restating: the planner calls read ctx's planner settings, and the hardware test restates a
    controller record as ctx's WBC settings and prm.gains. Returns the tuple of Context.rollout, or of Context.rollout_estimated with ep."""
    B = rbd0.shape[0]
    var = None if plant_variations is None else _padded(plant_variations, B, hb.default_plant_variation())
    ter = None
    if terrains is not None:
        assert prm.min_base_height == 0
        ter = _padded(terrains, B, flat_terrain(prm.sim.ground_height))
    lat = None if mpc_latencies is None else np.array([mpc_latencies[i] if i < len(mpc_latencies) else 0 for i in range(B)])
    captured = {}                                        # instance: (index of its captured goal, that goal's target)
    hw = None
    lim = np.array(prm.torque_limit[:])
    if hardware is not None:
        from hardware_ref import call_hardware           # hardware_ref imports this module
        hw = _padded(hardware, B, call_hardware(prm, ep))
        lim = np.array([h.torque_limit[:] for h in hw])
    rbd = rbd0.copy()
    act = hb.actuation_states(B)
    estop = np.zeros(B, dtype=np.uint8)
    st = hb.rollout_stats(B)
    held = rbd.copy()
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
            quat, w, acc, jp, jv = ctx.read_sensors(rbd, est, a, ep.noise, accel_dt=prm.sim.dt, hardware=hw)
            if odometry is not None:
                msg = ctx.read_odometry(rbd, est, a, ep.noise)
            flags = np.ones((B, 4), dtype=np.uint8)
            for i in range(B):
                if est[i].has_plan:
                    m = _mode_at(est[i], (a - 1) * prm.period)
                    flags[i] = [1 if (m in (1, 3) if c & 1 else m in (2, 3)) else 0 for c in range(4)]
            meas = ctx.estimator_update(prm.period, kf, quat, w, acc, jp, jv, flags, params=ep.kf)
            if odometry is not None:
                meas = ctx.fuse_odometry(kf, *msg, flags, meas, params=ep.kf)
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
        if lat is not None:
            due = latency_due(lat, a, prm.mpc_every)
            if due.any():
                ctx.policy_update(B, due)
        mpc = a % prm.mpc_every == 0
        if mpc:
            x0 = ctx.rbd_to_centroidal(meas)
            if ep is not None:
                x0[:, 9] = [est[i].yaw_obs for i in range(B)]
            cmd = cmd_vels[:, max(np.searchsorted(times, t, side="right") - 1, 0)]      # the last segment that has started
            if goals is not None:
                ctx.set_plan_targets(None)
                plain, _, pst = ctx.plan_references_gpu(hb.make_plan_inputs(np.full(B, t), horizon(ctx), x0, cmd, None, gaits, GAIT_START,
                                                                            joint_ik=False), np.zeros((B, 12)))
                assert (pst == 0).all()
                targets = [hb.reference_target(r) for r in plain]
                for i in range(min(B, len(goals))):
                    s = goals[i]
                    g = max([j for j in range(s.n_goal) if s.time[j] <= t], default=-1)
                    if g >= 0 and captured.get(i, (-1,))[0] != g:
                        captured[i] = (g, hb.goal_to_target(t, x0[i:i + 1], np.array(s.goal[g][:]))[0])
                    if i in captured:
                        targets[i] = captured[i][1]
                ctx.set_plan_targets((hb.HbTarget * B)(*targets))
            ins = hb.make_plan_inputs(np.full(B, t), horizon(ctx), x0, cmd, None, gaits, GAIT_START)
            info, _, _, _, ps = ctx.resident_plan_cycle(a == 0, 0.0, ins, meas)
            if lat is not None and a == 0 and (lat >= 1).any():
                ctx.policy_update(B, lat >= 1)
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
        if lat is None:
            xd, ud, md, sol, _, wst = ctx.resident_wbc(t, meas)
        else:
            ctx.policy_update(B, lat == 0)
            xd, ud, md, sol, _, wst = ctx.policy_wbc(t, meas)
        jcmd, _, estop = ctx.joint_command(prm.period, xd, ud, sol, md, meas, estop=estop, gains=prm.gains)
        tau = ctx.actuation(t, act, jcmd, rbd, prm.actuation_delay, hardware=hw)
        tau = np.clip(tau, -lim, lim)
        rbd, _, _ = ctx.sim_step(rbd, tau, prm.sim, wrench=None if pushes is None else wrench_numpy(pushes, t, B), variation=var, terrain=ter)
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


# ---------------------------------------------------------------------------------------------------------------- per-robot settings
# Every per-robot setting of the episodes (Context.set_<name>, hb_rollout_set_*) has one contract. The checks below take the setting's name
# and each test file's own data.
FRICTION = [1.0, 0.8, 1.0, 0.6, 1.0, 0.9]          # ground friction scales of six robots
PUSH = [[25.0, -15.0, 0.0]]                         # one push of 25 N forward and 15 N to the right


def small_terrains():
    """Three flat terrains, at GROUND, 5 mm above and 4 mm below it: 2 x 2 grids at (-2, -2), beyond which the robots stand on the
    clamped edge heights."""
    return hb.make_terrains(3, np.full((3, 2, 2), [[[0.0]], [[0.005]], [[-0.004]]]) + GROUND, 0.5, (-2.0, -2.0))


def random_goals(rbd0, B, seed):
    """Goal schedules of the first B - 1 of the robots: a goal 0.15-0.4 m away in a random direction given between two MPC ticks, a second
    one later for every other robot, and the goal at the start pose from the start for the robot at index 2."""
    rng = np.random.default_rng(seed)
    n = B - 1
    d = rng.uniform(0.15, 0.4, n); th = rng.uniform(-np.pi, np.pi, n)
    g1 = np.c_[rbd0[:n, 3] + d * np.cos(th), rbd0[:n, 4] + d * np.sin(th), rbd0[:n, 0] + rng.uniform(-0.6, 0.6, n)]
    g2 = g1 + np.c_[rng.uniform(-0.2, 0.2, (n, 2)), rng.uniform(-0.3, 0.3, n)]
    times = np.c_[np.full(n, 0.053), np.where(np.arange(n) % 2, 0.21, 1e9)]
    s = hb.make_goal_schedules(n, times, np.stack([g1, g2], axis=1))
    s[2].n_goal = 1; s[2].time[0] = 0.0
    s[2].goal[0][0], s[2].goal[0][1], s[2].goal[0][2] = rbd0[2, 3], rbd0[2, 4], rbd0[2, 0]
    return s


def use(ctx, **settings):
    """Sets each setting on ctx (Context.set_<name>(value)) and returns them: stepwise's keyword arguments for the same episode."""
    for name, value in settings.items():
        getattr(ctx, "set_" + name)(value)
    return settings


def array_of(records):
    """A ctypes array of the records (all of one type)."""
    return (type(records[0]) * len(records))(*records)


def logged_episode(ctx, rbd0, prm, ep, n_ticks=100, streams=50):
    """The episode of the instances rbd0 with GAITS and cmd_vels, logged every 10 ticks, as outputs(): estimated with ep (fresh estimation
    states from noise stream `streams`), truth without."""
    B = rbd0.shape[0]
    est = hb.estimation_states(B, streams) if ep is not None else None
    return outputs(device(ctx, rbd0, GAITS, cmd_vels(B), n_ticks, prm, 10, ep, est))


def assert_records_act_as_their_values(ctx, name, records, values, rbd0, prm, ep, n_ticks=100, streams=50):
    """The records of the setting cycled over the 2 len(records) instances rbd0 (logged_episode): instance i with record k gives bit for
    bit what it gives with the setting cleared and record k's values given another way, `with values(ctx, record, prm, ep) as (prm_k,
    ep_k)` (a context manager that undoes on exit what it changed on ctx); and every instance moves against the unset episode, so the
    records really act."""
    set_ = getattr(ctx, "set_" + name)
    n = len(records)
    set_(array_of([records[i % n] for i in range(2 * n)]))
    got = logged_episode(ctx, rbd0, prm, ep, n_ticks, streams)
    set_(None)
    for k, rec in enumerate(records):
        with values(ctx, rec, prm, ep) as (p, e):
            want = logged_episode(ctx, rbd0, p, e, n_ticks, streams)
        assert_episode_equal(got, want, rows_a=[k, k + n], rows_b=[k, k + n])
    ref = logged_episode(ctx, rbd0, prm, ep, n_ticks, streams)
    for i in range(2 * n):
        assert not np.array_equal(got[0][i], ref[0][i]), i


def _counted(ctx, run):
    c0 = ctx.launch_count
    out = run()
    return out, ctx.launch_count - c0


def assert_setting_episodes(ctx, name, rbd0, prm, full, one, other, row, part, padded, cont=None):
    """The setting on 200-tick episodes of the six instances rbd0, with log_every = 10: set to `cont` (default `full`), two calls split at
    tick 100 equal one; `one` (only instance 0 differs from the unset episode) moves instance 0 and leaves the others as unset; instance
    `row` of `other` equals instance `row` of `full`, whatever the other instances have; a permuted batch with the permuted setting gives the
    permuted result; `part`, a setting of the first k instances, moves them, leaves the others as unset and equals `padded`, the full
    setting it is documented to be; B = 0 clears the setting."""
    set_ = getattr(ctx, "set_" + name)
    B = rbd0.shape[0]
    vels = cmd_vels(B)

    def run(rbd=rbd0, gaits=GAITS, v=vels):
        return outputs(device(ctx, rbd, gaits, v, 200, prm, 10))

    set_(full if cont is None else cont)
    assert_continues(ctx, rbd0, GAITS, vels, 200, 100, prm, 10)
    set_(None)
    u = run()
    set_(one)
    p = run()
    assert not np.array_equal(p[0][0], u[0][0])
    assert_episode_equal(p, u, rows_a=slice(1, None), rows_b=slice(1, None))
    set_(full)
    f = run()
    set_(other)
    assert_episode_equal(f, run(), rows_a=[row], rows_b=[row])
    perm = [4, 0, 5, 2, 1, 3]
    set_((type(full[0]) * B)(*[full[i] for i in perm]))
    assert_episode_equal(f, run(rbd0[perm], [GAITS[i] for i in perm], vels[perm]), rows_a=perm)
    k = len(part)
    set_(part)
    pt = run()
    set_(padded)
    assert_episode_equal(pt, run())
    assert_episode_equal(pt, u, rows_a=slice(k, None), rows_b=slice(k, None))
    assert not np.array_equal(pt[0][:k], u[0][:k])
    assert getattr(ctx._lib, "hb_rollout_set_" + name)(ctx._h, 0, None) == 0
    assert_episode_equal(run(), u)


def assert_null_settings(ctx, name, run, nulls, some):
    """Each setting of `nulls`, and `some` set and then cleared, reproduce the unset episode `run()` bit for bit with the same launches.
    Returns the unset episode and its launch count."""
    set_ = getattr(ctx, "set_" + name)
    set_(None)
    ref, launches = _counted(ctx, run)
    for setting in list(nulls) + [None]:
        if setting is None:
            set_(some)
        set_(setting)
        out, n = _counted(ctx, run)
        assert n == launches, (n, launches)
        assert_episode_equal(ref, out)
    return ref, launches


def assert_rejected_settings(ctx, name, run, setting, bad, big):
    """With `setting` in force, every rejected call returns before any launch, -1 for each setting of `bad`, a null context, B < 0 and a NULL
    array, -4 for `big` (max_batch + 1 records), and keeps `setting`: run() is as before, with the same launches. Returns that episode and
    its launch count."""
    set_, call = getattr(ctx, "set_" + name), getattr(ctx._lib, "hb_rollout_set_" + name)
    set_(setting)
    want, launches = _counted(ctx, run)
    c0 = ctx.launch_count
    for b in bad:
        assert call(ctx._h, len(b), b) == -1
    assert call(None, 1, setting) == -1
    assert call(ctx._h, -1, setting) == -1
    assert call(ctx._h, 1, None) == -1
    assert len(big) == ctx.max_batch + 1 and call(ctx._h, len(big), big) == -4
    with pytest.raises(hb.HunterB200Error):
        set_(bad[0])
    assert ctx.launch_count == c0
    got, n = _counted(ctx, run)
    assert n == launches
    assert_episode_equal(want, got)
    return want, launches
