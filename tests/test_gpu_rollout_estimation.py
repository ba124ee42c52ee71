"""Estimated closed-loop episodes (hb_rollout_estimated_batch_dev): the controllers read the Kalman filter's estimate from simulated, seeded
noisy sensors. The sensors and their noise are checked against the numpy restatement in estimation_ref.py, the episode call bit for bit
against the same loop written with public calls, and against itself: continuation, permutation of instances, argument checks, launches."""
import ctypes as C
import math

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from estimation_ref import channel_normals, quat_zyx, sensors, shortest_angular_distance
from test_gpu_rollout_episodes import CMD_TIMES, GAIT_START, GAITS, _assert_stats_equal, _cmd_vels, _context, _horizon, _params, _start_states

pytestmark = pytest.mark.gpu

CHANNELS = ("orientation", "angular_velocity", "linear_acceleration", "joint_position", "joint_velocity")
SIGMAS = dict(orientation=0.002, angular_velocity=0.01, linear_acceleration=0.05, joint_position=0.001, joint_velocity=0.01)


def _torch():
    import torch
    return torch


def _noise(seed, scale=1.0):
    n = hb.HbSensorNoise()
    n.seed = seed
    for k, v in SIGMAS.items():
        setattr(n, k, scale * v)
    return n


def _est_params(seed=0, scale=1.0):
    ep = hb.default_estimation_params()
    ep.noise = _noise(seed, scale)
    return ep


def _est_bytes(est, B):
    return np.frombuffer(bytes(est), dtype=np.uint8).reshape(B, C.sizeof(hb.HbEstimationState)) if not hasattr(est, "cpu") else \
        est.cpu().numpy().reshape(B, C.sizeof(hb.HbEstimationState))


def _assert_est_equal(a, b, B):
    a, b = _est_bytes(a, B), _est_bytes(b, B)
    if not np.array_equal(a, b):
        bad = [f for f, _ in hb.HbEstimationState._fields_
               if not np.array_equal(a[:, getattr(hb.HbEstimationState, f).offset:][:, :getattr(hb.HbEstimationState, f).size],
                                     b[:, getattr(hb.HbEstimationState, f).offset:][:, :getattr(hb.HbEstimationState, f).size])]
        raise AssertionError("estimation state differs in %s" % bad)


def _random_rbd(B, seed):
    rng = np.random.default_rng(seed)
    rbd = sc.consistent_rbd(sc.random_initial_states(B, seed=seed), rng, 0.05)
    rbd[:, 0] = rng.uniform(-3.0, 3.0, B)
    rbd[B - 1, 0] = 4.2                     # a yaw beyond +-pi
    return rbd


def test_sensor_read_matches_restatement_without_noise():
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=8, device=0)
    B = 6
    rbd = _random_rbd(B, 3)
    est = hb.estimation_states(B)
    rng = np.random.default_rng(4)
    prev = rng.uniform(-0.5, 0.5, (B, 3))
    for i in range(1, B):                   # instance 0 stays unprimed: gravity only
        est[i].primed = 1
        for k in range(3):
            est[i].base_vel_prev[k] = prev[i, k]
    quat, w, a, jp, jv = ctx.read_sensors(rbd, est, 17, None, accel_dt=0.002)
    for i in range(B):
        rq, rw, ra, rjp, rjv = sensors(rbd[i], prev[i], i > 0, 0.002)
        np.testing.assert_allclose(quat[i], rq, rtol=0, atol=1e-13)
        np.testing.assert_allclose(w[i], rw, rtol=0, atol=1e-13)
        np.testing.assert_allclose(a[i], ra, rtol=0, atol=1e-13 * max(1.0, np.abs(ra).max()))
        assert np.array_equal(jp[i], rbd[i, 6:16]) and np.array_equal(jv[i], rbd[i, 22:32])
        assert est[i].primed == 1 and np.array_equal(np.array(est[i].base_vel_prev[:]), rbd[i, 19:22])
    assert abs(np.linalg.norm(a[0]) - 9.81) < 1e-12
    np.testing.assert_allclose(a[0], sc.rot_zyx(rbd[0, 0:3]).T @ [0, 0, 9.81], rtol=0, atol=1e-12)
    # the filter reads the wrapped yaw of the quaternion
    assert abs(math.atan2(2 * (quat[-1, 0] * quat[-1, 1] + quat[-1, 3] * quat[-1, 2]), quat[-1, 3] ** 2 + quat[-1, 0] ** 2 - quat[-1, 1] ** 2 - quat[-1, 2] ** 2)
               - (4.2 - 2 * math.pi)) < 1e-12
    ctx.close()


@pytest.mark.parametrize("seed", [1, (7 << 32) + 12345])
def test_sensor_noise_is_pinned(seed):
    """Noisy minus noiseless readings are sigma x the restated Philox normals, per channel; the same (seed, stream, tick) gives the same
    readings at another batch position and in another batch size."""
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=8, device=0)
    B, tick = 4, 70001
    rbd = _random_rbd(B, 5)
    rbd[3] = rbd[0]
    streams = [3, (1 << 33) + 1, 99, 3]          # instances 0 and 3: same stream, same state
    noise = _noise(seed)

    def states():
        st = hb.estimation_states(B)
        for i, s in enumerate(streams):
            st[i].noise_stream = s
            st[i].primed = 1
            for k in range(3):
                st[i].base_vel_prev[k] = 0.1 * (k + 1)
        return st

    clean = ctx.read_sensors(rbd, states(), tick, None)
    noisy = ctx.read_sensors(rbd, states(), tick, noise)
    for i in range(B):
        z = {ch: channel_normals(seed, ch, 3 if ch in ("orientation", "angular_velocity", "linear_acceleration") else 10, tick, streams[i]) for ch in CHANNELS}
        np.testing.assert_allclose(noisy[0][i], quat_zyx(rbd[i, 0:3] + SIGMAS["orientation"] * z["orientation"]), rtol=0, atol=1e-12)
        for k, ch in enumerate(CHANNELS[1:], start=1):
            np.testing.assert_allclose(noisy[k][i] - clean[k][i], SIGMAS[ch] * z[ch], rtol=0, atol=1e-12)
    for k in range(5):
        assert np.array_equal(noisy[k][0], noisy[k][3])
    st1 = hb.estimation_states(1)
    st1[0].noise_stream = streams[0]; st1[0].primed = 1
    for k in range(3):
        st1[0].base_vel_prev[k] = 0.1 * (k + 1)
    alone = ctx.read_sensors(rbd[3:4], st1, tick, noise)
    for k in range(5):
        assert np.array_equal(alone[k][0], noisy[k][3])
    # a channel with sigma 0 reads exactly
    quiet = _noise(seed); quiet.joint_velocity = 0.0
    part = ctx.read_sensors(rbd, states(), tick, quiet)
    assert np.array_equal(part[4], clean[4]) and np.array_equal(part[3], noisy[3])
    ctx.close()


def _mode_at(st, t):
    idx = 0
    while idx < st.n_events and st.event_times[idx] < t:
        idx += 1
    return st.modes[idx]


def _stepwise(ctx, rbd, gaits, cmd_vels, n_ticks, prm, ep, est, log_every):
    """The estimated episode as a Python loop over public calls, with the contact flags, the yaw unwrap and the stats restated."""
    B = rbd.shape[0]
    rbd = rbd.copy()
    act = hb.actuation_states(B)
    estop = np.zeros(B, dtype=np.uint8)
    st = hb.rollout_stats(B)
    es = hb.estimation_stats(B)
    kf = hb.kf_states(B)
    held = rbd.copy()
    lim = np.array(prm.torque_limit[:])
    times = np.array(CMD_TIMES)
    stance = np.zeros((B, 12))
    logs, est_logs = [], []
    for a in range(n_ticks):
        t = a * prm.period
        for i in range(B):
            r = rbd[i]
            why = (2 if (r[2] > np.pi / 2 or r[2] < -np.pi / 2) else 0) | (4 if prm.min_base_height != 0 and r[5] < prm.min_base_height else 0)
            if why and st["fail_tick"][i] < 0:
                st["fail_tick"][i] = a; st["fail_reason"][i] = why
            held[i] = r
        if log_every and a % log_every == 0:
            logs.append(rbd.copy())
        quat, w, acc, jp, jv = ctx.read_sensors(rbd, est, a, ep.noise, accel_dt=prm.sim.dt)
        tf = (a - 1) * prm.period
        flags = np.ones((B, 4), dtype=np.uint8)
        for i in range(B):
            if est[i].has_plan:
                m = _mode_at(est[i], tf)
                flags[i] = [1 if (m in (1, 3) if c & 1 else m in (2, 3)) else 0 for c in range(4)]
        e_rbd = ctx.estimator_update(prm.period, kf, quat, w, acc, jp, jv, flags, params=ep.kf)
        for i in range(B):
            est[i].yaw_obs = est[i].yaw_obs + shortest_angular_distance(est[i].yaw_obs, e_rbd[i, 0])
            if st["fail_tick"][i] < 0:
                d = [float(e_rbd[i, 19 + k] - rbd[i, 19 + k]) for k in range(3)]
                sq = d[0] * d[0] + d[1] * d[1] + d[2] * d[2]
                ve, dz = math.sqrt(sq), abs(float(e_rbd[i, 5] - rbd[i, 5]))
                if ve > es["max_vel_err"][i]:
                    es["max_vel_err"][i] = ve
                if dz > es["max_height_err"][i]:
                    es["max_height_err"][i] = dz
                es["sum_sq_vel_err"][i] += sq; es["sum_sq_height_err"][i] += dz * dz; es["count"][i] += 1
        if log_every and a % log_every == 0:
            est_logs.append(e_rbd.copy())
        mpc = a % prm.mpc_every == 0
        if mpc:
            x0 = ctx.rbd_to_centroidal(e_rbd)
            x0[:, 9] = [est[i].yaw_obs for i in range(B)]
            cmd = cmd_vels[:, max(np.searchsorted(times, t, side="right") - 1, 0)]
            ins = hb.make_plan_inputs(np.full(B, t), _horizon(ctx), x0, cmd, None, gaits, GAIT_START)
            info, _, _, _, ps = ctx.resident_plan_cycle(a == 0, 0.0, ins, e_rbd)
            refs, stance, _ = ctx.plan_references_gpu(hb.make_plan_inputs(np.full(B, t), _horizon(ctx), x0, cmd, ctx.contact_positions(x0), gaits, GAIT_START),
                                                      stance)
            for i in range(B):
                n = refs[i].n_events
                est[i].n_events = n
                for k in range(n):
                    est[i].event_times[k] = refs[i].event_times[k]
                for k in range(n + 1):
                    est[i].modes[k] = refs[i].modes[k]
                est[i].has_plan = 1
        xd, ud, md, sol, _, wst = ctx.resident_wbc(t, e_rbd)
        jcmd, _, estop = ctx.joint_command(prm.period, xd, ud, sol, md, e_rbd, estop=estop, gains=prm.gains)
        tau = ctx.actuation(t, act, jcmd, rbd, prm.actuation_delay)
        tau = np.clip(tau, -lim, lim)
        rbd, _, _ = ctx.sim_step(rbd, tau, prm.sim)
        for i in range(B):
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
    for i in range(B):
        est[i].kf = kf[i]
    log = np.stack(logs, axis=1) if log_every else None
    est_log = np.stack(est_logs, axis=1) if log_every else None
    return rbd, np.frombuffer(bytes(act), dtype=np.uint8), estop, st, log, est, es, est_log


def _device(ctx, rbd, gaits, cmd_vels, n_ticks, prm, ep, est, log_every, tick0=0, act=None, estop=None, stats=None, est_stats=None):
    torch = _torch()
    d_rbd = torch.from_numpy(np.ascontiguousarray(rbd)).cuda()
    d_est = est if hasattr(est, "cpu") else torch.from_numpy(np.frombuffer(bytes(est), dtype=np.uint8).copy()).cuda()
    cmds = hb.make_rollout_commands(gaits, GAIT_START, CMD_TIMES, cmd_vels)
    return ctx.rollout_estimated(d_rbd, cmds, n_ticks, tick0=tick0, params=prm, est_params=ep, est=d_est, act=act, estop=estop, stats=stats,
                                 est_stats=est_stats, log_every=log_every)


def _assert_est_stats_equal(a, b):
    for k in hb.ESTIMATION_STATS_DTYPE.names:
        assert np.array_equal(a[k], b[k]), (k, a[k], b[k])


@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
def test_estimated_episode_equals_the_stepwise_loop_bitwise(event_nodes):
    ctx = _context(event_nodes)
    B, n_ticks, log_every = 6, 200, 10
    rbd0 = _start_states(ctx, B, seed=11)
    vels = _cmd_vels(B)
    prm = _params(log_every)
    ep = _est_params(seed=2024)
    streams = 40
    d = _device(ctx, rbd0, GAITS, vels, n_ticks, prm, ep, hb.estimation_states(B, streams), log_every)
    r = _stepwise(ctx, rbd0, GAITS, vels, n_ticks, prm, ep, hb.estimation_states(B, streams), log_every)
    assert (r[3]["plan_rejects"] == 0).all(), r[3]
    assert np.array_equal(d[0].cpu().numpy(), r[0])
    assert np.array_equal(d[1].cpu().numpy(), r[1])
    assert np.array_equal(d[2].cpu().numpy(), r[2])
    _assert_stats_equal(d[3], r[3])
    assert np.array_equal(d[4].cpu().numpy(), r[4])
    _assert_est_equal(d[5], r[5], B)
    _assert_est_stats_equal(d[6], r[6])
    assert np.array_equal(d[7].cpu().numpy(), r[7])
    assert (d[6]["count"] > 0).all() and np.isfinite(r[0]).all()
    assert not np.array_equal(d[7].cpu().numpy(), d[4].cpu().numpy())      # the controllers did see an estimate, not the truth
    ctx.close()


def test_two_calls_continue_one_call_and_instances_permute():
    ctx = _context()
    B = 6
    rbd0 = _start_states(ctx, B, seed=12)
    vels = _cmd_vels(B)
    prm = _params(10)
    ep = _est_params(seed=5)
    one = _device(ctx, rbd0, GAITS, vels, 200, prm, ep, hb.estimation_states(B), 10)
    h = _device(ctx, rbd0, GAITS, vels, 100, prm, ep, hb.estimation_states(B), 10)
    two = ctx.rollout_estimated(h[0], hb.make_rollout_commands(GAITS, GAIT_START, CMD_TIMES, vels), 100, tick0=100, params=prm, est_params=ep, est=h[5],
                                act=h[1], estop=h[2], stats=h[3], est_stats=h[6], log_every=10)
    for k in (0, 1, 2, 5):
        assert np.array_equal(one[k].cpu().numpy(), two[k].cpu().numpy()), k
    _assert_stats_equal(one[3], two[3])
    _assert_est_stats_equal(one[6], two[6])
    for k in (4, 7):
        assert np.array_equal(one[k].cpu().numpy(), np.concatenate([h[k].cpu().numpy(), two[k].cpu().numpy()], axis=1)), k
    # permuting the instances together with their states and noise streams permutes the outcome
    perm = [4, 0, 5, 2, 1, 3]
    est_p = hb.estimation_states(B)
    for j, i in enumerate(perm):
        est_p[j].noise_stream = i
    p = _device(ctx, rbd0[perm], [GAITS[i] for i in perm], vels[perm], 200, prm, ep, est_p, 10)
    size = C.sizeof(hb.HbActuationState)
    assert np.array_equal(one[0].cpu().numpy()[perm], p[0].cpu().numpy())
    assert np.array_equal(one[1].cpu().numpy().reshape(B, size)[perm], p[1].cpu().numpy().reshape(B, size))
    assert np.array_equal(one[2].cpu().numpy()[perm], p[2].cpu().numpy())
    _assert_stats_equal(one[3][perm], p[3])
    assert np.array_equal(_est_bytes(one[5], B)[perm], _est_bytes(p[5], B))
    _assert_est_stats_equal(one[6][perm], p[6])
    for k in (4, 7):
        assert np.array_equal(one[k].cpu().numpy()[perm], p[k].cpu().numpy()), k
    ctx.close()


def test_standing_estimated_episode_keeps_the_robots_up():
    """test_standing_episode_keeps_the_robots_up through the estimator without sensor noise. Measured on an H100 80GB HBM3 (700 W): over the
    4 robots max_height_err = 2.8e-3 m and max_vel_err = 0.115 m/s (the filter starts from x_hat = 0, so the first ticks dominate both)."""
    B, n_ticks = 4, 200
    ctx = hb.Context(horizon_N=50, dt=0.02, max_batch=B, device=0)
    rbd0 = _start_states(ctx, B, seed=2)
    z0 = rbd0[:, 5].copy()
    prm = _params(1)
    cmds = hb.make_rollout_commands(["stance"] * B, 0.0, [0.0], [[0.0, 0.0, 0.0, 0.0]])
    torch = _torch()
    rbd, act, estop, st, log, est, es, est_log = ctx.rollout_estimated(torch.from_numpy(rbd0).cuda(), cmds, n_ticks, params=prm, log_every=1)
    rbd, log = rbd.cpu().numpy(), log.cpu().numpy()
    print("standing, no noise: max_height_err %.3e max_vel_err %.3e" % (es["max_height_err"].max(), es["max_vel_err"].max()))
    assert (st["fail_tick"] == -1).all() and (estop.cpu().numpy() == 0).all(), st
    assert np.isfinite(log).all() and np.isfinite(rbd).all()
    heights = np.vstack([log[:, -49:, 5].T, rbd[None, :, 5]])
    assert np.abs(heights - z0[None]).max() < 0.03, np.abs(heights - z0[None]).max()
    assert np.abs(rbd[:, 1:3]).max() < 0.1
    assert np.abs(rbd[:, 16:32]).max() < 1.0
    assert (es["count"] == n_ticks).all()
    assert es["max_height_err"].max() < 0.01 and es["max_vel_err"].max() < 0.3, es
    ctx.close()


def test_yaw_obs_follows_the_true_yaw_across_pi():
    """A turning trot from yaw 3.08 crosses +pi (to about 3.25 in 0.8 s): the filter's yaw wraps to about -pi, yaw_obs keeps following the
    plant's unwrapped yaw (measured on an H100: within 5.2e-3 rad with orientation noise of 2e-3 rad)."""
    B, calls, ticks = 2, 8, 50
    ctx = hb.Context(horizon_N=40, dt=0.02, max_batch=B, device=0)
    rbd0 = _start_states(ctx, B, seed=3)
    rbd0[:, 0] = 3.08
    prm = _params(1)
    cmds = hb.make_rollout_commands(["trot"] * B, 0.1, [0.0], [[0.0, 0.0, 0.0, 0.6]])
    ep = _est_params(seed=9)
    torch = _torch()
    r, act, estop, st, est, es = torch.from_numpy(rbd0).cuda(), None, None, None, None, None
    true_yaw, filt_yaw, gap = [], [], []
    for c in range(calls):
        r, act, estop, st, log, est, es, est_log = ctx.rollout_estimated(r, cmds, ticks, tick0=c * ticks, params=prm, est_params=ep, est=est, act=act,
                                                                         estop=estop, stats=st, est_stats=es, log_every=1)
        off = hb.HbEstimationState.yaw_obs.offset
        yaw_obs = _est_bytes(est, B)[:, off:off + 8].copy().view(np.float64)[:, 0]
        last_true = log.cpu().numpy()[:, -1, 0]
        gap.append(np.abs(yaw_obs - last_true).max())
        true_yaw.append(log.cpu().numpy()[:, :, 0]); filt_yaw.append(est_log.cpu().numpy()[:, :, 0])
    true_yaw = np.concatenate(true_yaw, axis=1); filt_yaw = np.concatenate(filt_yaw, axis=1)
    print("yaw: true max %.3f, filter min %.3f, max |yaw_obs - yaw| %.3e" % (true_yaw.max(), filt_yaw.min(), max(gap)))
    assert (st["fail_tick"] == -1).all(), st
    assert true_yaw.max() > math.pi + 0.05 and filt_yaw.min() < -math.pi + 0.2
    assert max(gap) < 0.05, gap
    ctx.close()


def test_argument_checks_and_launches():
    torch = _torch()
    ctx = _context()
    lib = ctx._lib
    B = 6
    P = lambda t: C.c_void_p(t.data_ptr())
    rbd = torch.from_numpy(_start_states(ctx, B, seed=14)).cuda()
    act = torch.zeros(B * C.sizeof(hb.HbActuationState), dtype=torch.uint8, device="cuda")
    estop = torch.zeros(B, dtype=torch.uint8, device="cuda")
    stats = torch.from_numpy(hb.rollout_stats(B).view(np.uint8).copy()).cuda()
    est = torch.from_numpy(np.frombuffer(bytes(hb.estimation_states(B)), dtype=np.uint8).copy()).cuda()
    cmds = hb.make_rollout_commands(GAITS, GAIT_START, CMD_TIMES, _cmd_vels(B))
    prm = _params()

    def call(Bc=B, ep=None, est_ptr=True, n=5):
        return lib.hb_rollout_estimated_batch_dev(ctx._h, Bc, C.c_int64(0), n, C.byref(prm), None if ep is False else C.byref(ep or _est_params()), cmds, P(rbd),
                                                  P(act), P(estop), P(stats), P(est) if est_ptr else None, None, None, None)

    c0 = ctx.launch_count
    for field, value in (("orientation", -0.1), ("joint_velocity", float("nan")), ("angular_velocity", float("inf"))):
        ep = _est_params()
        setattr(ep.noise, field, value)
        assert call(ep=ep) == -1, field
    assert call(ep=False) == -1 and call(est_ptr=False) == -1
    assert call(Bc=ctx.max_batch + 1) == -4
    q = torch.zeros((B, 4), dtype=torch.float64, device="cuda")
    bad = _noise(1); bad.linear_acceleration = -1.0
    assert lib.hb_sim_read_sensors_batch_dev(ctx._h, B, C.byref(bad), C.c_int64(0), C.c_double(0.002), P(rbd), P(est), P(q), P(q), P(q), P(q), P(q)) == -1
    assert lib.hb_sim_read_sensors_batch_dev(ctx._h, B, C.byref(_noise(1)), C.c_int64(-1), C.c_double(0.002), P(rbd), P(est), P(q), P(q), P(q), P(q), P(q)) == -1
    assert lib.hb_sim_read_sensors_batch_dev(ctx._h, B, C.byref(_noise(1)), C.c_int64(0), C.c_double(0.002), P(rbd), None, P(q), P(q), P(q), P(q), P(q)) == -1
    assert call(Bc=0) == 0
    assert ctx.launch_count == c0
    # launches: linear in MPC cycles and ticks, 3 more per tick (sensors + contact flags, filter, observation step) and 1 more per MPC cycle
    # (the plan's schedule copied into the estimation state) than the ground-truth episode
    vels = _cmd_vels(B)
    r0 = _start_states(ctx, B, seed=14)
    rows = {}
    for kind in ("truth", "estimated"):
        r = torch.from_numpy(r0).cuda()
        if kind == "truth":
            out = ctx.rollout(r, cmds, 10, params=prm)
        else:
            out = ctx.rollout_estimated(r, cmds, 10, params=prm, est_params=_est_params(1))
        tick0, res = 10, []
        for n in (10, 23, 7):
            cycles = sum(1 for a in range(tick0, tick0 + n) if a % prm.mpc_every == 0)
            c0 = ctx.launch_count
            if kind == "truth":
                out = ctx.rollout(out[0], cmds, n, tick0=tick0, params=prm, act=out[1], estop=out[2], stats=out[3])
            else:
                out = ctx.rollout_estimated(out[0], cmds, n, tick0=tick0, params=prm, est_params=_est_params(1), est=out[5], act=out[1], estop=out[2],
                                            stats=out[3], est_stats=out[6])
            res.append((cycles, n, ctx.launch_count - c0))
            tick0 += n
        M = np.array([[c, n] for c, n, _ in res[:2]], dtype=float)
        a, b = np.rint(np.linalg.solve(M, [d for _, _, d in res[:2]])).astype(int)
        for c, n, d in res:
            assert d == a * c + b * n, (res, a, b)
        rows[kind] = (a, b)
    assert rows["estimated"][0] == rows["truth"][0] + 1 and rows["estimated"][1] == rows["truth"][1] + 3, rows
    ctx.close()
