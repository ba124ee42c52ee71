"""Estimated closed-loop episodes (hb_rollout_estimated_batch_dev): the controllers read the Kalman filter's estimate from simulated, seeded
noisy sensors. The sensors and their noise are checked against the numpy restatement in estimation_ref.py, the episode call bit for bit
against the same loop written with public calls, and against itself: continuation, permutation of instances, argument checks, launches."""
import ctypes as C
import math

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from episode_ref import (CMD_TIMES, GAIT_START, GAITS, SIGMAS, assert_continues, assert_episode_equal, cmd_vels, context, device, est_params,
                         launch_coefficients, noise, params, start_states, stepwise)
from estimation_ref import channel_normals, quat_zyx, sensors

pytestmark = pytest.mark.gpu

CHANNELS = ("orientation", "angular_velocity", "linear_acceleration", "joint_position", "joint_velocity")


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
    sn = noise(seed)

    def states():
        st = hb.estimation_states(B)
        for i, s in enumerate(streams):
            st[i].noise_stream = s
            st[i].primed = 1
            for k in range(3):
                st[i].base_vel_prev[k] = 0.1 * (k + 1)
        return st

    clean = ctx.read_sensors(rbd, states(), tick, None)
    noisy = ctx.read_sensors(rbd, states(), tick, sn)
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
    alone = ctx.read_sensors(rbd[3:4], st1, tick, sn)
    for k in range(5):
        assert np.array_equal(alone[k][0], noisy[k][3])
    # a channel with sigma 0 reads exactly
    quiet = noise(seed); quiet.joint_velocity = 0.0
    part = ctx.read_sensors(rbd, states(), tick, quiet)
    assert np.array_equal(part[4], clean[4]) and np.array_equal(part[3], noisy[3])
    ctx.close()


@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
def test_estimated_episode_equals_the_stepwise_loop_bitwise(event_nodes):
    ctx = context(event_nodes)
    B, n_ticks, log_every = 6, 200, 10
    rbd0 = start_states(ctx, B, seed=11)
    vels = cmd_vels(B)
    prm = params(log_every)
    ep = est_params(seed=2024)
    streams = 40
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, streams))
    r = stepwise(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, streams))
    assert (r[3]["plan_rejects"] == 0).all(), r[3]
    assert_episode_equal(d, r)
    assert (d[6]["count"] > 0).all() and np.isfinite(r[0]).all()
    assert not np.array_equal(d[7].cpu().numpy(), d[4].cpu().numpy())      # the controllers did see an estimate, not the truth
    ctx.close()


def test_two_calls_continue_one_call_and_instances_permute():
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=12)
    vels = cmd_vels(B)
    prm = params(10)
    ep = est_params(seed=5)
    assert_continues(ctx, rbd0, GAITS, vels, 200, 100, prm, 10, ep)
    # permuting the instances together with their states and noise streams permutes the outcome
    perm = [4, 0, 5, 2, 1, 3]
    est_p = hb.estimation_states(B)
    for j, i in enumerate(perm):
        est_p[j].noise_stream = i
    one = device(ctx, rbd0, GAITS, vels, 200, prm, 10, ep)
    p = device(ctx, rbd0[perm], [GAITS[i] for i in perm], vels[perm], 200, prm, 10, ep, est_p)
    assert_episode_equal(one, p, rows_a=perm)
    ctx.close()


def test_standing_estimated_episode_keeps_the_robots_up():
    """test_standing_episode_keeps_the_robots_up through the estimator without sensor noise. Measured on an H100 80GB HBM3 (700 W): over the
    4 robots max_height_err = 2.8e-3 m and max_vel_err = 0.115 m/s (the filter starts from x_hat = 0, so the first ticks dominate both)."""
    import torch
    B, n_ticks = 4, 200
    ctx = hb.Context(horizon_N=50, dt=0.02, max_batch=B, device=0)
    rbd0 = start_states(ctx, B, seed=2)
    z0 = rbd0[:, 5].copy()
    prm = params(1)
    cmds = hb.make_rollout_commands(["stance"] * B, 0.0, [0.0], [[0.0, 0.0, 0.0, 0.0]])
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
    import torch
    B, calls, ticks = 2, 8, 50
    ctx = hb.Context(horizon_N=40, dt=0.02, max_batch=B, device=0)
    rbd0 = start_states(ctx, B, seed=3)
    rbd0[:, 0] = 3.08
    prm = params(1)
    cmds = hb.make_rollout_commands(["trot"] * B, 0.1, [0.0], [[0.0, 0.0, 0.0, 0.6]])
    ep = est_params(seed=9)
    r, act, estop, st, est, es = torch.from_numpy(rbd0).cuda(), None, None, None, None, None
    true_yaw, filt_yaw, gap = [], [], []
    for c in range(calls):
        r, act, estop, st, log, est, es, est_log = ctx.rollout_estimated(r, cmds, ticks, tick0=c * ticks, params=prm, est_params=ep, est=est, act=act,
                                                                         estop=estop, stats=st, est_stats=es, log_every=1)
        off = hb.HbEstimationState.yaw_obs.offset
        yaw_obs = est.cpu().numpy().reshape(B, -1)[:, off:off + 8].copy().view(np.float64)[:, 0]
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
    import torch
    ctx = context()
    lib = ctx._lib
    B = 6
    P = lambda t: C.c_void_p(t.data_ptr())
    rbd = torch.from_numpy(start_states(ctx, B, seed=14)).cuda()
    act = torch.zeros(B * C.sizeof(hb.HbActuationState), dtype=torch.uint8, device="cuda")
    estop = torch.zeros(B, dtype=torch.uint8, device="cuda")
    stats = torch.from_numpy(hb.rollout_stats(B).view(np.uint8).copy()).cuda()
    est = torch.from_numpy(np.frombuffer(bytes(hb.estimation_states(B)), dtype=np.uint8).copy()).cuda()
    cmds = hb.make_rollout_commands(GAITS, GAIT_START, CMD_TIMES, cmd_vels(B))
    prm = params()

    def call(Bc=B, ep=None, est_ptr=True, n=5):
        return lib.hb_rollout_estimated_batch_dev(ctx._h, Bc, C.c_int64(0), n, C.byref(prm), None if ep is False else C.byref(ep or est_params()), cmds, P(rbd),
                                                  P(act), P(estop), P(stats), P(est) if est_ptr else None, None, None, None)

    c0 = ctx.launch_count
    for field, value in (("orientation", -0.1), ("joint_velocity", float("nan")), ("angular_velocity", float("inf"))):
        ep = est_params()
        setattr(ep.noise, field, value)
        assert call(ep=ep) == -1, field
    assert call(ep=False) == -1 and call(est_ptr=False) == -1
    assert call(Bc=ctx.max_batch + 1) == -4
    q = torch.zeros((B, 4), dtype=torch.float64, device="cuda")
    bad = noise(1); bad.linear_acceleration = -1.0
    assert lib.hb_sim_read_sensors_batch_dev(ctx._h, B, C.byref(bad), C.c_int64(0), C.c_double(0.002), P(rbd), P(est), P(q), P(q), P(q), P(q), P(q)) == -1
    assert lib.hb_sim_read_sensors_batch_dev(ctx._h, B, C.byref(noise(1)), C.c_int64(-1), C.c_double(0.002), P(rbd), P(est), P(q), P(q), P(q), P(q), P(q)) == -1
    assert lib.hb_sim_read_sensors_batch_dev(ctx._h, B, C.byref(noise(1)), C.c_int64(0), C.c_double(0.002), P(rbd), None, P(q), P(q), P(q), P(q), P(q)) == -1
    assert call(Bc=0) == 0
    assert ctx.launch_count == c0
    # launches: linear in MPC cycles and ticks, 3 more per tick (sensors + contact flags, filter, observation step) and 1 more per MPC cycle
    # (the plan's schedule copied into the estimation state) than the ground-truth episode
    r0 = start_states(ctx, B, seed=14)
    truth = launch_coefficients(ctx, r0, GAITS, cmd_vels(B), prm)
    estimated = launch_coefficients(ctx, r0, GAITS, cmd_vels(B), prm, est_params(1))
    assert estimated[0] == truth[0] + 1 and estimated[1] == truth[1] + 3, (truth, estimated)
    ctx.close()
