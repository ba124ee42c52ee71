"""Simulated hardware in the episodes (hb_rollout_set_hardware): each robot's actuation delay, torque limits, sensor noise and calibration
offsets. The host calls with explicit records against numpy (hb_sim_read_sensors_hw, hb_actuation_hw); a record with zero offsets acts on
its robot exactly as the same values in params / est_params act on an unset episode, under both WBCs, both time grids, truth and
estimator; an episode with offsets equals the loop of public calls (episode_ref.stepwise); then the setting's contract and two properties."""
import ctypes as C
from collections import deque
from contextlib import contextmanager

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from episode_ref import (FRICTION, GAITS, PUSH, SIGMAS, array_of, assert_episode_equal, assert_null_settings, assert_records_act_as_their_values,
                         assert_rejected_settings, assert_setting_episodes, cmd_vels, context, device, est_params, outputs, params, random_goals,
                         small_terrains, start_states, stepwise, use)
from hardware_ref import call_hardware, sensors_hw

pytestmark = pytest.mark.gpu

B = 6
DEFAULT_LIMITS = np.array(hb.default_rollout_params().torque_limit[:])


def _sigmas(scale):
    return {"sigma_" + k: scale * v for k, v in SIGMAS.items()}


def _records():
    """Three records without offsets: a short delay with tight limits and twice the noise, a long delay with half the noise, no delay with
    tighter limits and exact sensors."""
    return [hb.make_hardware_settings(1, actuation_delay=0.004, torque_limit=0.8 * DEFAULT_LIMITS, **_sigmas(2.0))[0],
            hb.make_hardware_settings(1, actuation_delay=0.016, **_sigmas(0.5))[0],
            hb.make_hardware_settings(1, actuation_delay=0.0, torque_limit=0.6 * DEFAULT_LIMITS)[0]]


def _offsets(n):
    """Records with every kind of offset, per robot, some entries exactly 0.0, and per-robot delays, limits and sigmas."""
    rng = np.random.default_rng(5)
    enc = rng.uniform(-0.01, 0.01, (n, 10)); enc[:, 3] = 0.0
    return hb.make_hardware_settings(n, actuation_delay=np.linspace(0.0, 0.012, n), torque_limit=np.linspace(1.0, 0.7, n)[:, None] * DEFAULT_LIMITS,
                                     orientation_offset=rng.uniform(-0.015, 0.015, (n, 3)) * [1, 1, 0], gyro_bias=rng.uniform(-0.01, 0.01, (n, 3)),
                                     accel_bias=rng.uniform(-0.1, 0.1, (n, 3)), encoder_offset=enc,
                                     **{k: np.linspace(0.5, 1.5, n) * v for k, v in _sigmas(1.0).items()})


def _random_rbd(n, seed):
    rng = np.random.default_rng(seed)
    rbd = rng.normal(0.0, 0.3, (n, 32))
    rbd[:, 0] = rng.uniform(-3.0, 3.0, n)
    rbd[0, 6:16] = -0.0                                # -0.0 encoder readings: a 0.0 offset keeps them
    return rbd


def _states(n, prev):
    st = hb.estimation_states(n, 11)
    for i in range(n):
        st[i].primed = 1 if i else 0
        for k in range(3):
            st[i].base_vel_prev[k] = prev[i, k]
    return st


def _read_plain(ctx, rbd, est, tick, noise, accel_dt=0.002):
    """hb_sim_read_sensors itself (Context.read_sensors calls hb_sim_read_sensors_hw)."""
    n = rbd.shape[0]
    out = [np.zeros((n, 4)), np.zeros((n, 3)), np.zeros((n, 3)), np.zeros((n, 10)), np.zeros((n, 10))]
    assert ctx._lib.hb_sim_read_sensors(ctx._h, n, C.byref(noise), C.c_int64(tick), C.c_double(accel_dt), hb.api._ptr(rbd), est,
                                        *[hb.api._ptr(a) for a in out]) == 0
    return out


# ---------------------------------------------------------------------------------------------------------------- 1. sensor read
def test_sensor_read_matches_the_restatement():
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=8, device=0)
    rbd = _random_rbd(B, 3)
    prev = np.random.default_rng(4).normal(0.0, 0.2, (B, 3))
    hw = _offsets(B)
    seed, tick = (5 << 32) + 77, 23
    noise = hb.HbSensorNoise(); noise.seed = seed
    est = _states(B, prev)
    got = ctx.read_sensors(rbd, est, tick, noise, hardware=hw)
    for i in range(B):
        want = sensors_hw(rbd[i], prev[i], i > 0, 0.002, hw[i], seed, tick, 11 + i)
        for k, (g, w) in enumerate(zip(got, want)):
            np.testing.assert_allclose(g[i], w, rtol=0, atol=1e-12 * max(1.0, np.abs(w).max()), err_msg=str((i, k)))
        assert est[i].primed == 1 and np.array_equal(np.array(est[i].base_vel_prev[:]), rbd[i, 19:22])
    ctx.close()


def test_sensor_read_without_records_or_offsets_is_the_plain_read_bitwise():
    """hw = NULL, and records carrying the call's sigmas with zero offsets, read hb_sim_read_sensors' bits; so does the default record on a
    call without noise. -0.0 encoder readings stay -0.0."""
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=8, device=0)
    rbd = _random_rbd(B, 6)
    prev = np.random.default_rng(7).normal(0.0, 0.2, (B, 3))
    noise = est_params(seed=99).noise
    call = hb.make_hardware_settings(B, orientation_offset=[0.0, -0.0, 0.0], encoder_offset=np.r_[[-0.0] * 5, [0.0] * 5],
                                     **{"sigma_" + k: getattr(noise, k) for k in SIGMAS})
    for tick in (0, 41):
        want = _read_plain(ctx, rbd, _states(B, prev), tick, noise)
        for hw in (None, call):
            got = ctx.read_sensors(rbd, _states(B, prev), tick, noise, hardware=hw)
            for a, b in zip(got, want):
                assert np.array_equal(a, b) and np.array_equal(np.signbit(a), np.signbit(b))
    exact = _read_plain(ctx, rbd, _states(B, prev), 3, hb.HbSensorNoise())
    got = ctx.read_sensors(rbd, _states(B, prev), 3, None, hardware=hb.make_hardware_settings(B))
    for a, b in zip(got, exact):
        assert np.array_equal(a, b) and np.array_equal(np.signbit(a), np.signbit(b))
    assert np.signbit(got[3][0]).all()
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 2. actuation
def _actuation_numpy(delays, times, commands):
    """LeggedHWSim's buffer as a deque per robot (newest first, at most HB_ACT_CAPACITY): drop the oldest entries with stamp + delay < t, drop
    one more when full, push, apply the oldest. Returns the index of the command applied on each tick, (ticks, robots)."""
    n = len(delays)
    dq = [deque() for _ in range(n)]
    applied = np.zeros((len(times), n), dtype=int)
    for a, t in enumerate(times):
        for i in range(n):
            while dq[i] and dq[i][-1][0] + delays[i] < t:
                dq[i].pop()
            if len(dq[i]) == 16:
                dq[i].pop()
            dq[i].appendleft((t, a))
            applied[a, i] = dq[i][-1][1]
    return applied


def test_actuation_matches_the_deque_restatement():
    """Per-robot delays, 0 and one beyond the ring included: with kp = kd = 0 the applied torque is the feed-forward of the applied command,
    which names its tick; a larger delay applies an older command."""
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=8, device=0)
    delays = [0.0, 0.002, 0.005, 0.009, 0.0301, 1.0]
    hw = hb.make_hardware_settings(B, actuation_delay=delays)
    rbd = _random_rbd(B, 8)
    times = np.arange(40) * 0.002
    state = hb.actuation_states(B)
    applied = np.zeros((40, B), dtype=int)
    for a, t in enumerate(times):
        cmd = np.zeros((B, 10, 5))
        cmd[:, :, 4] = a + 1000.0 * np.arange(B)[:, None]
        tau = ctx.actuation(t, state, cmd, rbd, delay=0.009, hardware=hw)
        assert np.array_equal(tau, np.broadcast_to(tau[:, :1], (B, 10)))
        applied[a] = np.rint(tau[:, 0] - 1000.0 * np.arange(B)).astype(int)
        assert np.array_equal(tau[:, 0], applied[a] + 1000.0 * np.arange(B))
    assert np.array_equal(applied, _actuation_numpy(delays, times, None))
    assert (applied[:, 0] == np.arange(40)).all()                     # no delay: the newest command
    assert (np.diff(applied[-1]) <= 0).all() and applied[-1, -1] == 39 - 15   # older and older; beyond the ring: the oldest of a full ring
    ctx.close()


def test_actuation_without_records_is_the_plain_call_bitwise():
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=8, device=0)
    rng = np.random.default_rng(9)
    rbd = _random_rbd(B, 10)
    s1, s2 = hb.actuation_states(B), hb.actuation_states(B)
    for a in range(20):
        cmd = rng.normal(0.0, 1.0, (B, 10, 5))
        tau1 = ctx.actuation(a * 0.002, s1, cmd, rbd, delay=0.007)
        tau2 = np.zeros((B, 10))
        t = np.full(B, a * 0.002)
        assert ctx._lib.hb_actuation_batch(ctx._h, B, C.c_double(0.007), hb.api._ptr(t), s2, hb.api._ptr(np.ascontiguousarray(cmd)), hb.api._ptr(rbd),
                                           hb.api._ptr(tau2)) == 0
        assert np.array_equal(tau1, tau2) and bytes(s1) == bytes(s2)
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 3. records = call values
@contextmanager
def _on_the_call(ctx, rec, prm, ep):
    """Copies of prm and ep carrying rec's delay, limits and sigmas."""
    p = hb.HbRolloutParams.from_buffer_copy(bytes(prm))
    p.actuation_delay = rec.actuation_delay
    p.torque_limit[:] = rec.torque_limit[:]
    e = None
    if ep is not None:
        e = hb.HbEstimationParams.from_buffer_copy(bytes(ep))
        for k in SIGMAS:
            setattr(e.noise, k, getattr(rec, "sigma_" + k))
    yield p, e


@pytest.mark.parametrize("wbc", ["weighted", "hierarchical"])
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_records_equal_the_call_values_bitwise(wbc, event_nodes, estimated):
    ctx = context(event_nodes)
    ctx.set_wbc_formulation(wbc)
    rbd0 = start_states(ctx, B, seed=101)
    assert_records_act_as_their_values(ctx, "hardware", _records(), _on_the_call, rbd0, params(10), est_params(seed=2033) if estimated else None)
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 4. offsets through the loop
def test_offset_episode_equals_the_stepwise_loop_bitwise():
    """An estimated episode with offsets, delays, limits and sigmas per robot and one robot beyond the setting, with pushes, plant
    variations, a terrain, goals, an MPC latency and controller settings set alongside."""
    ctx = context()
    n_ticks, log_every = 120, 10
    rbd0 = start_states(ctx, B, seed=102)
    vels = cmd_vels(B)
    prm = params(log_every)
    kw = use(ctx, plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION, motor_strength=0.95),
             pushes=hb.make_push_schedules(B, 0.15, 0.05, PUSH), terrains=small_terrains(), goals=random_goals(rbd0, B, 102),
             mpc_latencies=[0, 2, 5, 1, 0, 3], hardware=_offsets(B - 1))
    # one controller record for every robot, which the loop of public calls restates as the context's WBC settings and params.gains
    w = ctx.wbc_settings(); w.swing_kp *= 1.2
    g = hb.default_pd_gains(); g.kp_big_stance = 45.0
    ctx.set_controller_settings(hb.make_controller_settings(B, wbc=w, gains=g))
    ep = est_params(seed=2034)
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 70))
    ctx.set_wbc_settings(w)
    prm.gains = g
    r = stepwise(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 70), **kw)
    assert_episode_equal(d, r)
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 5, 6. null settings
@pytest.mark.parametrize("wbc", ["weighted", "hierarchical"])
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_null_settings(wbc, estimated):
    """Records of the call's values on every robot, or on some, give the unset episode bit for bit with the same launches; in a truth
    episode so do records that differ only in their sensor fields (rollout has no sensors)."""
    ctx = context()
    ctx.set_wbc_formulation(wbc)
    rbd0 = start_states(ctx, B, seed=103)
    prm = params(5)
    ep = est_params(seed=9) if estimated else None
    call = array_of([call_hardware(prm, ep)] * B)
    nulls = [call, array_of([call_hardware(prm, ep)] * 3)]
    if not estimated:
        nulls += [hb.make_hardware_settings(B), _offsets(B)]
        for r in nulls[-1]:
            r.actuation_delay = prm.actuation_delay
            r.torque_limit[:] = prm.torque_limit[:]
    assert_null_settings(ctx, "hardware", lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 60, prm, 5, ep, hb.estimation_states(B, 50) if estimated else None),
                         nulls, array_of(_records() * 2))
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 7. the contract
def test_setting_contract():
    ctx = context()
    rbd0 = start_states(ctx, B, seed=104)
    r = _records()
    full = array_of([r[0], r[1], r[2], r[1], r[0], r[2]])
    one = hb.make_hardware_settings(B)
    one[0] = r[0]
    other = array_of([r[2], r[0], r[1], r[1], r[2], r[0]])       # instance 3 keeps its record
    part = array_of([r[1], r[2]])
    padded = hb.make_hardware_settings(B)
    padded[0], padded[1] = r[1], r[2]
    assert_setting_episodes(ctx, "hardware", rbd0, params(10), full, one, other, 3, part, padded)
    ctx.close()


def _bad():
    out = []
    for field, value in [("actuation_delay", -1e-3), ("actuation_delay", float("nan")), ("actuation_delay", float("inf")),
                         ("sigma_orientation", -1e-3), ("sigma_joint_velocity", float("inf")), ("gyro_bias", [0.0, float("nan"), 0.0]),
                         ("accel_bias", [0.0, 0.0, -float("inf")]), ("orientation_offset", [float("inf"), 0.0, 0.0])]:
        out.append(hb.make_hardware_settings(2, **{field: value}))
    for value in (0.0, -5.0, float("nan")):
        tl = hb.make_hardware_settings(2)
        tl[1].torque_limit[7] = value
        out.append(tl)
    enc = hb.make_hardware_settings(2)
    enc[0].encoder_offset[9] = float("nan")
    out.append(enc)
    return out


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_rejected_settings(estimated):
    ctx = context()
    rbd0 = start_states(ctx, B, seed=105)
    ep = est_params(seed=10) if estimated else None
    assert_rejected_settings(ctx, "hardware",
                             lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 40, params(5), 5, ep, hb.estimation_states(B, 50) if estimated else None),
                             array_of(_records() * 2), _bad(), hb.make_hardware_settings(ctx.max_batch + 1))
    # the host calls validate their records as the setter does
    rbd = _random_rbd(2, 1)
    for bad in _bad():
        with pytest.raises(hb.HunterB200Error):
            ctx.actuation(0.0, hb.actuation_states(2), np.zeros((2, 10, 5)), rbd, hardware=bad)
        with pytest.raises(hb.HunterB200Error):
            ctx.read_sensors(rbd, hb.estimation_states(2), 0, None, hardware=bad)
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 8. properties
def test_encoder_offsets_reach_the_estimate_exactly():
    """Without noise, the estimated joint positions are q_j + encoder_offset[j], one addition each, on every tick; a 0.0 offset leaves q_j."""
    ctx = context()
    rbd0 = start_states(ctx, B, seed=106)
    enc = np.random.default_rng(3).uniform(-0.02, 0.02, (B, 10)); enc[:, 4] = 0.0
    ctx.set_hardware(hb.make_hardware_settings(B, encoder_offset=enc))
    out = outputs(device(ctx, rbd0, GAITS, cmd_vels(B), 40, params(1), 1, est_params(seed=1, scale=0.0), hb.estimation_states(B, 50)))
    log, est_log = out[4], out[7]
    assert np.array_equal(est_log[:, :, 6:16], log[:, :, 6:16] + enc[:, None, :])
    ctx.close()
