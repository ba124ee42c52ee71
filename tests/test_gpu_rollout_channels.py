"""Recorded channels of the episodes (hb_rollout_set_channel): every channel equals the values the loop of public calls
(episode_ref.stepwise) computes on the same ticks, bit for bit, under both WBCs, both time grids, truth and estimator, and with every
per-robot setting; recording changes no episode output and adds one launch per recorded tick; split calls record what one call records;
buffers are written only where the contract says; the channels agree with each other, with the stats and with the log; argument checks."""
import ctypes as C

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from episode_ref import (FRICTION, GAITS, PUSH, assert_episode_equal, cmd_vels, context, device, est_params, outputs, params, random_goals,
                         small_terrains, start_states, stepwise, use)

pytestmark = pytest.mark.gpu

B = 6
SENTINEL = {np.float64: np.nan, np.int32: -7, np.uint8: 0xAB}


def _buffers(n, rows, names=None):
    """make_channels(n, rows, names), each filled with its type's sentinel."""
    bufs = hb.make_channels(n, rows, names)
    for name, t in bufs.items():
        t.fill_(SENTINEL[hb.CHANNELS[name][1]])
    return bufs


def _host(bufs):
    return {k: v.cpu().numpy() for k, v in bufs.items()}


def _untouched(a):
    return np.isnan(a).all() if a.dtype == np.float64 else (a == SENTINEL[a.dtype.type]).all()


def _written(a):
    return not np.isnan(a).any() if a.dtype == np.float64 else (a != SENTINEL[a.dtype.type]).all()


def _bitwise(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b, dtype=a.dtype)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _recorded(ctx, rbd0, n_ticks, prm, log_every, ep=None, est=None, names=None):
    """One episode call from tick 0 with the channels `names` (default: all) set: (outputs, {name: channel})."""
    bufs = _buffers(rbd0.shape[0], -(-n_ticks // log_every), names)
    ctx.set_channels(bufs)
    out = outputs(device(ctx, rbd0, GAITS, cmd_vels(rbd0.shape[0]), n_ticks, prm, log_every, ep, est))
    ctx.set_channels(None)
    return out, _host(bufs)


class _Observed:
    """The context for episode_ref.stepwise that also keeps what the loop of public calls computed on its logged ticks: every call goes to
    ctx unchanged and returns its result; the outputs of the policy + WBC, the joint command law, the sensor read and the MPC cycle of a
    tick, and the clipped torques and contact forces of its plant step (the last call of a tick), are kept as that tick's values of each
    channel of CHANNELS, (B, width) each, on every log_every-th plant step. The status' MPC entries are -1 on a tick without a cycle."""

    def __init__(self, ctx, log_every):
        self._ctx, self._every, self._tick, self._now = ctx, log_every, 0, {}
        self.rows = {}

    def __getattr__(self, name):
        return getattr(self._ctx, name)

    def _wbc(self, out):
        xd, ud, md, sol, _, wst = out
        self._now.update(x_des=xd, u_des=ud, wbc_solution=sol, mode=md.reshape(-1, 1), wbc_status=wst)
        return out

    def resident_wbc(self, *a, **kw):
        return self._wbc(self._ctx.resident_wbc(*a, **kw))

    def policy_wbc(self, *a, **kw):
        return self._wbc(self._ctx.policy_wbc(*a, **kw))

    def joint_command(self, *a, **kw):
        out = self._ctx.joint_command(*a, **kw)
        self._now["joint_command"] = out[0].reshape(out[0].shape[0], -1)
        return out

    def read_sensors(self, *a, **kw):
        out = self._ctx.read_sensors(*a, **kw)
        self._now["sensors"] = np.concatenate(out, axis=1)
        return out

    def resident_plan_cycle(self, *a, **kw):
        out = self._ctx.resident_plan_cycle(*a, **kw)
        self._now["cycle"] = (out[0]["status"], out[4])
        return out

    def sim_step(self, rbd, tau, *a, **kw):
        out = self._ctx.sim_step(rbd, tau, *a, **kw)
        if self._tick % self._every == 0:
            now = self._now
            none = np.full(rbd.shape[0], -1)
            info, plan = now.pop("cycle", (none, none))
            now.update(torque=np.array(tau), contact_force=out[1], contact_flag=out[2],
                       status=np.c_[now.pop("wbc_status"), info, plan].astype(np.int32))
            for k, v in now.items():
                self.rows.setdefault(k, []).append(np.array(v))
        self._tick += 1
        self._now = {}
        return out


def _loop(ctx, rbd0, n_ticks, prm, log_every, ep=None, est=None, **settings):
    """episode_ref.stepwise of the same episode as device(): (its outputs, {name: the values of each logged tick, (B, rows, width)})."""
    obs = _Observed(ctx, log_every)
    out = stepwise(obs, rbd0, GAITS, cmd_vels(rbd0.shape[0]), n_ticks, prm, log_every, ep, est, **settings)
    return out, {k: np.stack(v, axis=1) for k, v in obs.rows.items()}


def _assert_channels_are_the_loop(got, rec, estimated):
    assert set(rec) == set(hb.CHANNELS) - ({"sensors"} if not estimated else set())
    for name in hb.CHANNELS:
        if name == "sensors" and not estimated:
            assert _untouched(got[name])
            continue
        want = rec[name]
        assert _bitwise(got[name], want), (name, np.argwhere(got[name] != want)[:5])


# ---------------------------------------------------------------------------------------------------------------- 1. the loop of public calls
@pytest.mark.parametrize("wbc,event_nodes,estimated,log_every", [("weighted", False, False, 1), ("hierarchical", True, True, 3),
                                                                  ("weighted", True, True, 1), ("hierarchical", False, False, 3)])
def test_channels_equal_the_stepwise_loop(wbc, event_nodes, estimated, log_every):
    ctx = context(event_nodes)
    ctx.set_wbc_formulation(wbc)
    n_ticks = 100
    rbd0 = start_states(ctx, B, seed=301)
    prm = params(log_every)
    ep = est_params(seed=31) if estimated else None
    d, got = _recorded(ctx, rbd0, n_ticks, prm, log_every, ep, hb.estimation_states(B, 40) if estimated else None)
    r, rec = _loop(ctx, rbd0, n_ticks, prm, log_every, ep, hb.estimation_states(B, 40) if estimated else None)
    assert_episode_equal(d, r)
    _assert_channels_are_the_loop(got, rec, estimated)
    ctx.close()


@pytest.mark.parametrize("log_every", [1, 3])
def test_channels_with_every_setting_equal_the_stepwise_loop(log_every):
    """An estimated episode with pushes, plant variations, a terrain, goals, MPC latencies, hardware records and controller settings."""
    ctx = context()
    n_ticks = 90
    rbd0 = start_states(ctx, B, seed=302)
    prm = params(log_every)
    hw = hb.make_hardware_settings(B - 1, actuation_delay=np.linspace(0.0, 0.012, B - 1), sigma_joint_velocity=0.02,
                                   encoder_offset=np.full((B - 1, 10), 0.003), gyro_bias=[0.01, 0.0, -0.01])
    kw = use(ctx, plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION, motor_strength=0.95),
             pushes=hb.make_push_schedules(B, 0.05, 0.05, PUSH), terrains=small_terrains(), goals=random_goals(rbd0, B, 302),
             mpc_latencies=[0, 2, 5, 1, 0, 3], hardware=hw)
    w = ctx.wbc_settings(); w.swing_kp *= 1.2
    g = hb.default_pd_gains(); g.kp_big_stance = 45.0
    ctx.set_controller_settings(hb.make_controller_settings(B, wbc=w, gains=g))
    ep = est_params(seed=2035)
    d, got = _recorded(ctx, rbd0, n_ticks, prm, log_every, ep, hb.estimation_states(B, 70))
    ctx.set_controller_settings(None)
    ctx.set_wbc_settings(w)
    prm.gains = g
    r, rec = _loop(ctx, rbd0, n_ticks, prm, log_every, ep, hb.estimation_states(B, 70), **kw)
    assert_episode_equal(d, r)
    _assert_channels_are_the_loop(got, rec, True)
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 2, 6. observing only; launches
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_recording_only_observes_and_adds_one_launch_per_recorded_tick(estimated):
    ctx = context()
    n_ticks = 40
    rbd0 = start_states(ctx, B, seed=303)
    ep = est_params(seed=7) if estimated else None

    def run(log_every, bufs):
        ctx.set_channels(bufs)
        c0 = ctx.launch_count
        out = outputs(device(ctx, rbd0, GAITS, cmd_vels(B), n_ticks, params(log_every), log_every, ep, hb.estimation_states(B, 3) if ep else None))
        n = ctx.launch_count - c0
        ctx.set_channels(None)
        return out, n

    for log_every in (1, 3):
        plain, n0 = run(log_every, None)
        rows = -(-n_ticks // log_every)
        rec, n1 = run(log_every, _buffers(B, rows))
        assert_episode_equal(plain, rec)
        assert n1 == n0 + rows, (n0, n1, rows)
        if not estimated:                                   # a truth episode writes no sensors: the sensors alone add no launch
            sens, n2 = run(log_every, _buffers(B, rows, ["sensors"]))
            assert_episode_equal(plain, sens)
            assert n2 == n0
    # log_every == 0 records nothing and launches as without channels, whatever the channels' sizes (no logs to compare)
    plain, n0 = run(0, None)
    bufs = _buffers(1, 1)
    out, n1 = run(0, bufs)
    assert_episode_equal(*[[np.zeros(0) if x is None else x for x in o] for o in (plain, out)])
    assert n1 == n0
    assert all(_untouched(v) for v in _host(bufs).values())
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 3. continuation
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_split_calls_record_what_one_call_records(estimated):
    ctx = context()
    n_ticks, split, log_every = 60, 27, 3
    rbd0 = start_states(ctx, B, seed=304)
    vels = cmd_vels(B)
    prm = params(log_every)
    ep = est_params(seed=8) if estimated else None
    est = (lambda: hb.estimation_states(B, 5)) if estimated else (lambda: None)
    _, one = _recorded(ctx, rbd0, n_ticks, prm, log_every, ep, est())
    first_bufs, second_bufs = _buffers(B, split // log_every), _buffers(B, -(-(n_ticks - split) // log_every))
    ctx.set_channels(first_bufs)
    first = device(ctx, rbd0, GAITS, vels, split, prm, log_every, ep, est())
    ctx.set_channels(second_bufs)
    if ep is None:
        device(ctx, first[0], GAITS, vels, n_ticks - split, prm, log_every, tick0=split, act=first[1], estop=first[2], stats=first[3])
    else:
        device(ctx, first[0], GAITS, vels, n_ticks - split, prm, log_every, ep, first[5], tick0=split, act=first[1], estop=first[2], stats=first[3],
               est_stats=first[6])
    ctx.set_channels(None)
    a, b = _host(first_bufs), _host(second_bufs)
    for name in hb.CHANNELS:
        assert _bitwise(one[name], np.concatenate([a[name], b[name]], axis=1)), name
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 4. buffer edges
def test_writes_stay_inside_the_call():
    """Channels cleared by set_channels keep their sentinel, so does the sensors channel of a truth episode; instances at or beyond the call's
    B and rows at or beyond its ceil(n_ticks / log_every) are not written."""
    ctx = context()
    n_ticks, log_every = 20, 3
    rows = -(-n_ticks // log_every)
    rbd0 = start_states(ctx, B, seed=305)
    bufs = _buffers(B + 2, rows + 2)
    ctx.set_channels(bufs)
    kept = {k: v for k, v in bufs.items() if k not in ("u_des", "contact_flag")}
    ctx.set_channels(kept)
    device(ctx, rbd0, GAITS, cmd_vels(B), n_ticks, params(log_every), log_every)
    ctx.set_channels(None)
    got = _host(bufs)
    assert _untouched(got["u_des"]) and _untouched(got["contact_flag"]) and _untouched(got["sensors"])
    for name, a in got.items():
        assert _untouched(a[B:]) and _untouched(a[:, rows:]), name
        if name not in ("u_des", "contact_flag", "sensors"):
            assert _written(a[:B, :rows]), name
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 5. cross-checks
def test_channels_agree_with_the_stats_the_log_and_each_other():
    ctx = context()
    n_ticks = 150
    rbd0 = start_states(ctx, B, seed=306)
    prm = params(1)
    prm.actuation_delay = 0.0
    d, ch = _recorded(ctx, rbd0, n_ticks, prm, 1)
    st, log = d[3], d[4]
    up = st["fail_tick"] < 0
    assert up.sum() >= 4
    # the stats' torque maximum is the maximum over the recorded torques
    for i in np.nonzero(up)[0]:
        assert np.abs(ch["torque"][i]).max() == st["max_abs_torque"][i]
    # loaded and not stopped, the feed-forward of the command is the WBC's torque
    jc = ch["joint_command"].reshape(B, n_ticks, 10, 5)
    for i in np.nonzero(up)[0]:
        assert np.array_equal(jc[i, :, :, 4], ch["wbc_solution"][i, :, 28:38])
    # no delay: the applied torque is the clipped PD law of this tick's command on the state entering the tick (log)
    lim = np.array(prm.torque_limit[:])
    q, qd = log[:, :, 6:16], log[:, :, 22:32]
    law = jc[..., 2] * (jc[..., 0] - q) + jc[..., 3] * (jc[..., 1] - qd) + jc[..., 4]
    np.testing.assert_allclose(ch["torque"], np.clip(law, -lim, lim), rtol=0, atol=1e-12)
    # the flag says the normal force is positive; the status' MPC entries are -1 off the MPC ticks
    assert ((ch["contact_flag"] == 1) == (ch["contact_force"].reshape(B, n_ticks, 4, 3)[..., 2] > 0)).all()
    off = np.arange(n_ticks) % prm.mpc_every != 0
    assert (ch["status"][:, off, 1:] == -1).all()
    ctx.close()


def test_standing_robots_carry_their_weight():
    """Robots standing still: over the last 0.2 s of a 1 s episode the vertical contact forces of each add up to m g within 2 %."""
    ctx = context()
    n_ticks = 500
    rbd0 = start_states(ctx, B, seed=307)
    prm = params(1)
    bufs = _buffers(B, n_ticks, ["contact_force"])
    ctx.set_channels(bufs)
    d = outputs(device(ctx, rbd0, ["stance"] * B, np.zeros((B, 2, 4)), n_ticks, prm, 1))
    ctx.set_channels(None)
    assert (d[3]["fail_tick"] < 0).all()
    fz = bufs["contact_force"].cpu().numpy().reshape(B, n_ticks, 4, 3)[:, -100:, :, 2].sum(axis=2)
    weight = sc.TOTAL_MASS * 9.81
    assert np.abs(fz / weight - 1.0).max() < 0.02, np.abs(fz / weight - 1.0).max()
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 7. argument checks
def test_rejected_calls():
    ctx = context()
    lib = ctx._lib
    rbd0 = start_states(ctx, B, seed=308)
    n_ticks, log_every = 12, 3
    rows = n_ticks // log_every
    bufs = _buffers(B, rows, ["torque"])
    ctx.set_channels(bufs)
    tau = C.c_void_p(bufs["torque"].data_ptr())
    c0 = ctx.launch_count
    n_channels = len(hb.CHANNELS)
    for channel, n, r, buf in [(-1, B, rows, tau), (n_channels, B, rows, tau), (0, -1, rows, tau), (0, B, -1, tau), (0, B, rows, None),
                               (n_channels, 0, 0, None), (0, 0, -1, None)]:
        assert lib.hb_rollout_set_channel(ctx._h, channel, n, r, buf) == -1, (channel, n, r)
    assert lib.hb_rollout_set_channel(None, 0, B, rows, tau) == -1
    assert lib.hb_rollout_set_channel(ctx._h, 0, ctx.max_batch + 1, rows, tau) == -4
    assert ctx.launch_count == c0
    # the rejected calls kept the channel
    bufs["torque"].fill_(np.nan)
    device(ctx, rbd0, GAITS, cmd_vels(B), n_ticks, params(log_every), log_every)
    assert not np.isnan(bufs["torque"].cpu().numpy()).any()
    # an episode call with a set channel of too few instances or rows enqueues nothing and returns -1
    for n, r in [(B - 1, rows), (B, rows - 1)]:
        small = _buffers(n, r, ["mode"])
        ctx.set_channels(small)
        c0 = ctx.launch_count
        with pytest.raises(hb.HunterB200Error, match=r"\(-1\)"):
            device(ctx, rbd0, GAITS, cmd_vels(B), n_ticks, params(log_every), log_every)
        assert ctx.launch_count == c0
        assert _untouched(small["mode"].cpu().numpy())
    # clearing: B == 0 with a NULL buffer, then the call runs and writes nothing
    assert lib.hb_rollout_set_channel(ctx._h, hb.CHANNELS["mode"][0], 0, 0, None) == 0
    device(ctx, rbd0, GAITS, cmd_vels(B), n_ticks, params(log_every), log_every)
    assert _untouched(small["mode"].cpu().numpy())
    # the Python setter checks types and shapes, and clears every channel on an error
    ctx.set_channels(bufs)
    for bad in [{"nope": bufs["torque"]}, {"torque": bufs["torque"].float()}, {"torque": bufs["torque"][:, :, :5]},
                {"torque": bufs["torque"].cpu()}, {"mode": bufs["torque"]}]:
        with pytest.raises(ValueError):
            ctx.set_channels(bad)
    big = hb.make_channels(ctx.max_batch + 1, rows, ["torque", "mode"])
    with pytest.raises(hb.HunterB200Error, match=r"\(-4\)"):
        ctx.set_channels({"x_des": bufs["torque"].new_zeros((B, rows, 22)), **big})
    assert ctx._channels == {}
    bufs["torque"].fill_(np.nan)
    device(ctx, rbd0, GAITS, cmd_vels(B), n_ticks, params(log_every), log_every)
    assert _untouched(bufs["torque"].cpu().numpy())
    ctx.close()
