"""Planner settings on the device (hb_plan_set_settings): the device planner with records against the host planner with the same records,
the default record against no setting bit for bit, episodes with records against the loop of public calls bit for bit (both WBCs, both time
grids, truth and estimator, and alongside pushes, variations and a terrain), each record acting on its own robot alone with goals, a
latency and controller settings also set, the shared setting contract (null settings, launch counts, continuation, independence,
permutation, instances beyond the setting, clearing, argument checks), and what the records do to the robots on the plant: touchdowns at
the template's period, clearance that grows with swing_height, a template with a flight phase planned and tracked."""
from contextlib import contextmanager

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from episode_ref import (FRICTION, GAITS, GROUND, PUSH, array_of, assert_episode_equal, assert_null_settings, assert_records_act_as_their_values,
                         assert_rejected_settings, assert_setting_episodes, cmd_vels, context, device, est_params, launch_coefficients, outputs, params,
                         small_terrains, start_states, stepwise, use)
from planner_settings_ref import random_settings
from test_planner_settings_host import T, _bad_records, _cases

pytestmark = pytest.mark.gpu

B = 6


class _Lib:
    """The library as the shared setting checks of episode_ref.py call it: they name a per-robot setter hb_rollout_set_<name>, and the
    planner settings' setter is hb_plan_set_settings (every device planner path reads it, not only the episodes)."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        return getattr(self._lib, "hb_plan_set_settings" if name == "hb_rollout_set_planner_settings" else name)


class _Ctx:
    """A Context whose _lib is _Lib: everything else is the context's."""

    def __init__(self, ctx):
        self._ctx, self._lib = ctx, _Lib(ctx._lib)

    def __getattr__(self, name):
        return getattr(self._ctx, name)


def _records():
    """Three records; each changes the stance gait into stepping (instances 0 and 5 stand), a trot or standing-trot template and swing
    settings, so that each moves every robot it is given to."""
    return [
        hb.make_planner_settings(1, swing_height=0.06, gaits={"stance": (["L", "STANCE", "R", "STANCE"], [0.0, 0.25, 0.3, 0.55, 0.6]),
                                                              "trot": (["L", "R"], [0.0, 0.25, 0.5])})[0],
        hb.make_planner_settings(1, swing_height=0.03, swing_time_scale=0.2, feet_bias_y=0.12,
                                 gaits={"stance": (["L", "R"], [0.0, 0.3, 0.6]),
                                        "standing_trot": (["L", "STANCE", "R", "STANCE"], [0.0, 0.3, 0.4, 0.7, 0.8])})[0],
        hb.make_planner_settings(1, swing_height=0.05, feet_bias_x1=0.045, next_stance_z=0.021,
                                 gaits={"stance": (["L", "STANCE", "R", "STANCE"], [0.0, 0.2, 0.3, 0.5, 0.6]), "trot": (["L", "R"], [0.0, 0.35, 0.7]),
                                        "standing_trot": (["L", "STANCE", "R", "STANCE"], [0.0, 0.2, 0.25, 0.45, 0.5])})[0],
    ]


def _ref_fields(r):
    ne, nt = r.n_events, r.n_targets
    segs = [[np.array([list(r.segments[c][a][k][:]) for k in range(r.n_segments[c][a])]).reshape(-1, 6) for a in range(3)] for c in range(4)]
    return (ne, nt, np.array(r.event_times[:ne]), np.array(r.modes[:ne + 1]), np.array(r.target_times[:nt]),
            np.array([list(r.target_states[k][:]) for k in range(nt)]), segs)


def test_device_planner_matches_host_planner_with_settings():
    ctx = hb.Context(horizon_N=40, dt=0.02, max_batch=256, device=0)
    n = 200
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, seed=61)
    settings = random_settings(n, seed=62)
    ctx.set_planner_settings(settings)
    ins = hb.make_plan_inputs(t0, T, x0, cmd, feet, gaits, start)
    rd, lsd, st = ctx.plan_references_gpu(ins, latest)
    rh, lsh = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, settings=settings)
    assert (st == 0).all()
    np.testing.assert_allclose(lsd, lsh, rtol=0, atol=1e-14)
    for i in range(n):
        a, b = _ref_fields(rd[i]), _ref_fields(rh[i])
        assert a[0] == b[0] and a[1] == b[1]
        np.testing.assert_allclose(a[2], b[2], rtol=0, atol=1e-11)
        np.testing.assert_array_equal(a[3], b[3])
        np.testing.assert_allclose(a[4], b[4], rtol=0, atol=1e-11)
        np.testing.assert_allclose(a[5], b[5], rtol=0, atol=1e-8)
        for c in range(4):
            for ax in range(3):
                assert a[6][c][ax].shape == b[6][c][ax].shape
                np.testing.assert_allclose(a[6][c][ax], b[6][c][ax], rtol=0, atol=1e-11)
    # a template too short for the capacities: status -5 on the device as on the host, the others unaffected
    settings[7].gait[hb.GAIT_IDS[gaits[7]]] = hb.gait_template([3, 3], [0.0, 0.005, 0.01])
    ctx.set_planner_settings(settings)
    rd2, _, st2 = ctx.plan_references_gpu(ins, latest)
    assert st2[7] == -5 and (np.delete(st2, 7) == 0).all() and rd2[7].n_events == 0
    assert all(bytes(rd2[i]) == bytes(rd[i]) for i in range(n) if i != 7)
    ctx.close()


def _used_bytes(r):
    """The entries of an HbReference the counts make valid, as bytes (the device planner leaves the others as it finds them)."""
    ne, nt, *arrays = _ref_fields(r)
    return b"".join([np.array([ne, nt]).tobytes()] + [np.ascontiguousarray(a).tobytes() for a in arrays[:4]] +
                    [np.ascontiguousarray(g).tobytes() for c in arrays[4] for g in c])


def test_default_record_is_the_unset_device_planner_bitwise():
    ctx = hb.Context(horizon_N=40, dt=0.02, max_batch=128, device=0)
    n = 100
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, seed=63)
    ins = hb.make_plan_inputs(t0, T, x0, cmd, feet, gaits, start)
    ins_cycle = hb.make_plan_inputs(t0, T, x0, 0.5 * cmd, None, gaits, t0 + 0.1)
    from hunter_bipedal_control_b200 import scenarios as sc
    rbd = sc.consistent_rbd(x0)
    runs = []
    for setting in (None, hb.make_planner_settings(n), hb.make_planner_settings(n // 2), None):
        ctx.set_planner_settings(setting)
        rd, ls, st = ctx.plan_references_gpu(ins, latest)
        cyc = ctx.resident_plan_cycle(True, 0.002, ins_cycle, rbd)
        runs.append([_used_bytes(r) for r in rd] + [np.ascontiguousarray(a).tobytes() for a in (ls, st) + tuple(cyc)])
    for r in runs[1:]:
        assert r == runs[0]
    ctx.close()


@contextmanager
def _on_every_robot(ctx, rec, prm, ep):
    """rec as the planner settings of every robot, cleared on exit."""
    ctx.set_planner_settings(array_of([rec] * B))
    yield prm, ep
    ctx.set_planner_settings(None)


def _mixed(n=B):
    r = _records()
    return array_of([r[i % 3] for i in range(n)])


@pytest.mark.parametrize("wbc", ["weighted", "hierarchical"])
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_episode_equals_the_stepwise_loop_bitwise(wbc, event_nodes, estimated):
    ctx = context(event_nodes)
    ctx.set_wbc_formulation(wbc)
    log_every = 10
    n_ticks = 120 if estimated else 160
    rbd0 = start_states(ctx, B, seed=81)
    vels = cmd_vels(B)
    prm = params(log_every)
    kw = {}
    if wbc == "weighted" and not event_nodes:       # alongside pushes, plant variations and a terrain
        kw = use(ctx, terrains=small_terrains(), plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION),
                 pushes=hb.make_push_schedules(B, 0.15, 0.05, PUSH))
    ep = est_params(seed=2031) if estimated else None
    ctx.set_planner_settings(_mixed())
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 30) if estimated else None)
    r = stepwise(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 30) if estimated else None, **kw)
    assert_episode_equal(d, r)
    ctx.set_planner_settings(None)
    u = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 30) if estimated else None)
    for i in range(B):
        assert not np.array_equal(d[0][i].cpu().numpy(), u[0][i].cpu().numpy()), i
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_each_record_acts_on_its_robot_alone_with_every_other_setting(estimated):
    """With pushes, variations, a terrain, goals, MPC latencies and controller settings in force, robot i with record k in a mixed batch is
    bit for bit robot i of the batch in which every robot has record k."""
    ctx = context()
    rbd0 = start_states(ctx, B, seed=82)
    use(ctx, plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION, motor_strength=0.95), pushes=hb.make_push_schedules(B, 0.05, 0.05, PUSH),
        terrains=small_terrains(), goals=hb.make_goal_schedules(B, 0.15, [0.2, 0.0, 0.1]), mpc_latencies=[0, 1, 2, 0, 3, 1],
        controller_settings=hb.make_controller_settings(B, swing_kp=[150.0, 170.0, 160.0, 180.0, 140.0, 160.0]))
    assert_records_act_as_their_values(ctx, "planner_settings", _records(), _on_every_robot, rbd0, params(10),
                                       est_params(seed=2032) if estimated else None, n_ticks=150, streams=31)
    ctx.close()


@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_null_settings_and_launch_counts(event_nodes, estimated):
    """Default records give the unset episode bit for bit with the same launches, and the launches per MPC cycle and per tick are those of
    no setting."""
    ctx = context(event_nodes)
    rbd0 = start_states(ctx, B, seed=83)
    prm = params(5)
    ep = est_params(seed=9) if estimated else None
    null = hb.make_planner_settings(B)
    assert_null_settings(ctx, "planner_settings", lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 150, prm, 5, ep,
                                                                 hb.estimation_states(B, 50) if estimated else None),
                         (null, hb.make_planner_settings(3)), _mixed())
    ctx.set_planner_settings(None)
    plain = launch_coefficients(ctx, rbd0, GAITS, cmd_vels(B), params(0), ep)
    ctx.set_planner_settings(_mixed())
    assert launch_coefficients(ctx, rbd0, GAITS, cmd_vels(B), params(0), ep) == plain
    ctx.close()


def test_setting_contract():
    ctx = context()
    rbd0 = start_states(ctx, B, seed=84)
    r = _records()
    full = array_of([r[0], r[1], r[2], r[1], r[0], r[2]])
    one = hb.make_planner_settings(B)
    one[0] = r[0]
    other = array_of([r[2], r[0], r[1], r[1], r[2], r[0]])       # instance 3 keeps its record
    part = array_of([r[1], r[2]])
    padded = hb.make_planner_settings(B)
    padded[0], padded[1] = r[1], r[2]
    assert_setting_episodes(_Ctx(ctx), "planner_settings", rbd0, params(10), full, one, other, 3, part, padded)
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_rejected_settings(estimated):
    ctx = context()
    rbd0 = start_states(ctx, B, seed=85)
    ep = est_params(seed=10) if estimated else None
    bad = [rec for _, rec in _bad_records()]
    two = hb.make_planner_settings(2)
    two[1].gait[1].switching_times[1] = float("nan")     # a bad record after a good one
    assert_rejected_settings(_Ctx(ctx), "planner_settings",
                             lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 100, params(5), 5, ep, hb.estimation_states(B, 50) if estimated else None),
                             _mixed(), bad + [two], hb.make_planner_settings(ctx.max_batch + 1))
    ctx.close()


def _trot_episode(settings, n_ticks, seed):
    """len(settings) robots trotting at 0.3 m/s from t = 0.1 s, each with its record, logged every tick. Returns (stats, the toes' and heels'
    heights above the ground per tick (robots x ticks x 4))."""
    n = len(settings)
    ctx = context(max_batch=1024)
    rbd0 = start_states(ctx, n, seed)
    prm = params(1)
    ctx.set_planner_settings(settings)
    vels = np.zeros((n, 2, 4)); vels[:, :, 0] = 0.3
    out = outputs(device(ctx, rbd0, ["trot"] * n, vels, n_ticks, prm, 1))
    stats, log = out[3], out[4]                           # log: robots x ticks x 32
    rows = log.reshape(-1, 32)
    z = np.concatenate([ctx.contact_positions(ctx.rbd_to_centroidal(rows[k:k + 1024])) for k in range(0, len(rows), 1024)]).reshape(n, n_ticks, 4, 3)
    ctx.close()
    return stats, z[..., 2] - GROUND


def _touchdowns(h, lo=0.004, hi=0.012):
    """Tick indices where a foot height series comes down below lo after having been above hi."""
    out, up = [], False
    for k, v in enumerate(h):
        if v > hi:
            up = True
        elif v < lo and up:
            out.append(k); up = False
    return out


def test_touchdowns_follow_the_template_period():
    periods = [0.5, 0.5, 0.6, 0.6]
    settings = hb.make_planner_settings(4, gaits={"trot": [(["L", "R"], [0.0, p / 2, p]) for p in periods]})
    stats, h = _trot_episode(settings, 1250, seed=86)
    assert (stats["fail_tick"] == -1).all() and (stats["plan_rejects"] == 0).all()
    start = int(0.6 / 0.002)
    for i, p in enumerate(periods):
        for c in (0, 1):                                   # the toes
            td = np.array(_touchdowns(h[i, start:, c]))
            assert len(td) >= 3, (i, c, td)
            interval = 0.002 * np.median(np.diff(td))
            assert abs(interval - p) < 0.1 * p, (i, c, interval, p)


def test_clearance_grows_with_swing_height():
    heights = [0.02, 0.02, 0.04, 0.04]
    stats, h = _trot_episode(hb.make_planner_settings(4, swing_height=heights), 750, seed=87)
    assert (stats["fail_tick"] == -1).all() and (stats["plan_rejects"] == 0).all()
    clear = h[:, int(0.3 / 0.002):, :].max(axis=(1, 2))
    assert min(clear[2:]) > max(clear[:2]) + 0.008, clear


def test_template_with_a_flight_phase_is_planned_and_tracked():
    fly = hb.make_planner_settings(2, gaits={"trot": (["L", "FLY", "R", "FLY"], [0.0, 0.27, 0.3, 0.57, 0.6])})
    stats, h = _trot_episode(fly, 750, seed=88)
    assert (stats["plan_rejects"] == 0).all() and (stats["fail_tick"] == -1).all(), stats
    assert np.isfinite(h).all() and h[:, int(0.3 / 0.002):, :].max() > 0.02
