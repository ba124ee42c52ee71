"""Estimator maps on the device (hb_estimator_set_maps): the public filter call on maps against the restatement (estimator_map_ref.py);
unset, cleared, NULL and all-zero maps against no setting bit for bit, in the filter call and the estimated episode, with the truth
episodes untouched; the mapped estimated episode against the loop of public calls bit for bit (both WBCs, both time grids, with terrains,
planner maps, pushes, variations, goals, teleop, latencies, hardware settings and odometry alongside); the shared setting contract;
snapshots resumed with the same maps; and what the maps are for: the base-height estimate of robots standing on a plateau."""
import numpy as np
import pytest
import torch

import hunter_bipedal_control_b200 as hb
from episode_ref import (FRICTION, GAITS, GROUND, PUSH, array_of, assert_episode_equal, assert_null_settings, assert_rejected_settings,
                         assert_setting_episodes, cmd_vels, context, device, est_params, launch_coefficients, outputs, params, random_goals,
                         start_states, stepwise, use)
from estimator_map_ref import MappedKalmanFilterRef
from test_gpu_estimator_envelope import _kin, kf_arrays, kf_prm_dict, sensor_inputs
from test_gpu_height_maps import episode_maps
from test_gpu_rollout_hardware import _offsets
from test_gpu_rollout_odometry import _settings as odometry_settings
from test_gpu_rollout_teleop import mixed
import height_map_ref as M

pytestmark = pytest.mark.gpu

B = 6


# ---------------------------------------------------------------------------------------------------------------- 1. the filter call
def _filter_maps(n):
    """Stepped, sloped, random and plateau maps, by instance modulo 4, under the feet's neighbourhood (the filter starts at the origin)."""
    out = []
    for i in range(n):
        k = i % 4
        if k == 0:
            out.append(M.step_map(1, -0.04 + 0.02 * (i % 5), 0.03 + 0.01 * (i % 3), origin=(-0.6, -0.64))[0])
        elif k == 1:
            out.append(M.slope_map(1, 0.1 - 0.05 * (i % 5), axis=i % 2, spacing=0.03, n=30, origin=(-0.45, -0.45))[0])
        elif k == 2:
            out.append(M.random_maps(1, 100 + i, scale=0.04, spacing=0.05, n=20, origin=(-0.5, -0.5))[0])
        else:
            out.append(M.plateau(1, 0.1 * (i % 7) - 0.3)[0])
    return array_of(out)


def _points(m, c, k):
    """Foot c's lookup point on the map m at step k: a grid corner (c = 0), a point on a cell edge along x (1) and along y (2), and off
    the grid (3: beyond either end, with the other coordinate on or off the grid)."""
    o, s, nx, ny = m.origin, m.spacing, m.nx, m.ny
    i, j = (3 * k) % (nx - 1), (5 * k) % (ny - 1)
    if c == 0:
        return o[0] + i * s, o[1] + j * s
    if c == 1:
        return o[0] + (i + 0.37) * s, o[1] + j * s
    if c == 2:
        return o[0] + i * s, o[1] + (j + 0.61) * s
    return ((o[0] - 0.2 - 0.01 * k, o[1] + j * s), (o[0] + nx * s + 0.3, o[1] - 0.1), (o[0] + 0.5 * s, o[1] + ny * s + 0.05))[k % 3]


def test_filter_call_on_maps_matches_the_restatement():
    """64 instances: the 16 contact patterns over mapped instances (48, the maps of _filter_maps) and unmapped ones beyond the setting
    (16), 30 steps. Instances 16..31 have their feet put on grid corners, cell edges and off the grid before every step, in the device
    state and the restatement alike. Tolerances of test_gpu_estimator_envelope.py: 1e-9 on rbd and x_hat, 1e-9 relative on P, P exactly
    symmetric."""
    ctx = hb.Context(horizon_N=10, dt=0.02, max_batch=64, device=0)
    rng = np.random.default_rng(51)
    n, mapped = 64, 48
    maps = _filter_maps(mapped)
    ctx.set_estimator_maps(maps)
    st = hb.kf_states(n)
    refs = [MappedKalmanFilterRef(maps[i] if i < mapped else None) for i in range(n)]
    prm = kf_prm_dict(hb.default_kf_params())
    flags = np.array([[(p >> c) & 1 for c in range(4)] for p in range(16)] * 4, dtype=np.uint8)
    zyx = np.c_[rng.uniform(-np.pi, np.pi, n), rng.uniform(-0.3, 0.3, (n, 2))]
    for k in range(30):
        for i in range(16, 32):
            for c in range(4):
                px, py = _points(maps[i], c, k + i)
                st[i].x_hat[6 + 3 * c], st[i].x_hat[7 + 3 * c] = px, py
                refs[i].x[6 + 3 * c], refs[i].x[7 + 3 * c] = px, py
        quat, wl, al, jpos, jvel = sensor_inputs(rng, zyx + rng.normal(0, 1e-3, (n, 3)))
        rbd = ctx.estimator_update(0.002, st, quat, wl, al, jpos, jvel, flags)
        x, P = kf_arrays(st)
        for i, ref in enumerate(refs):
            rr = ref.update(0.002, quat[i], wl[i], al[i], jpos[i], jvel[i], flags[i], _kin, prm=prm)
            assert np.abs(rbd[i] - rr).max() < 1e-9, (k, i, np.abs(rbd[i] - rr).max())
            assert np.abs(x[i] - ref.x).max() < 1e-9, (k, i, np.abs(x[i] - ref.x).max())
            assert np.abs(P[i] - ref.P).max() < 1e-9 * max(1.0, np.abs(ref.P).max()), (k, i)
            assert np.array_equal(P[i], P[i].T)
    # a mapped update does not write feet_heights: they stay as hb_kf_reset left them
    assert (np.frombuffer(st, dtype=np.float64).reshape(n, -1)[:, 342:] == 0.0).all()
    ctx.close()


def test_unmapped_instances_are_the_filter_without_the_setting_bitwise():
    """Unset, cleared (B == 0 with and without an array), NULL and all-zero maps: the filter call gives the unset call's rbd and states bit
    for bit; instances beyond a setting too."""
    ctx = hb.Context(horizon_N=10, dt=0.02, max_batch=64, device=0)
    rng = np.random.default_rng(52)
    n = 40
    zyx = np.c_[rng.uniform(-np.pi, np.pi, n), rng.uniform(-0.3, 0.3, (n, 2))]
    ins = [sensor_inputs(rng, zyx) + ((rng.uniform(size=(n, 4)) > 0.3).astype(np.uint8),) for _ in range(8)]

    def run():
        st = hb.kf_states(n)
        return [ctx.estimator_update(0.002, st, *x).tobytes() for x in ins] + [bytes(st)]

    want = run()
    lib, h = ctx._lib, ctx._h
    for setting in ("zero", "zero_big", "cleared", "cleared_array", "null"):
        ctx.set_estimator_maps(_filter_maps(n))
        if setting == "zero":
            ctx.set_estimator_maps(M.zero_maps(n))
        elif setting == "zero_big":
            ctx.set_estimator_maps(hb.make_terrains(n // 2, np.zeros((64, 64)), 0.01, (-0.3, -0.3)))
        elif setting == "cleared":
            ctx.set_estimator_maps(None)
        elif setting == "cleared_array":
            assert lib.hb_estimator_set_maps(h, 0, _filter_maps(2)) == 0
        else:
            assert lib.hb_estimator_set_maps(h, 0, None) == 0
        assert run() == want, setting
    ctx.set_estimator_maps(_filter_maps(n // 2))
    got = run()
    assert got != want
    part = np.frombuffer(got[-1], dtype=np.float64).reshape(n, -1)
    assert np.array_equal(part[n // 2:], np.frombuffer(want[-1], dtype=np.float64).reshape(n, -1)[n // 2:])
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 2. null settings in episodes
def _with_channels(ctx, run, rows):
    """run() with every channel set on ctx: (the episode, the channels' contents)."""
    def go():
        ch = hb.make_channels(B, rows)
        for t in ch.values():
            t.fill_(7)
        ctx.set_channels(ch)
        out = run()
        torch.cuda.synchronize()
        got = {k: v.cpu().numpy().copy() for k, v in ch.items()}
        ctx.set_channels(None)
        return out, got
    return go


@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
def test_null_settings_launch_counts_and_truth_episodes(event_nodes):
    """Zero maps, and maps set then cleared, give the unset estimated episode bit for bit in every output (stats, est_stats, log, est_log)
    and every recorded channel, with the same launches; the launches per MPC cycle and per tick are those of no setting; truth episodes do
    not read the setting."""
    ctx = context(event_nodes)
    rbd0 = start_states(ctx, B, seed=111)
    prm = params(5)
    ep = est_params(seed=21)
    channels = []

    def run():
        out, ch = _with_channels(ctx, lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 150, prm, 5, ep, hb.estimation_states(B, 50)), 30)()
        channels.append(ch)
        return out

    assert_null_settings(ctx, "estimator_maps", run, (M.zero_maps(B), M.zero_maps(3), M.zero_maps(B, n=64, spacing=0.01)), episode_maps(rbd0))
    for ch in channels[1:]:
        assert ch.keys() == channels[0].keys()
        for k in ch:
            assert np.array_equal(ch[k], channels[0][k]), k
    ctx.set_estimator_maps(None)
    plain = launch_coefficients(ctx, rbd0, GAITS, cmd_vels(B), params(0), ep)
    ctx.set_estimator_maps(episode_maps(rbd0))
    assert launch_coefficients(ctx, rbd0, GAITS, cmd_vels(B), params(0), ep) == plain
    # the truth episode does not read the setting; the estimated one does
    mapped = outputs(device(ctx, rbd0, GAITS, cmd_vels(B), 150, prm, 5, ep, hb.estimation_states(B, 50)))
    truth, n = [], []
    for setting in (episode_maps(rbd0), None):
        ctx.set_estimator_maps(setting)
        c0 = ctx.launch_count
        truth.append(device(ctx, rbd0, GAITS, cmd_vels(B), 150, prm, 5))
        n.append(ctx.launch_count - c0)
    assert n[0] == n[1]
    assert_episode_equal(truth[0], truth[1])
    unset = outputs(device(ctx, rbd0, GAITS, cmd_vels(B), 150, prm, 5, ep, hb.estimation_states(B, 50)))
    assert sum(not np.array_equal(a, b) for a, b in zip(mapped[7], unset[7])) >= B - 1
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 3. the loop of public calls
@pytest.mark.parametrize("wbc", ["weighted", "hierarchical"])
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
def test_mapped_estimated_episode_equals_the_stepwise_loop_bitwise(wbc, event_nodes):
    """The estimated episode on estimator maps equals episode_ref.stepwise, whose filter call reads the same maps, bit for bit. On the
    weighted uniform grid with the terrains the maps describe, planner maps, pushes, variations, goals and teleop; on the hierarchical
    uniform grid with MPC latencies, hardware settings, odometry and goals; on event nodes with planner maps."""
    ctx = context(event_nodes)
    ctx.set_wbc_formulation(wbc)
    log_every, n_ticks = 10, 120
    rbd0 = start_states(ctx, B, seed=112)
    vels = cmd_vels(B)
    prm = params(log_every)
    maps = episode_maps(rbd0)
    kw, goals, teleop, planner_maps = {}, None, None, maps
    if wbc == "weighted" and not event_nodes:
        hm = np.ctypeslib.as_array(maps)["height"]
        ter = hb.make_terrains(B, hm[:, :40, :40] + GROUND, 0.02, rbd0[:, 3:5] - 0.4)
        kw = use(ctx, terrains=ter, plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION), pushes=hb.make_push_schedules(B, 0.15, 0.05, PUSH))
        goals, teleop = random_goals(rbd0, B, 112), mixed(B)
    if wbc == "hierarchical" and not event_nodes:
        kw = use(ctx, mpc_latencies=[5, 0, 2, 3], hardware=_offsets(B - 1), odometry=odometry_settings(B - 1))
        goals, planner_maps = random_goals(rbd0, B, 113), None
    if wbc == "weighted" and event_nodes:
        maps = array_of(list(maps)[:B - 2])                     # two robots beyond the setting
    if goals is not None:
        ctx.set_goals(goals)
    if teleop is not None:
        ctx.set_teleop(teleop)
    ep = est_params(seed=2051)
    ctx.set_height_maps(planner_maps)
    ctx.set_estimator_maps(maps)
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 30))
    loop = M.MapLoop(ctx, planner_maps if planner_maps is not None else [], prm.period, goals=goals, teleop=teleop)
    r = stepwise(loop, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 30), **kw)
    ctx.set_plan_targets(None)
    assert_episode_equal(d, r)
    ctx.set_estimator_maps(None)
    u = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 30))
    moved = [not np.array_equal(a, b) for a, b in zip(outputs(d)[7], outputs(u)[7])]
    assert sum(moved[:len(maps)]) >= len(maps) - 1 and not any(moved[len(maps):]), moved
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 4. the setting contract
class _Lib:
    """The library as the shared setting checks call it: they name a per-robot setter hb_rollout_set_<name>; the estimator maps' setter is
    hb_estimator_set_maps (the public filter call reads it too, not only the episodes)."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        return getattr(self._lib, "hb_estimator_set_maps" if name == "hb_rollout_set_estimator_maps" else name)


class _Estimated:
    """The context as assert_setting_episodes runs it: its episode calls (Context.rollout) go through the estimator, with noise-free
    sensors, so that the episode of a robot does not depend on its noise stream and a permuted batch is the permuted episode. A call from
    tick 0 starts from fresh estimation states, and a call from a later tick continues the estimation state and stats of the call before.
    It returns Context.rollout's five outputs, the log holding the true and the estimated state side by side (B, rows, 64); the
    estimation state and stats are compared by the other tests."""

    EP = est_params(scale=0.0)

    def __init__(self, ctx):
        self._ctx, self._lib = ctx, _Lib(ctx._lib)
        self._carry = None

    def __getattr__(self, name):
        return getattr(self._ctx, name)

    def rollout(self, rbd, cmds, n_ticks, tick0=0, params=None, act=None, estop=None, stats=None, log_every=0):
        est, est_stats = (None, None) if tick0 == 0 else self._carry
        out = self._ctx.rollout_estimated(rbd, cmds, n_ticks, tick0=tick0, params=params, est_params=self.EP, est=est, act=act, estop=estop,
                                          stats=stats, est_stats=est_stats, log_every=log_every)
        self._carry = (out[5], out[6])
        return out[:4] + (out[4] if out[4] is None else torch.cat([out[4], out[7]], dim=2),)


def test_setting_contract():
    ctx = context()
    rbd0 = start_states(ctx, B, seed=113)
    full = episode_maps(rbd0)
    one = M.zero_maps(B)
    one[0] = full[0]
    other = episode_maps(rbd0, rise=(-0.04, 0.05, 0.01, 0.0, -0.01, 0.02))
    other[3] = full[3]                                            # instance 3 keeps its map
    part = array_of([full[1], full[2]])
    padded = M.zero_maps(B)
    padded[0], padded[1] = full[1], full[2]
    # maps follow the robots' start positions, so permuting states and maps together is the permuted episode
    assert_setting_episodes(_Estimated(ctx), "estimator_maps", rbd0, params(10), full, one, other, 3, part, padded)
    ctx.close()


def test_rejected_settings():
    ctx = context()
    rbd0 = start_states(ctx, B, seed=114)
    ep = est_params(seed=23)
    bad = []
    for field, value in [("nx", 1), ("ny", 65), ("spacing", 0.0), ("spacing", float("nan"))]:
        r = M.zero_maps(1); setattr(r[0], field, value); bad.append(r)
    two = M.zero_maps(2)
    two[1].height[1][1] = float("inf")                        # a bad record after a good one
    assert_rejected_settings(_Estimated(ctx), "estimator_maps",
                             lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 100, params(5), 5, ep, hb.estimation_states(B, 50)),
                             episode_maps(rbd0), bad + [two], M.zero_maps(ctx.max_batch + 1))
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 5. snapshots
def test_snapshots_with_maps_continue_exactly():
    """Saved mid-episode with estimator and planner maps set and restored in a fresh context given the same maps: one call. Maps are not
    episode state: the row size is unchanged."""
    n1, n2 = 115, 85
    ctx = context()
    rbd0 = start_states(ctx, B, seed=115)
    vels = cmd_vels(B)
    ep = est_params(seed=24)
    maps = episode_maps(rbd0)
    plain_bytes = ctx.episode_state_bytes
    ctx.set_estimator_maps(maps)
    ctx.set_height_maps(maps)
    assert ctx.episode_state_bytes == plain_bytes
    one = device(ctx, rbd0, GAITS, vels, n1 + n2, params(5), 5, ep, hb.estimation_states(B, 40))
    first = device(ctx, rbd0, GAITS, vels, n1, params(5), 5, ep, hb.estimation_states(B, 40))
    snap = ctx.save_episodes(B, *first[:4], *first[5:7])
    ctx.close()
    ctx2 = context()
    ctx2.set_estimator_maps(maps)
    ctx2.set_height_maps(maps)
    r = ctx2.restore_episodes(snap)
    second = device(ctx2, r[0], GAITS, vels, n2, params(5), 5, ep, r[4], tick0=n1, act=r[1], estop=r[2], stats=r[3], est_stats=r[5])
    two = outputs(second)
    two[4] = np.concatenate([first[4].cpu().numpy(), two[4]], axis=1)
    two[7] = np.concatenate([first[7].cpu().numpy(), two[7]], axis=1)
    assert_episode_equal(one, two)
    ctx2.close()


# ---------------------------------------------------------------------------------------------------------------- 6. a property
# The base-height estimates of robots on a plateau with the map agree with those of the same robots on flat ground to this tolerance. It
# was a guess set before any measurement; the first run on an H100 measured at most 8.2e-5 m (printed by the test).
PLATEAU_TOL = 1e-3


def _up_rows(fail, log_every, n_rows):
    """The logged rows after row 0 at which none of the robots with fail ticks `fail` has failed."""
    return [k for k in range(1, n_rows) if all(f < 0 or k * log_every < f for f in fail)]


def test_plateau_base_height_estimate():
    """Robots 0-2 stand for 1 s on a plateau terrain at c, with the map c - g (g the flat ground), as planner and estimator map; robots
    3-5 are the same robots on the flat ground. Every filter starts at its robot's true base position and contact points, so that the
    plateau robots do not start c - g away from their estimate. With the estimator map the base-height estimate errors (estimate - truth)
    of the two groups agree to PLATEAU_TOL; without it, the plateau robots' estimate is low by about c - g. Noise-free sensors. The
    rise c - g is 2 cm: on a 15 cm rise the robots with a right height estimate stop on a joint limit after about 0.2 s (DESIGN §1
    "Estimator maps"), so rows are compared while every robot is up."""
    c, n_ticks, log_every = 0.04, 500, 10
    ctx = context()
    flat = start_states(ctx, 3, seed=116)
    rbd0 = np.concatenate([flat, flat])
    rbd0[:3, 5] += c - GROUND
    feet = ctx.contact_positions(ctx.rbd_to_centroidal(rbd0)).reshape(B, 4, 3) - [0.0, 0.0, hb.default_kf_params().foot_radius]

    def fresh():
        est = hb.estimation_states(B, 0)
        for i in range(B):
            est[i].kf.x_hat[0:3] = rbd0[i, 3:6].tolist()
            est[i].kf.x_hat[6:18] = feet[i].reshape(-1).tolist()
        return est

    prm = params(log_every)
    ep = est_params(scale=0.0)
    lift = M.plateau(3, c - GROUND)
    use(ctx, terrains=M.plateau(3, c), height_maps=lift)
    gaits, vels = ["stance"] * B, np.zeros((B, 2, 4))
    err = {}
    for name, setting in (("mapped", lift), ("blind", None)):
        ctx.set_estimator_maps(setting)
        out = outputs(device(ctx, rbd0, gaits, vels, n_ticks, prm, log_every, ep, fresh()))
        print(name, "fail_tick", out[3]["fail_tick"].tolist(), "fail_reason", out[3]["fail_reason"].tolist())
        assert (out[3]["fail_tick"][3:] < 0).all()
        err[name] = (out[7][:, :, 5] - out[4][:, :, 5], out[3]["fail_tick"])
    e, fail = err["mapped"]
    rows = _up_rows(fail, log_every, e.shape[1])
    assert len(rows) >= 8, rows
    d = e[:3, rows] - e[3:, rows]
    print("plateau at %g m: |estimate error on the plateau - on flat ground| over %d logged ticks, max %.3g m" % (c, len(rows), np.abs(d).max()))
    assert np.abs(d).max() < PLATEAU_TOL, d
    e, fail = err["blind"]
    rows = _up_rows(fail, log_every, e.shape[1])
    assert len(rows) >= 8, rows
    off = e[:3, rows] - e[3:, rows]
    print("without the estimator map: plateau - flat estimate error from %.4f to %.4f m (c - g = %g m)" % (off.min(), off.max(), c - GROUND))
    assert np.abs(off + (c - GROUND)).max() < 0.1 * (c - GROUND), off
    ctx.close()
