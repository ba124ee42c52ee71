"""Height maps on the device (hb_plan_set_maps): the three device planner paths on maps against the host planner on the same maps, unset and
all-zero maps against no setting bit for bit, the episodes' goal and teleop captures on maps against the host conversions, episodes with
maps against the loop of public calls bit for bit (both WBCs, both time grids, truth and estimator, alongside terrains, goals, teleop,
planner settings, latencies and pushes), the shared setting contract, and snapshots resumed with the same maps."""
import ctypes as C

import numpy as np
import pytest
import torch

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from episode_ref import (FRICTION, GAITS, GROUND, PUSH, array_of, assert_episode_equal, assert_null_settings,
                         assert_rejected_settings, assert_setting_episodes, cmd_vels, context, device, est_params, launch_coefficients, outputs,
                         params, random_goals, start_states, stepwise, use)
from planner_settings_ref import random_settings
from test_gpu_planner_settings import _ref_fields, _records, _used_bytes
from test_gpu_rollout_teleop import mixed
from test_height_maps_host import _cases, _map_cases, T
import height_map_ref as M

pytestmark = pytest.mark.gpu

B = 6


class _Lib:
    """The library as the shared setting checks of episode_ref.py call it: they name a per-robot setter hb_rollout_set_<name>, and the
    height maps' setter is hb_plan_set_maps (every device planner path reads it, not only the episodes)."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        return getattr(self._lib, "hb_plan_set_maps" if name == "hb_rollout_set_height_maps" else name)


class _Ctx:
    def __init__(self, ctx):
        self._ctx, self._lib = ctx, _Lib(ctx._lib)

    def __getattr__(self, name):
        return getattr(self._ctx, name)


def episode_maps(rbd0, n=None, rise=(0.03, -0.02, 0.05, 0.0, 0.04, -0.03)):
    """A step map per robot: flat around its start, a step of rise[i] 0.12 m ahead along world x and a 2 % slope along y, on a 2 cm grid
    around the start (the maps of terrains at GROUND + the map)."""
    n = rbd0.shape[0] if n is None else n
    xs, ys = 0.02 * np.arange(40) - 0.4, 0.02 * np.arange(40) - 0.4
    hm = np.stack([np.where(xs[None, :] >= 0.12, rise[i % len(rise)], 0.0) + 0.02 * ys[:, None] for i in range(n)])
    return hb.make_terrains(n, hm, 0.02, rbd0[:n, 3:5] - 0.4)


def _plan_batch_dev(ctx, ins, latest):
    """hb_plan_references_batch_dev on device copies of the inputs: (refs, latest_stance, status)."""
    n = len(ins)
    d_in = torch.frombuffer(bytearray(bytes(ins)), dtype=torch.uint8).cuda()
    d_ls = torch.tensor(latest, dtype=torch.float64).cuda()
    d_out = torch.zeros(n * C.sizeof(hb.HbReference), dtype=torch.uint8).cuda()
    d_st = torch.zeros(n, dtype=torch.int32).cuda()
    P = lambda t: C.c_void_p(t.data_ptr())
    assert ctx._lib.hb_plan_references_batch_dev(ctx._h, n, P(d_in), None, P(d_ls), P(d_out), P(d_st)) == 0
    torch.cuda.synchronize()
    refs = (hb.HbReference * n).from_buffer_copy(d_out.cpu().numpy().tobytes())
    return refs, d_ls.cpu().numpy(), d_st.cpu().numpy()


def _assert_plans_close(rd, rh, n):
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


@pytest.mark.parametrize("with_settings", [False, True], ids=["compiled_in", "settings"])
def test_device_planner_paths_match_the_host_planner_on_maps(with_settings):
    ctx = hb.Context(horizon_N=40, dt=0.02, max_batch=256, device=0)
    n = 200
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, seed=91)
    maps = _map_cases(n, 92)
    settings = random_settings(n, seed=93) if with_settings else None
    ctx.set_planner_settings(settings)
    ctx.set_height_maps(maps)
    ins = hb.make_plan_inputs(t0, T, x0, cmd, feet, gaits, start)
    rd, lsd, st = ctx.plan_references_gpu(ins, latest)
    rh, lsh = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, settings=settings, maps=maps)
    assert (st == 0).all()
    np.testing.assert_allclose(lsd, lsh, rtol=0, atol=1e-14)
    _assert_plans_close(rd, rh, n)
    rb, lsb, stb = _plan_batch_dev(ctx, ins, latest)
    assert (stb == 0).all() and lsb.tobytes() == lsd.tobytes()
    assert all(_used_bytes(rb[i]) == _used_bytes(rd[i]) for i in range(n))
    # the maps move every plan, and instances beyond the setting plan without one
    ctx.set_height_maps(None)
    ru, _, _ = ctx.plan_references_gpu(ins, latest)
    assert sum(_used_bytes(ru[i]) != _used_bytes(rd[i]) for i in range(n)) >= n - 4
    ctx.set_height_maps((hb.HbTerrain * 50)(*maps[:50]))
    rp, _, _ = ctx.plan_references_gpu(ins, latest)
    assert all(_used_bytes(rp[i]) == _used_bytes(rd[i] if i < 50 else ru[i]) for i in range(n))
    ctx.close()


def test_unset_and_zero_maps_are_the_unset_planner_bitwise():
    ctx = hb.Context(horizon_N=40, dt=0.02, max_batch=128, device=0)
    n = 100
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, seed=94)
    ins = hb.make_plan_inputs(t0, T, x0, cmd, feet, gaits, start)
    ins_cycle = hb.make_plan_inputs(t0, T, x0, 0.5 * cmd, None, gaits, t0 + 0.1)
    rbd = sc.consistent_rbd(x0)
    runs = []
    for setting in (None, M.zero_maps(n), hb.make_terrains(n // 2, np.zeros((64, 64)), 0.01, (-0.3, -0.3)), None):
        ctx.set_height_maps(setting)
        rd, ls, st = ctx.plan_references_gpu(ins, latest)
        rb, lsb, stb = _plan_batch_dev(ctx, ins, latest)
        cyc = ctx.resident_plan_cycle(True, 0.002, ins_cycle, rbd)
        runs.append([_used_bytes(r) for r in rd] + [_used_bytes(r) for r in rb] +
                    [np.ascontiguousarray(a).tobytes() for a in (ls, st, lsb, stb) + tuple(cyc)])
    for r in runs[1:]:
        assert r == runs[0]
    # maps move the resident cycle
    ctx.set_height_maps(_map_cases(n, 95))
    assert np.ascontiguousarray(ctx.resident_plan_cycle(True, 0.002, ins_cycle, rbd)[1]).tobytes() != runs[0][-4]
    ctx.close()


def test_episode_captures_on_maps_are_the_host_conversions():
    """With goals and teleop on maps, the episode equals the loop whose goal targets are hb_goal_to_target_maps of the tick's state and
    whose message targets are the device planner's cmd_vel targets on the same maps, bit for bit; a goal given at tick 0 is captured as the
    host conversion of the start state."""
    ctx = context()
    rbd0 = start_states(ctx, B, seed=96)
    maps = episode_maps(rbd0)
    prm = params(10)
    g0 = np.c_[rbd0[:, 3] + 0.3, rbd0[:, 4] + 0.1, rbd0[:, 0]]
    goals = hb.make_goal_schedules(B, 0.0, g0[:, None, :])
    teleop = mixed(B)
    teleop[0] = hb.make_teleop_settings(1, windows=[])[0]       # robot 0 keeps its tick-0 goal
    ctx.set_goals(goals)
    ctx.set_teleop(teleop)
    ctx.set_height_maps(maps)
    d = device(ctx, rbd0, GAITS, cmd_vels(B), 150, prm, 10)
    loop = M.MapLoop(ctx, maps, prm.period, goals=goals, teleop=teleop)
    r = stepwise(loop, rbd0, GAITS, cmd_vels(B), 150, prm, 10)
    ctx.set_plan_targets(None)
    assert_episode_equal(d, r)
    want = hb.goal_to_target(0.0, ctx.rbd_to_centroidal(rbd0), g0, maps=maps)
    assert loop._src[0] == 0 and bytes(loop._tg[0]) == bytes(want[0])
    assert loop._tg[5] is not None and bytes(loop._tg[5]) == bytes(want[5])      # robot 5 has no teleop record
    assert any(v == "msg" for v in loop._src.values())
    ctx.close()


@pytest.mark.parametrize("wbc", ["weighted", "hierarchical"])
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_episode_equals_the_stepwise_loop_bitwise(wbc, event_nodes, estimated):
    ctx = context(event_nodes)
    ctx.set_wbc_formulation(wbc)
    log_every = 10
    n_ticks = 120 if estimated else 160
    rbd0 = start_states(ctx, B, seed=97)
    vels = cmd_vels(B)
    prm = params(log_every)
    maps = episode_maps(rbd0)
    kw, goals, teleop = {}, None, None
    if wbc == "weighted" and not event_nodes:       # on the terrains the maps describe, with pushes, variations, goals and teleop
        hm = np.ctypeslib.as_array(maps)["height"]
        ter = hb.make_terrains(B, hm[:, :40, :40] + GROUND, 0.02, rbd0[:, 3:5] - 0.4)
        kw = use(ctx, terrains=ter, plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION), pushes=hb.make_push_schedules(B, 0.15, 0.05, PUSH))
        goals, teleop = random_goals(rbd0, B, 97), mixed(B)
    if wbc == "hierarchical" and not event_nodes:   # with planner settings, MPC latencies and goals
        ctx.set_planner_settings(array_of([_records()[i % 3] for i in range(B)]))
        kw = use(ctx, mpc_latencies=[5, 0, 2, 3])
        goals = random_goals(rbd0, B, 98)
    if goals is not None:
        ctx.set_goals(goals)
    if teleop is not None:
        ctx.set_teleop(teleop)
    ep = est_params(seed=2041) if estimated else None
    fresh = lambda: hb.estimation_states(B, 30) if estimated else None
    ctx.set_height_maps(maps)
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, fresh())
    loop = M.MapLoop(ctx, maps, prm.period, goals=goals, teleop=teleop)
    r = stepwise(loop, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, fresh(), **kw)
    ctx.set_plan_targets(None)
    assert_episode_equal(d, r)
    ctx.set_height_maps(None)
    u = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, fresh())
    moved = [not np.array_equal(a, b) for a, b in zip(d[0].cpu().numpy(), u[0].cpu().numpy())]
    assert sum(moved) >= B - 1, moved
    ctx.close()


@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_null_settings_and_launch_counts(event_nodes, estimated):
    """Zero maps give the unset episode bit for bit with the same launches, and the launches per MPC cycle and per tick are those of no
    setting."""
    ctx = context(event_nodes)
    rbd0 = start_states(ctx, B, seed=99)
    prm = params(5)
    ep = est_params(seed=12) if estimated else None
    assert_null_settings(ctx, "height_maps", lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 150, prm, 5, ep,
                                                            hb.estimation_states(B, 50) if estimated else None),
                         (M.zero_maps(B), M.zero_maps(3)), episode_maps(rbd0))
    ctx.set_height_maps(None)
    plain = launch_coefficients(ctx, rbd0, GAITS, cmd_vels(B), params(0), ep)
    ctx.set_height_maps(episode_maps(rbd0))
    assert launch_coefficients(ctx, rbd0, GAITS, cmd_vels(B), params(0), ep) == plain
    ctx.close()


def test_setting_contract():
    ctx = context()
    rbd0 = start_states(ctx, B, seed=100)
    full = episode_maps(rbd0)
    one = M.zero_maps(B)
    one[0] = full[0]
    other = episode_maps(rbd0, rise=(-0.04, 0.05, 0.01, 0.0, -0.01, 0.02))
    other[3] = full[3]                                            # instance 3 keeps its map
    part = (hb.HbTerrain * 2)(full[1], full[2])
    padded = M.zero_maps(B)
    padded[0], padded[1] = full[1], full[2]
    # the permutation check gives each robot its own map: maps follow the robots' start positions, so permuting states and maps together
    # is the permuted episode
    assert_setting_episodes(_Ctx(ctx), "height_maps", rbd0, params(10), full, one, other, 3, part, padded)
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_rejected_settings(estimated):
    ctx = context()
    rbd0 = start_states(ctx, B, seed=101)
    ep = est_params(seed=13) if estimated else None
    bad = []
    for field, value in [("nx", 1), ("ny", 65), ("spacing", 0.0), ("spacing", float("nan"))]:
        r = M.zero_maps(1); setattr(r[0], field, value); bad.append(r)
    two = M.zero_maps(2)
    two[1].height[1][1] = float("inf")                        # a bad record after a good one
    assert_rejected_settings(_Ctx(ctx), "height_maps",
                             lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 100, params(5), 5, ep, hb.estimation_states(B, 50) if estimated else None),
                             episode_maps(rbd0), bad + [two], M.zero_maps(ctx.max_batch + 1))
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_snapshots_with_maps_continue_exactly(estimated):
    """Saved with goals captured on maps and restored in a fresh context with the same maps and goals: one call. Maps are not episode state:
    the row size is unchanged."""
    n1, n2 = 115, 85
    ctx = context()
    rbd0 = start_states(ctx, B, seed=102)
    vels = cmd_vels(B)
    ep = est_params(seed=14) if estimated else None
    fresh = lambda: hb.estimation_states(B, 40) if estimated else None
    maps, goals = episode_maps(rbd0), random_goals(rbd0, B, 102)
    plain_bytes = ctx.episode_state_bytes
    ctx.set_height_maps(maps)
    assert ctx.episode_state_bytes == plain_bytes
    ctx.set_goals(goals)
    one = device(ctx, rbd0, GAITS, vels, n1 + n2, params(5), 5, ep, fresh())
    first = device(ctx, rbd0, GAITS, vels, n1, params(5), 5, ep, fresh())
    snap = ctx.save_episodes(B, *first[:4], *(first[5:7] if estimated else ()))
    ctx.close()
    ctx2 = context()
    ctx2.set_goals(goals)
    ctx2.set_height_maps(maps)
    r = ctx2.restore_episodes(snap)
    if estimated:
        second = device(ctx2, r[0], GAITS, vels, n2, params(5), 5, ep, r[4], tick0=n1, act=r[1], estop=r[2], stats=r[3], est_stats=r[5])
    else:
        second = device(ctx2, r[0], GAITS, vels, n2, params(5), 5, tick0=n1, act=r[1], estop=r[2], stats=r[3])
    two = outputs(second)
    two[4] = np.concatenate([first[4].cpu().numpy(), two[4]], axis=1)
    if estimated:
        two[7] = np.concatenate([first[7].cpu().numpy(), two[7]], axis=1)
    assert_episode_equal(one, two)
    ctx2.close()
