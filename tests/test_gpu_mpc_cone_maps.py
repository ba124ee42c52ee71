"""MPC cone maps on the device (hb_mpc_set_cone_maps): solves with tilted friction cones against the oracle given the same frames and
stance heights (mpc_cone_ref.py), on both time grids and every contact class, with instances beyond the setting and MPC maps on some
instances, the line search's decisions included; unset, cleared, NULL, all-zero and plateau cone maps against no setting bit for bit with
the same launches, in the solve calls and both episode calls; episodes on cone maps against the loop of public calls bit for bit (both
WBCs, both grids, truth and estimator, with terrains, planner, estimator, MPC and WBC maps, pushes, variations, goals, teleop and
latencies alongside); the shared setting contract; snapshots resumed with the same maps; and a stance on a plane steeper than the cone,
where the tilt binds."""
import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as S
from episode_ref import (FRICTION, GAITS, GROUND, PUSH, array_of, assert_episode_equal, assert_null_settings, assert_rejected_settings,
                         assert_setting_episodes, cmd_vels, context, device, est_params, outputs, params, random_goals, start_states,
                         stepwise, use)
import mpc_cone_ref as CO
from mpc_map_ref import stance_heights_batch
from test_gpu_height_maps import episode_maps
from test_gpu_mpc_maps import GAIT_CYCLE, _assert_iteration, _solve_maps
from test_gpu_rollout_teleop import mixed
from test_mpc_cone_maps_host import plane
import height_map_ref as M

pytestmark = pytest.mark.gpu

B = 6


# ---------------------------------------------------------------------------------------------------------------- 1. against the oracle
def test_uniform_grid_solves_on_cone_maps_match_the_oracle():
    """16 instances, four per contact-class cycle: 12 on cone maps (stepped, sloped, random, plateau), 4 beyond the setting, and MPC maps
    on the first 6; two SQP iterations each, against the oracle given the restated frames and heights: accepted step, trial count,
    branch, merits, violations and trajectories at the parity tolerances of the solve; the tilted solves differ from the flat ones."""
    N, dt, n = 20, 0.01, 16
    ctx = hb.Context(horizon_N=N, dt=dt, max_batch=n, device=0)
    x0, x_ref, swing, mode = S.make_batch(n, N, dt, gaits=[GAIT_CYCLE[i % 4] for i in range(n)], seed=77)
    cones, heights = _solve_maps(12), _solve_maps(6)
    F = CO.cone_frames_batch(cones, swing, mode)
    H = stance_heights_batch(heights, swing, mode)
    tilted = [not np.array_equal(F[i], np.tile(CO.IDENTITY, (N + 1, 4, 1))) for i in range(n)]
    assert sum(tilted[:12]) >= 6 and not any(tilted[12:])          # plateaus and steps away from the feet stay flat
    xt, ut = ctx.mpc_cold_start(x0, mode)
    ctx.set_mpc_maps(heights)
    flat = ctx.mpc_solve(x0, x_ref, swing, mode, xt, ut)
    ctx.set_mpc_cone_maps(cones)
    a1 = ctx.mpc_solve(x0, x_ref, swing, mode, xt, ut)
    a2 = ctx.mpc_solve(x0, x_ref, swing, mode, a1[0], a1[1])
    branches = []
    for i in range(n):
        xo, uo = xt[i], ut[i]
        for dev in (a1, a2):
            xo, uo, io, tr = CO.mpc_iteration(N, dt, x0[i], x_ref[i], swing[i], mode[i], xo, uo, record=True, stance_h=H[i], frames=F[i])
            branches.append(_assert_iteration(io, tr, dev[2], i, xo, uo, dev[0][i], dev[1][i], 1e-8))
    moved = [not np.array_equal(a1[1][i], flat[1][i]) for i in range(n)]
    assert moved == tilted, (moved, tilted)
    print("accepted branches:", {b: branches.count(b) for b in set(branches)})
    ctx.close()


def test_event_grid_solves_on_cone_maps_match_the_oracle():
    """The same on per-instance event-node grids (the shipped sqp.dt and horizon), with MPC maps on half the instances."""
    from test_gpu_event_nodes import CAP, DT, T, _cases
    n = 8
    ctx = hb.Context(horizon_N=CAP, dt=DT, max_batch=n, device=0, time_horizon=T, event_nodes=True)
    x0, compacts, refs = _cases(n, 2)
    tk, nn, st = ctx.time_grid(np.full(n, 0.004), refs)
    xr, sw, md = ctx.reference_expand_grid(tk, refs)
    cones, heights = _solve_maps(6), _solve_maps(4)
    F = CO.cone_frames_batch(cones, sw, md)
    H = stance_heights_batch(heights, sw, md)
    xt, ut = ctx.mpc_cold_start(x0, md)
    ctx.set_mpc_maps(heights)
    ctx.set_mpc_cone_maps(cones)
    a1 = ctx.mpc_solve_grid(x0, tk, nn, xr, sw, md, xt, ut)
    a2 = ctx.mpc_solve_grid(x0, tk, nn, xr, sw, md, a1[0], a1[1])
    assert (a1[2]["status"] == 0).all() and (a2[2]["status"] == 0).all()
    for i in range(n):
        k = int(nn[i])
        dts = np.diff(tk[i, :k + 1])
        xo, uo = xt[i, :k + 1], ut[i, :k]
        for dev in (a1, a2):
            xo, uo, io, tr = CO.mpc_iteration(k, dts, x0[i], xr[i, :k + 1], sw[i, :k + 1], md[i, :k + 1], xo, uo, record=True,
                                              stance_h=H[i, :k + 1], frames=F[i, :k + 1])
            _assert_iteration(io, tr, dev[2], i, xo, uo, dev[0][i, :k + 1], dev[1][i, :k], 1e-7)
    ctx.close()


def test_tilt_binds_on_a_plane_steeper_than_the_cone():
    """test_mpc_cone_maps_host's binding case on the device: stance on a 45 degree plane, where the vertical forces of the warm start lie
    outside the tilted cone. The mapped solve's merit rises by what the restatement adds, and its first step turns the forces towards the
    normal as the restatement's does (Fx falls in sum and on most nodes), matching it to the solve's tolerances."""
    N, dt, n = 20, 0.01, 2
    ctx = hb.Context(horizon_N=N, dt=dt, max_batch=n, device=0)
    x0, x_ref, swing, mode = S.make_batch(n, N, dt, gait="stance", seed=12)
    xt, ut = ctx.mpc_cold_start(x0, mode)
    flat = ctx.mpc_solve(x0, x_ref, swing, mode, xt, ut)
    ctx.set_mpc_cone_maps(array_of([plane(1.0, 0.0)]))
    tilt = ctx.mpc_solve(x0, x_ref, swing, mode, xt, ut)
    F = CO.cone_frames(plane(1.0, 0.0), swing[0], mode[0])
    a = CO.mpc_iteration(N, dt, x0[0], x_ref[0], swing[0], mode[0], xt[0], ut[0])
    b = CO.mpc_iteration(N, dt, x0[0], x_ref[0], swing[0], mode[0], xt[0], ut[0], frames=F)
    db, dd = b[2]["merit0"] - a[2]["merit0"], tilt[2]["merit0"][0] - flat[2]["merit0"][0]
    assert db > 0.1 and abs(dd - db) < 1e-7 * max(1.0, abs(b[2]["merit0"]))
    dFx = tilt[1][0][:, 0:12:3] - flat[1][0][:, 0:12:3]
    assert dFx.sum() < 0 and (dFx < 0).mean() >= 0.75, dFx
    assert np.abs(tilt[1][0] - b[1]).max() < 1e-6 * max(1.0, np.abs(b[1]).max())
    assert np.array_equal(tilt[1][1], flat[1][1])                       # beyond the setting: the flat cone
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 2. null settings
def _null_maps(n):
    return (M.zero_maps(n), M.zero_maps(max(1, n // 2)), M.zero_maps(n, n=64, spacing=0.01), M.plateau(n, 0.12))


def test_null_settings_in_the_solve_calls():
    """Zero maps (as many as the instances, fewer, on a fine grid), plateau maps, and maps set then cleared (None, B == 0 with an array,
    NULL): the solve, grid solve and control step give the unset calls' outputs bit for bit, with the same launches."""
    N, dt, n = 20, 0.01, 8
    ctx = hb.Context(horizon_N=N, dt=dt, max_batch=n, device=0)
    x0, x_ref, swing, mode = S.make_batch(n, N, dt, gaits=[GAIT_CYCLE[i % 4] for i in range(n)], seed=79)
    rbd = S.consistent_rbd(x0, np.random.default_rng(0), 0.01)
    xt, ut = ctx.mpc_cold_start(x0, mode)
    tk = np.tile(dt * np.arange(N + 1), (n, 1)); nn = np.full(n, N, dtype=np.int32)

    def run():
        c0 = ctx.launch_count
        a = ctx.mpc_solve(x0, x_ref, swing, mode, xt, ut)
        g = ctx.mpc_solve_grid(x0, tk, nn, x_ref, swing, mode, xt, ut)
        s = ctx.control_step(0.002, x0, x_ref, swing, mode, rbd, xt, ut)
        blobs = [np.asarray(v).tobytes() for v in (a[0], a[1], g[0], g[1], *s[:2], *s[3:])] + [bytes(np.asarray(a[2]).tobytes()),
                                                                                           bytes(np.asarray(g[2]).tobytes()), bytes(np.asarray(s[2]).tobytes())]
        return blobs, ctx.launch_count - c0

    want = run()
    lib, h = ctx._lib, ctx._h
    names = ("zero", "zero_few", "zero_fine", "plateau")
    for setting in names + ("cleared", "cleared_array", "null"):
        ctx.set_mpc_cone_maps(_solve_maps(n))
        if setting in names:
            ctx.set_mpc_cone_maps(_null_maps(n)[names.index(setting)])
        elif setting == "cleared":
            ctx.set_mpc_cone_maps(None)
        elif setting == "cleared_array":
            assert lib.hb_mpc_set_cone_maps(h, 0, _solve_maps(2)) == 0
        else:
            assert lib.hb_mpc_set_cone_maps(h, 0, None) == 0
        assert run() == want, setting
    ctx.set_mpc_cone_maps(_solve_maps(n))
    got = run()
    assert got[1] == want[1] and got[0] != want[0]
    ctx.close()


class _Lib:
    """The library as the shared setting checks call it: they name a per-robot setter hb_rollout_set_<name>; the MPC cone maps' setter
    is hb_mpc_set_cone_maps (every MPC path reads it, not only the episodes)."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        return getattr(self._lib, "hb_mpc_set_cone_maps" if name == "hb_rollout_set_mpc_cone_maps" else name)


class _Ctx:
    def __init__(self, ctx):
        self._ctx, self._lib = ctx, _Lib(ctx._lib)

    def __getattr__(self, name):
        return getattr(self._ctx, name)


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
def test_null_settings_in_episodes(event_nodes, estimated):
    """Zero and plateau cone maps, and maps set then cleared, give the unset episode bit for bit in every output and recorded channel,
    with the same launches; episodes on cone maps move the robots."""
    from test_gpu_estimator_maps import _with_channels
    ctx = context(event_nodes)
    rbd0 = start_states(ctx, B, seed=211)
    prm = params(5)
    ep = est_params(seed=31) if estimated else None
    channels = []

    def run():
        est = hb.estimation_states(B, 50) if estimated else None
        out, ch = _with_channels(ctx, lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 150, prm, 5, ep, est), 30)()
        channels.append(ch)
        return out

    ref, _ = assert_null_settings(ctx, "mpc_cone_maps", run, _null_maps(B), episode_maps(rbd0))
    for ch in channels[1:]:
        assert ch.keys() == channels[0].keys()
        for k in ch:
            assert np.array_equal(ch[k], channels[0][k]), k
    ctx.set_mpc_cone_maps(episode_maps(rbd0))
    mapped = outputs(run())
    ctx.set_mpc_cone_maps(None)
    assert sum(not np.array_equal(a, b) for a, b in zip(mapped[4], outputs(ref)[4])) >= B - 2
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 3. the loop of public calls
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
@pytest.mark.parametrize("wbc", ["weighted", "hierarchical"])
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
def test_cone_mapped_episode_equals_the_stepwise_loop_bitwise(wbc, event_nodes, estimated):
    """The episode on MPC cone maps equals episode_ref.stepwise, whose solve calls read the same maps, bit for bit. On the weighted
    uniform grid with the terrains the maps describe, planner, MPC and WBC maps, pushes, variations, goals and teleop (and estimator maps
    through the estimator); on the hierarchical uniform grid with MPC latencies, goals and MPC maps; on event nodes with planner maps,
    two robots beyond the setting."""
    ctx = context(event_nodes)
    ctx.set_wbc_formulation(wbc)
    log_every, n_ticks = 10, 120
    rbd0 = start_states(ctx, B, seed=212)
    vels = cmd_vels(B)
    prm = params(log_every)
    maps = episode_maps(rbd0)
    kw, goals, teleop, planner_maps = {}, None, None, maps
    if wbc == "weighted" and not event_nodes:
        hm = np.ctypeslib.as_array(maps)["height"]
        ter = hb.make_terrains(B, hm[:, :40, :40] + GROUND, 0.02, rbd0[:, 3:5] - 0.4)
        kw = use(ctx, terrains=ter, plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION), pushes=hb.make_push_schedules(B, 0.15, 0.05, PUSH))
        goals, teleop = random_goals(rbd0, B, 212), mixed(B)
        ctx.set_mpc_maps(maps)
        ctx.set_wbc_maps(maps)
        if estimated:
            ctx.set_estimator_maps(maps)
    if wbc == "hierarchical" and not event_nodes:
        kw = use(ctx, mpc_latencies=[5, 0, 2, 3])
        goals, planner_maps = random_goals(rbd0, B, 213), None
        ctx.set_mpc_maps(maps)
    if event_nodes:
        maps = array_of(list(maps)[:B - 2])
    if goals is not None:
        ctx.set_goals(goals)
    if teleop is not None:
        ctx.set_teleop(teleop)
    ep, mk = (est_params(seed=2052), lambda: hb.estimation_states(B, 30)) if estimated else (None, lambda: None)
    ctx.set_height_maps(planner_maps)
    ctx.set_mpc_cone_maps(maps)
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, mk())
    loop = M.MapLoop(ctx, planner_maps if planner_maps is not None else [], prm.period, goals=goals, teleop=teleop)
    r = stepwise(loop, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, mk(), **kw)
    ctx.set_plan_targets(None)
    assert_episode_equal(d, r)
    ctx.set_mpc_cone_maps(None)
    u = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, mk())
    moved = [not np.array_equal(a, b) for a, b in zip(outputs(d)[4], outputs(u)[4])]
    assert sum(moved[:len(maps)]) >= len(maps) - 2 and not any(moved[len(maps):]), moved
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 4. the setting contract
def test_setting_contract():
    ctx = context()
    rbd0 = start_states(ctx, B, seed=213)
    full = episode_maps(rbd0)
    one = M.zero_maps(B)
    one[0] = full[0]
    other = episode_maps(rbd0, rise=(-0.04, 0.05, 0.01, 0.0, -0.01, 0.02))
    other[3] = full[3]                                            # instance 3 keeps its map
    part = array_of([full[1], full[2]])
    padded = M.zero_maps(B)
    padded[0], padded[1] = full[1], full[2]
    assert_setting_episodes(_Ctx(ctx), "mpc_cone_maps", rbd0, params(10), full, one, other, 3, part, padded)
    ctx.close()


def test_rejected_settings():
    ctx = context()
    rbd0 = start_states(ctx, B, seed=214)
    bad = []
    for field, value in [("nx", 1), ("ny", 65), ("spacing", 0.0), ("spacing", float("nan"))]:
        r = M.zero_maps(1); setattr(r[0], field, value); bad.append(r)
    two = M.zero_maps(2)
    two[1].height[1][1] = float("inf")                        # a bad record after a good one
    assert_rejected_settings(_Ctx(ctx), "mpc_cone_maps", lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 100, params(5), 5),
                             episode_maps(rbd0), bad + [two], M.zero_maps(ctx.max_batch + 1))
    ctx.close()


def test_snapshots_with_cone_maps_continue_exactly():
    """Saved mid-episode with MPC cone, MPC and planner maps set and restored in a fresh context given the same maps: one call. Maps are
    not episode state: the row size is unchanged."""
    n1, n2 = 115, 85
    ctx = context()
    rbd0 = start_states(ctx, B, seed=215)
    vels = cmd_vels(B)
    maps = episode_maps(rbd0)
    plain_bytes = ctx.episode_state_bytes
    use(ctx, mpc_cone_maps=maps, mpc_maps=maps, height_maps=maps)
    assert ctx.episode_state_bytes == plain_bytes
    one = device(ctx, rbd0, GAITS, vels, n1 + n2, params(5), 5)
    first = device(ctx, rbd0, GAITS, vels, n1, params(5), 5)
    snap = ctx.save_episodes(B, *first[:4])
    ctx.close()
    ctx2 = context()
    use(ctx2, mpc_cone_maps=maps, mpc_maps=maps, height_maps=maps)
    r = ctx2.restore_episodes(snap)
    second = device(ctx2, r[0], GAITS, vels, n2, params(5), 5, tick0=n1, act=r[1], estop=r[2], stats=r[3])
    two = outputs(second)
    two[4] = np.concatenate([first[4].cpu().numpy(), two[4]], axis=1)
    assert_episode_equal(one, two)
    ctx2.close()
