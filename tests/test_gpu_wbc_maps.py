"""WBC maps on the device (hb_wbc_set_maps): the assembly on maps against the restated QP (wbc_map_ref.py), its pyramid rows bit for bit,
on stepped maps with contacts on the ramp cell, sloped, random, plateau and off-grid maps, every mode and stance_mode, with unmapped
instances in the batch; the fused weighted solve and the hierarchical solve and tasks against the restated solves; the tilted rows held
by every mapped stance force where they bind (mu = 0.5 on a 30 degree plane); unset, cleared, NULL and all-zero maps against no setting
bit for bit with the same launches, in the WBC calls and both episode calls; mapped episodes against the loop of public calls bit for
bit (both WBCs, both grids, truth and estimator, with terrains, the other three maps, pushes, variations, per-robot controller settings
and latencies); the shared setting contract; and snapshots resumed with the same maps."""
import math

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as S
from episode_ref import (FRICTION, GAITS, GROUND, PUSH, array_of, assert_episode_equal, assert_null_settings, assert_rejected_settings,
                         assert_setting_episodes, cmd_vels, context, device, est_params, outputs, params, start_states, stepwise, use)
from test_gpu_height_maps import episode_maps
from test_gpu_hierarchical_loop import _check_levels
import height_map_ref as M
import wbc_map_ref as W

pytestmark = pytest.mark.gpu

B = 6
MU = 0.7                                         # task.info frictionCoefficient, the context's and the oracle's default


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


def _cases(n, seed):
    """test_gpu_parity's WBC cases: every mode, forces sharing the weight over the stance contacts, stance_mode on some double stances."""
    rng = np.random.default_rng(seed)
    mode = np.array([3, 2, 1, 0, 3, 3] * ((n + 5) // 6), dtype=np.int32)[:n]
    x = np.tile(S.INITIAL_STATE, (n, 1)) + rng.uniform(-.04, .04, (n, 22))
    u = np.zeros((n, 22))
    for i in range(n):
        fl = S.mode_flags(int(mode[i]))
        for c in range(4):
            if fl[c]:
                u[i, 3 * c + 2] = S.TOTAL_MASS * 9.81 / max(1, sum(fl))
        u[i, 12:] = rng.uniform(-.3, .3, 10)
    rbd = S.consistent_rbd(x, rng, 0.01)
    stance = ((np.arange(n) % 6) == 5).astype(np.uint8)
    return x, u, rbd, mode, stance


def _plane(a, b, n=10, spacing=0.2, origin=(-1.0, -1.0)):
    xs = origin[0] + spacing * np.arange(n); ys = origin[1] + spacing * np.arange(n)
    return hb.make_terrains(1, a * xs[None, :] + b * ys[:, None], spacing, origin)[0]


# the kinds of map, by instance modulo 5; "exact": the gradient is the same at every point of the contact's cell, so the restated rows are
# the device's bit for bit even where the two contact positions differ in their last bits
KINDS = ["step", "slope", "random", "plateau", "off_grid"]
EXACT = {"step", "slope", "plateau", "off_grid"}


def _maps(rbd, n, scale=1.0):
    """Maps for instances 0 .. n-1 of rbd: a step whose one-cell ramp is under contact i mod 4, a slope along x or y, random heights, a
    plateau and a random map the contacts are off on both axes. scale: of the steps', slopes' and random maps' heights."""
    out = []
    for i in range(n):
        k = KINDS[i % 5]
        p = W.contact_positions(rbd[i])
        # grids offset by a fraction of a cell from the contacts, so that no contact lies on a cell edge, where the gradient jumps
        if k == "step":
            sp = 0.02
            org = (p[0] - 0.5 + 0.37 * sp, p[1] - 0.5 + 0.37 * sp)
            j = math.floor((p[3 * (i % 4)] - org[0]) / sp)
            out.append(M.step_map(1, org[0] + (j + 0.5) * sp, scale * (0.03 + 0.01 * (i % 3)), spacing=sp, n=64, origin=org)[0])
        elif k == "slope":
            out.append(M.slope_map(1, scale * (0.1 + 0.15 * (i % 3)), axis=i % 2, spacing=0.05, n=40, origin=(p[0] - 0.987, p[1] - 0.981))[0])
        elif k == "random":
            out.append(M.random_maps(1, 300 + i, scale=scale * 0.05, spacing=0.05, n=40, origin=(p[0] - 0.987, p[1] - 0.981))[0])
        elif k == "plateau":
            out.append(M.plateau(1, 0.05 * (i % 3) - 0.05)[0])
        else:
            out.append(hb.make_terrains(1, np.random.default_rng(i).uniform(-0.1, 0.1, (6, 6)), 0.1, (p[0] + 3.0, p[1] - 4.0))[0])
    return array_of(out)


# ---------------------------------------------------------------------------------------------------------------- 1. against the restatement
def test_assembly_on_maps_matches_the_restated_qp():
    """hb_wbc_assemble_batch on 30 mapped instances and 6 beyond the setting: the pyramid rows of every stance contact equal the restated
    rows bit for bit (to 1e-12 on random maps, whose gradient varies inside a cell), every other entry the oracle's at
    test_wbc_device_assembly_vs_oracle's tolerances; the step maps put a contact on the ramp cell."""
    n, nm = 36, 30
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=n, device=0)
    x, u, rbd, mode, stance = _cases(n, 41)
    maps = _maps(rbd, nm)
    ctx.set_wbc_maps(maps)
    H, g, A, lb, ub, m = ctx.wbc_assemble(x, u, rbd, mode, stance)
    tilted, on_ramp = 0, 0
    for i in range(n):
        mi = maps[i] if i < nm else None
        Hi, gi, Ai, lbi, ubi = W.wbc_assemble(x[i], u[i], rbd[i], mode[i], bool(stance[i]), mi, MU)
        assert m[i] == Ai.shape[0]
        assert np.abs(H[i] - Hi).max() < 1e-9 * max(1.0, np.abs(Hi).max()) and np.abs(g[i] - gi).max() < 1e-9 * max(1.0, np.abs(gi).max())
        r0, st = W.pyramid_rows(int(mode[i]))
        rows = slice(r0, r0 + 5 * len(st))
        if mi is None or KINDS[i % 5] in EXACT:
            assert A[i, rows].tobytes() == Ai[rows].tobytes(), i
        elif st:
            assert np.abs(A[i, rows] - Ai[rows]).max() < 1e-12, i
        other = np.ones(Ai.shape[0], dtype=bool); other[rows] = False
        assert np.abs(A[i, :m[i]][other] - Ai[other]).max() < 1e-9 * max(1.0, np.abs(Ai).max())
        fin = np.abs(lbi) < 1e19
        assert np.abs(lb[i, :m[i]][fin] - lbi[fin]).max() < 1e-8 * max(1.0, np.abs(lbi[fin]).max()) and (lb[i, :m[i]][~fin] <= -1e19).all()
        assert np.abs(ub[i, :m[i]] - ubi).max() < 1e-8 * max(1.0, np.abs(ubi).max())
        fr = W.frames(mi, rbd[i])
        tilted += any(fr[c] is not None for c in st)
        if mi is not None and KINDS[i % 5] == "step":
            on_ramp += fr[i % 4] is not None and abs(fr[i % 4][0][0]) > 0.5
    assert tilted >= 12 and on_ramp == 6, (tilted, on_ramp)
    ctx.close()


def test_fused_solve_on_maps_matches_the_restated_solve():
    """hb_wbc_solve_batch on the maps above against hbo.qp_solve on the restated QP, at test_wbc_solve_vs_oracle's tolerances."""
    n, nm = 36, 30
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=n, device=0)
    x, u, rbd, mode, stance = _cases(n, 42)
    maps = _maps(rbd, nm)
    flat, _ = ctx.wbc_solve(x, u, rbd, mode, stance)
    ctx.set_wbc_maps(maps)
    sol, st = ctx.wbc_solve(x, u, rbd, mode, stance)
    assert (st == 0).all()
    for i in range(n):
        so, sto = W.wbc_solve(x[i], u[i], rbd[i], mode[i], bool(stance[i]), maps[i] if i < nm else None, MU)
        assert sto == 0
        assert _rel(sol[i, 28:], so[28:]) < 1e-4 and _rel(sol[i], so) < 1e-4, i
    assert all(np.array_equal(sol[i], flat[i]) for i in range(nm, n))
    ctx.close()


def test_hierarchical_solve_and_tasks_on_maps_match_the_restated_cascade():
    """hb_hierarchical_wbc_solve_batch and hb_hierarchical_wbc_tasks_batch on the maps against oracle/hoqp.py's cascade on the restated
    assembly: the task0 inequality rows to 1e-12, the fused solution against the composition and against the cascade's levels at
    test_fused_equals_composition_and_oracle's criteria. The maps' heights are halved: on the full random map of instance 2 the oracle's
    own cascade fails a level. The composition (hb_hoqp_solve_batch on the tasks) is compared where it solves: on one of these problems
    its level 2 stops at the iteration limit."""
    n, nm = 20, 16
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=n, device=0)
    x, u, rbd, mode, _ = _cases(n, 43)
    maps = _maps(rbd, nm, 0.5)
    ctx.set_wbc_maps(maps)
    sol, st = ctx.hierarchical_wbc_solve(x, u, rbd, mode)
    pbs = ctx.hierarchical_wbc_tasks(x, u, rbd, mode)
    xc, _, stc = ctx.hoqp_solve(pbs)
    assert (st == 0).all() and (stc == 0).sum() >= n - 2, (st, stc)
    for i in range(n):
        tasks = hb.hoqp_tasks(pbs[i])
        so, levels, otasks = W.hierarchical_wbc(x[i], u[i], rbd[i], mode[i], maps[i] if i < nm else None, MU)
        assert np.abs(tasks[0][2] - otasks[0].d).max() < 1e-12 and np.abs(tasks[0][3] - otasks[0].f).max() == 0.0, i
        if stc[i] == 0:
            _check_levels(sol[i], tasks, (xc[i], xc[i], xc[i]))
        _check_levels(sol[i], [(t.a, t.b, t.d, t.f) for t in otasks], (levels[0].solution(), levels[1].solution(), so))
    ctx.close()


def test_mapped_forces_hold_the_tilted_rows_where_they_bind():
    """mu = 0.5 on a 30 degree plane (tan 30 > 0.5): the flat weighted WBC's stance forces leave the tilted cone by more than 1 N (on all but
    two of the eight states), the mapped WBC's satisfy every tilted row to 1e-9 max(1, |F|) with a tangential row active. (The
    HierarchicalWbc holds its inequalities through level 0's slack, and on this case its level 1 fails in about half of the states, in
    oracle/hoqp.py's cascade as on the device: DESIGN, "WBC maps".)"""
    n = 8
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=n, device=0)
    s = ctx.wbc_settings(); s.friction_coefficient = 0.5; ctx.set_wbc_settings(s)
    x, u, rbd, mode, stance = _cases(n, 44)
    mode[:] = 3; stance[:] = 0
    g = math.tan(math.radians(30.0))
    maps = array_of([_plane(*ab) for ab in [(g, 0.0), (0.0, g), (-g, 0.0), (0.0, -g)] * 2])     # uphill along t1 or t2: the pyramid's axes
    flat, st0 = ctx.wbc_solve(x, u, rbd, mode, stance)
    ctx.set_wbc_maps(maps)
    mapped, st1 = ctx.wbc_solve(x, u, rbd, mode, stance)
    assert (st0 == 0).all() and (st1 == 0).all()
    left = 0
    for i in range(n):
        fr = W.frames(maps[i], rbd[i])
        worst_flat, tangential = -np.inf, -np.inf
        for c in range(4):
            P = W.pyramid(fr[c], 0.5)
            F0, F1 = flat[i, 16 + 3 * c:19 + 3 * c], mapped[i, 16 + 3 * c:19 + 3 * c]
            worst_flat = max(worst_flat, (P @ F0).max())
            assert (P @ F1 <= 1e-9 * max(1.0, np.abs(F1).max())).all(), (i, c, P @ F1)
            tangential = max(tangential, (P[1:] @ F1).max() / max(1.0, np.abs(F1).max()))
        assert tangential > -1e-6, (i, tangential)
        left += worst_flat > 1.0
    assert left >= n - 2, left
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 2. null settings
def _null_maps(n):
    return (M.zero_maps(n), M.zero_maps(max(1, n // 2)), M.zero_maps(n, n=64, spacing=0.01))


def test_null_settings_in_the_wbc_calls():
    """Zero maps (as many as the instances, fewer, on a fine grid), and maps set then cleared (None, B == 0 with an array, NULL): the weighted
    solve and assembly, the hierarchical solve and tasks, and the control step under both WBCs give the unset calls' outputs bit for bit,
    with the same launches; maps move them. Each run is on a fresh context (the control step keeps the WBC's previous solution)."""
    N, dt, n = 20, 0.01, 8
    x, u, rbd, mode, stance = _cases(n, 45)
    x0, x_ref, swing, md = S.make_batch(n, N, dt, gait="trot", seed=80)
    rbd0 = S.consistent_rbd(x0, np.random.default_rng(1), 0.01)
    ctx = hb.Context(horizon_N=N, dt=dt, max_batch=n, device=0)
    xt, ut = ctx.mpc_cold_start(x0, md)
    ctx.close()

    def run(setting=None):
        ctx = hb.Context(horizon_N=N, dt=dt, max_batch=n, device=0)
        if setting is not None:
            ctx.set_wbc_maps(_maps(rbd, n))
            lib, h = ctx._lib, ctx._h
            if setting.startswith("zero"):
                ctx.set_wbc_maps(_null_maps(n)[("zero", "zero_few", "zero_fine").index(setting)])
            elif setting == "cleared":
                ctx.set_wbc_maps(None)
            elif setting == "cleared_array":
                assert lib.hb_wbc_set_maps(h, 0, _maps(rbd, 2)) == 0
            elif setting == "null":
                assert lib.hb_wbc_set_maps(h, 0, None) == 0
            else:
                ctx.set_wbc_maps(array_of([_plane(0.3, -0.2)] * n))
        c0 = ctx.launch_count
        out = [*ctx.wbc_solve(x, u, rbd, mode, stance), *ctx.hierarchical_wbc_solve(x, u, rbd, mode)]
        H, g, A, lb, ub, m = ctx.wbc_assemble(x, u, rbd, mode, stance)
        out += [H, g, m] + [a[i, :m[i]] for i in range(n) for a in (A, lb, ub)]                         # the rows written
        out += [a for pb in ctx.hierarchical_wbc_tasks(x, u, rbd, mode) for t in hb.hoqp_tasks(pb) for a in t]    # the rows written
        for form in ("weighted", "hierarchical"):
            ctx.set_wbc_formulation(form)
            s = ctx.control_step(0.002, x0, x_ref, swing, md, rbd0, xt, ut)
            out += [s[0], s[1], np.asarray(s[2]), *s[3:]]
        launches = ctx.launch_count - c0
        ctx.close()
        return [np.asarray(v).tobytes() for v in out], launches

    want = run()
    for setting in ("zero", "zero_few", "zero_fine", "cleared", "cleared_array", "null"):
        assert run(setting) == want, setting
    got = run("plane")
    assert got[1] == want[1] and got[0] != want[0]


class _Lib:
    """The library as the shared setting checks call it: they name a per-robot setter hb_rollout_set_<name>; the WBC maps' setter is
    hb_wbc_set_maps (every WBC path reads it, not only the episodes)."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        return getattr(self._lib, "hb_wbc_set_maps" if name == "hb_rollout_set_wbc_maps" else name)


class _Ctx:
    def __init__(self, ctx):
        self._ctx, self._lib = ctx, _Lib(ctx._lib)

    def __getattr__(self, name):
        return getattr(self._ctx, name)


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
def test_null_settings_in_episodes(event_nodes, estimated):
    """Zero maps, and maps set then cleared, give the unset episode bit for bit in every output and recorded channel, with the same
    launches; mapped episodes move the robots."""
    from test_gpu_estimator_maps import _with_channels
    ctx = context(event_nodes)
    rbd0 = start_states(ctx, B, seed=221)
    prm = params(5)
    ep = est_params(seed=41) if estimated else None
    channels = []

    def run():
        est = hb.estimation_states(B, 50) if estimated else None
        out, ch = _with_channels(ctx, lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 150, prm, 5, ep, est), 30)()
        channels.append(ch)
        return out

    ref, _ = assert_null_settings(ctx, "wbc_maps", run, _null_maps(B), episode_maps(rbd0))
    for ch in channels[1:]:
        assert ch.keys() == channels[0].keys()
        for k in ch:
            assert np.array_equal(ch[k], channels[0][k]), k
    ctx.set_wbc_maps(episode_maps(rbd0))
    mapped = outputs(run())
    ctx.set_wbc_maps(None)
    assert sum(not np.array_equal(a, b) for a, b in zip(mapped[4], outputs(ref)[4])) >= B - 2
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 3. the loop of public calls
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
@pytest.mark.parametrize("wbc", ["weighted", "hierarchical"])
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
def test_mapped_episode_equals_the_stepwise_loop_bitwise(wbc, event_nodes, estimated):
    """The episode on WBC maps equals episode_ref.stepwise, whose WBC calls read the same maps, bit for bit. On the weighted uniform grid
    with the terrains the maps describe, planner and MPC maps (and estimator maps through the estimator), pushes, variations and per-robot
    controller settings at mu = 0.5 (records equal to the context's settings, which the loop's calls run); on the hierarchical uniform
    grid with MPC latencies; on event nodes with planner maps, two robots beyond the setting."""
    ctx = context(event_nodes)
    ctx.set_wbc_formulation(wbc)
    log_every, n_ticks = 10, 120
    rbd0 = start_states(ctx, B, seed=222)
    vels = cmd_vels(B)
    prm = params(log_every)
    maps = episode_maps(rbd0)
    kw, planner_maps = {}, maps
    if wbc == "weighted" and not event_nodes:
        hm = np.ctypeslib.as_array(maps)["height"]
        ter = hb.make_terrains(B, hm[:, :40, :40] + GROUND, 0.02, rbd0[:, 3:5] - 0.4)
        kw = use(ctx, terrains=ter, plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION), pushes=hb.make_push_schedules(B, 0.15, 0.05, PUSH))
        s = ctx.wbc_settings(); s.friction_coefficient = 0.5; ctx.set_wbc_settings(s)
        ctx.set_controller_settings(hb.make_controller_settings(B, wbc=ctx.wbc_settings(), gains=prm.gains))
        ctx.set_mpc_maps(maps)
        if estimated:
            ctx.set_estimator_maps(maps)
    if wbc == "hierarchical" and not event_nodes:
        kw = use(ctx, mpc_latencies=[5, 0, 2, 3])
        planner_maps = None
    if event_nodes:
        maps = array_of(list(maps)[:B - 2])
    ep, mk = (est_params(seed=2062), lambda: hb.estimation_states(B, 30)) if estimated else (None, lambda: None)
    ctx.set_height_maps(planner_maps)
    ctx.set_wbc_maps(maps)
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, mk())
    loop = M.MapLoop(ctx, planner_maps if planner_maps is not None else [], prm.period)
    r = stepwise(loop, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, mk(), **kw)
    ctx.set_plan_targets(None)
    assert_episode_equal(d, r)
    ctx.set_wbc_maps(None)
    u = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, mk())
    moved = [not np.array_equal(a, b) for a, b in zip(outputs(d)[4], outputs(u)[4])]
    assert sum(moved[:len(maps)]) >= len(maps) - 2 and not any(moved[len(maps):]), moved
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 4. the setting contract
def test_setting_contract():
    ctx = context()
    rbd0 = start_states(ctx, B, seed=223)
    full = episode_maps(rbd0)
    one = M.zero_maps(B)
    one[0] = full[0]
    other = episode_maps(rbd0, rise=(-0.04, 0.05, 0.01, 0.0, -0.01, 0.02))
    other[3] = full[3]                                            # instance 3 keeps its map
    part = array_of([full[1], full[2]])
    padded = M.zero_maps(B)
    padded[0], padded[1] = full[1], full[2]
    assert_setting_episodes(_Ctx(ctx), "wbc_maps", rbd0, params(10), full, one, other, 3, part, padded)
    ctx.close()


def test_rejected_settings():
    ctx = context()
    rbd0 = start_states(ctx, B, seed=224)
    bad = []
    for field, value in [("nx", 1), ("ny", 65), ("spacing", 0.0), ("spacing", float("nan"))]:
        r = M.zero_maps(1); setattr(r[0], field, value); bad.append(r)
    two = M.zero_maps(2)
    two[1].height[1][1] = float("inf")                        # a bad record after a good one
    assert_rejected_settings(_Ctx(ctx), "wbc_maps", lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 100, params(5), 5),
                             episode_maps(rbd0), bad + [two], M.zero_maps(ctx.max_batch + 1))
    ctx.close()


def test_snapshots_with_maps_continue_exactly():
    """Saved mid-episode with WBC and planner maps set and restored in a fresh context given the same maps: one call. Maps are not episode
    state: the row size is unchanged."""
    n1, n2 = 115, 85
    ctx = context()
    rbd0 = start_states(ctx, B, seed=225)
    vels = cmd_vels(B)
    maps = episode_maps(rbd0)
    plain_bytes = ctx.episode_state_bytes
    use(ctx, wbc_maps=maps, height_maps=maps)
    assert ctx.episode_state_bytes == plain_bytes
    one = device(ctx, rbd0, GAITS, vels, n1 + n2, params(5), 5)
    first = device(ctx, rbd0, GAITS, vels, n1, params(5), 5)
    snap = ctx.save_episodes(B, *first[:4])
    ctx.close()
    ctx2 = context()
    use(ctx2, wbc_maps=maps, height_maps=maps)
    r = ctx2.restore_episodes(snap)
    second = device(ctx2, r[0], GAITS, vels, n2, params(5), 5, tick0=n1, act=r[1], estop=r[2], stats=r[3])
    two = outputs(second)
    two[4] = np.concatenate([first[4].cpu().numpy(), two[4]], axis=1)
    assert_episode_equal(one, two)
    ctx2.close()
