"""Link variations in the plant and the episodes (hb_rollout_set_link_variations, hb_sim_step_links): the varied plant step against the
numpy plant on link_ref's varied terms, exact identities (default records, robots without one), the base body scaled against the same
mass as a payload, momentum, energy and static load on varied bodies; the varied episode bit for bit against the loop of public calls
(episode_ref.stepwise on link_ref.LinkLoop) with every other setting alongside, the setting's contract, launches and snapshots."""
import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from episode_ref import (FRICTION, GAITS, PUSH, array_of, assert_episode_equal, assert_null_settings, assert_rejected_settings,
                         assert_setting_episodes, cmd_vels, context, device, est_params, launch_coefficients, outputs, params, plant_numpy,
                         random_goals, small_terrains, start_states, stepwise, use)
from bridge_ref import plant_bridged
from link_ref import LinkLoop, LinkOracle, body_motion, bodies, padded
from teleop_ref import TeleopLoop
from oracle import refs

pytestmark = pytest.mark.gpu

B = 6
nan, inf = float("nan"), float("inf")


def _same(a, b):
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.uint64), np.asarray(b, dtype=np.float64).view(np.uint64))


def _one_body(n, b, rng):
    """n records, each varying body b alone in mass, CoM and inertia."""
    ms, js = np.ones((n, 11)), np.ones((n, 11)); cs = np.zeros((n, 11, 3))
    ms[:, b] = rng.uniform(0.5, 2.0, n); js[:, b] = rng.uniform(0.5, 2.0, n); cs[:, b] = rng.uniform(-0.02, 0.02, (n, 3))
    return hb.make_link_variations(n, ms, cs, js)


def _all_bodies(n, rng):
    return hb.make_link_variations(n, rng.uniform(0.5, 2.0, (n, 11)), rng.uniform(-0.02, 0.02, (n, 11, 3)), rng.uniform(0.5, 2.0, (n, 11)))


def _step_inputs(n, seed):
    rng = np.random.default_rng(seed)
    rbd = sc.consistent_rbd(sc.random_initial_states(n, seed=seed + 40), rng, 0.02)
    rbd[:, 5] = rng.uniform(0.60, 0.64, n)               # some feet in the ground, some above it
    rbd[:, 16:19] = rng.uniform(-1.5, 1.5, (n, 3)); rbd[:, 22:32] = rng.uniform(-2, 2, (n, 10))
    return rbd, rng.uniform(-15, 15, (n, 10)), rng


def _close(got, want, tol=1e-9):
    return np.abs(got - want).max() < tol * max(1.0, np.abs(want).max())


# ---------------------------------------------------------------------------------------------------------------- 1. the plant step
@pytest.mark.parametrize("which", ["base", "hip", "thigh", "shank", "foot", "right_leg", "all"])
def test_varied_plant_step_matches_numpy(gpu_ctx, oracle, which):
    n = 6
    rbd, tau, rng = _step_inputs(n, 3 + len(which))
    L = _all_bodies(n, rng) if which == "all" else _one_body(n, {"base": 0, "hip": 1, "thigh": 3, "shank": 4, "foot": 5, "right_leg": 8}[which], rng)
    prm = hb.default_sim_params(); prm.substeps = 3
    nxt, cf, _ = gpu_ctx.sim_step(rbd, tau, prm, links=L)
    for i in range(n):
        ref, F, _ = plant_numpy(LinkOracle(oracle, L[i]), rbd[i], tau[i], prm)
        assert _close(nxt[i], ref), (i, np.abs(nxt[i] - ref).max())
        assert _close(cf[i], F, 1e-7), i


def test_varied_plant_step_with_every_other_plant_input(gpu_ctx, oracle):
    """Link variations together with a payload (on top), a wrench, a terrain and, on half the robots, a motor bridge."""
    n = 6
    rbd, tau, rng = _step_inputs(n, 11)
    L = _all_bodies(n, rng)
    V = hb.make_plant_variations(n, 2.0, [0.02, -0.01, 0.08], np.diag([0.01, 0.012, 0.008]), friction_scale=0.7, motor_strength=0.9)
    W = np.c_[rng.uniform(-40, 40, (n, 3)), rng.uniform(-5, 5, (n, 3))]
    T = hb.make_terrains(n, 0.6 + rng.uniform(0.0, 0.03, (n, 4, 4)), 0.1, rbd[:, 3:5] - 0.15)
    prm = hb.default_sim_params(); prm.substeps = 2
    nxt, cf, _ = gpu_ctx.sim_step(rbd, tau, prm, wrench=W, variation=V, terrain=T, links=L)
    for i in range(n):
        ref, F, _ = plant_numpy(LinkOracle(oracle, L[i]), rbd[i], tau[i], prm, W[i], V[i], T[i])
        assert _close(nxt[i], ref), (i, np.abs(nxt[i] - ref).max())
    br = hb.make_motor_bridges(n)
    jcmd = np.stack([rbd[:, 6:16], np.zeros((n, 10)), np.full((n, 10), 30.0), np.full((n, 10), 1.0), rng.uniform(-5, 5, (n, 10))], axis=2)
    mcmd = hb.bridge_encode(br, jcmd)
    lim = np.full(10, 40.0)
    nxt, _, _, applied = gpu_ctx.sim_step(rbd, mcmd, prm, variation=V, bridge=br, limits=lim, links=L)
    for i in range(n):
        ref, _, _, ap = plant_bridged(LinkOracle(oracle, L[i]), rbd[i], prm, br[i], mcmd[i], lim, V[i])
        assert _close(nxt[i], ref) and _close(applied[i], ap), i


# ---------------------------------------------------------------------------------------------------------------- 2. exact identities
def test_default_records_and_robots_without_one_are_the_unvaried_step_bitwise(gpu_ctx):
    n = 8
    rbd, tau, rng = _step_inputs(n, 21)
    prm = hb.default_sim_params()
    V = hb.make_plant_variations(n, 1.5, [0.0, 0.0, 0.05], np.diag([0.01, 0.01, 0.01]))
    plain = gpu_ctx.sim_step(rbd, tau, prm, variation=V)
    for x, y in zip(plain, gpu_ctx.sim_step(rbd, tau, prm, variation=V, links=hb.make_link_variations(n))):
        assert _same(x, y)
    L = _all_bodies(n, rng)
    for i in (0, 3, 4, 7):
        L[i] = hb.default_link_variation()
    mixed = gpu_ctx.sim_step(rbd, tau, prm, variation=V, links=L)
    for i in range(n):
        same = all(_same(x[i], y[i]) for x, y in zip(plain, mixed))
        assert same == (i in (0, 3, 4, 7)), i


def test_heavier_base_equals_the_same_mass_as_a_payload(gpu_ctx):
    """Body 0 with mass and inertia scale s against the nominal base carrying a payload of (s - 1) m0 at c0 with inertia (s - 1) I0: two
    paths through different code, equal to 1e-12 relative."""
    n = 6
    rbd, tau, rng = _step_inputs(n, 31)
    s = np.array([1.25, 1.5, 2.0, 1.1, 3.0, 1.75])
    ms = np.ones((n, 11)); ms[:, 0] = s
    L = hb.make_link_variations(n, ms, 0.0, ms)
    m0, c0, I0 = bodies()
    V = hb.make_plant_variations(n, (s - 1) * m0[0], c0[0], (s - 1)[:, None, None] * I0[0])
    prm = hb.default_sim_params()
    a, _, _ = gpu_ctx.sim_step(rbd, tau, prm, links=L)
    b, _, _ = gpu_ctx.sim_step(rbd, tau, prm, variation=V)
    assert np.abs(a - b).max() < 1e-12 * np.abs(b).max()
    assert not np.array_equal(a, gpu_ctx.sim_step(rbd, tau, prm)[0])


# ---------------------------------------------------------------------------------------------------------------- 3. physics
def _free_flight(substeps):
    prm = hb.default_sim_params()
    prm.ground_height = -100.0; prm.joint_armature = 0.0; prm.joint_damping = 0.0; prm.substeps = substeps
    return prm


def _qv(r):
    return (np.concatenate([r[3:6], r[0:3], r[6:16]]),
            np.concatenate([r[19:22], refs.euler_rates_from_global(r[0:3], r[16:19]), r[22:32]]))


def test_free_flight_momentum_changes_at_the_varied_weight(gpu_ctx):
    """Free flight with zero torques, no armature or damping: over 50 ticks the linear momentum sum_b m'_b v_b changes by m'_total g T. The
    O(h) error of semi-implicit Euler must shrink about 4x from 4 to 16 substeps and its Richardson extrapolation be below 2e-3 N s."""
    n = 3
    rng = np.random.default_rng(41)
    rbd = sc.consistent_rbd(sc.random_initial_states(n, seed=41))
    rbd[:, 16:19] = rng.uniform(-1, 1, (n, 3)); rbd[:, 22:] = rng.uniform(-1, 1, (n, 10))
    L = _all_bodies(n, rng)
    mt = np.array([bodies(L[i])[0].sum() for i in range(n)])

    def momentum(r):
        out = []
        for i in range(n):
            q, v = _qv(r[i])
            m = bodies(L[i])[0]
            out.append((m[:, None] * body_motion(q, v, bodies(L[i]))[1]).sum(axis=0))
        return np.array(out)

    err = {}
    for sub in (4, 16):
        prm = _free_flight(sub)
        r, p0 = rbd.copy(), momentum(rbd)
        for _ in range(50):
            r, _, fl = gpu_ctx.sim_step(r, np.zeros((n, 10)), prm, links=L)
            assert (fl == 0).all()
        err[sub] = momentum(r) - p0 - mt[:, None] * np.array([0.0, 0.0, -9.81]) * 50 * prm.dt
    assert np.abs(err[16]).max() < 0.3 * np.abs(err[4]).max() + 1e-6, err
    assert np.abs((4 * err[16] - err[4]) / 3).max() < 2e-3, err


def test_free_flight_energy_drift_is_no_worse_than_nominal(gpu_ctx, oracle):
    """Free flight conserves 1/2 v'M'v + sum_b m'_b g z_b: the drift of the varied plant shrinks with h as the nominal plant's does, and at
    each substep count stays within 3x of the nominal plant's from the same states."""
    n = 3
    rng = np.random.default_rng(43)
    rbd = sc.consistent_rbd(sc.random_initial_states(n, seed=43))
    rbd[:, 16:19] = rng.uniform(-1, 1, (n, 3)); rbd[:, 22:] = rng.uniform(-1, 1, (n, 10))
    L = _all_bodies(n, rng)

    def energy(r, links):
        E = np.zeros(n)
        for i in range(n):
            q, v = _qv(r[i])
            rec = None if links is None else links[i]
            M = LinkOracle(oracle, rec).rbd(q, v)["M"]
            body = bodies(rec)
            E[i] = 0.5 * v @ M @ v + 9.81 * (body[0] * body_motion(q, v, body)[0][:, 2]).sum()
        return E

    drift = {}
    for links in (None, L):
        for sub in (4, 16):
            prm = _free_flight(sub)
            r = rbd.copy()
            for _ in range(50):
                r, _, _ = gpu_ctx.sim_step(r, np.zeros((n, 10)), prm, links=links)
            drift[links is None, sub] = np.abs(energy(r, links) - energy(rbd, links)).max()
    for sub in (4, 16):
        assert drift[False, sub] <= 3 * drift[True, sub] + 1e-9, drift
    assert drift[False, 16] < 0.35 * drift[False, 4] + 1e-9, drift


def test_standing_robot_carries_its_varied_weight(gpu_ctx):
    """A robot held by a stiff joint PD law on the ground settles to summed normal forces of m'_total g within 2 %."""
    n = 4
    rbd = start_states(gpu_ctx, n, seed=7)
    q0 = rbd[:, 6:16].copy()
    s = np.ones((n, 11)); s[1, 0] = 0.7; s[2, 1:] = 1.5; s[3, [3, 8]] = 2.0
    L = hb.make_link_variations(n, s, [[0.0, 0.0, 0.0]] * 5 + [[0.0, 0.0, -0.01]] * 6, s)
    prm = hb.default_sim_params(); prm.ground_height = 0.02
    r = rbd.copy()
    for _ in range(1000):
        r, cf, _ = gpu_ctx.sim_step(r, 400.0 * (q0 - r[:, 6:16]) - 10.0 * r[:, 22:32], prm, links=L)
    want = np.array([bodies(L[i])[0].sum() for i in range(n)]) * 9.81
    assert np.abs(cf[:, 2::3].sum(axis=1) / want - 1).max() < 0.02


# ---------------------------------------------------------------------------------------------------------------- 4. episodes
def _records(n, seed=5):
    """Leg links heavier and lighter, a lower shank CoM, a lighter base, one default record."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        s, c = np.ones(11), np.zeros((11, 3))
        if k % 5 == 0:
            s[1:] = 1.3
        elif k % 5 == 1:
            s[[4, 9]] = 1.2; c[[4, 9], 2] = -0.02
        elif k % 5 == 2:
            s[0] = 0.85
        elif k % 5 == 3:
            s[:] = rng.uniform(0.8, 1.2, 11); c[:] = rng.uniform(-0.01, 0.01, (11, 3))
        out.append(hb.make_link_variations(1, s, c, s)[0])
    return array_of(out)


@pytest.mark.parametrize("wbc, event_nodes, estimated", [("weighted", False, False), ("hierarchical", True, True), ("weighted", True, True),
                                                         ("hierarchical", False, False)],
                         ids=["weighted-uniform-truth", "hierarchical-event_nodes-estimator", "weighted-event_nodes-estimator",
                              "hierarchical-uniform-truth"])
def test_varied_episode_equals_the_stepwise_loop_bitwise(wbc, event_nodes, estimated):
    """Link variations on all robots but the last, with pushes, plant variations, a terrain, goals, MPC latencies, hardware and controller
    settings, motor bridges and teleop set alongside."""
    ctx = context(event_nodes)
    ctx.set_wbc_formulation(wbc)
    n_ticks, log_every = 80, 10
    rbd0 = start_states(ctx, B, seed=301)
    vels = cmd_vels(B)
    prm = params(log_every)
    links = _records(B - 1)
    kw = use(ctx, plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION, motor_strength=0.95),
             pushes=hb.make_push_schedules(B, 0.05, 0.05, PUSH), terrains=small_terrains(), mpc_latencies=[0, 2, 5, 1, 0, 3],
             hardware=hb.make_hardware_settings(B, actuation_delay=np.linspace(0.0, 0.012, B), encoder_offset=np.linspace(-0.01, 0.01, 10)))
    bridges = hb.make_motor_bridges(3)
    goals, teleop = random_goals(rbd0, B, 301), hb.make_teleop_settings(4, period_ticks=5 * prm.mpc_every)
    ctx.set_motor_bridge(bridges); ctx.set_goals(goals); ctx.set_teleop(teleop); ctx.set_link_variations(links)
    g = hb.default_pd_gains(); g.kp_big_stance = 45.0
    ctx.set_controller_settings(hb.make_controller_settings(B, wbc=ctx.wbc_settings(), gains=g))
    ep = est_params(seed=3011) if estimated else None
    fresh = (lambda: hb.estimation_states(B, 70)) if estimated else (lambda: None)
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, fresh())
    prm.gains = g
    loop = LinkLoop(TeleopLoop(ctx, teleop, prm.period, goals), links, bridges, prm.torque_limit)
    r = stepwise(loop, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, fresh(), **kw)
    ctx.set_plan_targets(None)
    assert_episode_equal(d, r)
    ctx.set_link_variations(None)
    u = outputs(device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, fresh()))
    moved = [not np.array_equal(a, b) for a, b in zip(outputs(d)[0], u[0])]
    assert moved == [True, True, True, True, False, False], moved      # robot 4 has the default record, robot 5 none
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_default_records_are_the_unset_episode_bitwise(estimated):
    ctx = context()
    rbd0 = start_states(ctx, B, seed=302)
    ep = est_params(seed=21) if estimated else None
    assert_null_settings(ctx, "link_variations", lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 60, params(5), 5, ep,
                                                                hb.estimation_states(B, 50) if estimated else None),
                         [hb.make_link_variations(B), hb.make_link_variations(3)], _records(B))
    ctx.close()


def test_setting_contract():
    ctx = context()
    rbd0 = start_states(ctx, B, seed=303)
    r = list(_records(5))
    full = array_of([r[0], r[1], r[2], r[3], r[0], r[1]])
    one = array_of([r[0]])
    other = array_of([r[3], r[2], r[1], r[3], r[0], r[1]])       # instance 3 keeps its record
    part = array_of([r[2], r[0]])
    assert_setting_episodes(ctx, "link_variations", rbd0, params(10), full, one, other, 3, part, padded(part, B))
    ctx.close()


def _bad():
    out = []
    for field, b, v in [("mass_scale", 3, 0.0), ("mass_scale", 0, -1.0), ("mass_scale", 10, nan), ("inertia_scale", 2, 0.0),
                        ("inertia_scale", 7, inf), ("com_shift", 4, nan)]:
        recs = hb.make_link_variations(2)
        if field == "com_shift":
            recs[1].com_shift[b][2] = v
        else:
            getattr(recs[1], field)[b] = v
        out.append(recs)
    return out


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_rejected_settings(estimated):
    ctx = context()
    rbd0 = start_states(ctx, B, seed=304)
    ep = est_params(seed=11) if estimated else None
    assert_rejected_settings(ctx, "link_variations",
                             lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 40, params(5), 5, ep, hb.estimation_states(B, 50) if estimated else None),
                             _records(B), _bad(), hb.make_link_variations(ctx.max_batch + 1))
    rbd = np.zeros((2, 32))
    for bad in _bad():                                  # the host plant step validates its records as the setter does
        with pytest.raises(hb.HunterB200Error):
            ctx.sim_step(rbd, np.zeros((2, 10)), links=bad)
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_link_variations_add_no_launch(estimated):
    ctx = context()
    rbd0 = start_states(ctx, B, seed=305)
    vels = cmd_vels(B)
    prm = params(0)
    ep = est_params(seed=5) if estimated else None
    plain = launch_coefficients(ctx, rbd0, GAITS, vels, prm, ep)
    ctx.set_link_variations(_records(B))
    assert launch_coefficients(ctx, rbd0, GAITS, vels, prm, ep) == plain
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_snapshot_resumes_bitwise(estimated):
    """The setting holds no state: a save after 50 ticks restored into a fresh context with the same setting resumes as one call."""
    vels = cmd_vels(B)
    prm = params(1)
    ep = est_params(seed=12) if estimated else None
    fresh = (lambda: hb.estimation_states(B, 50)) if estimated else (lambda: None)

    def configured():
        c = context()
        c.set_link_variations(_records(B))
        return c
    ctx = configured()
    rbd0 = start_states(ctx, B, seed=306)
    one = device(ctx, rbd0, GAITS, vels, 100, prm, 1, ep, fresh())
    first = device(ctx, rbd0, GAITS, vels, 50, prm, 1, ep, fresh())
    snap = ctx.save_episodes(B, *first[:4], *(first[5:7] if estimated else ()))
    ctx.close()
    ctx2 = configured()
    r = ctx2.restore_episodes(snap)
    if estimated:
        second = device(ctx2, r[0], GAITS, vels, 50, prm, 1, ep, r[4], tick0=50, act=r[1], estop=r[2], stats=r[3], est_stats=r[5])
    else:
        second = device(ctx2, r[0], GAITS, vels, 50, prm, 1, tick0=50, act=r[1], estop=r[2], stats=r[3])
    two = outputs(second)
    two[4] = np.concatenate([first[4].cpu().numpy(), two[4]], axis=1)
    if estimated:
        two[7] = np.concatenate([first[7].cpu().numpy(), two[7]], axis=1)
    assert_episode_equal(one, two)
    ctx2.close()
