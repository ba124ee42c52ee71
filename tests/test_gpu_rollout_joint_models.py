"""Joint models in the plant and the episodes (hb_rollout_set_joint_models, hb_sim_step_joints): the plant step against the numpy plant
with joint_model_ref's terms, inside, at and beyond each bound, with every other plant input; the exact identities (no record, disabled
records, hb_sim_step_links against hb_sim_step_joints); the stop's settled penetration, the friction's dissipation and a stop that never
pulls; the episode bit for bit against the loop of public calls (episode_ref.stepwise on joint_model_ref.JointLoop) with every other
setting alongside; the setting's contract, launches and the stability rule."""
import ctypes as C

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import api
from hunter_bipedal_control_b200 import scenarios as sc
from episode_ref import (FRICTION, GAITS, PUSH, array_of, assert_episode_equal, assert_null_settings, assert_rejected_settings,
                         assert_setting_episodes, cmd_vels, context, device, est_params, launch_coefficients, outputs, params, plant_numpy,
                         random_goals, small_terrains, start_states, stepwise, use)
from bridge_ref import plant_bridged
from link_ref import LinkOracle, body_motion, bodies
from joint_model_ref import JointLoop, JointOracle, bad_records, disabled, padded
from teleop_ref import TeleopLoop
from oracle import refs

pytestmark = pytest.mark.gpu

B = 6
nan, inf = float("nan"), float("inf")


def _same(a, b):
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.uint64), np.asarray(b, dtype=np.float64).view(np.uint64))


def _close(got, want, tol=1e-9):
    return np.abs(got - want).max() < tol * max(1.0, np.abs(want).max())


def _qv(r):
    return (np.concatenate([r[3:6], r[0:3], r[6:16]]),
            np.concatenate([r[19:22], refs.euler_rates_from_global(r[0:3], r[16:19]), r[22:32]]))


def _step_inputs(n, seed):
    """States whose joints sit inside, exactly at and beyond (by 1 mrad to 60 mrad) their default bounds, with velocities both ways, inside
    and outside v_s = 0.01 rad/s."""
    rng = np.random.default_rng(seed)
    d = hb.default_joint_model()
    lo, hi = np.array(d.lower[:]), np.array(d.upper[:])
    rbd = sc.consistent_rbd(sc.random_initial_states(n, seed=seed + 40), rng, 0.02)
    rbd[:, 5] = rng.uniform(0.60, 0.64, n)
    rbd[:, 16:19] = rng.uniform(-1.0, 1.0, (n, 3))
    where = rng.integers(0, 5, (n, 10))          # 0 inside, 1 at upper, 2 at lower, 3 past upper, 4 past lower
    past = rng.uniform(1e-3, 0.06, (n, 10))
    q = np.where(where == 0, lo + rng.uniform(0.1, 0.9, (n, 10)) * (hi - lo), 0.0)
    q = np.where(where == 1, hi, q); q = np.where(where == 2, lo, q)
    q = np.where(where == 3, hi + past, q); q = np.where(where == 4, lo - past, q)
    rbd[:, 6:16] = q
    speed = np.where(rng.random((n, 10)) < 0.5, rng.uniform(0.0, 0.01, (n, 10)), rng.uniform(0.01, 3.0, (n, 10)))
    rbd[:, 22:32] = speed * rng.choice([-1.0, 1.0], (n, 10))
    return rbd, rng.uniform(-15, 15, (n, 10)), rng


def _records(n, rng):
    """Random records: friction losses 0 to 0.5 N m, v_s 0.012 to 0.05 rad/s, the default ranges (one side open on some joints), stop
    gains around the defaults."""
    d = hb.default_joint_model()
    lo = np.tile(np.array(d.lower[:]), (n, 1)); hi = np.tile(np.array(d.upper[:]), (n, 1))
    lo[rng.random((n, 10)) < 0.15] = -inf; hi[rng.random((n, 10)) < 0.15] = inf
    vs = rng.uniform(0.012, 0.05, n)                 # f / v_s <= 42: stable at one substep, 0.002 (1 + 42) <= 0.1
    return hb.make_joint_models(n, friction_loss=rng.uniform(0.0, 0.5, (n, 10)) * (rng.random((n, 10)) < 0.8), friction_velocity=vs,
                                lower=lo, upper=hi, stop_stiffness=rng.uniform(500.0, 5000.0, n), stop_damping=rng.uniform(20.0, 200.0, n))


def _prm(substeps=4):
    prm = hb.default_sim_params(); prm.substeps = substeps
    return prm


# ---------------------------------------------------------------------------------------------------------------- 1. the plant step
@pytest.mark.parametrize("substeps", [1, 4])
def test_plant_step_matches_numpy(gpu_ctx, oracle, substeps):
    n = 12
    rbd, tau, rng = _step_inputs(n, 5 + substeps)
    Jm = _records(n, rng)
    Jm[0] = hb.default_joint_model()
    prm = _prm(substeps)
    nxt, cf, fl = gpu_ctx.sim_step(rbd, tau, prm, joints=Jm)
    for i in range(n):
        ref, F, _ = plant_numpy(JointOracle(oracle, Jm[i], prm.joint_armature), rbd[i], tau[i], prm)
        assert _close(nxt[i], ref), (i, np.abs(nxt[i] - ref).max())
        assert _close(cf[i], F, 1e-7), i
    assert not _same(nxt, gpu_ctx.sim_step(rbd, tau, prm)[0])


def test_plant_step_with_every_other_plant_input(gpu_ctx, oracle):
    """Joint models with link variations, a payload, a wrench, a terrain and, on a second call, a motor bridge."""
    n = 6
    rbd, tau, rng = _step_inputs(n, 17)
    Jm = _records(n, rng)
    L = hb.make_link_variations(n, rng.uniform(0.7, 1.5, (n, 11)), rng.uniform(-0.01, 0.01, (n, 11, 3)), rng.uniform(0.7, 1.5, (n, 11)))
    V = hb.make_plant_variations(n, 2.0, [0.02, -0.01, 0.08], np.diag([0.01, 0.012, 0.008]), friction_scale=0.7, motor_strength=0.9)
    W = np.c_[rng.uniform(-40, 40, (n, 3)), rng.uniform(-5, 5, (n, 3))]
    T = hb.make_terrains(n, 0.6 + rng.uniform(0.0, 0.03, (n, 4, 4)), 0.1, rbd[:, 3:5] - 0.15)
    prm = _prm(2)
    nxt, cf, _ = gpu_ctx.sim_step(rbd, tau, prm, wrench=W, variation=V, terrain=T, links=L, joints=Jm)
    for i in range(n):
        ref, F, _ = plant_numpy(JointOracle(LinkOracle(oracle, L[i]), Jm[i], prm.joint_armature), rbd[i], tau[i], prm, W[i], V[i], T[i])
        assert _close(nxt[i], ref), (i, np.abs(nxt[i] - ref).max())
    br = hb.make_motor_bridges(n)
    jcmd = np.stack([rbd[:, 6:16], np.zeros((n, 10)), np.full((n, 10), 30.0), np.full((n, 10), 1.0), rng.uniform(-5, 5, (n, 10))], axis=2)
    mcmd = hb.bridge_encode(br, jcmd)
    lim = np.full(10, 40.0)
    nxt, _, _, applied = gpu_ctx.sim_step(rbd, mcmd, prm, variation=V, bridge=br, limits=lim, links=L, joints=Jm)
    for i in range(n):
        ref, _, _, ap = plant_bridged(JointOracle(LinkOracle(oracle, L[i]), Jm[i], prm.joint_armature), rbd[i], prm, br[i], mcmd[i], lim, V[i])
        assert _close(nxt[i], ref) and _close(applied[i], ap), i


# ---------------------------------------------------------------------------------------------------------------- 2. exact identities
def _step_links(ctx, rbd, tau, prm, variation=None):
    """hb_sim_step_links called directly: the plant step as it was before joint models."""
    rbd = rbd.copy(); B = rbd.shape[0]
    cf = np.zeros((B, 12)); fl = np.zeros((B, 4), dtype=np.uint8)
    assert ctx._lib.hb_sim_step_links(ctx._h, B, C.byref(prm), api._ptr(rbd), api._ptr(tau), None, variation, None, None, None, None, None,
                                      None, api._ptr(cf), api._ptr(fl)) == 0
    return rbd, cf, fl


def test_no_record_and_disabled_records_are_the_links_step_bitwise(gpu_ctx):
    n = 8
    rbd, tau, rng = _step_inputs(n, 21)
    prm = _prm()
    V = hb.make_plant_variations(n, 1.5, [0.0, 0.0, 0.05], np.diag([0.01, 0.01, 0.01]))
    plain = _step_links(gpu_ctx, rbd, tau, prm, V)
    for got in (gpu_ctx.sim_step(rbd, tau, prm, variation=V), gpu_ctx.sim_step(rbd, tau, prm, variation=V, joints=disabled(n))):
        for x, y in zip(plain, got):
            assert _same(x, y)
    Jm = _records(n, rng)
    for i in (0, 3, 4, 7):
        Jm[i] = disabled()[0]
    mixed = gpu_ctx.sim_step(rbd, tau, prm, variation=V, joints=Jm)
    for i in range(n):
        assert all(_same(x[i], y[i]) for x, y in zip(plain, mixed)) == (i in (0, 3, 4, 7)), i


# ---------------------------------------------------------------------------------------------------------------- 3. physics
def _free_flight(substeps=4):
    prm = hb.default_sim_params()
    prm.ground_height = -100.0; prm.substeps = substeps
    return prm


def test_constant_torque_settles_on_the_stop(gpu_ctx, oracle):
    """Free flight (no ground, so gravity loads no joint): a constant torque tau drives one joint into its stop, where it settles at the
    penetration r = tau / (k m_jj), m_jj the joint's diagonal of M + armature at the settled q. At rest the joint's row of the dynamics is
    m_jj (k r + b v_j) = tau - ((M + A) qdd + nle)_j - (d + f / v_s) v_j, so |m_jj k r - tau| <= E = |((M + A) qdd + nle)_j| +
    (m_jj b + d + f / v_s) |v_j|. E is evaluated at the last state, qdd from the last tick's velocity change; the test asserts
    |r - tau / (k m_jj)| <= 2 E / (k m_jj) + 1e-12 and that this bound is below 1e-4 of r (the joint has settled)."""
    cases = [(3, 5.0), (0, -4.0), (8, 8.0), (6, -3.0)]       # (joint, torque): knee and hip roll, both ends
    n = len(cases)
    rbd = np.tile(sc.consistent_rbd(sc.INITIAL_STATE[None, :]), (n, 1))
    tau = np.zeros((n, 10))
    for i, (j, t) in enumerate(cases):
        tau[i, j] = t
    d = hb.default_joint_model()
    Jm = hb.make_joint_models(n)
    prm = _free_flight()
    r = rbd.copy()
    for _ in range(1500):
        prev = r
        r, _, fl = gpu_ctx.sim_step(r, tau, prm, joints=Jm)
        assert (fl == 0).all()
    for i, (j, t) in enumerate(cases):
        q, v = _qv(r[i]); _, v0 = _qv(prev[i])
        o = oracle.rbd(q, v)
        M = o["M"] + np.diag(np.r_[np.zeros(6), np.full(10, prm.joint_armature)])
        k, mjj = 6 + j, M[6 + j, 6 + j]
        pen = q[k] - d.upper[j] if t > 0 else d.lower[j] - q[k]
        want = abs(t) / (d.stop_stiffness * mjj)
        E = abs((M @ ((v - v0) / prm.dt) + o["nle"])[k]) + (mjj * d.stop_damping + prm.joint_damping + d.friction_loss[j] / d.friction_velocity) * abs(v[k])
        tol = 2 * E / (d.stop_stiffness * mjj) + 1e-12
        assert tol < 1e-4 * want, (i, tol, want)
        assert abs(pen - want) <= tol, (i, pen, want, tol)


def test_friction_dissipates_in_free_flight(gpu_ctx, oracle):
    """Free flight with zero torques and initial joint velocities of up to 2 rad/s, friction loss on and no stops: the mechanical energy
    1/2 v'(M + A)v + sum_b m_b g z_b does not increase from tick to tick (to 1e-9 of its size, the rounding of the sum), and after 2 s every
    joint velocity is below v_s."""
    n = 3
    rng = np.random.default_rng(43)
    rbd = sc.consistent_rbd(sc.random_initial_states(n, seed=43))
    rbd[:, 22:] = rng.uniform(-2, 2, (n, 10))
    Jm = hb.make_joint_models(n, lower=-inf, upper=inf)
    prm = _free_flight()
    A = np.diag(np.r_[np.zeros(6), np.full(10, prm.joint_armature)])
    body = bodies()

    def energy(r):
        E = np.zeros(n)
        for i in range(n):
            q, v = _qv(r[i])
            E[i] = 0.5 * v @ (oracle.rbd(q, v)["M"] + A) @ v + 9.81 * (body[0] * body_motion(q, v, body)[0][:, 2]).sum()
        return E

    r, E0 = rbd.copy(), energy(rbd)
    for _ in range(1000):
        r, _, _ = gpu_ctx.sim_step(r, np.zeros((n, 10)), prm, joints=Jm)
        E1 = energy(r)
        assert (E1 <= E0 + 1e-9 * np.maximum(1.0, np.abs(E0))).all(), E1 - E0
        E0 = E1
    assert (np.abs(r[:, 22:32]) < Jm[0].friction_velocity).all(), np.abs(r[:, 22:32]).max()


def test_a_stop_never_pulls(gpu_ctx):
    """Joints past a bound but moving back inside fast enough that k r + b v has the sign of a pull: the stop is clipped to 0, so the
    step equals the step with that joint's bound removed, bit for bit; slower, it pushes and the steps differ."""
    n = 4
    rbd = np.tile(sc.consistent_rbd(sc.INITIAL_STATE[None, :]), (n, 1))
    rbd[:, 5] += 1.0                                     # off the ground
    d = hb.default_joint_model()
    k, b, r = d.stop_stiffness, d.stop_damping, 0.02
    v_zero = k * r / b                                   # the speed back inside at which k r + b v = 0
    rbd[0, 6 + 3], rbd[0, 22 + 3] = d.upper[3] + r, -3.0 * v_zero       # pulls: clipped
    rbd[1, 6 + 1], rbd[1, 22 + 1] = d.lower[1] - r, 3.0 * v_zero
    rbd[2, 6 + 3], rbd[2, 22 + 3] = d.upper[3] + r, -0.3 * v_zero       # pushes
    rbd[3, 6 + 1], rbd[3, 22 + 1] = d.lower[1] - r, 0.3 * v_zero
    prm = _free_flight(1)
    with_stop = gpu_ctx.sim_step(rbd, np.zeros((n, 10)), prm, joints=hb.make_joint_models(n, friction_loss=0.0))
    open_ = hb.make_joint_models(n, friction_loss=0.0)
    open_[0].upper[3] = inf; open_[2].upper[3] = inf; open_[1].lower[1] = -inf; open_[3].lower[1] = -inf
    without = gpu_ctx.sim_step(rbd, np.zeros((n, 10)), prm, joints=open_)
    assert _same(with_stop[0][:2], without[0][:2])
    assert not _same(with_stop[0][2], without[0][2]) and not _same(with_stop[0][3], without[0][3])
    assert with_stop[0][2, 22 + 3] < without[0][2, 22 + 3] and with_stop[0][3, 22 + 1] > without[0][3, 22 + 1]


# ---------------------------------------------------------------------------------------------------------------- 4. episodes
def _episode_records(n):
    """The default record, ranges narrowed to 0.03 rad around the start pose (the stops act from the first steps), friction only, stops only
    with stiff gains, one disabled record, cycled."""
    d = hb.default_joint_model()
    lo, hi = np.array(d.lower[:]), np.array(d.upper[:])
    q0 = sc.INITIAL_STATE[12:22]
    kinds = [hb.make_joint_models(1)[0],
             hb.make_joint_models(1, lower=q0 - 0.03, upper=q0 + 0.03)[0],
             hb.make_joint_models(1, lower=-inf, upper=inf, friction_loss=0.4, friction_velocity=0.02)[0],
             hb.make_joint_models(1, friction_loss=0.0, lower=np.maximum(lo, q0 - 0.05), upper=np.minimum(hi, q0 + 0.05), stop_stiffness=8000.0,
                                  stop_damping=300.0)[0],
             disabled()[0]]
    return array_of([kinds[k % len(kinds)] for k in range(n)])


@pytest.mark.parametrize("wbc, event_nodes, estimated", [("weighted", False, False), ("hierarchical", True, True), ("weighted", True, True),
                                                         ("hierarchical", False, False)],
                         ids=["weighted-uniform-truth", "hierarchical-event_nodes-estimator", "weighted-event_nodes-estimator",
                              "hierarchical-uniform-truth"])
def test_episode_equals_the_stepwise_loop_bitwise(wbc, event_nodes, estimated):
    """Joint models on all robots but the last, with pushes, plant and link variations, a terrain, goals, MPC latencies, hardware and
    controller settings, motor bridges and teleop set alongside."""
    ctx = context(event_nodes)
    ctx.set_wbc_formulation(wbc)
    n_ticks, log_every = 80, 10
    rbd0 = start_states(ctx, B, seed=401)
    vels = cmd_vels(B)
    prm = params(log_every)
    models = _episode_records(B - 1)
    links = hb.make_link_variations(2, [[1.0] + [1.2] * 10, [0.9] * 11], 0.0, 1.0)
    kw = use(ctx, plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION, motor_strength=0.95),
             pushes=hb.make_push_schedules(B, 0.05, 0.05, PUSH), terrains=small_terrains(), mpc_latencies=[0, 2, 5, 1, 0, 3],
             hardware=hb.make_hardware_settings(B, actuation_delay=np.linspace(0.0, 0.012, B), encoder_offset=np.linspace(-0.01, 0.01, 10)))
    bridges = hb.make_motor_bridges(3)
    goals, teleop = random_goals(rbd0, B, 401), hb.make_teleop_settings(4, period_ticks=5 * prm.mpc_every)
    ctx.set_motor_bridge(bridges); ctx.set_goals(goals); ctx.set_teleop(teleop); ctx.set_link_variations(links); ctx.set_joint_models(models)
    g = hb.default_pd_gains(); g.kp_big_stance = 45.0
    ctx.set_controller_settings(hb.make_controller_settings(B, wbc=ctx.wbc_settings(), gains=g))
    ep = est_params(seed=4011) if estimated else None
    fresh = (lambda: hb.estimation_states(B, 70)) if estimated else (lambda: None)
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, fresh())
    prm.gains = g
    loop = JointLoop(TeleopLoop(ctx, teleop, prm.period, goals), models, links, bridges, prm.torque_limit)
    r = stepwise(loop, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, fresh(), **kw)
    ctx.set_plan_targets(None)
    assert_episode_equal(d, r)
    ctx.set_joint_models(None)
    u = outputs(device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, fresh()))
    moved = [not np.array_equal(a, b) for a, b in zip(outputs(d)[0], u[0])]
    assert moved == [True, True, True, True, False, False], moved      # robot 4 has the disabled record, robot 5 none
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_disabled_and_cleared_records_are_the_unset_episode_bitwise(estimated):
    ctx = context()
    rbd0 = start_states(ctx, B, seed=402)
    ep = est_params(seed=21) if estimated else None
    assert_null_settings(ctx, "joint_models", lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 60, params(5), 5, ep,
                                                             hb.estimation_states(B, 50) if estimated else None),
                         [disabled(B), disabled(3)], _episode_records(B))
    ctx.close()


def test_setting_contract():
    ctx = context()
    rbd0 = start_states(ctx, B, seed=403)
    r = list(_episode_records(5))
    full = array_of([r[0], r[1], r[2], r[3], r[0], r[1]])
    one = array_of([r[1]])
    other = array_of([r[3], r[2], r[1], r[3], r[0], r[1]])       # instance 3 keeps its record
    part = array_of([r[1], r[0]])
    assert_setting_episodes(ctx, "joint_models", rbd0, params(10), full, one, other, 3, part, padded(part, B))
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_rejected_settings_and_the_stability_rule(estimated):
    ctx = context()
    rbd0 = start_states(ctx, B, seed=404)
    ep = est_params(seed=11) if estimated else None

    def run(prm=None):
        return device(ctx, rbd0, GAITS, cmd_vels(B), 40, prm or params(5), 5, ep, hb.estimation_states(B, 50) if estimated else None)
    want, launches = assert_rejected_settings(ctx, "joint_models", run, _episode_records(B), bad_records(),
                                              hb.make_joint_models(ctx.max_batch + 1))
    rbd = np.zeros((2, 32))
    for bad in bad_records():                          # the host plant step validates its records as the setter does
        with pytest.raises(hb.HunterB200Error):
            ctx.sim_step(rbd, np.zeros((2, 10)), joints=bad)
    # the stability rule: h (d + f / v_s) <= A for every record read, checked against each call's params before any launch
    steep = hb.make_joint_models(2, friction_loss=[0.2] * 9 + [2.5])
    with pytest.raises(hb.HunterB200Error):
        ctx.sim_step(rbd, np.zeros((2, 10)), joints=steep)
    prm = params(5); prm.sim.joint_armature = 0.0105 * 0.99
    c0 = ctx.launch_count
    with pytest.raises(hb.HunterB200Error):
        run(prm)                                         # the default records need A >= 0.0105 at the default substep
    assert ctx.launch_count == c0
    ctx.set_joint_models(array_of([hb.default_joint_model()] * B + [steep[1]]))     # beyond this call's B: not read
    run()
    ctx.set_joint_models(array_of([hb.default_joint_model()] * (B - 1) + [steep[1]]))
    c0 = ctx.launch_count
    with pytest.raises(hb.HunterB200Error):
        run()
    assert ctx.launch_count == c0
    prm = params(5); prm.sim.substeps = 1; prm.sim.joint_armature = 0.5      # h = 0.002: 0.002 (1 + 250) = 0.502 > 0.5
    with pytest.raises(hb.HunterB200Error):
        run(prm)
    prm.sim.joint_armature = 0.502 + 1e-9
    run(prm)
    ctx.set_joint_models(_episode_records(B))
    assert_episode_equal(want, run())
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_joint_models_add_no_launch(estimated):
    ctx = context()
    rbd0 = start_states(ctx, B, seed=405)
    vels = cmd_vels(B)
    prm = params(0)
    ep = est_params(seed=5) if estimated else None
    plain = launch_coefficients(ctx, rbd0, GAITS, vels, prm, ep)
    ctx.set_joint_models(_episode_records(B))
    assert launch_coefficients(ctx, rbd0, GAITS, vels, prm, ep) == plain
    ctx.close()
