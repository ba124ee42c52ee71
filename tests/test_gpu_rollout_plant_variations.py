"""Varied plants (hb_rollout_set_plant_variations, hb_sim_step_varied): a plant of its own for each robot, with a payload on the base, scaled
ground contact and motor strength. The varied plant step is checked against a numpy restatement, against exact identities, and against
momentum, energy and static balance; the varied episode bit for bit against the loop of public calls, and against the unvaried episode:
defaults, continuation, independence, permutation, instances beyond the setting, clearing, launch counts; then the argument checks."""
import ctypes as C

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from episode_ref import (GAITS, assert_episode_equal, assert_null_settings, assert_rejected_settings, assert_setting_episodes, cmd_vels, context,
                         device, est_params, launch_coefficients, params, plant_numpy, start_states, stepwise, use)
from oracle import refs

pytestmark = pytest.mark.gpu

BOX = np.diag([(0.2 ** 2 + 0.1 ** 2) / 12, (0.2 ** 2 + 0.1 ** 2) / 12, (0.2 ** 2 + 0.2 ** 2) / 12])    # 0.2 x 0.2 x 0.1 m box, per kg


def _full_inertia(rng, scale):
    """A random symmetric positive definite inertia with off-diagonal terms."""
    A = rng.normal(size=(3, 3))
    I = scale * (A @ A.T + 0.5 * np.eye(3))
    return np.triu(I) + np.triu(I, 1).T                   # exactly symmetric


def _variations():
    """Six instances: nominal (default); a 3 kg payload off-centre with a full inertia; slippery ground; soft, well-damped ground; weak and
    dead motors; everything at once."""
    rng = np.random.default_rng(3)
    V = hb.make_plant_variations(6)
    V[1] = hb.make_plant_variations(1, 3.0, [0.03, -0.02, 0.1], _full_inertia(rng, 0.004))[0]
    V[2] = hb.make_plant_variations(1, friction_scale=0.35)[0]
    V[3] = hb.make_plant_variations(1, stiffness_scale=0.5, damping_scale=2.0)[0]
    ms = np.ones(10); ms[[1, 6]] = 0.7; ms[4] = 0.0
    V[4] = hb.make_plant_variations(1, motor_strength=ms)[0]
    V[5] = hb.make_plant_variations(1, 2.0, [-0.02, 0.01, 0.08], _full_inertia(rng, 0.003), 0.6, 1.5, 0.7, np.linspace(0.8, 1.0, 10))[0]
    return V


def _one_varied(B, i, **kw):
    """B default variations, instance i varied by kw (make_plant_variations arguments)."""
    V = hb.make_plant_variations(B)
    V[i] = hb.make_plant_variations(1, **kw)[0]
    return V


def _step_inputs(B, seed):
    rng = np.random.default_rng(seed)
    x = sc.random_initial_states(B, seed=seed + 40)
    rbd = sc.consistent_rbd(x, rng, 0.02)
    rbd[:, 5] = rng.uniform(0.60, 0.64, B)               # some feet in the ground, some above it
    rbd[:, 1] = rng.uniform(-0.3, 0.3, B); rbd[:, 2] = rng.uniform(-0.3, 0.3, B)
    rbd[:, 16:19] = rng.uniform(-1.5, 1.5, (B, 3))       # base angular velocity: the payload's velocity-product terms act
    return rbd, rng.uniform(-15, 15, (B, 10)), rng


# ---------------------------------------------------------------------------------------------------------------- the plant step
def test_varied_plant_step_matches_numpy_restatement(gpu_ctx, oracle):
    B = 12
    rbd, tau, rng = _step_inputs(B, 8)
    V = hb.make_plant_variations(B, rng.uniform(0.5, 6.0, B), rng.uniform(-0.1, 0.15, (B, 3)), np.stack([_full_inertia(rng, 0.005) for _ in range(B)]),
                                 rng.uniform(0.2, 0.9, B), rng.uniform(0.4, 2.5, B), rng.uniform(0.3, 2.0, B), rng.uniform(0.2, 1.3, (B, 10)))
    W = np.c_[rng.uniform(-200, 200, (B, 3)), rng.uniform(-40, 40, (B, 3))]
    W[::2] = 0.0
    prm = hb.default_sim_params()
    nxt, cf, fl = gpu_ctx.sim_step(rbd, tau, prm, wrench=W, variation=V)
    base = gpu_ctx.sim_step(rbd, tau, prm, wrench=W)
    touched = 0
    for i in range(B):
        ref, F, _ = plant_numpy(oracle, rbd[i], tau[i], prm, W[i], V[i])
        assert np.abs(nxt[i] - ref).max() < 1e-9 * max(1.0, np.abs(ref).max()), (i, np.abs(nxt[i] - ref).max())
        assert np.abs(cf[i] - F).max() < 1e-7 * max(1.0, np.abs(F).max()), i
        assert np.array_equal(fl[i] != 0, F[2::3] > 0)
        touched += int((F[2::3] > 0).sum())
        assert np.abs(nxt[i] - base[0][i]).max() > 1e-6          # the variation acts
    assert 0 < touched < 4 * B
    # the payload alone (nominal ground and motors) against the restatement too
    P = hb.make_plant_variations(B, 4.0, [0.05, 0.02, 0.12], _full_inertia(rng, 0.01))
    nxt, cf, _ = gpu_ctx.sim_step(rbd, tau, prm, variation=P)
    for i in range(B):
        ref, F, _ = plant_numpy(oracle, rbd[i], tau[i], prm, variation=P[i])
        assert np.abs(nxt[i] - ref).max() < 1e-9 * max(1.0, np.abs(ref).max()), i
        assert np.abs(cf[i] - F).max() < 1e-7 * max(1.0, np.abs(F).max()), i


def test_exact_identities_of_the_varied_step(gpu_ctx):
    B = 8
    rbd, tau, rng = _step_inputs(B, 9)
    prm = hb.default_sim_params()
    lib, P = gpu_ctx._lib, (lambda a: C.c_void_p(a.ctypes.data))
    base = gpu_ctx.sim_step(rbd, tau, prm)

    def varied(w, v):
        r = rbd.copy(); cf = np.zeros((B, 12)); fl = np.zeros((B, 4), dtype=np.uint8)
        assert lib.hb_sim_step_varied(gpu_ctx._h, B, C.byref(prm), P(r), P(tau), None if w is None else P(w), v, P(cf), P(fl)) == 0
        return r, cf, fl

    def wrench_step(w):
        r = rbd.copy(); cf = np.zeros((B, 12)); fl = np.zeros((B, 4), dtype=np.uint8)
        assert lib.hb_sim_step_wrench(gpu_ctx._h, B, C.byref(prm), P(r), P(tau), None if w is None else P(w), P(cf), P(fl)) == 0
        return r, cf, fl

    # the default variation, a NULL variation and hb_sim_step_wrench are hb_sim_step_batch, bit for bit
    for got in (varied(None, hb.make_plant_variations(B)), varied(None, None), wrench_step(None), gpu_ctx.sim_step(rbd, tau, prm, variation=hb.make_plant_variations(B))):
        for a, b in zip(got, base):
            assert np.array_equal(a, b)
    # with a wrench: the default variation is hb_sim_step_wrench
    W = np.c_[rng.uniform(-100, 100, (B, 3)), rng.uniform(-20, 20, (B, 3))]
    for a, b in zip(varied(W, hb.make_plant_variations(B)), wrench_step(W)):
        assert np.array_equal(a, b)
    # motor strength s on tau is strength 1 on s * tau
    s = rng.uniform(0.0, 1.5, (B, 10)); s[0, 3] = 0.0
    ground = dict(friction_scale=0.5, stiffness_scale=1.3, damping_scale=0.8)
    got = gpu_ctx.sim_step(rbd, tau, prm, variation=hb.make_plant_variations(B, motor_strength=s, **ground))
    want = gpu_ctx.sim_step(rbd, s * tau, prm, variation=hb.make_plant_variations(B, **ground))
    for a, b in zip(got, want):
        assert np.array_equal(a, b)
    assert not np.array_equal(got[0], gpu_ctx.sim_step(rbd, tau, prm, variation=hb.make_plant_variations(B, **ground))[0])


def _payload_state(r, V):
    """World position and velocity of each payload's CoM, its angular velocity, rotation-dependent inertia: (x_c, v_c, omega, I_w)."""
    out = []
    for i in range(len(r)):
        R = refs.rot_zyx(r[i, 0:3]); c = np.array(V[i].payload_com[:]); Ic = np.array(V[i].payload_inertia[:]).reshape(3, 3)
        w = r[i, 16:19]
        out.append((r[i, 3:6] + R @ c, r[i, 19:22] + np.cross(w, R @ c), w, R @ Ic @ R.T))
    return out


def _free_flight_prm(substeps):
    prm = hb.default_sim_params()
    prm.ground_height = -100.0; prm.joint_armature = 0.0; prm.joint_damping = 0.0; prm.substeps = substeps
    return prm


def _free_flight_start(B, seed):
    rng = np.random.default_rng(seed)
    rbd = sc.consistent_rbd(sc.random_initial_states(B, seed=seed))
    rbd[:, 0:3] = [[0.7, 0.3, -0.2], [-1.2, -0.25, 0.35], [2.5, 0.1, 0.5]][:B]
    rbd[:, 16:] = 0.0
    rbd[:, 16:19] = rng.uniform(-1.0, 1.0, (B, 3))
    rbd[:, 22:] = rng.uniform(-1.0, 1.0, (B, 10))
    V = hb.make_plant_variations(B, [2.0, 4.0, 6.5][:B], rng.uniform(-0.08, 0.12, (B, 3)), np.stack([_full_inertia(rng, 0.01) for _ in range(B)]))
    return rbd, V, rng


def test_free_flight_momentum_balance_with_a_payload(gpu_ctx):
    """Free flight, a force f on the base origin, zero joint torques, no armature or joint damping: over T = 50 ticks the linear momentum of
    robot plus payload changes by (f + (m + m_p) g) T. The robot's part is rbd_to_centroidal's normalised momentum x its mass, the payload's
    m_p v_c with v_c = pdot + omega x R c. As in the pushed plant's balance test, semi-implicit Euler leaves an O(h T) error, so the test
    runs 4 and 16 substeps: the error must shrink about 4x and its Richardson extrapolation must be below 2e-3 N s. A wrong payload term
    leaves an O(1) error that does not shrink with h."""
    B = 3
    rbd, V, rng = _free_flight_start(B, 21)
    W = np.c_[rng.uniform(-80, 80, (B, 3)), np.zeros((B, 3))]
    m, mp, g = sc.TOTAL_MASS, np.array([V[i].payload_mass for i in range(B)]), np.array([0.0, 0.0, -9.81])

    def momentum(r):
        return gpu_ctx.rbd_to_centroidal(r)[:, :3] * m + mp[:, None] * np.array([s[1] for s in _payload_state(r, V)])

    n, err = 50, {}
    for substeps in (4, 16):
        prm = _free_flight_prm(substeps)
        T_ = n * prm.dt
        p0, r = momentum(rbd), rbd.copy()
        for _ in range(n):
            r, _, fl = gpu_ctx.sim_step(r, np.zeros((B, 10)), prm, wrench=W, variation=V)
            assert (fl == 0).all()
        err[substeps] = momentum(r) - p0 - (W[:, :3] + (m + mp)[:, None] * g) * T_
    e4, e16 = np.abs(err[4]).max(), np.abs(err[16]).max()
    assert e16 < 0.3 * e4 + 1e-6, (e4, e16)
    rich = (4 * err[16] - err[4]) / 3
    assert np.abs(rich).max() < 2e-3, (rich, err)


def test_free_flight_energy_with_a_payload(gpu_ctx, oracle):
    """Free flight with zero torques, no armature and no joint damping conserves the mechanical energy of robot plus payload: the robot's
    1/2 v'Mv + m g z_com from oracle.rbd, the payload's 1/2 m_p |v_c|^2 + 1/2 omega' I_w omega + m_p g z_c from its definition. The
    integrator drifts at O(h): the drift must shrink about 4x from 4 to 16 substeps and its Richardson extrapolation must be small against
    the kinetic energy. A wrong payload inertia or velocity-product term leaves a drift that does not shrink with h."""
    B = 3
    rbd, V, _ = _free_flight_start(B, 33)
    m = sc.TOTAL_MASS

    def energy(r):
        E = np.zeros(B)
        for i, (xc, vc, w, Iw) in enumerate(_payload_state(r, V)):
            q = np.concatenate([r[i, 3:6], r[i, 0:3], r[i, 6:16]])
            v = np.concatenate([r[i, 19:22], refs.euler_rates_from_global(r[i, 0:3], r[i, 16:19]), r[i, 22:32]])
            o = oracle.rbd(q, v)
            mp = V[i].payload_mass
            E[i] = 0.5 * v @ o["M"] @ v + m * 9.81 * o["com"][2] + 0.5 * mp * vc @ vc + 0.5 * w @ Iw @ w + mp * 9.81 * xc[2]
        return E

    n, drift = 50, {}
    E0 = energy(rbd)
    for substeps in (4, 16):
        prm = _free_flight_prm(substeps)
        r = rbd.copy()
        for _ in range(n):
            r, _, _ = gpu_ctx.sim_step(r, np.zeros((B, 10)), prm, variation=V)
        drift[substeps] = energy(r) - E0
    d4, d16 = np.abs(drift[4]).max(), np.abs(drift[16]).max()
    assert d16 < 0.35 * d4 + 1e-9, (d4, d16)
    rich = (4 * drift[16] - drift[4]) / 3
    assert np.abs(rich).max() < 0.05 * d4 + 1e-6, (rich, drift)


def test_standing_robot_carries_the_payload_on_its_contacts(gpu_ctx):
    """A robot held by a stiff joint PD law on the ground settles to summed normal contact forces of (m + m_p) g within 1 %, on soft and on
    stiff ground."""
    B = 4
    rbd = start_states(gpu_ctx, B, seed=5)
    q0 = rbd[:, 6:16].copy()
    mp = np.array([0.0, 2.0, 5.0, 7.5])
    V = hb.make_plant_variations(B, mp, np.where(mp[:, None] > 0, [0.0, 0.0, 0.1], 0.0), BOX[None] * mp[:, None, None], friction_scale=[1.0, 0.6, 0.4, 0.25],
                                 stiffness_scale=[1.0, 1.5, 2.0, 0.8], damping_scale=[1.0, 1.5, 1.0, 0.7])
    prm = hb.default_sim_params()
    prm.ground_height = 0.02
    r = rbd.copy()
    for _ in range(1000):
        tau = 400.0 * (q0 - r[:, 6:16]) - 10.0 * r[:, 22:32]
        r, cf, _ = gpu_ctx.sim_step(r, tau, prm, variation=V)
    fz = cf[:, 2::3].sum(axis=1)
    want = (sc.TOTAL_MASS + mp) * 9.81
    assert np.abs(fz / want - 1).max() < 0.01, (fz, want)
    assert np.abs(r[:, 16:]).max() < 0.05


# ---------------------------------------------------------------------------------------------------------------- varied episodes
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
def test_varied_episode_equals_the_stepwise_loop_bitwise(event_nodes):
    ctx = context(event_nodes)
    B, n_ticks, log_every = 6, 200, 10
    rbd0 = start_states(ctx, B, seed=11)
    vels = cmd_vels(B)
    prm = params(log_every)
    kw = use(ctx, plant_variations=_variations(), pushes=hb.make_push_schedules(B, 0.15, 0.05, [[30.0, -20.0, 0.0]]))
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every)
    r = stepwise(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, **kw)
    assert_episode_equal(d, r)
    ctx.set_plant_variations(None)
    u = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every)
    moved = [not np.array_equal(a, b) for a, b in zip(d[0].cpu().numpy(), u[0].cpu().numpy())]
    assert moved == [False, True, True, True, True, True], moved
    ctx.close()


def test_varied_estimated_episode_equals_the_stepwise_loop_bitwise():
    ctx = context()
    B, n_ticks, log_every = 6, 120, 10
    rbd0 = start_states(ctx, B, seed=11)
    vels = cmd_vels(B)
    prm = params(log_every)
    ep = est_params(seed=2024)
    kw = use(ctx, plant_variations=_variations(), pushes=hb.make_push_schedules(B, 0.1, 0.04, [[0.0, 40.0, 0.0]]))
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 40))
    r = stepwise(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 40), **kw)
    assert_episode_equal(d, r)
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_default_variations_change_nothing(estimated):
    ctx = context()
    B, n_ticks = 6, 100
    rbd0 = start_states(ctx, B, seed=13)
    vels = cmd_vels(B)
    prm = params(5)
    ep = est_params(seed=77) if estimated else None
    assert_null_settings(ctx, "plant_variations", lambda: device(ctx, rbd0, GAITS, vels, n_ticks, prm, 5, ep),
                         (hb.make_plant_variations(B), hb.make_plant_variations(3)), _variations())
    ctx.close()


def test_continuation_independence_permutation_and_instances_beyond_the_setting():
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=14)
    V = _variations()
    one = _one_varied(B, 0, payload_mass=4.0, payload_com=[0.02, 0.0, 0.1], payload_inertia=4.0 * BOX, friction_scale=0.5)
    W = _variations()
    for i in range(B):
        if i != 2:
            W[i] = hb.make_plant_variations(1, 1.0 + i, [0.0, 0.01 * i, 0.1], (1.0 + i) * BOX, stiffness_scale=0.8)[0]
    part = (hb.HbPlantVariation * 3)(*[V[i] for i in range(3)])
    padded = (hb.HbPlantVariation * B)(*[V[i] if i < 3 else hb.default_plant_variation() for i in range(B)])
    assert_setting_episodes(ctx, "plant_variations", rbd0, params(10), V, one, W, 2, part, padded)
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_variations_add_no_launch(estimated):
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=16)
    vels = cmd_vels(B)
    prm = params(0)
    ep = est_params(seed=5) if estimated else None
    plain = launch_coefficients(ctx, rbd0, GAITS, vels, prm, ep)
    ctx.set_plant_variations(_variations())
    assert launch_coefficients(ctx, rbd0, GAITS, vels, prm, ep) == plain
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- argument checks
def test_argument_checks_return_before_any_launch_and_keep_the_setting():
    ctx = context(max_batch=6)
    lib = ctx._lib
    B = 6
    rbd0 = start_states(ctx, B, seed=17)
    vels = cmd_vels(B)
    prm = params(10)
    V = _variations()
    assert C.sizeof(hb.HbPlantVariation) == 208
    nan, inf = float("nan"), float("inf")

    def bad(field, index, value):
        W = (hb.HbPlantVariation * B)(*V)
        s = W[1]
        if index is None:
            setattr(s, field, value)
        else:
            getattr(s, field)[index] = value
        return W

    cases = [("payload_mass", None, nan), ("payload_mass", None, -0.5), ("payload_mass", None, inf), ("payload_com", 1, nan),
             ("payload_com", 2, -inf), ("payload_inertia", 4, nan), ("payload_inertia", 1, 1e-4),      # not symmetric
             ("payload_inertia", 8, -1e-3),                                                             # negative diagonal
             ("friction_scale", None, -0.1), ("friction_scale", None, nan), ("stiffness_scale", None, 0.0), ("stiffness_scale", None, -1.0),
             ("stiffness_scale", None, inf), ("damping_scale", None, -0.1), ("damping_scale", None, nan), ("motor_strength", 3, -0.2),
             ("motor_strength", 9, nan), ("motor_strength", 0, inf)]
    rejected = [bad(field, index, value) for field, index, value in cases]
    # a negative 2 x 2 principal minor, and a negative determinant with every 2 x 2 minor >= 0
    for M in ([[0.01, 0.02, 0.0], [0.02, 0.01, 0.0], [0.0, 0.0, 0.01]], [[1.0, 1.0, 0.0], [1.0, 1.0, 1.0], [0.0, 1.0, 1.0]]):
        W = (hb.HbPlantVariation * B)(*V)
        for k in range(9):
            W[1].payload_inertia[k] = np.ravel(M)[k]
        rejected.append(W)
    # a zero mass with a CoM or an inertia
    for field, index in (("payload_com", 0), ("payload_inertia", 0)):
        W = (hb.HbPlantVariation * B)(*V)
        W[0].payload_mass = 0.0
        getattr(W[0], field)[index] = 0.01
        rejected.append(W)
    big = (hb.HbPlantVariation * (B + 1))(*([V[0]] * (B + 1)))
    assert_rejected_settings(ctx, "plant_variations", lambda: device(ctx, rbd0, GAITS, vels, 60, prm, 10), V, rejected, big)
    # the host plant step checks its variations as the setting does
    sp = hb.default_sim_params()
    r = np.zeros((B, 32)); t = np.zeros((B, 10))
    P = lambda a: C.c_void_p(a.ctypes.data)
    c0 = ctx.launch_count
    for field, index, value in cases[:4]:
        assert lib.hb_sim_step_varied(ctx._h, B, C.byref(sp), P(r), P(t), None, bad(field, index, value), None, None) == -1
    assert lib.hb_sim_step_varied(ctx._h, B + 1, C.byref(sp), P(np.zeros((B + 1, 32))), P(np.zeros((B + 1, 10))), None, big, None, None) == -4
    assert lib.hb_sim_step_varied(ctx._h, 0, C.byref(sp), P(r), P(t), None, None, None, None) == 0
    assert ctx.launch_count == c0
    ctx.close()
