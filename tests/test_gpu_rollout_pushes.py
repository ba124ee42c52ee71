"""Pushed episodes (hb_rollout_set_pushes, hb_sim_step_wrench): scheduled external wrenches on the base, applied by the plant of both episode
calls. The plant step with a wrench is checked against a numpy restatement and against momentum balance in free flight; the pushed episode
bit for bit against the loop of public calls with the documented wrench restated in numpy, and against the unpushed episode: causality,
null schedules, continuation, independence, permutation, instances beyond the schedules, estimated episodes; then the argument checks."""
import ctypes as C

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from episode_ref import (GAITS, assert_continues, assert_episode_equal, assert_null_settings, assert_rejected_settings, assert_setting_episodes,
                         cmd_vels, context, device, est_params, outputs, params, plant_numpy, start_states, stepwise)

pytestmark = pytest.mark.gpu


def _schedules():
    """Six instances: one push; two overlapping pushes; a push starting between ticks in mid-episode, with a couple; none; one after the
    episode; three pushes (from t = 0, one of zero duration, a couple only)."""
    S = (hb.HbPushSchedule * 6)()
    spec = [
        [(0.05, 0.1, (60.0, 0.0, 0.0), (0.0, 0.0, 0.0))],
        [(0.1, 0.08, (0.0, -50.0, 0.0), (0.0, 0.0, 0.0)), (0.14, 0.1, (20.0, 10.0, 0.0), (0.0, 0.0, 5.0))],
        [(0.2031, 0.05, (-40.0, 30.0, 10.0), (2.0, -3.0, 1.0))],
        [],
        [(1.0, 0.1, (100.0, 0.0, 0.0), (0.0, 0.0, 0.0))],
        [(0.0, 0.02, (0.0, 40.0, 0.0), (0.0, 0.0, 0.0)), (0.1, 0.0, (500.0, 0.0, 0.0), (0.0, 0.0, 0.0)), (0.3, 0.05, (0.0, 0.0, 0.0), (-3.0, 4.0, 0.0))],
    ]
    for s, pushes in zip(S, spec):
        s.n_push = len(pushes)
        for j, (t0, d, f, tq) in enumerate(pushes):
            s.t_start[j] = t0; s.duration[j] = d
            for c in range(3):
                s.force[j][c] = f[c]; s.torque[j][c] = tq[c]
    return S


def _one_push(B, i, t_start, duration, force, torque=(0.0, 0.0, 0.0)):
    """B schedules, only instance i pushed."""
    return hb.make_push_schedules(B, np.where(np.arange(B) == i, t_start, 0.0)[:, None], np.where(np.arange(B) == i, duration, 0.0)[:, None],
                                  np.where((np.arange(B) == i)[:, None, None], np.array(force, dtype=float)[None, None], 0.0),
                                  np.where((np.arange(B) == i)[:, None, None], np.array(torque, dtype=float)[None, None], 0.0))


# ---------------------------------------------------------------------------------------------------------------- the plant step
def test_plant_step_with_wrench_matches_numpy_restatement(gpu_ctx, oracle):
    B = 10
    rng = np.random.default_rng(8)
    x = sc.random_initial_states(B, seed=50)
    rbd = sc.consistent_rbd(x, rng, 0.02)
    rbd[:, 5] = rng.uniform(0.60, 0.64, B)               # some feet in the ground, some above it
    rbd[:, 1] = rng.uniform(-0.3, 0.3, B); rbd[:, 2] = rng.uniform(-0.3, 0.3, B)    # pitch and roll, so that T is not a permutation
    tau = rng.uniform(-15, 15, (B, 10))
    W = np.c_[rng.uniform(-300, 300, (B, 3)), rng.uniform(-60, 60, (B, 3))]
    prm = hb.default_sim_params()
    nxt, cf, fl = gpu_ctx.sim_step(rbd, tau, prm, wrench=W)
    base = gpu_ctx.sim_step(rbd, tau, prm)
    touched = 0
    for i in range(B):
        ref, F, _ = plant_numpy(oracle, rbd[i], tau[i], prm, W[i])
        assert np.abs(nxt[i] - ref).max() < 1e-9 * max(1.0, np.abs(ref).max()), i
        assert np.abs(cf[i] - F).max() < 1e-7 * max(1.0, np.abs(F).max())
        assert np.array_equal(fl[i] != 0, F[2::3] > 0)
        touched += int((F[2::3] > 0).sum())
        assert np.abs(nxt[i] - base[0][i]).max() > 1e-6          # the wrench acts
    assert 0 < touched < 4 * B
    # no wrench and an all-zero wrench are the plant step of hb_sim_step_batch, bit for bit
    zero = gpu_ctx.sim_step(rbd, tau, prm, wrench=np.zeros((B, 6)))
    r = rbd.copy(); cfn = np.zeros((B, 12)); fln = np.zeros((B, 4), dtype=np.uint8)
    assert gpu_ctx._lib.hb_sim_step_wrench(gpu_ctx._h, B, C.byref(prm), C.c_void_p(r.ctypes.data), C.c_void_p(tau.ctypes.data), None,
                                           C.c_void_p(cfn.ctypes.data), C.c_void_p(fln.ctypes.data)) == 0
    for got in (zero, (r, cfn, fln)):
        for a, b in zip(got, base):
            assert np.array_equal(a, b)


@pytest.mark.parametrize("kind", ["force", "couple"])
def test_free_flight_momentum_balance(gpu_ctx, kind):
    """Free flight (ground far below), zero joint torques, armature and joint damping: over T = 50 ticks the centroidal momentum
    (rbd_to_centroidal, normalised momentum x TOTAL_MASS) changes by (F + m g) T for a force at the base origin and by (m g T, tau T) for a
    pure couple tau. Independent of the numpy restatement: a wrong sign or a transposed T fails here.
    Tolerance: semi-implicit Euler updates v with M(q_n) and then moves q, so each substep changes the momentum A(q) v by h Q_ext + O(h^2),
    and over T / h substeps the error is O(h T). With the legs swinging freely (joint rates reach ~ 17 rad/s) it is ~ 0.08 N s at
    4 substeps, so the test runs 4 and 16 substeps: the error must shrink about 4x (first order), and the Richardson extrapolation
    (4 e_16 - e_4) / 3, which cancels the O(h) term, must be below 2e-3 N s (N m s), against changes of 0.4 .. 8 N s. A wrong sign or a
    transposed T leaves an O(1) error that does not shrink with h."""
    B = 3
    rng = np.random.default_rng(21)
    rbd = sc.consistent_rbd(sc.random_initial_states(B, seed=7))
    rbd[:, 0:3] = [[0.7, 0.3, -0.2], [-1.2, -0.25, 0.35], [2.5, 0.1, 0.5]]   # yaw, pitch, roll away from the identity
    rbd[:, 16:] = 0.0
    m, g = sc.TOTAL_MASS, np.array([0.0, 0.0, -9.81])
    if kind == "force":
        W = np.c_[rng.uniform(-80, 80, (B, 3)), np.zeros((B, 3))]
    else:
        W = np.c_[np.zeros((B, 3)), rng.uniform(-8, 8, (B, 3))]
    n = 50
    err = {}
    for substeps in (4, 16):
        prm = hb.default_sim_params()
        prm.ground_height = -100.0; prm.joint_armature = 0.0; prm.joint_damping = 0.0; prm.substeps = substeps
        T = n * prm.dt
        h0 = gpu_ctx.rbd_to_centroidal(rbd)[:, :6] * m
        r = rbd.copy()
        for _ in range(n):
            r, _, fl = gpu_ctx.sim_step(r, np.zeros((B, 10)), prm, wrench=W)
            assert (fl == 0).all()
        dh = gpu_ctx.rbd_to_centroidal(r)[:, :6] * m - h0
        want = np.c_[W[:, :3] * T + m * g * T, W[:, 3:] * T]
        # a force at the base origin also has a moment about the CoM: only the linear momentum is checked then
        err[substeps] = (dh - want)[:, :3] if kind == "force" else dh - want
    e4, e16 = np.abs(err[4]).max(), np.abs(err[16]).max()
    assert e16 < 0.3 * e4 + 1e-6, (e4, e16)
    rich = (4 * err[16] - err[4]) / 3
    assert np.abs(rich).max() < 2e-3, (rich, err)
    assert np.abs(W).max() * T > 0.4


# ---------------------------------------------------------------------------------------------------------------- pushed episodes
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
def test_pushed_episode_equals_the_stepwise_loop_bitwise(event_nodes):
    ctx = context(event_nodes)
    B, n_ticks, log_every = 6, 200, 10
    rbd0 = start_states(ctx, B, seed=11)
    vels = cmd_vels(B)
    prm = params(log_every)
    S = _schedules()
    ctx.set_pushes(S)
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every)
    r = stepwise(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, pushes=S)
    assert_episode_equal(d, r)
    ctx.set_pushes(None)
    u = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every)
    moved = [not np.array_equal(a, b) for a, b in zip(d[0].cpu().numpy(), u[0].cpu().numpy())]
    assert moved == [True, True, True, False, False, True], moved
    ctx.close()


def test_state_before_the_push_is_unchanged_and_the_state_after_it_moves():
    ctx = context()
    B, n_ticks = 6, 80
    rbd0 = start_states(ctx, B, seed=12)
    vels = cmd_vels(B)
    prm = params(1)
    u = outputs(device(ctx, rbd0, GAITS, vels, n_ticks, prm, 1))
    k = 50
    ctx.set_pushes(_one_push(B, 0, k * prm.period, 0.02, (0.0, 80.0, 0.0)))
    p = outputs(device(ctx, rbd0, GAITS, vels, n_ticks, prm, 1))
    assert np.array_equal(p[4][:, :k + 1], u[4][:, :k + 1])          # log row k: the state entering the tick the push starts
    assert not np.array_equal(p[4][0, k + 1], u[4][0, k + 1])
    assert np.array_equal(p[4][1:], u[4][1:]) and np.array_equal(p[0][1:], u[0][1:])
    ctx.close()


def _null_schedule_checks(ctx, run, B, horizon_t):
    """Null schedules (none, or pushes after the episode) change nothing; a rejected set keeps the previous, pushing setting."""
    nothing = hb.make_push_schedules(B, np.zeros((B, 0)), np.zeros((B, 0)), np.zeros((B, 0, 3)))
    later = hb.make_push_schedules(B, [horizon_t, horizon_t + 0.5], [0.1, 1.0], [[500.0, 0, 0], [0, 500.0, 0]], [[0, 0, 50.0], [0, 0, 0]])
    ref, launches = assert_null_settings(ctx, "pushes", run, (nothing, later), _schedules())
    bad = _one_push(B, 1, 0.02, 0.06, (0.0, -70.0, 0.0))
    bad[0].force[0][0] = float("nan")
    pushed = _one_push(B, 1, 0.02, 0.06, (0.0, -70.0, 0.0), (0.0, 0.0, 4.0))
    want, n = assert_rejected_settings(ctx, "pushes", run, pushed, [bad], (hb.HbPushSchedule * (ctx.max_batch + 1))())
    assert n == launches
    assert not np.array_equal(outputs(want)[0], outputs(ref)[0])


def test_null_schedules_change_nothing():
    ctx = context()
    B, n_ticks = 6, 100
    rbd0 = start_states(ctx, B, seed=13)
    vels = cmd_vels(B)
    prm = params(5)
    _null_schedule_checks(ctx, lambda: device(ctx, rbd0, GAITS, vels, n_ticks, prm, 5), B, n_ticks * prm.period)
    ctx.close()


def test_continuation_independence_permutation_and_unscheduled_instances():
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=14)
    S = _schedules()
    other = hb.make_push_schedules(B, 0.08, 0.1, [[0.0, 50.0, 0.0]])
    other[2] = S[2]
    padded = hb.make_push_schedules(B, 0.05, 0.2, [40.0, 40.0, 0.0])
    for i in range(3, B):
        padded[i].n_push = 0
    # continuation split inside a push window (ticks 75..124, split at tick 100); first 3 instances pushed as in `padded`
    assert_setting_episodes(ctx, "pushes", rbd0, params(10), S, _one_push(B, 0, 0.1, 0.1, (70.0, -30.0, 0.0), (0.0, 2.0, 0.0)), other, 2,
                            hb.make_push_schedules(3, 0.05, 0.2, [40.0, 40.0, 0.0]), padded,
                            cont=hb.make_push_schedules(B, 0.15, 0.1, np.linspace(-60, 60, B)[:, None, None] * np.array([1.0, 0.5, 0.0]),
                                                        [0.0, 0.0, 3.0]))
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- estimated episodes
def test_pushed_estimated_episode_equals_the_stepwise_loop_bitwise():
    ctx = context()
    B, n_ticks, log_every = 6, 120, 10
    rbd0 = start_states(ctx, B, seed=11)
    vels = cmd_vels(B)
    prm = params(log_every)
    ep = est_params(seed=2024)
    S = _schedules()
    ctx.set_pushes(S)
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 40))
    r = stepwise(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 40), pushes=S)
    assert_episode_equal(d, r)
    ctx.close()


def test_estimated_episodes_null_schedules_independence_and_continuation():
    ctx = context()
    B, n_ticks = 6, 100
    rbd0 = start_states(ctx, B, seed=15)
    vels = cmd_vels(B)
    prm = params(5)
    ep = est_params(seed=77)

    def run(rbd=rbd0, gaits=GAITS, v=vels, est=None):
        return device(ctx, rbd, gaits, v, n_ticks, prm, 5, ep, est)

    _null_schedule_checks(ctx, run, B, n_ticks * prm.period)
    # only instance 2 pushed: its estimation stats change, every other instance is the unpushed run
    ctx.set_pushes(None)
    u = outputs(run())
    ctx.set_pushes(_one_push(B, 2, 0.06, 0.08, (-60.0, 50.0, 0.0), (0.0, 0.0, -3.0)))
    p = outputs(run())
    assert not np.array_equal(p[6][2], u[6][2]) and not np.array_equal(p[0][2], u[0][2])
    keep = [0, 1, 3, 4, 5]
    assert_episode_equal(p, u, rows_a=keep, rows_b=keep)
    # two calls split inside the push window equal one call
    assert_continues(ctx, rbd0, GAITS, vels, n_ticks, 50, prm, 5, ep)
    # a permuted batch, with its schedules and noise streams permuted, gives the permuted result
    perm = [3, 5, 0, 1, 4, 2]
    S = _schedules()
    ctx.set_pushes(S)
    full = outputs(run())
    ctx.set_pushes((hb.HbPushSchedule * B)(*[S[i] for i in perm]))
    est_p = hb.estimation_states(B)
    for j, i in enumerate(perm):
        est_p[j].noise_stream = i
    q = outputs(run(rbd=rbd0[perm], gaits=[GAITS[i] for i in perm], v=vels[perm], est=est_p))
    assert_episode_equal(full, q, rows_a=perm)
    # schedules for the first 2 instances only: the others run unpushed
    ctx.set_pushes(None)
    u = outputs(run())
    ctx.set_pushes(hb.make_push_schedules(2, 0.04, 0.1, [0.0, 60.0, 0.0]))
    part = outputs(run())
    assert_episode_equal(part, u, rows_a=slice(2, None), rows_b=slice(2, None))
    assert not np.array_equal(part[0][:2], u[0][:2])
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- argument checks
def test_argument_checks_return_before_any_launch():
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=2, device=0)
    lib = ctx._lib
    assert C.sizeof(hb.HbPushSchedule) == 264
    c0 = ctx.launch_count

    def sched(n=3, **change):
        S = hb.make_push_schedules(n, [0.1, 0.2], [0.05, 0.05], [[10.0, 0, 0], [0, 10.0, 0]])
        for field, (j, value) in change.items():
            if field in ("force", "torque"):
                getattr(S[1], field)[j][2] = value
            elif field == "n_push":
                S[1].n_push = value
            else:
                getattr(S[1], field)[j] = value
        return S

    assert lib.hb_rollout_set_pushes(None, 1, sched()) == -1
    assert lib.hb_rollout_set_pushes(ctx._h, -1, sched()) == -1
    assert lib.hb_rollout_set_pushes(ctx._h, 1, None) == -1
    nan, inf = float("nan"), float("inf")
    for field, j, value in (("n_push", 0, -1), ("n_push", 0, hb.HB_MAX_PUSHES + 1), ("t_start", 1, nan), ("t_start", 0, -inf), ("force", 0, nan),
                            ("force", 1, inf), ("torque", 1, nan), ("torque", 0, -inf), ("duration", 0, -0.01), ("duration", 1, nan),
                            ("duration", 0, inf)):
        assert lib.hb_rollout_set_pushes(ctx._h, 2, sched(**{field: (j, value)})) == -1, (field, j, value)
    assert lib.hb_rollout_set_pushes(ctx._h, 3, sched()) == -4
    assert lib.hb_rollout_set_pushes(ctx._h, 0, None) == 0 and lib.hb_rollout_set_pushes(ctx._h, 0, sched()) == 0
    # a push beyond the used count is not read: n_push = 1 with a NaN in the second slot is valid
    ok = sched(t_start=(1, nan)); ok[1].n_push = 1
    assert lib.hb_rollout_set_pushes(ctx._h, 2, ok) == 0
    assert lib.hb_rollout_set_pushes(ctx._h, 0, None) == 0

    prm = hb.default_sim_params()
    rbd = np.zeros((3, 32)); tau = np.zeros((3, 10)); w = np.zeros((3, 6))
    P = lambda a: C.c_void_p(a.ctypes.data)

    def step(h=ctx._h, B=1, p=prm, r=rbd, t=tau):
        return lib.hb_sim_step_wrench(h, B, None if p is None else C.byref(p), None if r is None else P(r), None if t is None else P(t), P(w), None, None)

    assert step(h=None) == -1 and step(B=-1) == -1 and step(p=None) == -1 and step(r=None) == -1 and step(t=None) == -1
    for field, value in (("dt", 0.0), ("dt", nan), ("substeps", 0), ("substeps", 1001)):
        bad = hb.default_sim_params()
        setattr(bad, field, value)
        assert step(p=bad) == -1, field
    assert step(B=3) == -4
    assert step(B=0) == 0
    assert ctx.launch_count == c0
    ctx.close()
