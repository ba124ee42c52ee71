"""State estimator (SURVEY 8f row N3) across its envelope: the batched Kalman filter (kf_update_kernel) against KalmanFilterRef over
contact patterns, attitudes, step sizes, parameters, feet heights, a long trot and batch shapes; the momentum observer
(contact_force_kernel) against ContactForceObserverRef near the knee angle where a foot's wrench matrix loses rank, across the joint
ranges, and against the closed form of its filter recursion."""
import ctypes as C
import os

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from oracle import hbo
from oracle import refs as R

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
EPS = np.finfo(np.float64).eps
KF_NS = C.sizeof(hb.HbKfState) // 8                  # doubles per filter state: x_hat 18, P 324, feet heights 4


def _kin(q, v):
    r = hbo.rbd(q, v)
    return r["cpos"], r["J"] @ v


def quat_from_zyx(zyx):
    """(B, 3) ZYX angles (yaw, pitch, roll) -> (B, 4) quaternions (x, y, z, w) of Rz Ry Rx."""
    cz, sz = np.cos(0.5 * zyx[:, 0]), np.sin(0.5 * zyx[:, 0])
    cy, sy = np.cos(0.5 * zyx[:, 1]), np.sin(0.5 * zyx[:, 1])
    cx, sx = np.cos(0.5 * zyx[:, 2]), np.sin(0.5 * zyx[:, 2])
    return np.stack([cz * cy * sx - sz * sy * cx, cz * sy * cx + sz * cy * sx, sz * cy * cx - cz * sy * sx, cz * cy * cx + sz * sy * sx], axis=1)


def kf_arrays(st):
    """(x_hat [B, 18], P [B, 18, 18]) copied out of a ctypes array of HbKfState."""
    a = np.frombuffer(st, dtype=np.float64).reshape(len(st), KF_NS)
    return a[:, :18].copy(), a[:, 18:342].reshape(-1, 18, 18).copy()


def kf_prm_dict(prm):
    """HbKfParams -> the restatement's parameter dict (the same seven values in the same order)."""
    return dict(zip(R.KF_PARAMS, (getattr(prm, f) for f, _ in hb.HbKfParams._fields_)))


def sensor_inputs(rng, zyx):
    """One step of IMU and encoder readings at the ZYX attitudes zyx (B, 3)."""
    B = zyx.shape[0]
    wl = rng.normal(0, 0.5, (B, 3)); al = rng.normal(0, 1.0, (B, 3)) + np.array([0, 0, 9.81])
    jpos = np.clip(R.DEFAULT_JOINTS + rng.normal(0, 0.1, (B, 10)), R.JOINT_LOWER, R.JOINT_UPPER); jvel = rng.normal(0, 0.5, (B, 10))
    return quat_from_zyx(zyx), wl, al, jpos, jvel


class KfRun:
    """B device filter states beside B restatements, checked after every step to the suite's tolerances: 1e-9 on rbd and x_hat, 1e-9
    relative on P, and P exactly symmetric."""

    def __init__(self, B, prm=None, heights=None):
        self.st = hb.kf_states(B); self.refs = [R.KalmanFilterRef() for _ in range(B)]
        self.prm = prm; self.rprm = kf_prm_dict(prm or hb.default_kf_params())
        if heights is not None:
            for i in range(B):
                self.st[i].feet_heights[:] = [float(h) for h in heights[i]]
                self.refs[i].heights = np.array(heights[i], dtype=float)

    def step(self, ctx, dt, quat, wl, al, jpos, jvel, flags):
        rbd = ctx.estimator_update(dt, self.st, quat, wl, al, jpos, jvel, flags, params=self.prm)
        x, P = kf_arrays(self.st)
        for i, ref in enumerate(self.refs):
            rr = ref.update(dt, quat[i], wl[i], al[i], jpos[i], jvel[i], flags[i], _kin, prm=self.rprm)
            assert np.abs(rbd[i] - rr).max() < 1e-9, (i, np.abs(rbd[i] - rr).max())
            assert np.abs(x[i] - ref.x).max() < 1e-9, (i, np.abs(x[i] - ref.x).max())
            assert np.abs(P[i] - ref.P).max() < 1e-9 * max(1.0, np.abs(ref.P).max()), (i, np.abs(P[i] - ref.P).max())
            assert np.array_equal(P[i], P[i].T)
        return rbd, x, P


def test_kf_all_contact_patterns(gpu_ctx):
    """All 16 contact-flag patterns, one per instance (pattern 0: no foot in contact, every noise term x 100; pattern 15: all in
    contact), each held for 50 steps, then permuted between the instances for 50 more."""
    rng = np.random.default_rng(31)
    B = 16
    flags = np.array([[(p >> c) & 1 for c in range(4)] for p in range(B)], dtype=np.uint8)
    run = KfRun(B)
    zyx = np.c_[rng.uniform(-np.pi, np.pi, B), rng.uniform(-0.3, 0.3, (B, 2))]
    for k in range(100):
        if k == 50:
            flags = flags[rng.permutation(B)]
            assert sorted(int(f @ [1, 2, 4, 8]) for f in flags) == list(range(16))
        run.step(gpu_ctx, 0.002, *sensor_inputs(rng, zyx + rng.normal(0, 1e-3, (B, 3))), flags)


def test_kf_attitude_envelope(gpu_ctx):
    """Yaw at 0, +-pi/2 and +-(pi - 1e-3), drifting across +-pi; pitch up to +-1.5 rad (1 / cos(pitch) ~ 14 in the Euler rates); roll up
    to +-1.2 rad."""
    rng = np.random.default_rng(32)
    yaw = [0.0, np.pi / 2, -np.pi / 2, np.pi - 1e-3, -(np.pi - 1e-3)]
    pitch = [-1.5, -0.8, 0.0, 0.8, 1.5]
    roll = [-1.2, 0.0, 1.2]
    zyx0 = np.array([(z, y, x) for z in yaw for y in pitch for x in roll])
    B = zyx0.shape[0]
    drift = np.zeros((B, 3)); drift[:, 0] = np.where(np.abs(zyx0[:, 0]) > 3.0, np.sign(zyx0[:, 0]) * 4e-4, 0.0)   # across +-pi
    run = KfRun(B)
    flags = (rng.uniform(size=(B, 4)) > 0.3).astype(np.uint8)
    crossed = np.zeros(B, dtype=bool)
    for k in range(10):
        zyx = zyx0 + k * drift
        rbd, _, _ = run.step(gpu_ctx, 0.002, *sensor_inputs(rng, zyx), flags)
        crossed |= np.sign(rbd[:, 0]) != np.sign(zyx0[:, 0])
        np.testing.assert_allclose(rbd[:, 1:3], zyx[:, 1:3], rtol=0, atol=1e-12)
    assert crossed[np.abs(zyx0[:, 0]) > 3.0].all()          # every yaw near +-pi has wrapped to the other side


def test_kf_quaternion_sign_is_exact(gpu_ctx):
    """q and -q are one rotation; every term of the angle conversion is a product of two components, so the outputs and states are
    bitwise equal."""
    rng = np.random.default_rng(33)
    B = 48
    a, b = hb.kf_states(B), hb.kf_states(B)
    flags = (rng.uniform(size=(B, 4)) > 0.4).astype(np.uint8)
    for k in range(6):
        zyx = np.c_[rng.uniform(-np.pi, np.pi, B), rng.uniform(-1.5, 1.5, B), rng.uniform(-1.2, 1.2, B)]
        quat, wl, al, jpos, jvel = sensor_inputs(rng, zyx)
        ra = gpu_ctx.estimator_update(0.002, a, quat, wl, al, jpos, jvel, flags)
        rb = gpu_ctx.estimator_update(0.002, b, -quat, wl, al, jpos, jvel, flags)
        assert np.array_equal(ra, rb)
        assert bytes(a) == bytes(b)


@pytest.mark.parametrize("dt", [0.0005, 0.001, 0.002, 0.01, 0.02])
def test_kf_step_sizes(gpu_ctx, dt):
    rng = np.random.default_rng(int(dt * 1e5))
    B = 12
    run = KfRun(B)
    zyx = np.c_[rng.uniform(-np.pi, np.pi, B), rng.uniform(-0.5, 0.5, (B, 2))]
    for k in range(15):
        flags = (rng.uniform(size=(B, 4)) > 0.3).astype(np.uint8)
        run.step(gpu_ctx, dt, *sensor_inputs(rng, zyx), flags)


def _kf_param_sets():
    base = hb.default_kf_params()
    variant = hb.HbKfParams(*hb.parse_task_info(os.path.join(HERE, "golden", "task_wbc_variant.info")).kalman)
    out = {"default": base, "task_wbc_variant": variant}
    for s in (0.1, 10.0):                               # every noise value scaled, the foot radius kept
        out["noise_x%g" % s] = hb.HbKfParams(base.foot_radius, *[getattr(base, f) * s for f, _ in hb.HbKfParams._fields_[1:]])
    return out


@pytest.mark.parametrize("name", ["default", "task_wbc_variant", "noise_x0.1", "noise_x10"])
def test_kf_parameters(gpu_ctx, name):
    """The same hb_kf_params on the device and in the restatement: the defaults, the kalman block of a task.info variant, and every noise
    value scaled x0.1 and x10."""
    prm = _kf_param_sets()[name]
    if name == "task_wbc_variant":
        assert [getattr(prm, f) for f, _ in hb.HbKfParams._fields_] != [getattr(hb.default_kf_params(), f) for f, _ in hb.HbKfParams._fields_]
    rng = np.random.default_rng(34)
    B = 12
    run = KfRun(B, prm=prm)
    zyx = np.c_[rng.uniform(-np.pi, np.pi, B), rng.uniform(-0.5, 0.5, (B, 2))]
    for k in range(20):
        flags = (rng.uniform(size=(B, 4)) > 0.3).astype(np.uint8)
        run.step(gpu_ctx, 0.002, *sensor_inputs(rng, zyx), flags)


def test_kf_feet_heights(gpu_ctx):
    """Non-zero feet heights in the filter state enter the height rows of the innovation, in the device filter as in the restatement."""
    rng = np.random.default_rng(35)
    B = 16
    heights = rng.uniform(-0.15, 0.15, (B, 4))
    run = KfRun(B, heights=heights)
    zyx = np.c_[rng.uniform(-np.pi, np.pi, B), rng.uniform(-0.3, 0.3, (B, 2))]
    for k in range(20):
        flags = (rng.uniform(size=(B, 4)) > 0.3).astype(np.uint8)
        run.step(gpu_ctx, 0.002, *sensor_inputs(rng, zyx), flags)
    np.testing.assert_array_equal(np.frombuffer(run.st, dtype=np.float64).reshape(B, KF_NS)[:, 342:], heights)   # the filter keeps them


def test_kf_long_trot(gpu_ctx):
    """5 s at 500 Hz with the feet switching like a trot (one foot's two contact points, then the other's, with short double-support
    phases), yaw turning across +-pi: every step against the restatement, P exactly symmetric with its smallest eigenvalue >= -1e-9 |P|,
    and the decoupling of the xy position (LinearKalmanFilter.cpp:151-156) taken on some steps and not on others."""
    rng = np.random.default_rng(36)
    B, steps, dt, period = 4, 2500, 0.002, 0.6
    run = KfRun(B)
    phase = np.arange(B) * period / B
    yaw0 = rng.uniform(-np.pi, np.pi, B)
    decoupled = np.zeros((steps, B), dtype=bool)
    for k in range(steps):
        t = k * dt
        s = ((t + phase) % period) / period
        fa, fb = (s < 0.55) | (s > 0.95), s > 0.45          # foot a: contacts 0 and 2, foot b: contacts 1 and 3
        flags = np.stack([fa, fb, fa, fb], axis=1).astype(np.uint8)
        zyx = np.c_[yaw0 + 1.5 * t, 0.1 * np.sin(2 * np.pi * t / period + phase), 0.05 * np.cos(2 * np.pi * t / period + phase)]
        zyx[:, 0] = (zyx[:, 0] + np.pi) % (2 * np.pi) - np.pi
        quat, wl, al, jpos, jvel = sensor_inputs(rng, zyx)
        jpos = np.clip(R.DEFAULT_JOINTS + 0.2 * np.sin(2 * np.pi * t / period + phase[:, None] + np.arange(10)), R.JOINT_LOWER, R.JOINT_UPPER)
        _, _, P = run.step(gpu_ctx, dt, quat, wl, al, jpos, jvel, flags)
        for i in range(B):
            ev = np.linalg.eigvalsh(P[i])
            assert ev.min() >= -1e-9 * np.abs(ev).max(), (k, i, ev.min())
            decoupled[k, i] = run.refs[i].decoupled
    for i in range(B):
        assert decoupled[:, i].any() and not decoupled[:, i].all(), (i, decoupled[:, i].sum())
        assert decoupled[1:, i].any()                       # not only the first step, where P = 100 I


def test_kf_batch_shapes(gpu_ctx):
    """B = 1, 31, 32, 33 and max_batch against the restatement; an instance alone is bitwise equal to itself in a batch of 37, and
    permuting the instances permutes the results."""
    rng = np.random.default_rng(37)
    for B in (1, 31, 32, 33, gpu_ctx.max_batch):
        run = KfRun(B)
        zyx = np.c_[rng.uniform(-np.pi, np.pi, B), rng.uniform(-0.5, 0.5, (B, 2))]
        for k in range(2):
            run.step(gpu_ctx, 0.002, *sensor_inputs(rng, zyx), (rng.uniform(size=(B, 4)) > 0.3).astype(np.uint8))
    B, steps = 37, 3
    zyx = np.c_[rng.uniform(-np.pi, np.pi, B), rng.uniform(-1.0, 1.0, (B, 2))]
    ins = [sensor_inputs(rng, zyx) + ((rng.uniform(size=(B, 4)) > 0.3).astype(np.uint8),) for _ in range(steps)]
    st = hb.kf_states(B)
    out = [gpu_ctx.estimator_update(0.002, st, *x) for x in ins]
    full = np.frombuffer(st, dtype=np.float64).reshape(B, KF_NS).copy()
    for i in (0, 17, 31, 32, 36):
        s1 = hb.kf_states(1)
        for k, x in enumerate(ins):
            r1 = gpu_ctx.estimator_update(0.002, s1, *[a[i:i + 1] for a in x])
            assert np.array_equal(r1[0], out[k][i])
        assert np.array_equal(np.frombuffer(s1, dtype=np.float64), full[i])
    perm = rng.permutation(B)
    sp = hb.kf_states(B)
    for k, x in enumerate(ins):
        rp = gpu_ctx.estimator_update(0.002, sp, *[a[perm] for a in x])
        assert np.array_equal(rp, out[k][perm])
    assert np.array_equal(np.frombuffer(sp, dtype=np.float64).reshape(B, KF_NS), full[perm])


# ---- momentum observer and per-foot wrench --------------------------------------------------------------------------------------

def _q_of(rbd):
    """Generalised coordinates [p, zyx, q_j] of an rbd state, as the restatement forms them."""
    return np.concatenate([rbd[3:6], rbd[0:3], rbd[6:16]])


def _base_rbd(rng, B):
    x = sc.random_initial_states(B, seed=int(rng.integers(1 << 30)))
    rbd = sc.consistent_rbd(x)
    rbd[:, 16:32] = rng.uniform(-1.0, 1.0, (B, 16))
    return rbd


def _wrench_check(rbd, est, dist, legs=(0, 1)):
    """The device wrench of each instance and leg against the least-norm solution pinv(A) b of the oracle's A = S J' and the device's
    own disturbance b (the solve isolated): |w_dev - w| <= 100 cond(A) eps max|w| and |A w_dev - b| <= 100 eps |A| |w_dev|; the
    norms in entries 12-15 are those of w_dev. Returns (worst deviation / bound, worst residual / bound, cond(A)) per (instance, leg)."""
    out = []
    for i in range(rbd.shape[0]):
        q = _q_of(rbd[i])
        for leg in legs:
            A = R.foot_wrench_matrix(q, leg)
            b = dist[i, 6 + 5 * leg:11 + 5 * leg]
            w = np.linalg.pinv(A) @ b
            wd = est[i, 6 * leg:6 * leg + 6]
            cond = np.linalg.cond(A)
            dev = np.abs(wd - w).max() / (100.0 * cond * EPS * np.abs(w).max())
            res = np.abs(A @ wd - b).max() / (100.0 * EPS * np.linalg.norm(A, 2) * np.linalg.norm(wd))
            assert abs(est[i, 12 + leg] - np.linalg.norm(wd[:3])) <= 4 * EPS * est[i, 12 + leg]
            assert abs(est[i, 14 + leg] - np.linalg.norm(wd)) <= 4 * EPS * est[i, 14 + leg]
            out.append((dev, res, cond))
    return np.array(out)


def test_observer_wrench_near_singular_knee(gpu_ctx):
    """Each leg's S J' loses rank at one knee angle k* inside the knee's limits (the hip-pitch, knee and ankle origins in line), where
    cond(A) grows like 1.8 / |knee - k*|. At knee = k* +- delta, random hip pitch and ankle, either leg, the wrench must stay within the
    error of a backward-stable least-norm solve."""
    rng = np.random.default_rng(41)
    kstar = [R.singular_knee(leg, _q_of(sc.consistent_rbd(sc.INITIAL_STATE[None])[0])) for leg in (0, 1)]
    deltas = [1e-2, 1e-3, 1e-4, 1e-5, 1e-6]
    per, B = 12, 12 * len(deltas)
    rbd = _base_rbd(rng, B)
    leg_of = np.arange(B) % 2
    for n, d in enumerate(deltas):
        for j in range(per):
            i = n * per + j; leg = leg_of[i]; o = 6 + 5 * leg
            rbd[i, o + 2] = rng.uniform(R.JOINT_LOWER[5 * leg + 2], R.JOINT_UPPER[5 * leg + 2])       # hip pitch
            rbd[i, o + 3] = kstar[leg] + (d if j % 2 else -d)                                            # knee
            rbd[i, o + 4] = rng.uniform(R.JOINT_LOWER[5 * leg + 4], R.JOINT_UPPER[5 * leg + 4])       # ankle
    tau = rng.uniform(-20, 20, (B, 10))
    est, dist = gpu_ctx.contact_force_estimate(0.002, hb.observer_states(B), rbd, tau, 250.0)
    worst = []
    for n, d in enumerate(deltas):
        sl = slice(n * per, (n + 1) * per)
        r = _wrench_check(rbd[sl], est[sl], dist[sl], legs=(0, 1)).reshape(per, 2, 3)
        near = r[np.arange(per), leg_of[sl]]                  # the leg at k* +- delta
        assert near[:, 2].min() > 0.1 / d                     # the sweep reaches the conditioning it is meant to
        worst.append((d, r[..., 0].max(), r[..., 1].max(), near[:, 2].max()))
    for d, dev, res, cond in worst:
        print("knee - k* = +-%g: cond(A) up to %.2e, worst |w_dev - w| / bound %.3g, worst residual / bound %.3g" % (d, cond, dev, res))
    assert all(dev <= 1.0 and res <= 1.0 for _, dev, res, _ in worst), worst


def test_observer_joint_range(gpu_ctx):
    """A grid over each joint's [lower, upper] (the others at their defaults) and random joint vectors over the whole box, moderate base
    poses, three steps: the disturbance and the filter state to 1e-9 relative of the restatement, the wrench under the cond-scaled bound."""
    rng = np.random.default_rng(42)
    grid = []
    for j in range(10):
        for val in np.linspace(R.JOINT_LOWER[j], R.JOINT_UPPER[j], 7):
            qj = np.array(R.DEFAULT_JOINTS, dtype=float); qj[j] = val; grid.append(qj)
    grid += list(rng.uniform(R.JOINT_LOWER, R.JOINT_UPPER, (30, 10)))
    qj = np.array(grid); B = qj.shape[0]
    rbd = _base_rbd(rng, B); rbd[:, 6:16] = qj
    st = hb.observer_states(B)
    refs = [R.ContactForceObserverRef(250.0) for _ in range(B)]
    for k in range(3):
        rbd[:, 16:32] = rng.uniform(-1.0, 1.0, (B, 16))
        tau = rng.uniform(-20, 20, (B, 10))
        est, dist = gpu_ctx.contact_force_estimate(0.002, st, rbd, tau, 250.0)
        pf = np.frombuffer(st, dtype=np.float64).reshape(B, 16)
        for i in range(B):
            refs[i].update(rbd[i], tau[i], 0.002)
            s = max(1.0, np.abs(refs[i].disturbance).max())
            assert np.abs(dist[i] - refs[i].disturbance).max() < 1e-9 * s, (k, i)
            assert np.abs(pf[i] - refs[i].last).max() < 1e-9 * s, (k, i)
        r = _wrench_check(rbd, est, dist)
        assert r[:, 0].max() <= 1.0 and r[:, 1].max() <= 1.0, (k, r[:, 0].max(), r[:, 1].max())


@pytest.mark.parametrize("lam", [10.0, 250.0, 1000.0])
@pytest.mark.parametrize("dt", [1.0, 1.0 + 2.0 ** -40])
def test_observer_recursion_closed_form(gpu_ctx, lam, dt):
    """At v = 0 (p = M v = 0, C'v = 0) and a fixed tau the observer is a first-order low-pass of g - S' tau: after k steps from reset the
    disturbance is (1 - gamma^k)(g - S' tau), gamma = exp(-lambda dt). dt = 1 s is used as given, anything longer is replaced by 2 ms
    (StateEstimateBase.cpp:133-134)."""
    rng = np.random.default_rng(43)
    B = 6
    rbd = _base_rbd(rng, B); rbd[:, 16:32] = 0.0
    tau = rng.uniform(-20, 20, (B, 10))
    dt_used = dt if dt <= 1.0 else 0.002
    gamma = np.exp(-lam * dt_used)
    st = hb.observer_states(B)
    target = np.array([hbo.observer_terms(_q_of(rbd[i]), np.zeros(16))[1] - np.r_[np.zeros(6), tau[i]] for i in range(B)])
    for k in range(1, 9):
        est, dist = gpu_ctx.contact_force_estimate(dt, st, rbd, tau, lam)
        if gamma == 0.0:
            # lambda dt past exp's range: gamma underflows, beta = (1 - gamma) / (gamma dt) is infinite and beta p = inf * 0, so the
            # reference's disturbance is NaN; the kernel computes the same formula
            with np.errstate(divide="ignore", invalid="ignore"):
                ref = R.ContactForceObserverRef(lam); ref.update(rbd[0], tau[0], dt)
            assert np.isnan(ref.disturbance).all() and np.isnan(dist).all()
            return
        expect = (1.0 - gamma ** k) * target
        for i in range(B):
            assert np.abs(dist[i] - expect[i]).max() <= 1e-12 * np.abs(expect[i]).max(), (k, i, np.abs(dist[i] - expect[i]).max())


def test_observer_null_disturbance_dev():
    """hb_contact_force_estimate_batch_dev with a null disturbance_torque: the estimates and observer states are bitwise those of a call
    that writes the disturbance."""
    import torch
    ctx = hb.Context(horizon_N=10, dt=0.02, max_batch=64, device=0)
    try:
        rng = np.random.default_rng(44)
        B = 37
        P = lambda t: C.c_void_p(t.data_ptr())
        st0 = np.frombuffer(hb.observer_states(B), dtype=np.uint8).copy()
        sa, sb = torch.from_numpy(st0.copy()).cuda(), torch.from_numpy(st0.copy()).cuda()
        ea, eb = (torch.zeros((B, 16), dtype=torch.float64, device="cuda") for _ in range(2))
        dist = torch.zeros((B, 16), dtype=torch.float64, device="cuda")
        lib = hb.load_library()
        for k in range(4):
            rbd = torch.from_numpy(_base_rbd(rng, B)).cuda(); tau = torch.from_numpy(rng.uniform(-20, 20, (B, 10))).cuda()
            assert lib.hb_contact_force_estimate_batch_dev(ctx._h, B, C.c_double(250.0), C.c_double(0.002), P(sa), P(rbd), P(tau), P(ea), P(dist)) == 0
            assert lib.hb_contact_force_estimate_batch_dev(ctx._h, B, C.c_double(250.0), C.c_double(0.002), P(sb), P(rbd), P(tau), P(eb), None) == 0
            torch.cuda.synchronize()
            assert torch.equal(ea, eb) and torch.equal(sa, sb)
            assert torch.isfinite(dist).all() and (dist != 0).any()
    finally:
        ctx.close()
