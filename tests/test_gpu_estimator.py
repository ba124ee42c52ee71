"""State estimator (SURVEY 8f row N3): batched linear Kalman filter against the dense restatement of LinearKalmanFilter.cpp."""
import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from oracle import refs as R

pytestmark = pytest.mark.gpu


def _kin(oracle):
    def kin(q, v):
        r = oracle.rbd(q, v)
        return r["cpos"], r["J"] @ v
    return kin


def test_kalman_filter_tracks_restatement(oracle):
    ctx = hb.Context(horizon_N=20, dt=0.02, max_batch=64, device=0)
    B, steps, dt = 24, 12, 0.002
    rng = np.random.default_rng(12)
    st = hb.kf_states(B)
    ref = [R.KalmanFilterRef() for _ in range(B)]
    kin = _kin(oracle)
    jpos0 = np.clip(R.DEFAULT_JOINTS + rng.normal(0, 0.1, (B, 10)), R.JOINT_LOWER, R.JOINT_UPPER)
    for k in range(steps):
        ang = rng.normal(0, 0.2, (B, 3))
        quat = np.zeros((B, 4))
        for i in range(B):                      # small random orientation: quaternion (x, y, z, w)
            v = 0.5 * ang[i] * 0.3
            quat[i] = np.array([v[0], v[1], v[2], np.sqrt(1 - v @ v)])
        wl = rng.normal(0, 0.5, (B, 3)); al = rng.normal(0, 1.0, (B, 3)) + np.array([0, 0, 9.81])
        jpos = jpos0 + 0.01 * k; jvel = rng.normal(0, 0.5, (B, 10))
        flags = (rng.uniform(size=(B, 4)) > 0.3).astype(np.uint8)
        rbd = ctx.estimator_update(dt, st, quat, wl, al, jpos, jvel, flags)
        for i in range(B):
            rr = ref[i].update(dt, quat[i], wl[i], al[i], jpos[i], jvel[i], flags[i], kin)
            np.testing.assert_allclose(rbd[i], rr, rtol=0, atol=1e-9)
            np.testing.assert_allclose(np.array(st[i].x_hat[:]), ref[i].x, rtol=0, atol=1e-9)
            P = np.array(st[i].P[:]).reshape(18, 18)
            assert np.abs(P - ref[i].P).max() < 1e-9 * max(1.0, np.abs(ref[i].P).max())
            assert np.array_equal(P, P.T)
            if k == 0:      # first update: P = 100 I makes the xy determinant test of the reference fire (:151-156)
                assert np.all(P[0:2, 2:] == 0.0) and np.all(P[2:, 0:2] == 0.0)
    ctx.close()


def test_contact_force_observer_tracks_restatement(gpu_ctx):
    """Momentum observer + per-foot least-norm wrench (StateEstimateBase::estContactForce) over a sequence of measurements: the filter
    state, the disturbance torque and the 16 estimates against the restatement (different derivation of C'v, SVD solve)."""
    from hunter_bipedal_control_b200 import scenarios as sc
    B, steps = 20, 6
    rng = np.random.default_rng(21)
    st = hb.observer_states(B)
    ref = [R.ContactForceObserverRef(250.0) for _ in range(B)]
    x = sc.random_initial_states(B, seed=77)
    for k in range(steps):
        rbd = sc.consistent_rbd(x, rng, 0.03)
        rbd[:, 16:32] = rng.uniform(-1.0, 1.0, (B, 16))
        tau = rng.uniform(-20, 20, (B, 10))
        dt = 0.002 if k != 3 else 5.0              # dt > 1 s is replaced by 2 ms (:133-134)
        est, dist = gpu_ctx.contact_force_estimate(dt, st, rbd, tau, 250.0)
        for i in range(B):
            e = ref[i].update(rbd[i], tau[i], dt)
            sc_ = max(1.0, np.abs(ref[i].disturbance).max())
            assert np.abs(dist[i] - ref[i].disturbance).max() < 1e-9 * sc_
            assert np.abs(np.array(st[i].p_filtered[:]) - ref[i].last).max() < 1e-9 * sc_
            assert np.abs(est[i] - e).max() < 1e-7 * max(1.0, np.abs(e).max())
    # the settled filter is pinned by its closed form in test_gpu_estimator_envelope.py::test_observer_recursion_closed_form
