"""Odometry of the estimated episodes on the host (no GPU): the HbOdometrySetting mirror and make_odometry_settings, the numpy camera of
odometry_ref.py (history, the due rule, delay, drift, the Philox blocks 9 and 10), and its updateFromTopic against the oracle's kinematics."""
import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from estimation_ref import BLOCK, block_normals
from odometry_ref import BLOCK_DRIFT, BLOCK_POSITION, HISTORY, CameraRef, contact_positions_at, normals, update_from_topic


def test_make_odometry_settings_layout():
    s = hb.make_odometry_settings(4, [1, 5, 15, 0], delay_ticks=[0, 5, 15, 3], sigma_position=0.005, sigma_drift=[0.0, 0.0, 0.001, 0.0])
    assert len(s) == 4 and isinstance(s[0], hb.HbOdometrySetting)
    assert [x.period_ticks for x in s] == [1, 5, 15, 0] and [x.delay_ticks for x in s] == [0, 5, 15, 3]
    assert [x.sigma_position for x in s] == [0.005] * 4 and [x.sigma_drift for x in s] == [0.0, 0.0, 0.001, 0.0]
    assert hb.HB_ODOM_MAX_DELAY == 15 and HISTORY == hb.HB_ODOM_MAX_DELAY + 1
    none = hb.make_odometry_settings(3, 0)
    assert all(x.period_ticks == 0 and x.delay_ticks == 0 and x.sigma_position == 0.0 and x.sigma_drift == 0.0 for x in none)


@pytest.mark.parametrize("kw", [dict(period_ticks=-1), dict(delay_ticks=-1), dict(delay_ticks=16), dict(sigma_position=-1e-3),
                                dict(sigma_drift=np.nan), dict(sigma_position=np.inf), dict(period_ticks=1.5), dict(delay_ticks=[0, 1, 2]),
                                dict(period_ticks=2**32 + 5), dict(period_ticks=np.inf)],
                         ids=["negative_period", "negative_delay", "delay_above_max", "negative_sigma", "nan_drift", "inf_sigma", "fractional_period",
                              "wrong_shape", "period_beyond_int32", "inf_period"])
def test_make_odometry_settings_rejects(kw):
    args = dict(period_ticks=5)
    args.update(kw)
    with pytest.raises(ValueError):
        hb.make_odometry_settings(2, **args)


def _track(B, ticks, seed):
    rng = np.random.default_rng(seed)
    rbd = np.zeros((ticks, B, 32))
    rbd[:, :, 3:6] = np.cumsum(rng.normal(0.0, 1e-3, (ticks, B, 3)), axis=0) + [0.0, 0.0, 0.6]
    return rbd


def test_camera_due_rule_and_delay_without_noise():
    """With zero sigmas a message is due exactly on ticks a with a % period == 0 and a >= delay, and carries the position of tick a - delay;
    instances with period 0 and beyond the setting never have one."""
    periods, delays = [1, 5, 15, 3, 2, 0], [0, 5, 15, 2, 15, 4]
    B = len(periods) + 1
    s = hb.make_odometry_settings(len(periods), periods, delays)
    cam = CameraRef(s, B)
    ticks = 3 * HISTORY * 15
    track = _track(B, ticks, 1)
    for a in range(ticks):
        pos, has = cam.read(track[a], a, 7, np.arange(B))
        for i in range(B):
            want = i < len(periods) and periods[i] > 0 and a % periods[i] == 0 and a >= delays[i]
            assert has[i] == want, (i, a)
            if want:
                assert np.array_equal(pos[i], track[a - delays[i], i, 3:6])
            else:
                assert np.array_equal(pos[i], np.zeros(3))


def test_camera_noise_blocks_and_drift():
    """The position noise is sigma_position x block 10's normals and the bias a random walk of sigma_drift x block 9's, drawn per message
    from (seed, tick, stream) only; both blocks are new, after the sensors' blocks 0-8."""
    assert BLOCK_DRIFT > BLOCK["joint_velocity"] + 2 and BLOCK_POSITION == BLOCK_DRIFT + 1
    seed, streams = (3 << 32) + 11, np.array([4, 4, 9])
    s = hb.make_odometry_settings(3, 5, 2, sigma_position=[0.005, 0.0, 0.02], sigma_drift=[0.001, 0.001, 0.0])
    exact = CameraRef(hb.make_odometry_settings(3, 5, 2), 3)
    cam = CameraRef(s, 3)
    track = _track(3, 60, 2)
    walk = np.zeros((3, 3))
    for a in range(60):
        pos, has = cam.read(track[a], a, seed, streams)
        ref, ref_has = exact.read(track[a], a, seed, streams)
        assert np.array_equal(has, ref_has)
        if not has.any():
            continue
        for i in range(3):
            walk[i] += s[i].sigma_drift * normals(seed, BLOCK_DRIFT, a, streams[i])
            np.testing.assert_allclose(pos[i] - ref[i], walk[i] + s[i].sigma_position * normals(seed, BLOCK_POSITION, a, streams[i]), rtol=0, atol=1e-15)
    assert np.array_equal(normals(seed, BLOCK_DRIFT, 10, 4), np.array(block_normals(seed, 9, 10, 4)[:3]))
    assert not np.array_equal(normals(seed, BLOCK_DRIFT, 10, 4), normals(seed, BLOCK_POSITION, 10, 4))


def test_camera_clears_at_tick_zero():
    s = hb.make_odometry_settings(1, 1, 3, sigma_drift=0.01)
    cam = CameraRef(s, 1)
    track = _track(1, 20, 3)
    for a in range(20):
        cam.read(track[a], a, 1, [0])
    pos, has = cam.read(track[0], 0, 1, [0])
    assert has[0] == 0 and np.array_equal(cam.bias[0], np.zeros(3))
    assert np.array_equal(cam.hist[0, 1:], np.zeros((HISTORY - 1, 3))) and np.array_equal(cam.hist[0, 0], track[0, 0, 3:6])


def _estimates(B, seed):
    rng = np.random.default_rng(seed)
    rbd = np.zeros((B, 32))
    rbd[:, 0] = rng.uniform(-np.pi, np.pi, B); rbd[:, 1] = rng.uniform(-0.4, 0.4, B); rbd[:, 2] = rng.uniform(-0.4, 0.4, B)
    rbd[:, 3:6] = rng.normal(0.0, 0.5, (B, 3))
    rbd[:, 6:16] = rng.uniform(sc.JOINT_LOWER, sc.JOINT_UPPER, (B, 10))
    rbd[:, 16:32] = rng.normal(0.0, 0.5, (B, 16))
    return rbd


def test_update_from_topic_against_the_oracle_kinematics(oracle):
    """The fused feet are Pinocchio's contact positions at (pos, zyx, q) less the foot radius on z, restated as pos + the positions with the
    base at the origin (translation invariance, to rounding); feet heights move for the contact feet only; velocity and the estimated rbd
    beyond the position stay."""
    rng = np.random.default_rng(5)
    B = 16
    rbd = _estimates(B, 6)
    pos = rng.normal(0.0, 1.0, (B, 3))
    r = hb.default_kf_params().foot_radius
    for i in range(B):
        contact = [(i >> c) & 1 for c in range(4)]
        x0, h0 = rng.normal(0.0, 1.0, 18), rng.normal(0.0, 0.05, 4)
        fk = contact_positions_at(oracle, pos[i], rbd[i])
        at_origin = contact_positions_at(oracle, np.zeros(3), rbd[i])
        np.testing.assert_allclose(fk, np.tile(pos[i], 4) + at_origin, rtol=0, atol=1e-12 * (1 + np.abs(pos[i]).max()))
        x, h, rr = update_from_topic(x0, h0, rbd[i], pos[i], contact, r, fk)
        assert np.array_equal(x[0:3], pos[i]) and np.array_equal(x[3:6], x0[3:6])
        for c in range(4):
            assert np.array_equal(x[6 + 3 * c:8 + 3 * c], fk[3 * c:3 * c + 2]) and x[8 + 3 * c] == fk[3 * c + 2] - r
            assert h[c] == (x[8 + 3 * c] if contact[c] else h0[c])
        assert np.array_equal(rr[3:6], pos[i]) and np.array_equal(np.delete(rr, [3, 4, 5]), np.delete(rbd[i], [3, 4, 5]))
