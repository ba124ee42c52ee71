"""Simulated hardware records (no GPU): make_hardware_settings' defaults, broadcasting and errors, hb_default_hardware_setting against the
default episode, and the numpy sensor restatement on a record (hardware_ref.sensors_hw) in its documented order."""
import ctypes as C

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from estimation_ref import channel_normals, quat_zyx, sensors
from hardware_ref import sensors_hw
from hunter_bipedal_control_b200.scenarios import rot_zyx

SIGMAS = dict(orientation=0.002, angular_velocity=0.01, linear_acceleration=0.05, joint_position=0.001, joint_velocity=0.01)


def test_default_is_the_default_episode_without_noise():
    s = hb.default_hardware_setting()
    assert C.sizeof(hb.HbHardwareSetting) == 280
    p = hb.default_rollout_params()
    assert s.actuation_delay == p.actuation_delay == 0.009
    assert list(s.torque_limit) == list(p.torque_limit)
    sigmas = hb.HbHardwareSetting.sigma_orientation.offset
    assert bytes(s)[sigmas:] == bytes(280 - sigmas)              # every sigma and offset +0.0
    assert hb.load_library().hb_default_hardware_setting(None) == -1


def test_records_start_from_the_base():
    for r in hb.make_hardware_settings(3):
        assert bytes(r) == bytes(hb.default_hardware_setting())
    base = hb.default_hardware_setting(); base.actuation_delay = 0.02; base.gyro_bias[1] = 0.01
    s = hb.make_hardware_settings(2, base=base, sigma_joint_velocity=0.1)
    assert [r.actuation_delay for r in s] == [0.02, 0.02] and [r.gyro_bias[1] for r in s] == [0.01, 0.01]
    assert [r.sigma_joint_velocity for r in s] == [0.1, 0.1] and base.sigma_joint_velocity == 0.0


def test_scalars_broadcast_and_arrays_land_per_robot():
    B = 4
    tl = np.arange(B * 10, dtype=float).reshape(B, 10) + 1.0
    s = hb.make_hardware_settings(B, actuation_delay=[0.0, 0.004, 0.01, 0.03], sigma_orientation=0.003, torque_limit=tl,
                                  orientation_offset=[0.0, 0.01, -0.02], accel_bias=np.arange(B * 3, dtype=float).reshape(B, 3),
                                  encoder_offset=np.full(10, 0.002))
    for i, r in enumerate(s):
        assert r.actuation_delay == [0.0, 0.004, 0.01, 0.03][i] and r.sigma_orientation == 0.003
        assert np.array_equal(r.torque_limit[:], tl[i]) and list(r.orientation_offset) == [0.0, 0.01, -0.02]
        assert list(r.accel_bias) == [3.0 * i, 3.0 * i + 1, 3.0 * i + 2] and list(r.encoder_offset) == [0.002] * 10
        assert list(r.gyro_bias) == [0.0] * 3 and r.sigma_joint_position == 0.0
    s = hb.make_hardware_settings(B, torque_limit=np.full(10, 50.0))
    assert all(list(r.torque_limit) == [50.0] * 10 for r in s)


@pytest.mark.parametrize("kw", [dict(delay=0.01), dict(gyro_offset=[0.0, 0.0, 0.1]), dict(noise_orientation=0.1), dict(torque_limits=1.0)])
def test_unknown_names_raise(kw):
    with pytest.raises(ValueError, match="unknown field"):
        hb.make_hardware_settings(2, **kw)


@pytest.mark.parametrize("kw", [dict(actuation_delay=[0.0, 0.1, 0.2]), dict(torque_limit=np.ones(5)), dict(encoder_offset=np.ones((3, 10))),
                                dict(gyro_bias=[0.1, 0.2]), dict(accel_bias=np.ones((2, 4)))])
def test_shapes_that_do_not_broadcast_raise(kw):
    with pytest.raises(ValueError):
        hb.make_hardware_settings(2, **kw)


def test_exported():
    for name in ("hb_default_hardware_setting", "hb_rollout_set_hardware", "hb_actuation_hw", "hb_sim_read_sensors_hw"):
        assert name in hb.EXPORTED_SYMBOLS
        assert hasattr(hb.load_library(), name)


# ---------------------------------------------------------------------------------------------------------------- the restatement
def _rbd(seed):
    rng = np.random.default_rng(seed)
    r = rng.normal(0.0, 0.3, 32)
    r[2] = -0.0                           # a -0.0 roll: an offset of 0.0 keeps it
    r[8] = -0.0
    return r


def _noise(seed):
    n = hb.HbSensorNoise()
    n.seed = seed
    for k, v in SIGMAS.items():
        setattr(n, k, v)
    return n


def test_record_without_offsets_is_the_noisy_read_bitwise():
    """A record carrying the call's sigmas and zero offsets of either sign reads what sensors() reads with the call's noise, bit for bit."""
    rbd, prev = _rbd(1), np.array([0.1, -0.2, 0.05])
    hw = hb.make_hardware_settings(1, orientation_offset=[0.0, -0.0, -0.0], encoder_offset=np.r_[[-0.0] * 5, [0.0] * 5],
                                   **{"sigma_" + k: v for k, v in SIGMAS.items()})[0]
    want = sensors(rbd, prev, True, 0.002, _noise(77), tick=5, stream=3)
    got = sensors_hw(rbd, prev, True, 0.002, hw, seed=77, tick=5, stream=3)
    for a, b in zip(want, got):
        assert np.array_equal(a, b) and np.array_equal(np.signbit(a), np.signbit(b))
    clean = sensors_hw(rbd, prev, True, 0.002, hb.default_hardware_setting())
    assert np.signbit(clean[3][2]) and clean[3][2] == 0.0          # q_j[2] = rbd[8] = -0.0 stays -0.0
    for a, b in zip(sensors(rbd, prev, True, 0.002), clean):
        assert np.array_equal(a, b)


def test_offsets_come_before_the_noise():
    """Each reading is the true value, plus its offset (one addition), plus the record's sigma times the channel's normals."""
    rbd, prev = _rbd(2), np.array([0.0, 0.3, -0.1])
    off = dict(orientation_offset=[0.01, -0.02, 0.017], gyro_bias=[0.003, 0.0, -0.004], accel_bias=[0.2, -0.1, 0.0],
               encoder_offset=np.linspace(-0.01, 0.01, 10))
    hw = hb.make_hardware_settings(1, sigma_orientation=0.004, sigma_angular_velocity=0.02, sigma_linear_acceleration=0.0,
                                   sigma_joint_position=0.003, sigma_joint_velocity=0.05, **off)[0]
    seed, tick, stream = (3 << 32) + 9, 12, 41
    q, g, a, jp, jv = sensors_hw(rbd, prev, True, 0.002, hw, seed, tick, stream)
    R = rot_zyx(rbd[0:3])
    z = {ch: channel_normals(seed, ch, 3 if ch in ("orientation", "angular_velocity", "linear_acceleration") else 10, tick, stream) for ch in SIGMAS}
    ang = rbd[0:3] + np.where(np.asarray(off["orientation_offset"]) != 0.0, off["orientation_offset"], 0.0)
    np.testing.assert_array_equal(q, quat_zyx(ang + 0.004 * z["orientation"]))
    np.testing.assert_allclose(g, R.T @ rbd[16:19] + off["gyro_bias"] + 0.02 * z["angular_velocity"], rtol=0, atol=1e-15)
    acc = R.T @ ((rbd[19:22] - prev) / 0.002 + np.array([0.0, 0.0, 9.81]))
    np.testing.assert_allclose(a, acc + off["accel_bias"], rtol=0, atol=1e-12)           # sigma 0 draws nothing
    np.testing.assert_array_equal(jp, (rbd[6:16] + off["encoder_offset"]) + 0.003 * z["joint_position"])
    np.testing.assert_array_equal(jv, rbd[22:32] + 0.05 * z["joint_velocity"])        # the joint velocities get no offset
