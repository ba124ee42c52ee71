"""The simulated hardware (hb_rollout_set_hardware) restated for its tests (test_hardware_host.py, test_gpu_rollout_hardware.py, and
episode_ref.stepwise with `hardware`): the sensor read on a hardware record in numpy, and the record that restates a call's values."""
import hunter_bipedal_control_b200 as hb
from episode_ref import SIGMAS
from estimation_ref import channel_normals, quat_zyx, sensors


def add_offset(v, offset):
    """v + offset entry by entry, where an offset of exactly 0.0 (either sign) adds nothing: a -0.0 reading keeps its sign."""
    for k, o in enumerate(offset):
        if o != 0.0:
            v[k] += o


def sensors_hw(rbd, base_vel_prev, primed, accel_dt, hw, seed=0, tick=0, stream=0):
    """The readings of one instance on its hardware record hw (an HbHardwareSetting), in the documented order: the true value (as
    estimation_ref.sensors), plus the offset (ZYX angles, gyro, accelerometer, encoders; none on the joint velocities), plus hw's sigma
    times the channel's normals under the call's seed. Returns (quat, gyro, accel, joint_pos, joint_vel)."""
    _, gyro, acc, jp, jv = sensors(rbd, base_vel_prev, primed, accel_dt)
    ang = rbd[0:3].copy()
    for v, off in ((ang, hw.orientation_offset), (gyro, hw.gyro_bias), (acc, hw.accel_bias), (jp, hw.encoder_offset)):
        add_offset(v, off[:])
    for name, v in (("orientation", ang), ("angular_velocity", gyro), ("linear_acceleration", acc), ("joint_position", jp), ("joint_velocity", jv)):
        sigma = getattr(hw, "sigma_" + name)
        if sigma > 0:
            v += sigma * channel_normals(seed, name, len(v), tick, stream)
    return quat_zyx(ang), gyro, acc, jp, jv


def call_hardware(prm, ep=None):
    """The hardware record that restates a call's values: prm's actuation delay and torque limits, ep's noise sigmas (none without ep),
    no offsets."""
    h = hb.default_hardware_setting()
    h.actuation_delay = prm.actuation_delay
    h.torque_limit[:] = prm.torque_limit[:]
    if ep is not None:
        for k in SIGMAS:
            setattr(h, "sigma_" + k, getattr(ep.noise, k))
    return h
