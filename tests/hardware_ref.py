"""The simulated hardware (hb_rollout_set_hardware) restated for its tests (test_hardware_host.py, test_gpu_rollout_hardware.py): the sensor
read on a hardware record in numpy, the record that restates a call's values, and a context wrapper that turns episode_ref.stepwise into
the loop of public calls of an episode with the setting."""
import numpy as np

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


def unclipped(prm):
    """A copy of prm whose torque limits clip nothing (np.clip to +-inf returns its input bit for bit): the params of episode_ref.stepwise
    on a HardwareLoop, which clips per robot itself."""
    p = hb.HbRolloutParams.from_buffer_copy(bytes(prm))
    p.torque_limit[:] = [np.inf] * hb.NJ
    return p


class HardwareLoop:
    """A context whose read_sensors and actuation restate the simulated hardware of the episodes with public calls, for episode_ref.stepwise
    (run with unclipped(prm)): the records `hardware` set on ctx, padded beyond them with the call's values (call_hardware(prm, ep), prm and
    ep those of the episode call). read_sensors is hb_sim_read_sensors_hw on the records; actuation is hb_actuation_hw on them, the delay
    stepwise passes being each record's, and then each robot's torques clipped to its record's limits as rollout_saturate_kernel clips
    them. Everything else is the wrapped context's (which may itself be a wrapper)."""

    def __init__(self, ctx, hardware, prm, ep=None):
        self._ctx, self._hardware, self._call = ctx, hardware, call_hardware(prm, ep)

    def __getattr__(self, name):
        return getattr(self._ctx, name)

    def _records(self, B):
        return (hb.HbHardwareSetting * B)(*[self._hardware[i] if i < len(self._hardware) else self._call for i in range(B)])

    def read_sensors(self, rbd, est, tick, noise=None, accel_dt=0.002):
        return self._ctx.read_sensors(rbd, est, tick, noise, accel_dt=accel_dt, hardware=self._records(rbd.shape[0]))

    def actuation(self, time, state, command, rbd, delay=0.009):
        hw = self._records(rbd.shape[0])
        tau = self._ctx.actuation(time, state, command, rbd, delay, hardware=hw)
        lim = np.array([h.torque_limit[:] for h in hw])
        return np.clip(tau, -lim, lim)
