"""numpy restatement of the estimated-episode pieces that are not the filter itself: the Philox4x32-10 sensor noise, the simulated sensors
(hb_sim_read_sensors) and the observation step's yaw unwrap. Shared by test_estimation_host.py and test_gpu_rollout_estimation.py."""
import math

import numpy as np

from hunter_bipedal_control_b200.scenarios import rot_zyx

M32 = 0xFFFFFFFF
# noise blocks of the channels (hb_rollout.cuh): 4 normals per block, each channel starts at its own block
BLOCK = {"orientation": 0, "angular_velocity": 1, "linear_acceleration": 2, "joint_position": 3, "joint_velocity": 6}


def philox4x32_10(key, ctr):
    """Philox4x32-10 (Salmon et al., SC'11): 4 words of counter `ctr` under the 2-word key."""
    k0, k1 = key[0] & M32, key[1] & M32
    c = [x & M32 for x in ctr]
    for r in range(10):
        if r:
            k0 = (k0 + 0x9E3779B9) & M32; k1 = (k1 + 0xBB67AE85) & M32
        p0 = 0xD2511F53 * c[0]; p1 = 0xCD9E8D57 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k0) & M32, p1 & M32, ((p0 >> 32) ^ c[3] ^ k1) & M32, p0 & M32]
    return c


def block_normals(seed, block, tick, stream):
    """The 4 normals of one noise block: u = (w + 0.5) 2^-32, Box-Muller on (u0, u1) and (u2, u3)."""
    w = philox4x32_10((seed & M32, seed >> 32), (block, tick & M32, stream & M32, (stream >> 32) & M32))
    out = []
    for h in range(2):
        u0 = (w[2 * h] + 0.5) * 2.0 ** -32; u1 = (w[2 * h + 1] + 0.5) * 2.0 ** -32
        r = math.sqrt(-2.0 * math.log(u0))
        out += [r * math.cos(2.0 * math.pi * u1), r * math.sin(2.0 * math.pi * u1)]
    return out


def channel_normals(seed, channel, n, tick, stream):
    """The n normals a channel adds sigma times to its n values."""
    z = []
    for b in range((n + 3) // 4):
        z += block_normals(seed, BLOCK[channel] + b, tick, stream)
    return np.array(z[:n])


def quat_zyx(zyx):
    """(x, y, z, w) of Rz(yaw) Ry(pitch) Rx(roll)."""
    hz, hy, hx = 0.5 * zyx[0], 0.5 * zyx[1], 0.5 * zyx[2]
    cz, sz, cy, sy, cx, sx = math.cos(hz), math.sin(hz), math.cos(hy), math.sin(hy), math.cos(hx), math.sin(hx)
    return np.array([cz * cy * sx - sz * sy * cx, cz * sy * cx + sz * cy * sx, sz * cy * cx - cz * sy * sx, cz * cy * cx + sz * sy * sx])


def sensors(rbd, base_vel_prev, primed, accel_dt, noise=None, tick=0, stream=0):
    """Noiseless (noise=None) or noisy readings of one instance: (quat, gyro, accel, joint_pos, joint_vel)."""
    R = rot_zyx(rbd[0:3])
    aw = (rbd[19:22] - base_vel_prev) / accel_dt if primed else np.zeros(3)
    ang, gyro, acc = rbd[0:3].copy(), R.T @ rbd[16:19], R.T @ (aw + np.array([0.0, 0.0, 9.81]))
    jp, jv = rbd[6:16].copy(), rbd[22:32].copy()
    if noise is not None:
        for name, v in (("orientation", ang), ("angular_velocity", gyro), ("linear_acceleration", acc), ("joint_position", jp), ("joint_velocity", jv)):
            sigma = getattr(noise, name)
            if sigma > 0:
                v += sigma * channel_normals(noise.seed, name, len(v), tick, stream)
    return quat_zyx(ang), gyro, acc, jp, jv


def shortest_angular_distance(a_from, a_to):
    """ROS angles: normalize_angle(to - from), normalize_angle_positive = fmod(fmod(a, 2 pi) + 2 pi, 2 pi)."""
    two_pi = 2.0 * math.pi
    a = math.fmod(math.fmod(a_to - a_from, two_pi) + two_pi, two_pi)
    if a > math.pi:
        a -= two_pi
    return a
