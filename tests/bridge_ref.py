"""The motor bridge (hb_motor_bridge, hunter_b200.h) restated for its tests (test_motor_bridge_host.py, test_gpu_rollout_motor_bridge.py):
the protocol's codes in numpy float32, one rounded operation at a time, the frame maps and the motor PD; the bridged plant step on
episode_ref's numpy plant; and BridgeLoop, under which episode_ref.stepwise runs the bridged robots through the public calls."""
import ctypes as C

import numpy as np

from episode_ref import plant_numpy

F = np.float32
BITS = {"pos": 16, "vel": 12, "kp": 12, "kd": 9, "ff": 12}


def value(x, lo, hi, bits, quantise):
    """One value through the protocol on [lo, hi]: with quantise, rounded to float32, clamped, encoded with truncation (NaN: code 0) and
    decoded; without, clamped in double (NaN passes)."""
    x = float(x)
    if not quantise:
        return hi if x > hi else (lo if x < lo else x)
    flo, fhi, n = F(lo), F(hi), F((1 << bits) - 1)
    span = fhi - flo
    with np.errstate(over="ignore", invalid="ignore"):
        f = F(x)
    f = fhi if f > fhi else (flo if f < flo else f)
    code = 0 if np.isnan(f) else int(((f - flo) * n) / span)
    return float(F(F(F(code) * span) / n) + flo)


def code(x, lo, hi, bits):
    """The protocol's code of x (quantise = 1)."""
    flo, fhi, n = F(lo), F(hi), F((1 << bits) - 1)
    with np.errstate(over="ignore", invalid="ignore"):
        f = F(x)
    f = fhi if f > fhi else (flo if f < flo else f)
    return 0 if np.isnan(f) else int(((f - flo) * n) / (fhi - flo))


def command(r, j, c):
    """Joint j's hybrid command c = (posDes, velDes, kp, kd, ff) -> the decoded motor command (pos, vel, kp, kd, ff) of record r."""
    s, d, z, qz = r.command_scale[j], float(r.direction[j]), r.zero[j], r.quantise == 1
    return np.array([value(d * c[0] + z, -r.pos_max[j], r.pos_max[j], 16, qz), value(d * c[1], -r.vel_max[j], r.vel_max[j], 12, qz),
                     value(s * c[2], 0.0, r.kp_max[j], 12, qz), value(s * c[3], 0.0, r.kd_max[j], 9, qz),
                     value(s * c[4] * d, -r.ff_max[j], r.ff_max[j], 12, qz)])


def feedback(r, j, q, qd):
    """Joint j's readings (q, qd) through the encoders of record r: motor frame, protocol, joint frame (float32 with quantise)."""
    d, z, qz = float(r.direction[j]), r.zero[j], r.quantise == 1
    p = value(d * q + z, -r.pos_max[j], r.pos_max[j], 16, qz)
    v = value(d * qd, -r.vel_max[j], r.vel_max[j], 12, qz)
    if qz:
        return float((F(p) - F(z)) * F(d)), float(F(v) * F(d))
    return (p - z) * d, v * d


def commands(bridges, cmd):
    """command() over a batch: cmd (B, 10, 5) -> (B, 10, 5)."""
    return np.array([[command(bridges[i], j, cmd[i, j]) for j in range(10)] for i in range(len(cmd))])


def motor_torque(r, j, m, q, qd, lim):
    """The torque joint j receives from its motor at joint state (q, qd): the hybrid PD on the decoded command m in the motor frame, back
    to the joint frame, clipped to +-lim."""
    d = float(r.direction[j])
    t = d * (m[2] * (m[0] - (d * q + r.zero[j])) + m[3] * (m[1] - d * qd) + m[4])
    return -lim if t < -lim else (lim if t > lim else t)


def plant_bridged(oracle, rbd, prm, bridge, mcmd, lim, variation=None):
    """One bridged plant step of one robot on episode_ref.plant_numpy: on every substep the motor's torques (motor_torque of the record
    bridge, the decoded command mcmd (10, 5), the limits lim (10,)) at that substep's joint state, held over the substep. Returns (rbd_next,
    contact forces and flags of the last substep, the mean over the substeps of the clipped torques (10,))."""
    from hunter_bipedal_control_b200 import HbSimParams
    sub = HbSimParams.from_buffer_copy(bytes(prm))
    sub.dt, sub.substeps = prm.dt / prm.substeps, 1               # the substep of prm: the same h = dt / substeps
    applied = np.zeros(10)
    for _ in range(prm.substeps):
        t = np.array([motor_torque(bridge, j, mcmd[j], rbd[6 + j], rbd[22 + j], lim[j]) for j in range(10)])
        applied += t
        rbd, F, flags = plant_numpy(oracle, rbd, t, sub, variation=variation)
    return rbd, F, flags, applied / prm.substeps


def _rows(records, lo, hi):
    """Records lo .. hi - 1 of a ctypes array, in place (None stays None)."""
    if records is None:
        return None
    T = records._type_
    return (T * (hi - lo)).from_buffer(records, lo * C.sizeof(T))


class BridgeLoop:
    """The context episode_ref.stepwise runs on to restate an episode with a motor bridge set: the robots with a record (the first
    len(bridges)) read their sensors, run their actuation and step the plant through the calls with bridge=, the others through the
    calls without; every other call goes to ctx. The plant step clips a bridged robot to its limit (the hardware record's, when the
    actuation got records, else default_limit) and writes the mean applied torque into its rows of the torque array it is passed, the
    array whose maxima stepwise counts, as the episode counts the plant's mean."""

    def __init__(self, ctx, bridges, default_limit):
        self._ctx, self._bridges = ctx, bridges
        self._default = np.array(default_limit[:])
        self._mcmd = self._lim = None

    def __getattr__(self, name):
        return getattr(self._ctx, name)

    def _groups(self, B):
        nb = min(len(self._bridges), B)
        return [(lo, hi, mb) for lo, hi, mb in ((0, nb, _rows(self._bridges, 0, nb)), (nb, B, None)) if hi > lo]

    def read_sensors(self, rbd, est, tick, noise=None, accel_dt=0.002, hardware=None):
        reads = [self._ctx.read_sensors(rbd[lo:hi], _rows(est, lo, hi), tick, noise, accel_dt, hardware=_rows(hardware, lo, hi), bridge=mb)
                 for lo, hi, mb in self._groups(rbd.shape[0])]
        return tuple(np.concatenate(x) for x in zip(*reads))

    def actuation(self, time, state, command, rbd, delay=0.009, hardware=None):
        B = rbd.shape[0]
        tau, self._mcmd = np.zeros((B, 10)), np.zeros((B, 10, 5))
        self._lim = np.array([h.torque_limit[:] for h in hardware]) if hardware is not None else np.tile(self._default, (B, 1))
        for lo, hi, mb in self._groups(B):
            out = self._ctx.actuation(time, _rows(state, lo, hi), command[lo:hi], rbd[lo:hi], delay, hardware=_rows(hardware, lo, hi), bridge=mb)
            if mb is None:
                tau[lo:hi] = out
            else:
                self._mcmd[lo:hi] = out
        return tau

    def sim_step(self, rbd, tau, params=None, wrench=None, variation=None, terrain=None):
        B = rbd.shape[0]
        nxt, cf, fl = np.zeros((B, 32)), np.zeros((B, 12)), np.zeros((B, 4), dtype=np.uint8)
        for lo, hi, mb in self._groups(B):
            kw = dict(wrench=None if wrench is None else wrench[lo:hi], variation=_rows(variation, lo, hi), terrain=_rows(terrain, lo, hi))
            if mb is None:
                nxt[lo:hi], cf[lo:hi], fl[lo:hi] = self._ctx.sim_step(rbd[lo:hi], tau[lo:hi], params, **kw)
            else:
                nxt[lo:hi], cf[lo:hi], fl[lo:hi], tau[lo:hi] = self._ctx.sim_step(rbd[lo:hi], self._mcmd[lo:hi], params, bridge=mb,
                                                                                  limits=self._lim[lo:hi], **kw)
        return nxt, cf, fl
