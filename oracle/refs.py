"""CPU restatements of the steps around the solve. TEST INFRASTRUCTURE ONLY (tests/, smoke and the bench baseline may import it).

  P1  GaitSchedule::{insert,tile}ModeSequenceTemplate     legged_interface/src/gait/GaitSchedule.cpp:57-161
  P2  calculateVelAbs / walkGait / trotGait               legged_interface/src/SwitchedModelReferenceManager.cpp:185-249   (GaitSelectorRef)
  P3  SwingTrajectoryPlanner::update/calNextFootPos/...   legged_interface/src/foot_planner/SwingTrajectoryPlanner.cpp:164-358, 394-458
      CubicSpline / MultiCubicSpline                      legged_interface/src/foot_planner/{CubicSpline,MultiCubicSpline}.cpp
  P4  calculateJointRef + InverseKinematics::computeIK    SwitchedModelReferenceManager.cpp:251-300, foot_planner/InverseKinematics.cpp:20-231
  P5  cmdVelToTargetTrajectories                          legged_controllers/src/TargetTrajectoriesPublisher.cpp:41-130
  W6  joint command law                                   legged_controllers/src/LeggedController.cpp:186-257               (joint_command)
  N3  KalmanFilterEstimate::update                        legged_estimation/src/LinearKalmanFilter.cpp:24-185               (KalmanFilterRef)
  --  warm start of the next solve                        ocs2_sqp SqpSolver::initializeStateInputTrajectories (un-vendored) (warm_start_shift)
  constants                                               legged_controllers/config/hunter/{reference,task}.info

Unlike the product's flattened segment lists (csrc/hb_planner.h) the planner part follows the reference's own object structure: one
spline object per *phase index* and per axis, looked up by lower_bound on the event times; Eigen's pivoted QR is LAPACK's, the
kernel basis comes from numpy solves, the Kalman filter uses dense A, B, C matrices and np.linalg.solve -- so product and
restatement only agree if both follow the reference.

parity: these layers have no fixtures in the reference and it cannot be imported (C++ against OCS2 / ROS): pinned through the
reference's published constants, the properties in tests/test_planner.py and the leg kinematics against the MuJoCo-pinned oracle.
"""
import bisect
import math

import numpy as np

COM_HEIGHT = 0.57
NEXT_Z = 0.02
SWING_HEIGHT = 0.08
SWING_TIME_SCALE = 0.15
FEET_BIAS = [(0.11, 0.12, -0.57), (0.11, -0.12, -0.57), (-0.06, 0.12, -0.57), (-0.06, -0.12, -0.57)]
DEFAULT_JOINTS = None  # filled from the generated header below

GAITS = {
    "stance": ([3], [0.0, 0.5]),
    "trot": ([2, 1], [0.0, 0.3, 0.6]),
    "standing_trot": ([2, 3, 1, 3], [0.0, 0.25, 0.3, 0.55, 0.6]),
    "flying_trot": ([2, 0, 1, 0], [0.0, 0.15, 0.2, 0.35, 0.4]),
}


def _header_array(name):
    import os, re
    src = open(os.path.join(os.path.dirname(__file__), "..", "include", "hunter_model_constants.h")).read()
    m = re.search(name + r"\[[^\]]*\]\s*=\s*\{([^}]*)\}", src)
    return [float(v) for v in m.group(1).replace("\n", " ").split(",") if v.strip()]


def _header_value(name):
    import os, re
    src = open(os.path.join(os.path.dirname(__file__), "..", "include", "hunter_model_constants.h")).read()
    m = re.search(r"#define\s+" + name + r"\s+\(?([-+0-9.eE]+)", src)
    return float(m.group(1))


def constants_from_header():
    """The generated header carries the values parsed from reference.info / task.info; use them so the restatement follows the files."""
    global DEFAULT_JOINTS, COM_HEIGHT, NEXT_Z, SWING_HEIGHT, SWING_TIME_SCALE, FEET_BIAS
    DEFAULT_JOINTS = np.array(_header_array("HB_DEFAULT_JOINT_STATE"))
    COM_HEIGHT = _header_value("HB_COM_HEIGHT"); NEXT_Z = _header_value("HB_NEXT_POSITION_Z")
    SWING_HEIGHT = _header_value("HB_SWING_HEIGHT"); SWING_TIME_SCALE = _header_value("HB_SWING_TIME_SCALE")
    x1, x2, y, z = (_header_value("HB_FEET_BIAS_X1"), _header_value("HB_FEET_BIAS_X2"), _header_value("HB_FEET_BIAS_Y"), _header_value("HB_FEET_BIAS_Z"))
    FEET_BIAS = [(x1, y, z), (x1, -y, z), (x2, y, z), (x2, -y, z)]


constants_from_header()


def rot_zyx(e):
    z, y, x = e
    cz, sz, cy, sy, cx, sx = math.cos(z), math.sin(z), math.cos(y), math.sin(y), math.cos(x), math.sin(x)
    return np.array([[cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx],
                     [sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx],
                     [-sy, cy * sx, cy * cx]])


def stance_legs(mode):
    """modeNumber2StanceLeg (MotionPhaseDefinition.h:55-87): contacts l_toe, r_toe, l_heel, r_heel."""
    left, right = mode in (2, 3), mode in (1, 3)
    return [left, right, left, right]


class ModeSchedule:
    def __init__(self, events, modes):
        self.events, self.modes = list(events), list(modes)
        assert len(self.modes) == len(self.events) + 1

    def mode_at(self, t):
        return self.modes[bisect.bisect_left(self.events, t)]


def gait_schedule(gait, prev_event, start, final_time):
    """Initial {STANCE, STANCE} schedule, template inserted at `start`, tiled until final_time, closed by STANCE."""
    tm, tt = GAITS[gait]
    events, modes = [prev_event, start], [3, 3]
    while events[-1] < final_time:
        for i, m in enumerate(tm):
            modes.append(m)
            events.append(events[-1] + (tt[i + 1] - tt[i]))
    modes.append(3)
    return ModeSchedule(events, modes)


class Target:
    """TargetTrajectories with two samples; getDesiredState = clamped linear interpolation."""

    def __init__(self, times, states):
        self.times, self.states = list(times), [np.array(s, dtype=float) for s in states]

    def state(self, t):
        if t <= self.times[0]:
            return self.states[0].copy()
        if t >= self.times[-1]:
            return self.states[-1].copy()
        a = (t - self.times[0]) / (self.times[1] - self.times[0])
        return (1 - a) * self.states[0] + a * self.states[1]


def cmd_vel_to_target(cmd, time, state, time_to_target):
    pose = np.array(state[6:12], dtype=float)
    v = rot_zyx(pose[3:6]) @ np.array(cmd[:3], dtype=float)
    if abs(v[0]) < 0.06:
        v[0] = 0.0
    elif abs(v[1]) < 0.06:
        v[1] = 0.0
    target = np.array([pose[0] + v[0] * time_to_target, pose[1] + v[1] * time_to_target, COM_HEIGHT, pose[3] + cmd[3] * time_to_target, 0.0, 0.0])
    cur = pose.copy(); cur[4] = 0.0; cur[5] = 0.0
    cur[2] = pose[2] + max(-0.04, min(0.04, COM_HEIGHT - pose[2]))
    states = []
    for p in (cur, target):
        s = np.zeros(22); s[6:12] = p; s[12:22] = DEFAULT_JOINTS; s[0:3] = v
        states.append(s)
    return Target([time, time + time_to_target], states)


class CubicSpline:
    def __init__(self, n0, n1):
        (self.t0, p0, v0), (self.t1, p1, v1) = n0, n1
        self.dt = self.t1 - self.t0
        dp, dv = p1 - p0, v1 - v0
        self.c0 = p0; self.c1 = v0 * self.dt
        self.c2 = -(3.0 * v0 + dv) * self.dt + 3.0 * dp
        self.c3 = (2.0 * v0 + dv) * self.dt - 2.0 * dp

    def position(self, t):
        tn = (t - self.t0) / self.dt
        return self.c3 * tn ** 3 + self.c2 * tn ** 2 + self.c1 * tn + self.c0

    def velocity(self, t):
        tn = (t - self.t0) / self.dt
        return (3.0 * self.c3 * tn ** 2 + 2.0 * self.c2 * tn + self.c1) / self.dt


class MultiCubicSpline:
    def __init__(self, nodes):
        self.nodes = nodes
        self.splines = [CubicSpline(nodes[i], nodes[i + 1]) for i in range(len(nodes) - 1)]

    def _pick(self, t):
        for i in range(len(self.nodes) - 1):
            if self.nodes[i][0] <= t < self.nodes[i + 1][0]:
                return self.splines[i]
        if t < self.nodes[0][0]:
            return self.splines[0]
        return self.splines[-1]

    def position(self, t):
        return self._pick(t).position(t)

    def velocity(self, t):
        return self._pick(t).velocity(t)


def find_index(index, flags):
    n = len(flags)
    start = 0
    for ip in range(index - 1, -1, -1):
        if flags[ip] != flags[index]:
            start = ip
            break
    final = n - 2
    for ip in range(index + 1, n):
        if flags[ip] != flags[index]:
            final = ip - 1
            break
    return start, final


class SwingPlanner:
    """SwingTrajectoryPlanner: keeps latestStanceposition_ between updates."""

    def __init__(self, latest_stance=None):
        self.latest = np.zeros((4, 3)) if latest_stance is None else np.array(latest_stance, dtype=float).reshape(4, 3).copy()
        self.body_vel_cmd = np.zeros(6)
        self.current_feet = np.zeros((4, 3))

    def next_foot_pos(self, foot, current_time, stop_time, next_middle_time, next_middle_body_pos, current_body_pos, current_body_vel):
        roted_bias = rot_zyx(next_middle_body_pos[3:6]) @ np.array(FEET_BIAS[foot])
        rot = rot_zyx(current_body_pos[3:6])
        vel_cmd_linear = rot @ self.body_vel_cmd[:3]
        vel_cmd_angular = rot @ self.body_vel_cmd[3:]
        vel_linear = np.array(current_body_vel, dtype=float); vel_linear[2] = 0.0
        k = 0.03
        p_shoulder = (stop_time - current_time) * (0.5 * vel_linear + 0.5 * vel_cmd_linear) + roted_bias
        p_symmetry = (next_middle_time - stop_time) * vel_linear + k * (vel_linear - vel_cmd_linear)
        p_centrifugal = 0.5 * math.sqrt(current_body_pos[2] / 9.81) * np.cross(vel_linear, vel_cmd_angular)
        r = current_body_pos[:3] + p_shoulder + p_symmetry + p_centrifugal
        r[2] = NEXT_Z
        return r

    @staticmethod
    def swing_splines(t0, t1, a, b):
        out = []
        for ax in range(2):
            out.append(MultiCubicSpline([(t0, a[ax], 0.0),
                                         ((1 - 0.417) * t0 + 0.417 * t1, (1 - 0.650) * a[ax] + 0.650 * b[ax], 1.770 * (b[ax] - a[ax]) / (t1 - t0)),
                                         (t1, b[ax], 0.0)]))
        scaling = min(1.0, (t1 - t0) / SWING_TIME_SCALE)
        max_z = max(a[2], b[2]) + scaling * SWING_HEIGHT
        out.append(MultiCubicSpline([(t0, a[2], 0.0),
                                     ((1 - 0.251) * t0 + 0.251 * t1, 0.749 * max_z, 1.338 * (0.749 * (max_z - a[2])) / (0.251 * (t1 - t0))),
                                     ((1 - 0.630) * t0 + 0.630 * t1, 0.570 * max_z + (1 - 0.570) * b[2], 1.633 * 0.570 * (b[2] - max_z) / ((1 - 0.630) * (t1 - t0))),
                                     (t1, b[2], 0.0)]))
        return out

    def update(self, ms, target, init_time):
        self.events = ms.events
        legs = stance_legs(ms.mode_at(init_time + 0.001))
        for i in range(4):
            if legs[i]:
                self.latest[i] = self.current_feet[i]
            self.latest[i][2] = NEXT_Z
        last, nxt = self.latest.copy(), self.latest.copy()
        n = len(ms.modes)
        self.trajs = [[None] * n for _ in range(4)]
        for j in range(4):
            flags = [stance_legs(m)[j] for m in ms.modes]
            last_final = 0
            for p in range(n):
                si, fi = find_index(p, flags)
                if not flags[p]:
                    if si < 0 or fi >= n - 1:
                        raise RuntimeError("swing phase without take-off / touch-down")
                    ts, tf = ms.events[si], ms.events[fi]
                    if init_time < tf and fi > last_final:
                        last[j] = nxt[j]
                        if fi < n - 1:
                            _, fi2 = find_index(fi + 1, flags)
                            mid = 0.5 * (tf + ms.events[fi2])
                        else:
                            mid = tf
                        nxt[j] = self.next_foot_pos(j, init_time, tf, mid, target.state(mid)[6:12], target.state(init_time)[6:12], target.states[0][0:3])
                        last_final = fi
                    self.trajs[j][p] = self.swing_splines(ts, tf, last[j].copy(), nxt[j].copy())
                else:
                    ts, tf = ms.events[si], ms.events[fi]
                    if tf > ts:
                        self.trajs[j][p] = [MultiCubicSpline([(ts, nxt[j][a], 0.0), (tf, nxt[j][a], 0.0)]) for a in range(3)]
                    else:   # zero-length spline of the reference (never queried inside a solver window)
                        self.trajs[j][p] = None

    def foot(self, j, t):
        """(position(3), velocity(3)) of contact j at time t: phase index by lower_bound on the events (lookup::findIndexInTimeArray)."""
        p = bisect.bisect_left(self.events, t)
        sp = self.trajs[j][p]
        return np.array([s.position(t) for s in sp]), np.array([s.velocity(t) for s in sp])


# ------------------------------------------------------------------------------------------------------------------------------
# P4: joint references by inverse kinematics (SwitchedModelReferenceManager.cpp:251-300, InverseKinematics.cpp:20-231)
JOINT_XYZ = np.array(_header_array("HB_JOINT_XYZ")).reshape(11, 3)
JOINT_AXIS = np.array(_header_array("HB_JOINT_AXIS")).reshape(11, 3)
CONTACT_OFFSET = np.array(_header_array("HB_CONTACT_OFFSET")).reshape(4, 3)
JOINT_LOWER = np.array(_header_array("HB_JOINT_LOWER"))
JOINT_UPPER = np.array(_header_array("HB_JOINT_UPPER"))


def _rodrigues(a, q):
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + math.sin(q) * K + (1 - math.cos(q)) * (K @ K)


def leg_frame(leg, pose, qj):
    """Toe contact frame of leg (0 left, 1 right): position, rotation, world-aligned linear / angular Jacobians (3x5)."""
    R = rot_zyx(pose[3:6]); o = np.array(pose[0:3], dtype=float)
    origins, axes = [], []
    for i in range(5):
        b = 1 + 5 * leg + i
        o = o + R @ JOINT_XYZ[b]
        origins.append(o.copy()); axes.append(R @ JOINT_AXIS[b])
        R = R @ _rodrigues(JOINT_AXIS[b], qj[i])
    toe = o + R @ CONTACT_OFFSET[leg]
    Jl = np.stack([np.cross(axes[i], toe - origins[i]) for i in range(5)], axis=1)
    Ja = np.stack(axes, axis=1)
    return toe, R, Jl, Ja


def colpiv_qr_solve(A, b, threshold=0.01):
    """Eigen::ColPivHouseholderQR(threshold).solve: LAPACK pivoted QR picks the same columns (largest remaining norm)."""
    import scipy.linalg as sla
    Q, Rm, P = sla.qr(A, mode="economic", pivoting=True)
    d = np.abs(np.diag(Rm))
    rank = int(np.sum(d > threshold * d[0])) if d[0] > 0 else 0
    x = np.zeros(A.shape[1])
    if rank:
        c = Q[:, :rank].T @ b
        x[P[:rank]] = sla.solve_triangular(Rm[:rank, :rank], c)
    return x


def fullpiv_lu_kernel(J):
    """Eigen::FullPivLU::kernel: basis vectors e_j - sum_P (J_P^-1 J_j) e_p over the non-pivot columns j of complete pivoting."""
    M = np.array(J, dtype=float); m, n = M.shape
    cols = list(range(n)); rows = list(range(m))
    for k in range(m):
        sub = np.abs(M[k:, k:])
        i, j = np.unravel_index(np.argmax(sub), sub.shape)
        M[[k, k + i]] = M[[k + i, k]]; M[:, [k, k + j]] = M[:, [k + j, k]]
        cols[k], cols[k + j] = cols[k + j], cols[k]
        for r in range(k + 1, m):
            M[r, k:] -= M[r, k] / M[k, k] * M[k, k:]
    P, F = cols[:m], cols[m:]
    N = np.zeros((n, n - m))
    for c, j in enumerate(F):
        N[P, c] = -np.linalg.solve(J[:, P], J[:, j])
        N[j, c] = 1.0
    return N


def log3(R):
    tr = np.trace(R)
    theta = math.acos(max(-1.0, min(1.0, (tr - 1.0) / 2.0)))
    v = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    f = theta / (2.0 * math.sin(theta)) if theta > 1e-8 else 0.5 * (1.0 + theta * theta / 6.0)
    return f * v


def _ik_loop(leg, qj, err_of, step_of):
    err_tol, conv_tol, dt, max_it = 0.01, 0.001, 0.7, 5
    lo, hi = JOINT_LOWER[5 * leg:5 * leg + 5], JOINT_UPPER[5 * leg:5 * leg + 5]
    qj = np.array(qj, dtype=float)
    err = err_of(qj); last = np.linalg.norm(err)
    if last < err_tol:
        return qj
    it = 0
    while True:
        new_q = np.minimum(hi, np.maximum(lo, qj + dt * step_of(qj, err)))
        err = err_of(new_q); en = np.linalg.norm(err)
        if en > last or abs(en - last) < conv_tol:
            break
        last, qj = en, new_q
        if en < err_tol:
            break
        it += 1
        if it >= max_it:
            break
    return qj


def translation_ik(pose, qj, leg, des_p):
    def terr(q):
        return leg_frame(leg, pose, q)[0] - des_p

    def tstep(q, err):
        return -colpiv_qr_solve(leg_frame(leg, pose, q)[2], err)

    return _ik_loop(leg, qj, terr, tstep)


def rotation_ik(pose, qj, leg, R_des):
    def rerr(q):
        return log3(R_des.T @ leg_frame(leg, pose, q)[1])

    def rstep(q, err):
        _, R, Jl, Ja = leg_frame(leg, pose, q)
        N = fullpiv_lu_kernel(R.T @ Jl)
        return -N @ colpiv_qr_solve((R.T @ Ja) @ N, err)

    return _ik_loop(leg, qj, rerr, rstep)


def compute_ik(pose, qj, leg, des_p, R_des):
    return rotation_ik(pose, translation_ik(pose, qj, leg, des_p), leg, R_des)


def joint_references(sp, tg, init_time, final_time, init_state):
    """calculateJointRef: returns the resampled Target with IK joint references (or tg unchanged for short horizons)."""
    n = int(math.floor((final_time - init_time) / 0.15)) + 1
    if n <= 2:
        return tg
    Ts = [final_time if i == n - 1 else init_time + i * ((final_time - init_time) / (n - 1)) for i in range(n)]
    states = [tg.state(t) for t in Ts]
    states[0][12:22] = DEFAULT_JOINTS
    R_des = rot_zyx(init_state[9:12])
    for i in range(n):
        seed = states[max(i - 1, 0)][12:22].copy()
        for leg in range(2):
            des = sp.foot(leg, Ts[i])[0]
            states[i][12 + 5 * leg:17 + 5 * leg] = compute_ik(states[i][6:12], seed[5 * leg:5 * leg + 5], leg, des, R_des)
    return PiecewiseTarget(Ts, states)


class PiecewiseTarget(Target):
    def state(self, t):
        if t <= self.times[0]:
            return self.states[0].copy()
        if t >= self.times[-1]:
            return self.states[-1].copy()
        s = min(bisect.bisect_right(self.times, t) - 1, len(self.times) - 2)
        a = (t - self.times[s]) / (self.times[s + 1] - self.times[s])
        return (1 - a) * self.states[s] + a * self.states[s + 1]


def plan(t0, horizon, x0, cmd_vel, feet_pos, gait, gait_start, prev_event=None, time_to_target=None, latest_stance=None, joint_ik=True):
    """One instance: returns (ModeSchedule, Target, SwingPlanner) after update, mirroring SwitchedModelReferenceManager::modifyReferences."""
    prev_event = min(t0, gait_start) - 0.5 if prev_event is None else prev_event
    ttt = horizon if time_to_target is None else time_to_target
    ms = gait_schedule(gait, prev_event, gait_start, t0 + 2 * horizon)
    tg = cmd_vel_to_target(cmd_vel, t0, x0, ttt)
    sp = SwingPlanner(latest_stance)
    sp.body_vel_cmd = np.array([cmd_vel[0], cmd_vel[1], cmd_vel[2], cmd_vel[3], 0.0, 0.0])
    sp.current_feet = np.array(feet_pos, dtype=float).reshape(4, 3)
    sp.update(ms, tg, t0)
    if joint_ik:
        tg = joint_references(sp, tg, t0, t0 + horizon, np.asarray(x0, dtype=float))
    return ms, tg, sp


def sample(ms, tg, sp, times, post_event=True):
    """Node-sampled references: x_ref (n x 22), swing (n x 24: per contact pos(3), vel(3)), mode (n)."""
    n = len(times)
    x_ref = np.zeros((n, 22)); swing = np.zeros((n, 24)); mode = np.zeros(n, dtype=np.int32)
    for k, t in enumerate(times):
        x_ref[k] = tg.state(t)
        # the mode of the interval starting at t (a node on an event takes the post-event mode, as the SQP time discretisation does)
        mode[k] = ms.modes[bisect.bisect_right(ms.events, t + 1e-9)] if post_event else ms.mode_at(t)
        for j in range(4):
            p, v = sp.foot(j, t)
            swing[k, 6 * j:6 * j + 3] = p; swing[k, 6 * j + 3:6 * j + 6] = v
    return x_ref, swing, mode


def eval_compact(ref, times):
    """Evaluate a compact hb_reference (ctypes struct) at `times` on the CPU; restates the device expansion kernel for CPU tests."""
    n = len(times)
    x_ref = np.zeros((n, 22)); swing = np.zeros((n, 24)); mode = np.zeros(n, dtype=np.int32)
    ev = [ref.event_times[i] for i in range(ref.n_events)]
    tt = [ref.target_times[i] for i in range(ref.n_targets)]
    ts = [np.array(ref.target_states[i][:]) for i in range(ref.n_targets)]
    for k, t in enumerate(times):
        mode[k] = ref.modes[bisect.bisect_right(ev, t + 1e-9)]
        if len(tt) <= 1 or t <= tt[0]:
            x_ref[k] = ts[0]
        elif t >= tt[-1]:
            x_ref[k] = ts[-1]
        else:
            s = max(0, bisect.bisect_right(tt, t) - 1); s = min(s, len(tt) - 2)
            a = (t - tt[s]) / (tt[s + 1] - tt[s])
            x_ref[k] = (1 - a) * ts[s] + a * ts[s + 1]
        for c in range(4):
            for a in range(3):
                ns = ref.n_segments[c][a]
                if ns == 0:
                    continue
                s = 0
                while s + 1 < ns and t >= ref.segments[c][a][s][1]:
                    s += 1
                sg = ref.segments[c][a][s]
                cs = CubicSpline((sg[0], sg[2], sg[3]), (sg[1], sg[4], sg[5]))
                swing[k, 6 * c + a] = cs.position(t); swing[k, 6 * c + 3 + a] = cs.velocity(t)
    return x_ref, swing, mode


class GaitSelectorRef:
    """P2: calculateVelAbs + walkGait / trotGait (SwitchedModelReferenceManager.cpp:185-249) with a deque like the reference."""

    def __init__(self, gait_level=-1):
        from collections import deque
        self.hist = deque(); self.level = gait_level; self.avg = 0.0

    def update(self, cmd_vel, target0, gait_type=0):
        vc = np.zeros(4); vc[:3] = rot_zyx(target0[9:12]) @ np.array(cmd_vel[:3], dtype=float); vc[2] = 0.0; vc[3] = cmd_vel[3] / 3.0
        ve = np.array(target0[0:4], dtype=float); ve[2] = 0.0; ve[3] = ve[3] / 3.0
        self.hist.appendleft(float(np.linalg.norm(0.5 * vc + 0.5 * ve)))
        while len(self.hist) > 50:
            self.hist.pop()
        self.avg = sum(self.hist) / len(self.hist)
        insert = 0
        if gait_type == 0:
            if self.avg <= 0.02:
                if self.level != 0:
                    insert, self.level = 1, 0
            elif 0.03 < self.avg < 0.4:
                if self.level != 1:
                    insert, self.level = 1, 1
            elif self.avg >= 0.4:
                self.level = 3
        elif gait_type == 2:
            if self.level != 1:
                insert, self.level = 1, 1
        return self.level, insert


PD_DEFAULTS = dict(kp_position=10.0, kd_position=3.0, kp_big_stance=40.0, kp_big_swing=30.0, kd_big=2.0, kp_small_stance=30.0,
                   kp_small_swing=20.0, kd_small=2.0, kd_feet=0.01)     # legged_controllers/cfg/Tutorials.cfg:6-16


def joint_command(period, x_des, u_des, wbc_sol, mode_cmd, rbd, loaded=True, estop=False, gains=PD_DEFAULTS):
    """W6: joint command law of one instance (LeggedController.cpp:186-257). Returns (command 10x5, output_torque 10, estop)."""
    g = gains
    cmd = np.zeros((10, 5)); tau = np.zeros(10)
    pos_des = x_des[12:22] + 0.5 * wbc_sol[6:16] * period * period
    vel_des = u_des[12:22] + wbc_sol[6:16] * period
    legs = stance_legs(mode_cmd)
    for j in range(10):
        q, qd = rbd[6 + j], rbd[16 + 6 + j]
        if not estop and loaded and (q > JOINT_UPPER[j] + 0.02 or q < JOINT_LOWER[j] - 0.02):
            estop = True
        if not loaded:
            c = (x_des[12 + j], u_des[12 + j], g["kp_position"], g["kd_feet"] if j in (4, 9) else g["kd_position"], 0.0)
        else:
            contact = legs[j // 5]
            if j in (0, 1, 5, 6):
                kp, kd = (g["kp_small_stance"] if contact else g["kp_small_swing"]), g["kd_small"]
            elif j in (4, 9):
                kp, kd = (g["kp_small_stance"] if contact else g["kp_small_swing"]), g["kd_feet"]
            else:
                kp, kd = (g["kp_big_stance"] if contact else g["kp_big_swing"]), g["kd_big"]
            c = (pos_des[j], vel_des[j], kp, kd, wbc_sol[28 + j])
        if estop:
            c = (0.0, 0.0, 0.0, 1.0, 0.0)
        cmd[j] = c
        tau[j] = c[4] + c[2] * (c[0] - q) + c[3] * (c[1] - qd)
    return cmd, tau, estop


def warm_start_shift(t0_prev, t0_new, dt, x_prev, u_prev, x0, mode_new, mass, g=9.81):
    """SqpSolver::initializeStateInputTrajectories with a previous solution (restated from OCS2 ocs2_sqp, un-vendored): x[0] = x0;
    interval i: if t_{i+1} is inside the previous horizon, u[i] = prev input at t_i and x[i+1] = prev state at t_{i+1} (linear
    interpolation; the input trajectory repeats its last sample at the final node); otherwise the initializer
    (LeggedRobotInitializer.cpp:67-77): weight-compensating input for the mode of the interval, state kept."""
    N = u_prev.shape[0]
    t_end = t0_prev + N * dt
    u_ext = np.vstack([u_prev, u_prev[-1:]])

    def interp(arr, t):
        s = min(max((t - t0_prev) / dt, 0.0), float(N))
        k = min(int(math.floor(s)), N - 1)
        a = s - k
        return (1 - a) * arr[k] + a * arr[k + 1]

    x = np.zeros((N + 1, 22)); u = np.zeros((N, 22))
    x[0] = x0
    for i in range(N):
        ti, tn = t0_new + i * dt, t0_new + (i + 1) * dt
        if tn > t_end + 1e-9:
            legs = stance_legs(int(mode_new[i])); ns = sum(legs)
            for c in range(4):
                if legs[c]:
                    u[i, 3 * c + 2] = mass * g / ns
            x[i + 1] = x[i]
        else:
            u[i] = interp(u_ext, ti)
            x[i + 1] = interp(x_prev, tn)
    return x, u


# ------------------------------------------------------------------------------------------------------------------------------
# N3: KalmanFilterEstimate::update (legged_estimation/src/LinearKalmanFilter.cpp:24-185), dense matrices as in the reference
KF_PARAMS = dict(footRadius=0.02, imuProcessNoisePosition=0.02, imuProcessNoiseVelocity=0.02, footProcessNoisePosition=0.5,
                 footSensorNoisePosition=0.5, footSensorNoiseVelocity=0.1, footHeightSensorNoise=0.01)     # task.info:336-345


def quat_to_zyx(q):
    x, y, z, w = q
    a = min(-2.0 * (x * z - w * y), .99999)
    return np.array([math.atan2(2 * (x * y + w * z), w * w + x * x - y * y - z * z), math.asin(a),
                     math.atan2(2 * (y * z + w * x), w * w - x * x - y * y + z * z)])


def euler_rates_from_local(zyx, wl):
    sy, cy, sx, cx = math.sin(zyx[1]), math.cos(zyx[1]), math.sin(zyx[2]), math.cos(zyx[2])
    t = sx * wl[1] / cy + cx * wl[2] / cy
    return np.array([t, cx * wl[1] - sx * wl[2], wl[0] + sy * t])


def global_from_euler_rates(zyx, d):
    sz, cz, sy, cy = math.sin(zyx[0]), math.cos(zyx[0]), math.sin(zyx[1]), math.cos(zyx[1])
    return np.array([-sz * d[1] + cy * cz * d[2], cz * d[1] + cy * sz * d[2], d[0] - sy * d[2]])


def euler_rates_from_global(zyx, w):
    sz, cz, sy, cy = math.sin(zyx[0]), math.cos(zyx[0]), math.sin(zyx[1]), math.cos(zyx[1])
    r = (cz * w[0] + sz * w[1]) / cy
    return np.array([w[2] + sy * r, -sz * w[0] + cz * w[1], r])


class ContactForceObserverRef:
    """StateEstimateBase::estContactForce (legged_estimation/src/StateEstimateBase.cpp:130-206) restated: generalised-momentum observer and
    the SVD (least-norm) solve of the per-foot wrench, on the rigid-body terms of oracle/hb_oracle.cpp."""

    def __init__(self, cutoff_frequency=250.0):
        self.lam = cutoff_frequency
        self.last = np.zeros(16)                       # pSCgZinvlast_
        self.est = np.full(16, 50.0)                   # estContactforce_ (:60-61)
        self.disturbance = np.zeros(16)

    def update(self, rbd, tau_cmd, dt):
        from . import hbo
        if dt > 1:
            dt = 0.002
        gama = np.exp(-self.lam * dt); beta = (1 - gama) / (gama * dt)
        q = np.concatenate([rbd[3:6], rbd[0:3], rbd[6:16]])
        v = np.concatenate([rbd[19:22], euler_rates_from_global(rbd[0:3], rbd[16:19]), rbd[22:32]])
        p, g, ctv, J = hbo.observer_terms(q, v)
        pscg = beta * p + np.concatenate([np.zeros(6), tau_cmd]) + ctv - g
        filt = (1 - gama) * pscg + gama * self.last
        self.last = filt
        self.disturbance = beta * p - filt
        for i in range(2):
            S_JT = J[i][:, 6 + 5 * i:11 + 5 * i].T                       # S_li * Jac_i^T  (5 x 6)
            S_tau = self.disturbance[6 + 5 * i:11 + 5 * i]
            self.est[6 * i:6 * i + 6] = np.linalg.pinv(S_JT) @ S_tau    # bdcSvd(...).solve: least-norm least-squares solution
        for i in range(2):
            self.est[12 + i] = np.linalg.norm(self.est[6 * i:6 * i + 3])
            self.est[14 + i] = np.linalg.norm(self.est[6 * i:6 * i + 6])
        return self.est.copy()


def foot_wrench_matrix(q, leg):
    """S_l J_foot' of leg `leg` at the generalised coordinates q (5 x 6): the matrix of estContactForce's per-foot wrench solve."""
    from . import hbo
    J = hbo.observer_terms(q, np.zeros(16))[3]
    return J[leg][:, 6 + 5 * leg:11 + 5 * leg].T


def singular_knee(leg, q, lo=0.0, hi=0.05, tol=1e-14):
    """The knee angle of leg `leg` in [lo, hi] that minimises sigma_min / sigma_max of foot_wrench_matrix, the other coordinates from q:
    golden-section search (the ratio is unimodal there, |knee - k*| / 1.8 near its zero)."""
    def ratio(k):
        qk = np.array(q, dtype=float); qk[6 + 5 * leg + 3] = k
        s = np.linalg.svd(foot_wrench_matrix(qk, leg), compute_uv=False)
        return s[-1] / s[0]
    g = (math.sqrt(5.0) - 1.0) / 2.0
    c, d = hi - g * (hi - lo), lo + g * (hi - lo)
    fc, fd = ratio(c), ratio(d)
    while hi - lo > tol:
        if fc < fd:
            hi, d, fd = d, c, fc
            c = hi - g * (hi - lo); fc = ratio(c)
        else:
            lo, c, fc = c, d, fd
            d = lo + g * (hi - lo); fd = ratio(d)
    return 0.5 * (lo + hi)


class KalmanFilterRef:
    def __init__(self):
        self.x = np.zeros(18); self.P = 100.0 * np.eye(18); self.heights = np.zeros(4)
        self.a = np.eye(18); self.b = np.zeros((18, 3))
        c = np.zeros((28, 18))
        for i in range(4):
            c[3 * i:3 * i + 3, 0:3] = np.eye(3); c[12 + 3 * i:15 + 3 * i, 3:6] = np.eye(3)
        c[0:12, 6:18] = -np.eye(12)
        c[27, 17] = c[26, 14] = c[25, 11] = c[24, 8] = 1.0
        self.c = c

    def update(self, dt, quat, wl, al, jpos, jvel, contact, kin, prm=KF_PARAMS):
        """kin(q16, v16) -> (contact positions 12, contact velocities 12)."""
        zyx = quat_to_zyx(quat)
        wg = global_from_euler_rates(zyx, euler_rates_from_local(zyx, wl))
        a, b = self.a.copy(), self.b.copy()
        a[0:3, 3:6] = dt * np.eye(3); b[0:3] = 0.5 * dt * dt * np.eye(3); b[3:6] = dt * np.eye(3)
        q = np.eye(18)
        q[0:3, 0:3] *= (dt / 20.0) * prm["imuProcessNoisePosition"]
        q[3:6, 3:6] *= (dt * float(np.float32(9.81)) / 20.0) * prm["imuProcessNoiseVelocity"]
        q[6:18, 6:18] *= dt * prm["footProcessNoisePosition"]
        r = np.eye(28)
        r[0:12, 0:12] *= prm["footSensorNoisePosition"]; r[12:24, 12:24] *= prm["footSensorNoiseVelocity"]; r[24:28, 24:28] *= prm["footHeightSensorNoise"]
        qp = np.zeros(16); vp = np.zeros(16)
        qp[3:6] = zyx; qp[6:16] = jpos
        vp[3:6] = euler_rates_from_global(zyx, wg); vp[6:16] = jvel
        ee_pos, ee_vel = kin(qp, vp)
        ps = np.zeros(12); vs = np.zeros(12)
        for i in range(4):
            k = 1.0 if contact[i] else 100.0
            q[6 + 3 * i:9 + 3 * i, 6 + 3 * i:9 + 3 * i] *= k
            r[3 * i:3 * i + 3, 3 * i:3 * i + 3] *= k; r[12 + 3 * i:15 + 3 * i, 12 + 3 * i:15 + 3 * i] *= k; r[24 + i, 24 + i] *= k
            ps[3 * i:3 * i + 3] = -ee_pos[3 * i:3 * i + 3]; ps[3 * i + 2] += prm["footRadius"]
            vs[3 * i:3 * i + 3] = -ee_vel[3 * i:3 * i + 3]
        accel = rot_zyx(zyx) @ np.asarray(al, dtype=float) + np.array([0, 0, -9.81])
        y = np.concatenate([ps, vs, self.heights])
        self.x = a @ self.x + b @ accel
        pm = a @ self.P @ a.T + q
        ey = y - self.c @ self.x
        s = self.c @ pm @ self.c.T + r
        self.x = self.x + pm @ self.c.T @ np.linalg.solve(s, ey)
        p = (np.eye(18) - pm @ self.c.T @ np.linalg.solve(s, self.c)) @ pm
        p = (p + p.T) / 2.0
        self.decoupled = bool(np.linalg.det(p[0:2, 0:2]) > 0.000001)        # the branch of :151-156 this update took
        if self.decoupled:
            p[0:2, 2:18] = 0.0; p[2:18, 0:2] = 0.0; p[0:2, 0:2] /= 10.0
        self.P = p
        rbd = np.zeros(32)
        rbd[0:3] = zyx; rbd[3:6] = self.x[0:3]; rbd[6:16] = jpos; rbd[16:19] = wg; rbd[19:22] = self.x[3:6]; rbd[22:32] = jvel
        return rbd
