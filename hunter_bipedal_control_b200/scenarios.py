"""Synthetic workloads of SURVEY.md 8(d) (configs 1-5): initial states, mode schedules, targets, swing references.

Host-side input generation only (numpy). The reference's own reference manager (gait tiling, swing planner) is mirrored by
`trot_reference`: mode schedule from the gait template (reference.info:67-80), swing splines from genSwingTrajs
(SwingTrajectoryPlanner.cpp:314-358), targets from cmdVelToTargetTrajectories (TargetTrajectoriesPublisher.cpp:102-130).
"""
import numpy as np

INITIAL_STATE = np.array([0, 0, 0, 0, 0, 0, 0, 0, 0.63, 0, 0, 0, .1, 0, .4, .93, .53, -.1, 0, -.4, .93, -.53])
DEFAULT_JOINTS = INITIAL_STATE[12:]
JOINT_LOWER = np.array([-0.2, -0.5, -0.8, 0.0, -1.1, -0.5, -1.0, -1.2, 0.0, -1.1])
JOINT_UPPER = np.array([0.5, 1.0, 1.2, 1.5, 1.1, 0.2, 0.5, 0.8, 1.5, 1.1])
TOTAL_MASS = 12.586944
COM_HEIGHT = 0.63
FEET_BIAS = np.array([[0.034, 0.11, -0.63], [0.034, -0.11, -0.63], [-0.056, 0.11, -0.63], [-0.056, -0.11, -0.63]])
NEXT_Z = 0.02
SWING_HEIGHT, SWING_TIME_SCALE = 0.04, 0.15
GAITS = {
    "stance": ([3], [0.0, 0.5]),
    "trot": ([2, 1], [0.0, 0.3, 0.6]),
    "standing_trot": ([2, 3, 1, 3], [0.0, 0.25, 0.3, 0.55, 0.6]),
    "flying_trot": ([2, 0, 1, 0], [0.0, 0.15, 0.2, 0.35, 0.4]),
}


def mode_flags(mode):
    return [mode in (2, 3), mode in (1, 3), mode in (2, 3), mode in (1, 3)]


def rot_zyx(e):
    z, y, x = e
    cz, sz, cy, sy, cx, sx = np.cos(z), np.sin(z), np.cos(y), np.sin(y), np.cos(x), np.sin(x)
    return np.array([[cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx], [sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx],
                     [-sy, cy * sx, cy * cx]])


def random_initial_states(B, seed=20240901):
    """Config 2 perturbation of initialState (SURVEY 8d): one PCG64 stream per instance, seed + instance index."""
    x = np.tile(INITIAL_STATE, (B, 1))
    for i in range(B):
        rng = np.random.default_rng(seed + i)
        x[i, 6:8] += rng.uniform(-0.05, 0.05, 2)
        x[i, 8] = rng.uniform(0.60, 0.66)
        x[i, 9] = rng.uniform(-np.pi, np.pi)
        x[i, 10:12] = rng.uniform(-0.1, 0.1, 2)
        x[i, 0:6] = rng.uniform(-0.1, 0.1, 6)
        x[i, 12:] = np.clip(DEFAULT_JOINTS + rng.uniform(-0.05, 0.05, 10), JOINT_LOWER, JOINT_UPPER)
    return x


def tile_gait(gait, t_start, t_end, transition=0.1, phase=0.0):
    """GaitSchedule::tileModeSequenceTemplate (gait/GaitSchedule.cpp:123-161) after an initial stance of `transition` seconds."""
    modes_t, times_t = GAITS[gait]
    ev = []
    md = [3]
    t = t_start + transition - phase
    if gait == "stance":
        return np.array([]), [3]
    ev.append(t_start + transition)
    first = True
    while t < t_end:
        for i, m in enumerate(modes_t):
            seg_end = t + (times_t[i + 1] - times_t[i])
            if seg_end > t_start + transition + 1e-12:
                md.append(m)
                ev.append(seg_end)
            t = seg_end
        first = False
    md.append(3)
    return np.array(ev), md


def mode_at(ev, md, t):
    return md[int(np.searchsorted(ev, t + 1e-9, side="right"))] if len(ev) else md[0]


def hermite(t, t0, t1, p0, v0, p1, v1):
    T = t1 - t0
    tn = (t - t0) / T
    dp, dv = p1 - p0, v1 - v0
    c0, c1, c2, c3 = p0, v0 * T, -(3 * v0 + dv) * T + 3 * dp, (2 * v0 + dv) * T - 2 * dp
    return ((c3 * tn + c2) * tn + c1) * tn + c0, ((3 * c3 * tn + 2 * c2) * tn + c1) / T


def swing_segments(t0s, t1s, p_start, p_stop):
    """genSwingTrajs (SwingTrajectoryPlanner.cpp:314-358): x/y 3-node, z 4-node Hermite splines -> list per axis of (t0,t1,p0,v0,p1,v1)."""
    T = t1s - t0s
    segs = [[], [], []]
    a1, l1, k1 = 0.417, 0.650, 1.770
    for ax in range(2):
        tm = (1 - a1) * t0s + a1 * t1s
        pm = (1 - l1) * p_start[ax] + l1 * p_stop[ax]
        vm = k1 * (p_stop[ax] - p_start[ax]) / T
        segs[ax] = [(t0s, tm, p_start[ax], 0.0, pm, vm), (tm, t1s, pm, vm, p_stop[ax], 0.0)]
    scaling = min(1.0, T / SWING_TIME_SCALE)
    max_z = max(p_start[2], p_stop[2]) + scaling * SWING_HEIGHT
    za1, zl1, zk1, za2, zl2, zk2 = 0.251, 0.749, 1.338, 0.630, 0.570, 1.633
    tA = (1 - za1) * t0s + za1 * t1s; tB = (1 - za2) * t0s + za2 * t1s
    pA = zl1 * max_z; vA = zk1 * (zl1 * (max_z - p_start[2])) / (za1 * T)
    pB = zl2 * max_z + (1 - zl2) * p_stop[2]; vB = zk2 * zl2 * (p_stop[2] - max_z) / ((1 - za2) * T)
    segs[2] = [(t0s, tA, p_start[2], 0.0, pA, vA), (tA, tB, pA, vA, pB, vB), (tB, t1s, pB, vB, p_stop[2], 0.0)]
    return segs


def make_reference(x0, cmd_vel, gait, N, dt, t0=0.0, phase=0.0):
    """Node-sampled references (x_ref [(N+1)x22], swing [(N+1)x24], mode [(N+1)]) for one instance, plus the compact description."""
    T = N * dt
    ev, md = tile_gait(gait, t0, t0 + 2 * T, 0.1, phase)
    times = t0 + dt * np.arange(N + 1)
    mode = np.array([mode_at(ev, md, t) for t in times], dtype=np.int32)
    # target (cmdVelToTargetTrajectories): pose advanced by the rotated command over the horizon
    R = rot_zyx(x0[9:12])
    v = R @ np.array([cmd_vel[0], cmd_vel[1], 0.0])
    cur = np.concatenate([np.zeros(6), x0[6:12], DEFAULT_JOINTS]); cur[8] = COM_HEIGHT; cur[10:12] = 0
    tgt = cur.copy(); tgt[6] += v[0] * T; tgt[7] += v[1] * T; tgt[9] += cmd_vel[3] * T
    cur[0:3] = v; tgt[0:3] = v
    al = ((times - t0) / T)[:, None]
    x_ref = (1 - al) * cur[None] + al * tgt[None]
    # swing references: stance feet stay at their current foothold (z = 0.02), swing feet move by v * (swing + half stance) (Raibert-style)
    yaw = x0[9]
    Ry = rot_zyx([yaw, 0, 0])
    foot0 = np.array([x0[6:9] + Ry @ b for b in FEET_BIAS]); foot0[:, 2] = NEXT_Z
    swing = np.zeros((N + 1, 4, 6))
    segments = [[[] for _ in range(3)] for _ in range(4)]
    bounds = np.concatenate([[t0 - 1.0], ev, [t0 + 10.0]]) if len(ev) else np.array([t0 - 1.0, t0 + 10.0])
    for c in range(4):
        pos = foot0[c].copy()
        p = 0
        while p < len(md):
            fl = mode_flags(md[p])[c]
            q = p
            while q + 1 < len(md) and mode_flags(md[q + 1])[c] == fl:
                q += 1
            ts, te = bounds[p], bounds[q + 1]
            if fl:
                for a in range(3):
                    segments[c][a].append((ts, te, pos[a], 0.0, pos[a], 0.0))
            else:
                nxt = pos + np.array([v[0], v[1], 0.0]) * (te - ts) * 2.0
                nxt[2] = NEXT_Z
                sg = swing_segments(ts, te, pos, nxt)
                for a in range(3):
                    segments[c][a].extend(sg[a])
                pos = nxt
            p = q + 1
        for a in range(3):
            segs = segments[c][a]
            for k, t in enumerate(times):
                s = 0
                while s + 1 < len(segs) and t >= segs[s][1]:
                    s += 1
                pv = hermite(t, *segs[s])
                swing[k, c, a] = pv[0]; swing[k, c, 3 + a] = pv[1]
    compact = dict(events=ev, modes=md, target_times=np.array([t0, t0 + T]), target_states=np.stack([cur, tgt]), segments=segments)
    return x_ref, swing.reshape(N + 1, 24), mode, compact


def sample_reference(compact, times):
    """Evaluate a compact reference description (make_reference's 4th value) at arbitrary node times, the way the device expansion does:
    mode in force on the interval starting at t, clamped linear target interpolation, cubic-Hermite swing segments."""
    times = np.asarray(times, dtype=np.float64)
    ev, md = compact["events"], compact["modes"]
    tt, ts = compact["target_times"], compact["target_states"]
    n = len(times)
    mode = np.array([mode_at(ev, md, t) for t in times], dtype=np.int32)
    x_ref = np.zeros((n, 22))
    for k, t in enumerate(times):
        if len(tt) <= 1 or t <= tt[0]:
            x_ref[k] = ts[0]
        elif t >= tt[-1]:
            x_ref[k] = ts[-1]
        else:
            s = 0
            while s + 2 < len(tt) and tt[s + 1] <= t:
                s += 1
            al = (t - tt[s]) / (tt[s + 1] - tt[s])
            x_ref[k] = (1 - al) * ts[s] + al * ts[s + 1]
    swing = np.zeros((n, 4, 6))
    for c in range(4):
        for a in range(3):
            segs = compact["segments"][c][a]
            for k, t in enumerate(times):
                s = 0
                while s + 1 < len(segs) and t >= segs[s][1]:
                    s += 1
                pv = hermite(t, *segs[s])
                swing[k, c, a] = pv[0]; swing[k, c, 3 + a] = pv[1]
    return x_ref, swing.reshape(n, 24), mode


def event_time_grid(t0, T, dt, events, capacity, dt_min=1e-9):
    """Time discretisation with event nodes (SURVEY 8a row S1, ocs2::timeDiscretizationWithEvents with the pre-/post-event node pair collapsed):
    steps of dt, a node on every mode switch inside the horizon (the grid re-anchors there), last node = t0 + T."""
    tf = t0 + T
    ev = [e for e in events if e > t0 + 1e-9]
    nodes = [t0]
    cur, ei = t0, 0
    while cur < tf:
        nx = cur + dt
        if ei < len(ev) and nx >= ev[ei]:
            nx = ev[ei]; ei += 1
        if nx >= tf:
            nx = tf
        if nx > cur + dt_min or len(nodes) == 1:
            if len(nodes) - 1 == capacity:
                nodes[-1] = tf
                break
            nodes.append(nx)
        else:
            nodes[-1] = nx
        cur = nx
    return np.array(nodes)


def make_batch(B, N=100, dt=0.01, gait="trot", cmd_vel=(0.2, 0.0, 0.0, 0.0), seed=20240901, gaits=None, cmd_vels=None, return_compact=False):
    x0 = random_initial_states(B, seed)
    x_ref = np.zeros((B, N + 1, 22)); swing = np.zeros((B, N + 1, 24)); mode = np.zeros((B, N + 1), dtype=np.int32)
    compacts = []
    for i in range(B):
        g = gaits[i] if gaits is not None else gait
        cv = cmd_vels[i] if cmd_vels is not None else cmd_vel
        x_ref[i], swing[i], mode[i], c = make_reference(x0[i], cv, g, N, dt)
        compacts.append(c)
    if return_compact:
        return x0, x_ref, swing, mode, compacts
    return x0, x_ref, swing, mode


def consistent_rbd(x, rng=None, noise=0.0):
    """rbd measurement [zyx, p, qj, omega_world, v, qj_dot] (StateEstimateBase.cpp:73-106) at the configuration of x with small velocities."""
    B = x.shape[0]
    rbd = np.zeros((B, 32))
    rbd[:, 0:3] = x[:, 9:12]; rbd[:, 3:6] = x[:, 6:9]; rbd[:, 6:16] = x[:, 12:22]
    if rng is not None:
        rbd[:, 0:16] += noise * rng.uniform(-1, 1, (B, 16))
        rbd[:, 16:32] = rng.uniform(-0.3, 0.3, (B, 16))
    return rbd


def pack_references(compacts, horizon):
    """Compact descriptions returned by make_reference (4th value) -> ctypes array of HbReference for the device expansion."""
    from .api import HbReference, HB_MAX_SEGMENTS
    refs = (HbReference * len(compacts))()
    for r, c in zip(np.ctypeslib.as_array(refs), compacts):
        ne, nm, nt = len(c["events"]), len(c["modes"]), len(c["target_times"])
        r["n_events"] = ne; r["event_times"][:ne] = c["events"]; r["modes"][:nm] = c["modes"]
        r["n_targets"] = nt; r["target_times"][:nt] = c["target_times"]; r["target_states"][:nt] = c["target_states"]
        for cc in range(4):
            for a in range(3):
                segs = [sg for sg in c["segments"][cc][a] if sg[0] <= horizon + 1e-9]      # only what the horizon can see
                if len(segs) > HB_MAX_SEGMENTS:
                    raise ValueError("too many swing segments for hb_reference")
                r["n_segments"][cc, a] = len(segs)
                r["segments"][cc, a, :len(segs)] = np.reshape(segs, (-1, 6))
    return refs
