"""The solve's time axis restated in float64 numpy from OCS2's structure (not from the kernels): where the nodes lie
(timeDiscretizationWithEvents), what the references are at them (getIntervalStart), how the previous solution seeds the next grid
(initializeStateInputTrajectories) and what the policy gives between solves (evaluatePolicy). The repository's own rules on top of
OCS2 are separate functions or named steps, each said in its docstring."""
import bisect

import numpy as np

from oracle import refs as R

DT_MIN = 1e-9                 # nodes closer than this to their predecessor replace it (the repository's dt_min)
NONE, PRE_EVENT, POST_EVENT = 0, 1, 2


def time_discretization_with_events(t0, tf, dt, events, dt_min=DT_MIN):
    """ocs2::timeDiscretizationWithEvents: the annotated nodes [(time, event)], the pre-/post-event pairs included."""
    nodes = [(t0, NONE)]
    ei = bisect.bisect_left(events, t0)               # lookup::findIndexInTimeArray: lower_bound
    nxt = nodes[-1]
    while nodes[-1][0] < tf:
        t, ev = nxt[0] + dt, NONE
        if ei < len(events) and t >= events[ei]:      # an event has passed: land on it
            t, ev = events[ei], PRE_EVENT
            ei += 1
        if t >= tf:
            t, ev = tf, NONE
        nxt = (t, ev)
        if t > nodes[-1][0] + dt_min:
            nodes.append(nxt)
        else:                                         # points are close together: overwrite the old point
            nodes[-1] = nxt
    out = []
    for node in nodes:
        out.append(node)
        if node[1] == PRE_EVENT:
            out.append((node[0], POST_EVENT))
    return out


def collapse_event_pairs(annotated):
    """Each pre-/post-event pair as one node (identity jump map, no cost, no constraint on it): the node keeps the time, and the interval
    it starts is the post-event one."""
    return np.array([t for t, ev in annotated if ev != POST_EVENT])


def event_node_grid(t0, T, dt, events, capacity, dt_min=DT_MIN):
    """The repository's event-node grid: (node times, status). OCS2's discretisation of [t0, t0 + T] collapsed to one node per event,
    with three rules of the repository on top:
    1. switches at or within dt_min after t0 are in force at t0: they leave the event list, so node 0 stays at the time of the measured
       state (OCS2 moves node 0 onto such a switch, up to dt_min later);
    2. node 0 is never replaced: a horizon T <= dt_min keeps the one interval [t0, t0 + T] (OCS2 leaves the single node t0 + T);
    3. capacity: a grid of more than `capacity` intervals keeps its first `capacity` nodes and ends at t0 + T (the last interval is
       stretched over what it covers), status 1; otherwise status 0."""
    tf = t0 + T
    ev = [e for e in events if e > t0 + dt_min]
    g = collapse_event_pairs(time_discretization_with_events(t0, tf, dt, ev, dt_min))
    if len(g) == 1:
        g = np.array([t0, tf])
    if len(g) - 1 > capacity:
        return np.append(g[:capacity], tf), 1
    return g, 0


# ---------------------------------------------------------------------------------------------------------------- references at the nodes
def interval_mode(events, modes, t, dt_min=DT_MIN):
    """Mode of the interval starting at t (OCS2's getIntervalStart: the interval is evaluated just after its start node, so a node on a
    switch sees the post-event mode). 'Just after' is within dt_min, the tolerance the grid merges nodes with: a switch within dt_min
    after t is in force on the interval (rule 1 of event_node_grid; on uniform grids the rule of DESIGN §2 item 2)."""
    return modes[bisect.bisect_right(events, t + dt_min)]


def mode_at_time(events, modes, t):
    """ModeSchedule::modeAtTime: lower_bound on the switching times, so the earlier mode holds at a switching time."""
    return R.ModeSchedule(events, modes).mode_at(t)


def segment_at(segments, t):
    """The CubicSpline piece of one (foot, axis) list of contiguous segments (t0, t1, p0, v0, p1, v1) that holds t from the right: the
    piece starting at a knot is the one used there, the first piece extrapolates before the list and the last one after it (as
    getZpositionConstraint evaluates the reference's spline)."""
    starts = [s[0] for s in segments]
    s = segments[min(max(bisect.bisect_right(starts, t) - 1, 0), len(segments) - 1)]
    return R.CubicSpline((s[0], s[2], s[3]), (s[1], s[4], s[5]))


def sample_reference(ref, times):
    """Node-sampled references of a reference description ref = dict(events, modes, target_times, target_states, segments[4][3]) at the
    node times: x_ref (n x 22: TargetTrajectories, clamped linear interpolation), swing (n x 24: per foot position(3), velocity(3)),
    mode (n: interval_mode)."""
    n = len(times)
    tg = R.PiecewiseTarget(ref["target_times"], ref["target_states"])
    x_ref = np.array([tg.state(t) for t in times]).reshape(n, 22)
    swing = np.zeros((n, 24))
    mode = np.array([interval_mode(ref["events"], ref["modes"], t) for t in times], dtype=np.int32)
    for c in range(4):
        for a in range(3):
            segs = ref["segments"][c][a]
            if not segs:
                continue
            for k, t in enumerate(times):
                sp = segment_at(segs, t)
                swing[k, 6 * c + a] = sp.position(t)
                swing[k, 6 * c + 3 + a] = sp.velocity(t)
    return x_ref, swing, mode


def pack_reference(ref, out):
    """Fill one HbReference struct (a record of numpy.ctypeslib.as_array of the ctypes array) from a reference description."""
    ne, nt = len(ref["events"]), len(ref["target_times"])
    out["n_events"] = ne; out["event_times"][:ne] = ref["events"]; out["modes"][:ne + 1] = ref["modes"]
    out["n_targets"] = nt; out["target_times"][:nt] = ref["target_times"]; out["target_states"][:nt] = ref["target_states"]
    for c in range(4):
        for a in range(3):
            segs = ref["segments"][c][a]
            out["n_segments"][c, a] = len(segs)
            if segs:
                out["segments"][c, a, :len(segs)] = np.reshape(segs, (-1, 6))


# ---------------------------------------------------------------------------------------------------------------- warm start and policy
def initializer_input(mode, mass, g=9.81):
    """LeggedRobotInitializer::compute: the stance feet share the robot's weight in z, everything else zero."""
    legs = R.stance_legs(int(mode))
    u = np.zeros(22)
    for c in range(4):
        if legs[c]:
            u[3 * c + 2] = mass * g / sum(legs)
    return u


def interpolate(t, times, values):
    """LinearInterpolation::interpolate: clamped to the first / last sample outside the time range; inside, the interval
    [times[i], times[i + 1]] found by lower_bound (a query on an interior node ends the interval before it). Returns (value, i, alpha),
    value = alpha values[i] + (1 - alpha) values[i + 1]."""
    n = len(times) - 1
    if t <= times[0]:
        return values[0].copy(), 0, 1.0
    if t >= times[n]:
        return values[n].copy(), n - 1, 0.0
    i = bisect.bisect_left(times, t) - 1
    al = (times[i + 1] - t) / (times[i + 1] - times[i])
    return al * values[i] + (1.0 - al) * values[i + 1], i, al


def warm_start(prev_times, x_prev, u_prev, new_times, x0, new_modes, mass):
    """SqpSolver::initializeStateInputTrajectories from the previous solution (its node times prev_times, states x_prev, inputs u_prev)
    onto the node times new_times: interval i interpolates the previous solution while t_{i+1} <= t_end + 1e-9 (t_end the previous
    final time), u_i = previous input at t_i (the input trajectory repeats its last sample at the final node) and x_{i+1} = previous state at
    t_{i+1}; from the first interval past it on, the initializer (state kept, weight-compensating input of the interval's mode). x[0] is
    the measured state x0 (DESIGN §2 deviation 1)."""
    n = len(new_times) - 1
    u_ext = np.vstack([u_prev, u_prev[-1:]])
    t_end = prev_times[-1]
    x = np.zeros((n + 1, 22)); u = np.zeros((n, 22))
    x[0] = x0
    fallback = False
    for i in range(n):
        fallback = fallback or new_times[i + 1] > t_end + 1e-9
        if fallback:
            u[i] = initializer_input(new_modes[i], mass)
            x[i + 1] = x[i]
        else:
            u[i] = interpolate(new_times[i], prev_times, u_ext)[0]
            x[i + 1] = interpolate(new_times[i + 1], prev_times, x_prev)[0]
    return x, u


def evaluate_policy(times, x, u, node_modes, t):
    """MPC_MRT_Interface::evaluatePolicy with the feed-forward controller on a solution with node times `times` (n + 1 of them), states
    x (n + 1), inputs u (n), node modes: (x(t), u(t), node rule mode). x and u: LinearInterpolation on the node times, the input trajectory
    repeating its last sample, clamped before the first node and after the last. The node rule gives the mode of the node starting the
    interval LinearInterpolation picks (at an interior node: the interval ending there). Where the grid has every switch as a node this
    is modeAtTime(t) (mode_at_time); on a uniform grid, and over the stretched last interval of a capacity-exhausted grid, a switch between
    two nodes is not seen before the next node (DESIGN §2 item 2)."""
    n = len(times) - 1
    xs, i, _ = interpolate(t, times, x)
    us = interpolate(t, times, np.vstack([u, u[-1:]]))[0]
    return xs, us, int(node_modes[i])
