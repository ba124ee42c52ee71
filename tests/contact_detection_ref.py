"""Contact detection restated in numpy from the reference: SwingTrajectoryPlanner::update / updateFootSchedule / findIndex
(SwingTrajectoryPlanner.cpp:164-260, 364-430) store per phase p of each foot the start and stop [eventTimes[startIndex], eventTimes[finalIndex]];
threadSaftyGetStartStopTime (:510-532) picks the phase lookup::findIndexInTimeArray finds for the time, clamped to size - 1; and
StateEstimateBase::estContactState (StateEstimateBase.cpp:208-226) turns the observer's F_z into flags. Where the reference indexes
eventTimes[-1] (a schedule of one phase), and without a plan, the times are [t, t], as hunter_b200.h documents."""
import bisect

import numpy as np

import hunter_bipedal_control_b200 as hb

INITIAL_FORCE = 50.0          # estContactforce_.fill(50) (StateEstimateBase.cpp:61-62)


def contact_flag(mode, c):
    """modeNumber2StanceLeg: contact c (l_f1, r_f1, l_f2, r_f2) is in stance in modes 3 (both legs) and 2 (left) or 1 (right)."""
    return mode in (1, 3) if c & 1 else mode in (2, 3)


def find_index(index, stock):
    """SwingTrajectoryPlanner::findIndex: (startTimesIndex, finalTimesIndex) of phase `index` of one foot's contact flags."""
    n = len(stock)
    start = 0
    for ip in range(index - 1, -1, -1):
        if stock[ip] != stock[index]:
            start = ip
            break
    final = n - 2
    for ip in range(index + 1, n):
        if stock[ip] != stock[index]:
            final = ip - 1
            break
    return start, final


def phase_times(has_plan, events, modes, t):
    """[[s_c, e_c] for c in 0..3]: the start / stop time array of each foot (startStopTime_, one entry per phase) at the phase of t."""
    n = len(events)
    if not has_plan or n < 1:
        return np.full((4, 2), t)
    idx = min(n - 1, bisect.bisect_left(list(events), t))      # lookup::findIndexInTimeArray: std::lower_bound
    out = np.zeros((4, 2))
    for c in range(4):
        stock = [contact_flag(m, c) for m in modes[:n + 1]]
        per_phase = [(events[s], events[f]) for s, f in (find_index(p, stock) for p in range(n + 1))]
        out[c] = per_phase[idx]
    return out


def contact_state(record, t, times, force, cmd):
    """estContactState with the record's threshold and fractions: the flags from the schedule's cmd (4) at t."""
    out = [int(bool(x)) for x in cmd]
    for c in range(4):
        s, e = times[c]
        P = e - s
        fz = force[6 * (c % 2) + 2]
        if not cmd[c] and t - s > record.swing_fraction * P:
            out[c] = int(fz > record.threshold)
        if cmd[c] and t - s < record.stance_fraction * P:
            out[c] = int(fz > record.threshold)
    return out


def schedule_of(st):
    """(has_plan, events, modes) of an HbEstimationState."""
    n = min(st.n_events, hb.api.HB_MAX_EVENTS)
    return st.has_plan, list(st.event_times[:n]), list(st.modes[:n + 1])


def detect(records, t, est, force, cmd):
    """The rule on a batch: est (B HbEstimationState), force [B,16], cmd [B,4]; records None leaves cmd. Returns [B,4] uint8."""
    cmd = np.asarray(cmd, dtype=np.uint8)
    if records is None:
        return cmd.copy()
    return np.array([contact_state(records[i], t, phase_times(*schedule_of(est[i]), t), force[i], cmd[i]) for i in range(len(est))],
                    dtype=np.uint8)


def set_schedule(st, events, modes):
    """Stores the schedule (events, modes) in the HbEstimationState st, with has_plan = 1."""
    st.has_plan = 1
    st.n_events = len(events)
    for k, x in enumerate(events):
        st.event_times[k] = x
    for k, m in enumerate(modes):
        st.modes[k] = m


def schedule_flags(st, t):
    """The schedule's flags at t (the episode's sensor read): mode_at, all 1 without a plan."""
    if not st.has_plan:
        return [1, 1, 1, 1]
    has, ev, md = schedule_of(st)
    m = md[bisect.bisect_left(ev, t)]
    return [int(contact_flag(m, c)) for c in range(4)]
