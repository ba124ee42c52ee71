"""Height maps for their tests (test_height_maps_host.py, test_gpu_height_maps.py): map builders, oracle/refs.py's planner with a map
(the rules of hunter_b200.h's "height maps" on top of the oracle's own planner), numpy restatements of the two target conversions, and
MapLoop, the context episode_ref.stepwise runs on to restate an episode whose goals and teleop targets are built on maps.

The map lookup h(x, y) is episode_ref.terrain_height: Python floats round every product on its own, as the planner's lookup does."""
import math

import numpy as np

import hunter_bipedal_control_b200 as hb
from episode_ref import terrain_height
from oracle import refs as R
from teleop_ref import message_due, publisher_step

COM = R.COM_HEIGHT


def h(m, x, y):
    """h(x, y) of the height map m (an HbTerrain), 0 without one."""
    return 0.0 if m is None else terrain_height(m, float(x), float(y))[0]


# ---------------------------------------------------------------------------------------------------------------- maps
def plateau(B, c):
    """B flat maps at height c."""
    return hb.make_terrains(B, np.full((2, 2), float(c)), 1.0, (-1.0, -1.0))


def step_map(B, x_step, rise, spacing=0.02, n=64, origin=(-0.6, -0.64)):
    """B maps with a step of `rise` along world x at x_step (a one-cell ramp), flat on either side."""
    xs = origin[0] + spacing * np.arange(n)
    row = np.where(xs >= x_step, rise, 0.0)
    return hb.make_terrains(B, np.tile(row, (n, 1)), spacing, origin)


def slope_map(B, grade, spacing=0.05, n=40, origin=(-1.0, -1.0), axis=0):
    """B maps rising at `grade` (dz / ds) along world x (axis 0) or y (axis 1) through the origin of the grid's centre."""
    s = origin[axis] + spacing * np.arange(n)
    z = grade * s
    hm = np.tile(z, (n, 1)) if axis == 0 else np.tile(z[:, None], (1, n))
    return hb.make_terrains(B, hm, spacing, origin)


def random_maps(B, seed, scale=0.05, spacing=0.07, n=24, origin=(-0.8, -0.8)):
    """B maps of independent random heights in [-scale, scale]."""
    rng = np.random.default_rng(seed)
    return hb.make_terrains(B, rng.uniform(-scale, scale, (B, n, n)), spacing, origin)


def zero_maps(B, n=5, spacing=0.3, origin=(-0.5, -0.5)):
    return hb.make_terrains(B, np.zeros((n, n)), spacing, origin)


# ---------------------------------------------------------------------------------------------------------------- the planner on a map
class MappedSwingPlanner(R.SwingPlanner):
    """oracle/refs.py's SwingTrajectoryPlanner with the map m: lift-off and touch-down on the map, the swing z shape built above the lower
    end's ground, the centrifugal term on the body height above the map."""

    def __init__(self, m, latest_stance=None):
        super().__init__(latest_stance)
        self.m = m

    def next_foot_pos(self, foot, current_time, stop_time, next_middle_time, next_middle_body_pos, current_body_pos, current_body_vel):
        cur = np.array(current_body_pos, dtype=float)
        cur[2] = cur[2] - h(self.m, cur[0], cur[1])         # only the centrifugal term reads z; r.z is replaced below
        r = super().next_foot_pos(foot, current_time, stop_time, next_middle_time, next_middle_body_pos, cur, current_body_vel)
        r[2] = R.NEXT_Z + h(self.m, r[0], r[1])
        return r

    def swing_splines(self, t0, t1, a, b):
        h_lo = min(a[2], b[2]) - R.NEXT_Z
        a, b = np.array(a, dtype=float), np.array(b, dtype=float)
        a[2] = a[2] - h_lo; b[2] = b[2] - h_lo
        out = R.SwingPlanner.swing_splines(t0, t1, a, b)
        out[2] = R.MultiCubicSpline([(t, p + h_lo, v) for t, p, v in out[2].nodes])
        return out

    def update(self, ms, target, init_time):
        """SwingPlanner.update with every lift-off point on the map."""
        self.events = ms.events
        legs = R.stance_legs(ms.mode_at(init_time + 0.001))
        for i in range(4):
            if legs[i]:
                self.latest[i] = self.current_feet[i]
            self.latest[i][2] = R.NEXT_Z + h(self.m, self.latest[i][0], self.latest[i][1])
        last, nxt = self.latest.copy(), self.latest.copy()
        n = len(ms.modes)
        self.trajs = [[None] * n for _ in range(4)]
        for j in range(4):
            flags = [R.stance_legs(md)[j] for md in ms.modes]
            last_final = 0
            for p in range(n):
                si, fi = R.find_index(p, flags)
                if not flags[p]:
                    if si < 0 or fi >= n - 1:
                        raise RuntimeError("swing phase without take-off / touch-down")
                    ts, tf = ms.events[si], ms.events[fi]
                    if init_time < tf and fi > last_final:
                        last[j] = nxt[j]
                        if fi < n - 1:
                            _, fi2 = R.find_index(fi + 1, flags)
                            mid = 0.5 * (tf + ms.events[fi2])
                        else:
                            mid = tf
                        nxt[j] = self.next_foot_pos(j, init_time, tf, mid, target.state(mid)[6:12], target.state(init_time)[6:12], target.states[0][0:3])
                        last_final = fi
                    self.trajs[j][p] = self.swing_splines(ts, tf, last[j].copy(), nxt[j].copy())
                else:
                    ts, tf = ms.events[si], ms.events[fi]
                    self.trajs[j][p] = [R.MultiCubicSpline([(ts, nxt[j][a], 0.0), (tf, nxt[j][a], 0.0)]) for a in range(3)] if tf > ts else None


def body_height(m, pose):
    """z' of the targets: the pose's height moved towards HB_COM_HEIGHT above the map, by at most 0.04."""
    dz = COM + h(m, pose[0], pose[1]) - pose[2] if m is not None else COM - pose[2]
    dz = min(dz, 0.04) if dz > 0 else max(dz, -0.04)
    return pose[2] + dz


def cmd_vel_target_oracle(m, cmd, time, state, time_to_target):
    """oracle/refs.py's cmd_vel target with both samples' body heights on the map m."""
    tg = R.cmd_vel_to_target(cmd, time, state, time_to_target)
    if m is not None:
        tg.states[0][8] = body_height(m, state[6:12])
        tg.states[1][8] = COM + h(m, tg.states[1][6], tg.states[1][7])
    return tg


def plan(m, t0, horizon, x0, cmd_vel, feet_pos, gait, gait_start, prev_event=None, time_to_target=None, latest_stance=None, joint_ik=True):
    """oracle/refs.py's plan on the map m (None: refs.plan itself): (ModeSchedule, Target, MappedSwingPlanner) after update."""
    if m is None:
        return R.plan(t0, horizon, x0, cmd_vel, feet_pos, gait, gait_start, prev_event, time_to_target, latest_stance, joint_ik)
    prev_event = min(t0, gait_start) - 0.5 if prev_event is None else prev_event
    ttt = horizon if time_to_target is None else time_to_target
    ms = R.gait_schedule(gait, prev_event, gait_start, t0 + 2 * horizon)
    tg = cmd_vel_target_oracle(m, cmd_vel, t0, x0, ttt)
    sp = MappedSwingPlanner(m, latest_stance)
    sp.body_vel_cmd = np.array([cmd_vel[0], cmd_vel[1], cmd_vel[2], cmd_vel[3], 0.0, 0.0])
    sp.current_feet = np.array(feet_pos, dtype=float).reshape(4, 3)
    sp.update(ms, tg, t0)
    if joint_ik:
        tg = R.joint_references(sp, tg, t0, t0 + horizon, np.asarray(x0, dtype=float))
    return ms, tg, sp


# ---------------------------------------------------------------------------------------------------------------- the conversions
def goal_target_numpy(m, t, x, goal):
    """(times, states) of hb_goal_to_target_maps for one instance, in Python floats with every operation rounded on its own."""
    pose = [float(v) for v in x[6:12]]
    z = body_height(m, pose)
    zg = z + (h(m, goal[0], goal[1]) - h(m, pose[0], pose[1])) if m is not None else z
    dx, dy = float(goal[0]) - pose[0], float(goal[1]) - pose[1]
    reach = max(abs(float(goal[2]) - pose[3]) / R._header_value("HB_TARGET_ROTATION_VELOCITY"),
                math.sqrt(dx * dx + dy * dy) / R._header_value("HB_TARGET_DISPLACEMENT_VELOCITY"))
    cur = [pose[0], pose[1], z, pose[3], 0.0, 0.0]
    tgt = [float(goal[0]), float(goal[1]), zg, float(goal[2]), 0.0, 0.0]
    rows = [cur, tgt] if reach > 0.0 else [tgt]
    states = np.zeros((len(rows), 22))
    for k, p in enumerate(rows):
        states[k, 6:12] = p; states[k, 12:] = R.DEFAULT_JOINTS
    return np.array([t, t + reach][:len(rows)]), states


def cmd_vel_heights_numpy(m, x, sample1_xy):
    """The two body heights of hb_cmd_vel_to_target_maps for one instance whose sample 1 lies at sample1_xy."""
    return body_height(m, [float(v) for v in x[6:12]]), COM + h(m, *sample1_xy)


# ---------------------------------------------------------------------------------------------------------------- episodes
class MapLoop:
    """The context episode_ref.stepwise runs on to restate an episode with height maps set on ctx (`maps`), goals (`goals`, the schedules
    set on ctx) and teleoperation (`teleop`, the records set on ctx; `period` the tick period). The device planner calls read ctx's maps
    themselves; this restates the captures of rollout_plan_inputs_kernel: goals converted by hb_goal_to_target_maps on the robot's map, and
    the teleop messages' targets and the cmd_vel targets of the other robots taken from the device planner's joint_ik = 0 plan on the maps
    (the host conversion's libm trigonometry differs from the device's in the last bits). Every instance gets its target through
    hb_plan_set_targets. Every other call goes to ctx."""

    def __init__(self, ctx, maps, period, goals=None, teleop=None):
        self._ctx, self._maps, self._goals, self._period = ctx, maps, goals, period
        self._teleop = teleop if teleop is not None else []
        self.last, self._seen, self._src, self._tg = {}, {}, {}, {}

    def __getattr__(self, name):
        return getattr(self._ctx, name)

    def _map(self, i):
        return self._maps[i] if i < len(self._maps) else None

    def resident_plan_cycle(self, cold_start, t_rel, ins, rbd):
        B = len(ins)
        v = np.ctypeslib.as_array(ins)
        t = float(v["t0"][0])
        a = int(round(t / self._period))
        if cold_start:
            self.last, self._seen, self._src, self._tg = {}, {}, {}, {}
        x0 = v["x0"].copy()
        tele = range(min(B, len(self._teleop)))
        msg = []
        for i in range(B):
            if i < len(self._goals or []):
                s = self._goals[i]
                g = max([j for j in range(s.n_goal) if s.time[j] <= t], default=-1)
                had = self._seen.get(i, -1) if i in tele else self._src.get(i, -1)
                if g >= 0 and g != had:
                    m = self._map(i)
                    self._src[i] = g
                    self._tg[i] = hb.goal_to_target(t, x0[i:i + 1], np.array(s.goal[g][:]), maps=None if m is None else (hb.HbTerrain * 1)(m))[0]
                if i in tele:
                    self._seen[i] = g if g >= 0 else had
            if i in tele:
                last = self.last.get(i, np.zeros(4))
                if message_due(self._teleop[i], a):
                    last = publisher_step(last, v["cmd_vel"][i], self._teleop[i].change_limit)
                    msg.append(i)
                self.last[i] = last
                v["cmd_vel"][i] = last
        self._ctx.set_plan_targets(None)
        plain_in = hb.make_plan_inputs(v["t0"], v["horizon"][0], x0, v["cmd_vel"], None, v["gait"], v["gait_start"], v["prev_event"],
                                       v["time_to_target"], joint_ik=False)
        plain, _, pst = self._ctx.plan_references_gpu(plain_in, np.zeros((B, 12)))
        assert (pst == 0).all()
        targets = [hb.reference_target(r) for r in plain]
        for i in msg:
            self._src[i], self._tg[i] = "msg", targets[i]
        for i in self._tg:
            targets[i] = self._tg[i]
        self._ctx.set_plan_targets((hb.HbTarget * B)(*targets))
        return self._ctx.resident_plan_cycle(cold_start, t_rel, ins, rbd)
