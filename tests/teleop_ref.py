"""Teleoperation (hb_rollout_set_teleop) restated for its tests: the message rule and the publisher step in numpy, and TeleopLoop, the
context episode_ref.stepwise runs on to restate an episode with teleop (and goals) set through public calls. Float64 min, max and add are
exact, so the restated publisher reproduces the device's filtered command bit for bit."""
import numpy as np

import hunter_bipedal_control_b200 as hb


def message_due(s, a):
    """Whether the joystick of HbTeleopSetting s sends a message on absolute tick a: inside a window [on, off), on the period from its on."""
    return any(s.on_tick[w] <= a < s.off_tick[w] and (a - s.on_tick[w]) % s.period_ticks == 0 for w in range(s.n_window))


def publisher_step(last, cmd, limit):
    """TargetTrajectoriesPublisher's cmdVelCallback on the filtered command last (vx, vy, vz, yaw rate) for the message cmd, with the
    change limits (vx, vy, yaw rate): each change clipped, vx, vy and the yaw rate in that order, vz set to 0. Returns the new last."""
    out = [float(v) for v in last]
    for k, lim in ((0, limit[0]), (1, limit[1]), (3, limit[2])):
        d = float(cmd[k]) - out[k]
        d = min(d, lim) if d > 0 else max(d, -lim)
        out[k] += d
    out[2] = 0.0
    return np.array(out)


def publish(s, cmds, ticks):
    """The filtered commands of the record s after the messages of absolute ticks `ticks`, cmds[k] the cmd_vel at ticks[k]: (ticks of
    the messages, the filtered command after each)."""
    last, sent, lasts = np.zeros(4), [], []
    for a, c in zip(ticks, cmds):
        if message_due(s, a):
            last = publisher_step(last, c, s.change_limit)
            sent.append(a); lasts.append(last)
    return sent, np.array(lasts).reshape(-1, 4)


class TeleopLoop:
    """The context episode_ref.stepwise runs on to restate an episode with teleop (`teleop`, the records set on ctx) and goals (`goals`,
    the schedules set on ctx; stepwise then gets none): each resident_plan_cycle call of an MPC tick runs, per instance, the goal capture
    (a teleoperated instance compares the goal in force with the one it last saw), then the message due on the tick (publisher_step on the
    tick's cmd_vel), and plans on cmd_vel = last for the teleoperated instances. Every instance gets its target through
    hb_plan_set_targets: the captured one, or the cmd_vel target of its (filtered) command. Both come from the device planner with
    joint_ik = 0, as stepwise takes the plain cmd_vel targets: cmd_vel_to_target computes the same target on the host with libm's
    trigonometry, which the device's differs from in the last bits. Every other call goes to ctx."""

    def __init__(self, ctx, teleop, period, goals=None):
        self._ctx, self._teleop, self._goals, self._period = ctx, teleop, goals, period
        self.last = {}                                  # teleoperated instance: its filtered command
        self._seen, self._src, self._tg = {}, {}, {}    # the goal it last saw; the source of its captured target ("msg" or a goal), the target

    def __getattr__(self, name):
        return getattr(self._ctx, name)

    def resident_plan_cycle(self, cold_start, t_rel, ins, rbd):
        B = len(ins)
        v = np.ctypeslib.as_array(ins)
        t = float(v["t0"][0])
        a = int(round(t / self._period))
        if cold_start:
            self.last, self._seen, self._src, self._tg = {}, {}, {}, {}
        x0 = v["x0"].copy()
        tele = [i for i in range(min(B, len(self._teleop)))]
        msg = []
        for i in range(B):
            if i < len(self._goals or []):
                s = self._goals[i]
                g = max([j for j in range(s.n_goal) if s.time[j] <= t], default=-1)
                had = self._seen.get(i, -1) if i in tele else self._src.get(i, -1)
                if g >= 0 and g != had:
                    self._src[i], self._tg[i] = g, hb.goal_to_target(t, x0[i:i + 1], np.array(s.goal[g][:]))[0]
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
