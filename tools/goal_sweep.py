#!/usr/bin/env python3
"""Goal sweep of the closed-loop episodes (hb_rollout_set_goals + hb_rollout_batch_dev): prints one JSON line.

  python tools/goal_sweep.py [--repeats R] [--timed K] [--batch B] [--yaw-change RAD] [--settle S] [--estimator [--sensor-noise SCALE]]
                             [--wbc hierarchical]

The workload of tools/bench_rollout.py (B robots, default 1024, from the randomised poses of bench.py's configs[1], N = 100, dt = 10 ms,
ground at 0.02 m, failure below a base height of 0.3 m), trotting from t = 0.1 s with cmd_vel 0, so that only the goal moves them. At
t = GOAL_TIME every robot is given one goal (hb_goal_schedule): its start position moved by a distance d along a world heading h, and its
start yaw turned by --yaw-change. The 32 cells (4 distances x 8 headings) share the batch, 1/32 of the robots each; episode r of R shifts
the assignment by r. The episode runs until GOAL_TIME + the longest reaching time (goalToTargetTrajectories: max(|dyaw| / 1.57,
d / 0.5)) + --settle seconds. Per distance (over the headings) and per cell: survival, and over the survivors the final position error
(horizontal distance of the base origin from the goal) and yaw error (wrapped), median and 90th percentile, and the fraction within
5 cm and 0.1 rad.

The line also times, in the same invocation, the goal batch against the same batch with zero-goal schedules and with no goals set,
alternately, with device events around the episode call, and reports the launch counts of the three (goals add no launch), whether
zero-goal schedules and unset give the same outcome, and the card's name and power limit and the clocks sampled during the timed
episodes.
"""
import json
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import GROUND, Episodes, Tally, cells, failure_checks, report, sweep_args, workload  # noqa: E402

DISTANCES = [0.25, 0.5, 1.0, 2.0]                        # [m]
HEADINGS = [k * 45.0 for k in range(8)]                  # [deg], world frame
GOAL_TIME = 0.5                                          # [s]
V_DISP, V_ROT = 0.5, 1.57                                # targetDisplacementVelocity, targetRotationVelocity (reference.info:1-2)


def main():
    def extra(ap):
        ap.add_argument("--yaw-change", type=float, default=0.0, metavar="RAD", help="goal yaw - start yaw")
        ap.add_argument("--settle", type=float, default=2.0, metavar="S", help="seconds after the longest reaching time")
    args = sweep_args("goal_sweep.py", "timed goal / zero-goal / unset episode triples", len(DISTANCES) * len(HEADINGS), extra, repeats=1,
                      timed=2, valid=lambda a: a.settle >= 0.0 and math.isfinite(a.yaw_change), needs="--settle >= 0, a finite --yaw-change, ")
    yaw_change, settle = args.yaw_change, args.settle
    reach_max = max(max(DISTANCES) / V_DISP, abs(yaw_change) / V_ROT)
    T_episode = GOAL_TIME + reach_max + settle
    h = Episodes("goal_sweep.py", args, 0)
    hb, ctx, prm, B, rbd0 = h.hb, h.ctx, h.prm, h.B, h.rbd0
    h.ticks = int(round(T_episode / prm.period))
    h.cmds = hb.make_rollout_commands("trot", np.full(B, 0.1), [0.0], [[0.0, 0.0, 0.0, 0.0]])

    def goals_of(shift):
        di, hi = cells(B, len(DISTANCES), len(HEADINGS), shift)
        d, th = np.array(DISTANCES)[di], np.radians(np.array(HEADINGS)[hi])
        g = np.c_[rbd0[:, 3] + d * np.cos(th), rbd0[:, 4] + d * np.sin(th), rbd0[:, 0] + yaw_change]
        return g, di, hi

    def schedules(shift):
        return hb.make_goal_schedules(B, GOAL_TIME, goals_of(shift)[0][:, None, :])

    nd, nh = len(DISTANCES), len(HEADINGS)
    pos_err = [[[] for _ in range(nh)] for _ in range(nd)]
    yaw_err = [[[] for _ in range(nh)] for _ in range(nd)]
    tally = Tally(nh, nd)                       # [distance, heading]
    for r, run in h.sweep(ctx.set_goals, schedules):
        g, di, hi = goals_of(r)
        ok = run.stats["fail_tick"] < 0
        pe = np.hypot(run.rbd[:, 3] - g[:, 0], run.rbd[:, 4] - g[:, 1])
        ye = np.abs(np.mod(run.rbd[:, 0] - g[:, 2] + np.pi, 2 * np.pi) - np.pi)
        tally.add(hi, di, run.stats)
        for i in np.nonzero(ok)[0]:
            pos_err[di[i]][hi[i]].append(float(pe[i])); yaw_err[di[i]][hi[i]].append(float(ye[i]))

    def summary(p, y, n_up, n_total):
        p, y = np.array(p), np.array(y)
        out = {"survival": float(n_up / n_total) if n_total else None, "robots": int(n_total)}
        if len(p):
            out.update({"pos_err_median_m": float(np.median(p)), "pos_err_p90_m": float(np.percentile(p, 90)),
                        "yaw_err_median_rad": float(np.median(y)), "yaw_err_p90_rad": float(np.percentile(y, 90)),
                        "within_5cm_0.1rad": float(((p < 0.05) & (y < 0.1)).mean())})
        return out

    up, total = tally.up, tally.total
    per_distance = {str(d): summary(sum(pos_err[a], []), sum(yaw_err[a], []), up[a].sum(), total[a].sum()) for a, d in enumerate(DISTANCES)}
    per_cell = {"%g m / %g deg" % (d, hd): summary(pos_err[a][b], yaw_err[a][b], up[a, b], total[a, b])
                for a, d in enumerate(DISTANCES) for b, hd in enumerate(HEADINGS)}

    # goal, zero-goal and unset episodes alternate
    none = hb.make_goal_schedules(B, np.zeros((B, 0)), np.zeros((B, 0, 3)))
    runs, clocks, timing = h.alternate(ctx.set_goals, [("goals", schedules(0)), ("zero_goals", none), ("unset", None)], args.timed,
                                       launches=True)
    print(json.dumps({
        "metric": "goals: fraction of the trotting robots within 5 cm and 0.1 rad of a goal 0.5 m away, %.1f s after it is given"
                  % (T_episode - GOAL_TIME), "value": per_distance["0.5"].get("within_5cm_0.1rad"), "unit": "fraction",
        **report(args, clocks), "per_distance": per_distance, "per_cell": per_cell, "fail_reasons": tally.reasons, "timing": timing,
        "config": {"workload": workload(h, "; %d distances x %d headings, %d episodes" % (nd, nh, args.repeats), "trot with cmd_vel 0 from t = 0.1 s",
                                        T_episode, 2),
                   "goal": "given at t = %g s: start position + d (cos h, sin h), start yaw %+g rad; settle %g s after the longest reaching "
                           "time (%g s)" % (GOAL_TIME, yaw_change, settle, reach_max),
                   "errors": "over the robots still up at the end: |base xy - goal xy|, |wrap(base yaw - goal yaw)|",
                   "failure_checks": failure_checks(), "ground_m": GROUND}}))


if __name__ == "__main__":
    main()
