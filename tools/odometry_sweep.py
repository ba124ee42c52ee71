#!/usr/bin/env python3
"""Odometry sweep of the estimated episodes (hb_rollout_set_odometry + hb_rollout_estimated_batch_dev): prints one JSON line.

  python tools/odometry_sweep.py [--batch B] [--timed K] [--sensor-noise SCALE] [--settle S] [--wbc hierarchical]

The goal workload of tools/goal_sweep.py through the state estimator (B robots, default 1024, from the randomised poses of bench.py's
configs[1], trotting with cmd_vel 0 from t = 0.1 s; at t = GOAL_TIME each robot is given a goal 0.5 m or 1 m away in one of 8 headings, 16
cells sharing the batch; sensor noise SCALE x NOISE_SIGMAS, default 1). The episode runs until GOAL_TIME + 2 s (the 1 m goal's reaching time)
+ --settle seconds. Every robot of an episode gets the same tracking camera; the sweep runs one episode without a camera, then every camera
of PERIODS x DELAYS x POSITION_NOISE and DRIFTING. Per camera: survival and, over the survivors, the final goal error per distance (median and
90th percentile of the horizontal distance, the fraction within 5 cm and 0.1 rad), and the estimate's horizontal position error against
the true state over the episode (est_log against log, every LOG_EVERY-th tick while the robot is up: rms and max), beside the same numbers
without a camera from the same invocation.

The line also times, in the same invocation, a camera (100 Hz, 5 mm) against all-period-0 records and no setting, alternately, with device
events around the episode call, and reports the launch counts of the three (odometry adds no launch), whether the period-0 records give
the outcome of no setting, and the card's name and power limit and the clocks sampled during the timed episodes.
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import Episodes, cells, failure_checks, parser, report, sensor_noise, workload  # noqa: E402

DISTANCES = [0.5, 1.0]                                   # [m]
HEADINGS = [k * 45.0 for k in range(8)]                  # [deg], world frame
GOAL_TIME = 0.5                                          # [s]
V_DISP = 0.5                                             # targetDisplacementVelocity (reference.info:1)
PERIODS = [1, 5, 15]                                     # [ticks]: 500 / 100 / 33 Hz at 2 ms
DELAYS = [0, 5, 15]                                      # [ticks]
POSITION_NOISE = [0.0, 0.005, 0.02]                      # [m]
DRIFTING = dict(period_ticks=5, delay_ticks=5, sigma_position=0.005, sigma_drift=0.001)
LOG_EVERY = 10


def main():
    ncell = len(DISTANCES) * len(HEADINGS)
    ap = parser("robots per episode (a multiple of %d)" % ncell)
    ap.set_defaults(estimator=True, sensor_noise=1.0)
    ap.add_argument("--timed", type=int, default=3, help="timed camera / period-0 / unset episode triples")
    ap.add_argument("--settle", type=float, default=2.0, metavar="S", help="seconds after the 1 m goal's reaching time")
    args = ap.parse_args()
    if args.batch < ncell or args.batch % ncell or args.sensor_noise < 0 or not args.settle >= 0.0:
        raise SystemExit("odometry_sweep.py: --batch a multiple of %d, --sensor-noise >= 0, --settle >= 0" % ncell)
    args.estimator = True
    T_episode = GOAL_TIME + max(DISTANCES) / V_DISP + args.settle
    h = Episodes("odometry_sweep.py", args, 0)
    hb, ctx, prm, B, rbd0 = h.hb, h.ctx, h.prm, h.B, h.rbd0
    h.ticks = int(round(T_episode / prm.period))
    h.cmds = hb.make_rollout_commands("trot", np.full(B, 0.1), [0.0], [[0.0, 0.0, 0.0, 0.0]])
    di, hi = cells(B, len(DISTANCES), len(HEADINGS), 0)
    d, th = np.array(DISTANCES)[di], np.radians(np.array(HEADINGS)[hi])
    goal = np.c_[rbd0[:, 3] + d * np.cos(th), rbd0[:, 4] + d * np.sin(th), rbd0[:, 0]]
    ctx.set_goals(hb.make_goal_schedules(B, GOAL_TIME, goal[:, None, :]))
    n_log = -(-h.ticks // LOG_EVERY)

    def summary(setting):
        ctx.set_odometry(setting)
        run = h.episode(log_every=LOG_EVERY, est_log=True)
        st, rbd, log, est_log = run.stats, run.rbd, run.log, run.est_log
        up = st["fail_tick"] < 0
        pe = np.hypot(rbd[:, 3] - goal[:, 0], rbd[:, 4] - goal[:, 1])
        ye = np.abs(np.mod(rbd[:, 0] - goal[:, 2] + np.pi, 2 * np.pi) - np.pi)
        out = {"survival": float(up.mean())}
        for a, dist in enumerate(DISTANCES):
            sel = up & (di == a)
            p, y = pe[sel], ye[sel]
            out[str(dist)] = {"survival": float((di == a)[up].sum() / (di == a).sum())}
            if len(p):
                out[str(dist)].update({"pos_err_median_m": float(np.median(p)), "pos_err_p90_m": float(np.percentile(p, 90)),
                                       "within_5cm_0.1rad": float(((p < 0.05) & (y < 0.1)).mean())})
        # the estimate's horizontal error on the logged ticks before each robot's failure (all of them for survivors)
        rows = np.arange(n_log) * LOG_EVERY
        alive = np.where(st["fail_tick"][:, None] < 0, True, rows[None, :] < st["fail_tick"][:, None])
        exy = np.hypot(est_log[:, :, 3] - log[:, :, 3], est_log[:, :, 4] - log[:, :, 4])[alive]
        out["est_xy_err_rms_m"] = float(np.sqrt(np.mean(exy ** 2)))
        out["est_xy_err_max_m"] = float(exy.max())
        return out

    summary(None)                                       # warm-up episode
    results = {"none": summary(None)}
    for per in PERIODS:
        for dly in DELAYS:
            for sp in POSITION_NOISE:
                results["period %d / delay %d / noise %g m" % (per, dly, sp)] = summary(hb.make_odometry_settings(B, per, dly, sp))
    results["period %(period_ticks)d / delay %(delay_ticks)d / noise %(sigma_position)g m / drift %(sigma_drift)g m" % DRIFTING] = \
        summary(hb.make_odometry_settings(B, **DRIFTING))

    # camera, period-0 records and no setting alternate
    runs, clocks, timing = h.alternate(ctx.set_odometry, [("odometry", hb.make_odometry_settings(B, 5, 0, 0.005)),
                                                          ("zero_periods", hb.make_odometry_settings(B, 0)), ("unset", None)], args.timed,
                                       launches=True)
    print(json.dumps({
        "metric": "odometry: fraction of the surviving robots within 5 cm and 0.1 rad of a goal 0.5 m away through the estimator with a "
                  "100 Hz, 5 mm tracking camera", "value": results["period 5 / delay 0 / noise 0.005 m"]["0.5"].get("within_5cm_0.1rad"),
        "unit": "fraction", **report(args, clocks, estimator=False), "cameras": results, "timing": timing,
        "config": {"workload": workload(h, ", through the estimator", "trot with cmd_vel 0 from t = 0.1 s", T_episode, 2),
                   "goal": "given at t = %g s: start position + d (cos h, sin h), d in %s m, h in 8 headings, start yaw" % (GOAL_TIME, DISTANCES),
                   "errors": "goal: over the robots still up at the end; estimate: |est xy - true xy| every %d ticks while up" % LOG_EVERY,
                   "failure_checks": failure_checks()},
        **sensor_noise(args)}))


if __name__ == "__main__":
    main()
