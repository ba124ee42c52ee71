#!/usr/bin/env python3
"""Teleoperation sweep of the episodes (hb_rollout_set_teleop): prints one JSON line.

  python tools/teleop_sweep.py [--repeats R] [--timed K] [--batch B] [--wbc weighted|hierarchical]

B robots (default 1024) from the randomised poses of bench.py's configs[1] trot in place from t = 0.1 s; at t = 1 s each gets one command
step, a forward velocity of 0.1 .. 0.6 m/s or a yaw rate of 0.75 or 1.5 rad/s (the robots are spread over the eight steps, the
assignment shifting between the R repeats), and runs to t = 3 s, once on the true state and once through the state estimator (sensor
noise at 1 x NOISE_SIGMAS of episode_harness.py). Each repeat runs the batch once per publisher:
  unset      no setting: the command segment in force reaches the planner as it is, its target rebuilt on every MPC tick;
  default    hb_default_teleop_setting: messages at 10 Hz, the change per message limited to 0.1 m/s, 0.05 m/s and 0.3 rad/s, each
             message converted once into a target;
  unlimited  the default joystick without a change limit.
Per step and publisher: survival (robots up at the end), the RMS tracking error of the robots up over the last second (body-frame
horizontal velocity against the step for forward steps, world yaw rate against it for yaw steps), and the time from the step until the
0.1 s moving average of the forward speed or yaw rate first reaches 90 % of the step (mean over the robots up that reach it, and the
share that do). The line also times, alternately, episodes with every robot on a record that never fires (no window), on a record that
fires on every MPC tick, and with no setting, through the estimator. All with the card's name and power limit.
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import NOISE_SIGMAS, Episodes, Tally, failure_checks, report, sweep_args, workload  # noqa: E402
from bench import SEED, ClockSampler  # noqa: E402  (episode_harness put the repository root on the path)

TICKS, LOG_EVERY, T_STEP = 1500, 5, 1.0              # 3 s, logged every 10 ms, the step at 1 s
STEPS = [("vx", 0.1), ("vx", 0.2), ("vx", 0.3), ("vx", 0.4), ("vx", 0.5), ("vx", 0.6), ("yaw", 0.75), ("yaw", 1.5)]
PUBLISHERS = ["unset", "default", "unlimited"]
SMOOTH = 0.1                                          # [s] the moving average of the rise time


def publisher(hb, name, B):
    if name == "unset":
        return None
    return hb.make_teleop_settings(B) if name == "default" else hb.make_teleop_settings(B, change_limit=[float("inf")] * 3)


def main():
    args = sweep_args("teleop_sweep.py", "timed rounds of the never-firing record, the every-MPC-tick record and no setting", len(STEPS),
                      repeats=1)
    h = Episodes("teleop_sweep.py", args, TICKS)
    hb, ctx, B = h.hb, h.ctx, h.B
    rows = (TICKS + LOG_EVERY - 1) // LOG_EVERY
    t_log = np.arange(rows) * LOG_EVERY * h.prm.period
    after, last_second = t_log >= T_STEP, t_log >= t_log[-1] - 1.0 + 1e-9
    win = int(round(SMOOTH / (LOG_EVERY * h.prm.period)))
    line = {"metric": "teleop sweep: survival of %d robots per step and publisher after a command step at t = %.0f s" % (B // len(STEPS) * args.repeats, T_STEP),
            "unit": "fraction surviving", "steps": ["%s %.2f" % s for s in STEPS], "publishers": PUBLISHERS}
    for estimated in (False, True):
        args.estimator = estimated
        for k, v in NOISE_SIGMAS.items():
            setattr(h.ep.noise, k, v if estimated else 0.0)
        tally = Tally(len(STEPS), len(PUBLISHERS))
        err_sum, err_n = np.zeros((len(PUBLISHERS), len(STEPS))), np.zeros((len(PUBLISHERS), len(STEPS)))
        rise_sum, rise_n, rise_of = (np.zeros((len(PUBLISHERS), len(STEPS))) for _ in range(3))
        for r in range(args.repeats):
            col = (np.arange(B) + r) % len(STEPS)
            v = np.zeros((B, 2, 4))
            for c, (kind, size) in enumerate(STEPS):
                v[col == c, 1, 0 if kind == "vx" else 3] = size
            h.cmds = hb.make_rollout_commands("trot", np.full(B, 0.1), [0.0, T_STEP], v)
            if r == 0:
                h.episode(log_every=LOG_EVERY)                               # warm-up
            for p, name in enumerate(PUBLISHERS):
                ctx.set_teleop(publisher(hb, name, B))
                run = h.episode(log_every=LOG_EVERY)
                tally.add(col, np.full(B, p), run.stats)
                up = run.stats["fail_tick"] < 0
                log = run.log
                yaw = log[:, :, 0]
                vx = np.cos(yaw) * log[:, :, 19] + np.sin(yaw) * log[:, :, 20]
                vy = -np.sin(yaw) * log[:, :, 19] + np.cos(yaw) * log[:, :, 20]
                wz = log[:, :, 18]
                fwd = np.array([STEPS[c][0] == "vx" for c in col])
                target = np.array([STEPS[c][1] for c in col])[:, None]
                e2 = np.where(fwd[:, None], (vx - target) ** 2 + vy ** 2, (wz - target) ** 2)[:, last_second]
                speed = np.where(fwd[:, None], vx, wz)
                kernel = np.ones(win) / win
                avg = np.array([np.convolve(s, kernel, mode="full")[:rows] for s in speed])
                reached = (avg >= 0.9 * target) & after[None, :]
                has = reached.any(axis=1)
                rise = np.where(has, t_log[np.argmax(reached, axis=1)] - T_STEP, 0.0)
                np.add.at(err_sum[p], col[up], e2[up].sum(axis=1)); np.add.at(err_n[p], col[up], e2.shape[1])
                np.add.at(rise_sum[p], col[up & has], rise[up & has]); np.add.at(rise_n[p], col[up & has], 1)
                np.add.at(rise_of[p], col[up], 1)
        ctx.set_teleop(None)
        key = "estimator" if estimated else "truth"
        steps = ["%s %.2f" % s for s in STEPS]
        line[key] = {"survival": {name: dict(zip(steps, tally.survival()[p].tolist())) for p, name in enumerate(PUBLISHERS)},
                     "tracking_err_rms_last_second": {name: dict(zip(steps, [float(np.sqrt(s / n)) if n else None for s, n in zip(err_sum[p], err_n[p])]))
                                                     for p, name in enumerate(PUBLISHERS)},
                     "time_to_90pct_s": {name: dict(zip(steps, [float(s / n) if n else None for s, n in zip(rise_sum[p], rise_n[p])]))
                                         for p, name in enumerate(PUBLISHERS)},
                     "share_reaching_90pct": {name: dict(zip(steps, (rise_n[p] / np.maximum(rise_of[p], 1)).tolist())) for p, name in enumerate(PUBLISHERS)},
                     "wbc_fallbacks_per_robot": {name: (tally.fallbacks[p] / np.maximum(tally.total[p], 1)).tolist() for p, name in enumerate(PUBLISHERS)},
                     "fail_reasons": tally.reasons}
    line["value"] = line["estimator"]["survival"]["default"]["vx 0.50"]

    # timing through the estimator: a record that never fires, one that fires on every MPC tick, and no setting, alternated
    sampler = ClockSampler(args.device); sampler.start()
    never, every = hb.make_teleop_settings(B, windows=[]), hb.make_teleop_settings(B, h.prm.mpc_every)
    ms, launches = {"never_fires": [], "every_mpc_tick": [], "unset": []}, {}
    for _ in range(max(1, args.timed)):
        for name, value in (("never_fires", never), ("every_mpc_tick", every), ("unset", None)):
            ctx.set_teleop(value)
            run = h.episode()
            ms[name].append(run.ms); launches[name] = int(run.launches)
    timing = {}
    for name, v in ms.items():
        timing["ms_per_episode_" + name] = float(np.median(v)); timing["ms_per_episode_%s_range" % name] = [min(v), max(v)]
    for name in ("never_fires", "every_mpc_tick"):
        timing["%s_minus_unset_ms" % name] = timing["ms_per_episode_" + name] - timing["ms_per_episode_unset"]
    timing["rounds"] = max(1, args.timed)
    timing["launches_equal"] = len(set(launches.values())) == 1
    line["timing"] = timing
    line.update(report(args, sampler.stop(), estimator=False))
    line["config"] = {"workload": workload(h, "; %d robots per step, each publisher on the whole batch, %d repeats" % (B // len(STEPS), args.repeats),
                                           motion="trot in place from t = 0.1 s, one command step at t = %.0f s" % T_STEP,
                                           robots="robots, on the true state and through the estimator"),
                      "noise_sigmas_estimator": NOISE_SIGMAS, "noise_seed": SEED, "survival": "robots up at the end of the episode",
                      "failure_checks": failure_checks(), "timing": "through the estimator"}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
