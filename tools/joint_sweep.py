#!/usr/bin/env python3
"""Joint-model sweep of the closed-loop episodes (hb_rollout_set_joint_models): do range stops and friction loss in the plant change who
falls, and why? Prints one JSON line.

  python tools/joint_sweep.py [--timed K] [--batch B] [--wbc W] [--push FORCE]

The workload of the episode harness (B robots, default 1024, from the randomised poses of bench.py's configs[1], N = 100, dt = 10 ms,
ground at 0.02 m, failure below a base height of 0.3 m), trotting from t = 0.1 s at 0, 0.25 and 0.5 m/s (robot i at speed i mod 3) for
1.5 s (750 ticks), each cell once on the true state and once through the estimator (no sensor noise). --push FORCE also pushes every robot
sideways with FORCE newtons at the base for 0.1 s from t = 0.5 s, the push of push_sweep.py.

Cells (every robot of an episode has the same record): no record; friction only (f = 0.2 N m, v_s = 0.01 rad/s, no stops); stops only
(the default ranges and gains, f = 0); the default record (hb_default_joint_model); and the default stops with the friction loss scaled by
0.5, 2 and 4 (scale 0 is "stops only", 1 the default record). Per cell and speed: survival, the emergency stops, the largest penetration
past a range and the share of robot-ticks with some joint past its range (from the true state logged on every tick, over the robots'
ticks before they fell), and the velocity-tracking error of the survivors: the mean over them of | |horizontal base displacement from
t = 0.5 s to the end| / 1 s - commanded speed |. Fail reasons are counted per cell.

The line also times, in the same invocation, the default record on every robot against all-disabled records (f = 0, no bounds) and no
setting, alternately, with device events around the episode call (median of --timed rounds, default 3), and reports the launch counts of
the three, and the card's name and power limit and the clocks sampled during the timed episodes. It asserts that the disabled records,
and the "no record" cell run after every other cell (the setting cleared), give the unset outcome bit for bit.
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import PUSH_DURATION, PUSH_T, Episodes, failure_checks, parser, report, workload  # noqa: E402

TICKS = 750
SPEEDS = [0.0, 0.25, 0.5]
SCALES = [0.5, 2.0, 4.0]


def records(hb, B):
    """The sweep's cells as (name, B records or None)."""
    inf = float("inf")
    cells = [("none", None), ("friction_only", hb.make_joint_models(B, lower=-inf, upper=inf)), ("stops_only", hb.make_joint_models(B, friction_loss=0.0)),
             ("default", hb.make_joint_models(B))]
    return cells + [("stops_friction_x%g" % s, hb.make_joint_models(B, friction_loss=0.2 * s)) for s in SCALES]


def past_range(hb, log, stats, ticks):
    """(largest penetration past a range [rad], share of robot-ticks with some joint past its range) over each robot's ticks before it fell."""
    d = hb.default_joint_model()
    q = log[:, :, 6:16]
    pen = np.maximum(np.maximum(q - np.array(d.upper[:]), np.array(d.lower[:]) - q), 0.0).max(axis=2)    # B x ticks
    alive = np.arange(ticks)[None, :] < np.where(stats["fail_tick"] < 0, ticks, stats["fail_tick"])[:, None]
    return float(np.where(alive, pen, 0.0).max()), float(((pen > 0) & alive).sum() / max(1, alive.sum()))


def main():
    ap = parser("robots per episode (at least 3)")
    ap.add_argument("--timed", type=int, default=3, help="timed default / disabled / unset episode triples")
    ap.add_argument("--push", type=float, default=0.0, metavar="FORCE", help="push every robot sideways with FORCE [N] at t = 0.5 s for 0.1 s")
    args = ap.parse_args()
    if args.batch < 3 or args.estimator or args.sensor_noise:
        raise SystemExit("joint_sweep.py: --batch >= 3; the sweep runs truth and estimator episodes itself, without sensor noise")
    h = Episodes("joint_sweep.py", args, TICKS)
    hb, ctx, prm, B = h.hb, h.ctx, h.prm, h.B
    speed = np.array(SPEEDS)[np.arange(B) % len(SPEEDS)]
    h.cmds = hb.make_rollout_commands("trot", np.full(B, 0.1), [0.0], np.c_[speed, np.zeros((B, 3))][:, None, :])
    if args.push:
        ctx.set_pushes(hb.make_push_schedules(B, PUSH_T, PUSH_DURATION, [[0.0, args.push, 0.0]]))
    fail = hb.ROLLOUT_FAIL
    t_from = int(round(0.5 / prm.period))
    out = {}
    unset = {}
    cells = records(hb, B)
    for estimated in (False, True):
        mode = "estimator" if estimated else "truth"
        table = {}
        for name, recs in cells[1:] + cells[:1]:           # "none" last: the setting cleared after the others
            ctx.set_joint_models(recs)
            run = h.episode(estimated=estimated, log_every=1)
            if name == "none":
                unset[mode] = run
            row = {}
            for k, v in enumerate(SPEEDS):
                m = speed == v
                st = run.stats[m]
                up = st["fail_tick"] < 0
                pen, share = past_range(hb, run.log[m], st, TICKS)
                disp = np.hypot(*(run.log[m][:, -1, 3:5] - run.log[m][:, t_from, 3:5]).T) / ((TICKS - 1 - t_from) * prm.period)
                row["%g" % v] = {"survival": float(up.mean()), "estops": int(((st["fail_reason"] & fail["estop"]) != 0).sum()),
                                 "fail_reasons": {n: int(((st["fail_reason"] & b) != 0)[~up].sum()) for n, b in fail.items()},
                                 "max_penetration_rad": pen, "ticks_past_range": share,
                                 "speed_error_m_per_s": float(np.abs(disp[up] - v).mean()) if up.any() else None}
            table[name] = row
        out[mode] = table

    # the default record, all-disabled records and no setting alternate (truth episodes)
    inf = float("inf")
    h.args.estimator = False
    disabled = hb.make_joint_models(B, friction_loss=0.0, lower=-inf, upper=inf)
    runs, clocks, timing = h.alternate(ctx.set_joint_models, [("default", hb.make_joint_models(B)), ("disabled", disabled), ("unset", None)],
                                       args.timed, launches=True)
    ref = runs["unset"][-1]
    cleared = unset["truth"]
    timing["cleared_same_outcome_as_unset"] = bool(np.array_equal(cleared.stats, ref.stats) and np.array_equal(cleared.rbd, ref.rbd))
    assert timing["disabled_same_outcome_as_unset"] and timing["cleared_same_outcome_as_unset"], timing
    est_up = {n: float(np.mean([r["survival"] for r in out["estimator"][n].values()])) for n in out["estimator"]}
    print(json.dumps({
        "metric": "robots that fall, and emergency stops, with the plant's joints given range stops and friction loss (%.1f s trot%s)"
                  % (TICKS * prm.period, ", pushed %g N" % args.push if args.push else ""),
        "value": {n: sum(r["estops"] for r in out["truth"][n].values()) for n in out["truth"]}, "unit": "emergency stops per %d robots" % B,
        **report(args, clocks, estimator=False), "truth": out["truth"], "estimator": out["estimator"], "estimator_mean_survival": est_up,
        "timing": timing,
        "config": {"workload": workload(h, "; %d joint-model cells x truth / estimator" % len(cells),
                                        motion="trot at 0, 0.25 and 0.5 m/s from t = 0.1 s" + (", pushed %g N sideways at t = %g s for %g s"
                                                                                                % (args.push, PUSH_T, PUSH_DURATION) if args.push else "")),
                   "cells": "none; friction_only f = 0.2 N m, v_s = 0.01 rad/s, no stops; stops_only: default ranges and gains, f = 0; default: "
                            "hb_default_joint_model; stops_friction_xS: default stops, f = 0.2 S",
                   "failure_checks": failure_checks()}}))


if __name__ == "__main__":
    main()
