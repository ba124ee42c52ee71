#!/usr/bin/env python3
"""Gait sweep of the closed-loop episodes (hb_plan_set_settings): prints one JSON line.

  python tools/gait_sweep.py [--periods LO:HI:N] [--heights LO:HI:N] [--repeats R] [--timed K] [--batch B]
                             [--estimator [--sensor-noise SCALE]] [--wbc weighted|hierarchical]

A grid over the trot template's period (two phases L, R of half a period each; default 0.4 .. 0.8 s in 5 steps, the shipped 0.6 s among
them) x swing_height (default 0.02 .. 0.10 m in 5 steps, the shipped 0.04 m among them), every other planner setting at its shipped value.
The workload of tools/bench_rollout.py (B robots, default 1024, trotting at 0.3 m/s from t = 0.1 s from the randomised poses of bench.py's
configs[1]) runs for 2 s (1000 ticks) in one episode call, the grid's cells sharing the batch: robot i takes cell (i + r) mod cells in
episode r of R, so every cell has B / cells robots or one more. Per cell, over its robots in the R episodes:
  survival         the fraction up at the end of the episode;
  velocity error   RMS over the surviving robots and the logged ticks from t = 0.5 s of the base's horizontal velocity error against the
                   command, in the base's heading frame (forward 0.3 m/s, lateral 0), from the true state [m/s];
  clearance        the mean over the surviving robots of the highest contact point above the ground over the logged ticks from
                   t = 0.3 s, from the true state [m] (the swing apex the feet reach).
The log holds the true state every 5 ticks (10 ms). In the same invocation the tool times, alternately, one episode with the grid's records,
one with hb_default_planner_settings records on every robot and one with no setting (K rounds), and reports whether the default records
gave the unset outcome and the same launches, with the card's name, power limit and the clocks sampled meanwhile.
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import GROUND, Episodes, cells, failure_checks, noise_ok, parser, report, workload  # noqa: E402

TICKS, LOG_EVERY, V_CMD = 1000, 5, 0.3
T_VEL, T_CLEAR = 0.5, 0.3


def axis(spec, default, name):
    lo, hi, n = (spec or default).split(":")
    lo, hi, n = float(lo), float(hi), int(n)
    if not (0 <= lo < hi and n >= 2) or (name == "periods" and lo <= 0):
        raise SystemExit("gait_sweep.py: --%s LO:HI:N with 0 <= LO < HI (LO > 0 for periods) and N >= 2 expected, got %r" % (name, spec))
    return np.linspace(lo, hi, n)


def heights_above_ground(ctx, log):
    """Height of every contact point above the ground at every logged state (B x rows x 4)."""
    B, rows = log.shape[:2]
    flat = log.reshape(-1, 32)
    z = np.concatenate([ctx.contact_positions(ctx.rbd_to_centroidal(flat[k:k + B])).reshape(-1, 4, 3)[:, :, 2] for k in range(0, len(flat), B)])
    return z.reshape(B, rows, 4) - GROUND


def main():
    ap = parser("robots per episode (at least the number of cells)")
    ap.add_argument("--periods", default=None, metavar="LO:HI:N", help="trot periods [s] (default 0.4:0.8:5)")
    ap.add_argument("--heights", default=None, metavar="LO:HI:N", help="swing heights [m] (default 0.02:0.10:5)")
    ap.add_argument("--repeats", type=int, default=2, help="episodes per grid (the robot -> cell assignment shifts between them)")
    ap.add_argument("--timed", type=int, default=3, help="timed rounds of the grid, default records and no setting")
    args = ap.parse_args()
    periods, heights = axis(args.periods, "0.4:0.8:5", "periods"), axis(args.heights, "0.02:0.10:5", "heights")
    nx, ny = len(periods), len(heights)
    if args.batch < nx * ny or args.repeats < 1 or not noise_ok(args):
        raise SystemExit("gait_sweep.py: --batch >= %d, --repeats >= 1, --sensor-noise takes a scale >= 0 and needs --estimator" % (nx * ny))
    h = Episodes("gait_sweep.py", args, TICKS)
    hb, ctx, prm, B = h.hb, h.ctx, h.prm, h.B

    def grid(shift):
        """The records of every robot and its cell index (row-major: heights down, periods across) for the assignment shifted by `shift`."""
        col, row = cells(B, nx, ny, shift)
        recs = hb.make_planner_settings(B, swing_height=heights[row], gaits={"trot": [(["L", "R"], [0.0, p / 2, p]) for p in periods[col]]})
        return recs, row * nx + col

    n, up, sq, nsq, clear = (np.zeros(nx * ny) for _ in range(5))
    rejects = np.zeros(nx * ny)
    ctx.set_planner_settings(grid(0)[0])
    h.episode()                                 # warm-up episode
    t_log = np.arange(-(-TICKS // LOG_EVERY)) * LOG_EVERY * prm.period
    for r in range(args.repeats):
        recs, cell = grid(r)
        ctx.set_planner_settings(recs)
        run = h.episode(log_every=LOG_EVERY)
        ok = run.stats["fail_tick"] < 0
        log = run.log
        yaw, vx, vy = log[:, :, 0], log[:, :, 19], log[:, :, 20]
        fwd, lat = np.cos(yaw) * vx + np.sin(yaw) * vy, -np.sin(yaw) * vx + np.cos(yaw) * vy
        err2 = ((fwd - V_CMD) ** 2 + lat ** 2)[:, t_log >= T_VEL]
        top = heights_above_ground(ctx, log)[:, t_log >= T_CLEAR].max(axis=(1, 2))
        for k in range(nx * ny):
            m = cell == k
            n[k] += m.sum(); up[k] += (m & ok).sum(); rejects[k] += run.stats["plan_rejects"][m].sum()
            sq[k] += err2[m & ok].sum(); nsq[k] += err2[m & ok].size; clear[k] += top[m & ok].sum()
    survival = up / n
    vel_err = np.sqrt(sq / np.maximum(nsq, 1))
    clearance = clear / np.maximum(up, 1)
    at = lambda k: {"period_s": float(periods[k % nx]), "swing_height_m": float(heights[k // nx]), "survival": float(survival[k]),
                    "velocity_error_rms_mps": float(vel_err[k]), "clearance_m": float(clearance[k])}
    shipped = int(np.argmin(np.abs(heights - 0.04))) * nx + int(np.argmin(np.abs(periods - 0.6)))
    order = sorted(range(nx * ny), key=lambda k: (-survival[k], vel_err[k], k))

    # one episode with the grid's records, one with default records, one unset, alternated
    recs, _ = grid(0)
    _, clocks, timing = h.alternate(ctx.set_planner_settings, [("grid", recs), ("default_records", hb.make_planner_settings(B)), ("unset", None)],
                                    args.timed)
    ctx.set_planner_settings(None)

    print(json.dumps({
        "metric": "gait sweep: survival, velocity tracking and foot clearance over a %d x %d grid of trot period x swing height" % (nx, ny),
        "value": float(survival[order[0]]), "unit": "fraction surviving (best cell)", **report(args, clocks),
        "periods_s": [float(p) for p in periods], "swing_heights_m": [float(v) for v in heights],
        "survival": survival.reshape(ny, nx).tolist(), "velocity_error_rms_mps": vel_err.reshape(ny, nx).tolist(),
        "clearance_m": clearance.reshape(ny, nx).tolist(), "plan_rejects": rejects.reshape(ny, nx).astype(int).tolist(),
        "shipped_cell": at(shipped), "best_cell": at(order[0]), "timing": timing,
        "config": {"workload": workload(h, "; %d or %d robots per cell, %d episodes (assignment shifted)" % (B // (nx * ny), -(-B // (nx * ny)), args.repeats),
                                        "trot at %.1f m/s from t = 0.1 s" % V_CMD),
                   "survival": "robots up at the end of the episode",
                   "velocity_error": "RMS of the horizontal base velocity error in the heading frame, surviving robots, t >= %.1f s" % T_VEL,
                   "clearance": "mean over surviving robots of the highest contact point above the ground, t >= %.1f s" % T_CLEAR,
                   "failure_checks": failure_checks()}}))


if __name__ == "__main__":
    main()
