#!/usr/bin/env python3
"""Controller gain sweep of the closed-loop episodes (hb_rollout_set_controller_settings): prints one JSON line.

  python tools/gain_sweep.py [--x FIELD:LO:HI] [--y FIELD:LO:HI] [--push N] [--repeats R] [--timed K] [--batch B]
                             [--estimator [--sensor-noise SCALE]] [--wbc weighted|hierarchical]

An 8 x 8 grid over two fields of hb_controller_setting (any field of hb_wbc_settings or hb_pd_gains), each at 8 geometrically spaced values
from LO to HI. The default grid is the WBC's swing_kp x base_angular_kp, each from 1/4 to 2^1.5 times the shipped task.info value in
half-octave steps, so that the shipped values are a grid point. The workload of tools/bench_rollout.py (B robots, default 1024, trotting at
0.3 m/s from the randomised poses of bench.py's configs[1]) runs for 1.5 s (750 ticks); the 64 cells share the batch, B / 64 robots each,
every robot on its cell's record and the shipped values elsewhere; episode r of R shifts the assignment by r. --push N pushes every robot
with N newtons along +x at the base origin from t = 0.5 s for 0.1 s (push_sweep.py's push). Per cell: survival (the fraction of its robots
up at the end) and the WBC fallbacks per robot; the cell of the shipped values and the best cell (highest survival, then fewest fallbacks).

The line also times, in the same invocation and alternately, the grid as one call against the same grid the way it runs without the
setting: 64 calls of B / 64 robots, each after hb_wbc_set_settings with the cell's WBC settings and with the cell's PD gains in
params.gains. It reports both times (device events summed over the calls, and host time to the last synchronise), both launch counts,
whether every cell's final stats and states are bitwise equal between the two ways, and the fused WBC kernel's time per call (hb_profile)
with the setting in force and without, with the card's name and power limit.
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import PUSH_DURATION, PUSH_T, Episodes, Tally, cell_members, cells, failure_checks, report, sweep_args, workload  # noqa: E402
from bench import ClockSampler  # noqa: E402  (episode_harness put the repository root on the path)

TICKS, NX, NY = 750, 8, 8
DEFAULT_X, DEFAULT_Y = "swing_kp", "base_angular_kp"
FACTORS = 2.0 ** np.arange(-2.0, 2.0, 0.5)          # 1/4 .. 2^1.5 in half octaves; index 4 is the shipped value


def axis(spec, default_field, shipped):
    """(field, 8 values) of --x / --y: FIELD:LO:HI, or FIELD alone / nothing for FACTORS times the shipped value."""
    parts = (spec or default_field).split(":")
    field = parts[0]
    if field not in shipped:
        raise SystemExit("gain_sweep.py: unknown field %r (one of %s)" % (field, ", ".join(sorted(shipped))))
    if len(parts) == 1:
        return field, shipped[field] * FACTORS
    if len(parts) != 3:
        raise SystemExit("gain_sweep.py: FIELD:LO:HI expected, got %r" % spec)
    lo, hi = float(parts[1]), float(parts[2])
    if not (0 < lo < hi):
        raise SystemExit("gain_sweep.py: 0 < LO < HI expected, got %r" % spec)
    return field, np.geomspace(lo, hi, NX)


def main():
    def extra(ap):
        ap.add_argument("--x", default=None, metavar="FIELD:LO:HI", help="grid columns (default %s, 1/4 .. 2.8 x shipped)" % DEFAULT_X)
        ap.add_argument("--y", default=None, metavar="FIELD:LO:HI", help="grid rows (default %s, 1/4 .. 2.8 x shipped)" % DEFAULT_Y)
        ap.add_argument("--push", type=float, default=0.0, metavar="N", help="push every robot with N newtons along +x at t = 0.5 s")
    args = sweep_args("gain_sweep.py", "timed rounds of one call and 64 calls", NX * NY, extra)
    h = Episodes("gain_sweep.py", args, TICKS)
    hb, ctx, prm, B = h.hb, h.ctx, h.prm, h.B
    base = hb.make_controller_settings(1)[0]
    shipped = {f: float(getattr(base.wbc, f)) for f, t in hb.HbWbcSettings._fields_ if f != "torque_limits"}
    shipped.update({f: float(getattr(base.gains, f)) for f, _ in hb.HbPdGains._fields_})
    xf, xs = axis(args.x, DEFAULT_X, shipped)
    yf, ys = axis(args.y, DEFAULT_Y, shipped)
    if xf == yf:
        raise SystemExit("gain_sweep.py: --x and --y name the same field")
    if args.push:
        ctx.set_pushes(hb.make_push_schedules(B, PUSH_T, PUSH_DURATION, [args.push, 0.0, 0.0]))
    n_per = B // (NX * NY)

    def grid(shift):
        """The records of every robot for the assignment shifted by `shift`."""
        col, row = cells(B, NX, NY, shift)
        return hb.make_controller_settings(B, **{xf: xs[col], yf: ys[row]})

    # the grid, episode r on assignment shift r
    tally = Tally(NX, NY)
    for r, run in h.sweep(ctx.set_controller_settings, grid):
        tally.add(*cells(B, NX, NY, r), run.stats)
    survival, fallbacks = tally.survival().ravel(), (tally.fallbacks / tally.total).ravel()
    at = lambda k: {"cell": [int(k % NX), int(k // NX)], xf: float(xs[k % NX]), yf: float(ys[k // NX]), "survival": float(survival[k]),
                    "wbc_fallbacks_per_robot": float(fallbacks[k])}
    order = sorted(range(NX * NY), key=lambda k: (-survival[k], fallbacks[k], k))
    shipped_cell = [int(np.argmin(np.abs(np.log(xs / shipped[xf])))), int(np.argmin(np.abs(np.log(ys / shipped[yf]))))]

    # one call against 64 calls of B / 64 robots on the context's settings, alternated; assignment shift 0
    recs, members = grid(0), cell_members(B, NX, NY, 0)
    wbc0, gains0 = ctx.wbc_settings(), hb.HbPdGains.from_buffer_copy(bytes(prm.gains))

    def set_cell(k):                            # with --push, a call's robots take the first B / 64 push schedules, which are all alike
        ctx.set_wbc_settings(recs[members[k][0]].wbc)
        prm.gains = recs[members[k][0]].gains

    def restore():
        ctx.set_wbc_settings(wbc0); prm.gains = gains0

    sampler = ClockSampler(args.device); sampler.start()
    timing = h.one_call_against_per_cell_calls(ctx.set_controller_settings, recs, set_cell, restore, members)
    clocks = sampler.stop()
    # workload() reads h.ticks, which the WBC kernel profile below sets to 50
    sentence = workload(h, "; %d robots per cell, %d episodes (assignment shifted)" % (n_per, args.repeats))

    # the fused WBC kernel (hb_profile kind qp_ipm) per call on the whole batch, with the grid's setting in force and without
    h.ticks, wbc_ms = 50, {}
    for name, setting in (("set", recs), ("unset", None)):
        ctx.set_controller_settings(setting)
        h.episode()
        ctx.profile_enable(True)
        h.episode()
        q = ctx.profile_read()["qp_ipm"]
        ctx.profile_enable(False)
        wbc_ms[name] = q["ms"] / max(q["launches"], 1)
    ctx.set_controller_settings(None)
    timing.update(wbc_kernel_ms_per_call_set=wbc_ms["set"], wbc_kernel_ms_per_call_unset=wbc_ms["unset"])

    print(json.dumps({
        "metric": "controller gain sweep: survival of %d robots per cell over an 8 x 8 grid of %s x %s" % (n_per * args.repeats, xf, yf),
        "value": float(survival[order[0]]), "unit": "fraction surviving (best cell)", **report(args, clocks), "push_N": args.push,
        "x": {"field": xf, "values": [float(v) for v in xs]}, "y": {"field": yf, "values": [float(v) for v in ys]},
        "survival": survival.reshape(NY, NX).tolist(), "wbc_fallbacks_per_robot": fallbacks.reshape(NY, NX).tolist(),
        "shipped_cell": at(shipped_cell[1] * NX + shipped_cell[0]), "best_cell": at(order[0]), "timing": timing,
        "config": {"workload": sentence,
                   "survival": "robots up at the end of the episode", "failure_checks": failure_checks()}}))


if __name__ == "__main__":
    main()
