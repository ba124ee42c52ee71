#!/usr/bin/env python3
"""MPC latency sweep of the closed-loop episodes (hb_rollout_set_mpc_latencies + hb_rollout_batch_dev): prints one JSON line.

  python tools/latency_sweep.py [--ticks T] [--push N] [--timed K] [--batch B] [--estimator [--sensor-noise SCALE]] [--wbc hierarchical]

The workload of tools/bench_rollout.py (B robots, default 1024, from the randomised poses of bench.py's configs[1], N = 100, dt = 10 ms,
ground at 0.02 m, failure below a base height of 0.3 m), trotting at 0.3 m/s from t = 0.1 s. One episode per latency 0 .. 5 ticks (0-10 ms
at 500 Hz, MPC at 100 Hz), every robot with the same latency. With --push N every robot is pushed by a world-y force of N newtons at its
base for PUSH_DURATION from PUSH_TIME. Per latency: the share of robots that survive, the failure reasons, the MPC and WBC failure counts
(hb_rollout_stats' mpc_bad and wbc_fallbacks, summed over the robots) and the largest applied torque.

The line also times, in the same invocation, a latency of TIMED_LATENCY ticks against an all-zero setting and no setting, alternately, with
device events around the episode call, and reports the launch counts of the three, whether the all-zero setting gives the outcome of no
setting, and the card's name and power limit and the clocks sampled during the timed episodes.
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import GROUND, Episodes, failure_checks, noise_ok, parser, report, workload  # noqa: E402

LATENCIES = [0, 1, 2, 3, 4, 5]          # [ticks]
TIMED_LATENCY = 4                       # about the 7.8 ms of one 1024-robot MPC step in README
PUSH_TIME, PUSH_DURATION = 1.0, 0.1     # [s]


def main():
    ap = parser()
    ap.add_argument("--ticks", type=int, default=1000, help="ticks per episode (2 ms each)")
    ap.add_argument("--push", type=float, default=0.0, metavar="N", help="world-y push on every robot [N], 0: none")
    ap.add_argument("--timed", type=int, default=3, help="timed latency / zero / unset episode triples")
    args = ap.parse_args()
    if args.ticks < 1 or not noise_ok(args) or not np.isfinite(args.push):
        raise SystemExit("latency_sweep.py: --ticks >= 1, a finite --push, --sensor-noise takes a scale >= 0 and needs --estimator")
    h = Episodes("latency_sweep.py", args, args.ticks)
    hb, ctx, prm, B = h.hb, h.ctx, h.prm, h.B
    if max(LATENCIES) > prm.mpc_every:
        raise SystemExit("latency_sweep.py: latencies up to %d ticks need mpc_every >= %d" % (max(LATENCIES), max(LATENCIES)))
    if args.push:
        ctx.set_pushes(hb.make_push_schedules(B, PUSH_TIME, PUSH_DURATION, [0.0, args.push, 0.0]))
    ctx.set_mpc_latencies(np.full(B, TIMED_LATENCY))
    h.episode()                                   # warm-up episode
    per_latency = {}
    for d in LATENCIES:
        ctx.set_mpc_latencies(np.full(B, d))
        run = h.episode()
        st = run.stats
        up = st["fail_tick"] < 0
        per_latency[str(d)] = {
            "latency_ms": d * 1e3 * prm.period, "survival": float(up.mean()),
            "fail_reasons": {name: int(((st["fail_reason"] & bit) != 0)[~up].sum()) for name, bit in hb.ROLLOUT_FAIL.items()},
            "mpc_bad": int(st["mpc_bad"].sum()), "wbc_fallbacks": int(st["wbc_fallbacks"].sum()), "plan_rejects": int(st["plan_rejects"].sum()),
            "max_abs_torque": float(st["max_abs_torque"].max()), "ms_per_episode": run.ms}
    runs, clocks, timing = h.alternate(ctx.set_mpc_latencies, [("latency_%d" % TIMED_LATENCY, np.full(B, TIMED_LATENCY)),
                                                               ("zero_latency", np.zeros(B)), ("unset", None)], args.timed,
                                       launches=True)
    print(json.dumps({
        "metric": "MPC latency: share of trotting robots that survive %.1f s with a %d-tick (%.0f ms) MPC latency"
                  % (args.ticks * prm.period, TIMED_LATENCY, TIMED_LATENCY * 1e3 * prm.period),
        "value": per_latency[str(TIMED_LATENCY)]["survival"], "unit": "fraction", **report(args, clocks), "push_n": args.push,
        "per_latency": per_latency, "timing": timing,
        "config": {"workload": workload(h, "", "trot at 0.3 m/s from t = 0.1 s, MPC every %d ticks" % prm.mpc_every, digits=2),
                   "push": ("world-y %g N at the base from t = %g s for %g s" % (args.push, PUSH_TIME, PUSH_DURATION)) if args.push else None,
                   "failure_checks": failure_checks(), "ground_m": GROUND}}))


if __name__ == "__main__":
    main()
