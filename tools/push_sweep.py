#!/usr/bin/env python3
"""Push-recovery sweep of the closed-loop episodes (hb_rollout_set_pushes + hb_rollout_batch_dev): prints one JSON line.

  python tools/push_sweep.py [--repeats R] [--timed K] [--batch B] [--estimator [--sensor-noise SCALE]]

The workload of tools/bench_rollout.py (B robots, default 1024, trotting at 0.3 m/s from the randomised poses of bench.py's configs[1],
N = 100, dt = 10 ms, ground at 0.02 m, failure below a base height of 0.3 m), run for 1.5 s (750 ticks). Every robot gets one push at
t = 0.5 s for 0.1 s: a world-frame force at the base origin along +x, -x, +y or -y, of a magnitude from a grid (0 to 150 N in 10 N steps;
while some direction still has >= 90 % survival at the top of the grid, the grid is extended by another 16 steps, up to 1000 N). The
64 (direction, magnitude) cells of a grid block share the batch, 1/64 of the robots each; episode r of R shifts the assignment by r, so
every cell sees R x B / 64 different start poses. Survival of a cell = the fraction of its robots that were up when the push began and
are still up at the end of the episode.

The line also times, in the same invocation, the pushed batch (the first grid block) against the same batch with no schedules set,
alternately, with device events around the episode call, and reports the launch counts of both (pushes add no launch), with the card's
name and power limit and the clocks sampled during the timed episodes.

--estimator runs everything through hb_rollout_estimated_batch_dev (controllers on the Kalman filter's estimate from simulated sensors,
noise = SCALE x episode_harness's NOISE_SIGMAS).
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import PUSH_DURATION, PUSH_T, Episodes, Tally, cells, failure_checks, report, sweep_args, workload  # noqa: E402

TICKS = 750
DIRECTIONS = {"+x": (1.0, 0.0, 0.0), "-x": (-1.0, 0.0, 0.0), "+y": (0.0, 1.0, 0.0), "-y": (0.0, -1.0, 0.0)}
STEP_N, BLOCK, MAX_FORCE, SURVIVE = 10.0, 16, 1000.0, 0.9
BLOCKS = int(MAX_FORCE // (BLOCK * STEP_N)) + 1          # grid blocks up to the first one that ends above MAX_FORCE


def main():
    args = sweep_args("push_sweep.py", "timed pushed / zero-force / unpushed episode triples", len(DIRECTIONS) * BLOCK)
    h = Episodes("push_sweep.py", args, TICKS)
    hb, ctx, prm, B = h.hb, h.ctx, h.prm, h.B
    push_tick = int(round(PUSH_T / prm.period))

    def push_cells(block, shift):
        """(magnitude index, direction index) of every robot for grid block `block`, assignment shifted by `shift`."""
        c, d = cells(B, BLOCK, len(DIRECTIONS), shift)
        return block * BLOCK + c, d

    def schedules(block, shift):
        k, d = push_cells(block, shift)
        dirs = np.array(list(DIRECTIONS.values()))
        return hb.make_push_schedules(B, PUSH_T, PUSH_DURATION, (dirs[d] * (k * STEP_N)[:, None])[:, None, :])

    names = list(DIRECTIONS)
    tally = Tally(BLOCKS * BLOCK, len(names))
    ctx.set_pushes(schedules(0, 0))
    h.episode()                                 # warm-up episode
    for block in range(BLOCKS):
        for r in range(args.repeats):
            ctx.set_pushes(schedules(block, r))
            st = h.episode().stats
            tally.add(*push_cells(block, r), st, counts=(st["fail_tick"] < 0) | (st["fail_tick"] > push_tick))
        top = (block + 1) * BLOCK - 1
        if all(tally.up[:, top] < SURVIVE * np.maximum(tally.total[:, top], 1)):
            break

    fractions, survival, up, largest = tally.survival(), {}, {}, {}
    for a, n in enumerate(names):                # the magnitudes at which some robot was up when the push began
        ks = np.nonzero(tally.total[a])[0]
        survival[n] = {"%g" % (k * STEP_N): float(fractions[a, k]) for k in ks}
        up[n] = {"%g" % (k * STEP_N): int(tally.total[a, k]) for k in ks}
        good = [float(k * STEP_N) for k in ks if fractions[a, k] >= SURVIVE]
        largest[n] = max(good) if good else None

    # pushed, zero-force (schedules set, the trajectories of the unpushed batch: the cost of the wrench path alone) and unpushed episodes
    # alternate
    zero = hb.make_push_schedules(B, PUSH_T, PUSH_DURATION, [0.0, 0.0, 0.0])
    runs, clocks, timing = h.alternate(ctx.set_pushes, [("pushed", schedules(0, 0)), ("zero_force", zero), ("unpushed", None)], args.timed)
    timing.update(launches_pushed=int(runs["pushed"][-1].launches), launches_unpushed=int(runs["unpushed"][-1].launches))
    known = [v for v in largest.values() if v is not None]
    print(json.dumps({
        "metric": "push recovery: the largest %.1f s world-frame push at the base, over the four horizontal directions, that >= 90 %% of the "
                  "trotting robots survive" % PUSH_DURATION, "value": min(known) if len(known) == len(names) else None, "unit": "N",
        **report(args, clocks), "largest_force_90pct": largest, "survival": survival,
        "robots_up_at_push": up, "fail_reasons_after_push": tally.reasons,
        "upright_fraction_unpushed": float((runs["unpushed"][-1].stats["fail_tick"] < 0).mean()), "timing": timing,
        "config": {"workload": workload(h, "; one push per robot at t = %.1f s for %.1f s, %d episodes per grid block of %d magnitudes x 4 directions"
                                        % (PUSH_T, PUSH_DURATION, args.repeats, BLOCK)),
                   "survival": "robots up when the push began (fail_tick < 0 or after tick %d) that are still up at the end" % push_tick,
                   "failure_checks": failure_checks()}}))


if __name__ == "__main__":
    main()
