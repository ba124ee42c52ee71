#!/usr/bin/env python3
"""Leg-mass mismatch sweep of the closed-loop episodes (hb_rollout_set_link_variations + hb_rollout_batch_dev): prints one JSON line.

  python tools/link_sweep.py [--repeats R] [--timed K] [--batch B] [--wbc W] [--estimator [--sensor-noise SCALE]]

The workload of tools/bench_rollout.py (B robots, default 1024, trotting at 0.3 m/s from the randomised poses of bench.py's configs[1],
N = 100, dt = 10 ms, ground at 0.02 m, failure below a base height of 0.3 m), run for 1.5 s (750 ticks). Every robot's plant has leg links
of their own, which the controllers are not told about: the links of one group (hips: bodies 1, 2, 6, 7; thighs: 3, 8; shanks and feet:
4, 5, 9, 10; or every leg link) have s times the model's mass and s times its inertia (a link of the same shape and density scaled by s),
with s from 0.5 to 2.5. The 32 (scale, group) cells share the batch, 1/32 of the robots each; episode r of R shifts the assignment by r,
so every cell sees R x B / 32 different start poses. Per cell: survival (the fraction of its robots still up at the end) and the mean
horizontal base speed of the survivors (their base displacement in the ground plane over the episode time).

The line also times, in the same invocation, the varied batch against the same batch with all-default records and with none set,
alternately, with device events around the episode call, and reports the launch counts of the three (the setting adds no launch), whether
default and unset give the same outcome, and the card's name and power limit and the clocks sampled during the timed episodes.

--estimator runs everything through hb_rollout_estimated_batch_dev (controllers on the Kalman filter's estimate from simulated sensors,
noise = SCALE x episode_harness's NOISE_SIGMAS).
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import Episodes, Tally, cells, failure_checks, keyed, report, sweep_args, workload  # noqa: E402

TICKS = 750
SCALES = [0.5, 0.75, 1.0, 1.25, 1.5, 1.75, 2.0, 2.5]
GROUPS = {"hips": [1, 2, 6, 7], "thighs": [3, 8], "shanks_feet": [4, 5, 9, 10], "all_legs": list(range(1, 11))}


def tolerated(survival, threshold=0.9):
    """Per group (row), the smallest and largest scale of the run of cells around s = 1 whose survival is >= threshold (None when s = 1
    itself is below it)."""
    one = SCALES.index(1.0)
    out = []
    for row in survival:
        if row[one] < threshold:
            out.append(None)
            continue
        lo = hi = one
        while lo > 0 and row[lo - 1] >= threshold:
            lo -= 1
        while hi + 1 < len(SCALES) and row[hi + 1] >= threshold:
            hi += 1
        out.append([SCALES[lo], SCALES[hi]])
    return out


def main():
    args = sweep_args("link_sweep.py", "timed varied / default / unset episode triples", len(SCALES) * len(GROUPS))
    h = Episodes("link_sweep.py", args, TICKS)
    hb, ctx, prm, B, rbd0 = h.hb, h.ctx, h.prm, h.B, h.rbd0
    T_episode = TICKS * prm.period
    groups = list(GROUPS.values())

    def links(shift):
        si, gi = cells(B, len(SCALES), len(GROUPS), shift)
        s = np.ones((B, hb.NBODY))
        for i in range(B):
            s[i, groups[gi[i]]] = SCALES[si[i]]
        return hb.make_link_variations(B, mass_scale=s, inertia_scale=s)

    tally = Tally(len(SCALES), len(GROUPS))
    for r, run in h.sweep(ctx.set_link_variations, links):
        tally.add(*cells(B, len(SCALES), len(GROUPS), r), run.stats, value=np.hypot(*(run.rbd[:, 3:5] - rbd0[:, 3:5]).T) / T_episode)
    gk, sk = list(GROUPS), ["%g" % s for s in SCALES]
    survival = tally.survival().tolist()
    ranges = dict(zip(gk, tolerated(survival)))

    # varied, all-default and unset episodes alternate
    runs, clocks, timing = h.alternate(ctx.set_link_variations, [("varied", links(0)), ("default", hb.make_link_variations(B)), ("unset", None)],
                                       args.timed, launches=True)
    print(json.dumps({
        "metric": "leg-mass mismatch: the range of leg-link mass scales (inertia scaled alike, all ten leg links) over which >= 90 %% of the "
                  "trotting robots stay up for %.1f s" % T_episode, "value": ranges["all_legs"], "unit": "x nominal",
        **report(args, clocks), "scale_range_90pct": ranges, "survival": keyed(gk, sk, survival),
        "mean_speed_of_survivors_m_per_s": keyed(gk, sk, tally.mean()), "fail_reasons": tally.reasons,
        "upright_fraction_unset": float((runs["unset"][-1].stats["fail_tick"] < 0).mean()), "timing": timing,
        "config": {"workload": workload(h, "; %d leg-mass scales x %d link groups, %d episodes" % (len(SCALES), len(GROUPS), args.repeats)),
                   "groups": {k: "bodies " + ", ".join(map(str, v)) for k, v in GROUPS.items()},
                   "variation": "mass_scale = inertia_scale = s on the group's bodies, com_shift 0; the other bodies nominal",
                   "survival": "robots still up at the end of the episode", "failure_checks": failure_checks()}}))


if __name__ == "__main__":
    main()
