#!/usr/bin/env python3
"""Model-mismatch sweep of the closed-loop episodes (hb_rollout_set_plant_variations + hb_rollout_batch_dev): prints one JSON line.

  python tools/plant_sweep.py [--repeats R] [--timed K] [--batch B] [--estimator [--sensor-noise SCALE]]

The workload of tools/bench_rollout.py (B robots, default 1024, trotting at 0.3 m/s from the randomised poses of bench.py's configs[1],
N = 100, dt = 10 ms, ground at 0.02 m, failure below a base height of 0.3 m), run for 1.5 s (750 ticks). Every robot runs on a plant of
its own, which the controllers are not told about: a payload of 0 to 7.5 kg (0.5 kg steps) on the base, a solid 0.2 x 0.2 x 0.1 m box
with its CoM 0.1 m above the base origin, on ground whose friction coefficient is scaled by 1.0, 0.6, 0.4 or 0.25 (the WBC's friction cone
keeps mu = 0.7). The 64 (payload, friction) cells share the batch, 1/64 of the robots each; episode r of R shifts the assignment by r, so
every cell sees R x B / 64 different start poses. Per cell: survival (the fraction of its robots still up at the end) and the mean
horizontal base speed of the survivors (their base displacement in the ground plane over the episode time).

The line also times, in the same invocation, the varied batch against the same batch with all-default variations and with none set,
alternately, with device events around the episode call, and reports the launch counts of the three (variations add no launch), whether
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
MASSES = [0.5 * k for k in range(16)]                   # [kg]
FRICTION = [1.0, 0.6, 0.4, 0.25]
BOX, COM = (0.2, 0.2, 0.1), (0.0, 0.0, 0.1)             # payload box edges [m] (x, y, z) and CoM in the base frame


def box_inertia(m):
    a, b, c = BOX
    return np.diag([m * (b * b + c * c) / 12, m * (a * a + c * c) / 12, m * (a * a + b * b) / 12])


def main():
    args = sweep_args("plant_sweep.py", "timed varied / default / unset episode triples", len(MASSES) * len(FRICTION))
    h = Episodes("plant_sweep.py", args, TICKS)
    hb, ctx, prm, B, rbd0 = h.hb, h.ctx, h.prm, h.B, h.rbd0
    T_episode = TICKS * prm.period

    def variations(shift):
        mi, fi = cells(B, len(MASSES), len(FRICTION), shift)
        m = np.array(MASSES)[mi]
        return hb.make_plant_variations(B, m, np.where(m[:, None] > 0, COM, 0.0), np.stack([box_inertia(x) for x in m]),
                                        friction_scale=np.array(FRICTION)[fi])

    tally = Tally(len(MASSES), len(FRICTION))
    for r, run in h.sweep(ctx.set_plant_variations, variations):
        tally.add(*cells(B, len(MASSES), len(FRICTION), r), run.stats, value=np.hypot(*(run.rbd[:, 3:5] - rbd0[:, 3:5]).T) / T_episode)
    fk, mk = ["%g" % f for f in FRICTION], ["%g" % m for m in MASSES]
    # per friction scale: the heaviest payload up to which every cell keeps >= 90 % survival
    heaviest = dict(zip(fk, tally.largest(MASSES)))

    # varied, all-default and unset episodes alternate
    runs, clocks, timing = h.alternate(ctx.set_plant_variations, [("varied", variations(0)), ("default", hb.make_plant_variations(B)),
                                                                  ("unset", None)], args.timed, launches=True)
    print(json.dumps({
        "metric": "model mismatch: the heaviest unmodelled payload (0.2 x 0.2 x 0.1 m box, CoM 0.1 m above the base) that >= 90 %% of the "
                  "trotting robots carry for %.1f s, per friction scale" % T_episode, "value": heaviest.get("1"), "unit": "kg",
        **report(args, clocks), "heaviest_payload_90pct": heaviest, "survival": keyed(fk, mk, tally.survival().tolist()),
        "mean_speed_of_survivors_m_per_s": keyed(fk, mk, tally.mean()), "fail_reasons": tally.reasons,
        "upright_fraction_unset": float((runs["unset"][-1].stats["fail_tick"] < 0).mean()), "timing": timing,
        "config": {"workload": workload(h, "; %d payload masses x %d friction scales, %d episodes" % (len(MASSES), len(FRICTION), args.repeats)),
                   "payload": "solid box %g x %g x %g m, CoM (%g, %g, %g) m in the base frame" % (BOX + COM),
                   "friction": "plant mu = scale x %g; the WBC's friction cone keeps its nominal coefficient" % prm.sim.friction_mu,
                   "survival": "robots still up at the end of the episode", "failure_checks": failure_checks()}}))


if __name__ == "__main__":
    main()
