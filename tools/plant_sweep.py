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

from episode_harness import MIN_HEIGHT, NOISE_SIGMAS, Episodes, cells, gpu_identity, sweep_args  # noqa: E402
from bench import DT, HORIZON_N, SEED  # noqa: E402  (episode_harness put the repository root on the path)

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

    up = np.zeros((len(FRICTION), len(MASSES)), dtype=int)
    total = np.zeros_like(up)
    speed = np.zeros((len(FRICTION), len(MASSES)))
    reasons = {name: 0 for name in hb.ROLLOUT_FAIL}
    ctx.set_plant_variations(variations(0))
    h.episode()                                 # warm-up episode
    for r in range(args.repeats):
        ctx.set_plant_variations(variations(r))
        _, _, st, rbd, _ = h.episode()
        mi, fi = cells(B, len(MASSES), len(FRICTION), r)
        ok = st["fail_tick"] < 0
        v = np.hypot(*(rbd[:, 3:5] - rbd0[:, 3:5]).T) / T_episode
        np.add.at(total, (fi, mi), 1)
        np.add.at(up, (fi, mi), ok.astype(int))
        np.add.at(speed, (fi, mi), np.where(ok, v, 0.0))
        for name, bit in hb.ROLLOUT_FAIL.items():
            reasons[name] += int(((st["fail_reason"] & bit) != 0)[~ok].sum())
    survival = {"%g" % f: {"%g" % m: float(up[a, b] / total[a, b]) for b, m in enumerate(MASSES)} for a, f in enumerate(FRICTION)}
    mean_speed = {"%g" % f: {"%g" % m: (float(speed[a, b] / up[a, b]) if up[a, b] else None) for b, m in enumerate(MASSES)}
                  for a, f in enumerate(FRICTION)}
    heaviest = {}                               # per friction scale: the heaviest payload up to which every cell keeps >= 90 % survival
    for a, f in enumerate(FRICTION):
        heaviest["%g" % f] = None
        for b, m in enumerate(MASSES):
            if up[a, b] < 0.9 * total[a, b]:
                break
            heaviest["%g" % f] = m

    # varied, all-default and unset episodes alternate
    runs, clocks, timing = h.alternate(ctx.set_plant_variations, [("varied", variations(0)), ("default", hb.make_plant_variations(B)),
                                                                  ("unset", None)], args.timed)
    timing.update({"launches_" + n: int(runs[n][-1].launches) for n in runs})
    line = {"metric": "model mismatch: the heaviest unmodelled payload (0.2 x 0.2 x 0.1 m box, CoM 0.1 m above the base) that >= 90 %% of the "
                      "trotting robots carry for %.1f s, per friction scale" % T_episode, "value": heaviest.get("1"), "unit": "kg",
            "n_gpus": 1, "dtype": "f64", "data": "synthetic", "estimator": bool(args.estimator), "wbc": args.wbc,
            "heaviest_payload_90pct": heaviest, "survival": survival, "mean_speed_of_survivors_m_per_s": mean_speed, "fail_reasons": reasons,
            "upright_fraction_unset": float((runs["unset"][-1].stats["fail_tick"] < 0).mean()), "timing": timing,
            "config": {"workload": "%d robots, %.1f s simulated (%d ticks of %.0f ms), trot at 0.3 m/s from t = 0.1 s, initial poses of "
                                   "scenarios.random_initial_states(seed %d), N=%d dt=%.0f ms; %d payload masses x %d friction scales, %d episodes"
                                   % (B, T_episode, TICKS, 1e3 * prm.period, SEED, HORIZON_N, 1e3 * DT, len(MASSES), len(FRICTION), args.repeats),
                       "payload": "solid box %g x %g x %g m, CoM (%g, %g, %g) m in the base frame" % (BOX + COM),
                       "friction": "plant mu = scale x %g; the WBC's friction cone keeps its nominal coefficient" % prm.sim.friction_mu,
                       "survival": "robots still up at the end of the episode",
                       "failure_checks": "non-finite state, |roll| > pi/2, base z < %.2f m, emergency stop" % MIN_HEIGHT},
            "gpu": gpu_identity(args.device), "clocks": clocks}
    if args.estimator:
        line["sensor_noise"] = {k: args.sensor_noise * v for k, v in NOISE_SIGMAS.items()}
        line["noise_seed"] = SEED
    print(json.dumps(line))


if __name__ == "__main__":
    main()
