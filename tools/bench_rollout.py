#!/usr/bin/env python3
"""Closed-loop episode benchmark (hb_rollout_batch_dev): prints one JSON line.

  python tools/bench_rollout.py [--steps K] [--batch B] [--estimator [--sensor-noise SCALE]]

One episode = 1 s of simulated time (500 ticks of 2 ms, an MPC cycle every 5 ticks) for B robots (default 1024) in one
hb_rollout_batch_dev call: trot at 0.3 m/s from the randomised initial poses of bench.py's configs[1] (N = 100, dt = 10 ms), each robot
lowered until its lowest contact frame is 1 mm inside the ground. One warm-up episode, then K timed episodes from the same start (device
events around the call); the line reports the median, the card's name and power limit, and the clocks sampled during the timed episodes.

--estimator adds, in the same invocation, the same episodes through hb_rollout_estimated_batch_dev (controllers on the Kalman filter's
estimate from simulated sensors, noise = SCALE x NOISE_SIGMAS), timed alternately with the ground-truth ones, under the key "estimator".
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import Episodes, failure_checks, noise_ok, parser, report, sensor_noise  # noqa: E402
from bench import DT, HORIZON_N, SEED, ClockSampler  # noqa: E402  (episode_harness put the repository root on the path)

TICKS = 500


def main():
    ap = parser()
    ap.add_argument("--steps", type=int, default=5, help="timed episodes")
    args = ap.parse_args()
    if not noise_ok(args):
        raise SystemExit("bench_rollout.py: --sensor-noise takes a scale >= 0 and needs --estimator")
    h = Episodes("bench_rollout.py", args, TICKS)
    hb, prm, B = h.hb, h.prm, h.B
    cycles = sum(1 for k in range(TICKS) if k % prm.mpc_every == 0)

    def episode(estimated=False):
        return h.episode(estimated, est_stats=True)

    episode()                                   # warm-up episode
    if args.estimator:
        episode(True)
    sampler = ClockSampler(args.device); sampler.start()
    runs, est_runs = [], []
    for _ in range(max(1, args.steps)):         # ground-truth and estimated episodes alternate
        runs.append(episode())
        if args.estimator:
            est_runs.append(episode(True))
    clocks = sampler.stop()
    ms = [r.ms for r in runs]
    st = runs[-1].stats
    med = float(np.median(ms))
    sim_s = TICKS * prm.period
    reasons = {name: int(((st["fail_reason"] & bit) != 0).sum()) for name, bit in hb.ROLLOUT_FAIL.items()}
    line = {"metric": "closed-loop episodes: simulated robot-seconds per wall-second (Hunter, MPC 100 Hz + WBC 500 Hz + plant)", "value": B * sim_s / (med * 1e-3),
            "unit": "robot-s/s", **report(args, clocks, estimator=False), "steps": len(runs), "warmup": 1, "higher_is_better": True,
            "ms_per_episode": med, "ms_per_episode_range": [min(ms), max(ms)], "ms_per_mpc_period": med / cycles,
            "launches_per_mpc_period": runs[-1].launches / cycles, "gpu_launches": int(runs[-1].launches),
            "upright_fraction": float((st["fail_tick"] == -1).mean()), "fail_reasons": reasons,
            "same_outcome_every_episode": all(np.array_equal(r.stats, st) for r in runs),
            "stats": {"mpc_bad": int(st["mpc_bad"].sum()), "wbc_fallbacks": int(st["wbc_fallbacks"].sum()), "plan_rejects": int(st["plan_rejects"].sum()),
                      "max_abs_torque": float(st["max_abs_torque"].max())},
            "config": {"workload": "%d robots, %.1f s simulated (%d ticks of %.0f ms, %d MPC cycles), trot at 0.3 m/s from t = 0.1 s, initial poses of "
                                   "scenarios.random_initial_states(seed %d), N=%d dt=%.0f ms, one hb_rollout_batch_dev call per episode, device events "
                                   "around it" % (B, sim_s, TICKS, 1e3 * prm.period, cycles, SEED, HORIZON_N, 1e3 * DT),
                       "failure_checks": failure_checks()}}
    if args.estimator:
        ems = [r.ms for r in est_runs]
        est_st, es = est_runs[-1].stats, est_runs[-1].est_stats
        emed = float(np.median(ems))
        n = max(int(es["count"].sum()), 1)
        line["estimator"] = {
            "ms_per_episode": emed, "ms_per_episode_range": [min(ems), max(ems)], "ms_per_mpc_period": emed / cycles,
            "extra_ms_per_tick": (emed - med) / TICKS, "launches_per_mpc_period": est_runs[-1].launches / cycles, "gpu_launches": int(est_runs[-1].launches),
            "upright_fraction": float((est_st["fail_tick"] == -1).mean()), "upright_fraction_ground_truth": float((st["fail_tick"] == -1).mean()),
            "fail_reasons": {name: int(((est_st["fail_reason"] & bit) != 0).sum()) for name, bit in hb.ROLLOUT_FAIL.items()},
            "vel_err_rms": float(np.sqrt(es["sum_sq_vel_err"].sum() / n)), "vel_err_max": float(es["max_vel_err"].max()),
            "height_err_rms": float(np.sqrt(es["sum_sq_height_err"].sum() / n)), "height_err_max": float(es["max_height_err"].max()),
            "stats": {"mpc_bad": int(est_st["mpc_bad"].sum()), "wbc_fallbacks": int(est_st["wbc_fallbacks"].sum()),
                      "plan_rejects": int(est_st["plan_rejects"].sum()), "max_abs_torque": float(est_st["max_abs_torque"].max())},
            "same_outcome_every_episode": all(np.array_equal(r.stats, est_st) and np.array_equal(r.est_stats, es) for r in est_runs),
            **sensor_noise(args),
            "errors": "filter output against the true state entering each tick, counted while the robot is up: |v_hat - v| world base "
                      "velocity [m/s], |z_hat - z| [m]; rms over robots and ticks"}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
