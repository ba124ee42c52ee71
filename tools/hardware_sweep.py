#!/usr/bin/env python3
"""Simulated hardware sweep of the estimated episodes (hb_rollout_set_hardware): prints one JSON line.

  python tools/hardware_sweep.py [--offsets] [--repeats R] [--timed K] [--batch B] [--wbc weighted|hierarchical]

Every episode runs through the state estimator (hb_rollout_estimated_batch_dev). The workload of tools/bench_rollout.py (B robots, default
1024, trotting at 0.3 m/s from the randomised poses of bench.py's configs[1]) runs for 1.5 s (750 ticks); the 64 cells of an 8 x 8 grid
share the batch, B / 64 robots each, every robot on its cell's hardware record; episode r of R shifts the assignment by r.

Default grid: actuation delay (0, 4, ..., 28 ms) x sensor-noise scale (DELAYS x SCALES: every sigma SCALE x NOISE_SIGMAS of
episode_harness.py), no offsets. Per cell: survival (the fraction of its robots up at the end), the WBC fallbacks per robot and the
estimator's RMS velocity and height errors. The line also times, in the same invocation and alternately, the grid as one call against the
same grid the way it runs without the setting: 64 calls of B / 64 robots, each with the cell's delay in params.actuation_delay and its
sigmas in est_params.noise (each robot keeps its noise stream, so the two ways compute the same). It reports both times (device events
summed over the calls, and host time to the last synchronise), both launch counts and whether every cell's final stats and states are
bitwise equal between the two ways. Then it times, alternately, the episode with the grid's records, with records of the call's values on
every robot, and with no setting (at 1 x NOISE_SIGMAS), and checks that the second gives the third's outcome. All with the card's name and
power limit.

--offsets: the grid is a body-x accelerometer bias (0 ... 0.7 m/s^2) x an IMU roll mounting error (0 ... 1.75 deg), with the shipped
delay and limits and exact sensors otherwise. Per cell: survival, and the final position error: the horizontal distance between where each
surviving robot ends and where the same robot ends with ideal hardware (an episode without the setting). No per-call value can express an
offset, so this mode makes no comparison.
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import NOISE_SIGMAS, Episodes, Tally, cell_members, cells, failure_checks, report, sweep_args, workload  # noqa: E402
from bench import SEED, ClockSampler  # noqa: E402  (episode_harness put the repository root on the path)

TICKS, NX, NY = 750, 8, 8
DELAYS = 0.004 * np.arange(NX)                                      # [s]
SCALES = np.array([0.0, 0.5, 1.0, 2.0, 3.0, 4.0, 6.0, 8.0])          # x NOISE_SIGMAS
ACCEL_BIAS = 0.1 * np.arange(NX)                                     # body x [m/s^2]
ROLL_OFFSET = np.deg2rad(0.25 * np.arange(NY))                       # [rad]


def main():
    def extra(ap):
        ap.add_argument("--offsets", action="store_true", help="accelerometer bias x IMU roll offset instead of delay x noise")
    args = sweep_args("hardware_sweep.py", "timed rounds of one call and 64 calls", NX * NY, extra)
    args.estimator = True
    h = Episodes("hardware_sweep.py", args, TICKS)
    hb, ctx, prm, ep, B = h.hb, h.ctx, h.prm, h.ep, h.B
    n_per = B // (NX * NY)

    def sigmas(scale):
        return {"sigma_" + k: scale * v for k, v in NOISE_SIGMAS.items()}

    def grid(shift):
        """The records of every robot for the assignment shifted by `shift`."""
        col, row = cells(B, NX, NY, shift)
        if args.offsets:
            return hb.make_hardware_settings(B, accel_bias=np.c_[ACCEL_BIAS[col], np.zeros((B, 2))], orientation_offset=np.c_[np.zeros((B, 2)), ROLL_OFFSET[row]])
        return hb.make_hardware_settings(B, actuation_delay=DELAYS[col], **{k: SCALES[row] * v for k, v in sigmas(1.0).items()})

    ref = None
    if args.offsets:
        ctx.set_hardware(None)
        ref = h.episode(True, est_stats=True)   # ideal hardware: where each robot ends without offsets
    tally = Tally(NX, NY)
    vel, hgt, cnt, perr = np.zeros(NX * NY), np.zeros(NX * NY), np.zeros(NX * NY), [[] for _ in range(NX * NY)]
    for r, run in h.sweep(ctx.set_hardware, grid, estimated=True, est_stats=True):
        st, es = run.stats, run.est_stats
        tally.add(*cells(B, NX, NY, r), st)
        for k, m in enumerate(cell_members(B, NX, NY, r)):
            vel[k] += es["sum_sq_vel_err"][m].sum(); hgt[k] += es["sum_sq_height_err"][m].sum(); cnt[k] += es["count"][m].sum()
            if ref is not None:
                up = m[st["fail_tick"][m] < 0]
                perr[k] += list(np.hypot(*(run.rbd[up, 3:5] - ref.rbd[up, 3:5]).T))
    survival, cnt = tally.survival().ravel(), np.maximum(cnt, 1)
    axes = ({"field": "accel_bias[0]", "unit": "m/s^2", "values": ACCEL_BIAS.tolist()}, {"field": "orientation_offset[2]", "unit": "rad", "values": ROLL_OFFSET.tolist()}) \
        if args.offsets else ({"field": "actuation_delay", "unit": "s", "values": DELAYS.tolist()}, {"field": "sensor noise scale", "unit": "x NOISE_SIGMAS", "values": SCALES.tolist()})
    line = {"metric": "simulated hardware sweep: survival of %d robots per cell over an 8 x 8 grid of %s x %s" % (n_per * args.repeats, axes[0]["field"], axes[1]["field"]),
            "value": float(survival.mean()), "unit": "fraction surviving (mean over cells)", "x": axes[0], "y": axes[1],
            "survival": survival.reshape(NY, NX).tolist(), "wbc_fallbacks_per_robot": (tally.fallbacks / tally.total).tolist()}
    if args.offsets:
        line["final_position_error_m"] = {"median": [float(np.median(p)) if p else None for p in perr], "max": [float(np.max(p)) if p else None for p in perr]}
        for key in ("median", "max"):
            line["final_position_error_m"][key] = [line["final_position_error_m"][key][k * NX:(k + 1) * NX] for k in range(NY)]
    else:
        line["est_vel_err_rms"] = np.sqrt(vel / cnt).reshape(NY, NX).tolist()
        line["est_height_err_rms"] = np.sqrt(hgt / cnt).reshape(NY, NX).tolist()

    sampler = ClockSampler(args.device); sampler.start()
    timing = {}
    if not args.offsets:
        # one call against 64 calls of B / 64 robots on the call's values, alternated; assignment shift 0
        delay0, noise0 = prm.actuation_delay, hb.HbSensorNoise.from_buffer_copy(bytes(ep.noise))

        def set_cell(k):
            prm.actuation_delay = DELAYS[k % NX]
            for name, v in NOISE_SIGMAS.items():
                setattr(ep.noise, name, SCALES[k // NX] * v)

        def restore():
            prm.actuation_delay, ep.noise = delay0, noise0

        timing = h.one_call_against_per_cell_calls(ctx.set_hardware, grid(0), set_cell, restore, cell_members(B, NX, NY, 0), est_stats=True)
    # the grid's records, records of the call's values on every robot and no setting, alternated, at 1 x NOISE_SIGMAS
    for name, v in NOISE_SIGMAS.items():
        setattr(ep.noise, name, v)
    call = hb.make_hardware_settings(B, actuation_delay=prm.actuation_delay, torque_limit=prm.torque_limit[:], **sigmas(1.0))
    _, _, timing["episode"] = h.alternate(ctx.set_hardware, [("grid_records", grid(0)), ("call_value_records", call), ("unset", None)], args.timed)
    line["timing"] = timing
    line.update(report(args, sampler.stop(), estimator=False))
    line["config"] = {"workload": workload(h, "; %d robots per cell, %d episodes (assignment shifted)" % (n_per, args.repeats), robots="robots through the estimator"),
                      "noise_sigmas_at_scale_1": NOISE_SIGMAS, "noise_seed": SEED, "survival": "robots up at the end of the episode",
                      "failure_checks": failure_checks()}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
