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
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import MIN_HEIGHT, NOISE_SIGMAS, Episodes, cells, gpu_identity, sweep_args  # noqa: E402
from bench import DT, HORIZON_N, SEED, ClockSampler  # noqa: E402

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
        """The records of every robot and, per cell (row-major), its robots, for the assignment shifted by `shift`."""
        col, row = cells(B, NX, NY, shift)
        if args.offsets:
            recs = hb.make_hardware_settings(B, accel_bias=np.c_[ACCEL_BIAS[col], np.zeros((B, 2))], orientation_offset=np.c_[np.zeros((B, 2)), ROLL_OFFSET[row]])
        else:
            recs = hb.make_hardware_settings(B, actuation_delay=DELAYS[col], **{k: SCALES[row] * v for k, v in sigmas(1.0).items()})
        members = [np.nonzero(row * NX + col == k)[0] for k in range(NX * NY)]
        return recs, members

    def episode():
        return h.episode(True, est_stats=True)

    ref = None
    if args.offsets:
        ctx.set_hardware(None)
        ref = episode()                          # ideal hardware: where each robot ends without offsets
    surv, fb, n = np.zeros(NX * NY), np.zeros(NX * NY), np.zeros(NX * NY)
    vel, hgt, cnt, perr = np.zeros(NX * NY), np.zeros(NX * NY), np.zeros(NX * NY), [[] for _ in range(NX * NY)]
    ctx.set_hardware(grid(0)[0])
    episode()                                    # warm-up episode
    for r in range(args.repeats):
        recs, members = grid(r)
        ctx.set_hardware(recs)
        run = episode()
        st, es = run.stats, run.est_stats
        for k, m in enumerate(members):
            up = m[st["fail_tick"][m] < 0]
            surv[k] += len(up); fb[k] += st["wbc_fallbacks"][m].sum(); n[k] += len(m)
            vel[k] += es["sum_sq_vel_err"][m].sum(); hgt[k] += es["sum_sq_height_err"][m].sum(); cnt[k] += es["count"][m].sum()
            if ref is not None:
                perr[k] += list(np.hypot(*(run.rbd[up, 3:5] - ref.rbd[up, 3:5]).T))
    survival, fallbacks = surv / n, fb / n
    cnt = np.maximum(cnt, 1)
    axes = ({"field": "accel_bias[0]", "unit": "m/s^2", "values": ACCEL_BIAS.tolist()}, {"field": "orientation_offset[2]", "unit": "rad", "values": ROLL_OFFSET.tolist()}) \
        if args.offsets else ({"field": "actuation_delay", "unit": "s", "values": DELAYS.tolist()}, {"field": "sensor noise scale", "unit": "x NOISE_SIGMAS", "values": SCALES.tolist()})
    line = {"metric": "simulated hardware sweep: survival of %d robots per cell over an 8 x 8 grid of %s x %s" % (n_per * args.repeats, axes[0]["field"], axes[1]["field"]),
            "value": float(survival.mean()), "unit": "fraction surviving (mean over cells)", "n_gpus": 1, "dtype": "f64", "data": "synthetic",
            "wbc": args.wbc, "x": axes[0], "y": axes[1],
            "survival": survival.reshape(NY, NX).tolist(), "wbc_fallbacks_per_robot": fallbacks.reshape(NY, NX).tolist()}
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
        recs, members = grid(0)
        delay0, noise0 = prm.actuation_delay, hb.HbSensorNoise.from_buffer_copy(bytes(ep.noise))

        def one_call():
            ctx.set_hardware(recs)
            t0 = time.perf_counter()
            run = episode()
            return run, time.perf_counter() - t0

        def per_cell_calls():
            ctx.set_hardware(None)
            runs, t0 = [], time.perf_counter()
            for k, m in enumerate(members):
                prm.actuation_delay = DELAYS[k % NX]
                for name, v in NOISE_SIGMAS.items():
                    setattr(ep.noise, name, SCALES[k // NX] * v)
                runs.append(h.episode(True, est_stats=True, rows=m))
            wall = time.perf_counter() - t0
            prm.actuation_delay, ep.noise = delay0, noise0
            return runs, wall

        times = {"one_call_ms": [], "one_call_wall_ms": [], "per_cell_calls_ms": [], "per_cell_calls_wall_ms": []}
        equal = True
        for _ in range(max(1, args.timed)):
            one, w1 = one_call()
            many, w64 = per_cell_calls()
            times["one_call_ms"].append(one.ms); times["one_call_wall_ms"].append(1e3 * w1)
            times["per_cell_calls_ms"].append(sum(r.ms for r in many)); times["per_cell_calls_wall_ms"].append(1e3 * w64)
            for m, r in zip(members, many):
                equal &= bool(np.array_equal(one.stats[m], r.stats) and np.array_equal(one.rbd[m], r.rbd) and np.array_equal(one.est_stats[m], r.est_stats))
        timing = {k: float(np.median(v)) for k, v in times.items()}
        timing.update({k + "_range": [min(v), max(v)] for k, v in times.items()})
        timing.update(rounds=max(1, args.timed), launches_one_call=int(one.launches), launches_per_cell_calls=int(sum(r.launches for r in many)),
                      cells_bitwise_equal=equal)
    # the grid's records, records of the call's values on every robot and no setting, alternated, at 1 x NOISE_SIGMAS
    for name, v in NOISE_SIGMAS.items():
        setattr(ep.noise, name, v)
    call = hb.make_hardware_settings(B, actuation_delay=prm.actuation_delay, torque_limit=prm.torque_limit[:], **sigmas(1.0))
    _, _, alt = h.alternate(ctx.set_hardware, [("grid_records", grid(0)[0]), ("call_value_records", call), ("unset", None)], args.timed)
    timing["episode"] = alt
    line["timing"] = timing
    line["clocks"] = sampler.stop()
    line["config"] = {"workload": "%d robots through the estimator, %.1f s simulated (%d ticks of %.0f ms), trot at 0.3 m/s from t = 0.1 s, initial poses of "
                                  "scenarios.random_initial_states(seed %d), N=%d dt=%.0f ms; %d robots per cell, %d episodes (assignment shifted)"
                                  % (B, TICKS * prm.period, TICKS, 1e3 * prm.period, SEED, HORIZON_N, 1e3 * DT, n_per, args.repeats),
                      "noise_sigmas_at_scale_1": NOISE_SIGMAS, "noise_seed": SEED, "survival": "robots up at the end of the episode",
                      "failure_checks": "non-finite state, |roll| > pi/2, base z < %.2f m, emergency stop" % MIN_HEIGHT}
    line["gpu"] = gpu_identity(args.device)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
