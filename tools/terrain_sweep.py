#!/usr/bin/env python3
"""Terrain sweep of the closed-loop episodes (hb_rollout_set_terrains + hb_rollout_batch_dev): prints one JSON line.

  python tools/terrain_sweep.py [--repeats R] [--timed K] [--batch B] [--estimator [--sensor-noise SCALE]]

The workload of tools/bench_rollout.py (B robots, default 1024, trotting at 0.3 m/s from the randomised poses of bench.py's configs[1],
N = 100, dt = 10 ms, ground at 0.02 m, failure below a base height of 0.3 m, measured above the terrain), run for 1.5 s (750 ticks). Every
robot walks blind over a terrain of its own, which the planner, controllers and estimator are not told about: a 64 x 64 height field at
2.5 cm spacing centred on its start, with the ground at 0.02 m under the start pose and, across the robot's initial heading,
  - a step up or a step down of 0 to 15 cm (1 cm steps) whose edge lies 0.15 m ahead of the base origin, or
  - an incline or a decline of 0 to 15 degrees (1 degree steps) that starts 0.10 m ahead of it.
The height field is interpolated bilinearly between its samples, so a step is a ramp one cell (2.5 cm) wide; the plant has point
contacts only, so no foot meets the step's face. A robot whose foremost contact point starts less than 1.5 cells (3.75 cm, more than the
cell's diagonal) behind the edge or the ramp's start has them moved ahead to that distance, so that the ground under every start pose is
0.02 m exactly and the start states are those of bench_rollout (the randomised poses put the foremost contact point up to about 0.12 m
ahead of the base origin); the line reports how many robots that moves.

The 64 (kind, magnitude) cells share the batch, 1/64 of the robots each; episode r of R shifts the assignment by r, so every cell sees
R x B / 64 different start poses. Per cell: survival (the fraction of its robots still up at the end) and the mean horizontal base speed of
the survivors (their base displacement in the ground plane over the episode time). Per kind: the largest magnitude up to which every cell
keeps >= 90 % survival.

The line also times, in the same invocation, the terrain batch against the same batch on flat terrains at 0.02 m and with no terrain set,
alternately, with device events around the episode call, and reports the launch counts of the three (terrains add no launch), whether
flat and unset give the same outcome, and the card's name and power limit and the clocks sampled during the timed episodes.

--estimator runs everything through hb_rollout_estimated_batch_dev (controllers on the Kalman filter's estimate from simulated sensors,
noise = SCALE x bench_rollout's NOISE_SIGMAS).
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from bench_rollout import GROUND, MIN_HEIGHT, NOISE_SIGMAS, gpu_identity  # noqa: E402
from bench import DT, HORIZON_N, SEED, ClockSampler  # noqa: E402  (bench_rollout put the repository root on the path)

TICKS = 750
KINDS = ["step_up", "step_down", "incline", "decline"]
MAGNITUDES = list(range(16))                             # [cm] for steps, [deg] for slopes
GRID, SPACING = 64, 0.025
STEP_AHEAD, RAMP_AHEAD = 0.15, 0.10                      # [m] ahead of the base origin along the initial heading


def feature_distances(rbd0, feet):
    """Per robot, how far ahead of the base origin along the initial heading the step's edge and the ramp's start lie: STEP_AHEAD and
    RAMP_AHEAD, or 1.5 cells ahead of the foremost start contact point (feet, B x 4 x 3) when that is further."""
    front = ((feet[:, :, 0] - rbd0[:, 3, None]) * np.cos(rbd0[:, 0, None]) + (feet[:, :, 1] - rbd0[:, 4, None]) * np.sin(rbd0[:, 0, None])).max(axis=1)
    return np.maximum(STEP_AHEAD, front + 1.5 * SPACING), np.maximum(RAMP_AHEAD, front + 1.5 * SPACING)


def terrain_heights(rbd0, kind, magnitude, step_ahead, ramp_ahead):
    """(origin (B, 2), heights (B, GRID, GRID)) of one kind and magnitude per robot, centred on each start pose, with the step's edge and
    the ramp's start step_ahead / ramp_ahead (B,) ahead of the base origin."""
    origin = rbd0[:, 3:5] - 0.5 * (GRID - 1) * SPACING
    k = SPACING * np.arange(GRID)
    X = origin[:, 0, None, None] + k[None, None, :]
    Y = origin[:, 1, None, None] + k[None, :, None]
    d = (X - rbd0[:, 3, None, None]) * np.cos(rbd0[:, 0])[:, None, None] + (Y - rbd0[:, 4, None, None]) * np.sin(rbd0[:, 0])[:, None, None]
    m = np.asarray(magnitude, dtype=float)[:, None, None]
    kind = np.asarray(kind)[:, None, None]
    step = np.where(d >= step_ahead[:, None, None], 0.01 * m, 0.0)
    ramp = np.maximum(d - ramp_ahead[:, None, None], 0.0) * np.tan(np.radians(m))
    h = np.select([kind == "step_up", kind == "step_down", kind == "incline"], [step, -step, ramp], -ramp)
    return origin, GROUND + h


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=4, help="episodes of the grid (the robot -> cell assignment shifts between them)")
    ap.add_argument("--timed", type=int, default=3, help="timed terrain / flat / unset episode triples")
    ap.add_argument("--batch", type=int, default=1024, help="robots per episode (a multiple of 64)")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--estimator", action="store_true", help="run the episodes through the state estimator")
    ap.add_argument("--sensor-noise", type=float, default=0.0, metavar="SCALE", help="with --estimator: sensor noise, SCALE x NOISE_SIGMAS")
    args = ap.parse_args()
    ncell = len(KINDS) * len(MAGNITUDES)
    if args.batch < ncell or args.batch % ncell or args.repeats < 1 or args.sensor_noise < 0 or (args.sensor_noise and not args.estimator):
        raise SystemExit("terrain_sweep.py: --batch a multiple of %d, --repeats >= 1, --sensor-noise takes a scale >= 0 and needs --estimator" % ncell)
    import torch
    import hunter_bipedal_control_b200 as hb
    from hunter_bipedal_control_b200 import scenarios as S
    if not torch.cuda.is_available():
        raise SystemExit("terrain_sweep.py: no CUDA device visible; the product path has no CPU fallback")
    dev = torch.device("cuda", args.device)
    torch.cuda.set_device(dev)
    B = args.batch
    ctx = hb.Context(horizon_N=HORIZON_N, dt=DT, max_batch=B, device=args.device)
    x0 = S.random_initial_states(B, SEED)
    rbd0 = S.consistent_rbd(x0)
    feet = ctx.contact_positions(x0).reshape(B, 4, 3)
    rbd0[:, 5] -= feet[:, :, 2].min(axis=1) - (GROUND - 0.001)
    step_ahead, ramp_ahead = feature_distances(rbd0, feet)
    prm = hb.default_rollout_params()
    prm.sim.ground_height = GROUND
    prm.min_base_height = MIN_HEIGHT
    cmds = hb.make_rollout_commands("trot", np.full(B, 0.1), [0.0], [[0.3, 0.0, 0.0, 0.0]])
    ep = hb.default_estimation_params()
    ep.noise.seed = SEED
    for k, v in NOISE_SIGMAS.items():
        setattr(ep.noise, k, args.sensor_noise * v)
    stream = torch.cuda.ExternalStream(ctx.stream_handle, device=dev)
    lib = hb.load_library()
    P = lambda t: C.c_void_p(t.data_ptr())
    T_episode = TICKS * prm.period

    def episode():
        d_rbd = torch.from_numpy(rbd0).to(dev)
        d_act = torch.zeros(B * C.sizeof(hb.HbActuationState), dtype=torch.uint8, device=dev)
        d_estop = torch.zeros(B, dtype=torch.uint8, device=dev)
        d_st = torch.from_numpy(hb.rollout_stats(B).view(np.uint8).copy()).to(dev)
        if args.estimator:
            d_est = torch.from_numpy(np.frombuffer(bytes(hb.estimation_states(B)), dtype=np.uint8).copy()).to(dev)
        torch.cuda.synchronize(dev)
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        l0 = ctx.launch_count
        e0.record(stream)
        if args.estimator:
            rc = lib.hb_rollout_estimated_batch_dev(ctx._h, B, C.c_int64(0), TICKS, C.byref(prm), C.byref(ep), cmds, P(d_rbd), P(d_act), P(d_estop), P(d_st),
                                                    P(d_est), None, None, None)
        else:
            rc = lib.hb_rollout_batch_dev(ctx._h, B, C.c_int64(0), TICKS, C.byref(prm), cmds, P(d_rbd), P(d_act), P(d_estop), P(d_st), None)
        e1.record(stream)
        assert rc == 0, rc
        ctx.sync()
        return e0.elapsed_time(e1), ctx.launch_count - l0, d_st.cpu().numpy().view(hb.ROLLOUT_STATS_DTYPE), d_rbd.cpu().numpy()

    def cells(shift):
        """(magnitude index, kind index) of every robot, assignment shifted by `shift`."""
        c = (np.arange(B) + shift) % ncell
        return c % len(MAGNITUDES), c // len(MAGNITUDES)

    def terrains(shift):
        mi, ki = cells(shift)
        origin, h = terrain_heights(rbd0, np.array(KINDS)[ki], np.array(MAGNITUDES)[mi], step_ahead, ramp_ahead)
        return hb.make_terrains(B, h, SPACING, origin)

    up = np.zeros((len(KINDS), len(MAGNITUDES)), dtype=int)
    total = np.zeros_like(up)
    speed = np.zeros((len(KINDS), len(MAGNITUDES)))
    reasons = {name: 0 for name in hb.ROLLOUT_FAIL}
    ctx.set_terrains(terrains(0))
    episode()                                   # warm-up episode
    for r in range(args.repeats):
        ctx.set_terrains(terrains(r))
        _, _, st, rbd = episode()
        mi, ki = cells(r)
        ok = st["fail_tick"] < 0
        v = np.hypot(*(rbd[:, 3:5] - rbd0[:, 3:5]).T) / T_episode
        np.add.at(total, (ki, mi), 1)
        np.add.at(up, (ki, mi), ok.astype(int))
        np.add.at(speed, (ki, mi), np.where(ok, v, 0.0))
        for name, bit in hb.ROLLOUT_FAIL.items():
            reasons[name] += int(((st["fail_reason"] & bit) != 0)[~ok].sum())
    survival = {k: {str(m): float(up[a, b] / total[a, b]) for b, m in enumerate(MAGNITUDES)} for a, k in enumerate(KINDS)}
    mean_speed = {k: {str(m): (float(speed[a, b] / up[a, b]) if up[a, b] else None) for b, m in enumerate(MAGNITUDES)} for a, k in enumerate(KINDS)}
    largest = {}                                # per kind: the largest magnitude up to which every cell keeps >= 90 % survival
    for a, k in enumerate(KINDS):
        largest[k] = None
        for b, m in enumerate(MAGNITUDES):
            if up[a, b] < 0.9 * total[a, b]:
                break
            largest[k] = m

    # terrain, flat-terrain and unset episodes alternate
    flat_origin, flat_h = terrain_heights(rbd0, np.full(B, "step_up"), np.zeros(B), step_ahead, ramp_ahead)
    flat = hb.make_terrains(B, flat_h, SPACING, flat_origin)
    sampler = ClockSampler(args.device); sampler.start()
    on_terrain, flats, unset = [], [], []
    for _ in range(max(1, args.timed)):
        ctx.set_terrains(terrains(0))
        on_terrain.append(episode())
        ctx.set_terrains(flat)
        flats.append(episode())
        ctx.set_terrains(None)
        unset.append(episode())
    clocks = sampler.stop()
    tm, fm, um = [r[0] for r in on_terrain], [r[0] for r in flats], [r[0] for r in unset]
    lt, lf, lu = on_terrain[-1][1], flats[-1][1], unset[-1][1]
    line = {"metric": "terrain: the highest step [cm] that >= 90 %% of the trotting robots cross blind within %.1f s; per kind (steps in cm, "
                      "slopes in degrees) under largest_magnitude_90pct" % T_episode, "value": largest["step_up"], "unit": "cm",
            "n_gpus": 1, "dtype": "f64", "data": "synthetic", "estimator": bool(args.estimator),
            "largest_magnitude_90pct": largest, "survival": survival, "mean_speed_of_survivors_m_per_s": mean_speed, "fail_reasons": reasons,
            "upright_fraction_unset": float((unset[-1][2]["fail_tick"] < 0).mean()),
            "timing": {"ms_per_episode_terrain": float(np.median(tm)), "ms_per_episode_terrain_range": [min(tm), max(tm)],
                       "ms_per_episode_flat": float(np.median(fm)), "ms_per_episode_flat_range": [min(fm), max(fm)],
                       "ms_per_episode_unset": float(np.median(um)), "ms_per_episode_unset_range": [min(um), max(um)],
                       "terrain_minus_unset_ms": float(np.median(tm) - np.median(um)), "flat_minus_unset_ms": float(np.median(fm) - np.median(um)),
                       "flat_same_outcome_as_unset": all(np.array_equal(f[2], u[2]) and np.array_equal(f[3], u[3]) for f, u in zip(flats, unset)),
                       "episodes": len(tm), "launches_terrain": int(lt), "launches_flat": int(lf), "launches_unset": int(lu),
                       "launches_equal": lt == lf == lu},
            "config": {"workload": "%d robots, %.1f s simulated (%d ticks of %.0f ms), trot at 0.3 m/s from t = 0.1 s, initial poses of "
                                   "scenarios.random_initial_states(seed %d), N=%d dt=%.0f ms; %d kinds x %d magnitudes, %d episodes"
                                   % (B, T_episode, TICKS, 1e3 * prm.period, SEED, HORIZON_N, 1e3 * DT, len(KINDS), len(MAGNITUDES), args.repeats),
                       "terrain": "%d x %d height field at %g m centred on the start, ground %g m under the start; steps with the edge %g m "
                                  "ahead (a ramp one cell wide), slopes starting %g m ahead, across the initial heading"
                                  % (GRID, GRID, SPACING, GROUND, STEP_AHEAD, RAMP_AHEAD),
                       "robots_with_features_moved_ahead": {"step": int((step_ahead > STEP_AHEAD).sum()), "ramp": int((ramp_ahead > RAMP_AHEAD).sum()),
                                                            "max_step_ahead_m": float(step_ahead.max()), "max_ramp_ahead_m": float(ramp_ahead.max())},
                       "survival": "robots still up at the end of the episode",
                       "failure_checks": "non-finite state, |roll| > pi/2, base z above the terrain < %.2f m, emergency stop" % MIN_HEIGHT},
            "gpu": gpu_identity(args.device), "clocks": clocks}
    if args.estimator:
        line["sensor_noise"] = {k: args.sensor_noise * v for k, v in NOISE_SIGMAS.items()}
        line["noise_seed"] = SEED
    print(json.dumps(line))


if __name__ == "__main__":
    main()
