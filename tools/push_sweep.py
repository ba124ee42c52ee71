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

TICKS, PUSH_T, PUSH_DURATION = 750, 0.5, 0.1
DIRECTIONS = {"+x": (1.0, 0.0, 0.0), "-x": (-1.0, 0.0, 0.0), "+y": (0.0, 1.0, 0.0), "-y": (0.0, -1.0, 0.0)}
STEP_N, BLOCK, MAX_FORCE, SURVIVE = 10.0, 16, 1000.0, 0.9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=4, help="episodes per grid block (the robot -> cell assignment shifts between them)")
    ap.add_argument("--timed", type=int, default=3, help="timed pushed / unpushed episode pairs")
    ap.add_argument("--batch", type=int, default=1024, help="robots per episode (a multiple of 64)")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--estimator", action="store_true", help="run the episodes through the state estimator")
    ap.add_argument("--sensor-noise", type=float, default=0.0, metavar="SCALE", help="with --estimator: sensor noise, SCALE x NOISE_SIGMAS")
    args = ap.parse_args()
    ncell = len(DIRECTIONS) * BLOCK
    if args.batch < ncell or args.batch % ncell or args.repeats < 1 or args.sensor_noise < 0 or (args.sensor_noise and not args.estimator):
        raise SystemExit("push_sweep.py: --batch a multiple of %d, --repeats >= 1, --sensor-noise takes a scale >= 0 and needs --estimator" % ncell)
    import torch
    import hunter_bipedal_control_b200 as hb
    from hunter_bipedal_control_b200 import scenarios as S
    if not torch.cuda.is_available():
        raise SystemExit("push_sweep.py: no CUDA device visible; the product path has no CPU fallback")
    dev = torch.device("cuda", args.device)
    torch.cuda.set_device(dev)
    B = args.batch
    ctx = hb.Context(horizon_N=HORIZON_N, dt=DT, max_batch=B, device=args.device)
    x0 = S.random_initial_states(B, SEED)
    rbd0 = S.consistent_rbd(x0)
    rbd0[:, 5] -= ctx.contact_positions(x0).reshape(B, 4, 3)[:, :, 2].min(axis=1) - (GROUND - 0.001)
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
    push_tick = int(round(PUSH_T / prm.period))

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
        return e0.elapsed_time(e1), ctx.launch_count - l0, d_st.cpu().numpy().view(hb.ROLLOUT_STATS_DTYPE)

    def cells(block, shift):
        """(direction index, magnitude) of every robot for grid block `block`, assignment shifted by `shift`."""
        c = (np.arange(B) + shift) % ncell
        return c // BLOCK, (block * BLOCK + c % BLOCK) * STEP_N

    def schedules(block, shift):
        d, mag = cells(block, shift)
        dirs = np.array(list(DIRECTIONS.values()))
        return hb.make_push_schedules(B, PUSH_T, PUSH_DURATION, (dirs[d] * mag[:, None])[:, None, :])

    names = list(DIRECTIONS)
    up = {n: {} for n in names}
    survived = {n: {} for n in names}
    reasons = {name: 0 for name in hb.ROLLOUT_FAIL}
    ctx.set_pushes(schedules(0, 0))
    episode()                                   # warm-up episode
    block = 0
    while True:
        for r in range(args.repeats):
            ctx.set_pushes(schedules(block, r))
            _, _, st = episode()
            d, mag = cells(block, r)
            was_up = (st["fail_tick"] < 0) | (st["fail_tick"] > push_tick)
            ok = st["fail_tick"] < 0
            for i in np.nonzero(was_up)[0]:
                key = "%g" % mag[i]
                up[names[d[i]]][key] = up[names[d[i]]].get(key, 0) + 1
                survived[names[d[i]]][key] = survived[names[d[i]]].get(key, 0) + int(ok[i])
                for name, bit in hb.ROLLOUT_FAIL.items():
                    reasons[name] += int(not ok[i] and (st["fail_reason"][i] & bit) != 0)
        top = "%g" % ((block + 1) * BLOCK * STEP_N - STEP_N)
        if (block + 1) * BLOCK * STEP_N > MAX_FORCE or all(survived[n].get(top, 0) < SURVIVE * max(up[n].get(top, 0), 1) for n in names):
            break
        block += 1

    survival = {n: {k: survived[n][k] / up[n][k] for k in sorted(up[n], key=float)} for n in names}
    largest = {}
    for n in names:
        good = [float(k) for k, f in survival[n].items() if f >= SURVIVE]
        largest[n] = max(good) if good else None

    # pushed, zero-force (schedules set, the trajectories of the unpushed batch: the cost of the wrench path alone) and unpushed episodes
    # alternate
    zero = hb.make_push_schedules(B, PUSH_T, PUSH_DURATION, [0.0, 0.0, 0.0])
    sampler = ClockSampler(args.device); sampler.start()
    pushed, zeroed, unpushed = [], [], []
    for _ in range(max(1, args.timed)):
        ctx.set_pushes(schedules(0, 0))
        pushed.append(episode())
        ctx.set_pushes(zero)
        zeroed.append(episode())
        ctx.set_pushes(None)
        unpushed.append(episode())
    clocks = sampler.stop()
    pm, zm, um = [r[0] for r in pushed], [r[0] for r in zeroed], [r[0] for r in unpushed]
    lp, lu = pushed[-1][1], unpushed[-1][1]
    known = [v for v in largest.values() if v is not None]
    line = {"metric": "push recovery: the largest %.1f s world-frame push at the base, over the four horizontal directions, that >= 90 %% of the "
                      "trotting robots survive" % PUSH_DURATION, "value": min(known) if len(known) == len(names) else None, "unit": "N",
            "n_gpus": 1, "dtype": "f64", "data": "synthetic", "estimator": bool(args.estimator),
            "largest_force_90pct": largest, "survival": survival, "robots_up_at_push": up, "fail_reasons_after_push": reasons,
            "upright_fraction_unpushed": float((unpushed[-1][2]["fail_tick"] < 0).mean()),
            "timing": {"ms_per_episode_pushed": float(np.median(pm)), "ms_per_episode_pushed_range": [min(pm), max(pm)],
                       "ms_per_episode_unpushed": float(np.median(um)), "ms_per_episode_unpushed_range": [min(um), max(um)],
                       "pushed_minus_unpushed_ms": float(np.median(pm) - np.median(um)),
                       "ms_per_episode_zero_force": float(np.median(zm)), "ms_per_episode_zero_force_range": [min(zm), max(zm)],
                       "zero_force_minus_unpushed_ms": float(np.median(zm) - np.median(um)),
                       "zero_force_same_outcome_as_unpushed": all(np.array_equal(z[2], u[2]) for z, u in zip(zeroed, unpushed)), "episodes": len(pm),
                       "launches_pushed": int(lp), "launches_unpushed": int(lu), "launches_equal": lp == lu == zeroed[-1][1]},
            "config": {"workload": "%d robots, %.1f s simulated (%d ticks of %.0f ms), trot at 0.3 m/s from t = 0.1 s, initial poses of "
                                   "scenarios.random_initial_states(seed %d), N=%d dt=%.0f ms; one push per robot at t = %.1f s for %.1f s, %d "
                                   "episodes per grid block of %d magnitudes x 4 directions" % (B, TICKS * prm.period, TICKS, 1e3 * prm.period, SEED,
                                                                                                HORIZON_N, 1e3 * DT, PUSH_T, PUSH_DURATION, args.repeats, BLOCK),
                       "survival": "robots up when the push began (fail_tick < 0 or after tick %d) that are still up at the end" % push_tick,
                       "failure_checks": "non-finite state, |roll| > pi/2, base z < %.2f m, emergency stop" % MIN_HEIGHT},
            "gpu": gpu_identity(args.device), "clocks": clocks}
    if args.estimator:
        line["sensor_noise"] = {k: args.sensor_noise * v for k, v in NOISE_SIGMAS.items()}
        line["noise_seed"] = SEED
    print(json.dumps(line))


if __name__ == "__main__":
    main()
