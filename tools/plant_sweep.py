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
MASSES = [0.5 * k for k in range(16)]                   # [kg]
FRICTION = [1.0, 0.6, 0.4, 0.25]
BOX, COM = (0.2, 0.2, 0.1), (0.0, 0.0, 0.1)             # payload box edges [m] (x, y, z) and CoM in the base frame


def box_inertia(m):
    a, b, c = BOX
    return np.diag([m * (b * b + c * c) / 12, m * (a * a + c * c) / 12, m * (a * a + b * b) / 12])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=4, help="episodes of the grid (the robot -> cell assignment shifts between them)")
    ap.add_argument("--timed", type=int, default=3, help="timed varied / default / unset episode triples")
    ap.add_argument("--batch", type=int, default=1024, help="robots per episode (a multiple of 64)")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--estimator", action="store_true", help="run the episodes through the state estimator")
    ap.add_argument("--sensor-noise", type=float, default=0.0, metavar="SCALE", help="with --estimator: sensor noise, SCALE x NOISE_SIGMAS")
    args = ap.parse_args()
    ncell = len(MASSES) * len(FRICTION)
    if args.batch < ncell or args.batch % ncell or args.repeats < 1 or args.sensor_noise < 0 or (args.sensor_noise and not args.estimator):
        raise SystemExit("plant_sweep.py: --batch a multiple of %d, --repeats >= 1, --sensor-noise takes a scale >= 0 and needs --estimator" % ncell)
    import torch
    import hunter_bipedal_control_b200 as hb
    from hunter_bipedal_control_b200 import scenarios as S
    if not torch.cuda.is_available():
        raise SystemExit("plant_sweep.py: no CUDA device visible; the product path has no CPU fallback")
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
        """(payload index, friction index) of every robot, assignment shifted by `shift`."""
        c = (np.arange(B) + shift) % ncell
        return c % len(MASSES), c // len(MASSES)

    def variations(shift):
        mi, fi = cells(shift)
        m = np.array(MASSES)[mi]
        return hb.make_plant_variations(B, m, np.where(m[:, None] > 0, COM, 0.0), np.stack([box_inertia(x) for x in m]),
                                        friction_scale=np.array(FRICTION)[fi])

    up = np.zeros((len(FRICTION), len(MASSES)), dtype=int)
    total = np.zeros_like(up)
    speed = np.zeros((len(FRICTION), len(MASSES)))
    reasons = {name: 0 for name in hb.ROLLOUT_FAIL}
    ctx.set_plant_variations(variations(0))
    episode()                                   # warm-up episode
    for r in range(args.repeats):
        ctx.set_plant_variations(variations(r))
        _, _, st, rbd = episode()
        mi, fi = cells(r)
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
    default = hb.make_plant_variations(B)
    sampler = ClockSampler(args.device); sampler.start()
    varied, defaulted, unset = [], [], []
    for _ in range(max(1, args.timed)):
        ctx.set_plant_variations(variations(0))
        varied.append(episode())
        ctx.set_plant_variations(default)
        defaulted.append(episode())
        ctx.set_plant_variations(None)
        unset.append(episode())
    clocks = sampler.stop()
    vm, dm, um = [r[0] for r in varied], [r[0] for r in defaulted], [r[0] for r in unset]
    lv, ld, lu = varied[-1][1], defaulted[-1][1], unset[-1][1]
    line = {"metric": "model mismatch: the heaviest unmodelled payload (0.2 x 0.2 x 0.1 m box, CoM 0.1 m above the base) that >= 90 %% of the "
                      "trotting robots carry for %.1f s, per friction scale" % T_episode, "value": heaviest.get("1"), "unit": "kg",
            "n_gpus": 1, "dtype": "f64", "data": "synthetic", "estimator": bool(args.estimator),
            "heaviest_payload_90pct": heaviest, "survival": survival, "mean_speed_of_survivors_m_per_s": mean_speed, "fail_reasons": reasons,
            "upright_fraction_unset": float((unset[-1][2]["fail_tick"] < 0).mean()),
            "timing": {"ms_per_episode_varied": float(np.median(vm)), "ms_per_episode_varied_range": [min(vm), max(vm)],
                       "ms_per_episode_default": float(np.median(dm)), "ms_per_episode_default_range": [min(dm), max(dm)],
                       "ms_per_episode_unset": float(np.median(um)), "ms_per_episode_unset_range": [min(um), max(um)],
                       "varied_minus_unset_ms": float(np.median(vm) - np.median(um)), "default_minus_unset_ms": float(np.median(dm) - np.median(um)),
                       "default_same_outcome_as_unset": all(np.array_equal(d[2], u[2]) and np.array_equal(d[3], u[3]) for d, u in zip(defaulted, unset)),
                       "episodes": len(vm), "launches_varied": int(lv), "launches_default": int(ld), "launches_unset": int(lu),
                       "launches_equal": lv == ld == lu},
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
