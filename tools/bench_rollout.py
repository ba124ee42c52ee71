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
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import DT, HORIZON_N, SEED, ClockSampler  # noqa: E402

TICKS, GROUND, MIN_HEIGHT = 500, 0.02, 0.3
# sensor noise at --sensor-noise 1 (standard deviations): orientation [rad], gyro [rad/s], accelerometer [m/s^2], encoders [rad], [rad/s]
NOISE_SIGMAS = dict(orientation=0.005, angular_velocity=0.02, linear_acceleration=0.1, joint_position=0.001, joint_velocity=0.02)


def gpu_identity(index):
    """Card name and power limit, read in the run that measures."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True,
                             text=True, timeout=10).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1])}
    except Exception:
        return {"name": None, "power_limit_w": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="timed episodes")
    ap.add_argument("--batch", type=int, default=1024, help="robots per episode")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--estimator", action="store_true", help="also run the episodes through the state estimator")
    ap.add_argument("--sensor-noise", type=float, default=0.0, metavar="SCALE", help="with --estimator: sensor noise, SCALE x NOISE_SIGMAS")
    args = ap.parse_args()
    if args.sensor_noise < 0 or (args.sensor_noise and not args.estimator):
        raise SystemExit("bench_rollout.py: --sensor-noise takes a scale >= 0 and needs --estimator")
    import torch
    import hunter_bipedal_control_b200 as hb
    from hunter_bipedal_control_b200 import scenarios as S
    if not torch.cuda.is_available():
        raise SystemExit("bench_rollout.py: no CUDA device visible; the product path has no CPU fallback")
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
    cycles = sum(1 for k in range(TICKS) if k % prm.mpc_every == 0)
    stream = torch.cuda.ExternalStream(ctx.stream_handle, device=dev)
    lib = hb.load_library()
    P = lambda t: C.c_void_p(t.data_ptr())

    ep = hb.default_estimation_params()
    ep.noise.seed = SEED
    for k, v in NOISE_SIGMAS.items():
        setattr(ep.noise, k, args.sensor_noise * v)

    def episode(estimated=False):
        d_rbd = torch.from_numpy(rbd0).to(dev)
        d_act = torch.zeros(B * C.sizeof(hb.HbActuationState), dtype=torch.uint8, device=dev)
        d_estop = torch.zeros(B, dtype=torch.uint8, device=dev)
        d_st = torch.from_numpy(hb.rollout_stats(B).view(np.uint8).copy()).to(dev)
        if estimated:
            d_est = torch.from_numpy(np.frombuffer(bytes(hb.estimation_states(B)), dtype=np.uint8).copy()).to(dev)
            d_es = torch.from_numpy(hb.estimation_stats(B).view(np.uint8).copy()).to(dev)
        torch.cuda.synchronize(dev)
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        l0 = ctx.launch_count
        e0.record(stream)
        if estimated:
            rc = lib.hb_rollout_estimated_batch_dev(ctx._h, B, C.c_int64(0), TICKS, C.byref(prm), C.byref(ep), cmds, P(d_rbd), P(d_act), P(d_estop), P(d_st),
                                                    P(d_est), P(d_es), None, None)
        else:
            rc = lib.hb_rollout_batch_dev(ctx._h, B, C.c_int64(0), TICKS, C.byref(prm), cmds, P(d_rbd), P(d_act), P(d_estop), P(d_st), None)
        e1.record(stream)
        assert rc == 0, rc
        ctx.sync()
        run = (e0.elapsed_time(e1), ctx.launch_count - l0, d_st.cpu().numpy().view(hb.ROLLOUT_STATS_DTYPE))
        return run + (d_es.cpu().numpy().view(hb.ESTIMATION_STATS_DTYPE),) if estimated else run

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
    ms = [r[0] for r in runs]
    st = runs[-1][2]
    med = float(np.median(ms))
    sim_s = TICKS * prm.period
    reasons = {name: int(((st["fail_reason"] & bit) != 0).sum()) for name, bit in hb.ROLLOUT_FAIL.items()}
    line = {"metric": "closed-loop episodes: simulated robot-seconds per wall-second (Hunter, MPC 100 Hz + WBC 500 Hz + plant)", "value": B * sim_s / (med * 1e-3),
            "unit": "robot-s/s", "n_gpus": 1, "steps": len(runs), "warmup": 1, "higher_is_better": True, "dtype": "f64", "data": "synthetic",
            "ms_per_episode": med, "ms_per_episode_range": [min(ms), max(ms)], "ms_per_mpc_period": med / cycles,
            "launches_per_mpc_period": runs[-1][1] / cycles, "gpu_launches": int(runs[-1][1]),
            "upright_fraction": float((st["fail_tick"] == -1).mean()), "fail_reasons": reasons,
            "same_outcome_every_episode": all(np.array_equal(r[2], st) for r in runs),
            "stats": {"mpc_bad": int(st["mpc_bad"].sum()), "wbc_fallbacks": int(st["wbc_fallbacks"].sum()), "plan_rejects": int(st["plan_rejects"].sum()),
                      "max_abs_torque": float(st["max_abs_torque"].max())},
            "config": {"workload": "%d robots, %.1f s simulated (%d ticks of %.0f ms, %d MPC cycles), trot at 0.3 m/s from t = 0.1 s, initial poses of "
                                   "scenarios.random_initial_states(seed %d), N=%d dt=%.0f ms, one hb_rollout_batch_dev call per episode, device events "
                                   "around it" % (B, sim_s, TICKS, 1e3 * prm.period, cycles, SEED, HORIZON_N, 1e3 * DT),
                       "failure_checks": "non-finite state, |roll| > pi/2, base z < %.2f m, emergency stop" % MIN_HEIGHT},
            "gpu": gpu_identity(args.device), "clocks": clocks}
    if args.estimator:
        ems = [r[0] for r in est_runs]
        est_st, es = est_runs[-1][2], est_runs[-1][3]
        emed = float(np.median(ems))
        n = max(int(es["count"].sum()), 1)
        line["estimator"] = {
            "ms_per_episode": emed, "ms_per_episode_range": [min(ems), max(ems)], "ms_per_mpc_period": emed / cycles,
            "extra_ms_per_tick": (emed - med) / TICKS, "launches_per_mpc_period": est_runs[-1][1] / cycles, "gpu_launches": int(est_runs[-1][1]),
            "upright_fraction": float((est_st["fail_tick"] == -1).mean()), "upright_fraction_ground_truth": float((st["fail_tick"] == -1).mean()),
            "fail_reasons": {name: int(((est_st["fail_reason"] & bit) != 0).sum()) for name, bit in hb.ROLLOUT_FAIL.items()},
            "vel_err_rms": float(np.sqrt(es["sum_sq_vel_err"].sum() / n)), "vel_err_max": float(es["max_vel_err"].max()),
            "height_err_rms": float(np.sqrt(es["sum_sq_height_err"].sum() / n)), "height_err_max": float(es["max_height_err"].max()),
            "stats": {"mpc_bad": int(est_st["mpc_bad"].sum()), "wbc_fallbacks": int(est_st["wbc_fallbacks"].sum()),
                      "plan_rejects": int(est_st["plan_rejects"].sum()), "max_abs_torque": float(est_st["max_abs_torque"].max())},
            "same_outcome_every_episode": all(np.array_equal(r[2], est_st) and np.array_equal(r[3], es) for r in est_runs),
            "sensor_noise": {k: args.sensor_noise * v for k, v in NOISE_SIGMAS.items()}, "noise_seed": SEED,
            "errors": "filter output against the true state entering each tick, counted while the robot is up: |v_hat - v| world base "
                      "velocity [m/s], |z_hat - z| [m]; rms over robots and ticks"}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
