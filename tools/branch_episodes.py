#!/usr/bin/env python3
"""Push recovery against gait phase from forked episodes (Context.save_episodes / restore_episodes): prints one JSON line.

  python tools/branch_episodes.py [--batch B] [--phases P] [--speeds V ...] [--directions D] [--timed K] [--sensor-noise SCALE]
                                  [--wbc W] [--out FILE.npz]

1. Settle: one robot per speed (default 0.0, 0.25 and 0.5 m/s) trots from the standing pose of tools/episode_harness.py for 2 s.
2. Snapshot: the robots are saved at P phases (default 16) of the next gait cycle (0.6 s trot cycle, gait.info), one save every
   cycle / P.
3. Fork: each robot's snapshot at each phase is restored into B copies (default 1024), one cell each of D directions (default 16, evenly
   spaced in the horizontal plane) x B / D magnitudes (0, 10, 20, ... N).
4. Push: each copy gets one world-frame push at the base for 0.1 s from the fork tick (set_pushes), and runs 1.5 s on.
Both steps run through hb_rollout_batch_dev and, from their own settled robots, hb_rollout_estimated_batch_dev. A copy survives when it is
still up 1.5 s after the fork; per speed, phase and direction the line reports the smallest push that felled the copy (null: none did).

Timing: for the middle speed at phase 0, the forked sweep (a restore and the 1.5 s episode of the B copies) alternates with the same cells
re-simulated without a fork (B robots from standing through the whole prefix, with the push schedules), --timed times, with a host
clock around calls that return once the device has finished. Every cell of the re-simulated run must equal the forked cell bit for bit
(final state and stats); the line reports it. The card's name and power limit are read in the same run.
"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import GROUND, MIN_HEIGHT, NOISE_SIGMAS, gpu_identity, parser  # noqa: E402
from bench import DT, HORIZON_N, SEED  # noqa: E402  (episode_harness put the repository root on the path)

SETTLE_S, CYCLE_S, AFTER_S, PUSH_S, STEP_N = 2.0, 0.6, 1.5, 0.1, 10.0


def main():
    ap = parser("copies per snapshot (a multiple of --directions)")
    ap.add_argument("--phases", type=int, default=16)
    ap.add_argument("--speeds", type=float, nargs="+", default=[0.0, 0.25, 0.5])
    ap.add_argument("--directions", type=int, default=16)
    ap.add_argument("--timed", type=int, default=3, help="alternated forked / re-simulated rounds")
    ap.add_argument("--out", help="write every cell's survival to this .npz")
    args = ap.parse_args()
    if args.batch % args.directions or args.phases < 1 or args.timed < 1:
        raise SystemExit("branch_episodes.py: --batch a multiple of --directions, --phases >= 1, --timed >= 1")
    import torch
    import hunter_bipedal_control_b200 as hb
    from hunter_bipedal_control_b200 import scenarios as S
    if not torch.cuda.is_available():
        raise SystemExit("branch_episodes.py: no CUDA device visible; the product path has no CPU fallback")
    dev = torch.device("cuda", args.device)
    torch.cuda.set_device(dev)
    B, V, D = args.batch, len(args.speeds), args.directions
    prm = hb.default_rollout_params()
    prm.sim.ground_height, prm.min_base_height = GROUND, MIN_HEIGHT
    settle, step, after = (int(round(s / prm.period)) for s in (SETTLE_S, CYCLE_S / args.phases, AFTER_S))
    ep = hb.default_estimation_params()
    ep.noise.seed = SEED
    for k, v in NOISE_SIGMAS.items():
        setattr(ep.noise, k, args.sensor_noise * v)

    def context():
        ctx = hb.Context(horizon_N=HORIZON_N, dt=DT, max_batch=B, device=args.device)
        ctx.set_wbc_formulation(args.wbc)
        return ctx

    probe = context()
    x0 = np.tile(S.INITIAL_STATE, (1, 1))
    rbd0 = S.consistent_rbd(x0)
    rbd0[:, 5] -= probe.contact_positions(x0).reshape(1, 4, 3)[:, :, 2].min() - (GROUND - 0.001)
    probe.close()
    cmds = lambda speeds: hb.make_rollout_commands("trot", 0.1, [0.0], np.array([[[v, 0.0, 0.0, 0.0]] for v in speeds]))
    angle = 2 * np.pi * (np.arange(B) % D) / D
    mag = (np.arange(B) // D) * STEP_N
    force = np.stack([np.cos(angle), np.sin(angle), np.zeros(B)], axis=1) * mag[:, None]

    def pushes(tick):
        return hb.make_push_schedules(B, tick * prm.period, PUSH_S, force[:, None, :])

    def run(ctx, rbd, speeds, n, tick0, state, estimated):
        """One episode call; state: (act, estop, stats[, est, est_stats]), None entries and None fresh (est: noise stream i for robot i).
        Returns (outputs, ms): the host clock around the call, which returns once the device has finished the episode."""
        state = list(state or (None,) * 5)
        t0 = time.perf_counter()
        kw = dict(tick0=tick0, params=prm, act=state[0], estop=state[1], stats=state[2])
        if estimated:
            est = state[3]
            if est is None:
                est = torch.from_numpy(np.frombuffer(bytes(hb.estimation_states(len(speeds))), dtype=np.uint8).copy()).to(dev)
            out = ctx.rollout_estimated(rbd, cmds(speeds), n, est_params=ep, est=est, est_stats=state[4], **kw)
        else:
            out = ctx.rollout(rbd, cmds(speeds), n, **kw)
        return out, 1e3 * (time.perf_counter() - t0)

    def saved(out, estimated):
        return (out[1], out[2], out[3]) + ((out[5], out[6]) if estimated else ())

    result = {}
    timing = {}
    for estimated in (False, True):
        name = "estimated" if estimated else "truth"
        # 1-2: settle the robots, then a snapshot at every phase of the next cycle
        sctx = context()
        out, _ = run(sctx, torch.from_numpy(np.repeat(rbd0, V, axis=0)).to(dev), args.speeds, settle, 0, None, estimated)
        snaps = []
        for p in range(args.phases):
            if p:
                out, _ = run(sctx, out[0], args.speeds, step, settle + (p - 1) * step, saved(out, estimated), estimated)
            snaps.append(sctx.save_episodes(V, out[0], *saved(out, estimated)))
        up_at_fork = [bool(s) for s in snaps[-1].stats["fail_tick"] < 0]
        sctx.close()
        # 3-4: fork every snapshot into the push cells
        fctx = context()
        first_fall = np.full((V, args.phases, D), np.nan)
        alive = np.zeros((V, args.phases, B), dtype=bool)
        for v in range(V):
            for p in range(args.phases):
                fork = settle + p * step
                fctx.set_pushes(pushes(fork))
                r = fctx.restore_episodes(snaps[p], [v] * B)
                o, _ = run(fctx, r[0], [args.speeds[v]] * B, after, fork, r[1:], estimated)
                ok = o[3]["fail_tick"] < 0
                alive[v, p] = ok
                for d in range(D):
                    fell = mag[d::D][~ok[d::D]]
                    first_fall[v, p, d] = fell.min() if fell.size else np.nan
        # timing and the bitwise check: the middle speed at phase 0, forked against re-simulated from standing
        v = V // 2
        fork = settle
        fctx.set_pushes(pushes(fork))
        rctx = context()
        rctx.set_pushes(pushes(fork))
        ms_fork, ms_resim, equal = [], [], True
        for _ in range(args.timed):
            t0 = time.perf_counter()
            r = fctx.restore_episodes(snaps[0], [v] * B)          # synchronous
            f, ms = run(fctx, r[0], [args.speeds[v]] * B, after, fork, r[1:], estimated)
            ms_fork.append(1e3 * (time.perf_counter() - t0))
            state = None
            if estimated:                                          # the settled robot's noise stream in every cell
                est = hb.estimation_states(B)
                for i in range(B):
                    est[i].noise_stream = v
                state = (None, None, None, torch.from_numpy(np.frombuffer(bytes(est), dtype=np.uint8).copy()).to(dev), None)
            g, ms = run(rctx, torch.from_numpy(np.repeat(rbd0, B, axis=0)).to(dev), [args.speeds[v]] * B, fork + after, 0, state, estimated)
            ms_resim.append(ms)
            equal &= bool(torch.equal(f[0], g[0]) and np.array_equal(f[3], g[3]))
        rctx.close(); fctx.close()
        timing[name] = {"ms_forked_sweep": float(np.median(ms_fork)), "ms_forked_sweep_range": [min(ms_fork), max(ms_fork)],
                        "ms_resimulated_sweep": float(np.median(ms_resim)), "ms_resimulated_sweep_range": [min(ms_resim), max(ms_resim)],
                        "speedup": float(np.median(ms_resim) / np.median(ms_fork)), "rounds": args.timed,
                        "cells_bitwise_equal": equal, "cells_checked": B, "speed_checked": args.speeds[v]}
        result[name] = {"settled_robot_up": dict(zip(map(str, args.speeds), up_at_fork)),
                        "survival_by_speed_phase": {str(s): [float(alive[i, p].mean()) for p in range(args.phases)] for i, s in enumerate(args.speeds)},
                        "smallest_felling_push_N": {str(s): [[None if np.isnan(x) else float(x) for x in first_fall[i, p]] for p in range(args.phases)]
                                                    for i, s in enumerate(args.speeds)}}
        if args.out:
            np.savez(args.out.replace(".npz", "_%s.npz" % name), alive=alive, magnitude=mag, direction=angle, speeds=args.speeds)
    line = {"metric": "push recovery against gait phase from forked episodes: the smallest %.1f s push that fells a copy, per speed, phase and "
                      "direction" % PUSH_S, "unit": "N", "n_gpus": 1, "dtype": "f64", "data": "synthetic", "wbc": args.wbc, "results": result,
            "timing": timing,
            "config": {"workload": "%d copies per snapshot, %d phases of a %.1f s trot cycle after %.1f s of settling, speeds %s m/s, %d directions x "
                                   "%d magnitudes (step %.0f N), %.1f s after the fork, N=%d dt=%.0f ms" % (B, args.phases, CYCLE_S, SETTLE_S, args.speeds, D,
                                                                                                        B // D, STEP_N, AFTER_S, HORIZON_N, 1e3 * DT),
                       "survival": "up 1.5 s after the fork (failure checks: non-finite state, |roll| > pi/2, base z < %.2f m, estop)" % MIN_HEIGHT,
                       "sensor_noise": {k: args.sensor_noise * v for k, v in NOISE_SIGMAS.items()}},
            "gpu": gpu_identity(args.device)}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
