#!/usr/bin/env python3
"""Motor bridge sweep of the episodes (hb_rollout_set_motor_bridge): prints one JSON line.

  python tools/bridge_sweep.py [--repeats R] [--timed K] [--batch B] [--wbc weighted|hierarchical]

The workload of tools/bench_rollout.py (B robots, default 1024, trotting at 0.3 m/s from the randomised poses of bench.py's configs[1])
runs for 1.5 s (750 ticks), once on the true state and once through the state estimator (sensor noise at 1 x NOISE_SIGMAS of
episode_harness.py). The batch is split into five blocks of consecutive robots, one per cumulative part of the real robot's joint path:
  pd_substeps  the motor PD on every plant substep only (scale 1, quantise 0, ranges that never bind);
  clamps       + the protocol's clamps (kp, kd, position, velocity, ff ranges of each joint's X or D motor);
  quantised    + the protocol's float32 codes (quantise 1), scale 1 on every joint;
  default      + the 0.7 command scale on joints 0, 1, 5, 6 (hb_default_motor_bridge);
  none         no record: the simulated hardware's torque law, once per tick.
The last block has no record (it lies beyond the setting); episode r of R rotates the four bridged parts over the first four blocks.
Per part: survival (robots up at the end), the RMS velocity-tracking error of the robots up (body-frame horizontal base velocity against
the 0.3 m/s command, over the logged ticks from 0.5 s on), WBC fallbacks per robot, and from the recorded joint commands
(HB_CHANNEL_JOINT_COMMAND) the share of logged ticks of robots up on which each joint's ff clamp binds (|scale x ff| > ff_max), for the
scales 0.7 and 1.0 of the default record. The line also times, alternately, the sweep as one call against one call per part, with
whether every part's final stats and states are bitwise equal between the two ways, and the default record on every robot against no
setting. All with the card's name and power limit.
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import NOISE_SIGMAS, Episodes, Tally, failure_checks, report, sweep_args, workload  # noqa: E402
from bench import SEED, ClockSampler  # noqa: E402  (episode_harness put the repository root on the path)

TICKS, LOG_EVERY, TRACK_FROM = 750, 5, 0.5           # ticks, logged every LOG_EVERY ticks, tracking error from TRACK_FROM s on
PARTS = ["pd_substeps", "clamps", "quantised", "default", "none"]
FAR = 1e300
CMD_VX = 0.3


def part_records(hb, part, n):
    """n records of one bridged part."""
    if part == "default":
        return hb.make_motor_bridges(n)
    kw = dict(command_scale=1.0, quantise=1 if part == "quantised" else 0)
    if part == "pd_substeps":
        kw.update(kp_max=FAR, kd_max=FAR, pos_max=FAR, vel_max=FAR, ff_max=FAR)
    return hb.make_motor_bridges(n, **kw)


def main():
    args = sweep_args("bridge_sweep.py", "timed rounds of one call against one call per part, and of the default bridge against no setting",
                      1, repeats=2)
    h = Episodes("bridge_sweep.py", args, TICKS)
    hb, ctx, B = h.hb, h.ctx, h.B
    block = np.arange(B) * len(PARTS) // B                                  # the block of each robot; the last block has no record
    nb = int((block < len(PARTS) - 1).sum())

    def part_of_block(r):
        return [PARTS[(b + r) % 4] for b in range(4)] + ["none"]

    def settings(r):
        parts = part_of_block(r)
        recs = (hb.HbMotorBridge * nb)()
        for b in range(4):
            m = np.nonzero(block == b)[0]
            for i, rec in zip(m, part_records(hb, parts[b], len(m))):
                recs[i] = rec
        return recs

    rows = (TICKS + LOG_EVERY - 1) // LOG_EVERY
    ch = hb.make_channels(B, rows, names=["joint_command"])
    ctx.set_channels(ch)
    default = hb.default_motor_bridge()
    scale, ff_max = np.array(default.command_scale[:]), np.array(default.ff_max[:])
    t_log = np.arange(rows) * LOG_EVERY * h.prm.period
    line = {"metric": "motor bridge sweep: survival of %d robots per part over the cumulative parts of the real robot's joint path" % (B // len(PARTS) * args.repeats),
            "unit": "fraction surviving", "parts": PARTS}
    for estimated in (False, True):
        args.estimator = estimated
        for k, v in NOISE_SIGMAS.items():
            setattr(h.ep.noise, k, v if estimated else 0.0)
        tally = Tally(len(PARTS), 1)
        err_sum, err_n = np.zeros(len(PARTS)), np.zeros(len(PARTS))
        binds = {s: np.zeros(10) for s in ("0.7", "1.0")}
        bind_n = {s: 0 for s in binds}
        for r, run in h.sweep(ctx.set_motor_bridge, settings, log_every=LOG_EVERY):
            col = np.array([PARTS.index(part_of_block(r)[b]) for b in block])
            tally.add(col, np.zeros(B, dtype=int), run.stats)
            up = run.stats["fail_tick"] < 0
            log = run.log                                                 # B x rows x 32, true state
            yaw = log[:, :, 0]
            vx = np.cos(yaw) * log[:, :, 19] + np.sin(yaw) * log[:, :, 20]
            vy = -np.sin(yaw) * log[:, :, 19] + np.cos(yaw) * log[:, :, 20]
            e2 = ((vx - CMD_VX) ** 2 + vy ** 2)[:, t_log >= TRACK_FROM]
            np.add.at(err_sum, col[up], e2[up].sum(axis=1)); np.add.at(err_n, col[up], e2.shape[1])
            ff = ch["joint_command"].cpu().numpy().reshape(B, rows, 10, 5)[:, :, :, 4]
            for s, part in (("0.7", "default"), ("1.0", "quantised")):
                m = up & (col == PARTS.index(part))
                sc = scale if s == "0.7" else np.ones(10)
                binds[s] += (np.abs(sc * ff[m]) > ff_max).sum(axis=(0, 1))
                bind_n[s] += int(m.sum()) * rows
        key = "estimator" if estimated else "truth"
        line[key] = {"survival": dict(zip(PARTS, tally.survival()[0].tolist())),
                     "velocity_tracking_err_rms_mps": dict(zip(PARTS, [float(np.sqrt(s / n)) if n else None for s, n in zip(err_sum, err_n)])),
                     "wbc_fallbacks_per_robot": dict(zip(PARTS, (tally.fallbacks[0] / np.maximum(tally.total[0], 1)).tolist())),
                     "ff_clamp_binds_share_by_joint": {"scale_" + s: (binds[s] / max(bind_n[s], 1)).tolist() for s in binds},
                     "fail_reasons": tally.reasons}
    line["value"] = line["estimator"]["survival"]["default"]

    # timing through the estimator, with the channels cleared: the sweep as one call against one call per part, alternated
    ctx.set_channels(None)
    sampler = ClockSampler(args.device); sampler.start()
    members = [np.nonzero(block == b)[0] for b in range(len(PARTS))]
    parts0 = part_of_block(0)

    def set_cell(k):
        ctx.set_motor_bridge(None if parts0[k] == "none" else part_records(hb, parts0[k], len(members[k])))

    timing = h.one_call_against_per_cell_calls(ctx.set_motor_bridge, settings(0), set_cell, lambda: ctx.set_motor_bridge(None), members, est_stats=True)
    # the default bridge on every robot against no setting, alternated
    ms = {"default_bridge": [], "unset": []}
    launches = {}
    for _ in range(max(1, args.timed)):
        for name, value in (("default_bridge", hb.make_motor_bridges(B)), ("unset", None)):
            ctx.set_motor_bridge(value)
            run = h.episode()
            ms[name].append(run.ms); launches[name] = int(run.launches)
    for name, v in ms.items():
        timing["ms_per_episode_" + name] = float(np.median(v)); timing["ms_per_episode_%s_range" % name] = [min(v), max(v)]
    timing["default_bridge_minus_unset_ms"] = timing["ms_per_episode_default_bridge"] - timing["ms_per_episode_unset"]
    timing["launches_equal"] = launches["default_bridge"] == launches["unset"]
    line["timing"] = timing
    line.update(report(args, sampler.stop(), estimator=False))
    line["config"] = {"workload": workload(h, "; %d robots per part, %d episodes per mode (parts rotated over the blocks)" % (B // len(PARTS), args.repeats),
                                           robots="robots, on the true state and through the estimator"),
                      "noise_sigmas_estimator": NOISE_SIGMAS, "noise_seed": SEED, "survival": "robots up at the end of the episode",
                      "failure_checks": failure_checks(), "timing": "through the estimator"}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
