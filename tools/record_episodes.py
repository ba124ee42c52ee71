#!/usr/bin/env python3
"""Recorded channels of the episodes (hb_rollout_set_channel): prints one JSON line.

  python tools/record_episodes.py [--timed K] [--batch B] [--wbc weighted|hierarchical] [--out FILE.npz]

The workload of tools/bench_rollout.py (B robots, default 1024, from the randomised poses of bench.py's configs[1]) trots for 1.5 s (750
ticks) with the commanded speed spread over SPEEDS (robot i at SPEEDS[i % 5]), every channel recorded on every tick (log_every 1) along
with the state log, through hb_rollout_batch_dev and hb_rollout_estimated_batch_dev. Per call, K timed rounds (default 3) alternate the
episode without channels and with every channel set, after one warm-up of each; the line reports the median device time of each, the
overhead of recording, the launches, the bytes recorded, and whether the outcome (final stats, states, log and estimation stats) of the two
is bitwise equal in every round. Per commanded speed and call it reports the mechanical cost of transport of the robots that stayed up:
sum over ticks and joints of |tau q_dot| dt (tau from the torque channel, q_dot from the log row of the same tick) over m g times the
horizontal distance the base covered, its median and range, and the mean speed reached. All with the card's name and power limit.

--out FILE.npz writes the channels and the log of the last recorded episode of each call, keyed "<call>/<channel>" and "<call>/log".
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import Episodes, failure_checks, parser, report, workload  # noqa: E402
from bench import ClockSampler  # noqa: E402  (episode_harness put the repository root on the path)

TICKS = 750
SPEEDS = np.array([0.1, 0.2, 0.3, 0.4, 0.5])      # commanded forward speed [m/s]


def main():
    ap = parser()
    ap.add_argument("--timed", type=int, default=3, help="timed rounds of the episode without and with channels, per call")
    ap.add_argument("--out", help="write the channels and the log of the last recorded episode of each call to this .npz")
    args = ap.parse_args()
    h = Episodes("record_episodes.py", args, TICKS)
    hb, ctx, prm, B = h.hb, h.ctx, h.prm, h.B
    from hunter_bipedal_control_b200 import scenarios as S
    speed = SPEEDS[np.arange(B) % len(SPEEDS)]
    h.cmds = hb.make_rollout_commands("trot", np.full(B, 0.1), [0.0], np.c_[speed, np.zeros((B, 3))][:, None, :])
    bufs = hb.make_channels(B, TICKS)
    per_tick = {call: sum(w * np.dtype(t).itemsize for n, (_, t, w) in hb.CHANNELS.items() if call == "estimated" or n != "sensors")
                for call in ("truth", "estimated")}
    line = {"metric": "recorded channels: overhead of recording every channel on every tick of %d robots over %.1f s" % (B, TICKS * prm.period),
            "unit": "ms per episode"}
    saved = {}
    sampler = ClockSampler(args.device); sampler.start()
    for call, estimated in (("truth", False), ("estimated", True)):
        def episode(record):
            ctx.set_channels(bufs if record else None)
            return h.episode(estimated, est_stats=estimated, log_every=1)

        episode(False); episode(True)                       # warm-up
        runs = {False: [], True: []}
        for _ in range(max(1, args.timed)):
            for record in (False, True):
                runs[record].append(episode(record))
        ctx.set_channels(None)
        equal = all(np.array_equal(a.stats, b.stats) and np.array_equal(a.rbd, b.rbd) and np.array_equal(a.log, b.log)
                    and (not estimated or np.array_equal(a.est_stats, b.est_stats)) for a, b in zip(runs[False], runs[True]))
        ms = {r: [x.ms for x in runs[r]] for r in runs}
        rec = runs[True][-1]
        # mechanical cost of transport of the robots that stayed up, per commanded speed
        tau = bufs["torque"].cpu().numpy()
        energy = (np.abs(tau * rec.log[:, :, 22:32]).sum(axis=2) * prm.period).sum(axis=1)
        dist = np.hypot(*(rec.rbd[:, 3:5] - h.rbd0[:, 3:5]).T)
        up = rec.stats["fail_tick"] < 0
        cot = {}
        for s in SPEEDS:
            m = up & (speed == s)
            c = energy[m] / (S.TOTAL_MASS * 9.81 * dist[m])
            cot["%.1f" % s] = {"robots_up": int(m.sum()), "robots": int((speed == s).sum()),
                               "cost_of_transport_median": float(np.median(c)) if m.any() else None,
                               "cost_of_transport_range": [float(c.min()), float(c.max())] if m.any() else None,
                               "speed_reached_mean_m_s": float(dist[m].mean() / (TICKS * prm.period)) if m.any() else None}
        line[call] = {"ms_per_episode_unrecorded": float(np.median(ms[False])), "ms_per_episode_recorded": float(np.median(ms[True])),
                      "ms_per_episode_unrecorded_range": [min(ms[False]), max(ms[False])],
                      "ms_per_episode_recorded_range": [min(ms[True]), max(ms[True])],
                      "recording_overhead_ms": float(np.median(ms[True]) - np.median(ms[False])),
                      "recording_overhead_pct": float(100.0 * (np.median(ms[True]) / np.median(ms[False]) - 1.0)),
                      "launches_unrecorded": int(runs[False][-1].launches), "launches_recorded": int(runs[True][-1].launches),
                      "bytes_recorded_per_tick": int(per_tick[call] * B), "bytes_recorded_per_episode": int(per_tick[call] * B * TICKS),
                      "rounds": max(1, args.timed), "same_outcome_bitwise": bool(equal), "per_speed": cot}
        if args.out:
            saved.update({"%s/%s" % (call, n): t.cpu().numpy() for n, t in bufs.items() if estimated or n != "sensors"})
            saved["%s/log" % call] = rec.log
    line.update(report(args, sampler.stop(), estimator=False), value=line["truth"]["recording_overhead_ms"])
    line["config"] = {"workload": workload(h, ", no sensor noise; every channel and the log on every tick",
                                           "trot from t = 0.1 s at SPEEDS[i %% 5] = %s m/s" % SPEEDS.tolist()),
                      "failure_checks": failure_checks(),
                      "cost_of_transport": "sum over ticks and joints of |tau q_dot| dt / (m g horizontal distance), robots that stayed up"}
    if args.out:
        np.savez(args.out, **saved)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
