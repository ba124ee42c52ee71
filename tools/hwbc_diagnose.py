#!/usr/bin/env python3
"""Where the hierarchical WBC's closed-loop failures come from: prints one JSON line.

  python tools/hwbc_diagnose.py [--batch B] [--ticks T] [--wbc hierarchical] [--estimator [--sensor-noise SCALE]]

Runs the workload of tools/bench_rollout.py one tick per hb_rollout_batch_dev call (a continued episode is the one-call episode bit for
bit). Before every tick that starts no MPC cycle it evaluates the same WBC inputs with hb_resident_wbc_batch (policy of the resident
solution at the tick's time and state: the tick's own x_des, u_des, mode and WBC status; the call leaves the fallback state as the tick
leaves it). It then reports
  * the WBC status codes met in the loop, and how they split between robots that fail and robots that stay up, before their failure;
  * for every instance with a non-zero status and a sample of the solved ones, the same inputs solved by the composition
    (hb_hierarchical_wbc_tasks_batch + hb_hoqp_solve_batch): the cross table of the two status codes, and the largest difference of the
    two solutions where both solved, so a failure of the fused kernel that the composition does not share would show;
  * per failing robot, the WBC torque and joint state in the ticks before its failure.
Truth episodes only (--estimator is rejected: the tick's WBC inputs are then the estimator's, which this replay does not read)."""
import collections
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import Episodes, gpu_identity, parser  # noqa: E402
from bench import DT, HORIZON_N  # noqa: E402  (episode_harness put the repository root on the path)

SAMPLE = 32


def main():
    ap = parser()
    ap.add_argument("--ticks", type=int, default=500)
    args = ap.parse_args()
    if args.estimator:
        raise SystemExit("hwbc_diagnose.py: truth episodes only")
    h = Episodes("hwbc_diagnose.py", args, args.ticks)
    torch, hb, ctx, prm, B, dev = h.torch, h.hb, h.ctx, h.prm, h.B, h.dev
    ref = hb.Context(horizon_N=HORIZON_N, dt=DT, max_batch=B, device=args.device)   # same horizon: hb_create sizes the warm-shift kernel for it
    P = lambda t: C.c_void_p(t.data_ptr())
    d_rbd = torch.from_numpy(h.rbd0).to(dev)
    d_act = torch.zeros(B * C.sizeof(hb.HbActuationState), dtype=torch.uint8, device=dev)
    d_estop = torch.zeros(B, dtype=torch.uint8, device=dev)
    d_st = torch.from_numpy(hb.rollout_stats(B).view(np.uint8).copy()).to(dev)
    rng = np.random.default_rng(0)
    status = np.full((args.ticks, B), -1, dtype=np.int32)           # -1: tick not evaluated (MPC cycle tick) or robot already failed
    tau = np.full((args.ticks, B, 10), np.nan)
    qj = np.full((args.ticks, B, 10), np.nan)
    cross = collections.Counter()
    worst_rel, compared = 0.0, 0
    for a in range(args.ticks):
        ctx.sync()                                                  # the episode runs on the context's stream
        if a % prm.mpc_every and a >= prm.mpc_every:
            rbd = d_rbd.cpu().numpy()
            alive = d_st.cpu().numpy().view(hb.ROLLOUT_STATS_DTYPE)["fail_tick"] < 0
            xd, ud, md, sol, tq, st = ctx.resident_wbc(np.full(B, a * prm.period), rbd)
            status[a, alive] = st[alive]
            tau[a], qj[a] = tq, rbd[:, 6:16]
            bad = np.nonzero(alive & (st != 0))[0]
            good = np.nonzero(alive & (st == 0))[0]
            pick = np.concatenate([bad, rng.choice(good, min(SAMPLE, len(good)), replace=False)]) if len(good) else bad
            if len(pick):
                fs, fst = ref.hierarchical_wbc_solve(xd[pick], ud[pick], rbd[pick], md[pick])
                xc, _, cst = ref.hoqp_solve(ref.hierarchical_wbc_tasks(xd[pick], ud[pick], rbd[pick], md[pick]))
                assert np.array_equal(fst, st[pick])
                for f, c in zip(fst, cst):
                    cross["fused %d / composition %d" % (f, c)] += 1
                both = (fst == 0) & (cst == 0)
                if both.any():
                    rel = np.abs(fs - xc).max(axis=1) / np.maximum(1.0, np.abs(xc).max(axis=1))
                    worst_rel = max(worst_rel, float(rel[both].max()))
                    compared += int(both.sum())
        rc = h.lib.hb_rollout_batch_dev(ctx._h, B, C.c_int64(a), 1, C.byref(prm), h.cmds, P(d_rbd), P(d_act), P(d_estop), P(d_st), None)
        if rc != 0:
            raise SystemExit("hwbc_diagnose.py: hb_rollout_batch_dev at tick %d returned %d (%s)" % (a, rc, h.lib.hb_last_cuda_error(ctx._h).decode()))
    ctx.sync()
    stats = d_st.cpu().numpy().view(hb.ROLLOUT_STATS_DTYPE)
    failed = stats["fail_tick"] >= 0
    codes = collections.Counter(int(c) for c in status[status > 0].ravel())
    per = {}
    for name, rows in (("failing", np.nonzero(failed)[0]), ("upright", np.nonzero(~failed)[0])):
        s = status[:, rows]
        ev = s >= 0
        per[name] = {"robots": int(len(rows)), "evaluated_ticks": int(ev.sum()), "nonzero_status_ticks": int((s > 0).sum()),
                     "robots_with_a_nonzero_status": int((s > 0).any(axis=0).sum()),
                     "codes": {str(k): v for k, v in sorted(collections.Counter(int(c) for c in s[s > 0]).items())}}
    # the ticks before each failure
    lead = []
    limits = np.array(prm.torque_limit[:])
    for i in np.nonzero(failed)[0]:
        f = int(stats["fail_tick"][i])
        w = slice(max(0, f - 25), f)
        s = status[w, i]
        lead.append({"first_nonzero_tick_before_failure": (int(f - (np.nonzero(s > 0)[0][0] + w.start)) if (s > 0).any() else None),
                     "nonzero_in_last_25": int((s > 0).sum()),
                     "max_abs_tau_over_limit": float(np.nanmax(np.abs(tau[w, i]) / limits)) if np.isfinite(tau[w, i]).any() else None})
    first = [d["first_nonzero_tick_before_failure"] for d in lead]
    line = {"metric": "hierarchical WBC in the loop: status codes, fused kernel vs composition on the loop's own WBC inputs", "wbc": args.wbc,
            "ticks": args.ticks, "batch": B, "failed": int(failed.sum()),
            "fail_reasons": {n: int(((stats["fail_reason"] & bit) != 0).sum()) for n, bit in hb.ROLLOUT_FAIL.items()},
            "wbc_fallbacks": int(stats["wbc_fallbacks"].sum()), "status_codes": {str(k): v for k, v in sorted(codes.items())}, "by_outcome": per,
            "failing_robots_with_a_nonzero_status_in_the_25_ticks_before": int(sum(1 for x in first if x is not None)),
            "median_ticks_from_first_nonzero_to_failure": (float(np.median([x for x in first if x is not None])) if any(x is not None for x in first) else None),
            "median_max_abs_tau_over_limit_before_failure": float(np.median([d["max_abs_tau_over_limit"] for d in lead if d["max_abs_tau_over_limit"] is not None])) if lead else None,
            "fused_vs_composition": {"status_cross_table": dict(cross), "both_solved": compared, "max_rel_difference": worst_rel},
            "gpu": gpu_identity(args.device)}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
