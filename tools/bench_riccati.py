"""K2 (`riccati_kernel`) per control step against the number of co-resident blocks per SM.

The Riccati sweep runs one block per instance and 8 blocks per SM, so on the 132 SMs of an H100 a batch of 132 * b instances puts b
blocks on every SM. The time at 132 instances is the latency of one block's chain of 100 nodes; the slope over b is what each further
co-resident block costs, i.e. how far the kernel is bound by what an SM can issue and not by that chain. Times are CUDA events on the
launch stream (`hb_profile_enable`), configs[1] of bench.py (trot, N = 100). One JSON line; card name, power limit and the throttle
reasons seen during the timed steps are part of it.

  python tools/bench_riccati.py [--steps 20] [--warmup 3] [--batches 132,264,528,792,924,1056,1024]
"""
import argparse, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import hunter_bipedal_control_b200 as hb
import bench


def card(index):
    out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, timeout=10).stdout.strip().split(",")
    return {"name": out[0].strip(), "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batches", default="132,264,528,792,924,1056,1024")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_riccati.py: no CUDA device visible")
    steps, warmup = max(args.steps, 20), max(args.warmup, 3)
    batches = [int(b) for b in args.batches.split(",")]
    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    x0, x_ref, swing, mode, rbd = bench.workload(max(batches))      # instance i is the same in every batch
    to = lambda a, dt_=torch.float64: torch.from_numpy(np.ascontiguousarray(a)).to(dev, dtype=dt_)
    rows = []
    reasons = set()
    for B in batches:
        ctx = hb.Context(horizon_N=bench.HORIZON_N, dt=bench.DT, max_batch=B)
        stream = torch.cuda.ExternalStream(ctx.stream_handle, device=dev)
        d_x0, d_xref, d_swing, d_rbd, d_mode = to(x0[:B]), to(x_ref[:B]), to(swing[:B]), to(rbd[:B]), to(mode[:B], torch.int32)
        d_xt0 = torch.zeros((B, bench.HORIZON_N + 1, 22), dtype=torch.float64, device=dev)
        d_ut0 = torch.zeros((B, bench.HORIZON_N, 22), dtype=torch.float64, device=dev)
        ctx.mpc_cold_start_dev(d_x0, d_mode, d_xt0, d_ut0); ctx.sync()
        d_xt, d_ut = d_xt0.clone(), d_ut0.clone()
        d_info = torch.zeros((B, 7), dtype=torch.float64, device=dev); d_sol = torch.zeros((B, 38), dtype=torch.float64, device=dev)
        d_tau = torch.zeros((B, 10), dtype=torch.float64, device=dev); d_st = torch.zeros(B, dtype=torch.int32, device=dev)

        def step():
            with torch.cuda.stream(stream):
                d_xt.copy_(d_xt0, non_blocking=True); d_ut.copy_(d_ut0, non_blocking=True)      # every step is the cold-start solve
            ctx.control_step_dev(bench.T_POLICY, d_x0, d_xref, d_swing, d_mode, d_rbd, d_xt, d_ut, d_info, d_sol, d_tau, d_st)

        for _ in range(warmup):
            step()
        ctx.sync(); torch.cuda.synchronize(dev)
        ctx.profile_enable(True)
        sampler = bench.ClockSampler(0); sampler.start()
        for _ in range(steps):
            step()
        ctx.sync(); torch.cuda.synchronize(dev)
        clocks = sampler.stop()
        prof = ctx.profile_read()
        ctx.profile_enable(False)
        reasons.update(clocks["reasons"])
        rows.append({"batch": B, "blocks_per_sm": round(B / sms, 2), "mpc_riccati_ms": prof["mpc_riccati"]["ms"] / steps, "sm_mhz": clocks["sm_mhz"],
                     "converged": int((d_st == 0).sum().item())})
        del ctx
    # lone-block latency and the cost of each further co-resident block, from the batches that fill every SM equally
    full = [(r["batch"] // sms, r["mpc_riccati_ms"]) for r in rows if r["batch"] % sms == 0]
    fit = None
    if len(full) >= 2:
        slope, icpt = np.polyfit([b for b, _ in full], [t for _, t in full], 1)
        fit = {"ms_per_block_per_sm": float(slope), "ms_at_one_block": float(dict(full).get(1, icpt + slope))}
    print(json.dumps({"metric": "mpc_riccati ms per control step, configs[1], N=%d" % bench.HORIZON_N, "steps": steps, "warmup": warmup, "sms": sms,
                      "card": card(0), "throttle_reasons": sorted(reasons), "rows": rows, "fit": fit}))


if __name__ == "__main__":
    main()
