"""ms per WBC call at --batch robots, timed alternately in one process: WeightedWbc (wbc_fused_kernel), the hierarchical composition
(hwbc_tasks_kernel + hoqp_kernel, the kernels behind hb_hierarchical_wbc_tasks_batch and hb_hoqp_solve_batch_dev) and the fused hierarchical
kernel (hb_hierarchical_wbc_solve_batch_dev). Prints one JSON line with the card's name and power limit."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=20, help="calls per timed window")
    ap.add_argument("--rounds", type=int, default=5, help="alternations of the three")
    args = ap.parse_args()
    import torch
    import hunter_bipedal_control_b200 as hb
    from hunter_bipedal_control_b200 import scenarios as sc
    from episode_harness import gpu_identity
    if not torch.cuda.is_available():
        raise SystemExit("bench_hwbc: no CUDA device visible; the product path has no CPU fallback")
    B = args.batch
    ctx = hb.Context(horizon_N=4, dt=0.01, max_batch=B, device=0)
    rng = np.random.default_rng(0)
    mode = np.array([3, 2, 1, 0] * ((B + 3) // 4), dtype=np.int32)[:B]
    x = np.tile(sc.INITIAL_STATE, (B, 1)) + rng.uniform(-.04, .04, (B, 22))
    u = np.zeros((B, 22))
    for i in range(B):
        fl = sc.mode_flags(int(mode[i]))
        for c in range(4):
            if fl[c]:
                u[i, 3 * c + 2] = sc.TOTAL_MASS * 9.81 / max(1, sum(fl))
        u[i, 12:] = rng.uniform(-.3, .3, 10)
    rbd = sc.consistent_rbd(x, rng, 0.01)
    dev = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a), dtype=dt).cuda()
    xd, ud, rd, md = dev(x), dev(u), dev(rbd), dev(mode, torch.int32)
    sol = torch.zeros(B, 38, dtype=torch.float64, device="cuda"); st = torch.zeros(B, dtype=torch.int32, device="cuda")
    pbs = torch.zeros(B * C.sizeof(hb.HbHoqpProblem), dtype=torch.uint8, device="cuda")
    lib, h, p = ctx._lib, ctx._h, lambda t: C.c_void_p(t.data_ptr())
    tasks = ctx.hierarchical_wbc_tasks(x, u, rbd, mode)            # the composition's problems (hwbc_tasks_kernel)
    pbs.copy_(torch.from_numpy(np.frombuffer(bytes(tasks), dtype=np.uint8).copy()))

    def weighted():
        return lib.hb_wbc_solve_batch_dev(h, B, p(xd), p(ud), p(rd), p(md), None, p(sol), p(st))

    def hoqp():
        return lib.hb_hoqp_solve_batch_dev(h, B, p(pbs), p(sol), None, p(st))

    def fused():
        return lib.hb_hierarchical_wbc_solve_batch_dev(h, B, p(xd), p(ud), p(rd), p(md), p(sol), p(st))

    def tasks_kernel_ms():
        """hwbc_tasks_kernel alone: the host-pointer call's kernel, timed by the context's per-kernel events (kind wbc_assemble)."""
        ctx.profile_enable(True)
        for _ in range(args.reps):
            ctx.hierarchical_wbc_tasks(x, u, rbd, mode)
        ms = ctx.profile_read()["wbc_assemble"]
        ctx.profile_enable(False)
        return ms["ms"] / ms["launches"]

    stream = torch.cuda.ExternalStream(ctx.stream_handle)          # the library launches on the context's own stream

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ctx.sync()
        e0.record(stream)
        for _ in range(args.reps):
            assert f() == 0
        e1.record(stream)
        ctx.sync()
        return e0.elapsed_time(e1) / args.reps

    for f in (weighted, hoqp, fused):
        timed(f)
    tasks_kernel_ms()
    times = {k: [] for k in ("weighted", "hierarchical_composition", "hierarchical_fused", "composition_tasks_kernel", "composition_hoqp_kernel")}
    for _ in range(args.rounds):
        times["weighted"].append(timed(weighted))
        tk, hq = tasks_kernel_ms(), timed(hoqp)
        times["composition_tasks_kernel"].append(tk); times["composition_hoqp_kernel"].append(hq)
        times["hierarchical_composition"].append(tk + hq)
        times["hierarchical_fused"].append(timed(fused))
    fs, stf = ctx.hierarchical_wbc_solve(x, u, rbd, mode)
    xc, _, stc = ctx.hoqp_solve(tasks)
    ok = (stf == 0) & (stc == 0)
    line = {"metric": "ms per WBC call at %d robots" % B, "gpu": gpu_identity(0)}
    for k, v in times.items():
        line[k] = {"ms_median": float(np.median(v)), "ms_range": [float(min(v)), float(max(v))]}
    line["fused_vs_composition_max_rel"] = float((np.abs(fs - xc).max(axis=1) / np.maximum(1.0, np.abs(xc).max(axis=1)))[ok].max())
    line["status_nonzero"] = {"fused": np.unique(stf[stf != 0], return_counts=True)[1].tolist(), "fused_codes": np.unique(stf[stf != 0]).tolist(),
                              "composition": np.unique(stc[stc != 0], return_counts=True)[1].tolist(), "composition_codes": np.unique(stc[stc != 0]).tolist()}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
