"""Parity tests proper (run on an H100 with -m gpu): the CUDA path, called through the C ABI, against the CPU oracle on the same
seeded inputs, against the committed golden vectors, and -- at BASELINE.json's full sizes -- through size-independent
properties. Tolerances: 1e-4 relative on output torques (north_star); everything upstream of the QP is held to <= 1e-8."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TAU_RTOL = 1e-4   # BASELINE.json north_star: "output torques match the reference CPU path ... to 1e-4 relative"


def S():
    from hunter_bipedal_control_b200 import scenarios
    return scenarios


def rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


def test_extension_loaded_and_launch_counter(gpu_ctx):
    import hunter_bipedal_control_b200 as hb
    assert hb.load_library() is not None
    c0 = gpu_ctx.launch_count
    gpu_ctx.rbd_to_centroidal(np.zeros((1, 32)) + np.r_[np.zeros(5), 0.63, S().DEFAULT_JOINTS, np.zeros(16)])
    assert gpu_ctx.launch_count == c0 + 1


def test_flow_map_and_ee_jacobians_vs_oracle(gpu_ctx, oracle):
    sc = S()
    rng = np.random.default_rng(1)
    B = 24
    x = sc.random_initial_states(B, seed=5)
    u = rng.uniform(-30, 60, (B, 22)); u[:, 12:] = rng.uniform(-2, 2, (B, 10))
    pr = gpu_ctx.probe_flow_map(x, u)
    for i in range(B):
        f, A, Bm = oracle.flow_map(x[i], u[i])
        pos, vel, dp, dvx, dvu = oracle.ee_kinematics(x[i], u[i])
        assert np.abs(f - pr["f"][i]).max() < 1e-10
        assert np.abs(A - pr["A"][i]).max() < 1e-9 and np.abs(Bm - pr["B"][i]).max() < 1e-10
        assert np.abs(pos - pr["epos"][i]).max() < 1e-12 and np.abs(vel - pr["evel"][i]).max() < 1e-11
        assert np.abs(dp - pr["dpos_dx"][i]).max() < 1e-11
        assert np.abs(dvx - pr["dvel_dx"][i]).max() < 1e-9 and np.abs(dvu - pr["dvel_du"][i]).max() < 1e-11


def test_rbd_to_centroidal_vs_oracle(gpu_ctx, oracle):
    sc = S()
    rng = np.random.default_rng(2)
    x = sc.random_initial_states(16, seed=9)
    rbd = sc.consistent_rbd(x, rng, 0.05)
    xg = gpu_ctx.rbd_to_centroidal(rbd)
    for i in range(16):
        assert np.abs(oracle.rbd_to_centroidal(rbd[i]) - xg[i]).max() < 1e-12


def _wbc_cases(B, seed):
    sc = S()
    rng = np.random.default_rng(seed)
    mode = rng.choice([3, 3, 2, 1, 0], B).astype(np.int32)
    x = np.tile(sc.INITIAL_STATE, (B, 1)) + rng.uniform(-.05, .05, (B, 22))
    u = np.zeros((B, 22))
    for i in range(B):
        fl = sc.mode_flags(int(mode[i]))
        for c in range(4):
            if fl[c]:
                u[i, 3 * c + 2] = sc.TOTAL_MASS * 9.81 / sum(fl)
        u[i, 12:] = rng.uniform(-.5, .5, 10)
    rbd = sc.consistent_rbd(x, rng, 0.02)
    stance = (rng.uniform(size=B) < 0.15).astype(np.uint8) * (mode == 3)
    return x, u, rbd, mode, stance.astype(np.uint8)


def test_wbc_solve_vs_oracle(gpu_ctx, oracle):
    x, u, rbd, mode, stance = _wbc_cases(96, 21)
    sol, st = gpu_ctx.wbc_solve(x, u, rbd, mode, stance)
    assert (st == 0).all()
    so, sto = oracle.wbc_solve_batch(x, u, rbd, mode, stance, 1e-8, threads=4)
    assert (sto == 0).all()
    for i in range(len(mode)):
        assert rel(sol[i, 28:], so[i, 28:]) < TAU_RTOL, (i, mode[i])
        assert rel(sol[i], so[i]) < 1e-4


def test_wbc_device_assembly_vs_oracle(gpu_ctx, oracle):
    """hb_wbc_assemble_batch (W1-W3 in the qpOASES layout of WeightedWbc.cpp:24-42) against the oracle's assembly, entry by entry."""
    x, u, rbd, mode, stance = _wbc_cases(40, 23)
    H, g, A, lb, ub, m = gpu_ctx.wbc_assemble(x, u, rbd, mode, stance)
    for i in range(len(mode)):
        Hi, gi, Ai, lbi, ubi = oracle.wbc_assemble(x[i], u[i], rbd[i], int(mode[i]), bool(stance[i]))
        assert m[i] == Ai.shape[0]
        sc_ = max(1.0, np.abs(Hi).max())
        assert np.abs(H[i] - Hi).max() < 1e-9 * sc_ and np.abs(g[i] - gi).max() < 1e-9 * max(1.0, np.abs(gi).max())
        assert np.abs(A[i, :m[i]] - Ai).max() < 1e-9 * max(1.0, np.abs(Ai).max())
        fin = np.abs(lbi) < 1e19
        assert np.abs(lb[i, :m[i]][fin] - lbi[fin]).max() < 1e-8 * max(1.0, np.abs(lbi[fin]).max()) and (lb[i, :m[i]][~fin] <= -1e19).all()
        assert np.abs(ub[i, :m[i]] - ubi).max() < 1e-8 * max(1.0, np.abs(ubi).max())


def test_wbc_assembly_and_raw_qp_vs_oracle(gpu_ctx, oracle):
    """Config 5 path: raw (H, g, A, lbA, ubA) problems in qpOASES layout, mixed 56/58/60-row problems padded to 60 rows."""
    x, u, rbd, mode, stance = _wbc_cases(48, 22)
    B = len(mode)
    H = np.zeros((B, 38, 38)); g = np.zeros((B, 38)); A = np.zeros((B, 60, 38)); lb = np.full((B, 60), -1e20); ub = np.full((B, 60), 1e20)
    for i in range(B):
        Hi, gi, Ai, lbi, ubi = oracle.wbc_assemble(x[i], u[i], rbd[i], int(mode[i]), bool(stance[i]))
        m = Ai.shape[0]
        H[i] = Hi; g[i] = gi; A[i, :m] = Ai; lb[i, :m] = lbi; ub[i, :m] = ubi
    xs, st, it = gpu_ctx.wbc_qp(H, g, A, lb, ub)
    assert (st == 0).all() and (it < 40).all()
    xo, sto = oracle.wbc_qp_batch(H, g, A, lb, ub, 1e-8, threads=4)
    for i in range(B):
        assert rel(xs[i, 28:], xo[i, 28:]) < TAU_RTOL
        # KKT-free property checks on the device solution itself
        assert np.abs(A[i, :16] @ xs[i] - ub[i, :16]).max() < 1e-7
        assert (np.abs(xs[i, 28:]) <= np.tile([28, 60, 60, 60, 28], 2) + 1e-6).all()
    # fused path == assemble + raw solve
    sol, st2 = gpu_ctx.wbc_solve(x, u, rbd, mode, stance)
    # the fused path solves the reduced problem (tau, swing forces eliminated): same optimum up to the interior-point tolerance
    assert np.abs(sol - xs).max() < 1e-5 * max(1, np.abs(xs).max())
    assert max(rel(sol[i, 28:], xs[i, 28:]) for i in range(B)) < 0.1 * TAU_RTOL


def test_mpc_iteration_vs_golden_and_oracle(oracle):
    import hunter_bipedal_control_b200 as hb
    g = np.load(os.path.join(HERE, "golden", "path_golden.npz"))
    N, dt = int(g["N"]), float(g["dt"])
    ctx = hb.Context(horizon_N=N, dt=dt, max_batch=16)
    B = g["x0"].shape[0]
    xt, ut = ctx.mpc_cold_start(g["x0"], g["mode"])
    assert np.array_equal(xt, g["xt0"]) and np.array_equal(ut, g["ut0"])
    xt1, ut1, info = ctx.mpc_solve(g["x0"], g["x_ref"], g["swing"], g["mode"], xt, ut)
    assert (info["status"] == 0).all() and np.array_equal(info["alpha"], g["alpha"][:, 0])
    assert np.abs(xt1 - g["xt1"]).max() < 1e-8 and np.abs(ut1 - g["ut1"]).max() < 1e-6
    assert np.abs(info["merit1"] - g["merit"][:, 0]).max() < 1e-8 and np.abs(info["viol1"] - g["viol"][:, 0]).max() < 1e-9
    xt2, ut2, info2 = ctx.mpc_solve(g["x0"], g["x_ref"], g["swing"], g["mode"], xt1, ut1)
    assert np.array_equal(info2["alpha"], g["alpha"][:, 1])
    assert np.abs(xt2 - g["xt2"]).max() < 1e-8 and np.abs(ut2 - g["ut2"]).max() < 1e-6
    # WBC goldens
    sol, st = ctx.wbc_solve(g["wx"], g["wu"], g["wrbd"], g["wmode"], g["wstance"])
    assert (st == 0).all()
    for i in range(len(st)):
        assert rel(sol[i, 28:], g["wsol"][i, 28:]) < TAU_RTOL
    ctx.close()


def test_mpc_backtracking_line_search_vs_oracle(oracle):
    """A poor warm start forces alpha < 1 on some instances: the filter line search must take the same decisions."""
    import hunter_bipedal_control_b200 as hb
    sc = S()
    N, dt = 16, 0.02
    seeds = [9, 21, 1, 5, 13, 17, 25, 29]     # 9 and 21 back-track (alpha 0.5 / 0.25) with the recipe below
    B = len(seeds)
    ctx = hb.Context(horizon_N=N, dt=dt, max_batch=B)
    x0 = np.zeros((B, 22)); x_ref = np.zeros((B, N + 1, 22)); swing = np.zeros((B, N + 1, 24)); mode = np.zeros((B, N + 1), dtype=np.int32)
    xt = np.zeros((B, N + 1, 22)); ut = np.zeros((B, N, 22))
    for i, seed in enumerate(seeds):
        rng = np.random.default_rng(seed)
        a, b, c, d = sc.make_batch(1, N, dt, gait=["trot", "flying_trot", "standing_trot"][seed % 3], seed=1000 + seed)
        x0[i], x_ref[i], swing[i], mode[i] = a[0], b[0], c[0], d[0]
        xi, ui = oracle.mpc_cold_start(N, dt, x0[i], mode[i])
        for _ in range(3):                                     # converge, then push the joint trajectory far off
            xi, ui, _ = oracle.mpc_iteration(N, dt, x0[i], x_ref[i], swing[i], mode[i], xi, ui)
        xi[1:, 12:] += rng.uniform(-0.6, 0.6, (N, 10))
        xt[i], ut[i] = xi, ui
    xt1, ut1, info = ctx.mpc_solve(x0, x_ref, swing, mode, xt, ut)
    n_bt = 0
    for i in range(B):
        xo, uo, io = oracle.mpc_iteration(N, dt, x0[i], x_ref[i], swing[i], mode[i], xt[i], ut[i])
        assert io["alpha"] == info["alpha"][i] and io["n_trials"] == info["n_trials"][i]
        n_bt += io["alpha"] < 1.0
        assert np.abs(xo - xt1[i]).max() < 1e-7 * max(1, np.abs(xo).max())
        assert np.abs(uo - ut1[i]).max() < 1e-6 * max(1, np.abs(uo).max())
    assert n_bt >= 1
    ctx.close()


def test_mpc_full_size_vs_oracle_and_properties(gpu_ctx, oracle):
    """BASELINE config 2 shape (trot, N=100, dt=10 ms): oracle parity on a sample, size-independent properties on all."""
    sc = S()
    N, dt, B = 100, 0.01, 256
    gaits = [["stance", "trot", "standing_trot", "flying_trot"][i % 4] for i in range(B)]
    x0, x_ref, swing, mode = sc.make_batch(B, N, dt, gaits=gaits)
    xt, ut = gpu_ctx.mpc_cold_start(x0, mode)
    viol = []
    cur = (xt, ut)
    for it in range(3):
        nxt = gpu_ctx.mpc_solve(x0, x_ref, swing, mode, cur[0], cur[1])
        info = nxt[2]
        assert (info["status"] == 0).all()
        # filter line search property: an accepted step never increases both merit and violation
        acc = info["alpha"] > 0
        assert (acc.mean() > 0.95)
        assert ((info["merit1"] < info["merit0"]) | (info["viol1"] < info["viol0"]))[acc].all()
        assert np.array_equal(nxt[0][:, 0], x0)          # first node pinned to the measured state
        if it == 0:
            for i in (0, 1, 2, 3, 77, 255):
                xo, uo, io = oracle.mpc_iteration(N, dt, x0[i], x_ref[i], swing[i], mode[i], cur[0][i], cur[1][i])
                assert io["alpha"] == info["alpha"][i]
                assert np.abs(xo - nxt[0][i]).max() < 1e-7 * max(1, np.abs(xo).max())
                assert np.abs(uo - nxt[1][i]).max() < 1e-6 * max(1, np.abs(uo).max())
        viol.append(np.median(info["viol1"]))
        cur = (nxt[0], nxt[1])
    assert viol[2] < viol[0]
    # permutation invariance: instances are independent
    perm = np.random.default_rng(0).permutation(B)
    a = gpu_ctx.mpc_solve(x0[perm], x_ref[perm], swing[perm], mode[perm], xt[perm], ut[perm])
    b = gpu_ctx.mpc_solve(x0, x_ref, swing, mode, xt, ut)
    assert np.array_equal(a[0], b[0][perm]) and np.array_equal(a[1], b[1][perm])


def test_control_step_torques_vs_oracle(gpu_ctx, oracle):
    sc = S()
    N, dt, B = 100, 0.01, 32
    x0, x_ref, swing, mode = sc.make_batch(B, N, dt, gait="trot", seed=99)
    rbd = sc.consistent_rbd(x0, np.random.default_rng(3), 0.01)
    xt, ut = gpu_ctx.mpc_cold_start(x0, mode)
    xt1, ut1, info, sol, tau, st = gpu_ctx.control_step(0.002, x0, x_ref, swing, mode, rbd, xt, ut)
    assert (st == 0).all() and (info["status"] == 0).all()
    assert np.array_equal(tau, sol[:, 28:])
    for i in range(0, B, 4):
        xo, uo, io = oracle.mpc_iteration(N, dt, x0[i], x_ref[i], swing[i], mode[i], xt[i], ut[i])
        al = 0.002 / dt
        xd = (1 - al) * xo[0] + al * xo[1]; ud = (1 - al) * uo[0] + al * uo[1]
        so, sto = oracle.wbc_solve(xd, ud, rbd[i], int(mode[i][0]), False, 1e-8)
        assert sto == 0 and rel(tau[i], so[28:]) < TAU_RTOL


def test_reference_expand_matches_host_generator(gpu_ctx):
    import ctypes as C
    import hunter_bipedal_control_b200 as hb
    sc = S()
    N, dt = gpu_ctx.N, gpu_ctx.dt
    B = 6
    x0 = sc.random_initial_states(B, seed=3)
    refs = (hb.HbReference * B)()
    exp = []
    for i in range(B):
        gait = ["trot", "standing_trot", "flying_trot", "stance", "trot", "trot"][i]
        xr, sw, md, c = sc.make_reference(x0[i], (0.2, 0, 0, 0.1), gait, N, dt, phase=0.05 * i)
        exp.append((xr, sw, md))
        r = refs[i]
        r.n_events = len(c["events"])
        for k, t in enumerate(c["events"]):
            r.event_times[k] = t
        for k, m in enumerate(c["modes"]):
            r.modes[k] = m
        r.n_targets = 2
        for k in range(2):
            r.target_times[k] = c["target_times"][k]
            for j in range(22):
                r.target_states[k][j] = c["target_states"][k][j]
        for cc in range(4):
            for a in range(3):
                segs = [sg for sg in c["segments"][cc][a] if sg[0] <= N * dt + 1e-9]   # only what the horizon can see
                assert len(segs) <= 24
                r.n_segments[cc][a] = len(segs)
                for s, sg in enumerate(segs):
                    for j in range(6):
                        r.segments[cc][a][s][j] = sg[j]
    xr, sw, md = gpu_ctx.reference_expand(np.zeros(B), refs)
    for i in range(B):
        assert np.array_equal(md[i], exp[i][2])
        assert np.abs(xr[i] - exp[i][0]).max() < 1e-12 and np.abs(sw[i] - exp[i][1]).max() < 1e-12


def test_mirror_classes(oracle):
    import hunter_bipedal_control_b200 as hb
    sc = S()
    wbc = hb.WeightedWbc()
    with pytest.raises(hb.HunterB200Error):
        wbc.loadTasksSetting("/nonexistent/task.info", False)      # the reference throws on a missing task file too (boost read_info)
    wbc.loadTasksSetting(None, False)                              # no file: the shipped values stay in force
    x = sc.INITIAL_STATE; u = np.zeros(22); u[[2, 5, 8, 11]] = sc.TOTAL_MASS * 9.81 / 4
    rbd = np.r_[x[9:12], x[6:9], x[12:], np.zeros(16)]
    s1 = wbc.update(x, u, rbd, 3, 0.002)              # stance mode until setStanceMode(False)
    so, _ = oracle.wbc_solve(x, u, rbd, 3, True, 1e-8)
    assert s1.shape == (38,) and rel(s1[28:], so[28:]) < TAU_RTOL
    wbc.setStanceMode(False)
    s2 = wbc.update(x, u, rbd, 3, 0.002)
    so, _ = oracle.wbc_solve(x, u, rbd, 3, False, 1e-8)
    assert rel(s2[28:], so[28:]) < TAU_RTOL and wbc.getContactForceSize() == 12


def test_runtime_wbc_settings_from_task_info(oracle):
    """WbcBase::loadTasksSetting / WeightedWbc::loadTasksSetting / setKpKd honoured at run time: gains, limits and weights loaded from a
    task.info variant change the device WBC exactly as they change the restatement (assembly entry by entry, torques to 1e-4)."""
    import hunter_bipedal_control_b200 as hb
    ctx = hb.Context(horizon_N=10, dt=0.02, max_batch=64, device=0)
    x, u, rbd, mode, stance = _wbc_cases(32, 31)
    base, _ = ctx.wbc_solve(x, u, rbd, mode, stance)
    try:
        ctx.load_task_info(os.path.join(HERE, "golden", "task_wbc_variant.info"))
        s = ctx.wbc_settings()
        assert s.swing_kp == 140.0 and s.weight_contact_force == 0.02 and list(s.torque_limits) == [25.0, 55.0, 50.0, 58.0, 20.0]
        for variant in range(2):
            if variant == 1:
                ctx.set_kp_kd(90.0, 9.0)                       # WbcBase::setKpKd (WbcBase.h:65-69)
                s = ctx.wbc_settings()
                assert (s.swing_kp, s.swing_kd) == (90.0, 9.0)
            oracle.set_wbc_settings(s.as_array())
            H, g, A, lb, ub, m = ctx.wbc_assemble(x, u, rbd, mode, stance)
            sol, st = ctx.wbc_solve(x, u, rbd, mode, stance)
            assert (st == 0).all()
            changed = 0
            for i in range(len(mode)):
                Hi, gi, Ai, lbi, ubi = oracle.wbc_assemble(x[i], u[i], rbd[i], int(mode[i]), bool(stance[i]))
                assert np.abs(H[i] - Hi).max() < 1e-9 * max(1.0, np.abs(Hi).max()) and np.abs(g[i] - gi).max() < 1e-9 * max(1.0, np.abs(gi).max())
                assert np.abs(A[i, :m[i]] - Ai).max() < 1e-9 * max(1.0, np.abs(Ai).max()) and np.abs(ub[i, :m[i]] - ubi).max() < 1e-8 * max(1.0, np.abs(ubi).max())
                so, sto = oracle.wbc_solve(x[i], u[i], rbd[i], int(mode[i]), bool(stance[i]), 1e-8)
                assert sto == 0 and rel(sol[i, 28:], so[28:]) < TAU_RTOL, (variant, i)
                assert (np.abs(sol[i, 28:]) <= np.tile(list(s.torque_limits), 2) + 1e-6).all()
                changed += rel(sol[i, 28:], base[i, 28:]) > 1e-3
            assert changed > len(mode) // 2                    # the new settings do change the answer
    finally:
        oracle.set_wbc_settings(None)
        ctx.close()
