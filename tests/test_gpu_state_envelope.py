"""The MPC solve across the robot's state envelope (tests/state_envelope_ref.py) on the device, against the float64 oracle: far attitudes,
unwrapped yaw, far positions, large momentum, joints at their range ends, fast joints and large forces. The suite's other device-vs-oracle
checks of the centroidal model and the SQP iteration use near-nominal states only, and the closed-loop episodes, which run far outside that
box, compare the device with itself.

1. The flow map and contact kinematics that the linearisation uses (probe_flow_map), on every axis, with the suite's absolute bounds (f 1e-10,
   A 1e-9, B 1e-10, contact positions 1e-12, velocities 1e-11, dpos/dx 1e-11, dvel/dx 1e-9, dvel/du 1e-11). SCALED lists the entries whose
   bound is taken relative to max(1, |ref|) on an axis that makes them large, and why.
2. Two SQP iterations from the cold start on every solve case (all four gaits), on the uniform grid and on an event grid, plus poor warm
   starts whose line search back-tracks, so that it evaluates the flow map at trial points far from the linearisation. The suite's
   tolerances: alpha and n_trials equal, merit0 within 1e-8, x within 1e-7 and u within 1e-6 of max(1, |ref|).
3. Yaw + 2 pi k and horizontal shifts of the solve cases on the device alone, transformed back: within the host test's bounds, equal alpha.
4. Envelope instances mixed with nominal ones leave every nominal instance bitwise equal to its solve alone.
5. Near the vertical (pitch 1.55 to 1.5707963): status 0 with finite output matching the oracle (to its rounding floor), or a non-zero
   status with the iterate kept; the rest of the batch unchanged.
6. control_step torques against the oracle at the 1e-4 north-star tolerance: attitude to 0.5 rad, yaw to 1e3 rad, positions to 1e3 m,
   joints and hbar within random_initial_states' box. With hbar beyond it, or joints anywhere in their range, the device's WBC returns
   status 2 or 3 where the oracle's solves the problem; that is a strict expected failure with its own exception (WbcStatusMismatch).
7. The axes contain the x_des / u_des recorded through pushed, sloped and turning estimated episodes.

Rounding floor. Some instances are ill-conditioned: near the vertical (|A| grows like 100 / cos(pitch)) and where hbar is far from what
the joints can absorb after a poor warm start. There the oracle itself moves by 4e-7 (pitch 1.57), 3e-2 (pitch 1.5707), 1e-6 to 1e-4
(hbar +-1 with the poor warm start) and 1e-5 (one mixed state) when x0 and the warm start are perturbed by one ulp, and by the same amount
for perturbations up to 1e-13. No float64 implementation can agree with it more closely than that. An instance outside the suite's x / u
bounds is held to FLOOR times its rounding floor (state_envelope_ref.rounding_floor) instead, with alpha, n_trials and merit0 still exact;
the tests print which instances those are, and at most four per test may be."""
import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
import state_envelope_ref as E

pytestmark = pytest.mark.gpu

N, DT = 20, 0.02
THREADS = 8
BOUNDS = dict(f=1e-10, A=1e-9, B=1e-10, epos=1e-12, evel=1e-11, dpos_dx=1e-11, dvel_dx=1e-9, dvel_du=1e-11)
# entries held relative to max(1, |ref|), per axis. The mixed sample combines hbar to +-1, joint velocities to 10 rad/s and positions to
# 1e3 m, so f reaches 2e2 (14 at nominal states), the contact velocities 3e1 (3 at nominal states) and dvel/dx 3e1; joint velocities of
# 40 rad/s make f 40 and the contact velocities 2.4e1. A, B, the contact positions and dpos/dx, dvel/du keep their absolute bounds.
SCALED = {"mixed": ("f", "evel", "dvel_dx"), "joint_velocity": ("f", "evel", "dvel_dx")}
FLOOR = 5.0          # x / u bounds: the suite's, or FLOOR times the rounding floor of the instance (state_envelope_ref.rounding_floor)
INV_X, INV_U = 1e-10, 1e-9
# (state label, gait, seed): poor warm starts whose first oracle iteration back-tracks, chosen with the oracle alone
BACKTRACK = (("pitch +1.2", "trot", 9), ("ypr -3 -1.4 1", "flying_trot", 2), ("yaw 1000", "flying_trot", 7),
             ("position -1000 1000 0.63", "standing_trot", 7), ("all joints upper", "trot", 2), ("hbar all", "standing_trot", 0),
             ("mixed 3", "trot", 5))
NEAR_VERTICAL = (1.55, 1.56, 1.57, 1.5707, 1.5707963)


def _oracle_iterations(oracle, x0, xr, sw, md, xt, ut):
    o1 = oracle.mpc_iteration_batch(N, DT, x0, xr, sw, md, xt, ut, threads=THREADS)
    o2 = oracle.mpc_iteration_batch(N, DT, x0, xr, sw, md, o1[0], o1[1], threads=THREADS)
    return o1, o2


def _check_iteration(dev, orc, i, what, floor=(0.0, 0.0)):
    io, idv = orc[2][i], dev[2][i]
    assert idv["status"] == 0 == io["status"], (what, idv, io)
    assert io["alpha"] == idv["alpha"] and io["n_trials"] == idv["n_trials"], (what, io, idv)
    # merit0 of a second iteration is evaluated at the first one's result, which may differ by the rounding floor
    assert abs(io["merit0"] - idv["merit0"]) < max(1e-8, FLOOR * max(floor)) * max(1.0, abs(io["merit0"])), (what, io["merit0"], idv["merit0"])
    ex, eu = E.rel(dev[0][i], orc[0][i]), E.rel(dev[1][i], orc[1][i])
    assert ex < max(1e-7, FLOOR * floor[0]) and eu < max(1e-6, FLOOR * floor[1]), (what, ex, eu, floor)
    return ex, eu


def _floors(oracle, n, dts, case, iterations):
    """Rounding floor of `iterations` oracle iterations of one case (x0, x_ref, swing, mode, xt, ut) on n intervals."""
    def run(c):
        xt, ut = c[4], c[5]
        for _ in range(iterations):
            xt, ut, _ = oracle.mpc_iteration(n, dts, c[0], c[1], c[2], c[3], xt, ut)
        return xt, ut
    return E.rounding_floor(run, case)


@pytest.fixture(scope="module")
def ctx():
    c = hb.Context(horizon_N=N, dt=DT, max_batch=128, device=0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def cases(oracle):
    return E.solve_cases(N, DT, oracle)


@pytest.mark.parametrize("axis", E.AXES + ("mixed",))
def test_flow_map_on_every_axis_vs_oracle(axis, ctx, oracle):
    pts = E.all_points()[axis]
    x = np.stack([p[1] for p in pts]); u = np.stack([p[2] for p in pts])
    pr = ctx.probe_flow_map(x, u)
    worst = dict.fromkeys(BOUNDS, 0.0)
    bad = []
    for i, (label, _, _) in enumerate(pts):
        f, A, Bm = oracle.flow_map(x[i], u[i])
        pos, vel, dp, dvx, dvu = oracle.ee_kinematics(x[i], u[i])
        for k, ref in (("f", f), ("A", A), ("B", Bm), ("epos", pos), ("evel", vel), ("dpos_dx", dp), ("dvel_dx", dvx), ("dvel_du", dvu)):
            err = np.abs(pr[k][i] - ref).max()
            if k in SCALED.get(axis, ()):
                err /= max(1.0, np.abs(ref).max())
            worst[k] = max(worst[k], err)
            if not err < BOUNDS[k]:
                bad.append((label, k, err))
    print(axis, " ".join("%s %.1e" % kv for kv in worst.items()))
    assert not bad, bad


def _batch_with_backtracking(cases, oracle):
    st = {lab: x for _, lab, x, _ in E._case_states()}
    bt = [E.backtracking_case(st[lab], g, N, DT, s, oracle) for lab, g, s in BACKTRACK]
    return E.stack([c for _, _, _, c in cases] + bt), len(cases)


def _assert_case_values(axis, lab, case):
    """A solve case starts where its label says."""
    x0, xr, sw, md, xt, ut = case
    if lab.startswith("pitch"):
        assert x0[10] == float(lab.split()[1]), lab
    if axis == "yaw":
        assert abs(x0[9]) >= np.pi - 1e-12 and xr[0, 9] == x0[9], lab
    if axis == "position":
        assert np.abs(x0[6:8]).max() == 1e3, lab
    if axis == "momentum":
        assert np.abs(x0[0:6]).max() == E.ENVELOPE["momentum"], lab
    if axis == "joints" and lab.startswith("all"):
        assert np.array_equal(x0[12:], E.LOWER if "lower" in lab else E.UPPER), lab
    if axis == "joint_velocity":
        assert np.abs(ut[:, 12:]).max() == E.ENVELOPE["joint_velocity"], lab
    if lab.startswith("3mg on"):
        assert np.abs(ut[:, :12]).max() == 3 * E.WEIGHT, lab


def test_sqp_iterations_on_the_envelope_vs_oracle(ctx, cases, oracle):
    """Instances whose rounding floor exceeds the suite's bounds (hbar far from what the joints absorb, with a poor warm start, and one mixed
    state) are held to FLOOR times it: the oracle itself moves by 1e-6 to 1e-4 there when x0 and the warm start move by one ulp."""
    states = E._case_states()
    (x0, xr, sw, md, xt, ut), n_axis = _batch_with_backtracking(cases, oracle)
    B = x0.shape[0]
    xc, uc = ctx.mpc_cold_start(x0[:n_axis], md[:n_axis])
    for i, (axis, lab, _, c) in enumerate(cases):
        _assert_case_values(axis, lab, c)
        if states[i][3] is None:
            assert np.array_equal(xc[i], c[4]) and np.array_equal(uc[i], c[5]), lab
    dev1 = ctx.mpc_solve(x0, xr, sw, md, xt, ut)
    dev2 = ctx.mpc_solve(x0, xr, sw, md, dev1[0], dev1[1])
    orc = _oracle_iterations(oracle, x0, xr, sw, md, xt, ut)
    labels = [(a, lab, g) for a, lab, g, _ in cases] + [("backtracking", lab, g) for lab, g, _ in BACKTRACK]
    worst = {}
    widened = []
    for i in range(B):
        case = (x0[i], xr[i], sw[i], md[i], xt[i], ut[i])
        for it, (dev, o) in enumerate(((dev1, orc[0]), (dev2, orc[1]))):
            e = np.array([E.rel(dev[0][i], o[0][i]), E.rel(dev[1][i], o[1][i])])
            fl = (0.0, 0.0)
            if e[0] >= 1e-7 or e[1] >= 1e-6:
                fl = _floors(oracle, N, DT, case, it + 1)
                widened.append((labels[i][1], it, e.round(9).tolist(), np.round(fl, 9).tolist()))
            _check_iteration(dev, o, i, (it, labels[i]), fl)
            worst[labels[i][0]] = np.maximum(worst.get(labels[i][0], 0.0), e)
    assert all(orc[0][2][i]["alpha"] < 1.0 for i in range(n_axis, B))          # every poor warm start back-tracks
    assert {g for _, _, g in labels} == set(E.GAITS)
    for a, (ex, eu) in worst.items():
        print("%-15s max relative deviation x %.1e u %.1e" % (a, ex, eu))
    print("held to the rounding floor (label, iteration, deviation, floor):", widened)
    assert len(widened) <= 4


def test_sqp_iterations_on_an_event_grid_vs_oracle(oracle):
    """The solve cases on event-node grids: each instance's grid has a node on every mode switch of its reference (scenarios.event_time_grid)."""
    cap, T = 28, 0.4
    ctx = hb.Context(horizon_N=cap, dt=DT, max_batch=64, device=0, time_horizon=T, event_nodes=True)
    try:
        states = E._case_states()
        B = len(states)
        tk = np.zeros((B, cap + 1)); nn = np.zeros(B, dtype=np.int32)
        x0 = np.stack([s[2] for s in states])
        xr = np.zeros((B, cap + 1, 22)); sw = np.zeros((B, cap + 1, 24)); md = np.zeros((B, cap + 1), dtype=np.int32)
        for i in range(B):
            g = E.GAITS[i % 4]
            comp = sc.make_reference(x0[i], (0.3, 0.0, 0.0, 0.2), g, N, DT)[3]
            t = sc.event_time_grid(0.0, T, DT, comp["events"], cap)
            n = len(t) - 1
            nn[i] = n
            tk[i, :n + 1] = t; tk[i, n + 1:] = t[-1] + DT * np.arange(1, cap - n + 1)
            xr[i], sw[i], md[i] = sc.sample_reference(comp, tk[i])
        assert (nn > N).any() and len(set(nn.tolist())) > 1
        xt, ut = ctx.mpc_cold_start(x0, md)
        for i in range(B):
            if states[i][3] is not None:
                ut[i, :] = states[i][3]
        a1 = ctx.mpc_solve_grid(x0, tk, nn, xr, sw, md, xt, ut)
        a2 = ctx.mpc_solve_grid(x0, tk, nn, xr, sw, md, a1[0], a1[1])
        worst = np.zeros(2)
        widened = []
        for i in range(B):
            n = nn[i]
            dts = np.diff(tk[i, :n + 1])
            xo, uo = xt[i, :n + 1], ut[i, :n]
            for it, dev in enumerate((a1, a2)):
                xo, uo, io = oracle.mpc_iteration(n, dts, x0[i], xr[i, :n + 1], sw[i, :n + 1], md[i, :n + 1], xo, uo)
                e = np.array([E.rel(dev[0][i, :n + 1], xo), E.rel(dev[1][i, :n], uo)])
                fl = (0.0, 0.0)
                if e[0] >= 1e-7 or e[1] >= 1e-6:
                    case = (x0[i], xr[i, :n + 1], sw[i, :n + 1], md[i, :n + 1], xt[i, :n + 1], ut[i, :n])
                    fl = _floors(oracle, n, dts, case, it + 1)
                    widened.append((states[i][1], it, e.round(9).tolist(), np.round(fl, 9).tolist()))
                _check_iteration((dev[0][i:i + 1, :n + 1], dev[1][i:i + 1, :n], dev[2][i:i + 1]), ([xo], [uo], [io]), 0, (it, states[i][1]), fl)
                worst = np.maximum(worst, e)
        print("event grid: max relative deviation x %.1e u %.1e" % tuple(worst))
        print("held to the rounding floor (label, iteration, deviation, floor):", widened)
        assert len(widened) <= 4
    finally:
        ctx.close()


def test_yaw_turns_and_shifts_on_the_device(ctx, cases):
    """The exact transforms of the host test, on the device alone: the transformed solve, transformed back, within the host test's bounds."""
    batch = E.stack([c for _, _, _, c in cases])
    ref = ctx.mpc_solve(*batch)
    worst = np.zeros(4)
    for k in (1, 10, 159, 1000, -1000):
        t = ctx.mpc_solve(*E.yaw_turn(batch, k))
        xb = E.yaw_turn_back(t[0], k)
        for i, (_, lab, _, _) in enumerate(cases):
            assert t[2]["status"][i] == 0 and t[2]["alpha"][i] == ref[2]["alpha"][i] and t[2]["n_trials"][i] == ref[2]["n_trials"][i], (lab, k)
            ex, eu = E.rel(xb[i], ref[0][i]), E.rel(t[1][i], ref[1][i])
            assert ex < INV_X and eu < INV_U, (lab, k, ex, eu)
            worst[:2] = np.maximum(worst[:2], (ex, eu))
    for d in ((1e3, 1e3), (-1e3, 250.0), (0.37, -5e2)):
        t = ctx.mpc_solve(*E.shift(batch, d))
        xb = E.shift_back(t[0], d)
        for i, (_, lab, _, _) in enumerate(cases):
            assert t[2]["status"][i] == 0 and t[2]["alpha"][i] == ref[2]["alpha"][i] and t[2]["n_trials"][i] == ref[2]["n_trials"][i], (lab, d)
            ex, eu = E.rel(xb[i], ref[0][i]), E.rel(t[1][i], ref[1][i])
            assert ex < INV_X and eu < INV_U, (lab, d, ex, eu)
            worst[2:] = np.maximum(worst[2:], (ex, eu))
    print("device invariance: yaw turns x %.1e u %.1e, shifts x %.1e u %.1e" % tuple(worst))


def _nominal(B, seed):
    x0, xr, sw, md = sc.make_batch(B, N, DT, gaits=[E.GAITS[i % 4] for i in range(B)], seed=seed)
    from oracle import hbo
    xt = np.zeros((B, N + 1, 22)); ut = np.zeros((B, N, 22))
    for i in range(B):
        xt[i], ut[i] = hbo.mpc_cold_start(N, DT, x0[i], md[i])
    return x0, xr, sw, md, xt, ut


def test_envelope_instances_leave_nominal_ones_bitwise_unchanged(ctx, cases):
    nom = _nominal(8, 820)
    env = E.stack([c for _, _, _, c in cases])
    mixed = tuple(np.concatenate([a[:4], b, a[4:]]) for a, b in zip(nom, env))
    full = ctx.mpc_solve(*mixed)
    n_env = env[0].shape[0]
    for j in range(8):
        jj = j if j < 4 else j + n_env
        alone = ctx.mpc_solve(*(a[j:j + 1] for a in nom))
        assert np.array_equal(alone[0][0], full[0][jj]) and np.array_equal(alone[1][0], full[1][jj]), j
        assert alone[2][0].tobytes() == full[2][jj].tobytes(), j


def test_near_vertical_attitude(ctx, oracle):
    """Status 0 with finite output matching the oracle, or a non-zero status with the iterate kept (the line search's non-finite test);
    nominal neighbours bitwise unchanged."""
    nom = _nominal(4, 830)
    vert = [E.solve_case(E._x(pitch=p), E.GAITS[i % 4], N, DT, oracle=oracle) for i, p in enumerate(NEAR_VERTICAL)]
    vb = E.stack(vert)
    batch = tuple(np.concatenate([a[:2], b, a[2:]]) for a, b in zip(nom, vb))
    dev = ctx.mpc_solve(*batch)
    alone = ctx.mpc_solve(*nom)
    for j, jj in ((0, 0), (1, 1), (2, 2 + len(vert)), (3, 3 + len(vert))):
        assert np.array_equal(alone[0][j], dev[0][jj]) and np.array_equal(alone[1][j], dev[1][jj]) and alone[2][j].tobytes() == dev[2][jj].tobytes()
    for i, p in enumerate(NEAR_VERTICAL):
        k = 2 + i
        c = vert[i]
        xo, uo, io = oracle.mpc_iteration(N, DT, *c)
        st = dev[2]["status"][k]
        print("pitch %.7f: device status %d alpha %g trials %d; oracle status %d alpha %g trials %d; x %.1e u %.1e"
              % (p, st, dev[2]["alpha"][k], dev[2]["n_trials"][k], io["status"], io["alpha"], io["n_trials"],
                 E.rel(dev[0][k], xo), E.rel(dev[1][k], uo)))
        if st == 0:
            assert np.isfinite(dev[0][k]).all() and np.isfinite(dev[1][k]).all(), p
            fl = _floors(oracle, N, DT, c, 1)
            print("  rounding floor x %.1e u %.1e" % tuple(fl))
            _check_iteration(dev, ([None] * k + [xo], [None] * k + [uo], [None] * k + [io]), k, p, fl)
        else:
            assert np.array_equal(dev[0][k], c[4]) and np.array_equal(dev[1][k], c[5]), p


class WbcStatusMismatch(Exception):
    """The device's weighted WBC returns a non-zero status on a problem the oracle's WBC solves."""


def _control_step_states(momentum, joints_in_range, seed=840, B=24):
    rng = np.random.default_rng(seed)
    x0 = np.tile(E.X0, (B, 1))
    x0[:, 9] = rng.uniform(-1e3, 1e3, B); x0[:, 10:12] = rng.uniform(-0.5, 0.5, (B, 2))
    x0[:, 6:8] = rng.uniform(-1e3, 1e3, (B, 2))
    x0[:, 12:] = rng.uniform(E.LOWER, E.UPPER, (B, 10)) if joints_in_range else E.X0[12:] + rng.uniform(-0.05, 0.05, (B, 10))
    x0[:, 0:3] = rng.uniform(-momentum[0], momentum[0], (B, 3)); x0[:, 3:6] = rng.uniform(-momentum[1], momentum[1], (B, 3))
    if joints_in_range:
        x0[0, 12:] = E.LOWER; x0[1, 12:] = E.UPPER
    x0[2, 10] = 0.5; x0[3, 11] = -0.5
    return x0


def _control_step_torques_vs_oracle(ctx, oracle, momentum, joints_in_range):
    x0 = _control_step_states(momentum, joints_in_range)
    B = x0.shape[0]
    c = [E.solve_case(x0[i], E.GAITS[i % 4], N, DT, oracle=oracle) for i in range(B)]
    x0, xr, sw, md, xt, ut = E.stack(c)
    rbd = sc.consistent_rbd(x0)
    t_rel = 0.002
    xt1, ut1, info, sol, tau, st = ctx.control_step(t_rel, x0, xr, sw, md, rbd, xt, ut)
    worst = 0.0
    mismatched = []
    for i in range(B):
        xo, uo, io = oracle.mpc_iteration(N, DT, *c[i])
        assert info["status"][i] == 0 and io["alpha"] == info["alpha"][i], i
        al = t_rel / DT
        xd = (1 - al) * xo[0] + al * xo[1]; ud = (1 - al) * uo[0] + al * uo[1]
        so, sto = oracle.wbc_solve(xd, ud, rbd[i], int(md[i][0]), False, 1e-8)
        assert sto == 0, i
        if st[i] != 0:
            mismatched.append((i, int(st[i])))
            continue
        err = np.abs(so[28:] - tau[i]).max() / max(1.0, np.abs(so[28:]).max())
        assert err < 1e-4, (i, err)
        worst = max(worst, err)
    print("control_step torques, hbar to %s: max relative deviation %.1e; device WBC status mismatches %s" % (momentum, worst, mismatched))
    if mismatched:
        raise WbcStatusMismatch(mismatched)


def test_control_step_torques_on_the_upright_envelope_vs_oracle(ctx, oracle):
    """The north-star claim beyond the nominal box: attitude to 0.5 rad, yaw to +-1e3 rad, positions to 1e3 m, joints anywhere in their
    hbar within random_initial_states' +-0.1 and joints within its 0.05 of the default pose."""
    _control_step_torques_vs_oracle(ctx, oracle, (0.1, 0.1), False)


@pytest.mark.xfail(strict=True, raises=WbcStatusMismatch,
                   reason="with hbar beyond +-0.1 and the measured base velocity at rest (9 of 24 instances at +-0.5), or with joints drawn "
                          "anywhere in their range (1 of 24 at hbar +-0.1), the device's weighted WBC returns status 2 or 3 on instances the "
                          "oracle's WBC solves; attitude to 0.5 rad, yaw to 1e3 rad and positions to 1e3 m each leave every status 0. The "
                          "WBC's own envelope is another change")
def test_control_step_where_the_device_wbc_disagrees(ctx, oracle):
    _control_step_torques_vs_oracle(ctx, oracle, (0.5, 0.5), True)


VISITED_TICKS, VISITED_B = 750, 16


def _visited(name, setup, cmd_vel, estimated):
    """Extremes of x_des / u_des recorded on every tick of a 1.5 s episode of VISITED_B robots, up to each robot's failure tick."""
    import torch
    import episode_ref as R
    c = R.context(max_batch=VISITED_B)
    try:
        B = VISITED_B
        rbd0 = R.start_states(c, B, seed=7)
        setup(c, rbd0)
        bufs = hb.make_channels(B, VISITED_TICKS, names=["x_des", "u_des"])
        c.set_channels(bufs)
        cmds = hb.make_rollout_commands("trot", 0.1, [0.0], np.tile(np.asarray(cmd_vel, float), (B, 1, 1)))
        d = torch.from_numpy(np.ascontiguousarray(rbd0)).cuda()
        prm = R.params(1)
        out = (c.rollout_estimated(d, cmds, VISITED_TICKS, params=prm, est_params=R.est_params(3), log_every=1) if estimated
               else c.rollout(d, cmds, VISITED_TICKS, params=prm, log_every=1))
        c.set_channels(None)
        ft = out[3]["fail_tick"]
        xd, ud = bufs["x_des"].cpu().numpy(), bufs["u_des"].cpu().numpy()
        n = [VISITED_TICKS if t < 0 else int(t) for t in ft]
        return E.bounds_of(np.concatenate([xd[i, :n[i]] for i in range(B)]), np.concatenate([ud[i, :n[i]] for i in range(B)])), int((ft >= 0).sum())
    finally:
        c.close()


def test_axes_contain_the_visited_envelope():
    """x_des / u_des through a pushed episode (40 and 60 N for 0.1 s), a 15 degree incline and a turning estimated episode lie inside the
    axes. Measured on an H100: pitch 0.28, roll 0.17, linear hbar 0.73, angular hbar 0.07, joint velocity 36 rad/s, normal force 252 N
    (pushed); pitch 0.23 and joint velocity 12.5 rad/s (slope); joint velocity 10.1 rad/s (turning, estimated). The yaw and the position of
    1.5 s episodes stay below 1 rad and 1 m: their axes' reach comes from the unwrapped yaw and the distances of long episodes, not from
    this measurement."""
    B = VISITED_B

    def pushes(c, r):
        f = np.zeros((B, 1, 3)); f[:, 0, 1] = np.where(np.arange(B) % 2, 60.0, -40.0)
        c.set_pushes(hb.make_push_schedules(B, 0.6, 0.1, f))

    def slope(c, r):
        import episode_ref as R
        hh = R.GROUND + np.tan(np.radians(15.0)) * 0.1 * np.arange(64)[None, None, :] * np.ones((B, 64, 1))
        c.set_terrains(hb.make_terrains(B, hh, 0.1, np.c_[r[:, 3] + 0.1, r[:, 4] - 3.2]))

    runs = (("pushed", pushes, (0.3, 0, 0, 0), False), ("slope", slope, (0.3, 0, 0, 0), False),
            ("turning", lambda c, r: None, (0.4, 0, 0, 0.8), True))
    for name, setup, cmd, est in runs:
        b, failed = _visited(name, setup, cmd, est)
        print(name, "failed %d of %d" % (failed, B), {k: np.round(np.asarray(v), 3).tolist() for k, v in b.items() if k != "joints"})
        assert failed < B, name
        assert max(b["pitch"], b["roll"]) <= E.ENVELOPE["attitude"] and b["yaw"] <= E.ENVELOPE["yaw"], name
        assert b["position"] <= E.ENVELOPE["position"] and max(b["linear"], b["angular"]) <= E.ENVELOPE["momentum"], name
        lo, hi = b["joints"]
        assert (lo >= E.LOWER - 0.3).all() and (hi <= E.UPPER + 0.3).all(), name
        assert b["joint_velocity"] <= E.ENVELOPE["joint_velocity"] and b["force"] <= E.ENVELOPE["force"], name
