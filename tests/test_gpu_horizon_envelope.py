"""The MPC solve across its whole horizon envelope (1 <= horizon_N <= HB_MAX_HORIZON) against the float64 CPU oracle and the numpy
restatements of the steps around it. Every kernel of the SQP iteration maps nodes to threads in a way that depends on the horizon: node
pairs in the linearisation (odd N leaves a half-idle warp), a buffer and mbarrier phase picked by the parity of N - 1 in the Riccati sweep,
line-search trials evaluated one lane per node in rounds of 32, the warm shift staging (2N + 1) x 22 doubles in shared memory. So the
horizons here sit at the edges: 1, 2, 3, the 32-lane round boundaries, the 48 KB shared-memory default of the warm shift (N = 139 / 140),
and the cap. Tolerances are the suite's: alpha and trial counts equal, merit0 within 1e-8, x within 1e-7 and u within 1e-6 relative to
max(1, |ref|)."""
import os

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from hunter_bipedal_control_b200.api import HB_MAX_HORIZON
from oracle import refs as R

pytestmark = pytest.mark.gpu

ENVELOPE = (1, 2, 3, 31, 32, 33, 63, 64, 65, 139, 140, 200, HB_MAX_HORIZON)
GAITS = ("stance", "trot", "standing_trot", "flying_trot")
# Seeds of the back-tracking recipe (_backtracking_case) whose first oracle iteration takes alpha < 1 at that horizon, chosen with the oracle
# alone (the test asserts it again); with one horizon N = 1 has none.
BACKTRACK_SEEDS = {2: (4, 1), 3: (1, 2), 31: (12, 4), 32: (4, 7), 33: (4, 7), 63: (4, 5), 64: (5, 21), 65: (5, 15), 139: (17, 9),
                   140: (17, 9), 200: (14, 9), HB_MAX_HORIZON: (21, 6)}
EVENT_COUNTS = (1, 2, 31, 32, 33, 64, 65)          # active intervals of one batch on an odd-capacity event grid
SHIFTS = np.array([1.0, 0.3, 2.0, 1.3])            # warm-start shifts in units of dt: on the grid, off it
THREADS = min(8, os.cpu_count() or 1)


def _dt(N):
    return 0.005 if N == HB_MAX_HORIZON else 0.01    # 2.56 s at the cap


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


@pytest.fixture(scope="module")
def contexts():
    """Context of (horizon, max_batch, e2e_chunks), made once for the module; contexts of many horizons live in one process."""
    made = {}

    def get(N, max_batch=16, e2e_chunks=0):
        key = (N, max_batch, e2e_chunks)
        if key not in made:
            made[key] = hb.Context(horizon_N=N, dt=_dt(N), max_batch=max_batch, device=0, e2e_chunks=e2e_chunks)
        return made[key]
    yield get
    for ctx in made.values():
        ctx.close()


def _backtracking_case(N, dt, seed, oracle):
    """A poor warm start (test_mpc_backtracking_line_search_vs_oracle's recipe, amplitude 1.0): three oracle iterations, then the joint
    trajectory pushed far off. Returns (x0, x_ref, swing, mode, xt, ut) of one instance."""
    x0, xr, sw, md = sc.make_batch(1, N, dt, gait=["trot", "flying_trot", "standing_trot"][seed % 3], seed=1000 + seed)
    xt, ut = oracle.mpc_cold_start(N, dt, x0[0], md[0])
    for _ in range(3):
        xt, ut, _ = oracle.mpc_iteration(N, dt, x0[0], xr[0], sw[0], md[0], xt, ut)
    xt[1:, 12:] += np.random.default_rng(seed).uniform(-1.0, 1.0, (N, 10))
    return x0[0], xr[0], sw[0], md[0], xt, ut


def _assert_iteration(dev, orc, i, what):
    """Instance i of a device solve (xt, ut, info) against the oracle's (xt, ut, infos); returns the relative x and u deviations."""
    io = orc[2][i]
    assert dev[2]["status"][i] == 0, what
    assert io["alpha"] == dev[2]["alpha"][i] and io["n_trials"] == dev[2]["n_trials"][i], (what, io, dev[2][i])
    assert abs(io["merit0"] - dev[2]["merit0"][i]) < 1e-8 * max(1.0, abs(io["merit0"])), what
    ex, eu = _rel(dev[0][i], orc[0][i]), _rel(dev[1][i], orc[1][i])
    assert ex < 1e-7 and eu < 1e-6, (what, ex, eu)
    return ex, eu


@pytest.mark.parametrize("N", ENVELOPE)
def test_sqp_iterations_across_the_horizon_envelope_vs_oracle(N, contexts, oracle):
    """Two SQP iterations from the cold start on a mixed-gait batch, plus instances whose first step back-tracks, against the oracle."""
    dt, ctx = _dt(N), contexts(N)
    x0, xr, sw, md = sc.make_batch(len(GAITS), N, dt, gaits=GAITS, seed=300 + N)
    xt, ut = ctx.mpc_cold_start(x0, md)
    for i in range(len(GAITS)):
        xc, uc = oracle.mpc_cold_start(N, dt, x0[i], md[i])
        assert np.array_equal(xt[i], xc) and np.array_equal(ut[i], uc), i
    cases = [_backtracking_case(N, dt, s, oracle) for s in BACKTRACK_SEEDS.get(N, ())]
    if cases:
        x0, xr, sw, md, xt, ut = (np.concatenate([a, np.stack(b)]) for a, b in zip((x0, xr, sw, md, xt, ut), zip(*cases)))
    B = x0.shape[0]
    dev1 = ctx.mpc_solve(x0, xr, sw, md, xt, ut)
    dev2 = ctx.mpc_solve(x0, xr, sw, md, dev1[0], dev1[1])
    orc1 = oracle.mpc_iteration_batch(N, dt, x0, xr, sw, md, xt, ut, threads=THREADS)
    orc2 = oracle.mpc_iteration_batch(N, dt, x0, xr, sw, md, orc1[0], orc1[1], threads=THREADS)
    dev_x = dev_u = 0.0
    for it, (dev, orc) in enumerate(((dev1, orc1), (dev2, orc2))):
        for i in range(B):
            ex, eu = _assert_iteration(dev, orc, i, (N, it, i))
            dev_x, dev_u = max(dev_x, ex), max(dev_u, eu)
    backtracking = [i for i in range(B) if orc1[2][i]["alpha"] < 1.0]
    assert set(range(len(GAITS), B)) <= set(backtracking)          # the perturbed instances do take the trial rounds after the first
    assert backtracking or N == 1
    print("N=%d: max relative deviation from the oracle x %.2e u %.2e; back-tracking instances %s (alpha %s)"
          % (N, dev_x, dev_u, backtracking, [orc1[2][i]["alpha"] for i in backtracking]))


@pytest.fixture(scope="module")
def event_ctx():
    ctx = hb.Context(horizon_N=65, dt=0.015, max_batch=len(EVENT_COUNTS), device=0, time_horizon=0.8, event_nodes=True)
    yield ctx
    ctx.close()


def test_sqp_iterations_on_event_grids_of_every_active_count_vs_oracle(event_ctx, oracle):
    """One batch on an odd-capacity (65) event grid whose instances have 1, 2, 31, 32, 33, 64 and 65 active intervals, on hand-built
    non-uniform node times: two iterations against the oracle on each instance's own first n + 1 nodes; entries beyond n stay as they were."""
    cap, B = event_ctx.N, len(EVENT_COUNTS)
    rng = np.random.default_rng(17)
    nn = np.array(EVENT_COUNTS, dtype=np.int32)
    tk = np.zeros((B, cap + 1))
    for i in range(B):
        dts = rng.uniform(0.004, 0.016, cap)
        dts[rng.integers(0, cap, 3)] = 0.001                      # a few short intervals, as around an event node
        tk[i] = 0.003 * i + np.concatenate([[0.0], np.cumsum(dts)])
    x0 = sc.random_initial_states(B, seed=61)
    xr = np.zeros((B, cap + 1, 22)); sw = np.zeros((B, cap + 1, 24)); md = np.zeros((B, cap + 1), dtype=np.int32)
    for i in range(B):
        c = sc.make_reference(x0[i], (0.3, 0.0, 0.0, 0.1), GAITS[i % 4], cap, 0.016, phase=float(rng.uniform(0.0, 0.2)))[3]
        xr[i], sw[i], md[i] = sc.sample_reference(c, tk[i])
    xt, ut = event_ctx.mpc_cold_start(x0, md)
    for i, n in enumerate(EVENT_COUNTS):                          # distinct values beyond the active nodes, to see that they are kept
        xt[i, n + 1:] = rng.uniform(-1.0, 1.0, xt[i, n + 1:].shape)
        ut[i, n:] = rng.uniform(-1.0, 1.0, ut[i, n:].shape)
    a1 = event_ctx.mpc_solve_grid(x0, tk, nn, xr, sw, md, xt, ut)
    a2 = event_ctx.mpc_solve_grid(x0, tk, nn, xr, sw, md, a1[0], a1[1])
    for i, n in enumerate(EVENT_COUNTS):
        dts = np.diff(tk[i, :n + 1])
        xo, uo = oracle.mpc_cold_start(n, dts, x0[i], md[i, :n + 1])
        assert np.array_equal(xo, xt[i, :n + 1]) and np.array_equal(uo, ut[i, :n])
        for it, dev in enumerate((a1, a2)):
            xo, uo, io = oracle.mpc_iteration(n, dts, x0[i], xr[i, :n + 1], sw[i, :n + 1], md[i, :n + 1], xo, uo)
            _assert_iteration((dev[0][i:i + 1, :n + 1], dev[1][i:i + 1, :n], dev[2][i:i + 1]), ([xo], [uo], [io]), 0, (n, it))
            assert np.array_equal(dev[0][i, n + 1:], xt[i, n + 1:]) and np.array_equal(dev[1][i, n:], ut[i, n:]), (n, it)


def _references(N, dt, B, seed, gaits=("trot", "standing_trot", "stance", "trot")):
    """(x0, packed compact references, rbd) of B instances for resident cycles at horizon N: the events and swing segments a solve at
    t <= 0.1 s can see (the packed reference holds at most HB_MAX_EVENTS events and HB_MAX_SEGMENTS segments per axis)."""
    x0 = sc.random_initial_states(B, seed=seed)
    reach = N * dt + 0.1
    compacts = []
    for i in range(min(B, 8)):
        c = sc.make_reference(x0[i], (0.3, 0.0, 0.0, 0.1), gaits[i % len(gaits)], N, dt, phase=0.03 * i)[3]
        keep = int(np.searchsorted(c["events"], reach, side="right"))
        c["events"], c["modes"] = c["events"][:keep], c["modes"][:keep + 1]
        compacts.append(c)
    return x0, sc.pack_references([compacts[i % len(compacts)] for i in range(B)], reach), sc.consistent_rbd(x0)


def _check_warm_cycle(ctx, N, dt, B, seed, oracle):
    """A cold resident cycle at t = 0, then a warm one at shifts on the dt grid and off it: the resident trajectories equal the restated warm
    start (oracle/refs.warm_start_shift) followed by the ordinary control step on it, and the oracle's iteration from that warm start.
    Returns (t1, resident x, resident u, mode, rbd) after the warm cycle."""
    x0, refs, rbd = _references(N, dt, B, seed)
    info0, _, _, _ = ctx.resident_cycle(True, 0.002, np.zeros(B), x0, refs, rbd)
    assert (info0["status"] == 0).all()
    _, xprev, uprev = ctx.resident_read(B)
    t1 = SHIFTS[np.arange(B) % len(SHIFTS)] * dt
    x1 = xprev[:, 0] + 0.3 * (xprev[:, 1] - xprev[:, 0]) + 1e-3
    rbd1 = sc.consistent_rbd(x1)
    info, sol, tau, st = ctx.resident_cycle(False, 0.002, t1, x1, refs, rbd1)
    tr, xnew, unew = ctx.resident_read(B)
    assert np.array_equal(tr, t1)
    xr, sw, md = ctx.reference_expand(t1, refs)
    xw = np.zeros_like(xprev); uw = np.zeros_like(uprev)
    for i in range(B):
        xw[i], uw[i] = R.warm_start_shift(0.0, t1[i], dt, xprev[i], uprev[i], x1[i], md[i], sc.TOTAL_MASS)
    xt2, ut2, info2, sol2, tau2, st2 = ctx.control_step(0.002, x1, xr, sw, md, rbd1, xw, uw)
    assert np.array_equal(info["alpha"], info2["alpha"]) and (info["status"] == 0).all()
    assert np.abs(xnew - xt2).max() < 1e-9 and np.abs(unew - ut2).max() < 1e-7 * max(1.0, np.abs(ut2).max())
    assert np.abs(tau - tau2).max() < 1e-6 * np.abs(tau2).max() and np.array_equal(st, st2)
    orc = oracle.mpc_iteration_batch(N, dt, x1, xr, sw, md, xw, uw, threads=THREADS)
    dev = np.array([_assert_iteration((xnew, unew, info), orc, i, (N, "warm", i)) for i in range(B)])
    print("N=%d warm cycle: max relative deviation from the oracle x %.2e u %.2e" % (N, dev[:, 0].max(), dev[:, 1].max()))
    return t1, xnew, unew, md, rbd1


@pytest.mark.parametrize("N", (1, 33, 140, HB_MAX_HORIZON))
def test_warm_cycle_and_policy_at_long_horizons(N, contexts, oracle):
    """The warm shift of the resident solution at horizons below and above the 48 KB shared-memory default, then the policy evaluated at
    absolute times after the solve: at the solve time, on a node, between nodes, at the end of the horizon and beyond it (clamped, the
    last input repeated), against the linear interpolation of the resident trajectories."""
    dt, ctx = _dt(N), contexts(N)
    B = 8
    t1, xres, ures, md, rbd = _check_warm_cycle(ctx, N, dt, B, 70 + N, oracle)
    node = max(1, N // 2)
    for off in (0.0, node * dt, (node - 0.63) * dt, N * dt, N * dt + 0.05):
        t_now = t1 + off
        xd, ud, mode, _, _, _ = ctx.resident_wbc(t_now, rbd)
        s = np.clip((t_now - t1) / dt, 0.0, float(N))
        k = np.minimum(np.floor(s).astype(int), N - 1)
        al = s - k
        for i in range(B):
            xe = (1 - al[i]) * xres[i, k[i]] + al[i] * xres[i, k[i] + 1]
            ue = (1 - al[i]) * ures[i, k[i]] + al[i] * ures[i, min(k[i] + 1, N - 1)]
            assert _rel(xd[i], xe) < 1e-13 and _rel(ud[i], ue) < 1e-13, (off, i)
            # on a node where the mode changes the interval ending there holds (modeAtTime's earlier mode at a switch)
            ki = k[i] - 1 if al[i] == 0.0 and k[i] > 0 and md[i, k[i]] != md[i, k[i] - 1] else k[i]
            assert mode[i] == md[i, ki], (off, i)
    # beyond the horizon: the last state node and the last input sample, exactly
    assert np.array_equal(xd, xres[:, N]) and np.array_equal(ud, ures[:, N - 1])


def test_shorter_context_keeps_long_horizon_warm_cycles_launchable(oracle):
    """The shared-memory opt-in of the warm shift belongs to the kernel, for the whole process: creating a context with a shorter horizon
    after one that needs more than the 48 KB default must not make the longer one's warm cycles and episodes unlaunchable."""
    import episode_ref as E
    big = hb.Context(horizon_N=200, dt=0.01, max_batch=4, device=0)
    small = hb.Context(horizon_N=8, dt=0.01, max_batch=4, device=0)
    try:
        _check_warm_cycle(big, 200, 0.01, 4, 90, oracle)
        rbd0 = E.start_states(big, 4, seed=5)
        gaits = ["stance", "trot", "standing_trot", "trot"]
        prm = E.params()
        # 15 ticks: MPC cycles at ticks 0, 5 and 10, the last two warm
        E.assert_episode_equal(E.device(big, rbd0, gaits, E.cmd_vels(4), 15, prm, 5), E.stepwise(big, rbd0, gaits, E.cmd_vels(4), 15, prm, 5))
        _check_warm_cycle(small, 8, 0.01, 4, 91, oracle)
    finally:
        big.close()
        small.close()


@pytest.mark.parametrize("N", (1, 33, 140))
def test_batch_shape_leaves_every_instance_bitwise_unchanged(N, contexts):
    """An instance solved alone equals its copy in a batch of 37 (odd: with N = 1 and 33 the last linearisation block has an idle warp);
    host-pointer resident cycles split into three chunks (odd chunk offsets into the per-node scratch) equal one chunk, bit for bit."""
    dt = _dt(N)
    one, three = contexts(N, 197, 1), contexts(N, 197, 3)
    B = 37
    x0, xr, sw, md = sc.make_batch(B, N, dt, gaits=[GAITS[i % 4] for i in range(B)], seed=500 + N)
    xt, ut = one.mpc_cold_start(x0, md)
    full = one.mpc_solve(x0, xr, sw, md, xt, ut)
    for j in (0, B // 2, B - 1):
        alone = one.mpc_solve(*(a[j:j + 1] for a in (x0, xr, sw, md, xt, ut)))
        assert np.array_equal(alone[0][0], full[0][j]) and np.array_equal(alone[1][0], full[1][j]), j
        assert alone[2][0].tobytes() == full[2][j].tobytes(), j
    # three chunks of 65 / 66 / 66 instances (a chunk needs at least 64)
    B = 197
    x0, refs, rbd = _references(N, dt, B, 600 + N)
    t1 = SHIFTS[np.arange(B) % len(SHIFTS)] * dt
    runs = []
    for ctx in (one, three):
        c0 = ctx.launch_count
        cold = ctx.resident_cycle(True, 0.002, np.zeros(B), x0, refs, rbd)
        warm = ctx.resident_cycle(False, 0.002, t1, x0 + 1e-3, refs, rbd)
        runs.append((cold, warm, ctx.resident_read(B), ctx.launch_count - c0))
    for a, b in zip(runs[0][:3], runs[1][:3]):
        for u, v in zip(a, b):
            assert u.tobytes() == v.tobytes()
    assert (runs[0][1][0]["status"] == 0).all()
    assert runs[1][3] > runs[0][3]                                 # the three-chunk context did split the batch


def test_horizon_bounds():
    for N in (0, HB_MAX_HORIZON + 1):
        with pytest.raises(hb.HunterB200Error, match=r"invalid argument \(-1\)"):
            hb.Context(horizon_N=N, max_batch=1, device=0)
    for N in (1, HB_MAX_HORIZON):
        hb.Context(horizon_N=N, dt=_dt(N), max_batch=1, device=0).close()
