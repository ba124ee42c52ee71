"""The solve's time axis on the device at its edges, against the OCS2-structured restatement in tests/time_axis_ref.py: the event-node
grid (time_grid_kernel, row S1), the references on it (reference_expand_kernel, rows M10 / M12), the policy between solves
(policy_eval_kernel, row S8; the MRT buffer of policy_adopt_kernel) and the warm start between two grids (warm_shift_kernel). The
references are hand-built hb_reference structs, so switches, target samples and spline knots sit exactly where the edges are: on a
grid step and 1e-12 / 1e-9 / 2e-9 either side of one, on t0 and tf, coincident or closer than dt_min, beyond the capacities. Times
start at 1.0 so that t0 + (t - t0) is t exactly for every node time t the tests query (Sterbenz)."""
import ctypes as C

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from hunter_bipedal_control_b200.api import HB_MAX_EVENTS, HB_MAX_HORIZON, HB_MAX_SEGMENTS, HbReference, _check, _ptr
from oracle import refs as R
import time_axis_ref as TA

pytestmark = pytest.mark.gpu
DT, T = 0.015, 0.8
UDT = 0.015625                   # uniform grids: a dyadic step, so t0 + k dt is exact on both sides
LIFTOFF_VEL = 0.05               # swing_trajectory_config.liftOffVelocity (task.info:23)


@pytest.fixture(scope="module")
def contexts():
    made = {}

    def get(N, dt, T_=0.0, event_nodes=True, max_batch=16):
        key = (N, dt, T_, event_nodes, max_batch)
        if key not in made:
            made[key] = hb.Context(horizon_N=N, dt=dt, max_batch=max_batch, device=0, time_horizon=T_, event_nodes=event_nodes)
        return made[key]
    yield get
    for ctx in made.values():
        ctx.close()


def _steps(t0, dt, n):
    out, t = [], t0
    for _ in range(n):
        t = t + dt
        out.append(t)
    return out


def _reference(rng, t0, tf, events, nodes):
    """A hand-built reference: modes alternating at every event; target samples on nodes, on a switch and outside [t0, tf]; per foot z
    segments that follow its contact flag (a swing segment starts with the lift-off velocity), x segments with knots on nodes and
    between them (first knot after t0: the first segment extrapolates before it), no y segments on the right feet."""
    events = sorted(float(e) for e in events)
    modes = [int(rng.integers(0, 4))]
    for _ in events:
        modes.append(int((modes[-1] + rng.integers(1, 4)) % 4))
    inner = [e for e in events if t0 < e < tf]
    tt = sorted(set([t0 - 0.05, float(nodes[min(2, len(nodes) - 1)]), float(nodes[len(nodes) // 2]), tf + 0.05] + inner[:1]))
    ts = [rng.uniform(-1.0, 1.0, 22) for _ in tt]
    segs = [[[] for _ in range(3)] for _ in range(4)]
    for c in range(4):
        flags = [R.stance_legs(m)[c] for m in modes]
        knots = [t0 - 0.1] + [e for j, e in enumerate(events) if flags[j + 1] != flags[j]] + [tf + 0.1]
        phase = [flags[0]] + [flags[j + 1] for j, e in enumerate(events) if flags[j + 1] != flags[j]]
        for j in range(min(len(knots) - 1, HB_MAX_SEGMENTS)):
            if knots[j + 1] > knots[j]:
                z = 0.02 + 0.01 * c
                segs[c][2].append((knots[j], knots[j + 1], z, 0.0 if phase[j] else LIFTOFF_VEL, z + (0.0 if phase[j] else 0.03), 0.0))
        m = len(nodes) // 2
        xk = sorted(set(float(t) for t in (nodes[min(1, len(nodes) - 1)], nodes[m], 0.5 * (nodes[m] + nodes[min(m + 1, len(nodes) - 1)]), nodes[-1])))
        for j in range(len(xk) - 1):
            segs[c][0].append((xk[j], xk[j + 1], *rng.uniform(-0.3, 0.3, 4)))
        if c % 2 == 0:
            segs[c][1].append((t0 - 0.2, tf + 0.2, *rng.uniform(-0.3, 0.3, 4)))
    return dict(events=events, modes=modes, target_times=tt, target_states=np.array(ts), segments=segs)


def _pack(refs):
    arr = (HbReference * len(refs))()
    for r, rec in zip(refs, np.ctypeslib.as_array(arr)):
        TA.pack_reference(r, rec)
    return arr


def _padded(g, N):
    return np.concatenate([g, np.full(N + 1 - len(g), g[-1])])


# ------------------------------------------------------------------------------------------------------------------------------ the grid
def _grid_cases():
    """{(N, dt, T): [(t0, events)]}: every case of a context runs in one batch (instances with different interval counts)."""
    t0 = 1.0
    s = _steps(t0, DT, 60)
    tf = t0 + T
    main = []
    for k in (3, 17):
        for d in (0.0, 1e-12, -1e-12, 1e-9, -1e-9, 2e-9, -2e-9):
            main.append((t0, [s[k] + d, s[30] + 0.004]))
    main += [(t0, [s[4] + 0.003, s[4] + 0.011]), (t0, [s[4] + 0.002, s[4] + 0.006, s[4] + 0.013]), (t0, [s[6] + 0.004, s[6] + 0.004, s[9]]),
             (t0, [s[6] + 0.004, s[6] + 0.004 + 5e-10, s[9] + 0.001, s[9] + 0.001 + 1e-9]), (t0, [t0, s[5] + 0.001]), (t0, [t0 + 1e-12]),
             (t0, [t0 + 1e-9, s[8]]), (t0, [t0 + 2e-9]), (t0, [t0 - 0.2, t0 - 1e-9, s[2] + 0.005]), (t0, [s[10] + 0.002, tf]),
             (t0, [tf - 1e-9]), (t0, [s[10] + 0.002, tf + 1e-12, tf + 0.01]), (1.2, [1.25, 1.3])]
    ev = [s[2] + 0.004, s[20] + 0.001, s[33] + 0.009]
    n_full = len(TA.event_node_grid(t0, T, DT, ev, HB_MAX_HORIZON)[0]) - 1
    return {
        (64, DT, T): main,
        (n_full, DT, T): [(t0, ev), (t0, ev + [s[40] + 0.002]), (t0, ev[:1])],       # capacity reached exactly, exceeded by one, not reached
        (HB_MAX_HORIZON, 0.005, 2.5): [(t0, list(t0 + 0.003 + 0.0245 * np.arange(HB_MAX_EVENTS))), (t0, [t0 + 1.3, t0 + 2.2])],
        (33, DT, T): [(t0, ev), (t0, [])],
        (33, DT, 0.1234): [(t0, [s[2] + 0.004]), (t0, [])],
        (1, DT, 0.01): [(t0, []), (t0, [t0 + 0.004])],
        (2, DT, 0.01): [(t0, []), (t0, [t0 + 0.004]), (t0, [t0 + 0.004, t0 + 0.006])],
        (4, DT, 5e-10): [(t0, []), (t0, [t0 + 1e-10])],
    }


def _grid_dev(ctx, t0, refs):
    import torch
    B, N = len(t0), ctx.N
    t0_d = torch.tensor(t0, dtype=torch.float64, device="cuda")
    rf = torch.frombuffer(bytearray(bytes(refs)), dtype=torch.uint8).cuda()
    tk = torch.zeros((B, N + 1), dtype=torch.float64, device="cuda"); nn = torch.zeros(B, dtype=torch.int32, device="cuda")
    st = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    _check(ctx._lib.hb_time_grid_batch_dev(ctx._h, B, _ptr(t0_d), _ptr(rf), _ptr(tk), _ptr(nn), _ptr(st)), "hb_time_grid_batch_dev", ctx._h)
    ctx.sync()
    return tk.cpu().numpy(), nn.cpu().numpy(), st.cpu().numpy()


@pytest.mark.parametrize("key", list(_grid_cases()), ids=["N%d_dt%g_T%g" % k for k in _grid_cases()])
def test_event_grid_and_the_references_on_it(key, contexts):
    """Node times bit for bit, interval counts and status equal the restatement (host and device-pointer forms); nodes beyond nn repeat
    tk[nn]. The expansion on the grid: modes exactly, targets within 1e-12 (nodes on sample times, outside the samples), swing within
    1e-11 (nodes on knots: a lift-off node has the lift-off velocity; before the first and after the last segment the spline
    extrapolates). The swing tolerance is relative to values above 1: a spline extrapolated a second past a 25 ms segment reaches 1e4."""
    N, dt, T_ = key
    cases = _grid_cases()[key]
    ctx = contexts(N, dt, T_, max_batch=len(cases))
    rng = np.random.default_rng(N)
    t0 = np.array([c[0] for c in cases])
    grids = [TA.event_node_grid(c[0], T_, dt, sorted(c[1]), N) for c in cases]
    refs = [_reference(rng, c[0], c[0] + T_, c[1], g) for c, (g, _) in zip(cases, grids)]
    packed = _pack(refs)
    for tk, nn, st in (ctx.time_grid(t0, packed), _grid_dev(ctx, t0, packed)):
        for i, (g, status) in enumerate(grids):
            assert nn[i] == len(g) - 1 and st[i] == status, (i, nn[i], st[i], len(g) - 1, status)
            assert np.array_equal(tk[i], _padded(g, N)), (i, tk[i], g)
    xr, sw, md = ctx.reference_expand_grid(tk, packed)
    liftoffs = 0
    for i, (g, _) in enumerate(grids):
        xo, so, mo = TA.sample_reference(refs[i], _padded(g, N))
        assert np.array_equal(md[i], mo), (i, md[i], mo)
        assert np.abs(xr[i] - xo).max() <= 1e-12 and (np.abs(sw[i] - so) <= 1e-11 * np.maximum(1.0, np.abs(so))).all(), i
        for c in range(4):
            for sg in refs[i]["segments"][c][2]:
                if sg[3] == LIFTOFF_VEL and sg[0] in g:
                    k = int(np.flatnonzero(g == sg[0])[0])
                    assert abs(sw[i, k, 6 * c + 5] - LIFTOFF_VEL) <= 1e-11, (i, k)
                    liftoffs += 1
    if key == (64, DT, T):
        assert liftoffs > 0 and len(set(nn.tolist())) > 1


def test_uniform_expansion_on_nodes_that_hit_knots(contexts):
    """hb_reference_expand_batch on t0 + k dt with switches on nodes, 1e-12 after one (in force on the interval it starts) and between
    nodes, target samples and spline knots on nodes."""
    N, B = 40, 4
    ctx = contexts(N, UDT, event_nodes=False, max_batch=B)
    rng = np.random.default_rng(5)
    t0 = 1.0 + UDT * np.arange(B)
    refs = []
    for i in range(B):
        nodes = t0[i] + UDT * np.arange(N + 1)
        ev = [nodes[3], nodes[7] + 1e-12, nodes[11] + 0.3 * UDT, nodes[20], nodes[N], nodes[N] + 0.01]
        refs.append(_reference(rng, t0[i], nodes[N], ev, nodes))
    xr, sw, md = ctx.reference_expand(t0, _pack(refs))
    for i in range(B):
        xo, so, mo = TA.sample_reference(refs[i], t0[i] + UDT * np.arange(N + 1))
        assert np.array_equal(md[i], mo) and md[i, 7] == refs[i]["modes"][2], i
        assert np.abs(xr[i] - xo).max() <= 1e-12 and np.abs(sw[i] - so).max() <= 1e-11, i


# ------------------------------------------------------------------------------------------------------------------------------ the policy
def _solutions(rng, B, N):
    x = sc.INITIAL_STATE[None, None, :] + rng.uniform(-0.05, 0.05, (B, N + 1, 22))
    u = rng.uniform(-20.0, 60.0, (B, N, 22))
    return x, u


def _queries(g):
    """Node times, one ulp either side, mid-interval, before t0, the horizon end and past it."""
    q = [g[0] - 0.01, g[-1] + 0.05]
    for k, t in enumerate(g):
        q += [t, np.nextafter(t, -np.inf), np.nextafter(t, np.inf)]
        if k + 1 < len(g):
            q.append(t + 0.37 * (g[k + 1] - t))
    return q


def _check_policy(xd, ud, mode, g, x, u, nodes_md, t, events, modes, capped, i):
    """One instance's policy output at absolute time t against evaluate_policy (x, u within 1e-13 relative, the node rule exactly) and,
    where the grid holds every switch, against modeAtTime. Returns 1 when modeAtTime was checked at a switch node."""
    n = len(g) - 1
    xe, ue, me = TA.evaluate_policy(g, x[:n + 1], u[:n], nodes_md, t)
    assert np.abs(xd - xe).max() <= 1e-13 * max(1.0, np.abs(xe).max()) and np.abs(ud - ue).max() <= 1e-13 * max(1.0, np.abs(ue).max()), (i, t)
    assert mode == me, (i, t, mode, me)
    _, k, _ = TA.interpolate(t, g, x[:n + 1])
    if events is None or not (g[0] < t <= g[-1]) or (capped and k == n - 1) or any(g[k] < e < g[k + 1] for e in events):
        return 0
    assert mode == TA.mode_at_time(events, modes, t), (i, t)
    return int(t in events and t != g[0])


def test_grid_policy_at_nodes_switches_and_edges(contexts):
    """hb_policy_eval_grid_batch_dev on event grids (capacity-exhausted and nn < N included): x, u and the mode at every node and switch
    node, one ulp either side, mid-interval, before t0 and past the end."""
    import torch
    N = 64
    cases = _grid_cases()[(N, DT, T)][::3] + [(1.0, [1.0 + 0.003 + 0.0235 * j for j in range(HB_MAX_EVENTS)])]
    B = len(cases)
    ctx = contexts(N, DT, T, max_batch=16)
    rng = np.random.default_rng(11)
    grids = [TA.event_node_grid(c[0], T, DT, sorted(c[1]), N) for c in cases]
    assert any(st for _, st in grids)
    refs = [_reference(rng, c[0], c[0] + T, c[1], g) for c, (g, _) in zip(cases, grids)]
    tk = np.stack([_padded(g, N) for g, _ in grids]); nn = np.array([len(g) - 1 for g, _ in grids], dtype=np.int32)
    md = np.stack([TA.sample_reference(r, tk[i])[2] for i, r in enumerate(refs)])
    x, u = _solutions(rng, B, N)
    dev = {k: torch.tensor(v, device="cuda") for k, v in dict(tk=tk, nn=nn, md=md, x=x, u=u).items()}
    xd = torch.zeros((B, 22), dtype=torch.float64, device="cuda"); ud = torch.zeros_like(xd); mo = torch.zeros(B, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    at_switch = 0
    for i in range(B):
        for t in _queries(grids[i][0]):
            t_rel = t - tk[i, 0]
            _check(ctx._lib.hb_policy_eval_grid_batch_dev(ctx._h, B, C.c_double(t_rel), _ptr(dev["tk"]), _ptr(dev["nn"]), _ptr(dev["x"]), _ptr(dev["u"]),
                                                           _ptr(dev["md"]), _ptr(xd), _ptr(ud), _ptr(mo)), "hb_policy_eval_grid_batch_dev", ctx._h)
            ctx.sync()
            xs, us, ms = xd.cpu().numpy(), ud.cpu().numpy(), mo.cpu().numpy()
            for b in range(B):
                g, st = grids[b]
                at_switch += _check_policy(xs[b], us[b], ms[b], g, x[b], u[b], md[b], tk[b, 0] + t_rel, refs[b]["events"], refs[b]["modes"], st == 1, b)
    assert at_switch > 0


def test_uniform_policy_and_the_node_rule(contexts):
    """hb_policy_eval_batch_dev on the uniform grid: the same queries; the mode is the node rule. A switch between two nodes is not seen
    before the next node: mid-interval after it the policy keeps the node's mode while modeAtTime has switched (DESIGN §2 item 2)."""
    import torch
    N, B = 40, 3
    ctx = contexts(N, UDT, event_nodes=False, max_batch=B)
    rng = np.random.default_rng(12)
    rel = UDT * np.arange(N + 1)
    ev = [rel[3], rel[7] + 1e-12, rel[11] + 0.3 * UDT, rel[20]]
    modes = [3, 1, 2, 0, 3]
    md = np.tile(np.array([TA.interval_mode(ev, modes, t) for t in rel], dtype=np.int32), (B, 1))
    x, u = _solutions(rng, B, N)
    dev = {k: torch.tensor(v, device="cuda") for k, v in dict(md=md, x=x, u=u).items()}
    xd = torch.zeros((B, 22), dtype=torch.float64, device="cuda"); ud = torch.zeros_like(xd); mo = torch.zeros(B, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    node_rule_pinned = False
    for t in _queries(rel):
        _check(ctx._lib.hb_policy_eval_batch_dev(ctx._h, B, C.c_double(t), _ptr(dev["x"]), _ptr(dev["u"]), _ptr(dev["md"]), _ptr(xd), _ptr(ud), _ptr(mo)),
               "hb_policy_eval_batch_dev", ctx._h)
        ctx.sync()
        xs, us, ms = xd.cpu().numpy(), ud.cpu().numpy(), mo.cpu().numpy()
        for b in range(B):
            _check_policy(xs[b], us[b], ms[b], rel, x[b], u[b], md[b], t, None, None, False, b)
        if ev[2] < t < rel[12]:
            assert ms[0] == md[0, 11] != TA.mode_at_time(ev, modes, t), t
            node_rule_pinned = True
        if t in (rel[3], rel[20]):                 # a switch on a node: the earlier mode, as modeAtTime
            assert ms[0] == TA.mode_at_time(ev, modes, t), t
    assert node_rule_pinned


def _planted(ctx, rng, cases, N):
    grids = [TA.event_node_grid(c[0], T, DT, sorted(c[1]), N) for c in cases]
    refs = [_reference(rng, c[0], c[0] + T, c[1], g) for c, (g, _) in zip(cases, grids)]
    tk = np.stack([_padded(g, N) for g, _ in grids]); nn = np.array([len(g) - 1 for g, _ in grids], dtype=np.int32)
    md = np.stack([TA.sample_reference(r, tk[i])[2] for i, r in enumerate(refs)])
    return grids, refs, tk, nn, md


def test_resident_policy_and_the_mrt_split_on_event_grids(contexts):
    """hb_resident_wbc_batch after hb_resident_write_batch planted random trajectories on the edge grids, at per-instance node times and
    around them; then the MRT split: after hb_policy_update with a mask, hb_policy_wbc evaluates the solution each instance adopted, not
    the newer resident one."""
    N = 64
    cases = _grid_cases()[(N, DT, T)][::3]
    B = len(cases)
    ctx = contexts(N, DT, T, max_batch=16)
    rng = np.random.default_rng(13)
    grids, refs, tk, nn, md = _planted(ctx, rng, cases, N)
    sols = [_solutions(rng, B, N) for _ in range(3)]
    rbd = sc.consistent_rbd(np.tile(sc.INITIAL_STATE, (B, 1)))
    ctx.resident_write(tk[:, 0], *sols[0], mode=md, node_times=tk, n_intervals=nn)
    ctx.policy_update(B)
    queries = [_queries(g) for g, _ in grids]
    at_switch = 0
    for j in range(max(len(q) for q in queries)):
        t_now = np.array([q[min(j, len(q) - 1)] for q in queries])
        xd, ud, mo, _, _, _ = ctx.resident_wbc(t_now, rbd)
        for b in range(B):
            at_switch += _check_policy(xd[b], ud[b], mo[b], grids[b][0], sols[0][0][b], sols[0][1][b], md[b], t_now[b], refs[b]["events"],
                                       refs[b]["modes"], grids[b][1] == 1, b)
    assert at_switch > 0
    mask = (np.arange(B) % 2 == 0)
    ctx.resident_write(tk[:, 0], *sols[1], mode=md, node_times=tk, n_intervals=nn)
    ctx.policy_update(B, mask)
    ctx.resident_write(tk[:, 0], *sols[2], mode=md, node_times=tk, n_intervals=nn)
    for j in (0, 5, 17):
        t_now = np.array([q[min(j, len(q) - 1)] for q in queries])
        xp, up, mp, _, _, _ = ctx.policy_wbc(t_now, rbd)
        xr_, ur_, _, _, _, _ = ctx.resident_wbc(t_now, rbd)
        for b in range(B):
            s = sols[1] if mask[b] else sols[0]
            _check_policy(xp[b], up[b], mp[b], grids[b][0], s[0][b], s[1][b], md[b], t_now[b], None, None, False, b)
            _check_policy(xr_[b], ur_[b], mp[b], grids[b][0], sols[2][0][b], sols[2][1][b], md[b], t_now[b], None, None, False, b)


# ------------------------------------------------------------------------------------------------------------------------------ warm start
def _assert_warm(info, xnew, unew, dev, n, i, what):
    assert info["alpha"][i] == dev[2]["alpha"][i] and info["n_trials"][i] == dev[2]["n_trials"][i], (what, i)
    assert np.abs(xnew[i, :n + 1] - dev[0][i, :n + 1]).max() < 1e-9, (what, i)
    assert np.abs(unew[i, :n] - dev[1][i, :n]).max() < 1e-7 * max(1.0, np.abs(dev[1][i, :n]).max()), (what, i)


def _prev_solution(rng, B, N, x1):
    x = x1[:, None, :] + rng.uniform(-0.01, 0.01, (B, N + 1, 22))
    u = np.zeros((B, N, 22)); u[:, :, 2::3][:, :, :4] = sc.TOTAL_MASS * 9.81 / 4
    return x, u + rng.uniform(-1.0, 1.0, u.shape)


def test_uniform_warm_start_at_every_shift(contexts):
    """One warm hb_resident_cycle_batch from a planted solution at shifts of 0, k dt, off the grid and past the horizon (initializer
    only) equals control_step on the restated warm start and the restated references."""
    N = 40
    shifts = np.array([0.0, 3 * UDT, 1.3 * UDT, N * UDT + 0.01])
    B = len(shifts)
    ctx = contexts(N, UDT, event_nodes=False, max_batch=B)
    rng = np.random.default_rng(21)
    x1 = sc.random_initial_states(B, seed=21)
    xp, up = _prev_solution(rng, B, N, x1)
    ctx.resident_write(np.ones(B), xp, up)
    t1 = 1.0 + shifts
    refs = [_reference(rng, t1[i], t1[i] + N * UDT, [t1[i] + 0.1, t1[i] + 0.25, t1[i] + 0.4], t1[i] + UDT * np.arange(N + 1)) for i in range(B)]
    rbd = sc.consistent_rbd(x1)
    info, _, _, _ = ctx.resident_cycle(False, 0.002, t1, x1, _pack(refs), rbd)
    _, xnew, unew = ctx.resident_read(B)
    xr = np.zeros((B, N + 1, 22)); sw = np.zeros((B, N + 1, 24)); md = np.zeros((B, N + 1), dtype=np.int32)
    xw = np.zeros((B, N + 1, 22)); uw = np.zeros((B, N, 22))
    for i in range(B):
        nodes = t1[i] + UDT * np.arange(N + 1)
        xr[i], sw[i], md[i] = TA.sample_reference(refs[i], nodes)
        xw[i], uw[i] = TA.warm_start(1.0 + UDT * np.arange(N + 1), xp[i], up[i], nodes, x1[i], md[i], sc.TOTAL_MASS)
    assert (xw[3] == x1[3]).all()                              # past the horizon: the initializer everywhere
    dev = ctx.control_step(0.002, x1, xr, sw, md, rbd, xw, uw)
    for i in range(B):
        _assert_warm(info, xnew, unew, dev, N, i, shifts[i])


def test_event_grid_warm_start_between_edge_grids(contexts):
    """Warm starts between two event grids: interval counts that differ, a capacity-exhausted previous grid, new nodes exactly on
    previous nodes and switches, and a new node within 1e-9 of the previous end on either side (and 2e-9 past it). The resident cycle
    equals mpc_solve_grid on the restated grid, references and warm start."""
    N = 64
    ctx = contexts(N, DT, T, max_batch=16)
    rng = np.random.default_rng(22)
    t1 = 1.02
    s = _steps(t1, DT, 60)
    events = [s[4] + 0.004, s[9], s[21] + 0.0101, s[40] + 0.002]
    g_new = TA.event_node_grid(t1, T, DT, events, N)[0]
    prev = [TA.event_node_grid(1.0, T, DT, [1.0 + 0.05 * j for j in range(1, 9)], N)[0],            # interval counts differ
            TA.event_node_grid(1.0, 1.3, DT, [1.31, 1.52], N)[0],                                # capacity exhausted
            np.concatenate([[1.0], g_new[1:30], g_new[30:44] + 0.004, [g_new[50]]])]             # on new nodes and switch nodes
    j = 37
    for d in (-5e-10, 5e-10, -2e-9):                                                          # the previous end near new node j
        prev.append(np.concatenate([np.linspace(1.0, g_new[j] + d, 30)]))
    assert TA.event_node_grid(1.0, 1.3, DT, [1.31, 1.52], N)[1] == 1 and len(prev[0]) != len(g_new)
    B = len(prev)
    x1 = sc.random_initial_states(B, seed=22)
    xp, up = _prev_solution(rng, B, N, x1)
    ctx.resident_write(np.array([p[0] for p in prev]), xp, up, node_times=np.stack([_padded(p, N) for p in prev]),
                       n_intervals=np.array([len(p) - 1 for p in prev], dtype=np.int32))
    refs = [_reference(rng, t1, t1 + T, events, g_new) for _ in range(B)]
    rbd = sc.consistent_rbd(x1)
    info, _, _, _ = ctx.resident_cycle(False, 0.002, np.full(B, t1), x1, _pack(refs), rbd)
    _, xnew, unew = ctx.resident_read(B)
    tk_d, nn_d = ctx.resident_read_grid(B)
    n = len(g_new) - 1
    tk = np.tile(_padded(g_new, N), (B, 1))
    assert (nn_d == n).all() and np.array_equal(tk_d, tk)
    xr = np.zeros((B, N + 1, 22)); sw = np.zeros((B, N + 1, 24)); md = np.zeros((B, N + 1), dtype=np.int32)
    xw = np.zeros((B, N + 1, 22)); uw = np.zeros((B, N, 22))
    for i in range(B):
        xr[i], sw[i], md[i] = TA.sample_reference(refs[i], tk[i])
        xw[i, :n + 1], uw[i, :n] = TA.warm_start(prev[i], xp[i, :len(prev[i])], up[i, :len(prev[i]) - 1], g_new, x1[i], md[i], sc.TOTAL_MASS)
    # new node j lies within 1e-9 past the previous end: still interpolated (the previous end); 2e-9 past it: the initializer from there
    assert np.array_equal(xw[3, j], xp[3, 29]) and not np.array_equal(xw[4, j], xp[4, 29]) and np.array_equal(xw[5, j], xw[5, j - 1])
    dev = ctx.mpc_solve_grid(x1, tk, np.full(B, n, dtype=np.int32), xr, sw, md, xw, uw)
    for i in range(B):
        _assert_warm(info, xnew, unew, dev, n, i, i)
