"""The raw batched QP solver (qp_batch_kernel -> qp_solve_warp, hb_wbc_qp_batch and its device forms) across its advertised envelope,
1 <= n <= 80 and 0 <= m <= 160, on problems with a known optimum (tests/qp_ref.py):
  - every shape-dependent path: the register-window Cholesky (n 6, 7, 28), lane-per-column and entry-by-entry narrow-row updates, the wide
    row product with its 10-row chunks and second 32-column block, two-sided rows active at either side;
  - the row capacity (32 equalities, 96 one-sided entries) and status 4 beyond it;
  - the row classification (zero rows, free rows, |bound| >= 1e19, exact lb == ub);
  - bitwise agreement of the three entry points, and batch independence.
The tolerances follow from the solver's termination test (relative residuals 1e-10, complementarity 1e-12) on problems whose reduced
Hessian has eigenvalues >= 0.1 and whose multipliers and gaps are >= 0.5."""
import ctypes as C

import numpy as np
import pytest

import qp_ref as Q

pytestmark = pytest.mark.gpu
MAX_ITER = 40       # Context's default qp_max_iter


def _rho(ctx):
    return ctx.cfg.wbc_rho


def _solve_check(ctx, oracle, qps, what):
    """Solve a batch; every problem solves to x* and agrees with the CPU interior point. Returns (worst relative error, iterations)."""
    x, st, it = ctx.wbc_qp(*Q.stack(qps))
    assert (st == 0).all(), "%s: statuses %s, iterations %s" % (what, st, it)
    assert (it < MAX_ITER).all(), "%s: iterations %s" % (what, it)
    worst = 0.0
    for i, q in enumerate(qps):
        worst = max(worst, Q.check_solution(x[i], q, "%s[%d]" % (what, i)))
        xo, sto, _ = oracle.qp_solve(q.H, q.g, q.A, q.lb, q.ub, _rho(ctx))
        assert sto == 0
        d = np.abs(x[i] - xo).max() / max(1.0, np.abs(q.x).max())
        assert d <= Q.X_RTOL, "%s[%d]: |x - x_oracle| = %.3g (relative)" % (what, i, d)
    return worst, it


@pytest.mark.parametrize("n", Q.NS)
def test_known_optimum_envelope(gpu_ctx, oracle, n):
    worst, iters = 0.0, []
    for mix in Q.MIXES:
        for singular_h in (False, True):
            qps = Q.envelope_cell(n, mix, singular_h, _rho(gpu_ctx))
            w, it = _solve_check(gpu_ctx, oracle, qps, "n=%d %s singular_h=%s" % (n, mix, singular_h))
            worst = max(worst, w); iters += list(it)
    hist = dict(zip(*np.unique(iters, return_counts=True)))
    print("\nqp envelope n=%d: worst |x - x*| = %.2e (relative), iterations %s" % (n, worst, {int(k): int(v) for k, v in hist.items()}))


def test_path_boundaries(gpu_ctx, oracle):
    """n = 32 with 32 / 33 narrow entries and n = 33 with 32; active rows of span 8 and 9; two-sided rows active at the lower side for
    n <= 32 and n > 32; more than 10 active wide rows at n = 28 and n = 64."""
    for name, qps in Q.boundary_cases(_rho(gpu_ctx)).items():
        _solve_check(gpu_ctx, oracle, qps, name)


def test_row_capacity(gpu_ctx, oracle):
    """32 equalities, 96 one-sided entries, 48 two-sided rows and a 160-row problem solve; one equality or entry more returns status 4
    with x = 0 and no iteration, although the problem is feasible (test_qp_envelope_host.py solves it on the CPU)."""
    for name, (qps, expect) in Q.capacity_cases(_rho(gpu_ctx)).items():
        if expect == 0:
            _solve_check(gpu_ctx, oracle, qps, name)
        else:
            x, st, it = gpu_ctx.wbc_qp(*Q.stack(qps))
            assert (st == 4).all() and (x == 0).all() and (it == 0).all(), (name, st, it)


def _with_row(q, a, lb, ub, at=None):
    """q with one more row (appended, or inserted at index `at`)."""
    at = q.m if at is None else at
    ins = lambda v, r: np.insert(v, at, r, axis=0)
    return Q.Qp(q.H, q.g, ins(q.A, a), ins(q.lb, lb), ins(q.ub, ub), q.x, ins(q.bound, np.nan))


def _with_bounds(q, lb, ub):
    return Q.Qp(q.H, q.g, q.A, lb, ub, q.x, q.bound)


def _bits(ctx, qps):
    x, st, it = ctx.wbc_qp(*Q.stack(qps))
    return x.view(np.uint64), st, it


def _same_bits(a, b):
    return all(np.array_equal(u, v) for u, v in zip(a, b))


def test_row_classification(gpu_ctx, oracle):
    """Zero rows, free rows and |bound| >= 1e19 as the header describes them."""
    rho = _rho(gpu_ctx)
    base = Q.envelope_cell(29, "each", False, rho)
    ref = _bits(gpu_ctx, base)
    z = np.zeros(29)
    a = np.random.default_rng(5).standard_normal(29)
    # a zero row with 0 inside its bounds is dropped, and so is a nonzero row without a finite bound (+-1e19 included): appended, the
    # solver sees the same rows in the same order, so the result is the same to the bit
    for row in ((z, -1.0, 1.0), (z, 0.0, 0.0), (z, -Q.INF, Q.INF), (z, 1e-12, Q.INF), (z, -Q.INF, -1e-12),
                (a, -Q.INF, Q.INF), (a, -1e19, 1e19), (a, -1e19, Q.INF)):
        assert _same_bits(_bits(gpu_ctx, [_with_row(q, *row) for q in base]), ref), row[1:]
    # inserted among the other rows, the problem still solves to x*
    rng = np.random.default_rng(6)
    mixed = [_with_row(_with_row(q, z, -0.5, 2.0, at=int(rng.integers(0, q.m + 1))), a, -1e19, 1e19, at=int(rng.integers(0, q.m + 2)))
             for q in base]
    _solve_check(gpu_ctx, oracle, mixed, "zero and free rows inserted")
    # a zero row whose bounds exclude 0: status 2, x = 0, no iteration
    for lb, ub in ((1.0, Q.INF), (-Q.INF, -1.0), (1.0, 1.0), (2e-12, Q.INF)):
        x, st, it = gpu_ctx.wbc_qp(*Q.stack([_with_row(q, z, lb, ub, at=3) for q in base]))
        assert (st == 2).all() and (x == 0).all() and (it == 0).all(), (lb, ub, st)


def test_row_capacity_classification(gpu_ctx, oracle):
    """Which rows count towards the row capacity, seen from problems at the capacity."""
    rho = _rho(gpu_ctx)
    # |bound| >= 1e19 is no bound, the next double towards 0 is one: at the capacity of 96 entries the first solves and the second does
    # not fit; replacing +-1e20 by +-1e19 leaves the result unchanged to the bit
    full, _ = Q.capacity_cases(rho)["in96"]
    full_bits = _bits(gpu_ctx, full)
    for side, inf in (("lb", -1e19), ("ub", 1e19)):
        moved, beyond = [], []
        for q in full:
            r = int(np.flatnonzero(q.lb <= -1e19)[0] if side == "lb" else np.flatnonzero(q.ub >= 1e19)[0])
            for out, v in ((moved, inf), (beyond, np.nextafter(inf, 0.0))):
                lb, ub = q.lb.copy(), q.ub.copy()
                (lb if side == "lb" else ub)[r] = v
                out.append(_with_bounds(q, lb, ub))
        assert _same_bits(_bits(gpu_ctx, moved), full_bits), side
        x, st, it = gpu_ctx.wbc_qp(*Q.stack(beyond))
        assert (st == 4).all() and (x == 0).all(), (side, st)
    # a free row does not count towards the capacity
    _solve_check(gpu_ctx, oracle, [_with_row(q, np.ones(Q.CAP_N), -Q.INF, Q.INF, at=5) for q in full], "96 entries + a free row")
    # equality is exact lb == ub: 33 equalities exceed the capacity, 32 and a two-sided row one double wide do not
    over, _ = Q.capacity_cases(rho)["eq33"]
    x, st, it = gpu_ctx.wbc_qp(*Q.stack(over))
    assert (st == 4).all()
    nudged = []
    for q in over:
        ub = q.ub.copy()
        r = int(np.flatnonzero(q.lb == q.ub)[0])
        ub[r] = np.nextafter(ub[r], np.inf)
        nudged.append(_with_bounds(q, q.lb, ub))
    x, st, it = gpu_ctx.wbc_qp(*Q.stack(nudged))
    assert (st != 4).all() and (it > 0).all(), (st, it)


def _dev(t):
    return C.c_void_p(t.data_ptr())


def test_entry_points_bitwise(gpu_ctx):
    """hb_wbc_qp_batch, hb_wbc_qp_batch_dev and hb_wbc_qp_rows_batch_dev give the same bits; the rows form reads only the first m_rows[i]
    rows of each problem (the rest are NaN) with m_rows[i] over 0 .. m_alloc in one batch."""
    import torch
    ctx, lib = gpu_ctx, gpu_ctx._lib
    qps = Q.envelope_cell(38, "ineq", True, _rho(ctx))
    H, g, A, lb, ub = Q.stack(qps)
    B, n, m = len(qps), qps[0].n, qps[0].m
    x_host, st_host, it_host = ctx.wbc_qp(H, g, A, lb, ub)
    dev = [torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in (H, g, A, lb, ub)]
    torch.cuda.synchronize()

    def run_dev(rows=None, m_alloc=m, args=dev):
        x = torch.zeros((B if rows is None else rows.shape[0], n), dtype=torch.float64, device="cuda")
        st = torch.full((x.shape[0],), -1, dtype=torch.int32, device="cuda"); it = torch.full_like(st, -1)
        ptrs = [_dev(t) for t in args] + [_dev(x), _dev(st), _dev(it)]
        if rows is None:
            rc = lib.hb_wbc_qp_batch_dev(ctx._h, B, n, m_alloc, *ptrs)
        else:
            rc = lib.hb_wbc_qp_rows_batch_dev(ctx._h, x.shape[0], n, m_alloc, _dev(rows), *ptrs)
        assert rc == 0
        ctx.sync()
        return x.cpu().numpy().view(np.uint64), st.cpu().numpy(), it.cpu().numpy()

    host = (x_host.view(np.uint64), st_host, it_host)
    assert (st_host == 0).all()
    assert _same_bits(run_dev(), host)
    assert _same_bits(run_dev(rows=torch.full((B,), m, dtype=torch.int32, device="cuda")), host)
    # per-problem row counts 0 .. m_alloc, NaN beyond them
    m_alloc = m + 3
    nb = m_alloc + 1
    idx = np.arange(nb) % B
    m_rows = np.arange(nb, dtype=np.int32)
    Ar = np.full((nb, m_alloc, n), np.nan); lbr = np.full((nb, m_alloc), np.nan); ubr = np.full((nb, m_alloc), np.nan)
    for i in range(nb):
        k = min(m_rows[i], m)
        Ar[i, :k] = A[idx[i], :k]; lbr[i, :k] = lb[idx[i], :k]; ubr[i, :k] = ub[idx[i], :k]
        Ar[i, k:m_rows[i]] = 0.0; lbr[i, k:m_rows[i]] = -1.0; ubr[i, k:m_rows[i]] = 1.0      # zero rows past the problem's own m
    args = [torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in (H[idx], g[idx], Ar, lbr, ubr)]
    rows = torch.from_numpy(m_rows).cuda()
    torch.cuda.synchronize()
    xr, str_, itr = run_dev(rows=rows, m_alloc=m_alloc, args=args)
    for i in range(nb):
        k = int(m_rows[i])
        xi, sti, iti = ctx.wbc_qp(H[idx[i]][None], g[idx[i]][None], Ar[i, :k][None], lbr[i, :k][None], ubr[i, :k][None])
        assert np.array_equal(xr[i], xi[0].view(np.uint64)) and str_[i] == sti[0] and itr[i] == iti[0], (i, k, str_[i], sti[0])
    assert (str_[m_rows >= m] == 0).all()


def test_batch_independence(gpu_ctx):
    """A problem solved alone equals its copy at position 1000 of a 1025-problem batch of other problems with the same n."""
    import torch
    ctx = gpu_ctx
    qps = Q.envelope_cell(64, "each", False, _rho(ctx))
    H, g, A, lb, ub = Q.stack(qps)
    rng = np.random.default_rng(11)
    nb, at = 1025, 1000
    idx = np.arange(nb) % len(qps)
    gb = g[idx] * (1.0 + 0.01 * rng.uniform(-1.0, 1.0, (nb, g.shape[1])))      # distinct problems
    gb[at] = g[3]
    idx[at] = 3
    alone = ctx.wbc_qp(H[3:4], g[3:4], A[3:4], lb[3:4], ub[3:4])
    assert alone[1][0] == 0
    dev = [torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in (H[idx], gb, A[idx], lb[idx], ub[idx])]
    x = torch.zeros((nb, H.shape[1]), dtype=torch.float64, device="cuda")
    st = torch.full((nb,), -1, dtype=torch.int32, device="cuda"); it = torch.full_like(st, -1)
    torch.cuda.synchronize()
    assert ctx._lib.hb_wbc_qp_batch_dev(ctx._h, nb, H.shape[1], A.shape[1], *[_dev(t) for t in dev + [x, st, it]]) == 0
    ctx.sync()
    x, st, it = x.cpu().numpy(), st.cpu().numpy(), it.cpu().numpy()
    assert (st == 0).all()
    assert np.array_equal(x[at].view(np.uint64), alone[0][0].view(np.uint64)) and st[at] == alone[1][0] and it[at] == alone[2][0]


def test_qp_edge_cases(gpu_ctx):
    """Empty batch; unconstrained, equality-only and two-sided problems with a closed-form optimum; an infeasible zero row."""
    # empty batch
    x, st, it = gpu_ctx.wbc_qp(np.zeros((0, 4, 4)), np.zeros((0, 4)), np.zeros((0, 3, 4)), np.zeros((0, 3)), np.zeros((0, 3)))
    assert x.shape == (0, 4)
    # unconstrained, equality-only, two-sided, infeasible zero row, all-zero rows
    H = np.array([np.diag([1.0, 2, 3, 4])] * 4); g = np.array([[-1.0, -2, -3, -4]] * 4)
    A = np.zeros((4, 3, 4)); lb = np.full((4, 3), -1e20); ub = np.full((4, 3), 1e20)
    A[1, 0] = [1, 1, 1, 1]; lb[1, 0] = ub[1, 0] = 1.0                      # equality sum x = 1
    A[2, 0] = [1, 0, 0, 0]; lb[2, 0] = -0.25; ub[2, 0] = 0.25              # two-sided bound active at 0.25
    lb[3, 0] = 1.0                                                         # zero row demanding 0 >= 1 : infeasible
    x, st, it = gpu_ctx.wbc_qp(H, g, A, lb, ub)
    # optimum of 1/2 x'(diag(c) + rho I)x - c'x: x = c / d with d = c + rho; with sum x = 1: x = (c - lam) / d
    c = np.array([1.0, 2, 3, 4]); d = c + _rho(gpu_ctx)
    assert st[0] == 0 and np.abs(x[0] - c / d).max() < Q.X_RTOL
    lam = ((c / d).sum() - 1.0) / (1.0 / d).sum()
    assert st[1] == 0 and np.abs(x[1] - (c - lam) / d).max() < Q.X_RTOL
    assert st[2] == 0 and abs(x[2, 0] - 0.25) < Q.X_RTOL and np.abs(x[2, 1:] - c[1:] / d[1:]).max() < Q.X_RTOL
    assert st[3] == 2 and (x[3] == 0).all() and it[3] == 0
