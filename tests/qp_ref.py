"""Dense QPs with a known optimum for the batched interior-point solver (hb_wbc_qp_batch), and the checks of a solution (numpy only).

The solver's problem is  min 1/2 x'(H + rho I)x + g'x  s.t.  lb <= A x <= ub.  make_qp draws x*, the constraint rows, an active set with
multipliers in [0.5, 2] and gaps in [0.5, 2], then sets g so that x* satisfies the KKT conditions exactly. The active normals have full row
rank and the reduced Hessian is positive definite, so x* is the unique, well-determined optimum.
"""
import numpy as np

INF = 1e20          # qpOASES' INFTY; the solver reads |bound| >= 1e19 as no bound
X_RTOL = 1e-7       # |x - x*|_inf <= X_RTOL * max(1, |x*|_inf)
ROW_RTOL = 1e-8     # row feasibility / activity to ROW_RTOL * (1 + |bound|)
SIGMA_MIN = 0.05    # smallest singular value accepted for the active normals


class Row:
    """One inequality row: kind 'u' (ub only), 'l' (lb only) or 't' (both); act None (inactive) or the side 'u' / 'l' that is active at
    x*; nonzeros on columns c0 .. c1-1."""
    __slots__ = ("kind", "act", "c0", "c1")

    def __init__(self, kind, act, c0, c1):
        assert kind in "ult" and act in (None, "u", "l") and (act is None or kind in (act, "t")) and 0 <= c0 < c1
        self.kind, self.act, self.c0, self.c1 = kind, act, c0, c1


def random_rows(rng, n, kinds, active, span="mixed"):
    """Rows of the given kinds (a string over 'ult'); the first `active` of them active at a random side. span: 'narrow' (1..8 columns),
    'wide' (9..n), 'mixed' (either, when n > 8), or an int (exact width)."""
    rows = []
    for q, kind in enumerate(kinds):
        if isinstance(span, int):
            w = span
        elif span == "wide" or (span == "mixed" and n > 8 and rng.random() < 0.5):
            w = int(rng.integers(9, n + 1))
        else:
            w = int(rng.integers(1, min(8, n) + 1))
        c0 = int(rng.integers(0, n - w + 1))
        act = None
        if q < active:
            act = kind if kind != "t" else ("u" if rng.random() < 0.5 else "l")
        rows.append(Row(kind, act, c0, c0 + w))
    return rows


class Qp:
    """H [n,n], g [n], A [m,n], lb / ub [m], x* [n] and, per row, the active bound (NaN when the row is not active at x*)."""

    def __init__(self, H, g, A, lb, ub, x, bound):
        self.H, self.g, self.A, self.lb, self.ub, self.x, self.bound = H, g, A, lb, ub, x, bound

    @property
    def n(self):
        return self.g.size

    @property
    def m(self):
        return self.lb.size


def _unit_rows(rng, k, n, c0, c1):
    A = np.zeros((k, n))
    for i in range(k):
        A[i, c0[i]:c1[i]] = rng.standard_normal(c1[i] - c0[i])
        A[i] /= np.linalg.norm(A[i])
    return A


def _symmetric(M):
    return 0.5 * (M + M.T)       # fl(a + b) = fl(b + a): exactly symmetric


def make_qp(n, me, rows, rng, rho, singular_h=False, max_tries=200):
    """Known-optimum problem with n variables, me dense equality rows and the inequality rows `rows` (a list of Row). The rows are shuffled.
    singular_h: H has curvature only on the null space of the active normals and on half of their span (the WBC's situation, where
    H = A_w' A_w is singular); otherwise H = Q diag(lambda) Q' with lambda log-uniform in [0.1, 10]."""
    k_in = sum(r.act is not None for r in rows)
    assert me + k_in <= n, "more active rows than variables"
    xs = rng.standard_normal(n)
    for _ in range(max_tries):
        Aeq = np.linalg.qr(rng.standard_normal((n, me)))[0].T       # dense orthonormal rows (me <= n)
        Ain = _unit_rows(rng, len(rows), n, [r.c0 for r in rows], [r.c1 for r in rows])
        act = np.array([r.act is not None for r in rows], dtype=bool)
        Aact = np.vstack([Aeq, Ain[act]])
        if Aact.shape[0] == 0 or np.linalg.svd(Aact, compute_uv=False).min() >= SIGMA_MIN:
            break
    else:
        raise RuntimeError("no well-conditioned active set for n=%d me=%d rows=%d" % (n, me, len(rows)))
    k = Aact.shape[0]
    # H
    if singular_h:
        Vt = np.linalg.svd(Aact, full_matrices=True)[2] if k else np.eye(n)
        R, N = Vt[:k].T, Vt[k:].T            # span / null space of the active normals
        B = np.hstack([N, R[:, : k // 2]])
    else:
        B = np.linalg.qr(rng.standard_normal((n, n)))[0]
    lam = np.exp(rng.uniform(np.log(0.1), np.log(10.0), B.shape[1]))
    H = _symmetric((B * lam) @ B.T)
    # bounds and multipliers
    ax = Ain @ xs
    lb = np.full(len(rows), -INF); ub = np.full(len(rows), INF)
    g = -(H @ xs + rho * xs)
    bound_in = np.full(len(rows), np.nan)
    for i, r in enumerate(rows):
        gap_lo, gap_hi = rng.uniform(0.5, 2.0, 2)
        if r.kind in "ut":
            ub[i] = ax[i] if r.act == "u" else ax[i] + gap_hi
        if r.kind in "lt":
            lb[i] = ax[i] if r.act == "l" else ax[i] - gap_lo
        if r.act is not None:
            lam_i = rng.uniform(0.5, 2.0)
            g -= (lam_i if r.act == "u" else -lam_i) * Ain[i]
            bound_in[i] = ax[i]
    beq = Aeq @ xs
    if me:
        g -= Aeq.T @ rng.standard_normal(me)
    A = np.vstack([Aeq, Ain])
    lbA = np.concatenate([beq, lb]); ubA = np.concatenate([beq, ub]); bound = np.concatenate([beq, bound_in])
    p = rng.permutation(A.shape[0])
    return Qp(H, g, A[p], lbA[p], ubA[p], xs, bound[p])


def mix(rng, n, name):
    """(me, rows) of a named row mix: 'none', 'each' (one row of every kind and side), 'eq' (min(n, 32) equalities), 'ineq' (96 one-sided
    entries, 24 of them in two-sided rows)."""
    kmax = n if n <= 8 else n - n // 4           # active rows (equalities included) at most
    if name == "none":
        return 0, []
    if name == "each":
        me = 1
        spec = [("u", "u"), ("l", "l"), ("t", "l"), ("t", "u"), ("u", None), ("l", None), ("t", None)]
        rows = []
        k = me
        for kind, act in spec:
            if act is not None and k >= kmax:
                act = None
            k += act is not None
            rows += random_rows(rng, n, kind, 0)
            rows[-1].act = act
        return me, rows
    if name == "eq":
        me = min(n, 32)
        return me, random_rows(rng, n, "ult" * 2, 0)
    if name == "ineq":
        me = min(4, n // 4)
        kinds = "t" * 12 + "u" * 36 + "l" * 36               # 12 * 2 + 72 = 96 entries
        kinds = "".join(rng.permutation(list(kinds)))
        return me, random_rows(rng, n, kinds, min(kmax - me, max(1, n // 2)))
    raise ValueError(name)


def pad_rows(qps, m, rng, n_zero=None):
    """Bring every problem to m rows by inserting, at random positions, zero rows (bounds containing 0: dropped by the solver) and free
    rows (a nonzero row with both bounds at +-1e20: ignored). n_zero: how many of the inserted rows are zero rows (default half)."""
    out = []
    for q in qps:
        extra = m - q.m
        assert extra >= 0
        nz = extra // 2 if n_zero is None else n_zero
        A = np.zeros((extra, q.n))
        A[nz:] = rng.standard_normal((extra - nz, q.n))
        lb = np.full(extra, -INF); ub = np.full(extra, INF)
        lb[: nz] = np.where(rng.random(nz) < 0.5, -INF, -rng.uniform(0.0, 1.0, nz))
        ub[: nz] = np.where(rng.random(nz) < 0.5, INF, rng.uniform(0.0, 1.0, nz))
        At = np.vstack([q.A, A]); lbt = np.concatenate([q.lb, lb]); ubt = np.concatenate([q.ub, ub])
        bt = np.concatenate([q.bound, np.full(extra, np.nan)])
        p = rng.permutation(m)
        out.append(Qp(q.H, q.g, At[p], lbt[p], ubt[p], q.x, bt[p]))
    return out


def classify(q):
    """The solver's view of the rows (hb_wbc_qp_batch_dev): (equality rows, one-sided entries with a two-sided row counting twice,
    entries in its processing order, narrow among them (span <= 8 columns)). Zero rows and rows without finite bounds count nowhere."""
    me = entries = ordered = narrow = 0
    for a, lo, hi in zip(q.A, q.lb, q.ub):
        nz = np.flatnonzero(a)
        has_lo, has_hi = lo > -1e19, hi < 1e19
        if nz.size == 0 or not (has_lo or has_hi):
            continue
        if has_lo and has_hi and lo == hi:
            me += 1
            continue
        entries += int(has_lo) + int(has_hi)
        ordered += 1
        narrow += int(nz[-1] + 1 - nz[0] <= 8)
    return me, entries, ordered, narrow


def stack(qps):
    """Batch arrays (H, g, A, lb, ub) of problems with one n and one m."""
    return (np.stack([q.H for q in qps]), np.stack([q.g for q in qps]), np.stack([q.A for q in qps]).reshape(len(qps), -1, qps[0].n),
            np.stack([q.lb for q in qps]), np.stack([q.ub for q in qps]))


# ---------------------------------------------------------------- the problem sets shared by the CPU and the GPU tests
NS = (1, 2, 5, 6, 7, 8, 27, 28, 29, 31, 32, 33, 38, 64, 79, 80)   # raw n 6, 7, 28: register-window Cholesky; n <= 32: lane-per-column updates
MIXES = ("none", "each", "eq", "ineq")
PER_CELL = 8


def envelope_cell(n, mix_name, singular_h, rho):
    """PER_CELL known-optimum problems with n variables and one row mix, padded with two zero / free rows to one m ('none': m = 0)."""
    rng = np.random.default_rng([n, MIXES.index(mix_name), int(singular_h)])
    qps = [_draw(rng, lambda: mix(rng, n, mix_name), n, rho, singular_h) for _ in range(PER_CELL)]
    return pad_rows(qps, max(q.m for q in qps) + (0 if mix_name == "none" else 2), rng)


def _draw(rng, spec, n, rho, singular_h):
    """make_qp on spec() = (me, rows), drawing a new spec when its spans admit no well-conditioned active set (e.g. two active
    1-column rows on one column)."""
    for _ in range(50):
        me, rows = spec()
        try:
            return make_qp(n, me, rows, rng, rho, singular_h, max_tries=20)
        except RuntimeError:
            pass
    raise RuntimeError("no well-conditioned problem with n=%d" % n)


def _cell(seed, n, me, kinds, active, span, rho, count=PER_CELL, singular_h=False, pad=0, sides=None):
    """count problems with me equalities and rows of the given kinds, the first `active` of them active (at side `sides` when given)."""
    rng = np.random.default_rng(seed)

    def spec():
        rows = random_rows(rng, n, kinds, active, span)
        for r in rows[:active]:
            r.act = sides or r.act
        return me, rows
    qps = [_draw(rng, spec, n, rho, singular_h) for _ in range(count)]
    return pad_rows(qps, qps[0].m + pad, rng) if pad else qps


def _one_sided(k, rng_seed):
    return "".join(np.random.default_rng(rng_seed).choice(list("ul"), k))


def boundary_cases(rho):
    """Problems on either side of each shape-dependent path of the solver: name -> list of problems with one n and one m."""
    c = {}
    # narrow-row updates: lane per column (n <= 32 and <= 32 narrow entries) or entry by entry (otherwise)
    c["n32_narrow32"] = _cell(1, 32, 2, _one_sided(32, 1), 10, "narrow", rho)
    c["n32_narrow33"] = _cell(2, 32, 2, _one_sided(33, 2), 10, "narrow", rho)
    c["n33_narrow32"] = _cell(3, 33, 2, _one_sided(32, 3), 10, "narrow", rho)
    # the wide threshold: active rows of span exactly 8 (narrow) and 9 (wide)
    for n in (20, 38):
        c["n%d_span8" % n] = _cell(10 + n, n, 1, _one_sided(10, 10 + n), 6, 8, rho)
        c["n%d_span9" % n] = _cell(20 + n, n, 1, _one_sided(10, 20 + n), 6, 9, rho)
    # two-sided rows active at their lower side: the entry merged into its partner
    for n in (20, 40):
        c["n%d_two_sided_lower" % n] = _cell(30 + n, n, 1, "t" * 10, 6, "mixed", rho, sides="l")
    # more than 10 wide rows, more than 10 of them active: the 10-row chunk loop runs three times; n = 64 adds a second 32-column block
    c["n28_wide24"] = _cell(40, 28, 0, "t" * 4 + _one_sided(20, 40), 12, "wide", rho)
    c["n64_wide24"] = _cell(41, 64, 2, "t" * 4 + _one_sided(20, 41), 14, "wide", rho, singular_h=True)
    return c


CAP_N = 64


def capacity_cases(rho):
    """name -> (problems, expected status): at the row capacity (32 equalities, 96 one-sided entries, a two-sided row counting twice)
    the solver solves; one row beyond it returns status 4. Every problem is feasible with a known optimum."""
    n, k = CAP_N, 4
    return {
        "eq32": (_cell(50, n, 32, "ul", 0, "mixed", rho, k), 0),
        "in96": (_cell(51, n, 0, _one_sided(96, 51), 12, "mixed", rho, k), 0),
        "two48": (_cell(52, n, 0, "t" * 48, 12, "mixed", rho, k), 0),
        "m160": (_cell(53, n, 32, _one_sided(96, 53), 8, "mixed", rho, k, pad=32), 0),
        "eq33": (_cell(54, n, 33, "ul", 0, "mixed", rho, k), 4),
        "in97": (_cell(55, n, 0, _one_sided(97, 55), 12, "mixed", rho, k), 4),
        "two48_in1": (_cell(56, n, 0, "t" * 48 + "u", 12, "mixed", rho, k), 4),
    }


def solution_error(x, q):
    """(relative error of x against x*, worst row violation and worst active-row miss, each relative to 1 + |bound|)."""
    ex = np.abs(x - q.x).max() / max(1.0, np.abs(q.x).max())
    ax = q.A @ x
    viol = 0.0
    fin_lo = q.lb > -1e19; fin_hi = q.ub < 1e19
    if fin_lo.any():
        viol = max(viol, (np.maximum(q.lb[fin_lo] - ax[fin_lo], 0.0) / (1.0 + np.abs(q.lb[fin_lo]))).max())
    if fin_hi.any():
        viol = max(viol, (np.maximum(ax[fin_hi] - q.ub[fin_hi], 0.0) / (1.0 + np.abs(q.ub[fin_hi]))).max())
    act = ~np.isnan(q.bound)
    miss = (np.abs(ax[act] - q.bound[act]) / (1.0 + np.abs(q.bound[act]))).max() if act.any() else 0.0
    return ex, viol, miss


def check_solution(x, q, what=""):
    """x is x* to X_RTOL, every row is feasible and every active row is met to ROW_RTOL. Returns the relative error of x."""
    ex, viol, miss = solution_error(x, q)
    assert np.isfinite(x).all() and ex <= X_RTOL, "%s: |x - x*| = %.3g (relative)" % (what, ex)
    assert viol <= ROW_RTOL, "%s: row violation %.3g" % (what, viol)
    assert miss <= ROW_RTOL, "%s: active row missed by %.3g" % (what, miss)
    return ex
