"""Cases of the MPC's filter line search (step S6: forward_linesearch2_kernel, the oracle's mpc_iteration), one per kind of decision it
takes, and the checks of their decisions on the oracle's per-trial record.

Each trial alpha = 1, 1/2, ... is decided by one of three branches, chosen by the trial's violation vn and the start's violation v0:
  violation  vn > g_max (0.01)                                     accept if vn < (1 - gamma_c) v0
  armijo     vn < g_min (1e-6), v0 < g_min and alpha armijo < 0    accept if merit < merit0 + 1e-4 alpha armijo
  filter     every other trial                                     accept if merit < merit0 - gamma_c v0 or vn < (1 - gamma_c) v0
A case is (name, N, dt or dts, x0, x_ref, swing, mode, xt, ut, expected), expected being the (branch, accepted) of every trial in order.
The name says what the trials do; make_cases asserts it, with check_margins, on the oracle's record.

Margin: every comparison a decision rests on clears its threshold by at least MARGIN_FACTOR times the tolerance the GPU test holds merits
and violations to (TOL relative to max(1, |value|)), so a kernel that agrees with the oracle within that tolerance takes the same decisions.
Iterations near convergence, where merit differences are round-off, are never cases.

Not covered, for want of a case with that margin: a trial with vn < g_min and v0 < g_min whose descent metric is not negative (filter
branch by the sign of armijo alone). Every such trial found sits at convergence, where armijo is round-off (about 1e-15). So a kernel
that dropped the sign test from the Armijo condition would pass these cases.

The recipes, all on a stance reference at rest:
  converged    INITIAL_STATE iterated to its violation floor (about 2e-8: below g_min), the base of the Armijo and reference-move cases;
  x_ref moves  the base x reference moved: the step scales with the move, and so trials alpha = 2^-j of a move 2^j d sit where the first
               trial of move d does. Moves of d 2^(k-1) are accepted by the filter at trial k after k - 1 violation rejections;
  squeeze      an internal normal-force pattern (+f on the left toe and right heel, -f on the others: no net force or moment) added to
               the converged warm start: the violation stays at its floor while the merit drops by about f^2 / 100;
  unloaded     the base reference lowered by 0.8 m and iterated to its floor (about 4e-7): the heels carry under 1 N at node 0, in the
               steep part of the normal-force barrier. The squeeze there at node 0 makes the quadratic model undershoot the merit, so
               alpha = 1 decreases it by less than the model predicts, or increases it; its amplitude is bisected to a chosen decrease.
               With half the squeeze at the other nodes as well, |armijo| grows to about 0.02 while vn stays below g_min, and alpha = 1
               can decrease the merit by between 1e-4 and 1e-3 times armijo with a margin to both (a between-factors case);
  cold start   the cold start of a perturbed initial state (violation accept at alpha 1), of INITIAL_STATE (filter accept on the
               violation alone: the merit rises), or of INITIAL_STATE in left support over the whole horizon (the robot falls: violation
               rejections, then a violation accept).
"""
import numpy as np

from hunter_bipedal_control_b200 import scenarios as sc

G_MAX, G_MIN, GAMMA_C, ARMIJO_FACTOR = 0.01, 1e-6, 1e-6, 1e-4
MAX_TRIALS = 14
TOL = 1e-8                      # the GPU test's tolerance on merits, violations and armijo, relative to max(1, |oracle|)
MARGIN_FACTOR = 10.0
SQUEEZE = np.array([1.0, -1.0, -1.0, 1.0])      # normal-force pattern over contacts (left toe, right toe, left heel, right heel)
VN_MOVE0 = 0.0033      # vn at alpha = 1 of the smallest base x reference move: a quarter of it is far below g_max, twice it far above

# grids of the GPU test: the BASELINE horizon, one just past a 32-lane trial round, and a non-uniform event grid
_EVENT_DTS = np.full(40, 0.01)
_EVENT_DTS[[5, 17, 18, 30]] = (0.002, 0.004, 0.006, 0.0015)
_EVENT_DTS[[9, 24]] = 0.014
EVENT_TIMES = np.concatenate([[0.0], np.cumsum(_EVENT_DTS)])      # node times handed to the kernel, which takes dt_k = t_k+1 - t_k
GRIDS = {"baseline": (100, 0.01), "n33": (33, 0.01), "event": (40, np.diff(EVENT_TIMES))}
# base reference drop of the unloaded-heels cases, by grid. On the short grids the heels unload only with drops of 1.15 m or more, and
# there the trials near the Armijo bound have vn of about 1e-6: those cases are dropped on them
DROP = {"baseline": 0.8}


def _tol(v):
    return MARGIN_FACTOR * TOL * max(1.0, abs(v))


def decide(trial, info):
    """The branch a trial falls in and its decision, restated: (branch, accepted)."""
    vn, v0, m, m0 = trial["viol"], info["viol0"], trial["merit"], info["merit0"]
    am = trial["alpha"] * info["armijo"]
    if vn > G_MAX:
        return "violation", vn < (1.0 - GAMMA_C) * v0
    if vn < G_MIN and v0 < G_MIN and am < 0.0:
        return "armijo", m < m0 + ARMIJO_FACTOR * am
    return "filter", m < m0 - GAMMA_C * v0 or vn < (1.0 - GAMMA_C) * v0


def margins(trial, info):
    """(what, distance from its threshold, required distance) of every comparison the trial's decision rests on."""
    vn, v0, m, m0, arm = trial["viol"], info["viol0"], trial["merit"], info["merit0"], info["armijo"]
    am = trial["alpha"] * arm
    tv, tm = _tol(max(vn, v0)), _tol(max(abs(m), abs(m0)))
    out = [("vn vs g_max", abs(vn - G_MAX), tv)]
    branch, _ = decide(trial, info)
    if branch == "violation":
        return out + [("vn vs (1 - gamma) v0", abs(vn - (1.0 - GAMMA_C) * v0), tv)]
    if branch == "armijo":
        return out + [("vn vs g_min", G_MIN - vn, tv), ("v0 vs g_min", G_MIN - v0, tv), ("armijo sign", -arm, _tol(arm)),
                      ("merit vs Armijo", abs(m - m0 - ARMIJO_FACTOR * am), tm)]
    # filter: the Armijo branch is ruled out by vn or v0 above g_min (no case rules it out by the sign of armijo alone)
    out.append(("vn or v0 vs g_min", max(vn, v0) - G_MIN, tv))
    return out + [("merit vs filter", abs(m - m0 + GAMMA_C * v0), tm), ("vn vs (1 - gamma) v0", abs(vn - (1.0 - GAMMA_C) * v0), tv)]


def check_margins(trials, info):
    """Every trial's decision restated from its record, and clear of its thresholds by the margin; returns the smallest ratio of margin to
    required distance."""
    worst = np.inf
    for t in trials:
        assert decide(t, info) == (t["branch"], t["accepted"]), (t, info)
        for what, d, need in margins(t, info):
            assert d >= need, (what, d, need, t, info)
            worst = min(worst, d / need)
    return worst


def pattern(trials):
    return [(t["branch"], t["accepted"]) for t in trials]


def _stance(N, x0=None):
    """A stance reference at rest from x0 (INITIAL_STATE by default). It is the same at every node time, so one sampling serves every
    grid of N intervals."""
    x0 = sc.INITIAL_STATE.copy() if x0 is None else x0
    xr, sw, md, _ = sc.make_reference(x0, (0.0, 0.0, 0.0, 0.0), "stance", N, 0.01)
    return x0, xr, sw, md


def _converge(oracle, N, dt, x0, xr, sw, md, iters):
    xt, ut = oracle.mpc_cold_start(N, dt, x0, md)
    for _ in range(iters):
        xt, ut, _ = oracle.mpc_iteration(N, dt, x0, xr, sw, md, xt, ut)
    return xt, ut


def _record(oracle, N, dt, c, max_trials=MAX_TRIALS):
    x0, xr, sw, md, xt, ut = c
    _, _, info, trials = oracle.mpc_iteration(N, dt, x0, xr, sw, md, xt, ut, max_trials=max_trials, record=True)
    return info, trials


def _squeezed(ut, f0, f=0.0):
    """The squeeze added to the warm-start input: amplitude f0 at node 0, f at the other nodes."""
    u = ut.copy()
    u[0, 2:12:3] += f0 * SQUEEZE
    u[1:, 2:12:3] += f * SQUEEZE
    return u


def _bisect(h, lo, hi, iters=40):
    """A root of h in [lo, hi] (h(lo) < 0 < h(hi))."""
    assert h(lo) < 0.0 < h(hi), (h(lo), h(hi))
    for _ in range(iters):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if h(mid) < 0.0 else (lo, mid)
    return hi


def make_cases(oracle, grid):
    """Every case of one grid (a GRIDS key), in a fixed order: list of (name, N, dt, x0, x_ref, swing, mode, xt, ut, expected). Asserts
    each case's named trials and margins on the oracle."""
    N, dt = GRIDS[grid]
    cases = []

    def add(name, c, expected, holds=None):
        """holds(last trial, info): what else the name promises of the last trial, asserted on the record."""
        info, trials = _record(oracle, N, dt, c)
        assert pattern(trials) == expected, (grid, name, pattern(trials))
        check_margins(trials, info)
        assert holds is None or holds(trials[-1], info), (grid, name, trials[-1], info)
        cases.append((name, N, dt) + tuple(c) + (expected,))

    merit_lower = lambda t, i: t["merit"] < i["merit0"] - GAMMA_C * i["viol0"]
    viol_lower = lambda t, i: t["viol"] < (1.0 - GAMMA_C) * i["viol0"]

    acc = lambda b: [(b, True)]
    V, A, F = "violation", "armijo", "filter"
    x0, xr, sw, md = _stance(N)
    xt, ut = _converge(oracle, N, dt, x0, xr, sw, md, 5)
    # violation branch: a cold start accepted at alpha = 1; a falling one accepted after back-tracking
    xp = sc.random_initial_states(1, seed=0)[0]
    xpr, swp, mdp = _stance(N, xp)[1:]
    add("violation/alpha1/cold-start", (xp, xpr, swp, mdp) + oracle.mpc_cold_start(N, dt, xp, mdp), acc(V))
    ms = np.full_like(md, 2)
    trials = _record(oracle, N, dt, (x0, xr, sw, ms) + oracle.mpc_cold_start(N, dt, x0, ms))[1]
    assert len(trials) >= 2, grid
    add("violation/backtracked/single-support-cold-start", (x0, xr, sw, ms) + oracle.mpc_cold_start(N, dt, x0, ms),
        [(V, False)] * (len(trials) - 1) + acc(V))
    # filter branch: a reference move lowers the merit while the violation rises from its floor; the cold start of the resting state
    # removes most of its violation while the merit rises
    def moved(d):
        xm = xr.copy(); xm[:, 6] += d
        return (x0, xm, sw, md, xt, ut)
    move0 = 0.03 * np.sqrt(VN_MOVE0 / _record(oracle, N, dt, moved(0.03), max_trials=1)[1][0]["viol"])      # vn grows with the move squared
    add("filter/alpha1/merit-only", moved(move0), acc(F), lambda t, i: merit_lower(t, i) and not viol_lower(t, i))
    add("filter/alpha1/violation-only", (x0, xr, sw, md) + oracle.mpc_cold_start(N, dt, x0, md), acc(F),
        lambda t, i: viol_lower(t, i) and not merit_lower(t, i))
    # Armijo branch: the squeeze at the floor, accepted at alpha = 1 with a decrease of half the model's (alpha armijo / 2)
    add("armijo/alpha1/squeeze", (x0, xr, sw, md, xt, _squeezed(ut, 2.0, 2.0)), acc(A),
        lambda t, i: abs((t["merit"] - i["merit0"]) / i["armijo"] - 0.5) < 0.05)
    # the unloaded heels: alpha = 1 rejected by the Armijo test (the merit above the Armijo bound by 3 margins), alpha = 1/2 accepted
    if grid in DROP:
        xd = xr.copy(); xd[:, 8] -= DROP[grid]
        xdt, udt = _converge(oracle, N, dt, x0, xd, sw, md, 14)

        def excess(f):
            info, trials = _record(oracle, N, dt, (x0, xd, sw, md, xdt, _squeezed(udt, f)), max_trials=1)
            return trials[0]["merit"] - info["merit0"] - ARMIJO_FACTOR * info["armijo"] - 3.0 * _tol(info["merit0"])
        add("armijo/backtracked/unloaded-heels", (x0, xd, sw, md, xdt, _squeezed(udt, _bisect(excess, 1.0, 2.5))), [(A, False)] + acc(A))

        # alpha = 1 accepted with a merit decrease between ARMIJO_FACTOR and ten times it (times alpha armijo), midway in that band: the
        # squeeze of half amplitude at the other nodes raises |armijo| to about 0.02 so that the band holds a margin on either side
        def in_band(f):
            info, trials = _record(oracle, N, dt, (x0, xd, sw, md, xdt, _squeezed(udt, f, 0.5)), max_trials=1)
            return trials[0]["merit"] - info["merit0"] - 5.5 * ARMIJO_FACTOR * info["armijo"]

        def between_factors(t, i):
            dm, am, tol = t["merit"] - i["merit0"], t["alpha"] * i["armijo"], _tol(i["merit0"])
            return 10.0 * ARMIJO_FACTOR * am + tol <= dm <= ARMIJO_FACTOR * am - tol
        add("armijo/alpha1/between-factors", (x0, xd, sw, md, xdt, _squeezed(udt, _bisect(in_band, 1.0, 3.5), 0.5)), acc(A), between_factors)
    # every trial count (the merit-only case takes one): the move move0 * 2^(k-1) is rejected by the violation test k - 1 times, then
    # accepted by the filter; twice the move that takes all 14 trials is rejected at every one
    for k in range(2, MAX_TRIALS + 1):
        add("trials/%02d/move-x" % k, moved(move0 * 2.0 ** (k - 1)), [(V, False)] * (k - 1) + acc(F))
    add("rejected/move-x", moved(move0 * 2.0 ** MAX_TRIALS), [(V, False)] * MAX_TRIALS)
    return cases


def stack(cases):
    """(x0, x_ref, swing, mode, xt, ut) of a batch of cases of one grid."""
    return tuple(np.stack([c[3 + i] for c in cases]) for i in range(6))

