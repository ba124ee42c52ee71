"""Float64 numpy restatement of the MPC stage cost's 52 relaxed-barrier penalties per node, a classifier of their regions, and the case
generator of the penalty-envelope tests.

The penalties (LeggedInterface.cpp:317-357, FrictionConeConstraint.cpp:78-233, task.info frictionConeSoftConstraint):
  joint positions   DoubleSidedPenalty(lower, upper, RelaxedBarrierPenalty(mu 1, delta 0.1))       10 joints x 2 sides
  joint velocities  DoubleSidedPenalty(-limit, limit, RelaxedBarrierPenalty(mu 1, delta 0.1))      10 joints x 2 sides
  normal forces     DoubleSidedPenalty(0, 350, RelaxedBarrierPenalty(mu 0.1, delta 1))             4 contacts x 2 sides
  friction cones    RelaxedBarrierPenalty(mu 0.1, delta 5) of 0.7 F_z - sqrt(F_x^2 + F_y^2 + 25)    stance contacts only
RelaxedBarrierPenalty is -mu log(h) above delta and the quadratic extension mu (-log(delta) + ((h - 2 delta) / delta)^2 / 2 - 1/2) at or
below it, which continues into violation (h <= 0). The cone's Hessian carries OCS2's hessianDiagonalShift: -1e-6 on every diagonal entry
of the constraint's state and input Hessians, so the cost's Q and R diagonals take -1e-6 d1 from each stance cone."""
import numpy as np

from hunter_bipedal_control_b200 import scenarios as sc
from oracle import refs as R

NX = NU = 22
NJ = 10
JOINT_LOWER = np.array(R._header_array("HB_JOINT_LOWER"))
JOINT_UPPER = np.array(R._header_array("HB_JOINT_UPPER"))
JOINT_VEL = np.array(R._header_array("HB_JOINT_VEL_LIMIT"))
Q_DIAG = np.array(R._header_array("HB_Q_DIAG"))
POS = (R._header_value("HB_LIMIT_POS_MU"), R._header_value("HB_LIMIT_POS_DELTA"))          # (mu, delta)
VEL = (R._header_value("HB_LIMIT_VEL_MU"), R._header_value("HB_LIMIT_VEL_DELTA"))
FORCE = (R._header_value("HB_LIMIT_FORCE_MU"), R._header_value("HB_LIMIT_FORCE_DELTA"))
FORCE_MAX = R._header_value("HB_LIMIT_FORCE_MAX")
CONE = (R._header_value("HB_FRICTION_BARRIER_MU"), R._header_value("HB_FRICTION_BARRIER_DELTA"))
FRICTION_MU = R._header_value("HB_FRICTION_MU")
FRICTION_REG = R._header_value("HB_FRICTION_REGULARIZATION")
HESSIAN_SHIFT = R._header_value("HB_FRICTION_HESSIAN_SHIFT")
SOFT_SWING_WEIGHT = R._header_value("HB_SOFT_SWING_WEIGHT")
XY_POSITION_GAIN = R._header_value("HB_XY_POSITION_GAIN")
TOTAL_MASS = R._header_value("HB_TOTAL_MASS")
GRAVITY = R._header_value("HB_GRAVITY")
assert POS == (1.0, 0.1) and VEL == (1.0, 0.1) and FORCE == (0.1, 1.0) and CONE == (0.1, 5.0) and FORCE_MAX == 350.0

REGIONS = ("interior", "band", "violated")


def relaxed_barrier(h, mu, delta):
    """OCS2 RelaxedBarrierPenalty: value, first and second derivative in h."""
    if h > delta:
        return -mu * np.log(h), -mu / h, mu / (h * h)
    z = (h - 2.0 * delta) / delta
    return mu * (-np.log(delta) + 0.5 * z * z - 0.5), mu * (h - 2.0 * delta) / (delta * delta), mu / (delta * delta)


def double_sided(h, lo, hi, mu, delta):
    """OCS2 DoubleSidedPenalty: p(h - lo) + p(hi - h)."""
    a, b = relaxed_barrier(h - lo, mu, delta), relaxed_barrier(hi - h, mu, delta)
    return a[0] + b[0], a[1] - b[1], a[2] + b[2]


def cone(F):
    """Friction cone 0.7 F_z - sqrt(F_x^2 + F_y^2 + 25) of one contact force: value, gradient and Hessian in F."""
    Fx, Fy, Fz = F
    t2 = Fx * Fx + Fy * Fy + FRICTION_REG
    tn = np.sqrt(t2)
    t32 = tn * t2
    H = np.zeros((3, 3))
    H[0, 0] = -(Fy * Fy + FRICTION_REG) / t32
    H[0, 1] = H[1, 0] = Fx * Fy / t32
    H[1, 1] = -(Fx * Fx + FRICTION_REG) / t32
    return FRICTION_MU * Fz - tn, np.array([-Fx / tn, -Fy / tn, FRICTION_MU]), H


def stance(mode):
    return sc.mode_flags(int(mode))


def penalties(x, u, mode):
    """The penalties' share of one node's stage cost (unscaled by dt) and of its quadratic model: dict cost, q, r, Q, R."""
    o = dict(cost=0.0, q=np.zeros(NX), r=np.zeros(NU), Q=np.zeros((NX, NX)), R=np.zeros((NU, NU)))
    for j in range(NJ):
        v, d1, d2 = double_sided(x[12 + j], JOINT_LOWER[j], JOINT_UPPER[j], *POS)
        o["cost"] += v; o["q"][12 + j] += d1; o["Q"][12 + j, 12 + j] += d2
        v, d1, d2 = double_sided(u[12 + j], -JOINT_VEL[j], JOINT_VEL[j], *VEL)
        o["cost"] += v; o["r"][12 + j] += d1; o["R"][12 + j, 12 + j] += d2
    for c in range(4):
        i = 3 * c + 2
        v, d1, d2 = double_sided(u[i], 0.0, FORCE_MAX, *FORCE)
        o["cost"] += v; o["r"][i] += d1; o["R"][i, i] += d2
    for c, on in enumerate(stance(mode)):
        if not on:
            continue
        h, g, H = cone(u[3 * c:3 * c + 3])
        v, d1, d2 = relaxed_barrier(h, *CONE)
        s = slice(3 * c, 3 * c + 3)
        o["cost"] += v; o["r"][s] += d1 * g; o["R"][s, s] += d2 * np.outer(g, g) + d1 * H
        o["Q"][np.diag_indices(NX)] -= HESSIAN_SHIFT * d1; o["R"][np.diag_indices(NU)] -= HESSIAN_SHIFT * d1
    return o


def arguments(x, u, mode):
    """The 52 barrier arguments of one node: {(family, index, side): (h, delta)}; side is "lo" or "hi" (the cone's is "lo"). The cone of a
    swing contact is inactive and maps to None."""
    a = {}
    for j in range(NJ):
        a[("pos", j, "lo")] = (x[12 + j] - JOINT_LOWER[j], POS[1]); a[("pos", j, "hi")] = (JOINT_UPPER[j] - x[12 + j], POS[1])
        a[("vel", j, "lo")] = (u[12 + j] + JOINT_VEL[j], VEL[1]); a[("vel", j, "hi")] = (JOINT_VEL[j] - u[12 + j], VEL[1])
    for c, on in enumerate(stance(mode)):
        a[("force", c, "lo")] = (u[3 * c + 2], FORCE[1]); a[("force", c, "hi")] = (FORCE_MAX - u[3 * c + 2], FORCE[1])
        a[("cone", c, "lo")] = (cone(u[3 * c:3 * c + 3])[0], CONE[1]) if on else None
    assert len(a) == 52
    return a


def region(h, delta):
    return "interior" if h > delta else ("band" if h > 0.0 else "violated")


def classify(x, u, mode):
    """Region of each of the 52 arguments of one node: interior (h > delta), band (0 < h <= delta), violated (h <= 0), None if inactive."""
    return {k: (None if v is None else region(*v)) for k, v in arguments(x, u, mode).items()}


def linearisation_points(case):
    """(x, u, mode) of every node of the first SQP iteration: x0 at node 0, then xt[k], ut[k]."""
    return [(case["x0"] if k == 0 else case["xt"][k], case["ut"][k], case["mode"][k]) for k in range(len(case["ut"]))]


# ---------------------------------------------------------------- case generator
N, DT = 20, 0.02
MODES = (3, 2, 1, 0)                       # stance, left support (contacts 0, 2), right support (1, 3), flight
# band arguments at 0.7 delta: between delta / 2 and delta, where a misplaced branch point of the quadratic extension shows
H_LIMIT = {"interior": 0.15, "band": 0.07, "violated": -0.02}      # joint position (rad) / velocity (rad/s) arguments
H_FORCE = {("hi", "band"): 0.7, ("hi", "violated"): -1.0, ("lo", "band"): 0.7, ("lo", "violated"): -0.5}
H_CONE = {"interior": 6.0, "band": 3.5, "violated": -1.0}
CONE_DIRS = {"x": (1.0, 0.0), "y": (0.0, 1.0), "oblique": (np.cos(0.5), -np.sin(0.5)), "zero": (0.0, 0.0)}


def _base(mode, oracle):
    x0 = sc.INITIAL_STATE.copy()
    xr, sw, _, _ = sc.make_reference(x0, (0.2, 0.0, 0.0, 0.0), "stance", N, DT)
    md = np.full(N + 1, mode, dtype=np.int32)
    xt, ut = oracle.mpc_cold_start(N, DT, x0, md)
    return dict(x0=x0, xr=xr, sw=sw, mode=md, xt=xt, ut=ut)


def _case(name, targets, mode, oracle, edit):
    """One instance: the cold start of a constant-mode horizon, edited by edit(x0, xt, ut). targets: {(family, index, side): region} the
    name promises at every linearisation point."""
    c = _base(mode, oracle)
    edit(c["x0"], c["xt"], c["ut"])
    c.update(name=name, targets=targets)
    return c


def _set_joint(j, v):
    def edit(x0, xt, ut):
        x0[12 + j] = v; xt[:, 12 + j] = v
    return edit


def _set_input(i, v):
    def edit(x0, xt, ut):
        ut[:, i] = v
    return edit


def _set_cone(c, region_, d):
    def edit(x0, xt, ut):
        h = H_CONE[region_]
        if d == "zero":
            ut[:, 3 * c:3 * c + 3] = (0.0, 0.0, (h + np.sqrt(FRICTION_REG)) / FRICTION_MU)
        else:
            ft = np.sqrt((FRICTION_MU * ut[0, 3 * c + 2] - h) ** 2 - FRICTION_REG)
            ut[:, 3 * c] = ft * CONE_DIRS[d][0]; ut[:, 3 * c + 1] = ft * CONE_DIRS[d][1]
    return edit


def _mixed(x0, xt, ut):
    """One node per BarrierSum group with arguments on both sides of delta, and both sides of a joint's range in use at once."""
    for j, side, reg in ((0, "lo", "band"), (1, "hi", "violated"), (2, "hi", "band"), (3, "lo", "interior")):
        v = JOINT_LOWER[j] + H_LIMIT[reg] if side == "lo" else JOINT_UPPER[j] - H_LIMIT[reg]
        x0[12 + j] = v; xt[:, 12 + j] = v
    for j, side, reg in ((4, "lo", "band"), (5, "hi", "violated"), (6, "hi", "band")):
        ut[:, 12 + j] = (-1 if side == "lo" else 1) * (JOINT_VEL[j] - H_LIMIT[reg])


MIXED_TARGETS = {("pos", 0, "lo"): "band", ("pos", 1, "hi"): "violated", ("pos", 2, "hi"): "band", ("pos", 3, "lo"): "interior",
                 ("pos", 4, "lo"): "interior", ("vel", 4, "lo"): "band", ("vel", 5, "hi"): "violated", ("vel", 6, "hi"): "band",
                 ("vel", 7, "lo"): "interior"}


def make_cases(oracle):
    """Every case of the penalty envelope, in a fixed order: list of dicts (name, targets, x0, xr, sw, mode, xt, ut)."""
    cases = [_case("base/m%d" % m, {}, m, oracle, lambda *a: None) for m in MODES]
    # joint positions (on x0 and the warm start) and velocities (on ut): every joint, both sides, three regions; the whole grid in stance
    # and again in single support or flight (mode by joint)
    for kind in ("pos", "vel"):
        for modes in ((3,) * NJ, tuple((2, 1, 0)[j % 3] for j in range(NJ))):
            for j in range(NJ):
                for side in ("lo", "hi"):
                    for reg, h in H_LIMIT.items():
                        if kind == "pos":
                            edit = _set_joint(j, JOINT_LOWER[j] + h if side == "lo" else JOINT_UPPER[j] - h)
                        else:
                            edit = _set_input(12 + j, (-1 if side == "lo" else 1) * (JOINT_VEL[j] - h))
                        cases.append(_case("%s/j%d/%s/%s/m%d" % (kind, j, side, reg, modes[j]), {(kind, j, side): reg}, modes[j], oracle, edit))
    # normal forces of stance contacts: in the band below 350 N, beyond it, in (0, 1] and below 0
    for m in (3, 2, 1):
        for c in (c for c in range(4) if stance(m)[c]):
            for (side, reg), h in H_FORCE.items():
                cases.append(_case("force/c%d/%s/%s/m%d" % (c, side, reg, m), {("force", c, side): reg}, m, oracle,
                                   _set_input(3 * c + 2, h if side == "lo" else FORCE_MAX - h)))
    # friction cones of stance contacts: above delta, in the band, violated; tangential force along x, y, oblique, and none
    for m in (3, 2, 1):
        for c in (c for c in range(4) if stance(m)[c]):
            for reg in REGIONS:
                for d in CONE_DIRS:
                    cases.append(_case("cone/c%d/%s/%s/m%d" % (c, reg, d, m), {("cone", c, "lo"): reg}, m, oracle, _set_cone(c, reg, d)))
    for m in MODES:
        cases.append(_case("mixed/m%d" % m, MIXED_TARGETS, m, oracle, _mixed))
    return cases


def stack(cases):
    """(x0, x_ref, swing, mode, xt, ut) of a batch of cases."""
    return tuple(np.stack([c[k] for c in cases]) for k in ("x0", "xr", "sw", "mode", "xt", "ut"))


def family(case):
    return case["name"].split("/")[0]
