"""The robot's state envelope for the MPC solve's tests: named axes of states and inputs well outside the near-nominal box of
scenarios.random_initial_states, whole solve cases on them, the two exact transforms of a solve case and a central-difference Jacobian with
Richardson extrapolation. Plain numpy on top of scenarios and the float64 oracle; no device code.

State x = [hbar (linear 0:3, angular 3:6, normalised by the mass), base position 6:9, ZYX Euler angles 9:12 (yaw, pitch, roll), joints
12:22]; input u = [contact forces 0:12 (four contacts, x y z each), joint velocities 12:22].

Each axis sits alone on the default pose (every other coordinate as in scenarios.INITIAL_STATE, the weight spread over the four contacts,
joints at rest); MIXED draws every coordinate from the whole envelope at once. The axes reach:
  attitude  roll and pitch to +-1.4 rad, and combined yaw / pitch / roll
  yaw       +-pi, 2 pi k + small offsets (k to 159), +-1e3 rad (an estimated episode's unwrapped yaw grows without bound)
  position  1e3 m along x, y and z
  momentum  linear and angular hbar to +-1, ten times random_initial_states' range
  joints    every joint at its lower and at its upper limit, in turn and all together; both knees at 0 and at refs.singular_knee
  joint_velocity  +-40 rad/s, one joint at a time and all together (episodes command up to 36 rad/s)
  force     no force at all, 3 m g on one contact, 3 m g spread with tangential parts
"""
import numpy as np

from hunter_bipedal_control_b200 import scenarios as sc
from oracle import refs as R

X0 = sc.INITIAL_STATE.copy()
WEIGHT = sc.TOTAL_MASS * 9.81
LOWER, UPPER = sc.JOINT_LOWER, sc.JOINT_UPPER
KNEES = (3, 8)                                   # joint indices of the left and right knee (limits [0, 1.5])
GAITS = ("stance", "trot", "standing_trot", "flying_trot")
BOX = dict(attitude=0.1, momentum=0.1, joints=0.05, position=0.05)   # random_initial_states' half-widths (yaw is drawn in [-pi, pi])
ENVELOPE = dict(attitude=1.4, yaw=1e3, position=1e3, momentum=1.0, joint_velocity=40.0, force=3.0 * WEIGHT)


def stance_input():
    u = np.zeros(22)
    u[[2, 5, 8, 11]] = WEIGHT / 4
    return u


def singular_knees():
    """The knee angle of each leg at the default pose where its foot wrench matrix is closest to singular (refs.singular_knee)."""
    q = np.concatenate([X0[6:9], X0[9:12], X0[12:]])
    return [R.singular_knee(leg, q) for leg in (0, 1)]


def _x(**kw):
    x = X0.copy()
    for k, v in kw.items():
        x[dict(yaw=9, pitch=10, roll=11)[k]] = v
    return x


def axis_points(name):
    """[(label, x, u)] of one axis, alone on the default pose."""
    u0 = stance_input()
    out = []
    if name == "attitude":
        for p in (0.5, 1.0, 1.2, 1.4):
            out += [("pitch %+g" % s, _x(pitch=s), u0) for s in (p, -p)]
        out += [("roll %+g" % s, _x(roll=s), u0) for s in (0.8, -0.8, 1.4, -1.4)]
        for y, p, r in ((2.0, 1.2, -0.8), (-3.0, -1.4, 1.0), (0.7, 1.4, 1.4), (-1.0, -0.9, -1.4)):
            out.append(("ypr %g %g %g" % (y, p, r), _x(yaw=y, pitch=p, roll=r), u0))
    elif name == "yaw":
        for y in (np.pi, -np.pi, 2 * np.pi + 1e-3, 20 * np.pi - 1e-3, 2 * np.pi * 159 + 0.3, -2 * np.pi * 37 + 0.5, 1e3, -1e3):
            out.append(("yaw %.6g" % y, _x(yaw=y), u0))
    elif name == "position":
        for p in ((1e3, 0, 0.63), (0, -1e3, 0.63), (-1e3, 1e3, 0.63), (1e3, 1e3, 1e3)):
            x = X0.copy(); x[6:9] = p
            out.append(("position %g %g %g" % p, x, u0))
    elif name == "momentum":
        for i in range(6):
            for s in (1.0, -1.0):
                x = X0.copy(); x[i] = s
                out.append(("hbar[%d] %+g" % (i, s), x, u0))
        x = X0.copy(); x[0:6] = [1, -1, 1, -1, 1, -1]
        out.append(("hbar all", x, u0))
    elif name == "joints":
        for j in range(10):
            for side, lim in (("lower", LOWER), ("upper", UPPER)):
                x = X0.copy(); x[12 + j] = lim[j]
                out.append(("joint %d %s" % (j, side), x, u0))
        for side, lim in (("lower", LOWER), ("upper", UPPER)):
            x = X0.copy(); x[12:] = lim
            out.append(("all joints %s" % side, x, u0))
        x = X0.copy(); x[12 + np.array(KNEES)] = 0.0
        out.append(("knees 0", x, u0))
        x = X0.copy(); x[12 + np.array(KNEES)] = singular_knees()
        out.append(("knees singular", x, u0))
    elif name == "joint_velocity":
        for j in range(10):
            for s in (40.0, -40.0):
                u = u0.copy(); u[12 + j] = s
                out.append(("qdot %d %+g" % (j, s), X0, u))
        u = u0.copy(); u[12:] = 40.0 * np.array([1, -1] * 5)
        out.append(("qdot all", X0, u))
    elif name == "force":
        out.append(("no force", X0, np.zeros(22)))
        for c in range(4):
            u = np.zeros(22); u[3 * c + 2] = 3 * WEIGHT
            out.append(("3mg on contact %d" % c, X0, u))
        u = np.zeros(22); u[:12] = np.tile([0.3, -0.2, 1.0], 4) * 3 * WEIGHT / 4
        out.append(("3mg spread", X0, u))
    else:
        raise KeyError(name)
    return out


AXES = ("attitude", "yaw", "position", "momentum", "joints", "joint_velocity", "force")


def mixed_points(n, seed):
    """n (label, x, u) with every coordinate drawn from the whole envelope at once."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        x = X0.copy(); u = np.zeros(22)
        x[0:6] = rng.uniform(-1, 1, 6)
        x[6:8] = rng.uniform(-1e3, 1e3, 2); x[8] = rng.uniform(0.3, 1e3)
        x[9] = rng.uniform(-1e3, 1e3); x[10:12] = rng.uniform(-1.4, 1.4, 2)
        x[12:] = rng.uniform(LOWER, UPPER)
        u[:12] = rng.uniform(-0.5, 1.0, 12) * 3 * WEIGHT / 4
        u[12:] = rng.uniform(-10, 10, 10)
        out.append(("mixed %d" % i, x, u))
    return out


def all_points(n_mixed=8, seed=11):
    """{axis: [(label, x, u)]}: every axis and the mixed sample."""
    pts = {a: axis_points(a) for a in AXES}
    pts["mixed"] = mixed_points(n_mixed, seed)
    return pts


# ------------------------------------------------------------------------------------------------------------ solve cases
def solve_case(x0, gait, N, dt, cmd_vel=(0.3, 0.0, 0.0, 0.2), oracle=None, u_warm=None):
    """(x0, x_ref, swing, mode, xt, ut) of one instance: the reference scenarios.make_reference builds from x0, and the oracle's cold
    start; u_warm (22,) replaces every input sample of the warm start (inputs far from the cold start's)."""
    x_ref, swing, mode, _ = sc.make_reference(x0, cmd_vel, gait, N, dt)
    if oracle is None:
        from oracle import hbo as oracle
    xt, ut = oracle.mpc_cold_start(N, dt, x0, mode)
    if u_warm is not None:
        ut[:] = u_warm
    return x0.copy(), x_ref, swing, mode, xt, ut


def _case_states():
    """[(axis, label, x0, u_warm)]: the axis values the solve cases start at (u_warm None: the cold start's inputs)."""
    out = []
    for lab, x, _ in axis_points("attitude"):
        if lab in ("pitch +1.2", "pitch -1.2", "pitch +1.4", "roll +0.8", "roll -1.4", "ypr 2 1.2 -0.8", "ypr -3 -1.4 1"):
            out.append(("attitude", lab, x, None))
    for lab, x, _ in axis_points("yaw"):
        out.append(("yaw", lab, x, None))
    for lab, x, _ in axis_points("position")[:3]:
        out.append(("position", lab, x, None))
    for lab, x, _ in axis_points("momentum"):
        if lab in ("hbar[0] +1", "hbar[1] -1", "hbar[2] +1", "hbar[3] +1", "hbar[5] -1", "hbar all"):
            out.append(("momentum", lab, x, None))
    for lab, x, _ in axis_points("joints"):
        if lab.startswith(("all", "knees")) or lab in ("joint 2 upper", "joint 7 lower", "joint 4 upper", "joint 9 lower"):
            out.append(("joints", lab, x, None))
    for lab, _, u in axis_points("joint_velocity"):
        if lab in ("qdot 3 +40", "qdot 8 -40", "qdot all"):
            out.append(("joint_velocity", lab, X0, u))
    for lab, _, u in axis_points("force"):
        if lab in ("no force", "3mg on contact 0", "3mg on contact 3", "3mg spread"):
            out.append(("force", lab, X0, u))
    rng = np.random.default_rng(23)
    for i in range(6):
        x = X0.copy()
        x[0:6] = rng.uniform(-1, 1, 6)
        x[6:8] = rng.uniform(-1e3, 1e3, 2); x[9] = rng.uniform(-1e3, 1e3); x[10:12] = rng.uniform(-1.2, 1.2, 2)
        x[12:] = rng.uniform(LOWER, UPPER)
        out.append(("mixed", "mixed %d" % i, x, None))
    return out


def solve_cases(N, dt, oracle=None):
    """[(axis, label, gait, case)]: every solve state with the gaits in turn, so that each axis meets several gaits and all four occur."""
    out = []
    for i, (axis, lab, x0, uw) in enumerate(_case_states()):
        g = GAITS[i % len(GAITS)]
        out.append((axis, lab, g, solve_case(x0, g, N, dt, oracle=oracle, u_warm=uw)))
    return out


def stack(cases):
    """(x0, x_ref, swing, mode, xt, ut) of a batch from a list of single-instance cases."""
    return tuple(np.stack(a) for a in zip(*cases))


def backtracking_case(x0, gait, N, dt, seed, oracle, amplitude=1.0):
    """The poor warm start of the line-search tests on an envelope state: three oracle iterations from the cold start, then the joint
    trajectory pushed off by uniform(-amplitude, amplitude), so that the next iteration's line search evaluates the flow map at trial
    points far from the linearisation."""
    x0, xr, sw, md, xt, ut = solve_case(x0, gait, N, dt, oracle=oracle)
    for _ in range(3):
        xt, ut, _ = oracle.mpc_iteration(N, dt, x0, xr, sw, md, xt, ut)
    xt = xt.copy()
    xt[1:, 12:] += np.random.default_rng(seed).uniform(-amplitude, amplitude, (N, 10))
    return x0, xr, sw, md, xt, ut


# ------------------------------------------------------------------------------------------------------------ exact transforms
def yaw_turn(case, k):
    """The solve case with yaw + 2 pi k in x0, the reference and the warm start: the same problem, since yaw enters the model only
    through its sine and cosine."""
    x0, xr, sw, md, xt, ut = (np.array(a, copy=True) for a in case)
    c = 2 * np.pi * k
    x0[..., 9] += c; xr[..., 9] += c; xt[..., 9] += c
    return x0, xr, sw, md, xt, ut


def yaw_turn_back(xt, k):
    xt = np.array(xt, copy=True)
    xt[..., 9] -= 2 * np.pi * k
    return xt


def shift(case, d):
    """The solve case moved horizontally by d = (dx, dy): x0, the reference, the swing references' px / py and the warm start; the
    model is invariant under horizontal translation (and the stance feet's height constraint sees only z)."""
    x0, xr, sw, md, xt, ut = (np.array(a, copy=True) for a in case)
    d = np.asarray(d, dtype=np.float64)
    x0[..., 6:8] += d; xr[..., 6:8] += d; xt[..., 6:8] += d
    for c in range(4):
        sw[..., 6 * c:6 * c + 2] += d
    return x0, xr, sw, md, xt, ut


def shift_back(xt, d):
    xt = np.array(xt, copy=True)
    xt[..., 6:8] -= np.asarray(d, dtype=np.float64)
    return xt


# ------------------------------------------------------------------------------------------------------------ differences
def richardson_jacobian(fn, z, h):
    """d fn / d z by central differences with one Richardson step: (4 D(h / 2) - D(h)) / 3 with D(h) = (fn(z + h e) - fn(z - h e)) / 2h,
    error O(h^4) instead of O(h^2), so h can be large enough that rounding (eps |fn| / h) stays small too. h: scalar or per coordinate.
    The divisor is the distance between the two points as represented, so a coordinate of 1e3 (yaw, position) loses nothing to the
    rounding of z +- h."""
    z = np.asarray(z, dtype=np.float64)
    hs = np.broadcast_to(np.asarray(h, dtype=np.float64), z.shape)
    cols = []
    for k in range(z.size):
        def D(step):
            zp, zm = z.copy(), z.copy()
            zp[k] += step; zm[k] -= step
            return (np.asarray(fn(zp)) - np.asarray(fn(zm))) / (zp[k] - zm[k])
        cols.append((4 * D(hs[k] / 2) - D(hs[k])) / 3)
    return np.stack(cols, axis=-1)


def rounding_floor(run, case, reps=8, seed=0):
    """How far float64 rounding alone moves a solve: the largest relative change (x, u) of run(case) -> (xt, ut, ...) when x0 and the warm
    start are perturbed by one unit in the last place at random, over `reps` draws. A well-conditioned case moves by ~1e-13; an
    ill-conditioned one (near the vertical, or where hbar is far from what the joints can absorb) by up to 1e-2, whatever the size of the
    perturbation below 1e-13, so no float64 implementation can agree with another more closely than this."""
    rng = np.random.default_rng(seed)
    ref = run(case)
    w = np.zeros(2)
    for _ in range(reps):
        d = [np.array(a, copy=True) for a in case]
        for k in (0, 4, 5):
            d[k] = d[k] * (1 + np.finfo(np.float64).eps * rng.choice([-1.0, 1.0], d[k].shape))
        out = run(tuple(d))
        w = np.maximum(w, (rel(out[0], ref[0]), rel(out[1], ref[1])))
    return w


def rel(a, b):
    """max |a - b| / max(1, |b|): the suite's relative measure."""
    return np.abs(np.asarray(a) - b).max() / max(1.0, np.abs(b).max())


def bounds_of(x, u):
    """The extremes a set of states / inputs reaches, per envelope coordinate: |roll|, |pitch|, |yaw|, |horizontal position|, base height,
    |linear hbar|, |angular hbar|, joints (min, max), |joint velocity|, max normal force, max |force|."""
    x = np.asarray(x).reshape(-1, 22); u = np.asarray(u).reshape(-1, 22)
    f = u[:, :12].reshape(-1, 4, 3)
    return dict(roll=np.abs(x[:, 11]).max(), pitch=np.abs(x[:, 10]).max(), yaw=np.abs(x[:, 9]).max(), position=np.abs(x[:, 6:8]).max(),
                height=(x[:, 8].min(), x[:, 8].max()), linear=np.abs(x[:, 0:3]).max(), angular=np.abs(x[:, 3:6]).max(),
                joints=(x[:, 12:].min(axis=0), x[:, 12:].max(axis=0)), joint_velocity=np.abs(u[:, 12:]).max(),
                normal_force=f[:, :, 2].max(), force=np.abs(f).max())
