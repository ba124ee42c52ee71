"""Link variations (hb_link_variation, hunter_b200.h) restated for their tests (test_link_variations_host.py,
test_gpu_rollout_link_variations.py): the bodies of a record, the rigid-body terms M(q) and nle(q, v) on any bodies by recursive
Newton-Euler in numpy, the oracle's terms with a record's changes added (LinkOracle, which episode_ref.plant_numpy and
bridge_ref.plant_bridged take in place of the oracle), and LinkLoop, under which episode_ref.stepwise runs every plant step on the records."""
import ctypes as C

import numpy as np

import hunter_bipedal_control_b200 as hb
from bridge_ref import BridgeLoop, _rows

G = 9.81


def _header(name, shape):
    from oracle import refs
    return np.array(refs._header_array(name)).reshape(shape)


NB = 11
PARENT = [-1, 0, 1, 2, 3, 4, 0, 6, 7, 8, 9]
XYZ, AXIS = _header("HB_JOINT_XYZ", (NB, 3)), _header("HB_JOINT_AXIS", (NB, 3))
MASS, COM, INERTIA = _header("HB_BODY_MASS", (NB,)), _header("HB_BODY_COM", (NB, 3)), _header("HB_BODY_INERTIA", (NB, 3, 3))
GROUPS = {"hips": [1, 2, 6, 7], "thighs": [3, 8], "shanks_feet": [4, 5, 9, 10], "legs": list(range(1, 11))}


def bodies(record=None):
    """(m (11,), c (11, 3), I (11, 3, 3)) of the record's bodies, each value one rounded product or sum as documented; None: the model's."""
    if record is None:
        return MASS.copy(), COM.copy(), INERTIA.copy()
    r = np.ctypeslib.as_array((hb.HbLinkVariation * 1)(record))[0]
    return r["mass_scale"] * MASS, COM + r["com_shift"], r["inertia_scale"][:, None, None] * INERTIA


def _rot(axis, th):
    """Rotations about the unit axis by the angles th (L,): (L, 3, 3)."""
    K = np.array([[0.0, -axis[2], axis[1]], [axis[2], 0.0, -axis[0]], [-axis[1], axis[0], 0.0]])
    s, c = np.sin(th)[:, None, None], np.cos(th)[:, None, None]
    return np.eye(3) + s * K + (1.0 - c) * (K @ K)


def _T(zyx):
    sz, cz, sy, cy = np.sin(zyx[0]), np.cos(zyx[0]), np.sin(zyx[1]), np.cos(zyx[1])
    return np.array([[0.0, -sz, cz * cy], [0.0, cz, sz * cy], [1.0, 0.0, -sy]])


def _base(q, v, a):
    """The base of each lane: orientation R0, T, angular velocity, angular acceleration and origin acceleration (lanes of v, a: (L, 16))."""
    from oracle import refs
    R0, T = refs.rot_zyx(q[3:6]), _T(q[3:6])
    d = v[:, 3:6]
    w1 = d[:, :1] * T[:, 0]; w2 = w1 + d[:, 1:2] * T[:, 1]
    w0 = d @ T.T
    wd0 = a[:, 3:6] @ T.T + np.cross(w1, T[:, 1]) * d[:, 1:2] + np.cross(w2, T[:, 2]) * d[:, 2:3]
    return R0, T, w0, wd0, a[:, 0:3].copy()


def rnea(q, v, a, gravity, body=None):
    """tau = M(q) a + C(q, v) v (+ g(q) with gravity) for the lanes v, a (L, 16) on the bodies body = (m, c, I) (None: the model's):
    recursive Newton-Euler over the tree, world axes, moments about each body's origin. Returns (L, 16)."""
    m, c, I = bodies() if body is None else body
    L = v.shape[0]
    R0, T, w0, wd0, pd0 = _base(q, v, a)
    R = [None] * NB; w = [None] * NB; wd = [None] * NB; pd = [None] * NB; ax = [None] * NB; d = [None] * NB
    R[0], w[0], wd[0], pd[0] = np.broadcast_to(R0, (L, 3, 3)), w0, wd0, pd0
    for b in range(1, NB):
        P = PARENT[b]
        d[b] = R[P] @ XYZ[b]
        ax[b] = R[P] @ AXIS[b]
        pd[b] = pd[P] + np.cross(wd[P], d[b]) + np.cross(w[P], np.cross(w[P], d[b]))
        R[b] = R[P] @ _rot(AXIS[b], np.full(L, q[5 + b]))
        wd[b] = wd[P] + ax[b] * a[:, 5 + b:6 + b] + np.cross(w[P], ax[b]) * v[:, 5 + b:6 + b]
        w[b] = w[P] + ax[b] * v[:, 5 + b:6 + b]
    f, n = [None] * NB, [None] * NB
    for b in range(NB):
        r = R[b] @ c[b]
        F = m[b] * (pd[b] + np.cross(wd[b], r) + np.cross(w[b], np.cross(w[b], r)))
        if gravity:
            F = F + m[b] * G * np.array([0.0, 0.0, 1.0])
        Iw = R[b] @ I[b] @ np.swapaxes(R[b], 1, 2)
        n[b] = np.einsum("lij,lj->li", Iw, wd[b]) + np.cross(w[b], np.einsum("lij,lj->li", Iw, w[b])) + np.cross(r, F)
        f[b] = F
    tau = np.zeros((L, 16))
    for b in range(NB - 1, 0, -1):                     # children before parents
        tau[:, 5 + b] = np.einsum("li,li->l", ax[b], n[b])
        P = PARENT[b]
        f[P] = f[P] + f[b]; n[P] = n[P] + n[b] + np.cross(d[b], f[b])
    tau[:, 0:3] = f[0]
    tau[:, 3:6] = n[0] @ T
    return tau


def terms(q, v, body=None):
    """(M (16, 16), nle (16,)) on the bodies body (None: the model's): M's columns from unit accelerations, nle with v and gravity."""
    M = rnea(q, np.zeros((16, 16)), np.eye(16), False, body).T
    nle = rnea(q, np.asarray(v, dtype=float)[None], np.zeros((1, 16)), True, body)[0]
    return M, nle


def changes(q, v, record):
    """(dM, dnle): the record's bodies' terms minus the model's."""
    M1, n1 = terms(q, v, bodies(record))
    M0, n0 = terms(q, v)
    return M1 - M0, n1 - n0


def body_motion(q, v, body=None):
    """Per body: the world CoM position (11, 3), CoM velocity (11, 3), angular velocity (11, 3) and world inertia about the CoM (11, 3, 3)."""
    from oracle import refs
    m, c, I = bodies() if body is None else body
    R = [refs.rot_zyx(q[3:6])] + [None] * (NB - 1)
    p = [np.asarray(q[0:3], dtype=float)] + [None] * (NB - 1)
    w = [_T(q[3:6]) @ v[3:6]] + [None] * (NB - 1)
    vo = [np.asarray(v[0:3], dtype=float)] + [None] * (NB - 1)
    for b in range(1, NB):
        P = PARENT[b]
        dd = R[P] @ XYZ[b]
        p[b] = p[P] + dd; vo[b] = vo[P] + np.cross(w[P], dd)
        R[b] = R[P] @ _rot(AXIS[b], np.array([q[5 + b]]))[0]
        w[b] = w[P] + (R[P] @ AXIS[b]) * v[5 + b]
    pc = np.array([p[b] + R[b] @ c[b] for b in range(NB)])
    vc = np.array([vo[b] + np.cross(w[b], R[b] @ c[b]) for b in range(NB)])
    return pc, vc, np.array(w), np.array([R[b] @ I[b] @ R[b].T for b in range(NB)])


class LinkOracle:
    """The oracle (oracle.hbo) with the rigid-body terms of a record: rbd(q, v) is the oracle's, with M and nle changed by changes(q, v,
    record). The default record changes nothing, so it is the oracle's bit for bit."""

    def __init__(self, oracle, record):
        self._oracle, self._record = oracle, record

    def __getattr__(self, name):
        return getattr(self._oracle, name)

    def rbd(self, q, v):
        r = self._oracle.rbd(q, v)
        if self._record is not None:
            dM, dn = changes(np.asarray(q, dtype=float), np.asarray(v, dtype=float), self._record)
            r["M"] = r["M"] + dM; r["nle"] = r["nle"] + dn
        return r


def padded(links, B):
    """The B records of the setting links: links, then the default record beyond them."""
    d = hb.default_link_variation()
    return (hb.HbLinkVariation * B)(*[links[i] if i < len(links) else d for i in range(B)])


class LinkLoop(BridgeLoop):
    """The context episode_ref.stepwise runs on to restate an episode with link variations set (`links`, the records set on ctx): every
    plant step is the one with links=, padded with the default record; with `bridges` (the motor bridges set on ctx) the bridged robots
    read, actuate and step through the calls with bridge=, as under BridgeLoop. Every other call goes to ctx (which may be a TeleopLoop)."""

    def __init__(self, ctx, links, bridges=None, default_limit=None):
        super().__init__(ctx, bridges if bridges is not None else (hb.HbMotorBridge * 0)(),
                         default_limit if default_limit is not None else hb.default_rollout_params().torque_limit)
        self._links = links

    def sim_step(self, rbd, tau, params=None, wrench=None, variation=None, terrain=None):
        B = rbd.shape[0]
        lk = padded(self._links, B)
        nxt, cf, fl = np.zeros((B, 32)), np.zeros((B, 12)), np.zeros((B, 4), dtype=np.uint8)
        for lo, hi, mb in self._groups(B):
            kw = dict(wrench=None if wrench is None else wrench[lo:hi], variation=_rows(variation, lo, hi), terrain=_rows(terrain, lo, hi),
                      links=_rows(lk, lo, hi))
            if mb is None:
                nxt[lo:hi], cf[lo:hi], fl[lo:hi] = self._ctx.sim_step(rbd[lo:hi], tau[lo:hi], params, **kw)
            else:
                nxt[lo:hi], cf[lo:hi], fl[lo:hi], tau[lo:hi] = self._ctx.sim_step(rbd[lo:hi], self._mcmd[lo:hi], params, bridge=mb,
                                                                                  limits=self._lim[lo:hi], **kw)
        return nxt, cf, fl
