"""The joint models of the plant restated in numpy (hunter_b200.h, "joint models"): each robot's range stops and friction loss as
generalised forces on its joints, in the order the header pins, for episode_ref.plant_numpy and bridge_ref.plant_bridged through an oracle
wrapper, and for episode_ref.stepwise through a wrapper context whose every plant step passes the records."""
import numpy as np

import hunter_bipedal_control_b200 as hb
from bridge_ref import _rows
from link_ref import LinkLoop, padded as padded_links

NJ = 10


def disabled(B=1):
    """B records that act on nothing: no friction loss, no bound (the gains are arbitrary and nonzero)."""
    return hb.make_joint_models(B, friction_loss=0.0, lower=-np.inf, upper=np.inf, stop_stiffness=1e4, stop_damping=50.0)


inf, nan = float("inf"), float("nan")
# One broken range of the header per entry: (field, joint or None, value)
BAD = [("friction_loss", 3, nan), ("friction_loss", 0, -0.1), ("friction_loss", 9, inf), ("friction_velocity", None, 0.0),
       ("friction_velocity", None, -1e-3), ("friction_velocity", None, nan), ("friction_velocity", None, inf), ("lower", 2, nan),
       ("upper", 5, nan), ("lower", 4, 1.1), ("lower", 1, 2.0), ("upper", 0, -inf), ("lower", 7, inf), ("stop_stiffness", None, -1.0),
       ("stop_stiffness", None, nan), ("stop_stiffness", None, inf), ("stop_damping", None, -1e-9), ("stop_damping", None, nan),
       ("stop_damping", None, inf)]


def bad_records():
    """Two-record arrays whose second record breaks one range of the header, one per BAD entry."""
    out = []
    for field, j, v in BAD:
        recs = hb.make_joint_models(2)
        if j is None:
            setattr(recs[1], field, v)
        else:
            getattr(recs[1], field)[j] = v
        out.append(recs)
    return out


def friction(m, j, v):
    """The friction loss of joint j of record m at velocity v: -f_j clamp(v / v_s, -1, 1)."""
    return -m.friction_loss[j] * min(1.0, max(-1.0, v / m.friction_velocity))


def stop(m, j, q, v, mjj):
    """The range stop of joint j of record m at q, v, with mjj the joint's diagonal of M + armature: never pulling towards the stop."""
    if q > m.upper[j]:
        return min(0.0, -mjj * (m.stop_stiffness * (q - m.upper[j]) + m.stop_damping * v))
    if q < m.lower[j]:
        return max(0.0, mjj * (m.stop_stiffness * (m.lower[j] - q) - m.stop_damping * v))
    return 0.0


def joint_forces(m, q, v, M, armature):
    """The joint model's generalised forces on the 16 coordinates at q, v (the base rows 0), with M the substep's mass matrix."""
    out = np.zeros(16)
    for j in range(NJ):
        k = 6 + j
        out[k] = friction(m, j, v[k]) + stop(m, j, q[k], v[k], M[k, k] + armature)
    return out


def stable(prm, records):
    """The stability rule: h (joint_damping + f_j / v_s) <= joint_armature on every joint of every record."""
    h = prm.dt / prm.substeps
    return all(h * (prm.joint_damping + r.friction_loss[j] / r.friction_velocity) <= prm.joint_armature for r in records for j in range(NJ))


class JointOracle:
    """An oracle (oracle.hbo, or link_ref.LinkOracle) whose rbd(q, v) carries the joint model `record` in nle: plant_numpy and
    plant_bridged solve (M + A) qdd = rhs - nle, so subtracting the joint forces from nle adds them to the right-hand side. A payload
    changes only M's base block, so the joint diagonal the stop reads is the oracle's."""

    def __init__(self, oracle, record, armature):
        self._oracle, self._record, self._armature = oracle, record, armature

    def __getattr__(self, name):
        return getattr(self._oracle, name)

    def rbd(self, q, v):
        r = self._oracle.rbd(q, v)
        if self._record is not None:
            r["nle"] = r["nle"] - joint_forces(self._record, np.asarray(q, dtype=float), np.asarray(v, dtype=float), r["M"], self._armature)
        return r


def padded(models, B):
    """The B records of the setting models: models, then disabled records beyond them (the plant without a record, bit for bit)."""
    d = disabled()[0]
    return (hb.HbJointModel * B)(*[models[i] if i < len(models) else d for i in range(B)])


class JointLoop(LinkLoop):
    """The context episode_ref.stepwise runs on to restate an episode with joint models set (`models`, the records set on ctx): every
    plant step is the one with joints=, padded with disabled records, and with the link variations `links` (the default record when
    None); `bridges` as under LinkLoop. Every other call goes to ctx."""

    def __init__(self, ctx, models, links=None, bridges=None, default_limit=None):
        super().__init__(ctx, links if links is not None else (hb.HbLinkVariation * 0)(), bridges, default_limit)
        self._models = models

    def sim_step(self, rbd, tau, params=None, wrench=None, variation=None, terrain=None):
        B = rbd.shape[0]
        lk, jm = padded_links(self._links, B), padded(self._models, B)
        nxt, cf, fl = np.zeros((B, 32)), np.zeros((B, 12)), np.zeros((B, 4), dtype=np.uint8)
        for lo, hi, mb in self._groups(B):
            kw = dict(wrench=None if wrench is None else wrench[lo:hi], variation=_rows(variation, lo, hi), terrain=_rows(terrain, lo, hi),
                      links=_rows(lk, lo, hi), joints=_rows(jm, lo, hi))
            if mb is None:
                nxt[lo:hi], cf[lo:hi], fl[lo:hi] = self._ctx.sim_step(rbd[lo:hi], tau[lo:hi], params, **kw)
            else:
                nxt[lo:hi], cf[lo:hi], fl[lo:hi], tau[lo:hi] = self._ctx.sim_step(rbd[lo:hi], self._mcmd[lo:hi], params, bridge=mb,
                                                                                  limits=self._lim[lo:hi], **kw)
        return nxt, cf, fl
