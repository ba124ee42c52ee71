"""The varied plant restated for its tests (test_gpu_rollout_plant_variations.py), on top of the shared episode reference episode_ref.py:
the payload terms and the varied plant step in numpy, and the varied episode as episode_ref's loop of public calls with every plant step
taken on the robots' varied plants."""
import numpy as np

import hunter_bipedal_control_b200 as hb
from episode_ref import T, stepwise

G = 9.81


def payload_terms(q, v, variation):
    """The payload of a plant variation in the base coordinates (p, zyx) of q, v: (M_p, nle_p), the 6 x 6 base block it adds to M and the 6
    entries it adds to nle, from the documented formulas: with omega = T zyx_dot, r = R c and I_w = R I_c R', column k of M_p is
    [F; T' n] for F = m (pdd + omega_dot x r), n = I_w omega_dot + r x F at a unit acceleration of coordinate k and v = 0; nle_p is the
    same with omega_dot0 = (omega_1 x a_pitch) dpitch + (omega_2 x a_roll) droll, F = m (omega_dot0 x r + omega x (omega x r)) + m g e_z,
    n = I_w omega_dot0 + omega x I_w omega + r x F."""
    from oracle import refs
    m = variation.payload_mass
    c = np.array(variation.payload_com[:]); Ic = np.array(variation.payload_inertia[:]).reshape(3, 3)
    R, Tm = refs.rot_zyx(q[3:6]), T(q[3:6])
    r, Iw = R @ c, R @ Ic @ R.T
    M = np.zeros((6, 6))
    for k in range(6):
        a = np.zeros(6); a[k] = 1.0
        wd = Tm @ a[3:]
        F = m * (a[:3] + np.cross(wd, r))
        M[:, k] = np.r_[F, Tm.T @ (Iw @ wd + np.cross(r, F))]
    dz = v[3:6]
    w1 = Tm[:, 0] * dz[0]; w2 = w1 + Tm[:, 1] * dz[1]; w = Tm @ dz
    wd0 = np.cross(w1, Tm[:, 1]) * dz[1] + np.cross(w2, Tm[:, 2]) * dz[2]
    F = m * (np.cross(wd0, r) + np.cross(w, np.cross(w, r))) + m * G * np.array([0.0, 0.0, 1.0])
    n = Iw @ wd0 + np.cross(w, Iw @ w) + np.cross(r, F)
    return M, np.r_[F, Tm.T @ n]


def plant_numpy_varied(oracle, rbd, tau, prm, variation, wrench=None):
    """One plant step of one robot on its varied plant: episode_ref.plant_numpy with the ground stiffness, damping and friction scaled, the
    joint torques scaled by the motor strengths and, with a payload, payload_terms added to M and nle. Returns (rbd_next, contact forces of
    the last substep)."""
    from oracle import refs
    q = np.concatenate([rbd[3:6], rbd[0:3], rbd[6:16]])
    v = np.concatenate([rbd[19:22], refs.euler_rates_from_global(rbd[0:3], rbd[16:19]), rbd[22:32]])
    h = prm.dt / prm.substeps
    k_g = prm.ground_stiffness * variation.stiffness_scale
    d_g = prm.ground_damping * variation.damping_scale
    mu = prm.friction_mu * variation.friction_scale
    tau = np.array(variation.motor_strength[:]) * tau
    F = np.zeros(12)
    for _ in range(prm.substeps):
        r = oracle.rbd(q, v)
        M, nle = r["M"].copy(), r["nle"].copy()
        if variation.payload_mass > 0:
            Mp, nlep = payload_terms(q, v, variation)
            M[:6, :6] += Mp; nle[:6] += nlep
        cvel = r["J"] @ v
        F = np.zeros(12)
        for c in range(4):
            depth = prm.ground_height - r["cpos"][3 * c + 2]
            if depth > 0:
                fz = max(0.0, k_g * depth - d_g * cvel[3 * c + 2])
                ft = -prm.tangential_damping * cvel[3 * c:3 * c + 2]
                n = np.linalg.norm(ft)
                if n > mu * fz:
                    ft = ft * (mu * fz / n if n > 0 else 0.0)
                F[3 * c:3 * c + 3] = [ft[0], ft[1], fz]
        rhs = np.concatenate([np.zeros(6), tau - prm.joint_damping * v[6:]]) + r["J"].T @ F - nle
        if wrench is not None:
            rhs = rhs + np.concatenate([wrench[:3], T(q[3:6]).T @ wrench[3:], np.zeros(10)])
        qdd = np.linalg.solve(M + np.diag(np.r_[np.zeros(6), np.full(10, prm.joint_armature)]), rhs)
        v = v + h * qdd
        q = q + h * v
    out = np.zeros(32)
    out[0:3] = q[3:6]; out[3:6] = q[0:3]; out[6:16] = q[6:]
    out[16:19] = refs.global_from_euler_rates(q[3:6], v[3:6]); out[19:22] = v[0:3]; out[22:32] = v[6:]
    return out, F


class _VariedPlant:
    """A context whose plant steps run on the given varied plants (Context.sim_step with variation=; instances beyond them get the default
    variation); every other call is the context's own."""

    def __init__(self, ctx, variations, B):
        self._ctx = ctx
        self._v = (hb.HbPlantVariation * B)(*[variations[i] if i < len(variations) else hb.default_plant_variation() for i in range(B)])

    def sim_step(self, rbd, tau, params=None, wrench=None):
        return self._ctx.sim_step(rbd, tau, params, wrench=wrench, variation=self._v)

    def __getattr__(self, name):
        return getattr(self._ctx, name)


def stepwise_varied(ctx, rbd0, gaits, cmd_vels, n_ticks, prm, log_every, variations, ep=None, est=None, pushes=None):
    """episode_ref.stepwise with every plant step on the varied plants set on ctx (hb_sim_step_varied)."""
    return stepwise(_VariedPlant(ctx, variations, rbd0.shape[0]), rbd0, gaits, cmd_vels, n_ticks, prm, log_every, ep, est, pushes)
