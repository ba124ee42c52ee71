"""The terrain restated for its tests (test_gpu_rollout_terrain.py), on top of the shared episode reference episode_ref.py and the varied
plant's plant_variation_ref.py: the documented height and gradient of a height field, the plant step on a terrain in numpy, and the
terrain episode as episode_ref's loop of public calls with every plant step taken on the robots' terrains."""
import math

import numpy as np

import hunter_bipedal_control_b200 as hb
from episode_ref import T, stepwise
from plant_variation_ref import payload_terms


def _axis(x, origin, spacing, n):
    """(cell index, fraction, clamped) of world coordinate x along one grid axis; NaN clamps to 0 as the kernel does."""
    u = (x - origin) / spacing
    clamped = False
    if not u >= 0.0:
        u, clamped = 0.0, True
    elif u > n - 1:
        u, clamped = float(n - 1), True
    i = min(int(math.floor(u)), n - 2)
    return i, u - i, clamped


def terrain_height(t, x, y):
    """(h, g_x, g_y) of the HbTerrain t at world (x, y), as hunter_b200.h documents it."""
    i, a, cx = _axis(x, t.origin[0], t.spacing, t.nx)
    j, b, cy = _axis(y, t.origin[1], t.spacing, t.ny)
    h00, h01, h10, h11 = t.height[j][i], t.height[j][i + 1], t.height[j + 1][i], t.height[j + 1][i + 1]
    h0 = h00 + a * (h01 - h00)
    h1 = h10 + a * (h11 - h10)
    d0, d1 = h01 - h00, h11 - h10
    gx = 0.0 if cx else (d0 + b * (d1 - d0)) / t.spacing
    gy = 0.0 if cy else (h1 - h0) / t.spacing
    return h0 + b * (h1 - h0), gx, gy


def contact_numpy(p, v, t, k, d, ct, mu):
    """(force (3,), normal force) of one contact point at p with velocity v on the HbTerrain t, with ground stiffness k, damping d,
    tangential damping ct and friction coefficient mu: the flat path where the gradient is zero, the sloped path elsewhere."""
    h, gx, gy = terrain_height(t, p[0], p[1])
    if gx == 0.0 and gy == 0.0:
        depth = h - p[2]
        if not depth > 0:
            return np.zeros(3), 0.0
        fz = max(0.0, k * depth - d * v[2])
        ft = -ct * v[:2]
        n = np.linalg.norm(ft)
        if n > mu * fz:
            ft = ft * (mu * fz / n if n > 0 else 0.0)
        return np.array([ft[0], ft[1], fz]), fz
    L = math.sqrt(1.0 + gx * gx + gy * gy)
    n = np.array([-gx, -gy, 1.0]) / L
    depth = (h - p[2]) / L
    if not depth > 0:
        return np.zeros(3), 0.0
    vn = float(v @ n)
    fn = max(0.0, k * depth - d * vn)
    ft = -ct * (v - vn * n)
    tl = np.linalg.norm(ft)
    if tl > mu * fn:
        ft = ft * (mu * fn / tl if tl > 0 else 0.0)
    return fn * n + ft, fn


def plant_numpy_terrain(oracle, rbd, tau, prm, terrain, variation=None, wrench=None):
    """One plant step of one robot on the terrain (an HbTerrain), on its varied plant (None: nominal) and with an external wrench (None:
    none): episode_ref.plant_numpy with each contact from contact_numpy and, with a variation, plant_variation_ref's scaled ground, motor
    strengths and payload terms. Returns (rbd_next, contact forces of the last substep (12,), contact flags of the last substep (4,))."""
    from oracle import refs
    q = np.concatenate([rbd[3:6], rbd[0:3], rbd[6:16]])
    v = np.concatenate([rbd[19:22], refs.euler_rates_from_global(rbd[0:3], rbd[16:19]), rbd[22:32]])
    h = prm.dt / prm.substeps
    k_g, d_g, mu = prm.ground_stiffness, prm.ground_damping, prm.friction_mu
    if variation is not None:
        k_g, d_g, mu = k_g * variation.stiffness_scale, d_g * variation.damping_scale, mu * variation.friction_scale
        tau = np.array(variation.motor_strength[:]) * tau
    F, flags = np.zeros(12), np.zeros(4, dtype=bool)
    for _ in range(prm.substeps):
        r = oracle.rbd(q, v)
        M, nle = r["M"].copy(), r["nle"].copy()
        if variation is not None and variation.payload_mass > 0:
            Mp, nlep = payload_terms(q, v, variation)
            M[:6, :6] += Mp; nle[:6] += nlep
        cvel = r["J"] @ v
        F = np.zeros(12)
        for c in range(4):
            F[3 * c:3 * c + 3], fn = contact_numpy(r["cpos"][3 * c:3 * c + 3], cvel[3 * c:3 * c + 3], terrain, k_g, d_g, prm.tangential_damping, mu)
            flags[c] = fn > 0
        rhs = np.concatenate([np.zeros(6), tau - prm.joint_damping * v[6:]]) + r["J"].T @ F - nle
        if wrench is not None:
            rhs = rhs + np.concatenate([wrench[:3], T(q[3:6]).T @ wrench[3:], np.zeros(10)])
        qdd = np.linalg.solve(M + np.diag(np.r_[np.zeros(6), np.full(10, prm.joint_armature)]), rhs)
        v = v + h * qdd
        q = q + h * v
    out = np.zeros(32)
    out[0:3] = q[3:6]; out[3:6] = q[0:3]; out[6:16] = q[6:]
    out[16:19] = refs.global_from_euler_rates(q[3:6], v[3:6]); out[19:22] = v[0:3]; out[22:32] = v[6:]
    return out, F, flags


def flat_terrain(height, center=(0.0, 0.0), spacing=0.5):
    """One flat HbTerrain at `height`: a 2 x 2 grid around `center`."""
    return hb.make_terrains(1, np.full((2, 2), height), spacing, np.asarray(center) - 0.5 * spacing)[0]


class _TerrainPlant:
    """A context whose plant steps run on the given terrains (Context.sim_step with terrain=; instances beyond them stand on a flat terrain
    at the ground height, which is the flat plant bit for bit) and, when given, the varied plants (instances beyond them: the default
    variation); every other call is the context's own."""

    def __init__(self, ctx, terrains, B, ground_height, variations=None):
        self._ctx = ctx
        self._t = (hb.HbTerrain * B)(*[terrains[i] if i < len(terrains) else flat_terrain(ground_height) for i in range(B)])
        self._v = None if variations is None else (hb.HbPlantVariation * B)(
            *[variations[i] if i < len(variations) else hb.default_plant_variation() for i in range(B)])

    def sim_step(self, rbd, tau, params=None, wrench=None):
        return self._ctx.sim_step(rbd, tau, params, wrench=wrench, variation=self._v, terrain=self._t)

    def __getattr__(self, name):
        return getattr(self._ctx, name)


def stepwise_terrain(ctx, rbd0, gaits, cmd_vels, n_ticks, prm, log_every, terrains, variations=None, ep=None, est=None, pushes=None):
    """episode_ref.stepwise with every plant step on the terrains (and the varied plants) set on ctx (hb_sim_step_terrain). Its height
    check is the absolute one, so it restates the terrain episode only with prm.min_base_height = 0 (episode_ref.params)."""
    assert prm.min_base_height == 0
    plant = _TerrainPlant(ctx, terrains, rbd0.shape[0], prm.sim.ground_height, variations)
    return stepwise(plant, rbd0, gaits, cmd_vels, n_ticks, prm, log_every, ep, est, pushes)
