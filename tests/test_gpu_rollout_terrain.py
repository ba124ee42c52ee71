"""Terrain (hb_rollout_set_terrains, hb_sim_step_terrain): a height field under each robot of the episodes. The plant step on a terrain is
checked against a numpy restatement and against exact identities with the flat plant; independently of the restatement, against yaw and
translation invariance and the friction cone about the local normal. The terrain episode is checked bit for bit against the loop of
public calls, the terrain-relative height check on its own, and the setting against unset episodes: flat terrains, continuation,
independence, permutation, instances beyond the setting, clearing, launch counts; then the argument checks."""
import ctypes as C
import math

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from episode_ref import (FRICTION, GAITS, GROUND, PUSH, assert_episode_equal, assert_null_settings, assert_rejected_settings, assert_setting_episodes,
                         cmd_vels, context, device, est_params, launch_coefficients, outputs, params, plant_numpy, start_states, stepwise, terrain_height,
                         use)

pytestmark = pytest.mark.gpu

S = 0.025                                                # grid spacing of the episode terrains [m]
RZ = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])      # +pi/2 about the world z axis, exact


def _P(a):
    return C.c_void_p(a.ctypes.data)


def _step_inputs(B, seed):
    """Random poses with the base at 0.60-0.64 m and a spinning base, and random joint torques."""
    rng = np.random.default_rng(seed)
    x = sc.random_initial_states(B, seed=seed + 40)
    rbd = sc.consistent_rbd(x, rng, 0.02)
    rbd[:, 5] = rng.uniform(0.60, 0.64, B)
    rbd[:, 1] = rng.uniform(-0.3, 0.3, B); rbd[:, 2] = rng.uniform(-0.3, 0.3, B)
    rbd[:, 16:19] = rng.uniform(-1.5, 1.5, (B, 3))
    return rbd, rng.uniform(-15, 15, (B, 10)), rng


def _feet(oracle, r):
    """World positions (4 x 3) of the contact points of the rbd state r."""
    from oracle import refs
    q = np.concatenate([r[3:6], r[0:3], r[6:16]])
    v = np.concatenate([r[19:22], refs.euler_rates_from_global(r[0:3], r[16:19]), r[22:32]])
    return oracle.rbd(q, v)["cpos"].reshape(4, 3)


def _grid(origin, n, m, spacing):
    """World (X, Y) of the samples of an n x m (ny x nx) grid."""
    return np.meshgrid(origin[0] + spacing * np.arange(m), origin[1] + spacing * np.arange(n))


def _plant_terrains(oracle, rbd, rng):
    """Eight terrains, one per robot, placed against the robot's contact points: a plane with the lowest contact point exactly on a grid
    corner; a plane with it exactly on a cell edge (a plane, because there the cell is chosen by the last bit of the position, and a
    plane has the same gradient in both cells); a step between two plateaus; a seeded rough field; a rough grid far from the robot (every
    coordinate clamped: the flat path at the corner's height); a grid beside the robot in x only (x clamped: the sloped path along y); a
    rough field with every contact point on a plateau cell (the flat path at four heights); a steep rough field. Each touches the robot."""
    T = hb.make_terrains(8, np.zeros((2, 2)), 1.0)
    for i in range(8):
        f = _feet(oracle, rbd[i])
        zlo = f[:, 2].min() + 0.002
        low = f[np.argmin(f[:, 2])]
        if i == 0:
            o = low[:2] - [7 * S, 5 * S]
            X, Y = _grid(o, 20, 24, S)
            T[i] = hb.make_terrains(1, low[2] + 0.2 * (X - low[0]) - 0.1 * (Y - low[1]), S, o)[0]
        elif i == 1:
            o = low[:2] - [9 * S, 6.4 * S]
            X, Y = _grid(o, 24, 24, S)
            T[i] = hb.make_terrains(1, low[2] - 0.15 * (X - low[0]) + 0.25 * (Y - low[1]), S, o)[0]
        elif i == 2:
            o = rbd[i, 3:5] - 0.4
            X, _ = _grid(o, 33, 33, S)
            T[i] = hb.make_terrains(1, np.where(X < rbd[i, 3] + 0.013, zlo, zlo + 0.01), S, o)[0]
        elif i == 3:
            o = rbd[i, 3:5] - 0.5
            T[i] = hb.make_terrains(1, zlo + rng.uniform(-0.01, 0.01, (21, 21)), 0.05, o)[0]
        elif i == 4:
            h = rng.uniform(-0.05, 0.05, (6, 6)); h[0, 0] = zlo
            T[i] = hb.make_terrains(1, h, 0.1, rbd[i, 3:5] + 3.0)[0]
        elif i == 5:
            o = np.array([rbd[i, 3] + 1.0, rbd[i, 4] - 0.5])
            X, Y = _grid(o, 11, 4, 0.1)
            T[i] = hb.make_terrains(1, zlo + 0.1 * (Y - rbd[i, 4]) + rng.uniform(-0.02, 0.02, (11, 1)) * (X - o[0]), 0.1, o)[0]
        elif i == 6:
            o = rbd[i, 3:5] - 0.5
            h = zlo + rng.uniform(-0.01, 0.01, (41, 41))
            for c in range(4):
                ci, cj = int((f[c, 0] - o[0]) / S), int((f[c, 1] - o[1]) / S)
                h[cj:cj + 2, ci:ci + 2] = f[c, 2] + 0.001 * (c + 1)
            T[i] = hb.make_terrains(1, h, S, o)[0]
        else:
            o = rbd[i, 3:5] - 0.6
            T[i] = hb.make_terrains(1, zlo + rng.uniform(-0.05, 0.05, (13, 13)), 0.1, o)[0]
        if i in (0, 1, 3, 5, 7):                         # lowered or raised so that the deepest contact point is 2 mm inside
            t = T[i]
            dz = max(terrain_height(t, *f[c, :2])[0] - f[c, 2] for c in range(4)) - 0.002
            h = np.array(t.height)[:t.ny, :t.nx] - dz
            T[i] = hb.make_terrains(1, h, t.spacing, t.origin[:])[0]
    return T


def _variations(B, rng):
    return hb.make_plant_variations(B, rng.uniform(0.5, 4.0, B), rng.uniform(-0.1, 0.1, (B, 3)), np.diag([0.01, 0.02, 0.015]),
                                    rng.uniform(0.3, 1.0, B), rng.uniform(0.5, 2.0, B), rng.uniform(0.5, 2.0, B), rng.uniform(0.5, 1.2, (B, 10)))


# ---------------------------------------------------------------------------------------------------------------- the plant step
def test_terrain_plant_step_matches_numpy_restatement(gpu_ctx, oracle):
    B = 8
    rbd, tau, rng = _step_inputs(B, 31)
    T = _plant_terrains(oracle, rbd, rng)
    prm = hb.default_sim_params()
    V = _variations(B, rng)
    W = np.c_[rng.uniform(-150, 150, (B, 3)), rng.uniform(-30, 30, (B, 3))]
    flat = gpu_ctx.sim_step(rbd, tau, prm)
    touched = 0
    for var, wr in ((None, None), (V, W)):
        nxt, cf, fl = gpu_ctx.sim_step(rbd, tau, prm, wrench=wr, variation=var, terrain=T)
        for i in range(B):
            ref, F, flags = plant_numpy(oracle, rbd[i], tau[i], prm, None if wr is None else wr[i], None if var is None else var[i], T[i])
            assert np.abs(nxt[i] - ref).max() < 1e-9 * max(1.0, np.abs(ref).max()), (i, np.abs(nxt[i] - ref).max())
            assert np.abs(cf[i] - F).max() < 1e-7 * max(1.0, np.abs(F).max()), (i, cf[i], F)
            assert np.array_equal(fl[i] != 0, flags), (i, fl[i], flags)
            touched += int(flags.sum())
            assert np.abs(nxt[i] - flat[0][i]).max() > 1e-6                 # the terrain acts
    assert 0 < touched < 8 * B


def test_exact_identities_of_the_terrain_step(gpu_ctx):
    B = 6
    rbd, tau, rng = _step_inputs(B, 32)
    prm = hb.default_sim_params()
    lib = gpu_ctx._lib
    V = _variations(B, rng)
    W = np.c_[rng.uniform(-100, 100, (B, 3)), rng.uniform(-20, 20, (B, 3))]

    def terrain_step(t, w=None, v=None, p=prm):
        r = rbd.copy(); cf = np.zeros((B, 12)); fl = np.zeros((B, 4), dtype=np.uint8)
        assert lib.hb_sim_step_terrain(gpu_ctx._h, B, C.byref(p), _P(r), _P(tau), None if w is None else _P(w), v, t, _P(cf), _P(fl)) == 0
        return r, cf, fl

    def same(a, b):
        for x, y in zip(a, b):
            assert np.array_equal(x, y)

    # a NULL terrain is hb_sim_step_varied
    same(terrain_step(None, W, V), gpu_ctx.sim_step(rbd, tau, prm, wrench=W, variation=V))
    same(terrain_step(None), gpu_ctx.sim_step(rbd, tau, prm))
    # a flat terrain at sim.ground_height is no terrain: under the robots, and far from them (clamped)
    near = hb.make_terrains(B, np.full((8, 8), prm.ground_height), 0.1, rbd[:, 3:5] - 0.35)
    far = hb.make_terrains(B, np.full((3, 5), prm.ground_height), 0.1, rbd[:, 3:5] + [[-4.0, 2.0]])
    for t in (near, far):
        same(terrain_step(t), gpu_ctx.sim_step(rbd, tau, prm))
        same(terrain_step(t, W, V), gpu_ctx.sim_step(rbd, tau, prm, wrench=W, variation=V))
    # a flat terrain at c is the flat plant with ground_height = c, for robots inside and outside the grid
    c = 0.0173
    pc = hb.default_sim_params(); pc.ground_height = c
    org = rbd[:, 3:5] - 0.35
    org[1::2] += 5.0                                                         # odd robots outside their grid
    Tc = hb.make_terrains(B, np.full((8, 8), c), 0.1, org)
    want = gpu_ctx.sim_step(rbd, tau, pc)
    same(terrain_step(Tc), want)
    assert not np.array_equal(want[0], gpu_ctx.sim_step(rbd, tau, prm)[0])
    assert (want[2] != 0).any()


def _on_plane(ctx, B, seed, gx, gy, c=0.0):
    """B perturbed standing poses lowered onto the planes h = c + gx[i] x + gy[i] y, the deepest contact point 2 mm inside."""
    rbd = start_states(ctx, B, seed)
    rng = np.random.default_rng(seed)
    rbd[:, 3:5] = rng.uniform(-0.2, 0.2, (B, 2))
    rbd[:, 19:22] = rng.uniform(-0.05, 0.05, (B, 3))
    f = ctx.contact_positions(ctx.rbd_to_centroidal(rbd)).reshape(B, 4, 3)
    gap = f[:, :, 2] - (c + gx[:, None] * f[:, :, 0] + gy[:, None] * f[:, :, 1])
    rbd[:, 5] -= gap.min(axis=1) + 0.002
    return rbd


def _plane_terrains(origins, n, gx, gy, c=0.0):
    B = len(origins)
    T = hb.make_terrains(B, np.zeros((2, 2)), 1.0)
    for i in range(B):
        X, Y = _grid(origins[i], n, n, S)
        T[i] = hb.make_terrains(1, c + gx[i] * X + gy[i] * Y, S, origins[i])[0]
    return T


def _run(ctx, rbd, T, steps, q0):
    r, prm = rbd.copy(), hb.default_sim_params()
    for _ in range(steps):
        r, cf, fl = ctx.sim_step(r, 60.0 * (q0 - r[:, 6:16]) - 2.0 * r[:, 22:32], prm, terrain=T)
    return r, cf, fl


def test_yaw_invariance_on_a_plane(gpu_ctx):
    """A robot on the plane h = g x and the same robot yawed by +pi/2 about the world z axis on the plane h = g y, on the grid rotated to
    match, agree to 1e-9 after 5 plant steps: their states and contact forces are rotations of each other."""
    B = 3
    g = np.array([0.12, -0.25, 0.35])
    rbd = _on_plane(gpu_ctx, B, 41, g, np.zeros(B))
    n = 32
    oa = rbd[:, 3:5] - 0.5 * (n - 1) * S
    Ta = _plane_terrains(oa, n, g, np.zeros(B))
    rot = rbd.copy()
    for i in range(B):
        rot[i, 0] += 0.5 * np.pi
        for a in (3, 16, 19):
            rot[i, a:a + 3] = RZ @ rbd[i, a:a + 3]
    ob = np.c_[-(oa[:, 1] + (n - 1) * S), oa[:, 0]]                      # the rotated grid's sample (0, 0)
    Tb = _plane_terrains(ob, n, np.zeros(B), g)
    q0 = rbd[:, 6:16]
    ra, fa, la = _run(gpu_ctx, rbd, Ta, 5, q0)
    rb, fb, lb = _run(gpu_ctx, rot, Tb, 5, q0)
    assert (la != 0).sum() >= B
    back = rb.copy()
    back[:, 0] -= 0.5 * np.pi
    for i in range(B):
        for a in (3, 16, 19):
            back[i, a:a + 3] = RZ.T @ rb[i, a:a + 3]
    assert np.abs(back - ra).max() < 1e-9 * max(1.0, np.abs(ra).max()), np.abs(back - ra).max()
    fb_back = np.einsum("ij,bcj->bci", RZ.T, fb.reshape(B, 4, 3)).reshape(B, 12)
    assert np.abs(fb_back - fa).max() < 1e-9 * max(1.0, np.abs(fa).max()), np.abs(fb_back - fa).max()
    assert np.array_equal(la, lb)
    flat, _, _ = _run(gpu_ctx, rbd, hb.make_terrains(B, np.zeros((n, n)), S, oa), 5, q0)
    assert np.abs(flat - ra).max() > 1e-6                                  # the slope acts


def test_translation_invariance_on_a_plane(gpu_ctx):
    """A robot moved by (dx, 0, g dx) on the plane h = c + g x gives the moved result to 1e-9."""
    B = 3
    g, c, dx = np.array([0.2, -0.3, 0.1]), 0.05, 0.35
    rbd = _on_plane(gpu_ctx, B, 42, g, np.zeros(B), c)
    o = rbd[:, 3:5] - [0.4, 0.6]
    T = _plane_terrains(o, 50, g, np.zeros(B), c)
    moved = rbd.copy()
    moved[:, 3] += dx; moved[:, 5] += g * dx
    q0 = rbd[:, 6:16]
    ra, fa, la = _run(gpu_ctx, rbd, T, 5, q0)
    rb, fb, lb = _run(gpu_ctx, moved, T, 5, q0)
    assert (la != 0).sum() >= B
    rb[:, 3] -= dx; rb[:, 5] -= g * dx
    assert np.abs(rb - ra).max() < 1e-9 * max(1.0, np.abs(ra).max()), np.abs(rb - ra).max()
    assert np.abs(fb - fa).max() < 1e-9 * max(1.0, np.abs(fa).max())
    assert np.array_equal(la, lb)


def test_contact_forces_lie_in_the_friction_cone_about_the_local_normal(gpu_ctx):
    """On planes of several gradients, with the robots sliding, every returned contact force F satisfies F.n >= 0 and
    |F - (F.n) n| <= mu F.n (1 + 1e-12) about the plane's normal n, and some lie on the cone's surface (friction saturated)."""
    B = 8
    rng = np.random.default_rng(43)
    gx, gy = rng.uniform(-0.6, 0.6, B), rng.uniform(-0.6, 0.6, B)
    rbd = _on_plane(gpu_ctx, B, 43, gx, gy)
    rbd[:, 19:22] = rng.uniform(-0.8, 0.8, (B, 3))
    rbd[:, 5] -= 0.004
    T = _plane_terrains(rbd[:, 3:5] - 0.5, 40, gx, gy)
    prm = hb.default_sim_params()
    onsurface = 0
    for var in (None, hb.make_plant_variations(B, friction_scale=rng.uniform(0.1, 1.0, B))):
        _, cf, fl = gpu_ctx.sim_step(rbd, np.zeros((B, 10)), prm, variation=var, terrain=T)
        assert (fl != 0).any()
        for i in range(B):
            n = np.array([-gx[i], -gy[i], 1.0]) / math.sqrt(1.0 + gx[i] ** 2 + gy[i] ** 2)
            mu = prm.friction_mu * (1.0 if var is None else var[i].friction_scale)
            for k in range(4):
                F = cf[i, 3 * k:3 * k + 3]
                fn = F @ n
                ft = np.linalg.norm(F - fn * n)
                assert fn >= 0.0 and ft <= mu * fn * (1 + 1e-12) + 1e-12, (i, k, fn, ft, mu)
                assert (fl[i, k] != 0) == (fn > 0)
                onsurface += fn > 0 and ft > mu * fn * (1 - 1e-9)
    assert onsurface > 0


# ---------------------------------------------------------------------------------------------------------------- terrain episodes
def _profile_terrains(rbd0, profiles, rng=None):
    """One 64 x 64 terrain at spacing S per profile, centred on the robot's base: ground at GROUND + f(d), d the distance ahead of the base
    origin along the robot's initial heading; "flat", "step_up" / "step_down" (2 cm, 6 cm ahead), "ramp", "rough" (seeded +-3 mm)."""
    T = hb.make_terrains(len(profiles), np.zeros((2, 2)), 1.0)
    for i, kind in enumerate(profiles):
        o = rbd0[i, 3:5] - 31.5 * S
        X, Y = _grid(o, 64, 64, S)
        d = (X - rbd0[i, 3]) * math.cos(rbd0[i, 0]) + (Y - rbd0[i, 4]) * math.sin(rbd0[i, 0])
        if kind == "flat":
            h = np.zeros_like(X)
        elif kind == "step_up":
            h = np.where(d > 0.06, 0.02, 0.0)
        elif kind == "step_down":
            h = np.where(d > 0.06, -0.02, 0.0)
        elif kind == "ramp":                             # 4 degrees up through the start, level again 0.3 m behind it
            h = np.maximum(d, -0.3) * math.tan(math.radians(4.0))
        else:
            h = rng.uniform(-0.003, 0.003, X.shape)
        T[i] = hb.make_terrains(1, GROUND + h, S, o)[0]
    return T


PROFILES = ["flat", "ramp", "step_up", "rough", "step_down"]          # instance 5 of the six stands beyond the setting


@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
def test_terrain_episode_equals_the_stepwise_loop_bitwise(event_nodes):
    ctx = context(event_nodes)
    B, n_ticks, log_every = 6, 200, 10
    rbd0 = start_states(ctx, B, seed=51)
    vels = cmd_vels(B)
    prm = params(log_every)
    kw = use(ctx, terrains=_profile_terrains(rbd0, PROFILES, np.random.default_rng(51)),
             plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION, stiffness_scale=[1.0, 1.0, 1.3, 1.0, 0.8, 1.0]),
             pushes=hb.make_push_schedules(B, 0.15, 0.05, PUSH))
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every)
    r = stepwise(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, **kw)
    assert_episode_equal(d, r)
    ctx.set_terrains(None)
    u = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every)
    moved = [not np.array_equal(a, b) for a, b in zip(d[0].cpu().numpy(), u[0].cpu().numpy())]
    assert not moved[0] and not moved[5] and moved[1] and moved[3], moved
    ctx.close()


def test_terrain_estimated_episode_equals_the_stepwise_loop_bitwise():
    ctx = context()
    B, n_ticks, log_every = 6, 120, 10
    rbd0 = start_states(ctx, B, seed=52)
    vels = cmd_vels(B)
    prm = params(log_every)
    ep = est_params(seed=2025)
    kw = use(ctx, terrains=_profile_terrains(rbd0, PROFILES, np.random.default_rng(52)),
             plant_variations=hb.make_plant_variations(B, 1.5, [0.0, 0.0, 0.1], np.diag([0.01, 0.01, 0.01])),
             pushes=hb.make_push_schedules(B, 0.1, 0.04, [[0.0, 30.0, 0.0]]))
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 40))
    r = stepwise(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 40), **kw)
    assert_episode_equal(d, r)
    ctx.close()


def test_the_height_check_measures_above_the_terrain():
    """One-tick episodes with min_base_height = 0.3: the base height of an instance with a terrain is measured above the terrain at the
    base's (x, y), that of an instance beyond the setting from z = 0."""
    ctx = context()
    B = 4
    rbd0 = start_states(ctx, B, seed=53)
    rbd0[:, 5] = [0.5, 0.25, 0.25, 0.5]
    prm = params(0)
    prm.min_base_height = 0.3
    vels = cmd_vels(B)
    T = hb.make_terrains(2, np.stack([np.full((4, 4), 0.3), np.full((4, 4), -0.2)]), 0.2, rbd0[:2, 3:5] - 0.3)

    def failed():
        st = outputs(device(ctx, rbd0, GAITS[:B], vels, 1, prm, 0))[3]
        return [bool(st["fail_tick"][i] == 0 and st["fail_reason"][i] & hb.ROLLOUT_FAIL["height"]) for i in range(B)]

    ctx.set_terrains(T)
    # 0.5 above a 0.3 m plateau: 0.2 m; 0.25 above a -0.2 m hollow: 0.45 m; beyond the setting: 0.25 and 0.5 m from z = 0
    assert failed() == [True, False, True, False]
    ctx.set_terrains(None)
    assert failed() == [False, True, True, False]
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_flat_terrains_at_the_ground_height_change_nothing(estimated):
    ctx = context()
    B, n_ticks = 6, 100
    rbd0 = start_states(ctx, B, seed=54)
    vels = cmd_vels(B)
    prm = params(5)
    ep = est_params(seed=78) if estimated else None
    flat = _profile_terrains(rbd0, ["flat"] * B)
    assert_null_settings(ctx, "terrains", lambda: device(ctx, rbd0, GAITS, vels, n_ticks, prm, 5, ep), (flat, (hb.HbTerrain * 3)(*flat[:3])),
                         _profile_terrains(rbd0, PROFILES, np.random.default_rng(0)))
    ctx.close()


def test_continuation_independence_permutation_and_instances_beyond_the_setting():
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=55)
    T = _profile_terrains(rbd0, PROFILES + ["ramp"], np.random.default_rng(55))
    only0 = _profile_terrains(rbd0, ["flat"] * B)
    only0[0] = _profile_terrains(rbd0, ["ramp"])[0]
    other = _profile_terrains(rbd0, ["rough", "step_up", "ramp", "ramp", "rough", "step_down"], np.random.default_rng(9))
    other[3] = T[3]
    padded = _profile_terrains(rbd0, ["flat"] * B)
    for i in range(3):
        padded[i] = T[i]
    assert_setting_episodes(ctx, "terrains", rbd0, params(10), T, only0, other, 3, (hb.HbTerrain * 3)(*[T[i] for i in range(3)]), padded)
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_terrains_add_no_launch(estimated):
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=56)
    vels = cmd_vels(B)
    prm = params(0)
    ep = est_params(seed=6) if estimated else None
    plain = launch_coefficients(ctx, rbd0, GAITS, vels, prm, ep)
    ctx.set_terrains(_profile_terrains(rbd0, PROFILES + ["rough"], np.random.default_rng(1)))
    assert launch_coefficients(ctx, rbd0, GAITS, vels, prm, ep) == plain
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- argument checks
def test_argument_checks_return_before_any_launch_and_keep_the_setting():
    ctx = context(max_batch=6)
    lib = ctx._lib
    B = 6
    rbd0 = start_states(ctx, B, seed=57)
    vels = cmd_vels(B)
    prm = params(10)
    T = _profile_terrains(rbd0, PROFILES + ["ramp"], np.random.default_rng(57))
    assert C.sizeof(hb.HbTerrain) == 32800
    nan, inf = float("nan"), float("inf")

    def bad(field, value, index=None):
        W = (hb.HbTerrain * B)(*T)
        s = W[2]
        if field == "height":
            s.height[index[0]][index[1]] = value
        elif index is None:
            setattr(s, field, value)
        else:
            getattr(s, field)[index] = value
        return W

    cases = [("nx", 1), ("nx", 0), ("nx", -3), ("nx", 65), ("ny", 1), ("ny", 65), ("origin", nan, 0), ("origin", inf, 1),
             ("origin", -inf, 0), ("spacing", 0.0), ("spacing", -0.025), ("spacing", nan), ("spacing", inf), ("height", nan, (0, 0)),
             ("height", inf, (63, 63)), ("height", -inf, (10, 40))]
    big = (hb.HbTerrain * (B + 1))(*([T[0]] * (B + 1)))
    assert_rejected_settings(ctx, "terrains", lambda: device(ctx, rbd0, GAITS, vels, 60, prm, 10), T, [bad(*case) for case in cases], big)
    # samples beyond nx / ny are not read, so they are not checked either
    small = hb.make_terrains(B, np.full((3, 4), GROUND), 0.3, rbd0[:, 3:5] - 0.45)
    small[1].height[3][0] = nan; small[1].height[0][4] = inf
    assert lib.hb_rollout_set_terrains(ctx._h, B, small) == 0
    # the host plant step checks its terrains as the setting does
    sp = hb.default_sim_params()
    r = np.zeros((B, 32)); t = np.zeros((B, 10))
    c0 = ctx.launch_count
    for case in cases[:8] + cases[-3:]:
        assert lib.hb_sim_step_terrain(ctx._h, B, C.byref(sp), _P(r), _P(t), None, None, bad(*case), None, None) == -1, case
    assert lib.hb_sim_step_terrain(ctx._h, B + 1, C.byref(sp), _P(np.zeros((B + 1, 32))), _P(np.zeros((B + 1, 10))), None, None, big, None, None) == -4
    assert lib.hb_sim_step_terrain(ctx._h, 0, C.byref(sp), _P(r), _P(t), None, None, None, None, None) == 0
    assert ctx.launch_count == c0
    ctx.close()
