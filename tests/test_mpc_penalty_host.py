"""The MPC stage cost's relaxed-barrier penalties on the CPU: the float64 oracle's node LQ model against the numpy restatement
(penalty_ref) in every region of every penalty, finite differences of the oracle's cost in each region, continuity across h = delta,
and the case generator of test_gpu_mpc_penalty_envelope (each case sits where its name says, at every linearisation point)."""
import numpy as np
import pytest

import penalty_ref as P

H_FD = 1e-6


@pytest.fixture(scope="module")
def cases(oracle):
    return P.make_cases(oracle)


@pytest.fixture(scope="module")
def first_iteration(cases, oracle):
    return oracle.mpc_iteration_batch(P.N, P.DT, *P.stack(cases), threads=4)


def _unom(mode):
    fl = P.stance(mode)
    u = np.zeros(P.NU)
    for c in range(4):
        if fl[c]:
            u[3 * c + 2] = P.TOTAL_MASS * P.GRAVITY / sum(fl)
    return u


def _node(oracle, x, u, xr, sw, mode):
    return oracle.node_lq(P.DT, x, u, x, xr, sw, int(mode))


def _penalty_share(oracle, x, u, xr, sw, mode):
    """The oracle's node LQ model at (x, u) minus its tracking terms (Q_DIAG, the input cost R) and its xy swing soft constraint: what is
    left is the penalties' share of cost, q, r, Q, R (and P, which they do not touch)."""
    o = _node(oracle, x, u, xr, sw, mode)
    Rin = oracle.input_cost_R()
    dx, du = x - xr, u - _unom(mode)
    s = dict(cost=o["cost"] - 0.5 * P.Q_DIAG @ (dx * dx) - 0.5 * du @ Rin @ du, q=o["q"] - P.Q_DIAG * dx, r=o["r"] - Rin @ du,
             Q=o["Q"] - np.diag(P.Q_DIAG), R=o["R"] - Rin, P=o["P"].copy())
    pos, vel, dp, dvx, dvu = oracle.ee_kinematics(x, u)
    w = P.SOFT_SWING_WEIGHT
    for c, on in enumerate(P.stance(mode)):
        if on:
            continue
        for a in range(2):
            i = 3 * c + a
            h = vel[i] - sw[6 * c + 3 + a] + P.XY_POSITION_GAIN * (pos[i] - sw[6 * c + a])
            gx, gu = dvx[i] + P.XY_POSITION_GAIN * dp[i], dvu[i]
            s["cost"] -= 0.5 * w * h * h; s["q"] -= w * h * gx; s["r"] -= w * h * gu
            s["Q"] -= w * np.outer(gx, gx); s["R"] -= w * np.outer(gu, gu); s["P"] -= w * np.outer(gu, gx)
    return s


def test_restatement_derivatives_and_continuity_at_delta():
    """value -> slope -> curvature by central differences in every region of the four barrier configurations, and value, slope and
    curvature continuous across h = delta."""
    for mu, delta in (P.POS, P.VEL, P.FORCE, P.CONE):
        for h in (3.0 * delta, 1.5 * delta, 0.5 * delta, 0.0, -0.2 * delta, -2.0 * delta):
            e = 1e-6 * delta
            (vp, dp, _), (vm, dm, _), (_, d1, d2) = (P.relaxed_barrier(h + s, mu, delta) for s in (e, -e, 0.0))
            assert abs((vp - vm) / (2 * e) - d1) < 1e-7 * max(1.0, abs(d1)), (mu, delta, h)
            assert abs((dp - dm) / (2 * e) - d2) < 1e-6 * d2, (mu, delta, h)
        above, below = P.relaxed_barrier(delta * (1 + 1e-12), mu, delta), P.relaxed_barrier(delta, mu, delta)
        assert below[2] == mu / delta ** 2 and np.allclose(above, below, rtol=1e-10, atol=1e-10), (mu, delta)
    # the cone's gradient and Hessian in F
    for F in ((0.0, 0.0, 30.0), (12.0, 0.0, 30.0), (0.0, -9.0, 20.0), (8.0, -5.0, 40.0)):
        F = np.array(F)
        _, g, H = P.cone(F)
        for i in range(3):
            e = np.zeros(3); e[i] = 1e-5
            (hp, gp, _), (hm, gm, _) = P.cone(F + e), P.cone(F - e)
            assert abs((hp - hm) / 2e-5 - g[i]) < 1e-9 and np.abs((gp - gm) / 2e-5 - H[i]).max() < 1e-9, (F, i)


def test_oracle_node_lq_penalty_share_vs_restatement_in_every_region(cases, oracle):
    """At every linearisation point of every case: the oracle's penalty share of cost, q, r, Q and R equals the restatement; the regions
    seen cover interior, band and violated on both sides of every joint position and velocity limit and of the force bounds of every
    contact, in stance and in swing, and the three regions of every stance cone, in modes 0-3."""
    seen = set()
    for c in cases:
        for k, (x, u, mode) in enumerate(P.linearisation_points(c)):
            if k % 4 and k != 1:        # node 0 (x0), node 1 and every fourth node: the cases are uniform in k beyond node 0
                continue
            s = _penalty_share(oracle, x, u, c["xr"][k], c["sw"][k], mode)
            ref = P.penalties(x, u, mode)
            for key in ("cost", "q", "r", "Q", "R"):
                tol = 1e-11 * max(1.0, np.abs(ref[key]).max())
                assert np.abs(s[key] - ref[key]).max() < tol, (c["name"], k, key, np.abs(s[key] - ref[key]).max())
            assert np.abs(s["P"]).max() < 1e-12, (c["name"], k)
            fl = P.stance(mode)
            for (fam, i, side), reg in P.classify(x, u, mode).items():
                if reg is not None:
                    seen.add((fam, i, side, reg, ("stance" if fl[i] else "swing") if fam in ("force", "cone") else None, int(mode)))
    modes = {m for *_, m in seen}
    assert modes == {0, 1, 2, 3}
    cov = {(f, i, sd, r, st) for f, i, sd, r, st, _ in seen}
    for fam in ("pos", "vel"):
        assert all((fam, j, sd, r, None) in cov for j in range(P.NJ) for sd in ("lo", "hi") for r in P.REGIONS), fam
    for c in range(4):
        assert all(("force", c, sd, r, "stance") in cov for sd in ("lo", "hi") for r in P.REGIONS), c
        assert ("force", c, "lo", "violated", "swing") in cov and ("force", c, "hi", "interior", "swing") in cov, c
        assert all(("cone", c, "lo", r, "stance") in cov for r in P.REGIONS), c
    assert not any(f == "cone" and st == "swing" for f, _, _, _, st in cov)      # swing contacts carry no cone


def _fd_points(cases):
    """One linearisation point (node 1) per case of each (family, side, region, mode), and every mixed case."""
    pick = {}
    for c in cases:
        if len(c["targets"]) == 1:
            ((fam, _, side), reg), = c["targets"].items()
            key = (fam, side, reg, int(c["mode"][0]), c["name"].split("/")[3] if fam == "cone" else None)
        else:
            key = c["name"]
        pick.setdefault(key, c)
    return list(pick.values())


def test_oracle_cost_gradient_and_curvature_by_finite_differences(cases, oracle):
    """Central differences of the oracle's node cost against its q and r in each region (every argument at least 10 h_fd from delta),
    and of its q and r against the diagonal of Q / R on the penalised coordinates (the cone's whole 3x3 block), minus the cone's
    Hessian shift, in stance where the model is exact."""
    pts = _fd_points(cases)
    assert len(pts) > 40
    for c in pts:
        x, u, mode = P.linearisation_points(c)[1]
        xr, sw = c["xr"][1], c["sw"][1]
        for h, delta in (a for a in P.arguments(x, u, mode).values() if a is not None):
            assert abs(h - delta) > 10 * H_FD * max(1.0, np.abs(u).max()), c["name"]
        o = _node(oracle, x, u, xr, sw, mode)
        z = np.concatenate([x, u])
        for i in range(P.NX + P.NU):
            e = H_FD * max(1.0, abs(z[i]))
            zp, zm = z.copy(), z.copy(); zp[i] += e; zm[i] -= e
            op, om = _node(oracle, zp[:22], zp[22:], xr, sw, mode), _node(oracle, zm[:22], zm[22:], xr, sw, mode)
            g = o["q"][i] if i < P.NX else o["r"][i - P.NX]
            fd = (op["cost"] - om["cost"]) / (2 * e)
            assert abs(fd - g) < 1e-6 * max(1.0, abs(g)) + 1e-12 * max(1.0, abs(o["cost"])) / e, (c["name"], i, fd, g)
            if mode != 3 or i < 12:
                continue
            # curvature: the penalised diagonal, and the cone block of the contact (forces of one contact couple through the cone only)
            if i < P.NX:
                fdc, an = (op["q"][i] - om["q"][i]) / (2 * e), o["Q"][i, i] - _shift(u, mode)
            else:
                j = i - P.NX
                blk = slice(3 * (j // 3), 3 * (j // 3) + 3) if j < 12 else slice(j, j + 1)
                fdc, an = (op["r"][blk] - om["r"][blk]) / (2 * e), o["R"][j, blk].copy()
                an[j - blk.start] -= _shift(u, mode)
            assert np.abs(fdc - an).max() < 1e-5 * max(1e-2, np.abs(an).max()), (c["name"], i, fdc, an)


def _shift(u, mode):
    """hessianDiagonalShift's contribution to every diagonal entry of Q and R: -shift * sum of the stance cones' d1."""
    return -P.HESSIAN_SHIFT * sum(P.relaxed_barrier(P.cone(u[3 * c:3 * c + 3])[0], *P.CONE)[1] for c in range(4) if P.stance(mode)[c])


@pytest.mark.parametrize("fam", ("pos", "vel", "force", "cone"))
def test_oracle_value_slope_and_curvature_continuous_across_delta(fam, oracle):
    """The oracle's cost, q / r and Q / R at h = delta (quadratic side) and h = delta (1 + 1e-9) (log side) of one argument of each family
    (upper side for the bounds): the jumps are those of the smooth function, so value, slope and curvature are continuous."""
    mode = 3
    x = P.sc.INITIAL_STATE.copy(); u = _unom(mode)
    xr, sw, _, _ = P.sc.make_reference(x, (0.0, 0.0, 0.0, 0.0), "stance", 1, P.DT)
    mu, delta = {"pos": P.POS, "vel": P.VEL, "force": P.FORCE, "cone": P.CONE}[fam]
    out = []
    for h in (delta, delta * (1 + 1e-9)):
        x1, u1 = x.copy(), u.copy()
        if fam == "pos":
            x1[12 + 2] = P.JOINT_UPPER[2] - h; i = 12 + 2
        elif fam == "vel":
            u1[12 + 2] = P.JOINT_VEL[2] - h; i = P.NX + 12 + 2
        elif fam == "force":
            u1[3 * 1 + 2] = P.FORCE_MAX - h; i = P.NX + 3 * 1 + 2
        else:
            u1[3:6] = (0.0, 0.0, (h + np.sqrt(P.FRICTION_REG)) / P.FRICTION_MU); i = P.NX + 5
        key = (fam, 2, "hi") if fam in ("pos", "vel") else (fam, 1, "hi" if fam == "force" else "lo")
        assert P.arguments(x1, u1, mode)[key][0] == pytest.approx(h, rel=1e-12)
        o = _node(oracle, x1, u1, xr[0], sw[0], mode)
        g = np.concatenate([o["q"], o["r"]])[i]
        H = o["Q"][i, i] if i < P.NX else o["R"][i - P.NX, i - P.NX]
        out.append((o["cost"], g, H))
    (c0, g0, H0), (c1, g1, H1) = out
    dz = delta * 1e-9 / (P.FRICTION_MU if fam == "cone" else 1.0)       # the coordinate's step between the two points
    assert abs(c1 - c0) < 2 * abs(g0) * dz + 1e-13 * abs(c0), (fam, c0, c1)
    assert abs(g1 - g0) < 2 * abs(H0) * dz + 1e-13 * max(1.0, abs(g0)), (fam, g0, g1)
    assert abs(H1 - H0) < 1e-6 * abs(H0), (fam, H0, H1)
    assert H0 >= mu / delta ** 2 * (P.FRICTION_MU ** 2 if fam == "cone" else 1.0), (fam, H0)


def test_case_generator_places_every_case_and_exercises_the_line_search(cases, first_iteration):
    """Each case's targets hold at every linearisation point of the first iteration (x0 at node 0, then xt[k], ut[k]), band targets in
    (delta / 2, delta]; swing contacts keep F = 0; every case solves (status 0, finite); the stance baseline takes the full step and penalised stance cases back-track."""
    for c in cases:
        for k, (x, u, mode) in enumerate(P.linearisation_points(c)):
            cl, args = P.classify(x, u, mode), P.arguments(x, u, mode)
            for key, reg in c["targets"].items():
                assert cl[key] == reg, (c["name"], k, key, cl[key])
                if reg == "band":           # in the upper half of the band
                    assert args[key][0] > 0.5 * args[key][1], (c["name"], k, key)
            for cc, on in enumerate(P.stance(mode)):
                if not on:
                    assert not u[3 * cc:3 * cc + 3].any(), (c["name"], k)
    names = [c["name"] for c in cases]
    assert len(set(names)) == len(names)
    xt, ut, infos = first_iteration
    assert all(i["status"] == 0 for i in infos) and np.isfinite(xt).all() and np.isfinite(ut).all()
    alpha = {c["name"]: i["alpha"] for c, i in zip(cases, infos)}
    assert alpha["base/m3"] == 1.0
    back = {f: sum(1 for c in cases if P.family(c) == f and c["mode"][0] == 3 and alpha[c["name"]] < 1.0) for f in ("pos", "vel", "force", "mixed")}
    assert back["pos"] >= 3 and back["vel"] >= 40 and back["force"] >= 4 and back["mixed"] == 1, back
    # every family reaches the line search's later trials somewhere, and cones take the full step in stance
    assert all(any(P.family(c) == f and alpha[c["name"]] < 1.0 for c in cases) for f in ("pos", "vel", "force", "cone", "mixed"))
    assert all(alpha[c["name"]] == 1.0 for c in cases if P.family(c) == "cone" and c["mode"][0] == 3)
