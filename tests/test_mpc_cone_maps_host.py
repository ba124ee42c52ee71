"""MPC cone maps on the host (no GPU): the shared surface frame (hbplan::map_frame) against its Python restatement bit for bit, orthonormal
with n along (-gx, -gy, 1); the oracle given frames (mpc_cone_ref.py) -- identity and no frames are oracle/hbo.py bit for bit, flat maps
give identity frames, and a tilted cone's gradient and Hessian are the finite differences of its value and gradient; on a plane steeper
than atan(mu) vertical forces leave the tilted cone and the mapped iteration turns them towards the normal; the record check of
HB_SETTING_MPC_CONE_MAPS against HB_SETTING_TERRAINS and the Python constant against the header."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import api
from hunter_bipedal_control_b200 import scenarios as S
from oracle import hbo
from episode_ref import terrain_height
import height_map_ref as M
import mpc_cone_ref as CO
from mpc_map_ref import in_stance, stance_heights
import wbc_map_ref as W

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
HEADER = open(os.path.join(ROOT, "include", "hunter_b200.h")).read()
N, DT = 20, 0.01
MU = 0.7                                        # task.info frictionCoefficient (HB_FRICTION_MU)


def _problem(B=3, gait="trot", seed=5):
    x0, x_ref, swing, mode = S.make_batch(B, N, DT, gait=gait, seed=seed)
    xt, ut = zip(*(hbo.mpc_cold_start(N, DT, x0[i], mode[i]) for i in range(B)))
    return x0, x_ref, swing, mode, np.array(xt), np.array(ut)


def _equal(a, b):
    assert np.array_equal(np.asarray(a), np.asarray(b))


def plane(a, b, n=8, spacing=0.2, origin=(-0.9, -0.9)):
    """A map of the plane z = a x + b y around the scenarios' feet."""
    xs = origin[0] + spacing * np.arange(n); ys = origin[1] + spacing * np.arange(n)
    return hb.make_terrains(1, a * xs[None, :] + b * ys[:, None], spacing, origin)[0]


# ---------------------------------------------------------------------------------------------------------------- the shared frame
def test_map_frame_is_the_python_restatement_bit_for_bit():
    rng = np.random.default_rng(11)
    maps = [M.random_maps(1, 40 + s)[0] for s in range(3)] + [M.step_map(1, 0.0, 0.05)[0], M.slope_map(1, 0.3, axis=1)[0],
                                                              plane(0.4, -0.9), M.plateau(1, 0.1)[0], M.zero_maps(1)[0]]
    n_sloped = n_flat = 0
    for m in maps:
        for x, y in rng.uniform(-1.2, 1.2, (200, 2)):
            f = CO.map_frame(m, x, y)
            r = W.frame(m, x, y)
            if r is None:
                assert f is None; n_flat += 1
                continue
            n_sloped += 1
            assert f.tobytes() == np.array(r).tobytes()
            n, t1, t2 = f
            _, gx, gy = terrain_height(m, x, y)
            np.testing.assert_allclose(f @ f.T, np.eye(3), rtol=0, atol=1e-14)
            np.testing.assert_allclose(n, np.array([-gx, -gy, 1.0]) / math.sqrt(1 + gx * gx + gy * gy), rtol=0, atol=1e-15)
            np.testing.assert_allclose(np.cross(n, t1), t2, rtol=0, atol=1e-15)
            assert t1[1] == 0.0 and n[2] > 0
    assert n_sloped > 500 and n_flat > 300


def test_flat_maps_give_identity_frames():
    x0, x_ref, swing, mode, xt, ut = _problem(B=2)
    off_grid = hb.make_terrains(1, np.random.default_rng(4).uniform(-0.1, 0.1, (6, 6)), 0.1, (5.0, -7.0))[0]   # clamped on both axes
    for m in (None, M.zero_maps(1)[0], M.plateau(1, 0.15)[0], off_grid):
        _equal(CO.cone_frames(m, swing[0], mode[0]), np.tile(CO.IDENTITY, (N + 1, 4, 1)))
    fr = CO.cone_frames(plane(0.3, 0.2), swing[0], mode[0])
    for k in range(N + 1):
        for c in range(4):
            assert np.array_equal(fr[k, c], CO.IDENTITY) != in_stance(mode[0][k], c)      # tilted exactly on stance contacts
    fb = CO.cone_frames_batch([plane(0.3, 0.2)], swing, mode)
    _equal(fb[0], fr); _equal(fb[1], np.tile(CO.IDENTITY, (N + 1, 4, 1)))                  # beyond the maps: no map


# ---------------------------------------------------------------------------------------------------------------- the restated cone
@pytest.mark.parametrize("gait", ["trot", "stance", "flying_trot"])
def test_identity_frames_are_the_oracle(gait):
    x0, x_ref, swing, mode, xt, ut = _problem(gait=gait)
    ident = np.tile(CO.IDENTITY, (N + 1, 4, 1))
    for i in range(3):
        a = hbo.mpc_iteration(N, DT, x0[i], x_ref[i], swing[i], mode[i], xt[i], ut[i], record=True)
        for fr in (ident, None):
            b = CO.mpc_iteration(N, DT, x0[i], x_ref[i], swing[i], mode[i], xt[i], ut[i], record=True, frames=fr)
            _equal(a[0], b[0]); _equal(a[1], b[1]); assert a[2] == b[2] and a[3] == b[3]
        la = hbo.node_lq(DT, xt[i][3], ut[i][3], xt[i][4], x_ref[i][3], swing[i][3], int(mode[i][3]))
        for fr in (ident[3], None):
            lb = CO.node_lq(DT, xt[i][3], ut[i][3], xt[i][4], x_ref[i][3], swing[i][3], int(mode[i][3]), frames=fr)
            for k in la:
                _equal(la[k][:la["m"]] if k == "e" else la[k], lb[k][:lb["m"]] if k == "e" else lb[k])
    a = hbo.mpc_iteration_batch(N, DT, x0, x_ref, swing, mode, xt, ut)
    for fr in (np.tile(CO.IDENTITY, (3, N + 1, 4, 1)), None):
        b = CO.mpc_iteration_batch(N, DT, x0, x_ref, swing, mode, xt, ut, frames=fr)
        _equal(a[0], b[0]); _equal(a[1], b[1]); assert a[2] == b[2]


def test_frames_and_heights_together_are_each_alone_where_the_other_is_null():
    """With identity frames the restatement is mpc_map_ref's on the same heights, bit for bit."""
    import mpc_map_ref as MO
    x0, x_ref, swing, mode, xt, ut = _problem(gait="trot")
    for i in range(3):
        H = stance_heights(M.random_maps(1, 90 + i)[0], swing[i], mode[i])
        a = MO.mpc_iteration(N, DT, x0[i], x_ref[i], swing[i], mode[i], xt[i], ut[i], record=True, stance_h=H)
        b = CO.mpc_iteration(N, DT, x0[i], x_ref[i], swing[i], mode[i], xt[i], ut[i], record=True, stance_h=H,
                             frames=np.tile(CO.IDENTITY, (N + 1, 4, 1)))
        _equal(a[0], b[0]); _equal(a[1], b[1]); assert a[2] == b[2] and a[3] == b[3]


def _cone_terms(x, u, xn, xref, swing, mode, fr):
    """The cone's share of node_lq on frames fr: the node terms on them less the terms on identity frames (every other term is the same
    statement on the same values, so the difference is the tilted cone less the flat one)."""
    a = CO.node_lq(DT, x, u, xn, xref, swing, mode, frames=np.tile(CO.IDENTITY, (4, 1)))
    b = CO.node_lq(DT, x, u, xn, xref, swing, mode, frames=fr)
    return a, b


@pytest.mark.parametrize("grad", [(0.2, 0.0), (0.0, -0.35), (0.5, 0.4), (-0.8, 0.3)])
def test_tilted_cone_derivatives_are_finite_differences_of_its_value(grad):
    x0, x_ref, swing, mode, xt, ut = _problem(B=1, gait="trot", seed=9)
    k = 4
    md = int(mode[0][k])
    fr = np.tile(CO.IDENTITY, (4, 1))
    st = [c for c in range(4) if in_stance(md, c)]
    for c in st:
        fr[c] = CO.plane_frame(*grad)
    x, xn, xref, sw = xt[0][k], xt[0][k + 1], x_ref[0][k], swing[0][k]
    u = ut[0][k].copy()
    rng = np.random.default_rng(2)
    for c in st:
        u[3 * c:3 * c + 2] += rng.uniform(-30, 30, 2)                 # tangential forces: a cone off its axis
    a, b = _cone_terms(x, u, xn, xref, sw, md, fr)
    for key in ("Ad", "Bd", "b", "P", "q", "C", "D"):
        _equal(a[key], b[key])                                         # the cone acts on the cost, r and R (and the Q shift) only
    _equal(a["e"][:a["m"]], b["e"][:b["m"]])
    Q = b["Q"] - a["Q"]
    assert np.count_nonzero(Q - np.diag(np.diag(Q))) == 0              # the Hessian shift: the state diagonal only
    eps = 1e-4

    def at(v):
        p, q = _cone_terms(x, v, xn, xref, sw, md, fr)
        return q["cost"] - p["cost"], q["r"] - p["r"]
    for c in st:
        for i in range(3):
            up, um = u.copy(), u.copy()
            up[3 * c + i] += eps; um[3 * c + i] -= eps
            (cp, rp), (cm, rm) = at(up), at(um)
            g = (cp - cm) / (2 * eps)
            dr = b["r"][3 * c + i] - a["r"][3 * c + i]
            assert abs(g - dr) < 1e-6 * max(1.0, abs(dr)), (c, i, g, dr)
            h = (rp - rm) / (2 * eps)                                   # column 3c+i of the Hessian difference
            dR = b["R"][:, 3 * c + i] - a["R"][:, 3 * c + i]
            blk = slice(3 * c, 3 * c + 3)
            np.testing.assert_allclose(h[blk], dR[blk], rtol=0, atol=1e-6 * max(1.0, np.abs(dR[blk]).max()))
    assert np.abs(b["r"] - a["r"]).max() > 1e-3 and abs(b["cost"] - a["cost"]) > 1e-6


def test_tilt_binds_on_a_plane_steeper_than_the_cone():
    """Stance on a plane rising at 45 degrees along x (steeper than atan(0.7) = 35 degrees): the weight-compensating vertical forces are
    outside the tilted cone (h < 0) though well inside the flat one. The mapped iteration pays for it in its merit and turns every
    stance force towards the plane's normal (-1, 0, 1)/sqrt(2): Fx falls against the flat iteration's, in sum and on most nodes."""
    x0, x_ref, swing, mode, xt, ut = _problem(B=1, gait="stance", seed=12)
    g = 1.0
    m = plane(g, 0.0)
    fr = CO.cone_frames(m, swing[0], mode[0])
    assert not np.array_equal(fr[:N], np.tile(CO.IDENTITY, (N, 4, 1)))
    R = CO.plane_frame(g, 0.0).reshape(3, 3)
    for k in range(N):
        for c in range(4):
            F = ut[0][k][3 * c:3 * c + 3]
            Fl = R @ F
            assert MU * F[2] - math.sqrt(F[0] ** 2 + F[1] ** 2 + 25) > 0                    # inside the flat cone
            assert MU * Fl[2] - math.sqrt(Fl[0] ** 2 + Fl[1] ** 2 + 25) < 0                 # outside the tilted one
    a = CO.mpc_iteration(N, DT, x0[0], x_ref[0], swing[0], mode[0], xt[0], ut[0])
    b = CO.mpc_iteration(N, DT, x0[0], x_ref[0], swing[0], mode[0], xt[0], ut[0], frames=fr)
    assert b[2]["merit0"] > a[2]["merit0"] + 0.1
    dFx = b[1][:, 0::3][:, :4] - a[1][:, 0::3][:, :4]
    assert dFx.sum() < 0 and (dFx < 0).mean() >= 0.75, dFx


# ---------------------------------------------------------------------------------------------------------------- ABI
def test_exported_and_kind():
    lib = hb.load_library()
    assert "hb_mpc_set_cone_maps" in hb.EXPORTED_SYMBOLS and hasattr(lib, "hb_mpc_set_cone_maps")
    assert int(re.search(r"^#define HB_SETTING_MPC_CONE_MAPS (\d+)", HEADER, re.M).group(1)) == api.MPC_CONE_MAPS_SETTING_KIND == 19
    assert not re.search(r"^#define HB_SETTING_\w+ (10|16)\b", HEADER, re.M)                # 10 and 16 stay unassigned
    assert hasattr(hb.Context, "set_mpc_cone_maps")


def test_cone_map_records_are_checked_as_terrains():
    lib = hb.load_library()
    cases = [M.random_maps(3, 72)]
    for field, value in [("nx", 1), ("nx", 65), ("ny", 1), ("ny", 65), ("spacing", 0.0), ("spacing", -0.1), ("spacing", float("nan")),
                         ("spacing", float("inf"))]:
        r = M.random_maps(3, 72); setattr(r[1], field, value); cases.append(r)
    r = M.random_maps(3, 72); r[2].origin[1] = float("-inf"); cases.append(r)
    r = M.random_maps(3, 72); r[0].height[5][7] = float("nan"); cases.append(r)
    r = M.random_maps(3, 72); r[0].height[30][30] = float("nan"); cases.append(r)            # beyond the used samples: not read
    for recs in cases:
        a, b = C.c_int32(-7), C.c_int32(-7)
        ra = lib.hb_check_setting_records(api.HB_SETTING_TERRAINS, 3, recs, C.byref(a))
        rb = lib.hb_check_setting_records(api.MPC_CONE_MAPS_SETTING_KIND, 3, recs, C.byref(b))
        assert (ra, a.value) == (rb, b.value)
    assert [lib.hb_check_setting_records(19, 3, c, C.byref(C.c_int32())) for c in cases] == [0] + [-1] * 10 + [0]
    assert lib.hb_check_setting_records(19, 0, None, C.byref(C.c_int32())) == 0


def test_the_oracle_on_frames_rewrites_the_one_cone_statement():
    """mpc_cone_oracle.cpp takes over the oracle's cone through HB_FRICTION_BARRIER_MU and HB_FRICTION_BARRIER_DELTA: both must appear in
    the oracle once, as the barrier arguments of the cone's penalty, for the restatement to mean what it says."""
    src = open(os.path.join(ROOT, "oracle", "hb_oracle.cpp")).read()
    assert src.count("HB_FRICTION_BARRIER_MU") == 1 and src.count("HB_FRICTION_BARRIER_DELTA") == 1
    assert "Pen p = relaxed_barrier(h, HB_FRICTION_BARRIER_MU, HB_FRICTION_BARRIER_DELTA);" in src
