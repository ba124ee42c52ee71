"""MPC maps on the host (no GPU): the oracle given stance heights (mpc_map_ref.py) -- zero and no heights are oracle/hbo.py bit for bit, a
constant map and a shift of every height in the problem by the same constant leave the solve unchanged but for the base height, and the
heights act on the stance z rows' values only; the restated heights (mpc_map_ref.py) look the map up at the swing references of stance
contacts only; the record check of HB_SETTING_MPC_MAPS against HB_SETTING_TERRAINS and the Python constant against the header."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import api
from hunter_bipedal_control_b200 import scenarios as S
from oracle import hbo
import height_map_ref as M
import mpc_map_ref as MO
from mpc_map_ref import in_stance, stance_heights, stance_heights_batch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
HEADER = open(os.path.join(ROOT, "include", "hunter_b200.h")).read()
N, DT = 20, 0.01


def _problem(B=3, gait="trot", seed=5):
    x0, x_ref, swing, mode = S.make_batch(B, N, DT, gait=gait, seed=seed)
    xt, ut = zip(*(hbo.mpc_cold_start(N, DT, x0[i], mode[i]) for i in range(B)))
    return x0, x_ref, swing, mode, np.array(xt), np.array(ut)


def _same(a, b):
    assert np.asarray(a).tobytes() == np.asarray(b).tobytes()


@pytest.mark.parametrize("gait", ["trot", "stance", "flying_trot"])
def test_zero_heights_are_the_oracle_without_them(gait):
    x0, x_ref, swing, mode, xt, ut = _problem(gait=gait)
    zero = np.zeros((N + 1, 4))
    for i in range(3):
        a = hbo.mpc_iteration(N, DT, x0[i], x_ref[i], swing[i], mode[i], xt[i], ut[i], record=True)
        for sh in (zero, None):
            b = MO.mpc_iteration(N, DT, x0[i], x_ref[i], swing[i], mode[i], xt[i], ut[i], record=True, stance_h=sh)
            _same(a[0], b[0]); _same(a[1], b[1]); assert a[2] == b[2] and a[3] == b[3]
        la = hbo.node_lq(DT, xt[i][3], ut[i][3], xt[i][4], x_ref[i][3], swing[i][3], int(mode[i][3]))
        for sh in (zero[3], None):
            lb = MO.node_lq(DT, xt[i][3], ut[i][3], xt[i][4], x_ref[i][3], swing[i][3], int(mode[i][3]), stance_h=sh)
            for k in la:
                _same(la[k][:la["m"]] if k == "e" else la[k], lb[k][:lb["m"]] if k == "e" else lb[k])   # e beyond m: not written
    a = hbo.mpc_iteration_batch(N, DT, x0, x_ref, swing, mode, xt, ut)
    for sh in (np.zeros((3, N + 1, 4)), None):
        b = MO.mpc_iteration_batch(N, DT, x0, x_ref, swing, mode, xt, ut, stance_h=sh)
        _same(a[0], b[0]); _same(a[1], b[1]); assert a[2] == b[2]


def test_heights_act_on_the_stance_z_rows_values_only():
    x0, x_ref, swing, mode, xt, ut = _problem(gait="trot")
    rng = np.random.default_rng(3)
    seen = set()
    for i in range(3):
        for k in range(N):
            md = int(mode[i][k])
            hk = rng.uniform(-0.1, 0.1, 4)
            a = hbo.node_lq(DT, xt[i][k], ut[i][k], xt[i][k + 1], x_ref[i][k], swing[i][k], md)
            b = MO.node_lq(DT, xt[i][k], ut[i][k], xt[i][k + 1], x_ref[i][k], swing[i][k], md, stance_h=hk)
            for key in a:
                if key != "e":
                    _same(a[key], b[key])       # C, D (the row's Jacobian), the cost and the dynamics do not see the map
            row, want = 0, a["e"].copy()
            for c in range(4):
                if in_stance(md, c):
                    want[row + 2] -= 3 * hk[c]
                    row += 3
                else:
                    row += 4                    # zero force (3) and normal velocity (1): unchanged
            assert a["m"] == b["m"] == row
            np.testing.assert_allclose(b["e"][:row], want[:row], rtol=0, atol=1e-15)      # e beyond m: not written by the node LQ
            seen.add(md)
    assert seen >= {2, 3}                       # single support and double stance


@pytest.mark.parametrize("gait", ["trot", "stance"])
def test_constant_map_is_a_translation_of_the_problem(gait):
    x0, x_ref, swing, mode, xt, ut = _problem(gait=gait)
    c = 0.25
    hc = np.array([stance_heights(M.plateau(1, c)[0], swing[i], mode[i]) for i in range(3)])
    sx0, sxr, ssw, sxt = x0.copy(), x_ref.copy(), swing.copy(), xt.copy()
    sx0[:, 8] += c; sxr[:, :, 8] += c; sxt[:, :, 8] += c
    for f in range(4):
        ssw[:, :, 6 * f + 2] += c
    for i in range(3):
        a = hbo.mpc_iteration(N, DT, x0[i], x_ref[i], swing[i], mode[i], xt[i], ut[i], record=True)
        b = MO.mpc_iteration(N, DT, sx0[i], sxr[i], ssw[i], mode[i], sxt[i], ut[i], record=True, stance_h=hc[i])
        shift = np.zeros(22); shift[8] = c
        np.testing.assert_allclose(b[0], a[0] + shift, rtol=0, atol=1e-12)
        np.testing.assert_allclose(b[1], a[1], rtol=0, atol=1e-12 * max(1.0, np.abs(a[1]).max()))
        for key in ("merit0", "merit1", "viol0", "viol1", "armijo"):
            assert abs(b[2][key] - a[2][key]) <= 1e-12 * max(1.0, abs(a[2][key])), key
        assert (b[2]["alpha"], b[2]["n_trials"], b[2]["status"]) == (a[2]["alpha"], a[2]["n_trials"], a[2]["status"])
        assert [t["branch"] for t in b[3]] == [t["branch"] for t in a[3]]


def test_restated_heights_are_the_map_at_stance_swing_references_only():
    x0, x_ref, swing, mode, xt, ut = _problem(B=2, gait="trot")
    m = M.random_maps(1, 19)[0]
    H = stance_heights(m, swing[0], mode[0])
    n_stance = n_swing = 0
    for k in range(N + 1):
        for c in range(4):
            if in_stance(mode[0][k], c):
                assert H[k, c] == M.h(m, swing[0][k][6 * c], swing[0][k][6 * c + 1]); n_stance += 1
            else:
                assert H[k, c] == 0.0 and not np.signbit(H[k, c]); n_swing += 1
    assert n_stance > 0 and n_swing > 0
    Hb = stance_heights_batch([m], swing, mode)
    _same(Hb[0], H)
    assert Hb[1].tobytes() == np.zeros((N + 1, 4)).tobytes()            # beyond the maps: no map, +0
    assert (stance_heights(M.plateau(1, 0.1)[0], swing[1], mode[1]) == np.where(
        [[in_stance(md, c) for c in range(4)] for md in mode[1]], 0.1, 0.0)).all()


def test_exported_and_kind():
    lib = hb.load_library()
    assert "hb_mpc_set_maps" in hb.EXPORTED_SYMBOLS and hasattr(lib, "hb_mpc_set_maps")
    assert int(re.search(r"^#define HB_SETTING_MPC_MAPS (\d+)", HEADER, re.M).group(1)) == api.MPC_MAPS_SETTING_KIND == 17
    assert hasattr(hb.Context, "set_mpc_maps")


def test_mpc_map_records_are_checked_as_terrains():
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
        rb = lib.hb_check_setting_records(api.MPC_MAPS_SETTING_KIND, 3, recs, C.byref(b))
        assert (ra, a.value) == (rb, b.value)
    assert [lib.hb_check_setting_records(17, 3, c, C.byref(C.c_int32())) for c in cases] == [0] + [-1] * 10 + [0]
    assert lib.hb_check_setting_records(17, 0, None, C.byref(C.c_int32())) == 0


def test_the_oracle_on_heights_rewrites_the_one_stance_z_statement():
    """mpc_map_oracle.cpp appends its height term to the oracle's stance z row through HB_ZEROVEL_Z_OFFSET: that macro must appear in the
    oracle once, as the last term of that row's statement, for the restatement to mean what it says."""
    src = open(os.path.join(ROOT, "oracle", "hb_oracle.cpp")).read()
    assert src.count("HB_ZEROVEL_Z_OFFSET") == 1
    assert "if (a == 2) val += HB_ZEROVEL_Z_GAIN * epos[3 * c + 2] + HB_ZEROVEL_Z_OFFSET;" in src
