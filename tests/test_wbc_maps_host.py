"""WBC maps on the host (no GPU): the restatement (wbc_map_ref.py) against oracle/hbo.py -- zero, plateau and off-grid maps give
hbo.wbc_assemble's QP bit for bit; the frame on planes of several slopes and azimuths is orthonormal and its normal is the plane's; the
rotated pyramid admits a force just inside the cone and rejects one just outside; on a 30 degree plane at mu = 0.5 the flat WBC's
forces leave the tilted cone and the mapped WBC holds them on it; the record check of HB_SETTING_WBC_MAPS against HB_SETTING_TERRAINS and
the Python constant against the header."""
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
import height_map_ref as M
import wbc_map_ref as W

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
HEADER = open(os.path.join(ROOT, "include", "hunter_b200.h")).read()
MU = 0.7                                        # task.info frictionCoefficient (HB_WBC_FRICTION_MU), the oracle's


def _same(a, b):
    assert np.asarray(a).tobytes() == np.asarray(b).tobytes()


def _cases(B, seed):
    """Perturbed standing states in every mode, forces sharing the weight over the stance contacts (test_gpu_parity's cases)."""
    rng = np.random.default_rng(seed)
    mode = np.array([3, 2, 1, 0] * ((B + 3) // 4), dtype=np.int32)[:B]
    x = np.tile(S.INITIAL_STATE, (B, 1)) + rng.uniform(-.05, .05, (B, 22))
    u = np.zeros((B, 22))
    for i in range(B):
        fl = S.mode_flags(int(mode[i]))
        for c in range(4):
            if fl[c]:
                u[i, 3 * c + 2] = S.TOTAL_MASS * 9.81 / sum(fl)
        u[i, 12:] = rng.uniform(-.5, .5, 10)
    return x, u, S.consistent_rbd(x, rng, 0.02), mode


def plane(a, b, n=8, spacing=0.2, origin=(-0.7, -0.7)):
    """A map of the plane z = a x + b y."""
    xs = origin[0] + spacing * np.arange(n); ys = origin[1] + spacing * np.arange(n)
    return hb.make_terrains(1, a * xs[None, :] + b * ys[:, None], spacing, origin)[0]


FLAT_MAPS = {
    "zero": lambda: M.zero_maps(1)[0],
    "plateau": lambda: M.plateau(1, 0.15)[0],
    "off_grid": lambda: hb.make_terrains(1, np.random.default_rng(4).uniform(-0.1, 0.1, (6, 6)), 0.1, (5.0, -7.0))[0],   # clamped on both axes
}


@pytest.mark.parametrize("name", sorted(FLAT_MAPS))
@pytest.mark.parametrize("stance_mode", [False, True])
def test_flat_maps_are_the_oracle_bit_for_bit(name, stance_mode):
    m = FLAT_MAPS[name]()
    x, u, rbd, mode = _cases(8, 3)
    for i in range(8):
        assert W.frames(m, rbd[i]) == [None] * 4
        a = hbo.wbc_assemble(x[i], u[i], rbd[i], int(mode[i]), stance_mode)
        b = W.wbc_assemble(x[i], u[i], rbd[i], mode[i], stance_mode, m, MU)
        for p, q in zip(a, b):
            _same(p, q)


def test_the_flat_pyramid_is_the_oracles_rows():
    x, u, rbd, mode = _cases(4, 8)
    for i in range(4):
        A = hbo.wbc_assemble(x[i], u[i], rbd[i], int(mode[i]))[2]
        r0, st = W.pyramid_rows(int(mode[i]))
        assert A.shape[0] == r0 + 5 * len(st) + 3 * (4 - len(st))
        for k, c in enumerate(st):
            _same(A[r0 + 5 * k:r0 + 5 * k + 5, 16 + 3 * c:19 + 3 * c], W.pyramid(None, MU))


@pytest.mark.parametrize("deg", [3.0, 9.0, 20.0, 30.0, 45.0])
@pytest.mark.parametrize("azimuth", [0.0, 35.0, 90.0, 160.0, 250.0])
def test_frame_on_planes_is_orthonormal_about_the_planes_normal(deg, azimuth):
    g = math.tan(math.radians(deg))
    a, b = g * math.cos(math.radians(azimuth)), g * math.sin(math.radians(azimuth))
    m = plane(a, b)
    want = np.array([-a, -b, 1.0]) / math.sqrt(1 + a * a + b * b)
    for x, y in [(0.03, -0.11), (0.31, 0.2), (-0.4, 0.47)]:
        n, t1, t2 = W.frame(m, x, y)
        F = np.array([n, t1, t2])
        assert np.abs(F @ F.T - np.eye(3)).max() < 1e-15
        assert np.abs(np.cross(n, t1) - t2).max() < 1e-15 and t1[1] == 0.0
        assert np.abs(n - want).max() < 1e-13


@pytest.mark.parametrize("deg, azimuth", [(10.0, 0.0), (30.0, 60.0), (25.0, 200.0)])
def test_the_rotated_pyramid_admits_inside_and_rejects_outside(deg, azimuth):
    g = math.tan(math.radians(deg))
    n, t1, t2 = W.frame(plane(g * math.cos(math.radians(azimuth)), g * math.sin(math.radians(azimuth))), 0.1, 0.1)
    mu, fn = 0.5, 40.0
    P = W.pyramid((n, t1, t2), mu)
    for s1, s2 in [(1, 1), (1, -1), (-1, 1), (-1, -1), (1, 0), (0, -1)]:
        inside = fn * n + (1 - 1e-9) * mu * fn * (s1 * t1 + s2 * t2)
        assert (P @ inside <= 0).all()
        outside = fn * n + (1 + 1e-9) * mu * fn * (s1 * t1 + s2 * t2)
        assert (P @ outside > 0).any()
    assert (P @ (-fn * n) > 0).any()                     # pulling on the ground: the unilateral row


def _settings_with_mu(mu):
    """task.info's WBC settings (hb_default_wbc_settings) with friction coefficient mu, as the oracle's 17 values."""
    lib = hb.load_library()
    w = api.HbWbcSettings()
    assert lib.hb_default_wbc_settings(C.byref(w)) == 0
    w.friction_coefficient = mu
    return w.as_array()


def test_thirty_degree_plane_at_half_friction_binds_a_tangential_row():
    """The case the GPU test solves: standing on a 30 degree plane (tan 30 > 0.5), the flat WBC's stance forces leave the tilted cone; the
    mapped WBC's forces satisfy the tilted rows and hold a tangential one active."""
    m = plane(math.tan(math.radians(30.0)), 0.0)
    x, u, rbd, mode = _cases(4, 11)
    hbo.set_wbc_settings(_settings_with_mu(0.5))
    try:
        for i in [0]:                                   # mode 3: four stance contacts
            assert mode[i] == 3
            fr = W.frames(m, rbd[i])
            flat, st = hbo.wbc_solve(x[i], u[i], rbd[i], 3, False, 1e-8)
            assert st == 0
            mapped, st = W.wbc_solve(x[i], u[i], rbd[i], 3, False, m, 0.5)
            assert st == 0
            worst_flat, tangential = -np.inf, -np.inf
            for c in range(4):
                P = W.pyramid(fr[c], 0.5)
                F0, F1 = flat[16 + 3 * c:19 + 3 * c], mapped[16 + 3 * c:19 + 3 * c]
                worst_flat = max(worst_flat, (P @ F0).max())
                assert (P @ F1 <= 1e-9 * max(1.0, np.abs(F1).max())).all()
                tangential = max(tangential, (P[1:] @ F1).max())
            assert worst_flat > 1.0                     # newtons outside the tilted cone
            assert abs(tangential) < 1e-6               # a tangential row active
    finally:
        hbo.set_wbc_settings(None)


def test_exported_and_kind():
    lib = hb.load_library()
    assert "hb_wbc_set_maps" in hb.EXPORTED_SYMBOLS and hasattr(lib, "hb_wbc_set_maps")
    assert int(re.search(r"^#define HB_SETTING_WBC_MAPS (\d+)", HEADER, re.M).group(1)) == api.WBC_MAPS_SETTING_KIND == 18
    assert not hasattr(api, "HB_SETTING_WBC_MAPS")      # the module's HB_SETTING_* set stays the episode settings' ten kinds
    assert hasattr(hb.Context, "set_wbc_maps")


def test_wbc_map_records_are_checked_as_terrains():
    lib = hb.load_library()
    cases = [M.random_maps(3, 72)]
    for field, value in [("nx", 1), ("nx", 65), ("ny", 1), ("spacing", 0.0), ("spacing", float("nan"))]:
        r = M.random_maps(3, 72); setattr(r[1], field, value); cases.append(r)
    r = M.random_maps(3, 72); r[0].height[5][7] = float("nan"); cases.append(r)
    for recs in cases:
        a, b = C.c_int32(-7), C.c_int32(-7)
        ra = lib.hb_check_setting_records(api.HB_SETTING_TERRAINS, 3, recs, C.byref(a))
        rb = lib.hb_check_setting_records(api.WBC_MAPS_SETTING_KIND, 3, recs, C.byref(b))
        assert (ra, a.value) == (rb, b.value)
    assert [lib.hb_check_setting_records(18, 3, c, C.byref(C.c_int32())) for c in cases] == [0] + [-1] * 6
    assert lib.hb_check_setting_records(18, 0, None, C.byref(C.c_int32())) == 0
    assert lib.hb_check_setting_records(16, 3, cases[0], C.byref(C.c_int32())) == -1      # 16 stays unassigned
