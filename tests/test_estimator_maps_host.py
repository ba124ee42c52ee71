"""Estimator maps on the host (no GPU): the restatement (estimator_map_ref.py) against oracle/refs.py's KalmanFilterRef -- a zero map is
the filter without one and a plateau at c is the filter with every foot height c, bit for bit, and the lookup is at the predicted foot
xy; the record check of HB_SETTING_ESTIMATOR_MAPS against HB_SETTING_TERRAINS; the Python constant against the header; and
terrain_sweep.py's --estimator-maps argument check."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import api
from oracle import hbo
from oracle import refs as R
import height_map_ref as M
from estimator_map_ref import MappedKalmanFilterRef

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
HEADER = open(os.path.join(ROOT, "include", "hunter_b200.h")).read()


def _kin(q, v):
    r = hbo.rbd(q, v)
    return r["cpos"], r["J"] @ v


def _inputs(seed, steps):
    """steps of IMU and encoder readings near a standing pose, with contact flags that change between steps."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(steps):
        zyx = np.array([0.3, 0.05, -0.04]) + rng.normal(0, 0.02, 3)
        cz, sz, cy, sy, cx, sx = (f(0.5 * a) for a in zyx for f in (np.cos, np.sin))
        quat = np.array([cz * cy * sx - sz * sy * cx, cz * sy * cx + sz * cy * sx, sz * cy * cx - cz * sy * sx, cz * cy * cx + sz * sy * sx])
        wl = rng.normal(0, 0.3, 3); al = rng.normal(0, 0.5, 3) + [0, 0, 9.81]
        jpos = np.clip(R.DEFAULT_JOINTS + rng.normal(0, 0.05, 10), R.JOINT_LOWER, R.JOINT_UPPER); jvel = rng.normal(0, 0.3, 10)
        flags = (rng.uniform(size=4) > 0.3).astype(np.uint8)
        out.append((0.002, quat, wl, al, jpos, jvel, flags))
    return out


def _run(f, ins):
    """The filter f over the inputs: the rbd of every step and the final (x, P)."""
    rbd = [f.update(*x, _kin) for x in ins]
    return np.array(rbd), f.x.copy(), f.P.copy()


def _same(a, b):
    for u, v in zip(a, b):
        assert u.tobytes() == v.tobytes()


def test_zero_map_is_the_filter_without_a_map_bitwise():
    ins = _inputs(1, 40)
    want = _run(R.KalmanFilterRef(), ins)
    for zero in (M.zero_maps(1)[0], hb.make_terrains(1, np.zeros((64, 64)), 0.01, (-0.3, -0.3))[0]):
        _same(_run(MappedKalmanFilterRef(zero), ins), want)
    _same(_run(MappedKalmanFilterRef(None), ins), want)


@pytest.mark.parametrize("c", [0.23, -0.07, 1e-3])
def test_plateau_map_is_the_filter_with_those_heights_bitwise(c):
    ins = _inputs(2, 40)
    ref = R.KalmanFilterRef()
    ref.heights = np.full(4, c)
    want = _run(ref, ins)
    f = MappedKalmanFilterRef(M.plateau(1, c)[0])
    got = _run(f, ins)
    _same(got, want)
    assert (f.heights == 0.0).all()                     # the filter's own heights are not read or written on a map
    blind = _run(R.KalmanFilterRef(), ins)
    assert abs(got[1][2] - blind[1][2]) > 0.5 * abs(c)  # the map moves the base height


def _touched(m, pts):
    """The grid samples (j, i) the lookups at pts read."""
    from episode_ref import _axis
    out = set()
    for x, y in pts:
        i, _, _ = _axis(x, m.origin[0], m.spacing, m.nx)
        j, _, _ = _axis(y, m.origin[1], m.spacing, m.ny)
        out |= {(j, i), (j, i + 1), (j + 1, i), (j + 1, i + 1)}
    return out


def test_the_lookup_is_at_the_predicted_foot_xy():
    """A map that differs only at samples no foot lookup reads changes nothing; changing one sample a lookup reads moves the estimate."""
    ins = _inputs(3, 30)
    m = M.random_maps(1, 4, scale=0.03, spacing=0.04, n=40, origin=(-0.8, -0.8))[0]
    f = MappedKalmanFilterRef(m)
    want = _run(f, ins)
    assert len(f.lookups) == 4 * len(ins)
    # the first lookups are at the initial state's feet (all at the origin); the others at the previous estimates' feet
    assert f.lookups[:4] == [(0.0, 0.0)] * 4
    touched = _touched(m, f.lookups)
    far = hb.HbTerrain.from_buffer_copy(m)
    moved = 0
    for j in range(40):
        for i in range(40):
            if (j, i) not in touched:
                far.height[j][i] = 0.5 + 0.01 * (i + j)
                moved += 1
    assert moved > 1500
    _same(_run(MappedKalmanFilterRef(far), ins), want)
    near = hb.HbTerrain.from_buffer_copy(m)
    j, i = sorted(_touched(m, f.lookups[-4:]))[0]
    near.height[j][i] += 0.05
    assert _run(MappedKalmanFilterRef(near), ins)[1].tobytes() != want[1].tobytes()


def test_exported_and_kind():
    lib = hb.load_library()
    assert "hb_estimator_set_maps" in hb.EXPORTED_SYMBOLS and hasattr(lib, "hb_estimator_set_maps")
    assert int(re.search(r"^#define HB_SETTING_ESTIMATOR_MAPS (\d+)", HEADER, re.M).group(1)) == api.ESTIMATOR_MAPS_SETTING_KIND == 15
    assert not hasattr(api, "HB_SETTING_ESTIMATOR_MAPS")     # the module's HB_SETTING_* set stays the ten kinds of test_setting_records_host


def test_estimator_map_records_are_checked_as_terrains():
    lib = hb.load_library()
    cases = [M.random_maps(3, 71)]
    for field, value in [("nx", 1), ("nx", 65), ("ny", 1), ("ny", 65), ("spacing", 0.0), ("spacing", -0.1), ("spacing", float("nan")),
                         ("spacing", float("inf"))]:
        r = M.random_maps(3, 71); setattr(r[1], field, value); cases.append(r)
    r = M.random_maps(3, 71); r[2].origin[0] = float("inf"); cases.append(r)
    r = M.random_maps(3, 71); r[0].height[5][7] = float("nan"); cases.append(r)
    r = M.random_maps(3, 71); r[0].height[30][30] = float("nan"); cases.append(r)            # beyond the used samples: not read
    for recs in cases:
        a, b = C.c_int32(-7), C.c_int32(-7)
        ra = lib.hb_check_setting_records(api.HB_SETTING_TERRAINS, 3, recs, C.byref(a))
        rb = lib.hb_check_setting_records(api.ESTIMATOR_MAPS_SETTING_KIND, 3, recs, C.byref(b))
        assert (ra, a.value) == (rb, b.value)
    assert [lib.hb_check_setting_records(15, 3, c, C.byref(C.c_int32())) for c in cases] == [0] + [-1] * 10 + [0]
    assert lib.hb_check_setting_records(15, 0, None, C.byref(C.c_int32())) == 0
    assert lib.hb_check_setting_records(16, 3, cases[0], C.byref(C.c_int32())) == -1


@pytest.mark.parametrize("flags", [[], ["--height-maps"], ["--estimator"], ["--estimator", "--sensor-noise", "1"]],
                         ids=["alone", "height_maps", "estimator", "estimator_noise"])
def test_terrain_sweep_rejects_estimator_maps_without_height_maps_and_estimator(flags):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "terrain_sweep.py"), "--estimator-maps"] + flags,
                         capture_output=True, text=True, timeout=120)
    assert out.returncode != 0
    assert "--estimator-maps needs --height-maps --estimator" in out.stderr
