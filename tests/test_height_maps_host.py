"""Height maps on the host (no GPU): hb_plan_references_maps, hb_goal_to_target_maps and hb_cmd_vel_to_target_maps with NULL and all-zero
maps against the calls without maps bit for bit; the host planner on stepped, sloped and random maps against oracle/refs.py's planner
with the map rules (height_map_ref.py); plateau invariance; the touch-down heights; the two conversions against a numpy restatement bit for
bit; and the record check of HB_SETTING_HEIGHT_MAPS against HB_SETTING_TERRAINS."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import api
from oracle import refs as R
from planner_settings_ref import GAIT_NAMES, oracle_settings, random_settings
from test_planner_settings_host import T, _cases
import height_map_ref as M

HEADER = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include", "hunter_b200.h")).read()


def test_exported_and_kind():
    lib = hb.load_library()
    for name in ("hb_plan_set_maps", "hb_plan_references_maps", "hb_goal_to_target_maps", "hb_cmd_vel_to_target_maps"):
        assert name in hb.EXPORTED_SYMBOLS and hasattr(lib, name)
    assert int(re.search(r"^#define HB_SETTING_HEIGHT_MAPS (\d+)", HEADER, re.M).group(1)) == api.HEIGHT_MAPS_SETTING_KIND == 14
    assert not hasattr(api, "HB_SETTING_HEIGHT_MAPS")        # the module's HB_SETTING_* set stays the ten kinds of test_setting_records_host


def _plan(n, seed, maps=None, settings=None, targets=None, joint_ik=True):
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, seed)
    refs, ls = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, joint_ik=joint_ik, targets=targets, settings=settings,
                                  maps=maps)
    return bytes(refs), ls.tobytes()


def _goal_targets(n, seed):
    x0, gaits, cmd, t0, *_ = _cases(n, seed)
    rng = np.random.default_rng(seed + 1)
    goal = np.c_[x0[:, 6:8] + rng.uniform(-0.5, 0.5, (n, 2)), x0[:, 9] + rng.uniform(-1, 1, n)]
    return hb.goal_to_target(t0, x0, goal)


@pytest.mark.parametrize("joint_ik", [True, False], ids=["ik", "no_ik"])
@pytest.mark.parametrize("with_settings", [False, True], ids=["compiled_in", "settings"])
@pytest.mark.parametrize("with_targets", [False, True], ids=["cmd_vel", "targets"])
def test_null_and_zero_maps_are_the_planner_without_maps_bitwise(joint_ik, with_settings, with_targets):
    n, seed = 48, 11
    settings = random_settings(n, seed=12) if with_settings else None
    targets = _goal_targets(n, seed) if with_targets else None
    want = _plan(n, seed, None, settings, targets, joint_ik)
    lib = hb.load_library()
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, seed)
    ins = hb.make_plan_inputs(t0, T, x0, cmd, feet, gaits, start, joint_ik=joint_ik)
    refs, ls = (hb.HbReference * n)(), latest.copy()
    assert lib.hb_plan_references_maps(n, ins, targets, settings, None, C.c_void_p(ls.ctypes.data), refs) == 0
    assert (bytes(refs), ls.tobytes()) == want
    for zeros in (M.zero_maps(n), hb.make_terrains(n, np.zeros((64, 64)), 0.01, (-0.3, -0.3))):
        assert _plan(n, seed, zeros, settings, targets, joint_ik) == want


def test_null_and_zero_maps_are_the_conversions_without_maps_bitwise():
    n = 40
    x0, gaits, cmd, t0, *_ = _cases(n, 13)
    rng = np.random.default_rng(14)
    goal = np.c_[x0[:, 6:8] + rng.uniform(-0.5, 0.5, (n, 2)), x0[:, 9] + rng.uniform(-1, 1, n)]
    goal[3, :2] = x0[3, 6:8]; goal[3, 2] = x0[3, 9]                    # reaching time 0: one sample
    lib = hb.load_library()
    P = lambda a: C.c_void_p(a.ctypes.data)
    for make in (lambda: None, lambda: M.zero_maps(n)):
        g0, g1 = (hb.HbTarget * n)(), (hb.HbTarget * n)()
        assert lib.hb_goal_to_target(n, P(t0), P(x0), P(goal), g0) == 0
        assert lib.hb_goal_to_target_maps(n, P(t0), P(x0), P(goal), make(), g1) == 0
        assert bytes(g0) == bytes(g1) and g1[3].n == 1
        c0, c1 = (hb.HbTarget * n)(), (hb.HbTarget * n)()
        assert lib.hb_cmd_vel_to_target(n, P(t0), C.c_double(T), P(x0), P(cmd), c0) == 0
        assert lib.hb_cmd_vel_to_target_maps(n, P(t0), C.c_double(T), P(x0), P(cmd), make(), c1) == 0
        assert bytes(c0) == bytes(c1)


def _map_cases(n, seed):
    """One map per instance: steps up and down under the feet, slopes along x and y, and random fields."""
    out = []
    for i in range(n):
        k = i % 5
        if k == 0:
            out.append(M.step_map(1, 0.05, 0.04 + 0.01 * (i % 3))[0])
        elif k == 1:
            out.append(M.step_map(1, -0.08, -0.03)[0])
        elif k == 2:
            out.append(M.slope_map(1, 0.1 + 0.02 * (i % 4))[0])
        elif k == 3:
            out.append(M.slope_map(1, -0.08, axis=1)[0])
        else:
            out.append(M.random_maps(1, seed + i)[0])
    return (hb.HbTerrain * n)(*out)


def _compare_with_oracle(refs, ls, maps, x0, gaits, cmd, t0, start, feet, latest, settings=None, skip=()):
    for i in range(len(refs)):
        if i in skip:
            continue
        m = maps[i]
        if settings is None:
            ms, tg, sp = M.plan(m, t0[i], T, x0[i], cmd[i], feet[i], gaits[i], start[i], latest_stance=latest[i])
        else:
            with oracle_settings(settings[i]):
                ms, tg, sp = M.plan(m, t0[i], T, x0[i], cmd[i], feet[i], gaits[i], start[i], latest_stance=latest[i])
        np.testing.assert_allclose(ls[i], sp.latest.reshape(-1), rtol=0, atol=1e-15)
        times = np.linspace(t0[i], t0[i] + T, 97)
        times = np.array([t for t in times if min([abs(t - e) for e in ms.events]) > 1e-7])
        with (oracle_settings(settings[i]) if settings is not None else _nothing()):
            xr, sw, md = R.sample(ms, tg, sp, times)
        xc, sc, mc = R.eval_compact(refs[i], times)
        np.testing.assert_array_equal(mc, md)
        np.testing.assert_allclose(xc, xr, rtol=0, atol=1e-9)
        np.testing.assert_allclose(sc, sw, rtol=0, atol=1e-11)


class _nothing:
    def __enter__(self):
        return None

    def __exit__(self, *a):
        return False


@pytest.mark.parametrize("with_settings", [False, True], ids=["compiled_in", "settings"])
def test_host_planner_on_maps_matches_the_oracle(with_settings):
    n = 40
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, 21)
    maps = _map_cases(n, 22)
    settings = random_settings(n, seed=23) if with_settings else None
    refs, ls = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, settings=settings, maps=maps)
    blind, lsb = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, settings=settings)
    # a random template can keep a foot off the ground over the whole tiled window; the blind planner and the oracle already part there,
    # so such instances are left out of both comparisons
    skip = []
    for i in range(n):
        try:
            _compare_with_oracle(blind[i:i + 1], lsb[i:i + 1], [None], x0[i:i + 1], gaits[i:i + 1], cmd[i:i + 1], t0[i:i + 1], start[i:i + 1],
                                 feet[i:i + 1], latest[i:i + 1], None if settings is None else settings[i:i + 1])
        except AssertionError:
            skip.append(i)
    assert len(skip) <= 1, skip
    _compare_with_oracle(refs, ls, maps, x0, gaits, cmd, t0, start, feet, latest, settings, skip)
    # the maps move the plans
    assert sum(bytes(refs[i]) != bytes(blind[i]) for i in range(n)) >= n - 2


def test_plateau_invariance():
    """A flat map at c with x0's z, the feet and the latest stance raised by c is the blind plan with every z raised by c."""
    n, c = 40, 0.23
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, 31)
    blind, lsb = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest)
    up = lambda a: (a.reshape(n, 4, 3) + [0.0, 0.0, c]).reshape(n, 12)
    x0c = x0.copy(); x0c[:, 8] += c
    refs, ls = hb.plan_references(t0, T, x0c, cmd, up(feet), gaits, start, latest_stance=up(latest), maps=M.plateau(n, c))
    np.testing.assert_allclose(ls, up(lsb), rtol=0, atol=1e-12)
    for i in range(n):
        times = np.linspace(t0[i], t0[i] + T, 61)
        xb, sb, mb = R.eval_compact(blind[i], times)
        xm, sm, mm = R.eval_compact(refs[i], times)
        np.testing.assert_array_equal(mb, mm)
        sb = sb.reshape(len(times), 4, 6); sm = sm.reshape(len(times), 4, 6)
        np.testing.assert_allclose(sm[..., 2], sb[..., 2] + c, rtol=0, atol=1e-12)          # swing z
        np.testing.assert_allclose(np.delete(sm, 2, axis=-1), np.delete(sb, 2, axis=-1), rtol=0, atol=1e-12)
        xb[:, 8] += c
        np.testing.assert_allclose(xm[:, :12], xb[:, :12], rtol=0, atol=1e-12)
        np.testing.assert_allclose(xm[:, 12:], xb[:, 12:], rtol=0, atol=1e-9)               # IK joints


def test_touchdown_heights_are_next_stance_z_on_the_map():
    n = 40
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, 41)
    gaits = ["trot" if i % 2 else "standing_trot" for i in range(n)]
    maps = _map_cases(n, 42)
    refs, ls = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, maps=maps)
    checked = 0
    for i in range(n):
        for c in range(4):
            segs = [[refs[i].segments[c][a][k][:] for k in range(refs[i].n_segments[c][a])] for a in range(3)]
            for z in segs[2]:
                xy = [[g for g in segs[a] if g[0] == z[0] and g[1] == z[1]] for a in range(2)]
                if z[2] == z[4] and z[3] == z[5] == 0.0 and all(len(g) == 1 and g[0][2] == g[0][4] for g in xy):    # a stance segment
                    assert z[2] == R.NEXT_Z + M.h(maps[i], xy[0][0][2], xy[1][0][2])
                    checked += 1
        for c in range(4):                          # the lift-off points
            assert ls[i, 3 * c + 2] == R.NEXT_Z + M.h(maps[i], ls[i, 3 * c], ls[i, 3 * c + 1])
    assert checked > 2 * n


def test_conversions_on_maps_match_numpy_bitwise():
    n = 60
    x0, gaits, cmd, t0, *_ = _cases(n, 51)
    x0[:, 8] += np.random.default_rng(52).uniform(-0.08, 0.08, n)          # heights on either side of the 0.04 limit
    maps = _map_cases(n, 53)
    rng = np.random.default_rng(54)
    goal = np.c_[x0[:, 6:8] + rng.uniform(-0.5, 0.5, (n, 2)), x0[:, 9] + rng.uniform(-1, 1, n)]
    goal[5, :2] = x0[5, 6:8]; goal[5, 2] = x0[5, 9]
    g = hb.goal_to_target(t0, x0, goal, maps=maps)
    for i in range(n):
        tm, st = M.goal_target_numpy(maps[i], t0[i], x0[i], goal[i])
        k = g[i].n
        assert k == len(tm)
        assert np.array(g[i].time[:k]).tobytes() == tm.tobytes()
        assert np.array([g[i].state[j][:] for j in range(k)]).tobytes() == st.tobytes()
    c = hb.cmd_vel_to_target(t0, T, x0, cmd, maps=maps)
    c0 = hb.cmd_vel_to_target(t0, T, x0, cmd)
    moved = 0
    for i in range(n):
        a, b = np.ctypeslib.as_array(c)[i], np.ctypeslib.as_array(c0)[i]
        z0, z1 = M.cmd_vel_heights_numpy(maps[i], x0[i], b["state"][1, 6:8])
        assert (a["state"][0, 8], a["state"][1, 8]) == (z0, z1)
        sa = a["state"].copy(); sa[:2, 8] = b["state"][:2, 8]
        assert a["n"] == b["n"] and a["time"].tobytes() == b["time"].tobytes() and sa.tobytes() == b["state"].tobytes()   # only the heights move
        moved += a["state"][1, 8] != b["state"][1, 8]
    assert moved > n // 2


def test_bad_maps_are_rejected_by_the_host_calls():
    n = 2
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, 61)
    bad = M.zero_maps(n)
    bad[1].spacing = 0.0
    lib = hb.load_library()
    ins = hb.make_plan_inputs(t0, T, x0, cmd, feet, gaits, start)
    refs, ls = (hb.HbReference * n)(), latest.copy()
    P = lambda a: C.c_void_p(a.ctypes.data)
    assert lib.hb_plan_references_maps(n, ins, None, None, bad, P(ls), refs) == -1
    assert lib.hb_goal_to_target_maps(n, P(t0), P(x0), P(np.zeros((n, 3))), bad, (hb.HbTarget * n)()) == -1
    assert lib.hb_cmd_vel_to_target_maps(n, P(t0), C.c_double(T), P(x0), P(cmd), bad, (hb.HbTarget * n)()) == -1
    with pytest.raises(ValueError):
        hb.plan_references(t0, T, x0, cmd, feet, gaits, start, maps=M.zero_maps(3))


def test_height_map_records_are_checked_as_terrains():
    lib = hb.load_library()
    good = M.random_maps(3, 71)
    cases = [good]
    for field, value in [("nx", 1), ("nx", 65), ("ny", 1), ("ny", 65), ("spacing", 0.0), ("spacing", -0.1), ("spacing", float("nan")),
                         ("spacing", float("inf"))]:
        r = M.random_maps(3, 71); setattr(r[1], field, value); cases.append(r)
    r = M.random_maps(3, 71); r[2].origin[0] = float("inf"); cases.append(r)
    r = M.random_maps(3, 71); r[0].height[5][7] = float("nan"); cases.append(r)
    r = M.random_maps(3, 71); r[0].height[30][30] = float("nan"); cases.append(r)            # beyond the used samples: not read
    for recs in cases:
        a, b = C.c_int32(), C.c_int32()
        ra = lib.hb_check_setting_records(api.HB_SETTING_TERRAINS, 3, recs, C.byref(a))
        rb = lib.hb_check_setting_records(api.HEIGHT_MAPS_SETTING_KIND, 3, recs, C.byref(b))
        assert (ra, a.value) == (rb, b.value)
    assert [lib.hb_check_setting_records(14, 3, c, C.byref(C.c_int32())) for c in cases] == [0] + [-1] * 10 + [0]
