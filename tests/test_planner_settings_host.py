"""Planner settings on the host (no GPU): the default record and the parser against the shipped files and the header, the validity rules,
hb_plan_references_settings against hb_plan_references_targets and against oracle/refs.py planning with the same record over random
templates and swing settings, the capacity limits a short template runs into, and make_planner_settings."""
import ctypes as C
import os

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios
from oracle import refs as R
from planner_settings_ref import GAIT_NAMES, oracle_settings, random_settings, template_lists

N, DT = 40, 0.02
T = N * DT
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TASK, GAIT = os.path.join(GOLDEN, "hunter_config", "task.info"), os.path.join(GOLDEN, "hunter_config", "gait.info")
SWING_MACROS = dict(swing_height="HB_SWING_HEIGHT", swing_time_scale="HB_SWING_TIME_SCALE", next_stance_z="HB_NEXT_POSITION_Z",
                    feet_bias_x1="HB_FEET_BIAS_X1", feet_bias_x2="HB_FEET_BIAS_X2", feet_bias_y="HB_FEET_BIAS_Y", feet_bias_z="HB_FEET_BIAS_Z")
SHIPPED = {"stance": ([3], [0.0, 0.5]), "trot": ([2, 1], [0.0, 0.3, 0.6]), "standing_trot": ([2, 3, 1, 3], [0.0, 0.25, 0.3, 0.55, 0.6]),
           "flying_trot": ([2, 0, 1, 0], [0.0, 0.15, 0.2, 0.35, 0.4])}      # gait.info


def _cases(n, seed):
    """Plan inputs of n instances over the four gaits, started before or shortly after t0, with feet near their nominal footholds."""
    rng = np.random.default_rng(seed)
    x0 = scenarios.random_initial_states(n, seed=seed)
    gaits = [GAIT_NAMES[i % 4] for i in range(n)]
    cmd = np.stack([rng.uniform(-0.6, 0.8, n), rng.uniform(-0.2, 0.2, n), np.zeros(n), rng.uniform(-0.5, 0.5, n)], axis=1)
    t0 = rng.uniform(0.0, 3.0, n)
    start = t0 + rng.uniform(-1.3, 0.3, n)
    feet = np.zeros((n, 4, 3))
    for i in range(n):
        Ry = R.rot_zyx([x0[i, 9], 0, 0])
        for c in range(4):
            feet[i, c] = x0[i, 6:9] + Ry @ np.array(R.FEET_BIAS[c]) + rng.normal(0, 0.01, 3)
    latest = feet + rng.normal(0, 0.02, feet.shape)
    return x0, gaits, cmd, t0, start, feet.reshape(n, 12), latest.reshape(n, 12)


def _plan_rc(settings, n=1, seed=3, **over):
    """hb_plan_references_settings' return code on n instances of _cases with the records settings (ctypes array of n)."""
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, seed)
    kw = dict(t0=t0, horizon=T, x0=x0, cmd_vel=cmd, feet_pos=feet, gait=gaits, gait_start=start)
    kw.update(over)
    ins = hb.make_plan_inputs(**kw)
    refs = (hb.HbReference * n)()
    ls = latest.copy()
    return hb.load_library().hb_plan_references_settings(n, ins, None, settings, C.c_void_p(ls.ctypes.data), refs)


def test_default_record_is_the_compiled_in_planner():
    s = hb.default_planner_settings()
    assert C.sizeof(hb.HbGaitTemplate) == 112 and C.sizeof(hb.HbPlannerSettings) == 504
    for field, macro in SWING_MACROS.items():
        assert getattr(s, field) == R._header_value(macro), field
    for g, name in enumerate(GAIT_NAMES):
        assert template_lists(s.gait[g]) == SHIPPED[name]
        assert list(s.gait[g].modes[s.gait[g].n_phase:]) == [0] * (8 - s.gait[g].n_phase)
        assert list(s.gait[g].switching_times[s.gait[g].n_phase + 1:]) == [0.0] * (8 - s.gait[g].n_phase)


def test_parse_shipped_files_gives_the_default():
    assert bytes(hb.parse_planner_settings(TASK, GAIT)) == bytes(hb.default_planner_settings())


def test_parse_variant_files():
    s = hb.parse_planner_settings(os.path.join(GOLDEN, "task_swing_variant.info"), os.path.join(GOLDEN, "gait_variant.info"))
    assert (s.swing_height, s.swing_time_scale, s.next_stance_z) == (0.07, 0.2, 0.025)
    assert (s.feet_bias_x1, s.feet_bias_x2, s.feet_bias_y, s.feet_bias_z) == (0.04, -0.05, 0.12, -0.6)
    assert template_lists(s.gait[0]) == ([3], [0.0, 0.4])
    assert template_lists(s.gait[1]) == ([2, 3, 1, 3], [0.0, 0.3, 0.4, 0.7, 0.8])
    assert template_lists(s.gait[2]) == ([3, 0], [0.0, 0.25, 0.35])             # list order, not file order
    assert template_lists(s.gait[3]) == ([2, 3, 1, 3], [0.0, 0.35, 0.45, 0.8, 0.9])


def _write(tmp_path, name, text):
    p = tmp_path / name
    p.write_text(text)
    return str(p)


def test_missing_files_and_keys_follow_parse_task_info(tmp_path):
    d = hb.default_planner_settings()
    with pytest.raises(hb.HunterB200Error, match="-1"):
        hb.parse_planner_settings(str(tmp_path / "none.info"), GAIT)
    with pytest.raises(hb.HunterB200Error, match="-1"):
        hb.parse_planner_settings(TASK, str(tmp_path / "none.info"))
    with pytest.raises(hb.HunterB200Error):
        hb.parse_task_info(str(tmp_path / "none.info"))
    # absent sections and keys keep the defaults, as hb_parse_task_info's do
    empty = _write(tmp_path, "empty.info", "; nothing\n")
    assert bytes(hb.parse_planner_settings(empty, empty)) == bytes(d)
    task = _write(tmp_path, "task.info", "swing_trajectory_config\n{\n  swingHeight 0.09\n}\n")
    gait = _write(tmp_path, "gait.info", "list\n{\n  [0] stance\n  [1] fast\n  [2] nowhere\n}\n"
                                         "fast\n{\n  modeSequence\n  {\n    [0] L\n    [1] R\n  }\n  switchingTimes\n  {\n    [0] 0.0\n    [1] 0.2\n    [2] 0.4\n  }\n}\n")
    s = hb.parse_planner_settings(task, gait)
    assert s.swing_height == 0.09 and s.swing_time_scale == d.swing_time_scale and s.next_stance_z == d.next_stance_z
    assert template_lists(s.gait[1]) == ([2, 1], [0.0, 0.2, 0.4])
    for g in (0, 2, 3):                      # stance: not in the file; nowhere: not in the file; [3]: not in the list
        assert bytes(s.gait[g]) == bytes(d.gait[g])


@pytest.mark.parametrize("body", [
    "modeSequence\n{\n [0] L\n [1] JUMP\n}\nswitchingTimes\n{\n [0] 0.0\n [1] 0.2\n [2] 0.4\n}",          # unknown mode name
    "modeSequence\n{\n [0] L\n [1] R\n}\nswitchingTimes\n{\n [0] 0.0\n [1] 0.2\n}",                       # n modes, n times
    "modeSequence\n{\n [0] L\n}",                                                                            # no times
    "modeSequence\n{\n" + "".join(" [%d] L\n" % k for k in range(9)) + "}\nswitchingTimes\n{\n" + "".join(" [%d] %g\n" % (k, 0.1 * k) for k in range(10)) + "}",
    "modeSequence\n{\n [0] L\n [1] R\n}\nswitchingTimes\n{\n [0] 0.0\n [1] soon\n [2] 0.4\n}",           # not a number
    "modeSequence\n{\n [0] L\n [1] R\n}\nswitchingTimes\n{\n [0] 0.1\n [1] 0.2\n [2] 0.4\n}",            # does not start at 0
    "modeSequence\n{\n [0] L\n [1] R\n}\nswitchingTimes\n{\n [0] 0.0\n [1] 0.4\n [2] 0.4\n}",            # not strictly ascending
], ids=["mode_name", "counts", "no_times", "nine_phases", "not_a_number", "start", "ascending"])
def test_malformed_templates_are_rejected(tmp_path, body):
    gait = _write(tmp_path, "gait.info", "list\n{\n  [1] g\n}\ng\n{\n%s\n}\n" % body)
    with pytest.raises(hb.HunterB200Error, match="-1"):
        hb.parse_planner_settings(TASK, gait)


def test_unbalanced_file_is_rejected(tmp_path):
    with pytest.raises(hb.HunterB200Error, match="-1"):
        hb.parse_planner_settings(_write(tmp_path, "task.info", "swing_trajectory_config\n{\n  swingHeight 0.09\n"), GAIT)


def _bad_records():
    """(name, record) of every validity rule of hb_planner_settings, each broken once."""
    out = []

    def rec(fn):
        r = hb.make_planner_settings(1)
        fn(r[0])
        return r

    nan, inf = float("nan"), float("inf")
    out.append(("n_phase_0", rec(lambda r: setattr(r.gait[1], "n_phase", 0))))
    out.append(("n_phase_9", rec(lambda r: setattr(r.gait[2], "n_phase", 9))))
    out.append(("mode_neg", rec(lambda r: r.gait[1].modes.__setitem__(0, -1))))
    out.append(("mode_4", rec(lambda r: r.gait[3].modes.__setitem__(3, 4))))
    out.append(("start", rec(lambda r: r.gait[0].switching_times.__setitem__(0, 0.01))))
    out.append(("start_nan", rec(lambda r: r.gait[0].switching_times.__setitem__(0, nan))))
    out.append(("equal", rec(lambda r: r.gait[1].switching_times.__setitem__(2, 0.3))))
    out.append(("descending", rec(lambda r: r.gait[2].switching_times.__setitem__(2, 0.2))))
    out.append(("time_nan", rec(lambda r: r.gait[3].switching_times.__setitem__(4, nan))))
    out.append(("time_inf", rec(lambda r: r.gait[3].switching_times.__setitem__(4, inf))))
    for f, v in [("swing_height", -1e-3), ("swing_height", nan), ("swing_height", inf), ("swing_time_scale", 0.0), ("swing_time_scale", -0.1),
                 ("swing_time_scale", inf), ("swing_time_scale", nan), ("next_stance_z", nan), ("feet_bias_x1", inf), ("feet_bias_x2", -inf),
                 ("feet_bias_y", nan), ("feet_bias_z", inf)]:
        out.append(("%s=%g" % (f, v), hb.make_planner_settings(1, **{f: v})))
    return out


@pytest.mark.parametrize("name,rec", _bad_records(), ids=[n for n, _ in _bad_records()])
def test_every_validity_rule_rejects(name, rec):
    assert _plan_rc(rec) == -1
    with pytest.raises(hb.HunterB200Error):
        x0, gaits, cmd, t0, start, feet, latest = _cases(1, 3)
        hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, settings=rec)


def test_unused_entries_are_not_read():
    rec = hb.make_planner_settings(1, gaits={"trot": (["L", "R"], [0.0, 0.3, 0.6])})
    rec[0].gait[1].modes[5] = 17; rec[0].gait[1].switching_times[7] = float("nan")
    assert _plan_rc(rec) == 0


@pytest.mark.parametrize("with_targets", [False, True], ids=["cmd_vel", "targets"])
def test_null_and_default_settings_are_the_targets_planner_bitwise(with_targets):
    n = 64
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, seed=7)
    tg = None
    if with_targets:
        tg = hb.goal_to_target(t0, x0, np.stack([x0[:, 6] + 0.4, x0[:, 7] - 0.2, x0[:, 9] + 0.3], axis=1))
    want, lw = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, targets=tg)
    lib = hb.load_library()
    ins = hb.make_plan_inputs(t0, T, x0, cmd, feet, gaits, start)
    for settings in (None, hb.make_planner_settings(n), hb.parse_planner_settings(TASK, GAIT)):
        if isinstance(settings, hb.HbPlannerSettings):
            settings = (hb.HbPlannerSettings * n)(*[settings] * n)
        refs = (hb.HbReference * n)()
        ls = latest.copy()
        assert lib.hb_plan_references_settings(n, ins, tg, settings, C.c_void_p(ls.ctypes.data), refs) == 0
        assert bytes(refs) == bytes(want) and np.array_equal(ls, lw)


def test_matches_the_restatement_with_random_settings():
    """Random templates of 1..8 phases (FLY and STANCE among the modes) and random swing settings, per instance: the plan equals
    oracle/refs.py planning with the same record, at test_planner.py's tolerances."""
    n = 48
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, seed=19)
    settings = random_settings(n, seed=5)
    modes_seen = set()
    refs, ls = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, settings=settings)
    for i in range(n):
        with oracle_settings(settings[i]):
            ms, tg, sp = R.plan(t0[i], T, x0[i], cmd[i], feet[i], gaits[i], start[i], latest_stance=latest[i])
        np.testing.assert_allclose(ls[i], sp.latest.reshape(-1), rtol=0, atol=1e-15)
        times = np.concatenate([t0[i] + DT * np.arange(N + 1), t0[i] + np.random.default_rng(i).uniform(0, T, 40)])
        times = np.array([t for t in times if min([abs(t - e) for e in ms.events]) > 1e-7])
        xr, sw, md = R.sample(ms, tg, sp, times)
        xc, sc, mc = R.eval_compact(refs[i], times)
        np.testing.assert_array_equal(md, mc)
        np.testing.assert_allclose(xc, xr, rtol=0, atol=1e-9)
        np.testing.assert_allclose(sc, sw, rtol=0, atol=1e-11)
        modes_seen |= set(int(m) for m in mc)
        assert R.GAITS[gaits[i]] == SHIPPED[gaits[i]]          # restored after the block
    assert modes_seen == {0, 1, 2, 3}


def test_settings_move_the_plan():
    """Each kind of field acts: a record differing from the default in one field plans differently."""
    n = 8
    x0, gaits, cmd, t0, start, feet, latest = _cases(n, seed=29)
    gaits = ["trot"] * n
    base, _ = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest)
    for kw in (dict(swing_height=0.08), dict(swing_time_scale=0.5), dict(next_stance_z=0.03), dict(feet_bias_x1=0.05), dict(feet_bias_y=0.13),
               dict(gaits={"trot": (["L", "R"], [0.0, 0.25, 0.5])})):
        refs, _ = hb.plan_references(t0, T, x0, cmd, feet, gaits, start, latest_stance=latest, settings=hb.make_planner_settings(n, **kw))
        assert bytes(refs) != bytes(base), kw


@pytest.mark.parametrize("case", ["phases", "events", "segments"])
def test_templates_too_short_for_the_capacities(case):
    """A valid template that tiles more than 128 phases over [t0 - T, t0 + 2T], puts more than HB_MAX_EVENTS events into the horizon or
    more than HB_MAX_SEGMENTS segments on a foot gives -5."""
    if case == "phases":            # 2 x 0.005 s: about 480 phases
        rec, over = hb.make_planner_settings(1, gaits={"stance": (["STANCE", "STANCE"], [0.0, 0.005, 0.01])}), dict(gait="stance")
    elif case == "events":          # horizon 0.3 s: about 37 events inside it, 115 phases tiled
        rec, over = hb.make_planner_settings(1, gaits={"stance": (["STANCE", "STANCE"], [0.0, 0.008, 0.016])}), dict(gait="stance", horizon=0.3)
    else:                           # a trot of 2 x 0.03 s: 27 swings per foot in the horizon
        rec, over = hb.make_planner_settings(1, gaits={"trot": (["L", "R"], [0.0, 0.03, 0.06])}), dict(gait="trot")
    x0, _, _, t0, _, _, _ = _cases(1, 3)
    over.setdefault("horizon", T)
    assert _plan_rc(rec, gait_start=t0 - 5.0, **over) == -5
    assert _plan_rc(hb.make_planner_settings(1), gait_start=t0 - 5.0, **over) == 0


def test_make_planner_settings():
    d = hb.default_planner_settings()
    s = hb.make_planner_settings(3)
    assert all(bytes(r) == bytes(d) for r in s)
    base = hb.default_planner_settings(); base.feet_bias_y = 0.1
    s = hb.make_planner_settings(4, base=base, swing_height=[0.01, 0.02, 0.03, 0.04], swing_time_scale=0.2,
                                 gaits={"trot": (["L", "STANCE", "R", "STANCE"], [0.0, 0.2, 0.25, 0.45, 0.5]),
                                        3: [(["FLY"], [0.0, 0.1 * (i + 1)]) for i in range(4)]})
    assert base.feet_bias_y == 0.1 and bytes(base.gait[1]) == bytes(d.gait[1])
    for i, r in enumerate(s):
        assert r.swing_height == 0.01 * (i + 1) and r.swing_time_scale == 0.2 and r.feet_bias_y == 0.1 and r.next_stance_z == d.next_stance_z
        assert template_lists(r.gait[1]) == ([2, 3, 1, 3], [0.0, 0.2, 0.25, 0.45, 0.5])
        assert template_lists(r.gait[3]) == ([0], [0.0, 0.1 * (i + 1)])
        assert bytes(r.gait[0]) == bytes(d.gait[0]) and bytes(r.gait[2]) == bytes(d.gait[2])
    t = hb.gait_template([3, "L"], [0, 0.1, 0.3])
    s = hb.make_planner_settings(2, gaits={"standing_trot": t})
    assert bytes(s[0].gait[2]) == bytes(s[1].gait[2]) == bytes(t)
    for bad in (dict(swing_hieght=0.1), dict(swing_height=[0.1, 0.2, 0.3]), dict(gaits={"gallop": ([1], [0, 1])}),
                dict(gaits={5: ([1], [0, 1])}), dict(gaits={"trot": (["L", "JUMP"], [0, 0.1, 0.2])}), dict(gaits={"trot": (["L"], [0, 0.1, 0.2])}),
                dict(gaits={"trot": ([1] * 9, list(range(10)))}), dict(gaits={"trot": [(["L"], [0, 0.1])] * 3})):
        with pytest.raises((ValueError, KeyError)):
            hb.make_planner_settings(2, **bad)


def test_exported():
    lib = hb.load_library()
    for s in ("hb_default_planner_settings", "hb_parse_planner_settings", "hb_plan_references_settings", "hb_plan_set_settings"):
        assert s in hb.EXPORTED_SYMBOLS and hasattr(lib, s)
