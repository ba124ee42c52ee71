"""Teleoperation on the host (no GPU): the hb_teleop_setting record against the header and the reference's joystick and publisher, every
rejected record through hb_check_setting_records, the make_teleop_settings shapes, hand-computed publisher sequences of the numpy
restatement, and hb_cmd_vel_to_target against the target of a joint_ik = 0 host plan."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import api, scenarios
from teleop_ref import message_due, publish, publisher_step

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "hunter_b200.h")).read()
KIND = hb.HbTeleop.SETTING_KIND
INT32_MAX = 2 ** 31 - 1
nan, inf = float("nan"), float("inf")


def _check(records, n=None):
    bad = C.c_int32(7)
    rc = hb.load_library().hb_check_setting_records(KIND, len(records) if n is None else n, records, C.byref(bad))
    return rc, bad.value


def test_record_layout_and_kind_follow_the_header():
    assert C.sizeof(hb.HbTeleopSetting) == 64 and hb.HbTeleop is hb.HbTeleopSetting
    assert int(re.search(r"^#define HB_MAX_TELEOP_WINDOWS (\d+)", HEADER, re.M).group(1)) == hb.HB_MAX_TELEOP_WINDOWS == 4
    assert int(re.search(r"^#define HB_SETTING_TELEOP (\d+)", HEADER, re.M).group(1)) == KIND == 12
    assert not hasattr(api, "HB_SETTING_TELEOP")            # the module's HB_SETTING_* set stays the ten kinds of test_setting_records_host
    lib = hb.load_library()
    for name in ("hb_default_teleop_setting", "hb_rollout_set_teleop", "hb_cmd_vel_to_target"):
        assert name in hb.EXPORTED_SYMBOLS and hasattr(lib, name)
    assert lib.hb_default_teleop_setting(None) == -1
    assert lib.hb_rollout_set_teleop(None, 1, hb.make_teleop_settings(1)) == -1


def test_default_record_is_the_reference_joystick_and_publisher():
    """joy_teleop.launch: autorepeat_rate 10 Hz (a message every 50 ticks of 2 ms); the deadman held throughout; changeLimit_ (0.1, 0.05,
    ., 0.3) of TargetTrajectoriesPublisher.h:97 on vx, vy and the yaw rate."""
    d = hb.default_teleop_setting()
    assert d.period_ticks == 50 and d.n_window == 1 and d.on_tick[0] == 0 and d.off_tick[0] == INT32_MAX
    assert list(d.change_limit) == [0.1, 0.05, 0.3]
    assert list(d.on_tick[1:]) == [0] * 3 and list(d.off_tick[1:]) == [0] * 3
    assert bytes(hb.make_teleop_settings(1)[0]) == bytes(d)
    assert hb.default_rollout_params().period * d.period_ticks == pytest.approx(0.1)


# each case edits record AT of four default records
BAD = {
    "zero_period": [("period_ticks", (), 0)], "negative_period": [("period_ticks", (), -50)],
    "negative_windows": [("n_window", (), -1)], "too_many_windows": [("n_window", (), 5)],
    "negative_on": [("on_tick", (0,), -5)], "empty_window": [("off_tick", (0,), 0)], "reversed_window": [("on_tick", (0,), 10), ("off_tick", (0,), 5)],
    "overlap": [("n_window", (), 2), ("off_tick", (0,), 100), ("on_tick", (1,), 95), ("off_tick", (1,), 200)],
    "descending": [("n_window", (), 2), ("on_tick", (0,), 100), ("off_tick", (0,), 200), ("on_tick", (1,), 0), ("off_tick", (1,), 50)],
    "zero_limit": [("change_limit", (1,), 0.0)], "negative_limit": [("change_limit", (0,), -0.1)], "nan_limit": [("change_limit", (2,), nan)],
    "minus_inf_limit": [("change_limit", (2,), -inf)],
}
B, AT = 4, 1


def _edit(records, i, changes):
    v = np.ctypeslib.as_array(records)
    for name, index, value in changes:
        v[name][(i,) + index] = value


@pytest.mark.parametrize("case", sorted(BAD))
def test_every_rejected_record_is_named(case):
    records = hb.make_teleop_settings(B)
    assert _check(records) == (0, -1)
    _edit(records, AT, BAD[case])
    assert _check(records) == (-1, AT)
    assert _check(records, AT) == (0, -1)
    _edit(records, B - 1, BAD[case])
    assert _check(records) == (-1, AT)


def test_the_builder_names_the_first_rejected_record():
    with pytest.raises(ValueError, match="^teleop: record 1 is rejected by hb_rollout_set_teleop$"):
        hb.make_teleop_settings(3, windows=[[(0, 10)], [(20, 10)], [(30, 10)]])
    with pytest.raises(ValueError, match="^teleop: record 2 is rejected by hb_rollout_set_teleop$"):
        hb.make_teleop_settings(3, change_limit=[[1, 1, 1], [1, 1, 1], [1, 0, 1]])


def test_accepted_edge_records():
    r = hb.make_teleop_settings(3, period_ticks=[1, 5, 50], windows=[[], [(0, 1)], [(0, 50), (50, 100), (100, 150), (150, INT32_MAX)]],
                                change_limit=[inf, inf, inf])
    assert _check(r) == (0, -1)
    assert [x.n_window for x in r] == [0, 1, 4]
    _edit(r, 0, [("on_tick", (3,), -7), ("change_limit", (0,), inf)])       # entries beyond n_window are not read
    assert _check(r) == (0, -1)


def test_make_teleop_settings_shapes():
    r = hb.make_teleop_settings(3, period_ticks=[10, 20, 30], windows=[(0, 100), (200, 300)], change_limit=[[1, 2, 3], [4, 5, 6], [7, 8, 9]])
    v = np.ctypeslib.as_array(r)
    assert list(v["period_ticks"]) == [10, 20, 30] and list(v["n_window"]) == [2] * 3
    assert (v["on_tick"][:, :2] == [0, 200]).all() and (v["off_tick"][:, :2] == [100, 300]).all() and (v["on_tick"][:, 2:] == 0).all()
    assert (v["change_limit"] == [[1, 2, 3], [4, 5, 6], [7, 8, 9]]).all()
    r = hb.make_teleop_settings(2, windows=np.array([[[0, 50]], [[100, 150]]]))            # (B, n, 2)
    assert [(x.on_tick[0], x.off_tick[0]) for x in r] == [(0, 50), (100, 150)]
    r = hb.make_teleop_settings(2, windows=[[(0, 50), (60, 70)], []])                        # B ragged sequences
    assert [x.n_window for x in r] == [2, 0]
    assert hb.make_teleop_settings(2, windows=np.zeros((0, 2)))[1].n_window == 0
    for kw, msg in [(dict(period_ticks=[1, 2, 3]), "period_ticks"), (dict(period_ticks=2.5), "int32"), (dict(windows=[(0, 1.5)]), "int32"),
                    (dict(windows=[(0, 2 ** 31)]), "int32"), (dict(windows=[(0, 1)] * 5), "at most 4"), (dict(change_limit=[1, 2]), "change_limit"),
                    (dict(windows=[[(0, 1)]] * 3), "windows")]:
        with pytest.raises(ValueError, match=msg):
            hb.make_teleop_settings(2, **kw)


def test_message_rule():
    s = hb.make_teleop_settings(1, period_ticks=10, windows=[(20, 45), (100, 121)])[0]
    assert [a for a in range(150) if message_due(s, a)] == [20, 30, 40, 100, 110, 120]
    assert not any(message_due(hb.make_teleop_settings(1, windows=[])[0], a) for a in range(200))


def test_publisher_sequences():
    lim = hb.default_teleop_setting().change_limit
    # 0 -> 0.5 m/s forward: 0.1 per message, 0.5 exactly on the 5th message
    seq = [publisher_step(np.zeros(4), [0.5, 0, 0, 0], lim)]
    for _ in range(5):
        seq.append(publisher_step(seq[-1], [0.5, 0, 0, 0], lim))
    assert [s[0] for s in seq] == [0.1, 0.2, 0.30000000000000004, 0.4, 0.5, 0.5]
    # vy at 0.05 per message (0.12 on the third), vz dropped, the yaw rate at 0.3 per message
    last, seen = np.zeros(4), []
    for _ in range(3):
        last = publisher_step(last, [0.0, 0.12, 0.7, -1.0], lim)
        seen.append((last[1], last[2], last[3]))
    assert seen == [(0.05, 0.0, -0.3), (0.1, 0.0, -0.6), (0.12, 0.0, -0.8999999999999999)]
    # a negative step from 0.3: down by 0.1 per message, the fifth step the remaining 0.05 to -0.15
    last, xs = np.array([0.3, 0.0, 0.0, 0.0]), []
    for _ in range(6):
        last = publisher_step(last, [-0.15, 0, 0, 0], lim)
        xs.append(last[0])
    assert xs == [0.19999999999999998, 0.09999999999999998, -2.7755575615628914e-17, -0.10000000000000003, -0.15, -0.15]
    # no limit: the message, as last + (cmd - last) rounds it
    assert list(publisher_step(np.array([0.2, 0.1, 0.5, 0.3]), [-0.4, 0.3, 0.9, 1.2], [inf] * 3)) == [-0.4000000000000001, 0.3, 0.0, 1.2]
    # publish() over ticks: the default record at 10 Hz sends ticks 0, 50, 100, ...
    sent, lasts = publish(hb.default_teleop_setting(), [[0.5, 0, 0, 0]] * 300, range(300))
    assert sent == [0, 50, 100, 150, 200, 250] and lasts[4, 0] == 0.5


def test_cmd_vel_to_target_is_the_joint_ik_0_host_plan():
    n, T = 48, 0.8
    rng = np.random.default_rng(3)
    x0 = scenarios.random_initial_states(n, seed=3)
    cmd = np.stack([rng.uniform(-0.6, 0.8, n), rng.uniform(-0.2, 0.2, n), rng.uniform(-0.1, 0.1, n), rng.uniform(-0.5, 0.5, n)], axis=1)
    cmd[:4, :2] = [[0.03, 0.3], [0.3, 0.03], [0.03, 0.03], [0.0, 0.0]]          # the dead band on x, then on y, both, none moving
    t0 = rng.uniform(0.0, 3.0, n)
    plain, _ = hb.plan_references(t0, T, x0, cmd, np.zeros((n, 12)), "trot", t0 - 0.2, joint_ik=False)
    tg = hb.cmd_vel_to_target(t0, T, x0, cmd)
    for i in range(n):
        assert tg[i].n == plain[i].n_targets == 2
        assert bytes(tg[i].time)[:16] == bytes(plain[i].target_times)[:16]
        assert bytes(tg[i].state)[:2 * 22 * 8] == bytes(plain[i].target_states)[:2 * 22 * 8]
        assert not any(bytes(tg[i].state)[2 * 22 * 8:]) and not any(bytes(tg[i].time)[16:])
    assert bytes(hb.cmd_vel_to_target(t0[5], T, x0[5], cmd[5])[0]) == bytes(tg[5])          # scalar t, one state
    lib = hb.load_library()
    out = (hb.HbTarget * 2)()
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    t, x, c = np.zeros(2), np.tile(x0[0], (2, 1)), np.zeros((2, 4))
    assert lib.hb_cmd_vel_to_target(2, P(t), C.c_double(T), P(x), P(c), out) == 0
    assert lib.hb_cmd_vel_to_target(-1, P(t), C.c_double(T), P(x), P(c), out) == -1
    assert lib.hb_cmd_vel_to_target(2, P(t), C.c_double(nan), P(x), P(c), out) == -1
    for a, k in ((t, 1), (x, 22 + 9), (c, 7)):
        saved = a.flat[k]
        a.flat[k] = nan
        assert lib.hb_cmd_vel_to_target(2, P(t), C.c_double(T), P(x), P(c), out) == -1
        a.flat[k] = saved
    for k in range(5):
        args = [P(t), C.c_double(T), P(x), P(c), out]
        args[[0, 2, 3, 4][min(k, 3)]] = None
        assert lib.hb_cmd_vel_to_target(2, *args) == -1


def test_the_sweep_tool_parses_its_help():
    import subprocess
    import sys
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "teleop_sweep.py"), "--help"], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    assert out.stdout.startswith("usage: teleop_sweep.py") and "--batch" in out.stdout and "--repeats" in out.stdout
