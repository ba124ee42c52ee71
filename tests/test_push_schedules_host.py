"""Push schedules on the host (no GPU): the ctypes layout of hb_push_schedule and what make_push_schedules builds and rejects."""
import ctypes as C

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb


def test_layout_matches_the_header():
    assert C.sizeof(hb.HbPushSchedule) == 264
    assert hb.HbPushSchedule.t_start.offset == 8 and hb.HbPushSchedule.torque.offset == 264 - 96
    assert hb.HB_MAX_PUSHES == 4


def test_make_push_schedules_broadcasts():
    S = hb.make_push_schedules(3, [0.5, 0.7], 0.1, [[10.0, 0.0, 0.0], [0.0, -20.0, 0.0]])
    assert len(S) == 3 and all(s.n_push == 2 for s in S)
    assert [S[2].t_start[j] for j in range(2)] == [0.5, 0.7] and [S[1].duration[j] for j in range(2)] == [0.1, 0.1]
    assert list(S[0].force[1]) == [0.0, -20.0, 0.0] and list(S[0].torque[0]) == [0.0, 0.0, 0.0]
    S = hb.make_push_schedules(2, [[0.1], [0.2]], [[0.05], [0.0]], [[[1.0, 2.0, 3.0]], [[4.0, 5.0, 6.0]]], [0.0, 0.0, 7.0])
    assert S[1].t_start[0] == 0.2 and S[1].duration[0] == 0.0 and list(S[1].force[0]) == [4.0, 5.0, 6.0] and S[0].torque[0][2] == 7.0
    S = hb.make_push_schedules(2, 0.3, 0.1, [1.0, 0.0, 0.0])
    assert S[0].n_push == 1 and S[1].force[0][0] == 1.0
    S = hb.make_push_schedules(2, np.zeros((2, 0)), np.zeros((2, 0)), np.zeros((2, 0, 3)))
    assert S[0].n_push == 0 and S[1].n_push == 0


@pytest.mark.parametrize("case", ["too_many", "nan_start", "inf_force", "nan_torque", "negative_duration", "inf_duration", "shape"])
def test_make_push_schedules_rejects_what_the_c_call_rejects(case):
    t, d, f, tq = np.zeros((2, 1)), np.full((2, 1), 0.1), np.zeros((2, 1, 3)), None
    if case == "too_many":
        t, d, f = np.zeros((2, 5)), np.zeros((2, 5)), np.zeros((2, 5, 3))
    elif case == "nan_start":
        t[1, 0] = np.nan
    elif case == "inf_force":
        f[0, 0, 1] = np.inf
    elif case == "nan_torque":
        tq = [0.0, np.nan, 0.0]
    elif case == "negative_duration":
        d[0, 0] = -0.1
    elif case == "inf_duration":
        d[1, 0] = np.inf
    else:
        f = np.zeros((3, 1, 3))
    with pytest.raises(ValueError):
        hb.make_push_schedules(2, t, d, f, tq)
