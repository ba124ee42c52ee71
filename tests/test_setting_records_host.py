"""hb_check_setting_records on the host (no GPU): the setters' own record check, without a context, for every kind of per-robot setting.
Each record the builders' tests reject is rejected here as a raw record, with the index of the first rejected record; the builders'
records pass; and the builders raise with that index."""
import ctypes as C

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import api

B, AT = 4, 1              # the bad record sits at AT, and another after it: first_bad names the first
nan, inf = float("nan"), float("inf")

# kind: the records its builder makes, accepted by its setter
GOOD = {
    "pushes": (api.HB_SETTING_PUSHES, lambda: hb.make_push_schedules(B, 0.5, 0.1, [10.0, 0.0, 0.0])),
    "plant_variations": (api.HB_SETTING_PLANT_VARIATIONS,
                         lambda: hb.make_plant_variations(B, payload_mass=1.0, payload_com=[0.0, 0.0, 0.1], payload_inertia=np.diag([0.1] * 3))),
    "terrains": (api.HB_SETTING_TERRAINS, lambda: hb.make_terrains(B, np.zeros((4, 5)), 0.05)),
    "goals": (api.HB_SETTING_GOALS, lambda: hb.make_goal_schedules(B, [0.0, 1.0], [[1.0, 2.0, 0.5], [0.0, 0.0, -1.0]])),
    "odometry": (api.HB_SETTING_ODOMETRY, lambda: hb.make_odometry_settings(B, 5, 2, sigma_position=0.01, sigma_drift=0.001)),
    "controllers": (api.HB_SETTING_CONTROLLERS, lambda: hb.make_controller_settings(B)),
    "hardware": (api.HB_SETTING_HARDWARE, lambda: hb.make_hardware_settings(B)),
    "planner": (api.HB_SETTING_PLANNER, lambda: hb.make_planner_settings(B)),
    "targets": (api.HB_SETTING_TARGETS, lambda: hb.make_targets([[0.0, 1.0]] * B, [np.zeros((2, 22))] * B)),
    "latencies": (api.HB_SETTING_LATENCIES, lambda: (C.c_int32 * B)(0, 1, 5, 0)),
}

# kind: {case: [(field path, index within the record, value)]}. The cases of the five builders' tests, as records: a count or grid size
# a builder cannot even form is a record field here. One case for each other kind shows the switch reaches its predicate.
BAD = {
    "pushes": {"too_many": [("n_push", (), 5)], "negative_count": [("n_push", (), -1)], "nan_start": [("t_start", (0,), nan)],
               "inf_force": [("force", (0, 1), inf)], "nan_torque": [("torque", (0, 1), nan)], "negative_duration": [("duration", (0,), -0.1)],
               "inf_duration": [("duration", (0,), inf)]},
    "plant_variations": {
        "nan_mass": [("payload_mass", (), nan)], "negative_mass": [("payload_mass", (), -0.1)], "inf_com": [("payload_com", (1,), inf)],
        "asymmetric": [("payload_inertia", (1,), 0.01)], "negative_diagonal": [("payload_inertia", (8,), -0.01)],
        "negative_minor": [("payload_inertia", (1,), 0.2), ("payload_inertia", (3,), 0.2)],
        "negative_det": [("payload_inertia", (), [1.0, 1.0, 0.0, 1.0, 1.0, 1.0, 0.0, 1.0, 1.0])],
        "com_without_mass": [("payload_mass", (), 0.0), ("payload_inertia", (), 0.0)],
        "inertia_without_mass": [("payload_mass", (), 0.0), ("payload_com", (), 0.0)], "negative_friction": [("friction_scale", (), -0.5)],
        "zero_stiffness": [("stiffness_scale", (), 0.0)], "negative_damping": [("damping_scale", (), -1.0)],
        "negative_motor": [("motor_strength", (3,), -0.5)], "nan_motor": [("motor_strength", (9,), nan)]},
    "terrains": {"nx_small": [("nx", (), 1)], "ny_small": [("ny", (), 1)], "nx_large": [("nx", (), 65)], "ny_large": [("ny", (), 65)],
                 "nan_height": [("height", (2, 3), nan)], "inf_height": [("height", (0, 0), -inf)], "nan_origin": [("origin", (0,), nan)],
                 "inf_origin": [("origin", (1,), inf)], "zero_spacing": [("spacing", (), 0.0)], "negative_spacing": [("spacing", (), -0.05)],
                 "nan_spacing": [("spacing", (), nan)], "inf_spacing": [("spacing", (), inf)]},
    "goals": {"descending": [("time", (1,), -1.0)], "nan_time": [("time", (1,), nan)], "inf_goal": [("goal", (0, 1), inf)],
              "too_many": [("n_goal", (), 9)], "negative_count": [("n_goal", (), -1)]},
    "odometry": {"negative_period": [("period_ticks", (), -1)], "negative_delay": [("delay_ticks", (), -1)],
                 "delay_above_max": [("delay_ticks", (), 16)], "negative_sigma": [("sigma_position", (), -1e-3)],
                 "nan_drift": [("sigma_drift", (), nan)], "inf_sigma": [("sigma_position", (), inf)]},
    "controllers": {"zero_friction": [("wbc.friction_coefficient", (), 0.0)]},
    "hardware": {"negative_delay": [("actuation_delay", (), -1e-3)]},
    "planner": {"zero_time_scale": [("swing_time_scale", (), 0.0)]},
    "targets": {"no_sample": [("n", (), 0)]},
    "latencies": {"negative": [(None, (), -1)]},
}


def _check(kind, records, n=None):
    """(return code, *first_bad) of hb_check_setting_records on the first n records (all of them by default)."""
    bad = C.c_int32(7)
    rc = hb.load_library().hb_check_setting_records(kind, len(records) if n is None else n, records, C.byref(bad))
    return rc, bad.value


def _edit(records, i, changes):
    v = np.ctypeslib.as_array(records)
    for path, index, value in changes:
        field = v
        for name in path.split(".") if path else []:
            field = field[name]
        field[(i,) + index] = value


def test_every_kind_is_covered():
    kinds = sorted(v for k, v in vars(api).items() if k.startswith("HB_SETTING_"))      # the header's kinds (test_abi_layout.py)
    assert sorted(v for v, _ in GOOD.values()) == kinds and len(kinds) == 10 and set(BAD) == set(GOOD)


@pytest.mark.parametrize("name", sorted(GOOD))
def test_the_builders_records_pass(name):
    kind, good = GOOD[name]
    assert _check(kind, good()) == (0, -1)
    assert _check(kind, None, 0) == (0, -1)


@pytest.mark.parametrize("name, case", [(k, c) for k in sorted(BAD) for c in BAD[k]])
def test_a_rejected_record_is_named(name, case):
    kind, good = GOOD[name]
    records = good()
    _edit(records, AT, BAD[name][case])
    assert _check(kind, records) == (-1, AT)
    assert _check(kind, records, AT) == (0, -1)           # the records before it pass
    _edit(records, B - 1, BAD[name][case])
    assert _check(kind, records) == (-1, AT)


def test_malformed_calls_are_rejected():
    lib = hb.load_library()
    records = hb.make_push_schedules(2, 0.5, 0.1, [10.0, 0.0, 0.0])
    for kind in (-1, 10, 1 << 20):
        assert _check(kind, records) == (-1, -1)
    assert _check(api.HB_SETTING_PUSHES, None, 2) == (-1, -1)
    assert _check(api.HB_SETTING_PUSHES, records, -1) == (-1, -1)
    assert lib.hb_check_setting_records(api.HB_SETTING_PUSHES, 2, records, None) == -1


@pytest.mark.parametrize("name, build", [
    ("pushes", lambda: hb.make_push_schedules(3, [[0.0], [0.1], [0.2]], [[0.1], [-0.1], [-0.2]], [1.0, 0.0, 0.0])),
    ("plant_variations", lambda: hb.make_plant_variations(3, payload_mass=[1.0, -1.0, -2.0])),
    ("terrains", lambda: hb.make_terrains(3, np.zeros((2, 2)), [0.1, 0.0, -0.1])),
    ("goals", lambda: hb.make_goal_schedules(3, [[0.0, 1.0], [1.0, 0.0], [1.0, 0.0]], np.zeros((2, 3)))),
    ("odometry", lambda: hb.make_odometry_settings(3, 5, [0, 16, 17])),
])
def test_the_builders_name_the_first_rejected_record(name, build):
    with pytest.raises(ValueError, match="^%s: record 1 is rejected by hb_rollout_set_%s$" % (name, name)):
        build()
