"""Planner settings for the tests of hb_planner_settings (test_planner_settings_host.py, test_gpu_planner_settings.py): random valid
records, and the per-phase restatement of oracle/refs.py planning with a record. The restatement reads its gait templates and swing
constants from module globals (GAITS, SWING_HEIGHT, SWING_TIME_SCALE, NEXT_Z, FEET_BIAS); `oracle_settings` sets them from a record for
the duration of a with block, so the oracle's planner itself plans with the record."""
import contextlib

import numpy as np

import hunter_bipedal_control_b200 as hb
from oracle import refs as R

GAIT_NAMES = ["stance", "trot", "standing_trot", "flying_trot"]     # hb_plan_input.gait 0..3
_GLOBALS = ("GAITS", "SWING_HEIGHT", "SWING_TIME_SCALE", "NEXT_Z", "FEET_BIAS")


def template_lists(t):
    """(modes, switching_times) of an HbGaitTemplate as lists."""
    n = t.n_phase
    return [int(m) for m in t.modes[:n]], [float(x) for x in t.switching_times[:n + 1]]


@contextlib.contextmanager
def oracle_settings(rec):
    """oracle/refs.py plans with the HbPlannerSettings rec inside the block (its module constants restored after it)."""
    saved = {k: getattr(R, k) for k in _GLOBALS}
    try:
        R.GAITS = {GAIT_NAMES[g]: template_lists(rec.gait[g]) for g in range(4)}
        R.SWING_HEIGHT, R.SWING_TIME_SCALE, R.NEXT_Z = rec.swing_height, rec.swing_time_scale, rec.next_stance_z
        x1, x2, y, z = rec.feet_bias_x1, rec.feet_bias_x2, rec.feet_bias_y, rec.feet_bias_z
        R.FEET_BIAS = [(x1, y, z), (x1, -y, z), (x2, y, z), (x2, -y, z)]
        yield
    finally:
        for k, v in saved.items():
            setattr(R, k, v)


def random_template(rng, max_phases=hb.HB_GAIT_MAX_PHASES, lo=0.1, hi=0.3):
    """A template of 1..max_phases phases of random modes (FLY and STANCE included) and durations in [lo, hi)."""
    n = int(rng.integers(1, max_phases + 1))
    modes = [int(m) for m in rng.integers(0, 4, n)]
    return modes, np.concatenate([[0.0], np.cumsum(rng.uniform(lo, hi, n))]).tolist()


def random_settings(B, seed):
    """B valid records with a random template for every gait and random swing settings around the shipped ones."""
    rng = np.random.default_rng(seed)
    gaits = {g: [random_template(rng) for _ in range(B)] for g in range(4)}
    return hb.make_planner_settings(B, gaits=gaits, swing_height=rng.uniform(0.0, 0.1, B), swing_time_scale=rng.uniform(0.05, 0.4, B),
                                    next_stance_z=rng.uniform(0.0, 0.04, B), feet_bias_x1=rng.uniform(0.0, 0.06, B),
                                    feet_bias_x2=rng.uniform(-0.08, -0.02, B), feet_bias_y=rng.uniform(0.08, 0.14, B),
                                    feet_bias_z=rng.uniform(-0.66, -0.58, B))
