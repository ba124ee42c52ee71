"""Contact detection on the host (no GPU): the rule's body (hb_contact_state_host) against contact_detection_ref's restatement of the
reference on the shipped and variant gaits and on random schedules, its truth table, the default records from task.info, the record check
of kind 20, the builders and the header's layout."""
import ctypes as C
import os

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import api
import contact_detection_ref as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TASK = os.path.join(GOLDEN, "hunter_config", "task.info")


def _planned_states(settings=None):
    """Estimation states holding the schedules the host planner makes for every gait, over the horizon from t0 = 0.3."""
    gaits = list(hb.GAIT_IDS)
    B = len(gaits)
    x0 = np.zeros((B, 22)); x0[:, 8] = 0.9
    refs, _ = hb.plan_references(np.full(B, 0.3), 1.0, x0, np.zeros(4), np.zeros((B, 12)), gaits, 0.0,
                                 settings=None if settings is None else (type(settings) * B)(*[settings] * B))
    est = hb.estimation_states(B)
    for i in range(B):
        n = min(refs[i].n_events, api.HB_MAX_EVENTS)
        R.set_schedule(est[i], refs[i].event_times[:n], refs[i].modes[:n + 1])
    return est


def _random_states(rng, B):
    """Random schedules: 1 .. HB_MAX_EVENTS events, some of them repeated (ties) and runs of equal modes; the first without a plan."""
    est = hb.estimation_states(B)
    for i in range(1, B):
        n = int(rng.integers(1, api.HB_MAX_EVENTS + 1))
        ev = np.sort(np.round(rng.uniform(0.0, 2.0, n), 2))
        R.set_schedule(est[i], ev, rng.integers(0, 4, n + 1))
    return est


def _times_of(est, t):
    rec = hb.make_contact_detection_settings(len(est))
    return hb.contact_state_host(t, est, np.zeros((len(est), 16)), rec, np.ones((len(est), 4)))[1]


def _assert_phase_times(est, ts):
    for t in ts:
        got = _times_of(est, t)
        for i in range(len(est)):
            assert np.array_equal(got[i], R.phase_times(*R.schedule_of(est[i]), t)), (i, t)


def test_phase_times_on_the_shipped_gaits():
    est = _planned_states()
    ts = sorted(set(np.linspace(0.0, 1.5, 301)) | {x for s in est for x in s.event_times[:s.n_events]})     # the event times: ties
    _assert_phase_times(est, ts)


def test_phase_times_on_the_variant_gaits():
    s = hb.parse_planner_settings(os.path.join(GOLDEN, "task_swing_variant.info"), os.path.join(GOLDEN, "gait_variant.info"))
    est = _planned_states(s)
    _assert_phase_times(est, sorted(set(np.linspace(0.0, 1.5, 151)) | {x for e in est for x in e.event_times[:e.n_events]}))


def test_phase_times_on_random_schedules():
    rng = np.random.default_rng(3)
    est = _random_states(rng, 40)
    _assert_phase_times(est, list(np.round(rng.uniform(-0.5, 2.5, 60), 2)) + [0.0, 1.0, 2.0, 2.5])


def test_phase_times_edges():
    est = hb.estimation_states(4)
    R.set_schedule(est[1], [0.5], [3, 0])                            # one event: the clamp keeps phase 0
    R.set_schedule(est[2], [0.2, 0.4, 0.6], [3, 2, 3, 1])
    R.set_schedule(est[3], [0.3], [1, 2])
    est[3].n_events = 0                                             # one phase: [t, t], as without a plan
    got = _times_of(est, 0.7)
    assert np.array_equal(got[0], np.full((4, 2), 0.7)) and np.array_equal(got[3], np.full((4, 2), 0.7))
    assert np.array_equal(got[1], np.full((4, 2), 0.5))             # phase 1 clamped to 0: start index 0, final n - 2 = 0
    # t = 0.4 is an event time: it belongs to phase 1 (mode 2, left stance)
    t = _times_of(est, 0.4)[2]
    assert list(t[0]) == [0.2, 0.6] and list(t[1]) == [0.2, 0.4]    # left: stance run of phases 0..2 (start index 0); right: swing phase 1
    assert list(_times_of(est, 0.41)[2][1]) == [0.4, 0.6]           # phase 2 of 3 (clamped to n - 1): right stance run 2..3, stop n - 2


@pytest.mark.parametrize("cmd", [0, 1])
def test_truth_table(cmd):
    """Swing and stance x inside and outside each window x force below, at and above the threshold, for each contact and its leg."""
    r = hb.make_contact_detection_settings(1)[0]
    est = hb.estimation_states(1)
    mode = 3 if cmd else 0
    R.set_schedule(est[0], [1.0, 2.0], [mode ^ 3, mode, mode ^ 3])      # contact c in phase 1 = [1, 2] is cmd
    frac = r.swing_fraction if not cmd else r.stance_fraction
    for t, inside in [(1.0 + frac - 0.05, cmd == 1), (1.0 + frac + 0.05, cmd == 0), (1.0 + frac, False)]:
        for fz, loaded in [(r.threshold - 1.0, False), (r.threshold, False), (r.threshold + 1.0, True)]:
            for leg in (0, 1):
                force = np.zeros((1, 16)); force[0, 6 * leg + 2] = fz
                force[0, 6 * (1 - leg) + 2] = 1e3 if not loaded else -1e3        # the other leg says the opposite
                fl, _ = hb.contact_state_host(t, est, force, [r], np.full((1, 4), cmd))
                want = [(int(loaded) if inside else cmd) if c % 2 == leg else (int(not loaded) if inside else cmd) for c in range(4)]
                assert list(fl[0]) == want, (t, fz, leg)
                assert want == R.contact_state(r, t, R.phase_times(*R.schedule_of(est[0]), t), force[0], [cmd] * 4)


def test_initial_force_is_loaded_for_the_default_threshold():
    """Before the first observer output every F_z is 50: below task.info's 75, so a swing foot late in its phase stays in the air and a
    stance foot early in its phase is distrusted."""
    est = hb.estimation_states(1)
    R.set_schedule(est[0], [1.0, 2.0, 3.0], [3, 0, 3, 0])
    force = np.full((1, 16), R.INITIAL_FORCE)
    r = hb.make_contact_detection_settings(1)
    assert list(hb.contact_state_host(1.9, est, force, r, np.zeros((1, 4)))[0][0]) == [0, 0, 0, 0]
    assert list(hb.contact_state_host(2.1, est, force, r, np.ones((1, 4)))[0][0]) == [0, 0, 0, 0]
    r2 = hb.make_contact_detection_settings(1, threshold=49.0)
    assert list(hb.contact_state_host(1.9, est, force, r2, np.zeros((1, 4)))[0][0]) == [1, 1, 1, 1]


def test_rule_against_the_restatement_on_random_inputs():
    rng = np.random.default_rng(7)
    B = 40
    est = _random_states(rng, B)
    rec = hb.make_contact_detection_settings(B, threshold=rng.uniform(0, 100, B), swing_fraction=rng.uniform(0, 1, B),
                                             stance_fraction=rng.uniform(0, 1, B))
    for t in np.round(rng.uniform(-0.2, 2.2, 30), 2):
        force = rng.uniform(-20, 150, (B, 16))
        cmd = rng.integers(0, 2, (B, 4))
        got, _ = hb.contact_state_host(t, est, force, rec, cmd)
        assert np.array_equal(got, R.detect(rec, t, est, force, cmd)), t
        assert np.array_equal(hb.contact_state_host(t, est, force, None, cmd)[0], cmd)       # no records: unchanged


def test_default_records_from_task_info():
    d = hb.default_contact_detection()
    assert (d.cutoff_frequency, d.threshold, d.swing_fraction, d.stance_fraction) == (250.0, 75.0, 0.75, 0.25)
    assert bytes(hb.default_contact_detection(TASK)) == bytes(d)
    v = hb.default_contact_detection(os.path.join(GOLDEN, "task_wbc_variant.info"))
    assert (v.cutoff_frequency, v.threshold, v.swing_fraction, v.stance_fraction) == (200.0, 70.0, 0.75, 0.25)
    assert hb.load_library().hb_default_contact_detection(None, None) == -1


BAD = [dict(cutoff_frequency=0.0), dict(cutoff_frequency=-1.0), dict(cutoff_frequency=np.nan), dict(threshold=np.inf), dict(threshold=np.nan),
       dict(swing_fraction=-0.01), dict(swing_fraction=1.01), dict(swing_fraction=np.nan), dict(stance_fraction=-1e-9),
       dict(stance_fraction=1.5), dict(stance_fraction=np.nan)]


@pytest.mark.parametrize("bad", BAD, ids=[str(b) for b in BAD])
def test_every_rejected_record_is_named_by_index(bad):
    lib = hb.load_library()
    rec = hb.make_contact_detection_settings(5)
    (k, v), = bad.items()
    setattr(rec[3], k, v)
    first = C.c_int32()
    assert lib.hb_check_setting_records(20, 5, rec, C.byref(first)) == -1 and first.value == 3
    with pytest.raises(ValueError, match="record 2"):
        hb.make_contact_detection_settings(4, **{k: [0.5 if k != "threshold" else 1.0, 0.5 if k != "threshold" else 1.0, v, v]})
    with pytest.raises(hb.HunterB200Error):
        hb.contact_state_host(0.0, hb.estimation_states(5), np.zeros((5, 16)), rec, np.zeros((5, 4)))


def test_records_and_builders():
    lib = hb.load_library()
    assert hb.HbContactDetection.SETTING_KIND == 20 and not hasattr(api, "HB_SETTING_CONTACT_DETECTION")
    rec = hb.make_contact_detection_settings(3, threshold=[10.0, 20.0, 30.0], stance_fraction=0.0, swing_fraction=1.0)
    first = C.c_int32()
    assert lib.hb_check_setting_records(20, 3, rec, C.byref(first)) == 0 and first.value == -1
    assert [r.threshold for r in rec] == [10.0, 20.0, 30.0] and all(r.cutoff_frequency == 250.0 for r in rec)
    base = hb.default_contact_detection(); base.cutoff_frequency = 100.0
    assert all(r.cutoff_frequency == 100.0 for r in hb.make_contact_detection_settings(2, base=base))
    with pytest.raises(ValueError, match="unknown field"):
        hb.make_contact_detection_settings(2, cutoff=1.0)
    with pytest.raises(ValueError, match="expected"):
        hb.make_contact_detection_settings(2, threshold=[1.0, 2.0, 3.0])
    # kinds 10 and 16 stay unassigned
    for kind in (10, 16, 21):
        assert lib.hb_check_setting_records(kind, 1, rec, C.byref(first)) == -1


def test_header_layout_and_symbols():
    assert C.sizeof(hb.HbContactDetection) == 32
    assert [f for f, _ in hb.HbContactDetection._fields_] == ["cutoff_frequency", "threshold", "swing_fraction", "stance_fraction"]
    lib = hb.load_library()
    for name in ("hb_default_contact_detection", "hb_rollout_set_contact_detection", "hb_contact_state_estimate_async", "hb_contact_state_estimate",
                 "hb_rollout_contact_estimates", "hb_contact_state_host"):
        assert name in hb.EXPORTED_SYMBOLS and hasattr(lib, name)
    hdr = open(os.path.join(os.path.dirname(GOLDEN), "..", "include", "hunter_b200.h")).read()
    assert "#define HB_SETTING_CONTACT_DETECTION 20" in hdr
