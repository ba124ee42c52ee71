"""Joint models on the host (no GPU): the default record against the model constants and against both reference plants' joints (the
URDF under tests/golden/hunter_config and tests/golden/joint_model_mjcf.json from hunter.xml), every rejected record
(hb_check_setting_records), the stability rule's arithmetic, make_joint_models, the layout, and joint_model_ref's terms."""
import ctypes as C
import json
import os
import xml.etree.ElementTree as ET

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
import joint_model_ref as J
from oracle import refs as R

HERE = os.path.dirname(os.path.abspath(__file__))
KIND = hb.HbJointModel.SETTING_KIND
NAMES = ["leg_%s%d_joint" % (s, k) for s in "lr" for k in range(1, 6)]
nan, inf = float("nan"), float("inf")
JOINT_LOWER, JOINT_UPPER = np.array(R._header_array("HB_JOINT_LOWER")), np.array(R._header_array("HB_JOINT_UPPER"))


def _check(records):
    bad = C.c_int32(7)
    rc = hb.load_library().hb_check_setting_records(KIND, len(records), records, C.byref(bad))
    return rc, bad.value


def _arr(rec, name):
    return np.array(getattr(rec, name)[:]) if isinstance(getattr(rec, name), C.Array) else getattr(rec, name)


# ---------------------------------------------------------------------------------------------------------------- records
def test_kind_and_layout():
    assert KIND == 21 and C.sizeof(hb.HbJointModel) == 264
    offs = {n: getattr(hb.HbJointModel, n).offset for n, _ in hb.HbJointModel._fields_}
    assert offs == {"friction_loss": 0, "friction_velocity": 80, "lower": 88, "upper": 168, "stop_stiffness": 248, "stop_damping": 256}
    for name in ("hb_default_joint_model", "hb_rollout_set_joint_models", "hb_sim_step_joints"):
        assert name in hb.EXPORTED_SYMBOLS and hasattr(hb.load_library(), name)


def test_default_record_against_the_constants_and_mujoco_defaults():
    d = hb.default_joint_model()
    assert (_arr(d, "friction_loss") == 0.2).all() and d.friction_velocity == 0.01
    assert np.array_equal(_arr(d, "lower"), JOINT_LOWER) and np.array_equal(_arr(d, "upper"), JOINT_UPPER)
    tc, zeta, d_max = 0.02, 1.0, 0.95                        # MuJoCo's default solref and solimp's d_max
    assert d.stop_damping == 2.0 / (d_max * tc) and abs(d.stop_damping - 105.263) < 1e-3
    assert d.stop_stiffness == 1.0 / (d_max * tc * tc * zeta * zeta) and abs(d.stop_stiffness - 2631.579) < 1e-3
    assert bytes(hb.make_joint_models(1)[0]) == bytes(d)
    assert _check((hb.HbJointModel * 1)(d)) == (0, -1)


def test_default_record_against_the_urdf():
    root = ET.parse(os.path.join(HERE, "golden", "hunter_config", "hunter.urdf")).getroot()
    joints = {j.get("name"): j for j in root.findall("joint")}          # the robot's joints, not the transmissions' references
    d = hb.default_joint_model()
    for j, n in enumerate(NAMES):
        lim, dyn = joints[n].find("limit"), joints[n].find("dynamics")
        assert (float(lim.get("lower")), float(lim.get("upper"))) == (d.lower[j], d.upper[j]), n
        assert float(dyn.get("friction")) == d.friction_loss[j], n


def test_default_record_against_the_mjcf():
    with open(os.path.join(HERE, "golden", "joint_model_mjcf.json")) as f:
        g = json.load(f)
    assert g["joints"] == NAMES and g["autolimits"]
    d = hb.default_joint_model()
    assert np.array_equal(np.array(g["range"]), np.c_[_arr(d, "lower"), _arr(d, "upper")])
    assert np.array_equal(g["frictionloss"], _arr(d, "friction_loss"))


def test_disabled_records_pass():
    assert _check(J.disabled(3)) == (0, -1)
    one_sided = hb.make_joint_models(2, lower=-inf, upper=JOINT_UPPER, friction_loss=0.0, stop_stiffness=0.0, stop_damping=0.0)
    assert _check(one_sided) == (0, -1)


@pytest.mark.parametrize("case", range(len(J.BAD)), ids=["%s[%s]=%s" % b for b in J.BAD])
def test_rejected_records(case):
    assert _check(J.bad_records()[case]) == (-1, 1)


def test_builder_names_the_bad_record():
    with pytest.raises(ValueError, match="joint_models"):
        hb.make_joint_models(3, friction_velocity=[0.01, 0.0, 0.01])
    with pytest.raises(ValueError, match="joint_models"):
        hb.make_joint_models(2, lower=[[0.0], [2.0]])


def test_builder_broadcasts():
    B = 3
    v = np.ctypeslib.as_array(hb.make_joint_models(B, friction_loss=[[0.0], [0.1], [0.4]], upper=np.arange(1, 11), stop_stiffness=[1.0, 2.0, 3.0]))
    assert (v["friction_loss"] == np.array([0.0, 0.1, 0.4])[:, None]).all()
    assert (v["upper"] == np.arange(1, 11)).all() and (v["lower"] == JOINT_LOWER).all()
    assert (v["stop_stiffness"] == [1.0, 2.0, 3.0]).all() and (v["stop_damping"] == hb.default_joint_model().stop_damping).all()
    assert (v["friction_velocity"] == 0.01).all()
    with pytest.raises(ValueError, match="friction_loss"):
        hb.make_joint_models(B, friction_loss=np.zeros(4))
    with pytest.raises(ValueError, match="stop_damping"):
        hb.make_joint_models(B, stop_damping=np.zeros(2))


# ---------------------------------------------------------------------------------------------------------------- the stability rule
def test_stability_rule_arithmetic():
    """h (d + f / v_s) <= A: at the default params 0.002 / 4 (1 + 0.2 / 0.01) = 0.0105 <= 0.1, and the bound is reached at f / v_s = 199."""
    prm = hb.default_sim_params()
    h = prm.dt / prm.substeps
    assert (prm.dt, prm.substeps, prm.joint_damping, prm.joint_armature) == (0.002, 4, 1.0, 0.1)
    assert abs(h * (prm.joint_damping + 0.2 / 0.01) - 0.0105) < 1e-15
    assert J.stable(prm, [hb.default_joint_model()]) and J.stable(prm, J.disabled(2))
    gain = prm.joint_armature / h - prm.joint_damping                    # the largest f / v_s the rule admits: 199
    assert abs(gain - 199.0) < 1e-9
    assert J.stable(prm, hb.make_joint_models(1, friction_loss=1.9, friction_velocity=0.01))
    assert not J.stable(prm, hb.make_joint_models(1, friction_loss=2.0, friction_velocity=0.01))
    assert not J.stable(prm, hb.make_joint_models(1, friction_velocity=0.2 / 200))
    one = hb.make_joint_models(1, friction_loss=[0.2] * 9 + [2.5])       # one joint of one record suffices
    assert not J.stable(prm, one)
    prm.substeps = 1                                                      # h = 0.002: 0.002 (1 + 20) = 0.042 <= 0.1
    assert J.stable(prm, [hb.default_joint_model()])
    prm.joint_armature = 0.04
    assert not J.stable(prm, [hb.default_joint_model()]) and J.stable(prm, J.disabled(1))


# ---------------------------------------------------------------------------------------------------------------- the terms
def test_friction_and_stop_terms():
    d = hb.default_joint_model()
    assert abs(J.friction(d, 0, 0.005) + 0.1) < 1e-15 and J.friction(d, 0, -0.02) == 0.2 and J.friction(d, 0, 0.0) == 0.0
    up, lo = d.upper[3], d.lower[3]
    assert J.stop(d, 3, up, 5.0, 0.2) == 0.0 and J.stop(d, 3, lo, -5.0, 0.2) == 0.0           # at a bound: no stop
    r = 0.01
    assert J.stop(d, 3, up + r, 0.0, 0.2) == pytest.approx(-0.2 * d.stop_stiffness * r, rel=1e-12)
    assert J.stop(d, 3, lo - r, 0.0, 0.2) == pytest.approx(0.2 * d.stop_stiffness * r, rel=1e-12)
    v_back = d.stop_stiffness * r / d.stop_damping                                              # k r + b v = 0
    assert J.stop(d, 3, up + r, -2 * v_back, 0.2) == 0.0 and J.stop(d, 3, lo - r, 2 * v_back, 0.2) == 0.0   # never pulls
    assert J.stop(d, 3, up + r, -0.5 * v_back, 0.2) < 0.0 and J.stop(d, 3, lo - r, 0.5 * v_back, 0.2) > 0.0


def test_settled_penetration_under_a_load():
    """The static balance of the stop, m_jj k r = tau: with the default gains a 10 N m load on a joint with m_jj = 0.15 penetrates
    about 0.025 rad, past the joint command law's 0.02 rad emergency-stop margin."""
    d = hb.default_joint_model()
    r = 10.0 / (d.stop_stiffness * 0.15)
    assert 0.025 < r < 0.0255
    assert abs(J.stop(d, 0, d.upper[0] + r, 0.0, 0.15) + 10.0) < 1e-12


# ---------------------------------------------------------------------------------------------------------------- the sweep tool
def test_joint_sweep_parses_help_and_measures_past_the_range():
    import subprocess
    import sys
    tools = os.path.join(os.path.dirname(HERE), "tools")
    out = subprocess.run([sys.executable, os.path.join(tools, "joint_sweep.py"), "--help"], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.startswith("usage: joint_sweep.py") and "--push" in out.stdout, out.stderr
    sys.path.insert(0, tools)
    import joint_sweep
    d = hb.default_joint_model()
    log = np.zeros((2, 4, 32))
    log[:, :, 6:16] = 0.5 * (JOINT_LOWER + JOINT_UPPER)
    log[0, 1, 6 + 3] = d.upper[3] + 0.03                  # robot 0 past the knee's upper end on tick 1
    log[1, 2, 6 + 0] = d.lower[0] - 0.05                  # robot 1 past the hip's lower end on tick 2, after it fell on tick 2
    st = hb.rollout_stats(2); st["fail_tick"] = [-1, 2]
    pen, share = joint_sweep.past_range(hb, log, st, 4)
    assert abs(pen - 0.03) < 1e-12 and share == 1 / 6
