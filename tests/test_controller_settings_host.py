"""make_controller_settings (no GPU): the defaults are hb_default_wbc_settings and hb_default_pd_gains, scalars broadcast and per-robot
arrays land in their fields, unknown names and shapes that do not broadcast raise."""
import ctypes as C

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb


def _default_wbc():
    w = hb.HbWbcSettings()
    assert hb.load_library().hb_default_wbc_settings(C.byref(w)) == 0
    return w


def test_defaults_are_the_library_defaults():
    s = hb.make_controller_settings(3)
    assert C.sizeof(hb.HbControllerSetting) == 208
    for r in s:
        assert bytes(r.wbc) == bytes(_default_wbc())
        assert bytes(r.gains) == bytes(hb.default_pd_gains())


def test_base_records_are_copied():
    w = _default_wbc(); w.swing_kp = 123.0
    g = hb.default_pd_gains(); g.kd_feet = 0.5
    s = hb.make_controller_settings(2, wbc=w, gains=g)
    assert [r.wbc.swing_kp for r in s] == [123.0, 123.0] and [r.gains.kd_feet for r in s] == [0.5, 0.5]
    assert w.swing_kp == 123.0 and g.kd_feet == 0.5


def test_scalars_broadcast_and_arrays_land_per_robot():
    B = 4
    s = hb.make_controller_settings(B, swing_kp=[1.0, 2.0, 3.0, 4.0], weight_contact_force=0.02, kp_big_stance=np.arange(B) + 40.0,
                                    kd_feet=0.03, torque_limits=[10.0, 20.0, 30.0, 40.0, 50.0])
    d = _default_wbc()
    for i, r in enumerate(s):
        assert r.wbc.swing_kp == i + 1.0 and r.wbc.weight_contact_force == 0.02
        assert r.gains.kp_big_stance == 40.0 + i and r.gains.kd_feet == 0.03
        assert list(r.wbc.torque_limits) == [10.0, 20.0, 30.0, 40.0, 50.0]
        assert r.wbc.swing_kd == d.swing_kd and r.gains.kd_big == hb.default_pd_gains().kd_big
    tl = np.arange(B * 5, dtype=float).reshape(B, 5) + 1.0
    s = hb.make_controller_settings(B, torque_limits=tl)
    assert np.array_equal(np.array([list(r.wbc.torque_limits) for r in s]), tl)


@pytest.mark.parametrize("kw", [dict(swing_gain=1.0), dict(kp=1.0), dict(wbc_swing_kp=1.0)])
def test_unknown_names_raise(kw):
    with pytest.raises(ValueError, match="unknown field"):
        hb.make_controller_settings(2, **kw)


@pytest.mark.parametrize("kw", [dict(swing_kp=[1.0, 2.0, 3.0]), dict(torque_limits=[1.0, 2.0]), dict(torque_limits=np.ones((3, 5)))])
def test_shapes_that_do_not_broadcast_raise(kw):
    with pytest.raises(ValueError):
        hb.make_controller_settings(2, **kw)


def test_exported():
    assert "hb_rollout_set_controller_settings" in hb.EXPORTED_SYMBOLS
    assert hasattr(hb.load_library(), "hb_rollout_set_controller_settings")
