"""Plant variations on the host (no GPU): what make_plant_variations builds and rejects, and the library's default variation."""
import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb


def _view(V):
    return np.ctypeslib.as_array(V)


def test_default_plant_variation_is_the_python_default():
    d = hb.default_plant_variation()
    assert bytes(d) == bytes(hb.make_plant_variations(1)[0])
    assert d.payload_mass == 0.0 and list(d.payload_com) == [0.0] * 3 and list(d.payload_inertia) == [0.0] * 9
    assert (d.friction_scale, d.stiffness_scale, d.damping_scale) == (1.0, 1.0, 1.0) and list(d.motor_strength) == [1.0] * 10


def test_make_plant_variations_broadcasts():
    box = np.diag([0.1, 0.2, 0.3])
    V = _view(hb.make_plant_variations(3, payload_mass=[0.5, 1.0, 2.5], payload_com=[0.0, 0.0, 0.1], payload_inertia=box, friction_scale=0.4,
                                       motor_strength=np.linspace(0.5, 1.0, 10)))
    assert list(V["payload_mass"]) == [0.5, 1.0, 2.5]
    assert (V["payload_com"] == [0.0, 0.0, 0.1]).all() and (V["payload_inertia"] == box.reshape(9)).all()
    assert (V["friction_scale"] == 0.4).all() and (V["stiffness_scale"] == 1.0).all() and (V["damping_scale"] == 1.0).all()
    assert (V["motor_strength"] == np.linspace(0.5, 1.0, 10)).all()
    # per-instance arrays
    com = np.array([[0.0, 0.0, 0.0], [0.1, -0.02, 0.05]])
    inertia = np.stack([np.zeros((3, 3)), [[0.2, 0.01, 0.0], [0.01, 0.3, -0.02], [0.0, -0.02, 0.1]]])
    V = _view(hb.make_plant_variations(2, payload_mass=[0.0, 3.0], payload_com=com, payload_inertia=inertia, stiffness_scale=[0.5, 2.0],
                                       damping_scale=[0.0, 1.5], motor_strength=[[1.0], [0.0]]))
    assert (V["payload_com"] == com).all() and (V["payload_inertia"] == inertia.reshape(2, 9)).all()
    assert list(V["stiffness_scale"]) == [0.5, 2.0] and list(V["damping_scale"]) == [0.0, 1.5]
    assert (V["motor_strength"][0] == 1.0).all() and (V["motor_strength"][1] == 0.0).all()
    # the defaults: B nominal plants
    D = _view(hb.make_plant_variations(4))
    assert all(bytes(x) == bytes(hb.default_plant_variation()) for x in hb.make_plant_variations(4)) and len(D) == 4


@pytest.mark.parametrize("case", ["nan_mass", "negative_mass", "inf_com", "asymmetric", "negative_diagonal", "negative_minor", "negative_det",
                                  "com_without_mass", "inertia_without_mass", "negative_friction", "zero_stiffness", "negative_damping",
                                  "negative_motor", "nan_motor", "shape"])
def test_make_plant_variations_rejects_what_the_c_call_rejects(case):
    kw = dict(payload_mass=[1.0, 2.0], payload_com=[0.0, 0.0, 0.1], payload_inertia=np.diag([0.1, 0.1, 0.1]))
    I = np.diag([0.1, 0.1, 0.1])
    if case == "nan_mass":
        kw["payload_mass"] = [1.0, np.nan]
    elif case == "negative_mass":
        kw["payload_mass"] = [1.0, -0.1]
    elif case == "inf_com":
        kw["payload_com"] = [0.0, np.inf, 0.0]
    elif case == "asymmetric":
        I[0, 1] = 0.01; kw["payload_inertia"] = I
    elif case == "negative_diagonal":
        I[2, 2] = -0.01; kw["payload_inertia"] = I
    elif case == "negative_minor":
        I[0, 1] = I[1, 0] = 0.2; kw["payload_inertia"] = I             # diagonal >= 0, 2 x 2 minor 0.01 - 0.04 < 0
    elif case == "negative_det":
        kw["payload_inertia"] = np.array([[1.0, 1.0, 0.0], [1.0, 1.0, 1.0], [0.0, 1.0, 1.0]])    # 2 x 2 minors >= 0, determinant -1
    elif case == "com_without_mass":
        kw["payload_mass"] = [0.0, 1.0]; kw["payload_inertia"] = None
    elif case == "inertia_without_mass":
        kw["payload_mass"] = [0.0, 1.0]; kw["payload_com"] = [0.0, 0.0, 0.0]
    elif case == "negative_friction":
        kw["friction_scale"] = [0.5, -0.5]
    elif case == "zero_stiffness":
        kw["stiffness_scale"] = 0.0
    elif case == "negative_damping":
        kw["damping_scale"] = -1.0
    elif case == "negative_motor":
        ms = np.ones(10); ms[3] = -0.5; kw["motor_strength"] = ms
    elif case == "nan_motor":
        kw["motor_strength"] = [[1.0], [np.nan]]
    else:
        kw["payload_com"] = np.zeros((3, 3))
    with pytest.raises(ValueError):
        hb.make_plant_variations(2, **kw)
