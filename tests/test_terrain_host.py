"""Terrains on the host (no GPU): what make_terrains builds and rejects, and the height and gradient the tests restate."""
import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from episode_ref import terrain_height


def _view(T):
    return np.ctypeslib.as_array(T)


def test_make_terrains_broadcasts_and_writes_the_used_samples_only():
    h = np.arange(12, dtype=float).reshape(3, 4) * 0.01             # ny = 3, nx = 4
    V = _view(hb.make_terrains(2, h, 0.05))
    assert list(V["nx"]) == [4, 4] and list(V["ny"]) == [3, 3]
    assert (V["origin"] == 0.0).all() and (V["spacing"] == 0.05).all()
    assert (V["height"][:, :3, :4] == h).all()
    assert (V["height"][:, 3:, :] == 0).all() and (V["height"][:, :, 4:] == 0).all()
    # per-instance heights, spacings and origins
    hs = np.stack([h, -h])
    V = _view(hb.make_terrains(2, hs, [0.05, 0.1], [[1.0, -2.0], [0.5, 0.25]]))
    assert (V["height"][:, :3, :4] == hs).all()
    assert list(V["spacing"]) == [0.05, 0.1] and (V["origin"] == [[1.0, -2.0], [0.5, 0.25]]).all()
    # the largest grid, and the bytes of one instance
    big = np.random.default_rng(0).uniform(-0.1, 0.1, (hb.HB_TERRAIN_MAX, hb.HB_TERRAIN_MAX))
    T = hb.make_terrains(1, big, 0.025, (-0.8, -0.8))[0]
    assert T.nx == T.ny == hb.HB_TERRAIN_MAX and np.array_equal(np.array(T.height), big)
    raw = np.frombuffer(bytes(T), dtype=np.uint8)
    assert len(raw) == 32800
    assert np.array_equal(raw[:8].view(np.int32), [64, 64])
    assert np.array_equal(raw[8:32].view(np.float64), [-0.8, -0.8, 0.025])
    assert np.array_equal(raw[32:].view(np.float64).reshape(64, 64), big)


@pytest.mark.parametrize("case", ["nx_small", "ny_small", "nx_large", "ny_large", "ndim", "nan_height", "inf_height", "nan_origin",
                                  "inf_origin", "zero_spacing", "negative_spacing", "nan_spacing", "inf_spacing", "shape_heights",
                                  "shape_spacing", "shape_origin"])
def test_make_terrains_rejects_what_the_c_call_rejects(case):
    kw = dict(heights=np.zeros((4, 5)), spacing=0.05, origin=(0.0, 0.0))
    if case == "nx_small":
        kw["heights"] = np.zeros((4, 1))
    elif case == "ny_small":
        kw["heights"] = np.zeros((1, 4))
    elif case == "nx_large":
        kw["heights"] = np.zeros((4, 65))
    elif case == "ny_large":
        kw["heights"] = np.zeros((65, 4))
    elif case == "ndim":
        kw["heights"] = np.zeros(5)
    elif case == "nan_height":
        kw["heights"][2, 3] = np.nan
    elif case == "inf_height":
        kw["heights"][0, 0] = -np.inf
    elif case == "nan_origin":
        kw["origin"] = (np.nan, 0.0)
    elif case == "inf_origin":
        kw["origin"] = [[0.0, 0.0], [0.0, np.inf]]
    elif case == "zero_spacing":
        kw["spacing"] = 0.0
    elif case == "negative_spacing":
        kw["spacing"] = [0.05, -0.05]
    elif case == "nan_spacing":
        kw["spacing"] = np.nan
    elif case == "inf_spacing":
        kw["spacing"] = np.inf
    elif case == "shape_heights":
        kw["heights"] = np.zeros((3, 4, 5))
    elif case == "shape_spacing":
        kw["spacing"] = [0.05, 0.05, 0.05]
    else:
        kw["origin"] = (0.0, 0.0, 0.0)
    with pytest.raises(ValueError):
        hb.make_terrains(2, **kw)


def test_restated_height_and_gradient():
    """The restatement's lookup on hand-computed points: a plane is reproduced with its gradient, a plateau exactly, and a clamped axis
    has a zero gradient component with the edge's height."""
    s, o = 0.25, (-1.0, 2.0)
    X, Y = np.meshgrid(o[0] + s * np.arange(6), o[1] + s * np.arange(5))
    T = hb.make_terrains(1, 0.5 + 0.2 * X - 0.1 * Y, s, o)[0]
    for x, y in [(-0.6, 2.3), (-1.0, 2.0), (-0.5, 2.5), (0.24, 2.99)]:
        h, gx, gy = terrain_height(T, x, y)
        assert abs(h - (0.5 + 0.2 * x - 0.1 * y)) < 1e-15 and abs(gx - 0.2) < 1e-14 and abs(gy + 0.1) < 1e-14
    h, gx, gy = terrain_height(T, -3.0, 2.3)                       # x clamped to the first column
    assert gx == 0.0 and abs(gy + 0.1) < 1e-14 and abs(h - (0.5 + 0.2 * -1.0 - 0.1 * 2.3)) < 1e-15
    h, gx, gy = terrain_height(T, 5.0, 9.0)                        # both clamped: the far corner, flat
    assert gx == 0.0 and gy == 0.0 and abs(h - (0.5 + 0.2 * 0.25 - 0.1 * 3.0)) < 1e-15
    P = hb.make_terrains(1, np.full((3, 3), 0.1234567), 0.1)[0]
    assert terrain_height(P, 0.137, 0.05) == (0.1234567, 0.0, 0.0)
