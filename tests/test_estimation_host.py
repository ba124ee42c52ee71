"""Host-side checks of the estimated episodes (no GPU): the numpy Philox4x32-10 of the sensor noise reproduces the published known-answer
vectors, and the C layout of the estimation types matches the ctypes mirror (hb_estimation_reset writes at the offsets api.py reads)."""
import ctypes as C

import numpy as np

import hunter_bipedal_control_b200 as hb
from estimation_ref import block_normals, philox4x32_10, shortest_angular_distance


def test_philox_known_answers():
    assert philox4x32_10((0, 0), (0, 0, 0, 0)) == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    ones = 0xFFFFFFFF
    assert philox4x32_10((ones, ones), (ones, ones, ones, ones)) == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    assert philox4x32_10((0xA4093822, 0x299F31D0), (0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344)) == [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]


def test_noise_normals_are_standard():
    z = np.array([block_normals(7, b, t, 3) for b in range(4) for t in range(500)]).ravel()
    assert abs(z.mean()) < 0.03 and abs(z.std() - 1.0) < 0.03


def test_shortest_angular_distance():
    assert shortest_angular_distance(0.0, 0.5) == 0.5
    assert abs(shortest_angular_distance(3.0, -3.0) - (2 * np.pi - 6.0)) < 1e-15
    assert abs(shortest_angular_distance(-3.0, 3.0) + (2 * np.pi - 6.0)) < 1e-15
    assert abs(shortest_angular_distance(10.0, 0.1) - ((0.1 - 10.0) + 4 * np.pi)) < 1e-14


def test_estimation_reset_layout():
    st = hb.estimation_states(3, first_stream=(1 << 40) + 5)
    raw = np.frombuffer(bytes(st), dtype=np.uint8).reshape(3, -1)
    size = C.sizeof(hb.HbEstimationState)
    assert raw.shape[1] == size == 3216
    off = hb.HbEstimationState
    for i in range(3):
        row = raw[i]
        assert int(row[off.noise_stream.offset:off.noise_stream.offset + 8].view(np.uint64)[0]) == (1 << 40) + 5 + i
        P = row[off.kf.offset + hb.HbKfState.P.offset:][:324 * 8].view(np.float64).reshape(18, 18)
        assert np.array_equal(P, 100.0 * np.eye(18))
        assert row[off.yaw_obs.offset:off.yaw_obs.offset + 8].view(np.float64)[0] == 0.0
        for f in ("primed", "has_plan", "n_events"):
            o = getattr(off, f).offset
            assert row[o:o + 4].view(np.int32)[0] == 0
    # a non-zero yaw written through the mirror lands where the C side reads it: the reset overwrites it
    st[1].yaw_obs = 2.5
    assert hb.load_library().hb_estimation_reset(1, C.c_uint64(9), C.byref(st[1])) == 0
    assert st[1].yaw_obs == 0.0 and st[1].noise_stream == 9 and st[1].kf.P[0] == 100.0
    assert hb.load_library().hb_estimation_reset(1, C.c_uint64(0), None) == -1
    assert hb.load_library().hb_estimation_reset(-1, C.c_uint64(0), st) == -1


def test_default_estimation_params():
    p = hb.default_estimation_params()
    kf = hb.default_kf_params()
    assert bytes(p.kf) == bytes(kf)
    assert p.noise.seed == 0 and all(getattr(p.noise, k) == 0.0 for k in ("orientation", "angular_velocity", "linear_acceleration", "joint_position",
                                                                          "joint_velocity"))
    assert C.sizeof(hb.HbEstimationParams) == 104 and hb.ESTIMATION_STATS_DTYPE.itemsize == 40
    assert hb.load_library().hb_default_estimation_params(None) == -1
