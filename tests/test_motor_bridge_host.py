"""Motor bridge records and codec on the host (no GPU): the host codec (hb_motor_bridge_encode / _feedback) against the numpy float32
restatement (bridge_ref) bit for bit at every range edge, at and next to code boundaries, on +-0, +-inf and NaN; the known answers of the
shipped gains; the default record against the reference's constants; the record check; and make_motor_bridges."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from bridge_ref import BITS, code, command, feedback, value

nan, inf = float("nan"), float("inf")
X_JOINTS, D_JOINTS = [0, 1, 4, 5, 6, 9], [2, 3, 7, 8]


def _same(a, b):
    """Bitwise equality of float64 arrays (NaN payloads and zero signs included)."""
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.uint64), np.asarray(b, dtype=np.float64).view(np.uint64))


def _probe(lo, hi, bits):
    """Values on [lo, hi] and beyond: the edges, +-0, +-inf, NaN, each code boundary of a sample of codes, the float32 neighbours of each
    and a double between them."""
    n = (1 << bits) - 1
    f32 = np.float32
    flo, span = f32(lo), f32(hi) - f32(lo)
    ks = np.unique(np.r_[0, 1, 2, n // 2, n // 2 + 1, n - 2, n - 1, n, np.random.default_rng(bits).integers(0, n + 1, 60)])
    out = [lo, hi, -lo, -hi, 0.0, -0.0, inf, -inf, nan, 2 * hi, 2 * lo - 1.0, np.nextafter(hi, inf), np.nextafter(lo, -inf)]
    for k in ks:
        b = f32(f32(f32(k) * span) / f32(n)) + flo          # the decoded value of code k
        x = f32((f32(k) * span) / f32(n)) + flo             # where the encoder's product crosses k
        for v in (b, x):
            up, dn = np.nextafter(v, f32(inf)), np.nextafter(v, f32(-inf))
            out += [float(v), float(up), float(dn), 0.5 * (float(v) + float(up)), 0.5 * (float(v) + float(dn))]
    return np.array(out)


def _records(quantise):
    r = hb.default_motor_bridge()
    r.quantise = quantise
    return r


@pytest.mark.parametrize("quantise", [1, 0])
def test_host_codec_is_the_float32_restatement_bitwise(quantise):
    """Each field of the command, and both encoder readings, over the probe values of its range, on every joint of the default record
    (X and D motors, directions +1 and -1, hip scales 0.7 and 1)."""
    r = _records(quantise)
    for j in range(10):
        for k, (lo, hi, bits) in enumerate([(-12.5, 12.5, 16), (-18.0, 18.0, 12), (0.0, 500.0, 12), (0.0, 5.0, 9),
                                            (-r.ff_max[j], r.ff_max[j], 12)]):
            xs = _probe(lo, hi, bits)
            scale = [float(r.direction[j]), float(r.direction[j]), r.command_scale[j], r.command_scale[j], r.command_scale[j] * r.direction[j]][k]
            xs = np.r_[xs, xs / scale] if scale != 0 else xs      # values that land on the probes after the scale
            cmd = np.zeros((len(xs), 10, 5))
            cmd[:, j, k] = xs
            got = hb.bridge_encode([r] * len(xs), cmd)[:, j, k]
            want = [command(r, j, cmd[i, j])[k] for i in range(len(xs))]
            assert _same(got, want), (j, k)
        xs = np.r_[_probe(-12.5, 12.5, 16), _probe(-18.0, 18.0, 12)]
        q = np.zeros((len(xs), 10)); qd = np.zeros((len(xs), 10))
        q[:, j] = xs; qd[:, j] = xs[::-1]
        got_q, got_qd = hb.bridge_feedback([r] * len(xs), q, qd)
        want = np.array([feedback(r, j, q[i, j], qd[i, j]) for i in range(len(xs))])
        assert _same(got_q[:, j], want[:, 0]) and _same(got_qd[:, j], want[:, 1]), j


def test_codec_rules_on_special_values():
    """NaN encodes as code 0 (the range's low end), +-inf clamps, -0.0 is 0; without quantise NaN passes and nothing is rounded."""
    assert value(nan, -12.5, 12.5, 16, True) == -12.5 and code(nan, -12.5, 12.5, 16) == 0
    assert value(inf, -18.0, 18.0, 12, True) == 18.0 and value(-inf, -18.0, 18.0, 12, True) == -18.0
    assert code(inf, 0.0, 5.0, 9) == 511 and code(-inf, 0.0, 5.0, 9) == 0
    assert value(-0.0, -18.0, 18.0, 12, True) == value(0.0, -18.0, 18.0, 12, True)
    assert np.isnan(value(nan, -1.0, 1.0, 12, False)) and value(0.1, -1.0, 1.0, 12, False) == 0.1 and value(inf, -1.0, 1.0, 12, False) == 1.0
    r = hb.default_motor_bridge()
    cmd = np.zeros((1, 10, 5)); cmd[0, :, 0] = nan; cmd[0, :, 4] = inf
    out = hb.bridge_encode([r], cmd)[0]
    assert (out[:, 0] == -12.5).all()                                    # NaN position: code 0
    assert np.array_equal(out[:, 4], np.where(np.array(r.direction) > 0, np.array(r.ff_max), -np.array(r.ff_max)))


def test_known_answers_of_the_shipped_gains():
    r = hb.default_motor_bridge()
    cmd = np.zeros((1, 10, 5))
    cmd[0, :, 2] = 30.0; cmd[0, :, 3] = 0.01
    out = hb.bridge_encode([r], cmd)[0]
    assert round(out[4, 3], 6) == 0.009785                               # kd_feet 0.01 on a foot (scale 1)
    assert round(out[0, 2], 3) == 20.879 and round(out[2, 2], 3) == 29.915   # kp 30 on a hip (0.7 x 30 = 21) and on a knee
    assert round(out[0, 1], 4) == -0.0044                                # a zero velocity command
    assert round(out[0, 4], 4) == -0.0073 and round(out[2, 4], 4) == -0.0220   # a zero feed-forward on an X and on a D motor
    assert code(21.0, 0.0, 500.0, 12) == 171 and code(0.0, -18.0, 18.0, 12) == 2047
    # the hip's X motor accepts 30 N m of ff: 30 / 0.7 = 42.9 N m of commanded torque, of the WBC's 60
    cmd = np.zeros((1, 10, 5)); cmd[0, 1, 4] = 60.0
    assert hb.bridge_encode([r], cmd)[0, 1, 4] == -30.0                  # joint 1: direction -1
    assert hb.bridge_encode([r], cmd * 30.0 / 0.7 / 60.0 * 0.99)[0, 1, 4] > -30.0


def test_setting_kind_is_the_header_constant():
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "hunter_b200.h")).read()
    assert int(re.search(r"^#define HB_SETTING_MOTOR_BRIDGE (\d+)", header, re.M).group(1)) == hb.HbMotorBridge.SETTING_KIND


def test_default_record_is_the_reference():
    r = hb.default_motor_bridge()
    assert C.sizeof(hb.HbMotorBridge) == 608
    assert list(r.command_scale) == [0.7, 0.7, 1.0, 1.0, 1.0, 0.7, 0.7, 1.0, 1.0, 1.0]          # BridgeHW.cpp:74-85
    assert list(r.direction) == [1, -1, 1, 1, 1, 1, -1, 1, -1, 1]                               # BridgeHW.h:118
    assert list(r.zero) == [0.0] * 10                                                           # BridgeHW.h:120
    assert list(r.kp_max) == [500.0] * 10 and list(r.kd_max) == [5.0] * 10                      # motor_control.c:11-35
    assert list(r.pos_max) == [12.5] * 10 and list(r.vel_max) == [18.0] * 10
    assert [r.ff_max[j] for j in X_JOINTS] == [30.0] * 6 and [r.ff_max[j] for j in D_JOINTS] == [90.0] * 4
    assert r.quantise == 1
    assert BITS == {"pos": 16, "vel": 12, "kp": 12, "kd": 9, "ff": 12}
    assert hb.load_library().hb_default_motor_bridge(None) == -1


BAD = {"direction_zero": ("direction", 3, 0), "direction_two": ("direction", 0, 2), "direction_minus_two": ("direction", 9, -2),
       "nan_scale": ("command_scale", 1, nan), "negative_scale": ("command_scale", 5, -0.1), "inf_zero": ("zero", 2, inf),
       "nan_zero": ("zero", 7, nan), "zero_kp_max": ("kp_max", 0, 0.0), "negative_kd_max": ("kd_max", 4, -5.0),
       "inf_pos_max": ("pos_max", 6, inf), "nan_vel_max": ("vel_max", 8, nan), "zero_ff_max": ("ff_max", 2, 0.0),
       "quantise_two": ("quantise", None, 2), "quantise_negative": ("quantise", None, -1)}


@pytest.mark.parametrize("case", sorted(BAD))
def test_check_rejects(case):
    field, j, v = BAD[case]
    recs = (hb.HbMotorBridge * 4)(*[hb.default_motor_bridge()] * 4)
    for i in (1, 3):
        if j is None:
            setattr(recs[i], field, v)
        else:
            getattr(recs[i], field)[j] = v
    bad = C.c_int32(7)
    assert hb.load_library().hb_check_setting_records(hb.HbMotorBridge.SETTING_KIND, 4, recs, C.byref(bad)) == -1 and bad.value == 1
    with pytest.raises(hb.HunterB200Error):
        hb.bridge_encode(recs, np.zeros((4, 10, 5)))
    with pytest.raises(hb.HunterB200Error):
        hb.bridge_feedback(recs, np.zeros((4, 10)), np.zeros((4, 10)))


def test_check_accepts_the_builders_records():
    bad = C.c_int32(7)
    for recs in (hb.make_motor_bridges(3), hb.make_motor_bridges(2, quantise=0, command_scale=0.0, zero=[0.1] * 10)):
        assert hb.load_library().hb_check_setting_records(hb.HbMotorBridge.SETTING_KIND, len(recs), recs, C.byref(bad)) == 0 and bad.value == -1
    assert hb.load_library().hb_motor_bridge_encode(-1, None, None, None) == -1
    assert hb.load_library().hb_motor_bridge_encode(0, None, None, None) == 0


def test_make_motor_bridges():
    for r in hb.make_motor_bridges(3):
        assert bytes(r) == bytes(hb.default_motor_bridge())
    base = hb.default_motor_bridge(); base.quantise = 0
    r = hb.make_motor_bridges(3, base=base, command_scale=1.0, direction=[1, -1, 1, 1, 1, 1, 1, 1, 1, -1], ff_max=np.full((3, 10), 60.0),
                              quantise=[0, 1, 0])
    assert [x.quantise for x in r] == [0, 1, 0]
    assert all(list(x.command_scale) == [1.0] * 10 and x.direction[1] == -1 and x.direction[9] == -1 and list(x.ff_max) == [60.0] * 10 for x in r)
    assert list(r[0].pos_max) == [12.5] * 10
    with pytest.raises(ValueError, match="unknown field"):
        hb.make_motor_bridges(2, kp=1.0)
    with pytest.raises(ValueError, match="ff_max"):
        hb.make_motor_bridges(2, ff_max=np.ones((3, 10)))
    with pytest.raises(ValueError, match="int32 integers"):
        hb.make_motor_bridges(2, direction=0.5)
    with pytest.raises(ValueError, match="record 1 is rejected by hb_rollout_set_motor_bridge"):
        hb.make_motor_bridges(2, direction=[[1] * 10, [0] * 10])
    with pytest.raises(ValueError, match="record 0 is rejected"):
        hb.make_motor_bridges(2, kp_max=-1.0)
