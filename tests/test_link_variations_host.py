"""Link variations on the host (no GPU): make_link_variations and the default record, the record check (hb_check_setting_records), and
the varied rigid-body terms of link_ref (the restatement the GPU tests hold the plant to): the oracle's own terms with the default record,
the nominal terms of the numpy recursion against the oracle, the changes of varied bodies against MuJoCo, and the physics of M and nle on
varied bodies (symmetry and definiteness, total mass, kinetic and potential energy)."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
import link_ref as L

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
KIND = hb.HbLinkVariation.SETTING_KIND
nan, inf = float("nan"), float("inf")


def _check(records):
    bad = C.c_int32(7)
    rc = hb.load_library().hb_check_setting_records(KIND, len(records), records, C.byref(bad))
    return rc, bad.value


def _states(n, seed):
    rng = np.random.default_rng(seed)
    lo = np.array([-0.2, -0.5, -0.8, 0, -1.1, -0.5, -1, -1.2, 0, -1.1]); hi = np.array([0.5, 1, 1.2, 1.5, 1.1, 0.2, 0.5, 0.8, 1.5, 1.1])
    out = []
    for _ in range(n):
        q = np.r_[rng.uniform(-0.3, 0.3, 3) + [0, 0, 0.63], rng.uniform([-np.pi, -0.5, -0.5], [np.pi, 0.5, 0.5]), rng.uniform(lo, hi)]
        out.append((q, rng.uniform(-1.5, 1.5, 16)))
    return out


def _random_record(seed):
    rng = np.random.default_rng(seed)
    return hb.make_link_variations(1, rng.uniform(0.5, 2.0, 11), rng.uniform(-0.02, 0.02, (11, 3)), rng.uniform(0.5, 2.0, 11))[0]


# ---------------------------------------------------------------------------------------------------------------- records
def test_kind_and_layout():
    assert KIND == 13 and C.sizeof(hb.HbLinkVariation) == 440 and hb.NBODY == 11
    assert "hb_sim_step_links" in hb.EXPORTED_SYMBOLS and hasattr(hb.load_library(), "hb_sim_step_links")


def test_default_record():
    r = np.ctypeslib.as_array((hb.HbLinkVariation * 1)(hb.default_link_variation()))[0]
    assert (r["mass_scale"] == 1.0).all() and (r["inertia_scale"] == 1.0).all() and (r["com_shift"] == 0.0).all()
    assert bytes(hb.make_link_variations(1)[0]) == bytes(hb.default_link_variation())


def test_builder_broadcasts_over_robot_and_body():
    B = 3
    v = np.ctypeslib.as_array(hb.make_link_variations(B, mass_scale=[[1.0], [1.5], [2.0]], com_shift=[0.0, 0.0, -0.02], inertia_scale=np.arange(1, 12)))
    assert v.shape == (B,)
    assert (v["mass_scale"] == np.array([1.0, 1.5, 2.0])[:, None]).all()
    assert (v["com_shift"] == [0.0, 0.0, -0.02]).all()
    assert (v["inertia_scale"] == np.arange(1, 12)).all()
    shift = np.random.default_rng(0).normal(size=(B, 11, 3))
    assert (np.ctypeslib.as_array(hb.make_link_variations(B, com_shift=shift))["com_shift"] == shift).all()
    for bad in (dict(mass_scale=np.ones(10)), dict(com_shift=np.zeros((11, 2))), dict(inertia_scale=np.ones((2, 11)))):
        with pytest.raises(ValueError, match="link variations"):
            hb.make_link_variations(B, **bad)


@pytest.mark.parametrize("field, body, value", [("mass_scale", 4, 0.0), ("mass_scale", 0, -1.0), ("mass_scale", 10, nan), ("mass_scale", 3, inf),
                                                ("inertia_scale", 2, 0.0), ("inertia_scale", 9, -0.5), ("inertia_scale", 5, nan),
                                                ("com_shift", 7, nan), ("com_shift", 1, -inf)])
def test_a_rejected_record_is_named(field, body, value):
    records = hb.make_link_variations(4, mass_scale=1.3)
    assert _check(records) == (0, -1)
    v = np.ctypeslib.as_array(records)
    if field == "com_shift":
        v[field][2, body, 1] = value
    else:
        v[field][2, body] = value
    assert _check(records) == (-1, 2)
    with pytest.raises(ValueError, match="record 2 is rejected by hb_rollout_set_link_variations"):
        hb.make_link_variations(4, **{field: np.ctypeslib.as_array(records)[field]})


def test_small_positive_scales_and_large_shifts_pass():
    assert _check(hb.make_link_variations(2, mass_scale=1e-300, com_shift=5.0, inertia_scale=1e-300)) == (0, -1)


# ---------------------------------------------------------------------------------------------------------------- the varied terms
def test_default_record_is_the_oracle_bit_for_bit(oracle):
    lo = L.LinkOracle(oracle, hb.default_link_variation())
    for q, v in _states(4, 1):
        a, b = oracle.rbd(q, v), lo.rbd(q, v)
        for k in a:
            assert np.array_equal(a[k], b[k]), k


def test_the_recursion_restates_the_oracle(oracle):
    for q, v in _states(6, 2):
        r = oracle.rbd(q, v)
        M, nle = L.terms(q, v)
        assert np.abs(M - r["M"]).max() <= 1e-13 * np.abs(r["M"]).max()
        assert np.abs(nle - r["nle"]).max() <= 1e-13 * np.abs(r["nle"]).max()


def test_bodies_are_one_rounded_operation_each():
    rec = _random_record(3)
    r = np.ctypeslib.as_array((hb.HbLinkVariation * 1)(rec))[0]
    m, c, I = L.bodies(rec)
    assert np.array_equal(m, r["mass_scale"] * L.MASS) and np.array_equal(c, L.COM + r["com_shift"])
    assert np.array_equal(I, r["inertia_scale"][:, None, None] * L.INERTIA)


def _golden():
    return json.load(open(os.path.join(HERE, "golden", "rbd_mujoco_links.json")))


def _record(fields):
    return hb.make_link_variations(1, fields["mass_scale"], np.array(fields["com_shift"]), fields["inertia_scale"])[0]


def test_changes_against_mujoco():
    """The changes of M and nle from the nominal model, from MuJoCo on edited MJCF inertials (tests/golden/gen_rbd_mujoco_links.py), against
    link_ref's changes. The MJCF stores rounded inertials (test_oracle_rbd.py holds M and nle to 1e-5 relative), and the changes are
    products of the same rounded values, so each record's changes are held to 1e-5 of their own size (measured: <= 1.4e-6); the golden's 7
    digits round them by at most 5e-8 of that."""
    d = _golden()
    assert len(d["records"]) >= 8 and len(d["states"]) >= 2
    low = np.tril_indices(16)
    for rec in d["records"]:
        record = _record(rec)
        got = [L.changes(np.array(s["q"]), np.array(s["v"]), record) for s in d["states"]]
        for k, want in ((0, [np.array(m) for m in rec["dM"]]), (1, [np.array(n) for n in rec["dnle"]])):
            size = max(np.abs(w).max() for w in want)
            assert size > 1e-5, rec["name"]
            for g, w in zip(got, want):
                g = g[k][low] if k == 0 else g[k]
                assert np.abs(g - w).max() < 1e-5 * size, (rec["name"], "Mn"[k], np.abs(g - w).max(), size)


@pytest.mark.parametrize("seed", range(4))
def test_varied_mass_matrix(oracle, seed):
    rec = _random_record(10 + seed)
    m, _, _ = L.bodies(rec)
    lo = L.LinkOracle(oracle, rec)
    for q, v in _states(3, 20 + seed):
        M = lo.rbd(q, v)["M"]
        assert np.abs(M - M.T).max() < 1e-12 * np.abs(M).max()
        assert np.linalg.eigvalsh(0.5 * (M + M.T)).min() > 0
        assert np.abs(M[:3, :3] - m.sum() * np.eye(3)).max() < 1e-12 * m.sum()
        pc, vc, w, Iw = L.body_motion(q, v, L.bodies(rec))
        ke = sum(0.5 * m[b] * vc[b] @ vc[b] + 0.5 * w[b] @ Iw[b] @ w[b] for b in range(11))
        assert abs(0.5 * v @ M @ v - ke) < 1e-12 * ke


@pytest.mark.parametrize("seed", range(3))
def test_varied_gravity_is_the_potential_gradient(oracle, seed):
    rec = _random_record(30 + seed)
    body = L.bodies(rec)
    lo = L.LinkOracle(oracle, rec)

    def potential(q):
        return L.G * (body[0] * L.body_motion(q, np.zeros(16), body)[0][:, 2]).sum()

    for q, _ in _states(2, 40 + seed):
        g = lo.rbd(q, np.zeros(16))["nle"]
        h = 1e-6
        fd = np.array([(potential(q + h * e) - potential(q - h * e)) / (2 * h) for e in np.eye(16)])
        assert np.abs(g - fd).max() < 1e-6 * np.abs(g).max()


def test_sweep_tool_parses_help():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "link_sweep.py"), "--help"], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    assert out.stdout.startswith("usage: link_sweep.py") and all(a in out.stdout for a in ("--batch", "--wbc", "--estimator", "--sensor-noise"))
