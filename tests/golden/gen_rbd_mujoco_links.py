#!/usr/bin/env python3
"""Generate tests/golden/rbd_mujoco_links.json: M and nle of the Hunter with varied bodies (hb_link_variation), computed with the
reference's vendored MuJoCo 3.0.1 binary, on states of tests/golden/rbd_mujoco.json.

Usage: gen_rbd_mujoco_links.py REFERENCE_CHECKOUT. The MJCF is patched as gen_rbd_mujoco.py patches it (its probe and patch are reused).
For each record, the inertial of every varied body is then replaced (fullinertia) so that the body merged with its welded children (the
imu on the base, the toe and heel bodies on leg_l5 / leg_r5, as tools/gen_model.py merges them) has the record's parameters: mass
mass_scale m, CoM c + com_shift and inertia about it inertia_scale I, where m, c, I are the MJCF's merged values. The JSON holds the
records, the states and, per record and state, the changes of M and nle from the nominal model (reference coordinates, 7 significant
digits): dM as its lower triangle row by row (136 entries, M is symmetric), dnle (16 entries).
"""
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import gen_rbd_mujoco as g  # noqa: E402  (reads REFERENCE_CHECKOUT from sys.argv[1])

NAMES = ["base_link", "leg_l1_link", "leg_l2_link", "leg_l3_link", "leg_l4_link", "leg_l5_link",
         "leg_r1_link", "leg_r2_link", "leg_r3_link", "leg_r4_link", "leg_r5_link"]
WELDED = {0: ["imu_link"], 5: ["leg_l_f1_link", "leg_l_f2_link"], 10: ["leg_r_f1_link", "leg_r_f2_link"]}
STATES = (0, 1)      # of rbd_mujoco.json's cases: the default pose at rest, a random pose moving


def _inertial(xml, name):
    """(match, pos, mass, inertia about the CoM in the body frame) of body `name`'s inertial element, and the body's pos attribute."""
    m = re.search(r'<body name="%s"([^>]*)>\s*(<inertial[^>]*/>)' % name, xml, re.S)
    el = m.group(2)
    attr = lambda k: np.array([float(t) for t in re.search(r'\b%s="([^"]*)"' % k, el).group(1).split()])   # noqa: E731
    pos, mass, d = attr("pos"), float(attr("mass")[0]), attr("diaginertia")
    w, x, y, z = attr("quat") if re.search(r'\bquat="', el) else (1.0, 0.0, 0.0, 0.0)
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                  [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                  [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    bpos = np.array([float(t) for t in re.search(r'pos="([^"]*)"', m.group(1)).group(1).split()]) if 'pos="' in m.group(1) else np.zeros(3)
    return m, pos, mass, R @ np.diag(d) @ R.T, bpos


def _about_origin(m, c, Ic):
    return Ic + m * (np.dot(c, c) * np.eye(3) - np.outer(c, c))


def vary(xml, record):
    """The patched MJCF with the inertials of the bodies the record varies replaced."""
    for b, name in enumerate(NAMES):
        s, dc, si = record["mass_scale"][b], np.array(record["com_shift"][b]), record["inertia_scale"][b]
        if s == 1.0 and si == 1.0 and not dc.any():
            continue
        own, c0, m0, I0, _ = _inertial(xml, name)
        kids = []
        for k in WELDED.get(b, []):
            _, ck, mk, Ik, pk = _inertial(xml, k)
            kids.append((mk, pk + ck, Ik))            # the child's CoM in the parent's frame (welded without rotation)
        M = m0 + sum(k[0] for k in kids)
        C = (m0 * c0 + sum(k[0] * k[1] for k in kids)) / M
        Io = _about_origin(m0, c0, I0) + sum(_about_origin(*k) for k in kids)
        Ic = Io - M * (np.dot(C, C) * np.eye(3) - np.outer(C, C))         # the merged body about its CoM
        M1, C1, I1 = s * M, C + dc, si * Ic
        Io1 = _about_origin(M1, C1, I1) - sum(_about_origin(*k) for k in kids)
        m_own = M1 - sum(k[0] for k in kids)
        c_own = (M1 * C1 - sum(k[0] * k[1] for k in kids)) / m_own
        I_own = Io1 - m_own * (np.dot(c_own, c_own) * np.eye(3) - np.outer(c_own, c_own))
        assert m_own > 0 and np.linalg.eigvalsh(I_own).min() > 0, name
        el = '<inertial pos="%s" mass="%.17g" fullinertia="%s"/>' % (" ".join("%.17g" % x for x in c_own), m_own,
                                                                     " ".join("%.17g" % x for x in (I_own[0, 0], I_own[1, 1], I_own[2, 2],
                                                                                                     I_own[0, 1], I_own[0, 2], I_own[1, 2])))
        xml = xml[:own.start(2)] + el + xml[own.end(2):]
    return xml


def records():
    """(name, record): each body type alone, varied in mass, CoM and inertia at once; every leg link scaled; the base lightened."""
    def rec(**kw):
        r = dict(mass_scale=[1.0] * 11, com_shift=[[0.0] * 3 for _ in range(11)], inertia_scale=[1.0] * 11)
        for k, (bs, v) in kw.items():
            for b in bs:
                r[k][b] = v
        return r
    out = []
    for b, shift in ((0, [0.01, -0.005, 0.02]), (1, [0.0, 0.01, -0.01]), (2, [0.005, 0.0, -0.02]), (3, [0.0, 0.0, -0.02]),
                     (4, [0.0, 0.0, -0.02]), (5, [0.002, 0.0, -0.002])):
        out.append(("%s mass x1.2, com shift, inertia x1.5" % NAMES[b], rec(mass_scale=([b], 1.2), com_shift=([b], shift), inertia_scale=([b], 1.5))))
    legs = list(range(1, 11))
    out += [("all leg links x1.5", rec(mass_scale=(legs, 1.5), inertia_scale=(legs, 1.5))),
            ("base lightened x0.8", rec(mass_scale=([0], 0.8), inertia_scale=([0], 0.8)))]
    return out


def probe(exe, xml, states):
    p = os.path.join(tempfile.mkdtemp(), "hunter_links.xml")
    open(p, "w").write(xml)
    lines = []
    for q, v in states:
        R, T = g.Rzyx(q[3:6]), g.Tmap(q[3:6])
        lines.append(" ".join("%.17g" % a for a in np.concatenate([q[0:3], g.quat_from_R(R), q[6:], v[0:3], R.T @ T @ v[3:6], v[6:]])))
    out = subprocess.run([exe, p], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout.splitlines()
    Ms, ns = [], []
    for (q, v), line in zip(states, out[1:]):                 # the conversion of gen_rbd_mujoco.py to the reference's coordinates
        a = np.array([float(t) for t in line.split()])
        M, bias = a[:256].reshape(16, 16), a[256:272]
        R, T = g.Rzyx(q[3:6]), g.Tmap(q[3:6])
        G = np.eye(16); G[3:6, 3:6] = R.T @ T
        eps = 1e-6
        wdot = (g.Tmap(q[3:6] + eps * v[3:6]) @ v[3:6] - g.Tmap(q[3:6] - eps * v[3:6]) @ v[3:6]) / (2 * eps)
        Gdot_v = np.zeros(16); Gdot_v[3:6] = R.T @ wdot
        Ms.append(G.T @ M @ G)
        ns.append(G.T @ (M @ Gdot_v + bias))
    return Ms, ns


def main():
    if g.REF is None:
        sys.exit(__doc__)
    exe, xml = g.build_probe(), open(g.patched_xml()).read()
    cases = json.load(open(os.path.join(HERE, "rbd_mujoco.json")))["cases"]
    states = [(np.array(cases[k]["q"]), np.array(cases[k]["v"])) for k in STATES]
    M0, n0 = probe(exe, xml, states)
    out = dict(source="MuJoCo 3.0.1 (reference vendored binary) on patched mujoco/model/hunter/hunter.xml with edited inertials",
               states=[dict(q=q.tolist(), v=v.tolist()) for q, v in states], records=[])
    low = np.tril_indices(16)
    digits = lambda a: [float("%.7g" % x) for x in a]          # noqa: E731
    for name, r in records():
        M, n = probe(exe, vary(xml, r), states)
        out["records"].append(dict(name=name, **r, dM=[digits((M[k] - M0[k])[low]) for k in range(len(states))],
                                   dnle=[digits(n[k] - n0[k]) for k in range(len(states))]))
    json.dump(out, open(os.path.join(HERE, "rbd_mujoco_links.json"), "w"), separators=(",", ":"))
    print("wrote rbd_mujoco_links.json:", len(out["records"]), "records on", len(states), "states")


if __name__ == "__main__":
    main()
