"""Nodes outside the three regular classes of the Riccati sweep (stance nt = 12, single support nt = 9, flight nt = 6).

When the contact-velocity rows lose rank, the projection keeps more null-space inputs and the node takes the general path of
`riccati_node`, which reads its column classes from the record at run time. A vertical left foot does that: with the left hip
yaw at 0 and the left ankle at 0.53 - pi/2 (hip pitch 0.4, knee 0.93), the toe-heel line of the left foot is vertical, so the
z-velocity rows of its two contacts coincide. A flight node then has nt = 7 and a node with the left foot in swing nt = 10.
The CPU test checks that on the oracle; the GPU test runs a flying-trot SQP iteration through such nodes against the oracle."""
import numpy as np
import pytest

N, DT = 100, 0.01


def vertical_left_foot_state():
    from hunter_bipedal_control_b200 import scenarios as sc
    x = sc.INITIAL_STATE.copy()
    x[12] = 0.0                      # left hip yaw
    x[16] = 0.53 - np.pi / 2         # left ankle: foot pitched by -pi/2 from level
    return x


def oracle_nt(o):
    """Free inputs of the oracle's least-squares projection (project_constraints in oracle/hb_oracle.cpp): Gauss-Jordan on D'D with
    diagonal pivoting and the rank threshold 1e-9 of the largest diagonal entry."""
    D = o["D"][:o["m"]]
    G = D.T @ D
    tol = 1e-9 * max(np.diag(G).max(), 1e-300)
    piv = np.zeros(G.shape[0], bool)
    for _ in range(G.shape[0]):
        d = np.where(piv, -np.inf, np.diag(G))
        p = int(np.argmax(d))
        if not d[p] > tol:
            break
        piv[p] = True
        G[p] /= G[p, p]
        for i in range(G.shape[0]):
            if i != p:
                G[i] -= G[i, p] * G[p]
    return int((~piv).sum())


def flying_trot_case():
    from hunter_bipedal_control_b200 import scenarios as sc
    x0 = vertical_left_foot_state()
    x_ref, swing, mode, _ = sc.make_reference(x0, (0.2, 0.0, 0.0, 0.0), "flying_trot", N, DT)
    return x0, x_ref, swing, mode


def node_classes(oracle, x0, x_ref, swing, mode, xt, ut):
    """(mode, nt) of every node of the warm start, as the oracle's projection sees them."""
    out = []
    for k in range(N):
        xk = x0 if k == 0 else xt[k]
        o = oracle.node_lq(DT, xk, ut[k], xt[k + 1], x_ref[k], swing[k], int(mode[k]))
        out.append((int(mode[k]), oracle_nt(o)))
    return out


def test_vertical_foot_gives_irregular_nodes(oracle):
    x0, x_ref, swing, mode = flying_trot_case()
    xt, ut = oracle.mpc_cold_start(N, DT, x0, mode)
    classes = set(node_classes(oracle, x0, x_ref, swing, mode, xt, ut))
    assert (0, 7) in classes and (1, 10) in classes, classes       # flight and left-swing nodes with one extra null-space input
    assert (2, 9) in classes, classes                               # the right foot keeps left-stance nodes regular


@pytest.mark.gpu
def test_irregular_nodes_vs_oracle(gpu_ctx, oracle):
    x0, x_ref, swing, mode = flying_trot_case()
    xt, ut = gpu_ctx.mpc_cold_start(x0[None], mode[None])
    xo0, uo0 = oracle.mpc_cold_start(N, DT, x0, mode)
    assert np.abs(xt[0] - xo0).max() < 1e-12 and np.abs(ut[0] - uo0).max() < 1e-12
    classes = node_classes(oracle, x0, x_ref, swing, mode, xt[0], ut[0])
    assert sum(nt not in (12, 9, 6) for _, nt in classes) >= 10, classes
    xt1, ut1, info = gpu_ctx.mpc_solve(x0[None], x_ref[None], swing[None], mode[None], xt, ut)
    assert info["status"][0] == 0, info
    xo, uo, io = oracle.mpc_iteration(N, DT, x0, x_ref, swing, mode, xt[0], ut[0])
    assert io["status"] == 0 and io["alpha"] > 0, io
    assert abs(io["alpha"] - info["alpha"][0]) < 1e-12, (io, info)
    assert np.abs(xo - xt1[0]).max() < 1e-6 * max(1.0, np.abs(xo).max()), np.abs(xo - xt1[0]).max()
    assert np.abs(uo - ut1[0]).max() < 1e-5 * max(1.0, np.abs(uo).max()), np.abs(uo - ut1[0]).max()
