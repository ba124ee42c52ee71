"""WBC maps restated for their tests (test_wbc_maps_host.py, test_gpu_wbc_maps.py): each stance contact's friction pyramid about the map's
surface normal at the contact's measured position (hunter_b200.h, "WBC maps"), written into the oracle's own QPs. oracle/ is unchanged:
the weighted QP is hbo.wbc_assemble's with the pyramid rows rewritten, solved by hbo.qp_solve; the hierarchical cascade is
oracle/hoqp.py's hierarchical_wbc built on that rewritten assembly.

The frame's products are Python float products, each rounded on its own, as the device's mul_rn products are, and the lookup is
episode_ref.terrain_height (the planner's lookup), so a frame here is the device's bit for bit at the same contact position."""
import math

import numpy as np

from episode_ref import terrain_height
from oracle import hbo

NQ, NJ = 16, 10


def in_stance(mode, c):
    return mode in (1, 3) if c & 1 else mode in (2, 3)


def contact_positions(rbd):
    """The oracle's contact positions (12) at the measured configuration of an rbd state [zyx, p, q_j, omega, v, qd_j]."""
    r = np.asarray(rbd, dtype=float)
    q = np.concatenate([r[3:6], r[0:3], r[6:16]])
    return hbo.rbd(q, np.zeros(NQ))["cpos"]


def frame(m, x, y):
    """(n, t1, t2) of the WBC map m at world (x, y), or None where the gradient is zero (the flat rows stay)."""
    _, gx, gy = terrain_height(m, float(x), float(y))
    if gx == 0.0 and gy == 0.0:
        return None
    L = math.sqrt(1.0 + gx * gx + gy * gy)
    Lt = math.sqrt(1.0 + gx * gx)
    n = (-gx / L, -gy / L, 1.0 / L)
    t1 = (1.0 / Lt, 0.0, gx / Lt)
    t2 = (n[1] * t1[2] - n[2] * t1[1], n[2] * t1[0] - n[0] * t1[2], n[0] * t1[1] - n[1] * t1[0])
    return np.array(n), np.array(t1), np.array(t2)


def frames(m, rbd):
    """The four contacts' frames (None: flat) on map m at the measured contact positions of rbd; all None without a map."""
    if m is None:
        return [None] * 4
    p = contact_positions(rbd)
    return [frame(m, p[3 * c], p[3 * c + 1]) for c in range(4)]


def pyramid(f, mu):
    """The five rows (5 x 3) of one contact's pyramid: the flat rows for f None, else -n, t1 - mu n, -t1 - mu n, t2 - mu n, -t2 - mu n."""
    if f is None:
        return np.array([[0, 0, -1], [1, 0, -mu], [-1, 0, -mu], [0, 1, -mu], [0, -1, -mu]], dtype=float)
    n, t1, t2 = f
    mn = np.array([mu * n[a] for a in range(3)])
    return np.array([-n, t1 - mn, -t1 - mn, t2 - mn, -t2 - mn])


def pyramid_rows(mode):
    """(first row, contacts) of the pyramid rows in hbo.wbc_assemble's A: after the 16 EoM rows, 3 zero-force rows per swing contact and
    the 20 torque-limit rows, 5 rows per stance contact in contact order."""
    st = [c for c in range(4) if in_stance(mode, c)]
    return 16 + 3 * (4 - len(st)) + 2 * NJ, st


def rewrite(A, mode, fr, mu):
    """A copy of the constraint matrix A (hbo.wbc_assemble's) with the pyramid rows of each stance contact that has a frame in fr on it;
    the others keep the oracle's flat rows."""
    A = A.copy()
    r0, st = pyramid_rows(mode)
    for k, c in enumerate(st):
        if fr[c] is None:
            continue
        A[r0 + 5 * k:r0 + 5 * k + 5, :] = 0.0
        A[r0 + 5 * k:r0 + 5 * k + 5, NQ + 3 * c:NQ + 3 * c + 3] = pyramid(fr[c], mu)
    return A


def wbc_assemble(x_des, u_des, rbd, mode, stance_mode=False, m=None, mu=None):
    """hbo.wbc_assemble with the pyramids of map m (None: unchanged). mu: the oracle's friction coefficient in force (hbo.set_wbc_settings)."""
    H, g, A, lb, ub = hbo.wbc_assemble(x_des, u_des, rbd, int(mode), stance_mode)
    return H, g, rewrite(A, int(mode), frames(m, rbd), mu), lb, ub


def wbc_solve(x_des, u_des, rbd, mode, stance_mode=False, m=None, mu=None, rho=1e-8):
    """The weighted WBC on map m: hbo.qp_solve on the rewritten QP. Returns (solution, status)."""
    H, g, A, lb, ub = wbc_assemble(x_des, u_des, rbd, mode, stance_mode, m, mu)
    x, st, _ = hbo.qp_solve(H, g, A, lb, ub, rho)
    return x, st


def hierarchical_wbc(x_des, u_des, rbd, mode, m=None, mu=None):
    """oracle/hoqp.py's hierarchical_wbc on the assembly with map m's pyramids: its own construction, run while hbo.wbc_assemble is the
    rewritten one. Returns what hierarchical_wbc returns."""
    from oracle import hoqp
    plain = hbo.wbc_assemble
    fr = frames(m, rbd)

    def mapped(x, u, r, md, sm=False):
        H, g, A, lb, ub = plain(x, u, r, md, sm)
        return H, g, rewrite(A, int(md), fr, mu), lb, ub

    hbo.wbc_assemble = mapped
    try:
        return hoqp.hierarchical_wbc(x_des, u_des, rbd, int(mode))
    finally:
        hbo.wbc_assemble = plain
