"""ctypes loader for the CPU oracle (test infrastructure only).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module.
"""
import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
NX, NU, NQ = 22, 22, 16


class Horizon(C.Structure):
    _fields_ = [("N", C.c_int), ("dt", C.c_double), ("dts", C.c_void_p)]


def _horizon(N, dt):
    """dt: scalar (uniform grid) or an array of N interval lengths (non-uniform grid). Returns (Horizon, keep-alive array)."""
    if np.ndim(dt) == 0:
        return Horizon(N, float(dt), None), None
    dts = np.ascontiguousarray(dt, dtype=np.float64)
    assert dts.shape == (N,)
    return Horizon(N, float(dts[0]), dts.ctypes.data), dts


class SolveInfo(C.Structure):
    _fields_ = [("alpha", C.c_double), ("merit0", C.c_double), ("merit1", C.c_double), ("viol0", C.c_double),
                ("viol1", C.c_double), ("armijo", C.c_double), ("status", C.c_int), ("n_trials", C.c_int)]


class LsTrial(C.Structure):
    _fields_ = [("alpha", C.c_double), ("merit", C.c_double), ("viol", C.c_double), ("branch", C.c_int), ("accepted", C.c_int)]


LS_BRANCHES = ("violation", "armijo", "filter")      # HBO_LS_VIOLATION, HBO_LS_ARMIJO, HBO_LS_FILTER
LS_MAX_TRIALS = 14                                   # hb_config.line_search_max_trials by default: alpha = 1, 1/2, ... >= 1e-4


def build():
    subprocess.check_call(["make", "-s", "-C", _HERE])


def lib():
    global _LIB
    if _LIB is None:
        p = os.path.join(_HERE, "libhb_oracle.so")
        if not os.path.exists(p):
            build()
        _LIB = C.CDLL(p)
        _LIB.hbo_init()
        _LIB.hbo_qp_solve.restype = C.c_int
        _LIB.hbo_wbc_solve.restype = C.c_int
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _d(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def rbd(q, v):
    q, v = _d(q), _d(v)
    M = np.zeros((16, 16)); nle = np.zeros(16); J = np.zeros((12, 16)); dJv = np.zeros(12); A = np.zeros((6, 16))
    com = np.zeros(3); h = np.zeros(6); cpos = np.zeros(12)
    lib().hbo_rbd(_p(q), _p(v), _p(M), _p(nle), _p(J), _p(dJv), _p(A), _p(com), _p(h), _p(cpos))
    return dict(M=M, nle=nle, J=J, dJv=dJv, A=A, com=com, h=h, cpos=cpos)


def set_wbc_settings(values=None):
    """Override the WBC gains / limits / weights of the oracle (17 doubles in the order of hb_wbc_settings); None restores the shipped values."""
    if values is None:
        lib().hbo_set_wbc_settings(None)
    else:
        v = _d(values); assert v.size == 17
        lib().hbo_set_wbc_settings(_p(v))


def observer_terms(q, v):
    """p = M v, generalised gravity, C' v and the 6-D toe-frame Jacobians of both feet (momentum observer, StateEstimateBase.cpp:157-190)."""
    q, v = _d(q), _d(v)
    p = np.zeros(16); g = np.zeros(16); ctv = np.zeros(16); J = np.zeros((2, 6, 16))
    lib().hbo_observer_terms(_p(q), _p(v), _p(p), _p(g), _p(ctv), _p(J))
    return p, g, ctv, J


def rbd_to_centroidal(rbd_state):
    r = _d(rbd_state); x = np.zeros(22)
    lib().hbo_rbd_to_centroidal(_p(r), _p(x))
    return x


def flow_map(x, u, jac=True):
    x, u = _d(x), _d(u)
    f = np.zeros(22); A = np.zeros((22, 22)); B = np.zeros((22, 22))
    lib().hbo_flow_map(_p(x), _p(u), _p(f), _p(A) if jac else None, _p(B) if jac else None)
    return (f, A, B) if jac else f


def ee_kinematics(x, u):
    x, u = _d(x), _d(u)
    pos = np.zeros(12); vel = np.zeros(12); dp = np.zeros((12, 22)); dvx = np.zeros((12, 22)); dvu = np.zeros((12, 22))
    lib().hbo_ee_kinematics(_p(x), _p(u), _p(pos), _p(vel), _p(dp), _p(dvx), _p(dvu))
    return pos, vel, dp, dvx, dvu


def input_cost_R():
    R = np.zeros((22, 22)); lib().hbo_input_cost_R(_p(R)); return R


def node_lq(dt, x, u, xn, xref, swing, mode):
    x, u, xn, xref, swing = map(_d, (x, u, xn, xref, swing))
    o = dict(Ad=np.zeros((22, 22)), Bd=np.zeros((22, 22)), b=np.zeros(22), Q=np.zeros((22, 22)), R=np.zeros((22, 22)),
             P=np.zeros((22, 22)), q=np.zeros(22), r=np.zeros(22), C=np.zeros((16, 22)), D=np.zeros((16, 22)), e=np.zeros(16))
    m = C.c_int(0); cost = C.c_double(0)
    lib().hbo_node_lq(C.c_double(dt), _p(x), _p(u), _p(xn), _p(xref), _p(swing), C.c_int(mode), _p(o["Ad"]), _p(o["Bd"]), _p(o["b"]),
                      _p(o["Q"]), _p(o["R"]), _p(o["P"]), _p(o["q"]), _p(o["r"]), _p(o["C"]), _p(o["D"]), _p(o["e"]), C.byref(m), C.byref(cost))
    o["m"] = m.value; o["cost"] = cost.value
    return o


def mpc_cold_start(N, dt, x0, mode):
    hz, _keep = _horizon(N, dt); x0 = _d(x0); mode = np.ascontiguousarray(mode, dtype=np.int32)
    xt = np.zeros((N + 1, 22)); ut = np.zeros((N, 22))
    lib().hbo_mpc_cold_start(C.byref(hz), _p(x0), _p(mode), _p(xt), _p(ut))
    return xt, ut


def mpc_iteration(N, dt, x0, x_ref, swing, mode, xt, ut, max_trials=LS_MAX_TRIALS, record=False):
    """One SQP iteration with at most max_trials line-search trials. record: also return the line search's trials, one dict per trial
    (alpha, merit, viol, branch: one of LS_BRANCHES, accepted: bool), as a fourth result."""
    hz, _keep = _horizon(N, dt)
    x0, x_ref, swing = _d(x0), _d(x_ref), _d(swing)
    mode = np.ascontiguousarray(mode, dtype=np.int32)
    xt = _d(xt).copy(); ut = _d(ut).copy()
    info = SolveInfo()
    rows = (LsTrial * max(1, max_trials))()
    lib().hbo_mpc_iteration(C.byref(hz), C.c_int(max_trials), _p(x0), _p(x_ref), _p(swing), _p(mode), _p(xt), _p(ut), C.byref(info), rows)
    info = {k: getattr(info, k) for k, _ in SolveInfo._fields_}
    if not record:
        return xt, ut, info
    trials = [dict(alpha=r.alpha, merit=r.merit, viol=r.viol, branch=LS_BRANCHES[r.branch], accepted=bool(r.accepted))
              for r in rows[:info["n_trials"]]]
    return xt, ut, info, trials


def mpc_iteration_batch(N, dt, x0, x_ref, swing, mode, xt, ut, threads=1):
    hz, _keep = _horizon(N, dt)
    B = x0.shape[0]
    x0, x_ref, swing = _d(x0), _d(x_ref), _d(swing)
    mode = np.ascontiguousarray(mode, dtype=np.int32)
    xt = _d(xt).copy(); ut = _d(ut).copy()
    infos = (SolveInfo * B)()
    lib().hbo_mpc_iteration_batch(C.byref(hz), C.c_int(B), C.c_int(threads), _p(x0), _p(x_ref), _p(swing), _p(mode), _p(xt), _p(ut), infos)
    return xt, ut, [{k: getattr(i, k) for k, _ in SolveInfo._fields_} for i in infos]


def wbc_assemble(x_des, u_des, rbd_state, mode, stance_mode=False):
    x_des, u_des, r = _d(x_des), _d(u_des), _d(rbd_state)
    H = np.zeros((38, 38)); g = np.zeros(38); A = np.zeros((60, 38)); lb = np.zeros(60); ub = np.zeros(60); m = C.c_int(0)
    lib().hbo_wbc_assemble(_p(x_des), _p(u_des), _p(r), C.c_int(mode), C.c_int(int(stance_mode)), _p(H), _p(g), _p(A), _p(lb), _p(ub), C.byref(m))
    return H, g, A[:m.value].copy(), lb[:m.value].copy(), ub[:m.value].copy()


def wbc_terms(x_des, u_des, rbd_state, mode):
    """Pieces of the WBC problem for the hierarchical formulation: weighted task rows (Aw, bw), contact Jacobian J, dJ/dt v."""
    x_des, u_des, r = _d(x_des), _d(u_des), _d(rbd_state)
    Aw = np.zeros((24, 38)); bw = np.zeros(24); J = np.zeros((12, 16)); dJv = np.zeros(12); rw = C.c_int(0)
    lib().hbo_wbc_terms(_p(x_des), _p(u_des), _p(r), C.c_int(mode), _p(Aw), _p(bw), C.byref(rw), _p(J), _p(dJv))
    return Aw[:rw.value].copy(), bw[:rw.value].copy(), J, dJv


def qp_solve(H, g, A, lbA, ubA, rho):
    H, g, A, lbA, ubA = map(_d, (H, g, A, lbA, ubA))
    n = g.size; m = lbA.size; x = np.zeros(n); it = C.c_int(0)
    st = lib().hbo_qp_solve(C.c_int(n), C.c_int(m), _p(H), _p(g), _p(A), _p(lbA), _p(ubA), C.c_double(rho), _p(x), C.byref(it))
    return x, st, it.value


def wbc_solve(x_des, u_des, rbd_state, mode, stance_mode=False, rho=1e-6):
    x_des, u_des, r = _d(x_des), _d(u_des), _d(rbd_state)
    sol = np.zeros(38)
    st = lib().hbo_wbc_solve(_p(x_des), _p(u_des), _p(r), C.c_int(mode), C.c_int(int(stance_mode)), C.c_double(rho), _p(sol))
    return sol, st


def wbc_solve_batch(x_des, u_des, rbd_state, mode, stance_mode, rho=1e-6, threads=1):
    x_des, u_des, r = _d(x_des), _d(u_des), _d(rbd_state)
    B = x_des.shape[0]
    mode = np.ascontiguousarray(mode, dtype=np.int32); sm = np.ascontiguousarray(stance_mode, dtype=np.uint8)
    sol = np.zeros((B, 38)); st = np.zeros(B, dtype=np.int32)
    lib().hbo_wbc_solve_batch(C.c_int(B), C.c_int(threads), _p(x_des), _p(u_des), _p(r), _p(mode), _p(sm), C.c_double(rho), _p(sol), _p(st))
    return sol, st


def wbc_qp_batch(H, g, A, lbA, ubA, rho=1e-6, threads=1):
    H, g, A, lbA, ubA = map(_d, (H, g, A, lbA, ubA))
    B, n = g.shape; m = lbA.shape[1]
    x = np.zeros((B, n)); st = np.zeros(B, dtype=np.int32)
    lib().hbo_wbc_qp_batch(C.c_int(B), C.c_int(threads), C.c_int(n), C.c_int(m), _p(H), _p(g), _p(A), _p(lbA), _p(ubA), C.c_double(rho), _p(x), _p(st))
    return x, st
