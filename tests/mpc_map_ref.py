"""MPC maps for their tests (test_mpc_maps_host.py, test_gpu_mpc_maps.py): the stance heights a solve reads, restated from hunter_b200.h's
"MPC maps", and the CPU oracle given those heights (mpc_map_oracle.cpp: oracle/hb_oracle.cpp compiled as it is, with the stance z row's
offset lowered by 3 h), with oracle/hbo.py's node_lq, mpc_iteration and mpc_iteration_batch plus a stance_h argument.

At node k, contact c in stance there is held at 0.02 + h(m, swing[k][6c], swing[k][6c + 1]); every other entry is +0. The lookup is
height_map_ref.h (episode_ref.terrain_height, whose Python products round on their own as the device lookup's do), so these heights are
the device's bit for bit."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from height_map_ref import h
from oracle import hbo

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "mpc_map_oracle.cpp")
ORACLE = os.path.join(HERE, "..", "oracle")
_LIB = None


def in_stance(mode, c):
    """contact_flag of MotionPhaseDefinition.h: contacts 0, 2 (left toe, heel) stand in modes 2, 3; contacts 1, 3 in modes 1, 3."""
    return int(mode) in ((1, 3) if c & 1 else (2, 3))


def stance_heights(m, swing, mode):
    """(N+1) x 4 heights of one instance on the map m (an HbTerrain; None: no map, all +0). swing: (N+1) x 24, mode: N+1."""
    sw = np.asarray(swing, dtype=float).reshape(-1, 24)
    out = np.zeros((sw.shape[0], 4))
    if m is None:
        return out
    for k in range(sw.shape[0]):
        for c in range(4):
            if in_stance(mode[k], c):
                out[k, c] = h(m, sw[k, 6 * c], sw[k, 6 * c + 1])
    return out


def stance_heights_batch(maps, swing, mode):
    """B x (N+1) x 4 heights; maps[i] for instance i < len(maps), instances beyond it without a map."""
    maps = [] if maps is None else list(maps)
    return np.stack([stance_heights(maps[i] if i < len(maps) else None, swing[i], mode[i]) for i in range(len(swing))])


# ---------------------------------------------------------------------------------------------------------------- the oracle on heights
def lib():
    """mpc_map_oracle.cpp as a shared library, built once per source state into the temporary directory (the tree may be read-only) with
    the oracle's own compiler flags (oracle/Makefile)."""
    global _LIB
    if _LIB is None:
        deps = [SRC] + [os.path.join(ORACLE, f) for f in ("hb_oracle.cpp", "hb_oracle.hpp", "hb_rbd.hpp", "hb_dual.hpp")]
        deps.append(os.path.join(HERE, "..", "include", "hunter_model_constants.h"))
        key = hashlib.sha256(b"".join(open(f, "rb").read() for f in deps)).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), "hb_mpc_map_oracle_%s_%d.so" % (key, os.getuid()))
        if not os.path.exists(so):
            tmp = "%s.%d.tmp" % (so, os.getpid())
            subprocess.check_call(["g++", "-O3", "-march=x86-64-v3", "-std=c++17", "-fPIC", "-shared", "-o", tmp, SRC, "-lpthread"])
            os.replace(tmp, so)
        _LIB = C.CDLL(so)
        _LIB.hbo_init()
    return _LIB


def _heights(stance_h, shape):
    if stance_h is None:
        return None
    a = np.ascontiguousarray(stance_h, dtype=np.float64)
    assert a.shape == shape, (a.shape, shape)
    return a


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def node_lq(dt, x, u, xn, xref, swing, mode, stance_h=None):
    """hbo.node_lq; stance_h (4, optional): the ground under each contact of the node, a stance contact held at 0.02 + stance_h[c]."""
    x, u, xn, xref, swing = (np.ascontiguousarray(a, dtype=np.float64) for a in (x, u, xn, xref, swing))
    sh = _heights(stance_h, (4,))
    o = dict(Ad=np.zeros((22, 22)), Bd=np.zeros((22, 22)), b=np.zeros(22), Q=np.zeros((22, 22)), R=np.zeros((22, 22)),
             P=np.zeros((22, 22)), q=np.zeros(22), r=np.zeros(22), C=np.zeros((16, 22)), D=np.zeros((16, 22)), e=np.zeros(16))
    m = C.c_int(0); cost = C.c_double(0)
    lib().hbt_node_lq(C.c_double(dt), *map(_ptr, (x, u, xn, xref, swing)), C.c_int(int(mode)),
                      *(_ptr(o[k]) for k in ("Ad", "Bd", "b", "Q", "R", "P", "q", "r", "C", "D", "e")), C.byref(m), C.byref(cost), _ptr(sh))
    o["m"] = m.value; o["cost"] = cost.value
    return o


def mpc_iteration(N, dt, x0, x_ref, swing, mode, xt, ut, max_trials=hbo.LS_MAX_TRIALS, record=False, stance_h=None):
    """hbo.mpc_iteration; stance_h ((N+1) x 4, optional): the ground under each contact of every node, as node_lq's."""
    hz, _keep = hbo._horizon(N, dt)
    x0, x_ref, swing = (np.ascontiguousarray(a, dtype=np.float64) for a in (x0, x_ref, swing))
    mode = np.ascontiguousarray(mode, dtype=np.int32)
    xt = np.array(xt, dtype=np.float64); ut = np.array(ut, dtype=np.float64)
    sh = _heights(stance_h, (N + 1, 4))
    info = hbo.SolveInfo()
    rows = (hbo.LsTrial * max(1, max_trials))()
    lib().hbt_mpc_iteration(C.byref(hz), C.c_int(max_trials), *map(_ptr, (x0, x_ref, swing, mode, xt, ut)), C.byref(info), rows, _ptr(sh))
    info = {k: getattr(info, k) for k, _ in hbo.SolveInfo._fields_}
    if not record:
        return xt, ut, info
    trials = [dict(alpha=r.alpha, merit=r.merit, viol=r.viol, branch=hbo.LS_BRANCHES[r.branch], accepted=bool(r.accepted))
              for r in rows[:info["n_trials"]]]
    return xt, ut, info, trials


def mpc_iteration_batch(N, dt, x0, x_ref, swing, mode, xt, ut, stance_h=None):
    """hbo.mpc_iteration_batch on one thread; stance_h (B x (N+1) x 4, optional): each instance's as mpc_iteration's."""
    hz, _keep = hbo._horizon(N, dt)
    B = x0.shape[0]
    x0, x_ref, swing = (np.ascontiguousarray(a, dtype=np.float64) for a in (x0, x_ref, swing))
    mode = np.ascontiguousarray(mode, dtype=np.int32)
    xt = np.array(xt, dtype=np.float64); ut = np.array(ut, dtype=np.float64)
    sh = _heights(stance_h, (B, N + 1, 4))
    infos = (hbo.SolveInfo * B)()
    lib().hbt_mpc_iteration_batch(C.byref(hz), C.c_int(B), *map(_ptr, (x0, x_ref, swing, mode, xt, ut)), infos, _ptr(sh))
    return xt, ut, [{k: getattr(i, k) for k, _ in hbo.SolveInfo._fields_} for i in infos]
