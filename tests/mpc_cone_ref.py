"""MPC cone maps for their tests (test_mpc_cone_maps_host.py, test_gpu_mpc_cone_maps.py): the surface frames a solve's friction cones
stand on, restated from hunter_b200.h's "MPC cone maps", and the CPU oracle given those frames and the MPC maps' stance heights
(mpc_cone_oracle.cpp: mpc_map_oracle.cpp's oracle with each framed cone restated from FrictionConeConstraint.cpp), with oracle/hbo.py's
node_lq, mpc_iteration and mpc_iteration_batch plus stance_h and frames arguments.

At node k, stance contact c's cone bounds t_R_w F, with t_R_w = rows (t1, t2, n) of the frame of the map at (swing[k][6c],
swing[k][6c + 1]); a swing contact, flat ground (a zero gradient) and an instance without a map have the identity, which gives the
oracle's cone bit for bit. The frame is hbplan::map_frame itself (hbc_map_frame), which test_mpc_cone_maps_host.py checks against
wbc_map_ref.frame's Python restatement bit for bit."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from mpc_map_ref import in_stance
from oracle import hbo

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..")
SRC = os.path.join(HERE, "mpc_cone_oracle.cpp")
IDENTITY = np.eye(3).reshape(9)
_LIB = None


def lib():
    """mpc_cone_oracle.cpp as a shared library, built once per source state into the temporary directory (the tree may be read-only) with
    the oracle's own compiler flags (oracle/Makefile)."""
    global _LIB
    if _LIB is None:
        deps = [SRC, os.path.join(HERE, "mpc_map_oracle.cpp")]
        deps += [os.path.join(ROOT, "oracle", f) for f in ("hb_oracle.cpp", "hb_oracle.hpp", "hb_rbd.hpp", "hb_dual.hpp")]
        deps += [os.path.join(ROOT, "include", f) for f in ("hunter_model_constants.h", "hunter_b200.h")]
        deps.append(os.path.join(ROOT, "hunter_bipedal_control_b200", "csrc", "hb_planner.h"))
        key = hashlib.sha256(b"".join(open(f, "rb").read() for f in deps)).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), "hb_mpc_cone_oracle_%s_%d.so" % (key, os.getuid()))
        if not os.path.exists(so):
            tmp = "%s.%d.tmp" % (so, os.getpid())
            subprocess.check_call(["g++", "-O3", "-march=x86-64-v3", "-std=c++17", "-fPIC", "-shared", "-o", tmp, SRC, "-lpthread"])
            os.replace(tmp, so)
        _LIB = C.CDLL(so)
        _LIB.hbo_init()
    return _LIB


def map_frame(m, x, y):
    """hbplan::map_frame: the frame (n, t1, t2) of map m (an HbTerrain) at (x, y) as a 3 x 3 array, or None on flat ground."""
    f = np.zeros(9)
    if not lib().hbc_map_frame(C.byref(m), C.c_double(x), C.c_double(y), f.ctypes.data_as(C.c_void_p)):
        return None
    return f.reshape(3, 3)


def cone_frames(m, swing, mode):
    """(N+1) x 4 x 9 frames t_R_w (rows t1, t2, n) of one instance on the map m (None: no map, every frame the identity).
    swing: (N+1) x 24, mode: N+1."""
    sw = np.asarray(swing, dtype=float).reshape(-1, 24)
    out = np.tile(IDENTITY, (sw.shape[0], 4, 1))
    if m is None:
        return out
    for k in range(sw.shape[0]):
        for c in range(4):
            if in_stance(mode[k], c):
                f = map_frame(m, sw[k, 6 * c], sw[k, 6 * c + 1])
                if f is not None:
                    out[k, c] = np.concatenate([f[1], f[2], f[0]])
    return out


def cone_frames_batch(maps, swing, mode):
    """B x (N+1) x 4 x 9 frames; maps[i] for instance i < len(maps), instances beyond it without a map."""
    maps = [] if maps is None else list(maps)
    return np.stack([cone_frames(maps[i] if i < len(maps) else None, swing[i], mode[i]) for i in range(len(swing))])


def _arr(a, shape):
    if a is None:
        return None
    a = np.ascontiguousarray(a, dtype=np.float64)
    assert a.shape == shape, (a.shape, shape)
    return a


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def node_lq(dt, x, u, xn, xref, swing, mode, stance_h=None, frames=None):
    """hbo.node_lq; stance_h (4, optional): mpc_map_ref.node_lq's heights; frames (4 x 9, optional): each contact's t_R_w."""
    x, u, xn, xref, swing = (np.ascontiguousarray(a, dtype=np.float64) for a in (x, u, xn, xref, swing))
    sh, fr = _arr(stance_h, (4,)), _arr(frames, (4, 9))
    o = dict(Ad=np.zeros((22, 22)), Bd=np.zeros((22, 22)), b=np.zeros(22), Q=np.zeros((22, 22)), R=np.zeros((22, 22)),
             P=np.zeros((22, 22)), q=np.zeros(22), r=np.zeros(22), C=np.zeros((16, 22)), D=np.zeros((16, 22)), e=np.zeros(16))
    m = C.c_int(0); cost = C.c_double(0)
    lib().hbc_node_lq(C.c_double(dt), *map(_ptr, (x, u, xn, xref, swing)), C.c_int(int(mode)),
                      *(_ptr(o[k]) for k in ("Ad", "Bd", "b", "Q", "R", "P", "q", "r", "C", "D", "e")), C.byref(m), C.byref(cost),
                      _ptr(sh), _ptr(fr))
    o["m"] = m.value; o["cost"] = cost.value
    return o


def mpc_iteration(N, dt, x0, x_ref, swing, mode, xt, ut, max_trials=hbo.LS_MAX_TRIALS, record=False, stance_h=None, frames=None):
    """hbo.mpc_iteration; stance_h ((N+1) x 4) and frames ((N+1) x 4 x 9), both optional, as node_lq's for every node."""
    hz, _keep = hbo._horizon(N, dt)
    x0, x_ref, swing = (np.ascontiguousarray(a, dtype=np.float64) for a in (x0, x_ref, swing))
    mode = np.ascontiguousarray(mode, dtype=np.int32)
    xt = np.array(xt, dtype=np.float64); ut = np.array(ut, dtype=np.float64)
    sh, fr = _arr(stance_h, (N + 1, 4)), _arr(frames, (N + 1, 4, 9))
    info = hbo.SolveInfo()
    rows = (hbo.LsTrial * max(1, max_trials))()
    lib().hbc_mpc_iteration(C.byref(hz), C.c_int(max_trials), *map(_ptr, (x0, x_ref, swing, mode, xt, ut)), C.byref(info), rows,
                            _ptr(sh), _ptr(fr))
    info = {k: getattr(info, k) for k, _ in hbo.SolveInfo._fields_}
    if not record:
        return xt, ut, info
    trials = [dict(alpha=r.alpha, merit=r.merit, viol=r.viol, branch=hbo.LS_BRANCHES[r.branch], accepted=bool(r.accepted))
              for r in rows[:info["n_trials"]]]
    return xt, ut, info, trials


def mpc_iteration_batch(N, dt, x0, x_ref, swing, mode, xt, ut, stance_h=None, frames=None):
    """hbo.mpc_iteration_batch on one thread; stance_h (B x (N+1) x 4) and frames (B x (N+1) x 4 x 9), both optional."""
    hz, _keep = hbo._horizon(N, dt)
    B = x0.shape[0]
    x0, x_ref, swing = (np.ascontiguousarray(a, dtype=np.float64) for a in (x0, x_ref, swing))
    mode = np.ascontiguousarray(mode, dtype=np.int32)
    xt = np.array(xt, dtype=np.float64); ut = np.array(ut, dtype=np.float64)
    sh, fr = _arr(stance_h, (B, N + 1, 4)), _arr(frames, (B, N + 1, 4, 9))
    infos = (hbo.SolveInfo * B)()
    lib().hbc_mpc_iteration_batch(C.byref(hz), C.c_int(B), *map(_ptr, (x0, x_ref, swing, mode, xt, ut)), infos, _ptr(sh), _ptr(fr))
    return xt, ut, [{k: getattr(i, k) for k, _ in hbo.SolveInfo._fields_} for i in infos]


def plane_frame(gx, gy):
    """t_R_w (9) of a plane of gradient (gx, gy), in exact float64 arithmetic (numpy): rows t1, t2, n."""
    n = np.array([-gx, -gy, 1.0]) / np.sqrt(1.0 + gx * gx + gy * gy)
    t1 = np.array([1.0, 0.0, gx]) / np.sqrt(1.0 + gx * gx)
    return np.concatenate([t1, np.cross(n, t1), n])
