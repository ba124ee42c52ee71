"""The reference-side adapters (adapters/B200Wbc.h : legged::WbcBase, adapters/B200Mpc.h : ocs2::MPC_BASE) as real code: compiled against
minimal stand-ins of the reference / OCS2 headers (tests/adapter_stubs/), linked with libhunter_b200.so, and -- on the GPU -- driven the way
LeggedController drives wbc_ and mpc_, with the results checked against the same steps through the Python binding."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "hunter_bipedal_control_b200")
INC = ["-I" + os.path.join(ROOT, "adapters"), "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "tests", "adapter_stubs")]


def build_driver(out_dir):
    """The driver program, built in out_dir: the repository tree may be read-only."""
    exe = os.path.join(out_dir, "adapters_main")
    src = os.path.join(ROOT, "tests", "adapters_main.cpp")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror"] + INC + ["-o", exe, src, "-L" + PKG, "-l:libhunter_b200.so", "-Wl,-rpath," + PKG])
    return exe


def test_adapters_compile_and_link_against_the_c_abi(tmp_path):
    """Each header on its own (self-contained includes), then the driver program linked with the shared library."""
    for h in ("B200Wbc.h", "B200Mpc.h"):
        subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-Werror"] + INC + ["-x", "c++", "-"], input=('#include "%s"\n' % h).encode(), check=True)
    assert os.path.exists(build_driver(tmp_path))


@pytest.mark.gpu
def test_adapters_drive_the_gpu_path_like_the_controller(tmp_path):
    import hunter_bipedal_control_b200 as hb
    from hunter_bipedal_control_b200 import scenarios as sc
    from test_gpu_event_nodes import _shift_numpy
    exe = build_driver(tmp_path)
    task = os.path.join(ROOT, "tests", "golden", "task_wbc_variant.info")
    rng = np.random.default_rng(17)
    # ---- WBC cases: (mode, stance flag, setKpKd or not)
    cases = [(3, 1, 0.0, 0.0), (3, 0, 0.0, 0.0), (2, 0, 120.0, 11.0), (1, 0, 0.0, 0.0)]
    xs = np.tile(sc.INITIAL_STATE, (len(cases), 1)) + rng.uniform(-.03, .03, (len(cases), 22))
    us = np.zeros((len(cases), 22))
    for i, (m, _, _, _) in enumerate(cases):
        fl = sc.mode_flags(m)
        us[i, 2:12:3] = np.array(fl) * sc.TOTAL_MASS * 9.81 / sum(fl)
        us[i, 12:] = rng.uniform(-.3, .3, 10)
    rbds = sc.consistent_rbd(xs, rng, 0.01)
    # ---- MPC scenario at the shipped discretisation
    dt, T, cap = 0.015, 0.8, int(np.ceil(0.8 / 0.015)) + 12
    x0 = sc.random_initial_states(1, seed=5)[0]
    comp = sc.make_reference(x0, (0.3, 0.0, 0.0, 0.1), "trot", 54, dt, t0=0.0, phase=0.137)[3]
    cycles = [(0.0, x0), (0.01, x0 + 1e-3), (0.02, x0 + 2e-3)]
    scen = tmp_path / "scenario.txt"; outp = tmp_path / "out.txt"
    with open(scen, "w") as f:
        f.write(task + "\n%d\n" % len(cases))
        for i, (m, st, kp, kd) in enumerate(cases):
            f.write("%d %d %r %r\n" % (m, st, kp, kd) + " ".join(repr(float(v)) for v in np.r_[xs[i], us[i], rbds[i]]) + "\n")
        f.write("%r %r\n%d\n" % (dt, T, len(comp["events"])))
        f.write(" ".join(repr(float(e)) for e in comp["events"]) + "\n" + " ".join(str(int(m)) for m in comp["modes"]) + "\n")
        f.write("%d\n" % len(comp["target_times"]))
        for t, s in zip(comp["target_times"], comp["target_states"]):
            f.write(repr(float(t)) + " " + " ".join(repr(float(v)) for v in s) + "\n")
        for c in range(4):
            for a in range(3):
                segs = comp["segments"][c][a]
                f.write("%d\n" % len(segs) + "".join(" ".join(repr(float(v)) for v in sg) + "\n" for sg in segs))
        f.write("%d\n" % len(cycles))
        for t, x in cycles:
            f.write(repr(float(t)) + " " + " ".join(repr(float(v)) for v in x) + "\n")
    subprocess.run([exe, str(scen), str(outp)], check=True, timeout=300)
    lines = open(outp).read().splitlines()
    wbc_lines = [np.array(l.split()[1:], dtype=float) for l in lines if l.startswith("wbc")]
    mpc_lines = [np.array(l.split()[1:], dtype=float) for l in lines if l.startswith("mpc")]
    assert len(wbc_lines) == len(cases) and len(mpc_lines) == len(cycles)
    # ---- the same WBC calls through the Python binding: identical
    ctx = hb.Context(horizon_N=1, max_batch=1, device=0)
    ctx.load_task_info(task)
    for i, (m, st, kp, kd) in enumerate(cases):
        if kp > 0:
            ctx.set_kp_kd(kp, kd)
        sol, status = ctx.wbc_solve(xs[i:i + 1], us[i:i + 1], rbds[i:i + 1], [m], [st])
        assert status[0] == 0 and np.array_equal(sol[0], wbc_lines[i]), i
    ctx.close()
    # ---- the same MPC cycles: grid, references on the grid, warm start between grids, one SQP iteration
    ctx = hb.Context(horizon_N=cap, dt=dt, max_batch=1, device=0, time_horizon=T, event_nodes=True)
    refs = sc.pack_references([comp], 3.0)
    prev = None
    for (t, x), line in zip(cycles, mpc_lines):
        n1 = int(line[0]); body = line[1:1 + n1 * 45].reshape(n1, 45); u_mid = line[1 + n1 * 45:]
        tk, nn, st = ctx.time_grid(np.array([t]), refs)
        n = int(nn[0]); g = tk[0, :n + 1]
        assert n1 == n + 1 and np.abs(body[:, 0] - g).max() < 1e-12
        xr, sw, md = sc.sample_reference(comp, tk[0])
        if prev is None:
            xs0, us0 = ctx.mpc_cold_start(x[None], md[None])
            xs0, us0 = xs0[0], us0[0]
        else:
            xw, uw = _shift_numpy(prev[0], len(prev[0]) - 1, prev[1], prev[2], g, n, x, md)
            xs0 = np.zeros((cap + 1, 22)); us0 = np.zeros((cap, 22)); xs0[:n + 1] = xw; us0[:n] = uw
        xt, ut, info = ctx.mpc_solve_grid(x[None], tk, nn, xr[None], sw[None], md[None], xs0[None], us0[None])
        assert info["status"][0] == 0
        assert np.abs(body[:, 1:23] - xt[0, :n + 1]).max() < 1e-9 * max(1.0, np.abs(xt[0]).max())
        assert np.abs(body[:n, 23:] - ut[0, :n]).max() < 1e-8 * max(1.0, np.abs(ut[0]).max())
        assert np.array_equal(body[n, 23:], body[n - 1, 23:])                      # the last input sample is repeated at the final node
        k = int(np.clip(np.searchsorted(g, t + 0.002, side="right") - 1, 0, n - 1)); al = (t + 0.002 - g[k]) / (g[k + 1] - g[k])
        assert np.abs(u_mid - ((1 - al) * body[k, 23:] + al * body[k + 1, 23:])).max() < 1e-9 * max(1.0, np.abs(u_mid).max())
        prev = (g.copy(), xt[0, :n + 1].copy(), ut[0, :n].copy())
    ctx.close()
