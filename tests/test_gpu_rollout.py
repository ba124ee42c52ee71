"""SURVEY 8f row N2: the closed loop as a batched roll-out -- actuation model with command delay (LeggedHWSim.cpp:166-192), a batched
rigid-body plant, MPC at 100 Hz on the resident solution and policy + WeightedWbc + joint command law at 500 Hz (LeggedController::update)."""
import collections

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from episode_ref import GROUND, plant_numpy, start_states

pytestmark = pytest.mark.gpu


def test_actuation_delay_matches_deque_restatement(gpu_ctx):
    """cmdBuffer_ semantics: push the new command, drop entries older than `delay`, apply the oldest remaining one with the current joint state."""
    B, delay, period = 5, 0.009, 0.002
    rng = np.random.default_rng(3)
    st = hb.actuation_states(B)
    bufs = [collections.deque() for _ in range(B)]
    for k in range(40):
        t = np.full(B, period * (k + 1)) + (0.0005 if k > 20 else 0.0)       # a jitter in the tick times half way through
        cmd = rng.uniform(-1, 1, (B, 10, 5)); cmd[:, :, 2:4] = rng.uniform(0, 40, (B, 10, 2))
        rbd = rng.uniform(-0.5, 0.5, (B, 32))
        tau = gpu_ctx.actuation(t, st, cmd, rbd, delay)
        for i in range(B):
            buf = bufs[i]
            while buf and buf[-1][0] + delay < t[i]:
                buf.pop()
            buf.appendleft((t[i], cmd[i].copy()))
            c = buf[-1][1]
            ref = c[:, 2] * (c[:, 0] - rbd[i, 6:16]) + c[:, 3] * (c[:, 1] - rbd[i, 22:32]) + c[:, 4]
            assert np.abs(tau[i] - ref).max() < 1e-12
            assert st[i].count == len(buf)
    assert max(len(b) for b in bufs) >= 5      # 9 ms of delay at 500 Hz keeps five commands in flight


def test_plant_step_matches_numpy_restatement(gpu_ctx, oracle):
    from hunter_bipedal_control_b200 import scenarios as sc
    B = 10
    rng = np.random.default_rng(8)
    x = sc.random_initial_states(B, seed=50)
    rbd = sc.consistent_rbd(x, rng, 0.02)
    rbd[:, 5] = rng.uniform(0.60, 0.64, B)               # some feet in the ground, some above it
    tau = rng.uniform(-15, 15, (B, 10))
    prm = hb.default_sim_params()
    nxt, cf, fl = gpu_ctx.sim_step(rbd, tau, prm)
    touched = 0
    for i in range(B):
        ref, F, _ = plant_numpy(oracle, rbd[i], tau[i], prm)
        assert np.abs(nxt[i] - ref).max() < 1e-9 * max(1.0, np.abs(ref).max()), i
        assert np.abs(cf[i] - F).max() < 1e-7 * max(1.0, np.abs(F).max())
        assert np.array_equal(fl[i] != 0, F[2::3] > 0)
        touched += int((F[2::3] > 0).sum())
    assert 0 < touched < 4 * B


def test_dynamic_closed_loop_standing_rollout(oracle):
    """0.4 s of closed loop on the batched plant: MPC every 10 ms (warm-started resident solution), policy + WBC + joint command law +
    delayed actuation every 2 ms. The robots must keep standing: base height and attitude stay put, no emergency stop, torques inside limits."""
    from hunter_bipedal_control_b200 import scenarios as sc
    B, N, dt = 4, 50, 0.02
    ctx = hb.Context(horizon_N=N, dt=dt, max_batch=B, device=0)
    rbd = start_states(ctx, B, seed=2)                        # the contact springs start loaded with about the weight
    z0 = rbd[:, 5].copy()
    compacts = []
    for i in range(B):
        xi = ctx.rbd_to_centroidal(rbd[i:i + 1])[0]
        compacts.append(sc.make_reference(xi, (0.0, 0.0, 0.0, 0.0), "stance", N, dt)[3])
        compacts[-1]["target_times"] = np.array([0.0, 10.0])          # hold the pose
        compacts[-1]["target_states"][:, 8] = z0[i]
    refs = sc.pack_references(compacts, 3.0)
    act = hb.actuation_states(B)
    prm = hb.default_sim_params()
    prm.ground_height = GROUND
    estop = np.zeros(B, dtype=np.uint8)
    period = 0.002
    tau_lim = np.tile([28, 60, 60, 60, 28], 2)
    heights = []
    for tick in range(200):
        t = tick * period
        if tick % 5 == 0:
            x_meas = ctx.rbd_to_centroidal(rbd)
            info, _, _, st = ctx.resident_cycle(tick == 0, 0.0, np.full(B, t), x_meas, refs, rbd)
            assert (info["status"] == 0).all()
        xd, ud, md, sol, tau_ff, st = ctx.resident_wbc(t, rbd)
        assert (md == 3).all()
        cmd, tau_cmd, estop = ctx.joint_command(period, xd, ud, sol, md, rbd, estop=estop)
        tau = ctx.actuation(t, act, cmd, rbd, 0.009)
        tau = np.clip(tau, -tau_lim, tau_lim)                  # actuator saturation
        rbd, cf, fl = ctx.sim_step(rbd, tau, prm)
        assert np.isfinite(rbd).all()
        heights.append(rbd[:, 5].copy())
    heights = np.array(heights)
    assert (estop == 0).all()
    assert np.abs(heights[-50:] - z0[None]).max() < 0.03, np.abs(heights[-50:] - z0[None]).max()
    assert np.abs(rbd[:, 1:3]).max() < 0.1                                       # pitch, roll
    assert np.abs(rbd[:, 16:32]).max() < 1.0                                     # it came to rest
    assert (cf[:, 2::3].sum(axis=1) > 0.8 * sc.TOTAL_MASS * 9.81).all() and (cf[:, 2::3].sum(axis=1) < 1.2 * sc.TOTAL_MASS * 9.81).all()
    ctx.close()
