"""The motor bridge in the episodes (hb_rollout_set_motor_bridge): the device codec against the host codec, the bridged plant step against
the numpy plant's per-substep motor PD, a neutral bridge on a one-substep plant against the unbridged episode, a bridged episode against
the loop of public calls (episode_ref.stepwise on bridge_ref.BridgeLoop), the setting's contract, snapshots, and the encoders' quantisation grid."""
import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import scenarios as sc
from bridge_ref import BridgeLoop, plant_bridged
from episode_ref import (FRICTION, GAITS, PUSH, array_of, assert_episode_equal, assert_null_settings, assert_rejected_settings,
                         assert_setting_episodes, cmd_vels, context, device, est_params, outputs, params, random_goals, small_terrains,
                         start_states, stepwise, use)

pytestmark = pytest.mark.gpu

B = 6
FAR = 1e300                    # a range that never binds
nan, inf = float("nan"), float("inf")


def _same(a, b):
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.uint64), np.asarray(b, dtype=np.float64).view(np.uint64))


def _random_bridges(n, rng):
    """Records across the whole envelope: random scales, directions, zeros and ranges, quantise 0 and 1."""
    return hb.make_motor_bridges(n, command_scale=rng.uniform(0.0, 1.5, (n, 10)), direction=rng.choice([-1, 1], (n, 10)),
                                 zero=rng.uniform(-0.5, 0.5, (n, 10)) * (rng.random((n, 1)) < 0.7), kp_max=rng.uniform(50, 600, (n, 10)),
                                 kd_max=rng.uniform(0.5, 6, (n, 10)), pos_max=rng.uniform(1.0, 13.0, (n, 10)), vel_max=rng.uniform(2, 20, (n, 10)),
                                 ff_max=rng.uniform(5, 100, (n, 10)), quantise=rng.integers(0, 2, n))


def _neutral(n, directions):
    """Scale 1, the given directions, zero 0, no quantisation, ranges that never bind."""
    return hb.make_motor_bridges(n, command_scale=1.0, direction=directions, zero=0.0, kp_max=FAR, kd_max=FAR, pos_max=FAR, vel_max=FAR,
                                 ff_max=FAR, quantise=0)


# ---------------------------------------------------------------------------------------------------------------- 1. the codec
def test_device_codec_equals_the_host_codec_bitwise(gpu_ctx):
    """Commands through the actuation call (delay 0: the newest entry is applied) and joint readings through the sensor read (no noise),
    on 1024 random records, random values over and beyond each range and the special values."""
    rng = np.random.default_rng(1)
    n = 1024
    br = _random_bridges(n, rng)
    br[0] = hb.default_motor_bridge()
    cmd = np.stack([rng.uniform(-15, 15, (n, 10)), rng.uniform(-25, 25, (n, 10)), rng.uniform(-50, 700, (n, 10)), rng.uniform(-1, 8, (n, 10)),
                    rng.uniform(-120, 120, (n, 10))], axis=2)
    special = np.array([nan, inf, -inf, 0.0, -0.0, 1e39, -1e39, 12.5, -12.5, 18.0])
    cmd[1:11] = special[:, None, None]
    want = hb.bridge_encode(br, cmd)
    got = gpu_ctx.actuation(0.0, hb.actuation_states(n), cmd, np.zeros((n, 32)), delay=0.0, bridge=br)
    assert _same(got, want)
    rbd = sc.consistent_rbd(sc.random_initial_states(n, seed=3))
    rbd[:, 6:16] = rng.uniform(-14, 14, (n, 10)); rbd[:, 22:32] = rng.uniform(-22, 22, (n, 10))
    rbd[1:11, 6:16] = special[:, None]; rbd[1:11, 22:32] = special[::-1, None]
    _, _, _, jp, jv = gpu_ctx.read_sensors(rbd, hb.estimation_states(n), 0, bridge=br)
    wq, wqd = hb.bridge_feedback(br, rbd[:, 6:16], rbd[:, 22:32])
    assert _same(jp, wq) and _same(jv, wqd)
    assert not np.array_equal(jp[0], rbd[0, 6:16])          # the default record quantises


# ---------------------------------------------------------------------------------------------------------------- 2. the plant step
def test_bridged_plant_step_matches_the_numpy_motor_pd(gpu_ctx, oracle):
    rng = np.random.default_rng(8)
    n = 12
    rbd = sc.consistent_rbd(sc.random_initial_states(n, seed=48), rng, 0.02)
    rbd[:, 5] = rng.uniform(0.60, 0.64, n)
    jcmd = np.stack([rbd[:, 6:16] + rng.uniform(-0.2, 0.2, (n, 10)), rng.uniform(-1, 1, (n, 10)), rng.uniform(20, 60, (n, 10)),
                     rng.uniform(0.01, 3, (n, 10)), rng.uniform(-40, 40, (n, 10))], axis=2)
    br = _random_bridges(n, rng)
    br[0] = hb.default_motor_bridge()
    mcmd = hb.bridge_encode(br, jcmd)
    lim = rng.uniform(10, 60, (n, 10))
    V = hb.make_plant_variations(n, motor_strength=rng.uniform(0.5, 1.2, (n, 10)))
    for prm_sub, var in ((4, None), (3, V)):
        prm = hb.default_sim_params(); prm.substeps = prm_sub
        nxt, cf, _, applied = gpu_ctx.sim_step(rbd, mcmd, prm, variation=var, bridge=br, limits=lim)
        for i in range(n):
            ref, F, _, ap = plant_bridged(oracle, rbd[i], prm, br[i], mcmd[i], lim[i], None if var is None else var[i])
            assert np.abs(nxt[i] - ref).max() < 1e-9 * max(1.0, np.abs(ref).max()), (i, np.abs(nxt[i] - ref).max())
            assert np.abs(applied[i] - ap).max() < 1e-9 * max(1.0, np.abs(ap).max()), i
            assert np.abs(cf[i] - F).max() < 1e-7 * max(1.0, np.abs(F).max()), i
        assert (np.abs(applied) <= lim).all() and (np.abs(applied) == lim).any()


def test_neutral_bridge_on_one_substep_is_the_plain_plant_step_bitwise(gpu_ctx):
    rng = np.random.default_rng(9)
    n = 16
    rbd = sc.consistent_rbd(sc.random_initial_states(n, seed=49), rng, 0.02)
    jcmd = rng.normal(0.0, 5.0, (n, 10, 5))
    jcmd[:, :, 2:4] = np.abs(jcmd[:, :, 2:4])                # gains >= 0, as the joint command law writes them: the clamps never bind
    prm = hb.default_sim_params(); prm.substeps = 1
    lim = np.full(10, 25.0)
    for d in (np.ones(10, dtype=int), -np.ones(10, dtype=int), rng.choice([-1, 1], 10)):
        br = _neutral(n, d)
        tau = np.clip(gpu_ctx.actuation(0.0, hb.actuation_states(n), jcmd, rbd, delay=0.0), -lim, lim)
        mcmd = gpu_ctx.actuation(0.0, hb.actuation_states(n), jcmd, rbd, delay=0.0, bridge=br)
        a = gpu_ctx.sim_step(rbd, tau, prm)
        b = gpu_ctx.sim_step(rbd, mcmd, prm, bridge=br, limits=lim)
        for x, y in zip(a, b):
            assert _same(x, y)
        assert _same(b[3], tau)


# ---------------------------------------------------------------------------------------------------------------- 3. neutral episodes
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_neutral_bridge_is_the_unbridged_episode_bitwise(estimated):
    """On a one-substep plant, neutral records (directions +1 on some robots, -1 on others, mixed on the rest) give the unset episode bit
    for bit, with the same launches: null settings."""
    ctx = context()
    rbd0 = start_states(ctx, B, seed=201)
    prm = params(5); prm.sim.substeps = 1
    ep = est_params(seed=21) if estimated else None
    dirs = np.array([[1] * 10, [-1] * 10, [1, -1] * 5, [-1, 1, 1, -1, 1, 1, -1, -1, 1, -1], [1] * 10, [-1] * 10])
    assert_null_settings(ctx, "motor_bridge", lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 60, prm, 5, ep, hb.estimation_states(B, 50) if estimated else None),
                         [_neutral(B, dirs), _neutral(3, dirs[:3])], hb.make_motor_bridges(B))
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 4. the loop of public calls
def _records(n):
    """The default record, and the same without quantisation, with the 0.7 hip scale off, and with zero offsets."""
    out = []
    for k in range(n):
        r = hb.default_motor_bridge()
        if k % 4 == 1:
            r.quantise = 0
        elif k % 4 == 2:
            r.command_scale[:] = [1.0] * 10
        elif k % 4 == 3:
            r.zero[:] = list(np.linspace(-0.05, 0.05, 10))
        out.append(r)
    return array_of(out)


@pytest.mark.parametrize("wbc", ["weighted", "hierarchical"])
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_bridged_episode_equals_the_stepwise_loop_bitwise(wbc, event_nodes, estimated):
    """Bridges on all robots but the last, with pushes, plant variations, a terrain, goals, an MPC latency, hardware and controller
    settings set alongside."""
    ctx = context(event_nodes)
    ctx.set_wbc_formulation(wbc)
    n_ticks, log_every = 80, 10
    rbd0 = start_states(ctx, B, seed=202)
    vels = cmd_vels(B)
    prm = params(log_every)
    kw = use(ctx, plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION, motor_strength=0.95),
             pushes=hb.make_push_schedules(B, 0.05, 0.05, PUSH), terrains=small_terrains(), goals=random_goals(rbd0, B, 202),
             mpc_latencies=[0, 2, 5, 1, 0, 3], motor_bridge=_records(B - 1),
             hardware=hb.make_hardware_settings(B, actuation_delay=np.linspace(0.0, 0.012, B), encoder_offset=np.linspace(-0.01, 0.01, 10),
                                                torque_limit=np.linspace(1.0, 0.8, B)[:, None] * np.array(prm.torque_limit[:])))
    g = hb.default_pd_gains(); g.kp_big_stance = 45.0
    ctx.set_controller_settings(hb.make_controller_settings(B, wbc=ctx.wbc_settings(), gains=g))
    ep = est_params(seed=2035) if estimated else None
    fresh = (lambda: hb.estimation_states(B, 70)) if estimated else (lambda: None)
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, fresh())
    prm.gains = g
    loop = BridgeLoop(ctx, kw.pop("motor_bridge"), prm.torque_limit)
    r = stepwise(loop, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, fresh(), **kw)
    assert_episode_equal(d, r)
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 5. the contract
def test_setting_contract():
    ctx = context()
    rbd0 = start_states(ctx, B, seed=203)
    r = list(_records(4)) + [_neutral(1, [-1] * 10)[0]]
    full = array_of([r[0], r[1], r[2], r[3], r[4], r[0]])
    one = array_of([r[0]])
    other = array_of([r[3], r[2], r[1], r[3], r[0], r[1]])       # instance 3 keeps its record
    part = array_of([r[2], r[0]])
    assert_setting_episodes(ctx, "motor_bridge", rbd0, params(10), full, one, other, 3, part, part)
    ctx.close()


def _bad():
    out = []
    for field, j, v in [("direction", 3, 0), ("direction", 0, 2), ("command_scale", 1, nan), ("command_scale", 5, -0.1), ("zero", 2, inf),
                        ("kp_max", 0, 0.0), ("kd_max", 4, -5.0), ("pos_max", 6, inf), ("vel_max", 8, nan), ("ff_max", 2, 0.0), ("quantise", None, 2)]:
        recs = hb.make_motor_bridges(2)
        if j is None:
            setattr(recs[1], field, v)
        else:
            getattr(recs[1], field)[j] = v
        out.append(recs)
    return out


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_rejected_settings(estimated):
    ctx = context()
    rbd0 = start_states(ctx, B, seed=204)
    ep = est_params(seed=11) if estimated else None
    assert_rejected_settings(ctx, "motor_bridge",
                             lambda: device(ctx, rbd0, GAITS, cmd_vels(B), 40, params(5), 5, ep, hb.estimation_states(B, 50) if estimated else None),
                             _records(B), _bad(), hb.make_motor_bridges(ctx.max_batch + 1))
    rbd = np.zeros((2, 32))
    for bad in _bad():                                  # the host calls validate their records as the setter does
        with pytest.raises(hb.HunterB200Error):
            ctx.actuation(0.0, hb.actuation_states(2), np.zeros((2, 10, 5)), rbd, bridge=bad)
        with pytest.raises(hb.HunterB200Error):
            ctx.sim_step(rbd, np.zeros((2, 10, 5)), bridge=bad, limits=np.ones(10))
        with pytest.raises(hb.HunterB200Error):
            ctx.read_sensors(rbd, hb.estimation_states(2), 0, bridge=bad)
    with pytest.raises(hb.HunterB200Error):
        ctx.sim_step(rbd, np.zeros((2, 10, 5)), bridge=hb.make_motor_bridges(2), limits=np.r_[np.ones(9), 0.0])
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_snapshot_resumes_bitwise(estimated):
    """The bridge holds no state: a save after 50 ticks restored into a fresh context with the same settings resumes as one call, and the
    row size does not change."""
    plain = context()
    rbd0 = start_states(plain, B, seed=205)
    unbridged_bytes = plain.episode_state_bytes
    plain.close()
    vels = cmd_vels(B)
    prm = params(1)
    ep = est_params(seed=12) if estimated else None
    fresh = (lambda: hb.estimation_states(B, 50)) if estimated else (lambda: None)

    def configured():
        c = context()
        c.set_motor_bridge(_records(B))
        return c
    ctx = configured()
    bytes0 = ctx.episode_state_bytes
    one = device(ctx, rbd0, GAITS, vels, 100, prm, 1, ep, fresh())
    first = device(ctx, rbd0, GAITS, vels, 50, prm, 1, ep, fresh())
    snap = ctx.save_episodes(B, *first[:4], *(first[5:7] if estimated else ()))
    ctx.close()
    ctx2 = configured()
    assert ctx2.episode_state_bytes == bytes0 == unbridged_bytes
    r = ctx2.restore_episodes(snap)
    if estimated:
        second = device(ctx2, r[0], GAITS, vels, 50, prm, 1, ep, r[4], tick0=50, act=r[1], estop=r[2], stats=r[3], est_stats=r[5])
    else:
        second = device(ctx2, r[0], GAITS, vels, 50, prm, 1, tick0=50, act=r[1], estop=r[2], stats=r[3])
    two = outputs(second)
    two[4] = np.concatenate([first[4].cpu().numpy(), two[4]], axis=1)
    if estimated:
        two[7] = np.concatenate([first[7].cpu().numpy(), two[7]], axis=1)
    assert_episode_equal(one, two)
    ctx2.close()


# ---------------------------------------------------------------------------------------------------------------- 6. properties
def _on_grid(x, lo, hi, bits):
    """Whether each float64 x is one of the protocol's decoded values on [lo, hi] with `bits` bits."""
    f32, n = np.float32, np.float32((1 << bits) - 1)
    flo, span = f32(lo), f32(hi) - f32(lo)
    k0 = np.rint((x - lo) * float(n) / float(span)).astype(np.int64)
    hit = np.zeros(x.shape, dtype=bool)
    for dk in (-1, 0, 1):
        k = np.clip(k0 + dk, 0, int(n)).astype(np.float32)
        hit |= ((k * span) / n + flo).astype(np.float64) == x
    return hit


def test_quantised_encoders_put_every_reading_on_the_grid():
    """quantise = 1, zero 0 and no noise: every estimated joint position is on the 16-bit grid of its motor frame and every joint velocity
    the filter reads on the 12-bit grid, on every tick; the truth is not."""
    ctx = context()
    rbd0 = start_states(ctx, B, seed=206)
    br = hb.make_motor_bridges(B)
    ctx.set_motor_bridge(br)
    ch = hb.make_channels(B, 40, names=["sensors"])
    ctx.set_channels(ch)
    out = outputs(device(ctx, rbd0, GAITS, cmd_vels(B), 40, params(1), 1, est_params(seed=1, scale=0.0), hb.estimation_states(B, 50)))
    d = np.array(br[0].direction[:], dtype=float)
    sensors = ch["sensors"].cpu().numpy()
    assert _on_grid(d * out[7][:, :, 6:16], -12.5, 12.5, 16).all()
    assert _on_grid(d * sensors[:, :, 10:20], -12.5, 12.5, 16).all()
    assert _on_grid(d * sensors[:, :, 20:30], -18.0, 18.0, 12).all()
    assert not _on_grid(d * out[4][:, :, 6:16], -12.5, 12.5, 16).all()
    ctx.set_channels(None)
    ctx.close()
