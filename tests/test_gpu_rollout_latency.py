"""MPC latency in the batched episodes (hb_rollout_set_mpc_latencies) and the MRT split behind it (hb_policy_update, hb_policy_wbc). The latency
episode is checked bit for bit against the loop of public calls (episode_ref.stepwise: the adoptions through hb_policy_update, the 500 Hz tick
through hb_policy_wbc), with latencies 0, 1, 2, mpc_every - 1 and mpc_every and one instance beyond the setting, under both WBC formulations,
truth and estimator, both time grids, and together with pushes and plant variations; then the setting's contract (null settings, continuation
across a split between a cycle and its adoption, independence, permutation, instances beyond the setting, launch counts, argument checks) and
the MRT entry points on their own (adoption, the mask, the held policy, the shared WBC fallback)."""
import ctypes as C

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from episode_ref import (FRICTION, GAITS, GAIT_START, PUSH, assert_continues, assert_episode_equal, assert_null_settings, assert_rejected_settings,
                         assert_setting_episodes, cmd_vels, context, device, est_params, horizon, latency_due, outputs, params, start_states, stepwise,
                         use)

pytestmark = pytest.mark.gpu

EVERY = 5                                   # params()'s mpc_every (hb_default_rollout_params): 100 Hz MPC at 500 Hz
LATENCIES = [0, 1, 2, EVERY - 1, EVERY]                              # six robots: the sixth is beyond the setting


def _due_ticks(latencies, ticks, every):
    """The ticks of `ticks` on which some instance of the setting adopts (one launch each)."""
    return sum(1 for a in ticks if latency_due(np.array(latencies), a, every).any())


@pytest.mark.parametrize("wbc", ["weighted", "hierarchical"])
@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_latency_episode_equals_the_stepwise_loop_bitwise(wbc, event_nodes, estimated):
    ctx = context(event_nodes)
    ctx.set_wbc_formulation(wbc)
    B, log_every = 6, 10
    n_ticks = 120 if estimated else 160
    rbd0 = start_states(ctx, B, seed=81)
    vels = cmd_vels(B)
    prm = params(log_every)
    extra = {}
    if wbc == "weighted" and not event_nodes:         # the latency together with pushes and plant variations
        extra = dict(plant_variations=hb.make_plant_variations(B, friction_scale=FRICTION, motor_strength=0.95),
                     pushes=hb.make_push_schedules(B, 0.15, 0.05, PUSH))
    kw = use(ctx, mpc_latencies=LATENCIES, **extra)
    ep = est_params(seed=2027) if estimated else None
    d = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 50) if estimated else None)
    r = stepwise(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 50) if estimated else None, **kw)
    assert (outputs(d)[3]["wbc_fallbacks"] == 0).all() and (r[3]["wbc_fallbacks"] == 0).all()
    assert_episode_equal(d, r)
    # the latency really delays: the instances with d >= 1 move, latency 0 and the instance beyond the setting do not
    ctx.set_mpc_latencies(None)
    u = device(ctx, rbd0, GAITS, vels, n_ticks, prm, log_every, ep, hb.estimation_states(B, 50) if estimated else None)
    moved = [not np.array_equal(a, b) for a, b in zip(d[0].cpu().numpy(), u[0].cpu().numpy())]
    assert moved == [False, True, True, True, True, False], moved
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_zero_latencies_change_nothing(estimated):
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=82)
    vels = cmd_vels(B)
    ep = est_params(seed=6) if estimated else None
    assert_null_settings(ctx, "mpc_latencies", lambda: device(ctx, rbd0, GAITS, vels, 100, params(5), 5, ep), ([0] * B, [0] * 3),
                         [1, 2, 3, 4, 5, 0])
    ctx.close()


def _lat(values):
    return [C.c_int32(int(v)) for v in values]


def test_continuation_independence_permutation_and_instances_beyond_the_setting():
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=83)
    full = _lat([3, 1, 5, 2, 4, 3])
    one = _lat([2, 0, 0, 0, 0, 0])
    other = _lat([5, 4, 1, 2, 3, 1])              # instance 3 keeps its latency
    assert_setting_episodes(ctx, "mpc_latencies", rbd0, params(10), full, one, other, 3, _lat([3, 1, 5]), _lat([3, 1, 5, 0, 0, 0]))
    # splits between a cycle and its adoption: the cycle at tick 100, adopted at 103 (d = 3) and 101 (d = 1)
    ctx.set_mpc_latencies([3, 3, 1, 3, 5, 0])
    assert_continues(ctx, rbd0, GAITS, cmd_vels(B), 200, 101, params(1), 1)
    assert_continues(ctx, rbd0, GAITS, cmd_vels(B), 200, 102, params(1), 1, est_params(seed=3))
    ctx.close()


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
def test_launch_counts(estimated):
    """A latency setting adds one launch on every tick where an instance within it adopts, and one on the cold tick: checked against the
    unset episode over a cold call and warm calls of 10, 23 and 7 ticks, for several settings."""
    ctx = context()
    B = 6
    rbd0 = start_states(ctx, B, seed=84)
    vels = cmd_vels(B)
    ep = est_params(seed=4) if estimated else None
    prm = params(0)

    def counts():
        c0 = ctx.launch_count
        out = device(ctx, rbd0, GAITS, vels, 10, prm, 0, ep)
        n = [ctx.launch_count - c0]
        tick0 = 10
        for k in (10, 23, 7):
            c0 = ctx.launch_count
            out = device(ctx, out[0], GAITS, vels, k, prm, 0, ep, out[5] if ep else None, tick0=tick0, act=out[1], estop=out[2], stats=out[3],
                         est_stats=out[6] if ep else None)
            n.append(ctx.launch_count - c0)
            tick0 += k
        return n

    ctx.set_mpc_latencies(None)
    plain = counts()
    spans = [range(0, 10), range(10, 20), range(20, 43), range(43, 50)]
    for setting in ([1], [0, 2, 0], [5, 5], [1, 2, 3, 4, 5, 0], [4, 0, 0, 0, 0, 3]):
        ctx.set_mpc_latencies(setting)
        got = counts()
        want = [p + _due_ticks(setting, s, prm.mpc_every) + (1 if k == 0 and any(d >= 1 for d in setting) else 0)
                for k, (p, s) in enumerate(zip(plain, spans))]
        assert got == want, (setting, got, want, plain)
    ctx.close()


def test_argument_checks_return_before_any_launch_and_keep_the_setting():
    ctx = context(max_batch=6)
    lib = ctx._lib
    B = 6
    rbd0 = start_states(ctx, B, seed=85)
    vels = cmd_vels(B)
    arr = lambda v: (C.c_int32 * len(v))(*v)          # noqa: E731
    good = arr([1, 2, 3, 4, 5, 0])
    bad = [arr([1, 2, -1, 4, 5, 0]), arr([-2 ** 31, 0, 0, 0, 0, 0])]
    big = arr([1] * (B + 1))
    assert_rejected_settings(ctx, "mpc_latencies", lambda: device(ctx, rbd0, GAITS, vels, 30, params(10), 10), good, bad, big)
    # a latency above the episode's mpc_every: rejected by the episode call before any launch; the setting stays and runs at a slower cadence
    ctx.set_mpc_latencies([1, 6])
    prm = params(0)
    c0 = ctx.launch_count
    with pytest.raises(hb.HunterB200Error):
        device(ctx, rbd0, GAITS, vels, 10, prm, 0)
    assert ctx.launch_count == c0
    prm.mpc_every = 6
    out = outputs(device(ctx, rbd0, GAITS, vels, 20, prm, 0))
    assert (out[3]["fail_tick"] < 0).all()
    # a warm call in which an instance with a latency has never adopted a policy
    fresh = context(max_batch=6)
    first = device(fresh, rbd0, GAITS, vels, 10, params(0), 0)
    fresh.set_mpc_latencies([0, 0, 2])
    c0 = fresh.launch_count
    with pytest.raises(hb.HunterB200Error):
        device(fresh, first[0], GAITS, vels, 10, params(0), 0, tick0=10, act=first[1], estop=first[2], stats=first[3])
    assert fresh.launch_count == c0
    fresh.set_mpc_latencies([2, 0, 0])          # instance 0 has never adopted either
    with pytest.raises(hb.HunterB200Error):
        device(fresh, first[0], GAITS, vels, 10, params(0), 0, tick0=10, act=first[1], estop=first[2], stats=first[3])
    fresh.set_mpc_latencies([0, 0, 0])
    device(fresh, first[0], GAITS, vels, 10, params(0), 0, tick0=10, act=first[1], estop=first[2], stats=first[3])
    fresh.close()
    ctx.close()


def _mrt_context(event_nodes):
    ctx = context(event_nodes, max_batch=8)
    B = 8
    rbd0 = start_states(ctx, B, seed=86)
    return ctx, B, rbd0


def _cycle(ctx, B, rbd, t, cold):
    x0 = ctx.rbd_to_centroidal(rbd)
    ins = hb.make_plan_inputs(np.full(B, t), horizon(ctx), x0, cmd_vels(B)[:, 1], None, ["trot"] * B, GAIT_START)
    info, _, _, st, ps = ctx.resident_plan_cycle(cold, 0.0, ins, rbd)
    assert (info["status"] == 0).all() and (st == 0).all() and (ps == 0).all()


def _wbc_equal(a, b, rows=slice(None)):
    for x, y in zip(a, b):
        assert np.array_equal(x[rows], y[rows])


@pytest.mark.parametrize("event_nodes", [False, True], ids=["uniform", "event_nodes"])
def test_mrt_entry_points_adopt_hold_and_mask(event_nodes):
    """policy_update then policy_wbc equals resident_wbc bit for bit; after the next cycle the held policy is the resident one of a second
    context that stopped one cycle earlier; a mask adopts only the flagged instances."""
    ctx, B, rbd = _mrt_context(event_nodes)
    held, _, _ = _mrt_context(event_nodes)
    lib = ctx._lib
    d_rbd = rbd.copy()
    t_rbd = rbd.copy()
    assert lib.hb_policy_wbc(ctx._h, B, *([None] * 9)) == -1
    with pytest.raises(hb.HunterB200Error):              # no adopted policy yet
        ctx.policy_wbc(0.0, rbd)
    with pytest.raises(hb.HunterB200Error):              # no resident solution to adopt
        ctx.policy_update(B)
    for c in (ctx, held):
        _cycle(c, B, rbd, 0.0, True)
    ctx.policy_update(B)
    for t in (0.0, 0.002, 0.006):
        a = ctx.policy_wbc(t, rbd)
        assert (a[5] == 0).all()
        _wbc_equal(a, ctx.resident_wbc(t, rbd))
    # the next cycle at t = 0.01 on ctx only: ctx's adopted policy is still the first solve, held's resident solution too
    d_rbd[:, 5] += 0.002; d_rbd[:, 19] += 0.05
    _cycle(ctx, B, d_rbd, 0.01, False)
    for t in (0.012, 0.014, 0.016):
        a = ctx.policy_wbc(t, t_rbd)
        _wbc_equal(a, held.resident_wbc(t, t_rbd))
        assert not np.array_equal(a[0], ctx.resident_wbc(t, t_rbd)[0])
    # a mask adopts only the flagged instances
    mask = np.arange(B) % 3 == 1
    before = ctx.policy_wbc(0.014, t_rbd)
    ctx.policy_update(B, mask)
    after = ctx.policy_wbc(0.014, t_rbd)
    now = ctx.resident_wbc(0.014, t_rbd)
    _wbc_equal(after, now, mask)
    _wbc_equal(after, before, ~mask)
    assert not any(np.array_equal(before[0][i], now[0][i]) for i in np.nonzero(mask)[0])
    ctx.close(); held.close()


def test_policy_wbc_shares_the_weighted_fallback_and_checks_its_arguments():
    """The WeightedWbc fallback state is the context's, whichever of resident_wbc and policy_wbc solved last: a policy_wbc whose QP does not
    solve returns the last good solution of a resident_wbc, and the other way round."""
    ctx, B, rbd = _mrt_context(False)
    _cycle(ctx, B, rbd, 0.0, True)
    ctx.policy_update(B)
    bad = rbd.copy()
    bad[1:3, 6] = np.nan                              # a joint angle the WBC cannot take: its QP does not solve
    good = ctx.resident_wbc(0.004, rbd)
    got = ctx.policy_wbc(0.004, bad)
    assert (got[5][1:3] != 0).all() and (got[5][[0, 3, 4, 5, 6, 7]] == 0).all()
    assert np.array_equal(got[3][1:3], good[3][1:3]) and np.array_equal(got[4][1:3], good[4][1:3])
    good = ctx.policy_wbc(0.006, rbd)
    got = ctx.resident_wbc(0.006, bad)
    assert np.array_equal(got[3][1:3], good[3][1:3]) and (got[5][1:3] != 0).all()
    # argument checks of the MRT entry points: empty batch, negative batch, NULL required pointers, capacity; no launch
    lib, h = ctx._lib, ctx._h
    dummy = np.zeros(1 << 12)
    P = C.c_void_p(dummy.ctypes.data)
    c0 = ctx.launch_count
    for name in ("hb_policy_wbc", "hb_policy_wbc_async"):
        spec = [P, P, None, P, P, P, P, None, None]
        f = getattr(lib, name)
        assert f(h, 0, *spec) == 0 and f(h, -1, *spec) == -1
        for k in (0, 1, 3, 4, 5, 6):
            assert f(h, 1, *[None if j == k else a for j, a in enumerate(spec)]) == -1, (name, k)
    assert lib.hb_policy_wbc(h, B + 1, *spec) == -4
    assert lib.hb_policy_update(h, 0, None) == 0 and lib.hb_policy_update(h, -1, None) == -1 and lib.hb_policy_update(None, 1, None) == -1
    assert lib.hb_policy_update(h, B + 1, None) == -4
    assert ctx.launch_count == c0
    ctx.close()
