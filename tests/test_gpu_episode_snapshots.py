"""Episode snapshots (hb_episode_save_async / hb_episode_restore, Context.save_episodes / restore_episodes): an episode saved after n1
ticks and restored into a fresh context continues bit for bit as one call of n1 + n2 ticks, under every per-robot setting; forks,
permutations and identity restores; forked noise streams; launches; and the rejected calls, which change nothing."""
import ctypes as C

import numpy as np
import pytest
import torch

import hunter_bipedal_control_b200 as hb
from episode_ref import (FRICTION, GAITS, N, PUSH, _resume, assert_episode_equal, cmd_vels, context, device, est_params, outputs, params,
                         random_goals, small_terrains, start_states)

pytestmark = pytest.mark.gpu

B = 6
N1, N2 = 37, 43          # the split: after the cycle of tick 35, before its adoption at 38 under a latency of 3


def _documented_bytes(n, grid):
    pad = lambda b: (b + 7) // 8 * 8
    sol = pad(8) + pad(8 * (n + 1) * 22) + pad(8 * n * 22) + (pad(8 * (n + 1)) if grid else 0) + pad(4 * (n + 1)) + (pad(4) if grid else 0)
    camera = 8 * (hb.HB_ODOM_MAX_DELAY + 1) * 3 + 8 * 3
    return hb.api.HB_EPISODE_HEADER_BYTES + sol + pad(8 * 38) + pad(8 * 12) + pad(4) + pad(C.sizeof(hb.HbTarget)) + sol + pad(camera)


def _headers(snap):
    return snap.rows[:, :32].cpu().numpy().copy().view(np.int64)


def configured(grid, wbc, rbd0):
    """A context with every per-robot setting of the episodes (the same data every time it is called) and every channel."""
    ctx = context(grid)
    ctx.set_wbc_formulation(wbc)
    ctx.set_pushes(hb.make_push_schedules(4, [[0.06], [0.07], [0.02], [0.09]], 0.03, PUSH))
    ctx.set_plant_variations(hb.make_plant_variations(B, friction_scale=FRICTION))
    ctx.set_terrains(small_terrains())
    ctx.set_goals(random_goals(rbd0, B, 5))
    ctx.set_mpc_latencies([3, 0, 5, 2])
    ctx.set_odometry(hb.make_odometry_settings(5, [4, 4, 3, 0, 5], [6, 0, 2, 0, 9], 0.002, 0.001))
    g = hb.default_pd_gains()
    ctx.set_controller_settings(hb.make_controller_settings(2, kp_big_stance=[g.kp_big_stance, 1.1 * g.kp_big_stance]))
    ctx.set_hardware(hb.make_hardware_settings(4, actuation_delay=[0.009, 0.004, 0.012, 0.0], sigma_joint_position=0.001))
    d = hb.default_planner_settings()
    ctx.set_planner_settings(hb.make_planner_settings(3, swing_height=[d.swing_height, 1.2 * d.swing_height, 0.8 * d.swing_height]))
    return ctx


@pytest.mark.parametrize("estimated", [False, True], ids=["truth", "estimator"])
@pytest.mark.parametrize("grid", [False, True], ids=["uniform", "event_nodes"])
@pytest.mark.parametrize("wbc", ["weighted", "hierarchical"])
def test_resume_in_a_fresh_context_is_bit_exact(wbc, grid, estimated):
    """n1 ticks, save, a new context with the same configuration and settings, restore, n2 ticks: the same as one call of n1 + n2 ticks,
    every output and every recorded channel. A state buffer missing from the row shows up here as a difference."""
    rbd0 = start_states(context(grid), B, 11)
    vels = cmd_vels(B)
    prm = params()
    ep = est_params(7) if estimated else None
    fresh = lambda: hb.estimation_states(B, 50) if estimated else None
    ctx = configured(grid, wbc, rbd0)
    ch = hb.make_channels(B, N1 + N2)
    ctx.set_channels(ch)
    one = device(ctx, rbd0, GAITS, vels, N1 + N2, prm, 1, ep, fresh())
    want = {k: v.clone() for k, v in ch.items()}
    first = device(ctx, rbd0, GAITS, vels, N1, prm, 1, ep, fresh())
    got = {k: v[:, :N1].clone() for k, v in ch.items()}
    snap = ctx.save_episodes(B, *first[:4], *(first[5:7] if estimated else ()))
    ctx.close()
    ctx2 = configured(grid, wbc, rbd0)
    ch2 = hb.make_channels(B, N2)
    ctx2.set_channels(ch2)
    r = ctx2.restore_episodes(snap)
    if estimated:
        second = device(ctx2, r[0], GAITS, vels, N2, prm, 1, ep, r[4], tick0=N1, act=r[1], estop=r[2], stats=r[3], est_stats=r[5])
    else:
        second = device(ctx2, r[0], GAITS, vels, N2, prm, 1, tick0=N1, act=r[1], estop=r[2], stats=r[3])
    two = outputs(second)
    two[4] = np.concatenate([first[4].cpu().numpy(), two[4]], axis=1)
    if estimated:
        two[7] = np.concatenate([first[7].cpu().numpy(), two[7]], axis=1)
    assert_episode_equal(one, two)
    for name in ch:
        joined = torch.cat([got[name], ch2[name]], dim=1)
        assert torch.equal(want[name], joined), name
    h = _headers(snap)
    assert (h[:, 0] == N).all() and (h[:, 1] == int(grid)).all() and (h[:, 2] == ctx2.episode_state_bytes).all()
    flags = hb.api.HB_EPISODE_HAS_SOLUTION | hb.api.HB_EPISODE_HAS_FALLBACK
    assert list(h[:, 3]) == [flags | (hb.api.HB_EPISODE_HAS_POLICY if i in (0, 2, 3) else 0) for i in range(B)]


@pytest.mark.parametrize("grid", [False, True], ids=["uniform", "event_nodes"])
def test_state_bytes_follow_the_documented_layout(grid):
    for n in (4, N, 41):
        ctx = hb.Context(horizon_N=n, dt=0.02, max_batch=2, device=0, time_horizon=0.6 if grid else 0.0, event_nodes=grid)
        assert ctx.episode_state_bytes == _documented_bytes(n, grid), n
        ctx.close()


def _run(ctx, rbd, gaits, vels, n, tick0=0, act=None, estop=None, stats=None, log_every=1):
    return device(ctx, rbd, gaits, vels, n, params(), log_every, tick0=tick0, act=act, estop=estop, stats=stats)


def test_fork_permutation_identity_and_launches():
    """src = [k] * B gives every instance instance k's own continuation; a permutation the permuted one; an identity save and restore
    changes nothing, with one launch each and the episode's launches unchanged."""
    ctx = context()
    rbd0 = start_states(ctx, B, 3)
    vels = cmd_vels(B)
    first = _run(ctx, rbd0, GAITS, vels, N1)
    c0 = ctx.launch_count
    snap = ctx.save_episodes(B, *first[:4])
    assert ctx.launch_count == c0 + 1
    cont_ref = _resume(ctx, first, GAITS, vels, N2, N1, params(), 1, None)
    c0 = ctx.launch_count
    r = ctx.restore_episodes(snap)
    assert ctx.launch_count == c0 + 1
    c0 = ctx.launch_count
    cont = _run(ctx, r[0], GAITS, vels, N2, N1, *r[1:])
    launches = ctx.launch_count - c0
    assert_episode_equal(cont_ref, cont)
    first_again = _run(ctx, rbd0, GAITS, vels, N1)        # the same prefix without a snapshot: the same launches afterwards
    c0 = ctx.launch_count
    _resume(ctx, first_again, GAITS, vels, N2, N1, params(), 1, None)
    assert ctx.launch_count - c0 == launches
    other = context()
    for src in ([4] * B, [1] * B, [5, 3, 0, 4, 1, 2]):
        r = other.restore_episodes(snap, src)
        out = _run(other, r[0], [GAITS[i] for i in src], vels[src], N2, N1, *r[1:])
        assert_episode_equal(out, cont_ref, rows_b=src)


def test_forked_copies_match_their_unforked_twin_until_their_push():
    ctx = context()
    rbd0 = start_states(ctx, B, 4)
    vels = cmd_vels(B)
    first = _run(ctx, rbd0, GAITS, vels, N1)
    snap = ctx.save_episodes(B, *first[:4])
    k = 2
    twin = outputs(_resume(ctx, first, GAITS, vels, N2, N1, params(), 1, None))
    at = [N1 + 3 + 5 * i for i in range(B)]                    # instance i pushed from tick at[i] on
    fork = context()
    fork.set_pushes(hb.make_push_schedules(B, np.array(at, dtype=float)[:, None] * params().period, 0.02, [[60.0, 40.0, 0.0]]))
    r = fork.restore_episodes(snap, [k] * B)
    out = outputs(_run(fork, r[0], [GAITS[k]] * B, vels[[k] * B], N2, N1, *r[1:]))
    for i in range(B):
        rows = at[i] - N1 + 1                                   # log rows of the states entering ticks N1 .. at[i]
        assert np.array_equal(out[4][i, :rows], twin[4][k, :rows]), i
        assert not np.array_equal(out[4][i, rows], twin[4][k, rows]), i


def test_forked_noise_streams():
    """Forked estimated copies share their source's noise stream and stay identical; reseeded, they differ, and copy j equals the source's
    own continuation with stream S + j from the fork tick on."""
    ctx = context()
    rbd0 = start_states(ctx, B, 6)
    vels = cmd_vels(B)
    ep = est_params(9)
    first = device(ctx, rbd0, GAITS, vels, N1, params(), 1, ep, hb.estimation_states(B, 50))
    snap = ctx.save_episodes(B, *first[:4], *first[5:7])
    k, S = 1, 1000
    fork = context()
    run = lambda r: outputs(device(fork, r[0], [GAITS[k]] * B, vels[[k] * B], N2, params(), 1, ep, r[4], tick0=N1, act=r[1], estop=r[2],
                                   stats=r[3], est_stats=r[5]))
    same = run(fork.restore_episodes(snap, [k] * B))
    for i in range(1, B):
        assert_episode_equal(same, same, rows_a=[0], rows_b=[i])
    r = list(fork.restore_episodes(snap, [k] * B))
    hb.reseed(r[4], S)
    apart = run(r)
    assert not np.array_equal(apart[0][0], apart[0][1])
    for j in (0, 3):
        r = ctx.restore_episodes(snap)
        hb.reseed(r[4].view(B, -1)[k].view(-1), S + j)          # the source's instance k on stream S + j from the fork tick on
        ref = device(ctx, r[0], GAITS, vels, N2, params(), 1, ep, r[4], tick0=N1, act=r[1], estop=r[2], stats=r[3], est_stats=r[5])
        assert_episode_equal(apart, ref, rows_a=[j], rows_b=[k])


def test_rejected_calls_change_nothing():
    lib = hb.load_library()
    ctx = context()
    rbd0 = start_states(ctx, B, 8)
    vels = cmd_vels(B)
    first = _run(ctx, rbd0, GAITS, vels, N1)
    snap = ctx.save_episodes(B, *first[:4])
    want = outputs(_resume(ctx, first, GAITS, vels, N2, N1, params(), 1, None))
    ctx.restore_episodes(snap)
    rows = snap.rows
    small = hb.Context(horizon_N=N - 10, dt=0.02, max_batch=8, device=0)
    grid = context(event_nodes=True)
    fresh = context()
    empty = fresh.save_episodes(2, *_run(fresh, rbd0[:2], GAITS[:2], vels[:2], 0)[:4])       # no solution yet
    assert not (_headers(empty)[:, 3] & hb.api.HB_EPISODE_HAS_SOLUTION).any()
    src = lambda *i: (C.c_int32 * len(i))(*i)
    c0 = ctx.launch_count
    p = C.c_void_p(rows.data_ptr())
    assert lib.hb_episode_restore(small._h, 1, None, 1, p) == -1                # horizon_N
    assert lib.hb_episode_restore(grid._h, 1, None, 1, p) == -1                 # time grid
    assert lib.hb_episode_restore(ctx._h, 1, src(B), B, p) == -1                # src beyond the rows
    assert lib.hb_episode_restore(ctx._h, 2, src(0, -1), B, p) == -1
    assert lib.hb_episode_restore(ctx._h, B + 1, None, B, p) == -1              # more instances than rows
    assert lib.hb_episode_restore(ctx._h, 2, None, 2, C.c_void_p(empty.rows.data_ptr())) == -1      # no solution
    assert lib.hb_episode_restore(ctx._h, 9, src(*[0] * 9), B, p) == -4         # beyond max_batch
    assert lib.hb_episode_restore(ctx._h, 1, None, 1, None) == -1               # NULL rows
    assert lib.hb_episode_restore(ctx._h, 0, None, 0, None) == 0
    out = torch.empty_like(rows)
    q = C.c_void_p(out.data_ptr())
    assert lib.hb_episode_save_async(ctx._h, 1, src(8), q) == -1                # src beyond max_batch
    assert lib.hb_episode_save_async(ctx._h, 1, src(-1), q) == -1
    assert lib.hb_episode_save_async(ctx._h, 9, None, q) == -4
    assert lib.hb_episode_save_async(ctx._h, 1, None, None) == -1
    assert lib.hb_episode_save_async(ctx._h, 0, None, None) == 0
    with pytest.raises(ValueError):
        small.restore_episodes(snap)                                            # rows of another size
    with pytest.raises(ValueError):
        ctx.restore_episodes(snap, [B])
    assert ctx.launch_count == c0
    assert_episode_equal(want, _run(ctx, snap.rbd.clone(), GAITS, vels, N2, N1, snap.act.clone(), snap.estop.clone(), snap.stats.copy()))
    # warm calls after an incomplete restore are rejected as in the context that saved the rows
    part = context()
    r = part.restore_episodes(snap, [0, 1])
    with pytest.raises(hb.HunterB200Error):
        _run(part, torch.cat([r[0], snap.rbd[2:]]), GAITS, vels, 5, N1)
    lat = context()
    lat.set_mpc_latencies([2])
    r = lat.restore_episodes(snap)                                              # rows without an adopted policy
    with pytest.raises(hb.HunterB200Error):
        _run(lat, *r[:1], GAITS, vels, 5, N1, *r[1:])


def test_fallback_flags_must_stay_a_prefix():
    """Rows with a solution but no previous WBC solution (a context whose solution was written, not solved) restore only where the
    instances that have one stay a prefix."""
    ctx = context()
    rbd0 = start_states(ctx, B, 9)
    vels = cmd_vels(B)
    snap = ctx.save_episodes(B, *_run(ctx, rbd0, GAITS, vels, 10)[:4])
    w = context()
    w.resident_write(np.zeros(2), np.zeros((2, N + 1, 22)), np.zeros((2, N, 22)))
    written = w.save_episodes(2, snap.rbd[:2], snap.act[:2 * C.sizeof(hb.HbActuationState)], snap.estop[:2], snap.stats[:2])
    assert list(_headers(written)[:, 3]) == [hb.api.HB_EPISODE_HAS_SOLUTION] * 2
    mixed = hb.EpisodeSnapshot(torch.cat([snap.rows[:1], written.rows[:1]]), snap.rbd[:2], snap.act[:2 * C.sizeof(hb.HbActuationState)],
                               snap.estop[:2], snap.stats[:2])
    t = context()
    _run(t, rbd0, GAITS, vels, 5)                                # every instance holds a previous WBC solution
    c0 = t.launch_count
    with pytest.raises(hb.HunterB200Error):
        t.restore_episodes(written)                               # instances 2 .. 5 would keep one that 0 and 1 lack
    with pytest.raises(hb.HunterB200Error):
        t.restore_episodes(mixed, [1, 0])                         # a gap
    assert t.launch_count == c0
    u = context()
    u.restore_episodes(mixed)                                     # instance 0 has one, instance 1 none: a prefix
    u.restore_episodes(snap)                                      # and all six again
    assert u.launch_count == 2


def test_restore_before_set_goals_forgets_the_capture():
    ctx = context()
    rbd0 = start_states(ctx, B, 12)
    vels = cmd_vels(B)
    goals = random_goals(rbd0, B, 5)
    ctx.set_goals(goals)
    first = _run(ctx, rbd0, GAITS, vels, N1)                     # goals captured on tick 30
    snap = ctx.save_episodes(B, *first[:4])
    kept = outputs(_resume(ctx, first, GAITS, vels, N2, N1, params(), 1, None))
    ctx.restore_episodes(snap)
    ctx.set_goals(goals)
    forgot = outputs(_run(ctx, snap.rbd.clone(), GAITS, vels, N2, N1, snap.act.clone(), snap.estop.clone(), snap.stats.copy()))
    other = context()
    other.set_goals(goals)
    r = other.restore_episodes(snap)
    other.set_goals(goals)
    assert_episode_equal(forgot, _run(other, r[0], GAITS, vels, N2, N1, *r[1:]))
    assert not np.array_equal(forgot[0], kept[0])
