"""Episode snapshots without a GPU: the entry points are exported and reject a null context, EpisodeSnapshot checks that its buffers hold
the same instances, the index checks of Context.save_episodes / restore_episodes, the .npz round trip and reseed. The row size of each
configuration needs a context, so test_gpu_episode_snapshots.py checks it against the documented layout."""
import ctypes as C

import numpy as np
import pytest
import torch

import hunter_bipedal_control_b200 as hb
from hunter_bipedal_control_b200 import api

ACT, EST = C.sizeof(hb.HbActuationState), C.sizeof(hb.HbEstimationState)


def _snapshot(n, estimated, row_bytes=96, seed=0):
    g = torch.Generator().manual_seed(seed)
    byte = lambda *s: torch.randint(0, 256, s, dtype=torch.uint8, generator=g)
    stats = hb.rollout_stats(n)
    stats["fail_tick"] = np.arange(n) - 1; stats["max_abs_torque"] = np.linspace(0.0, 3.0, n)
    est = est_stats = None
    if estimated:
        est = byte(n * EST)
        est_stats = hb.estimation_stats(n); est_stats["count"] = np.arange(n) + 7; est_stats["sum_sq_vel_err"] = 0.5
    return hb.EpisodeSnapshot(byte(n, row_bytes), torch.rand((n, 32), dtype=torch.float64, generator=g), byte(n * ACT), byte(n), stats, est, est_stats)


def test_entry_points_are_exported_and_reject_a_null_context():
    lib = hb.load_library()
    for name in ("hb_episode_state_bytes", "hb_episode_save_async", "hb_episode_restore"):
        assert name in hb.EXPORTED_SYMBOLS and hasattr(lib, name)
    rows = (C.c_uint8 * 64)()
    assert lib.hb_episode_state_bytes(None) == -1
    assert lib.hb_episode_save_async(None, 1, None, rows) == -1
    assert lib.hb_episode_restore(None, 1, None, 1, rows) == -1


@pytest.mark.parametrize("estimated", [False, True])
def test_snapshot_checks_its_buffers_hold_the_same_instances(estimated):
    s = _snapshot(3, estimated)
    assert len(s) == 3 and s.estimated == estimated
    parts = dict(rows=s.rows, rbd=s.rbd, act=s.act, estop=s.estop, stats=s.stats, est=s.est, est_stats=s.est_stats)
    short = dict(rows=s.rows[:2], rbd=s.rbd[:2], act=s.act[:2 * ACT], estop=s.estop[:2], stats=s.stats[:2])
    if estimated:
        short.update(est=s.est[:2 * EST], est_stats=s.est_stats[:2])
    for name, value in short.items():
        with pytest.raises(ValueError):
            hb.EpisodeSnapshot(**dict(parts, **{name: value}))
    with pytest.raises(ValueError):             # est and est_stats go together
        hb.EpisodeSnapshot(**dict(parts, est=None if estimated else torch.zeros(3 * EST, dtype=torch.uint8)))


def test_episode_index_checks():
    assert api._episode_index(None, 3, 3, "f") == [0, 1, 2]
    assert api._episode_index(np.array([2, 2, 0, 1]), 4, 3, "f") == [2, 2, 0, 1]
    for src, B, n in (([3], 1, 3), ([-1], 1, 3), ([0, 1], 3, 3), (None, 4, 3)):
        with pytest.raises(ValueError):
            api._episode_index(src, B, n, "f")


@pytest.mark.parametrize("estimated", [False, True])
def test_npz_round_trip_is_exact(tmp_path, estimated):
    s = _snapshot(5, estimated, seed=3)
    s.save(tmp_path / "snap.npz")
    t = hb.EpisodeSnapshot.load(tmp_path / "snap.npz", device="cpu")
    assert t.estimated == estimated
    for k in hb.EpisodeSnapshot._TENSORS:
        a, b = getattr(s, k), getattr(t, k)
        assert (a is None) == (b is None), k
        if a is not None:
            assert a.dtype == b.dtype and torch.equal(a, b), k
    assert t.stats.dtype == hb.ROLLOUT_STATS_DTYPE and np.array_equal(t.stats, s.stats)
    if estimated:
        assert t.est_stats.dtype == hb.ESTIMATION_STATS_DTYPE and np.array_equal(t.est_stats, s.est_stats)


def test_reseed_sets_each_noise_stream_and_nothing_else():
    est = torch.from_numpy(np.frombuffer(bytes(hb.estimation_states(4, first_stream=9)), dtype=np.uint8).copy())
    before = est.clone()
    assert hb.reseed(est, 2**40 + 5) is est
    rec = (hb.HbEstimationState * 4).from_buffer_copy(est.numpy().tobytes())
    assert [r.noise_stream for r in rec] == [2**40 + 5 + i for i in range(4)]
    off = hb.HbEstimationState.noise_stream.offset
    keep = np.ones(EST, dtype=bool); keep[off:off + 8] = False
    assert torch.equal(est.view(4, EST)[:, keep], before.view(4, EST)[:, keep])
