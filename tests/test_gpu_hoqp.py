"""SURVEY 8f row N4: HoQP / HierarchicalWbc on the device against the CPU restatement (oracle/hoqp.py, itself checked against the reference's own
unit test legged_wbc/test/HoQp_test.cpp in tests/test_oracle_hoqp.py)."""
import ctypes

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb
from oracle.hoqp import HoQp, Task

pytestmark = pytest.mark.gpu


def eigen_random(libc, rows, cols):
    m = np.zeros((rows, cols))
    for c in range(cols):
        for r in range(rows):
            m[r, c] = -1.0 + 2.0 * libc.rand() / 2147483647.0
    return m


def _oracle_chain(levels):
    h = None
    out = []
    for (a, b, d, f) in levels:
        n = a.shape[1] if a is not None and a.size else d.shape[1]
        h = HoQp(Task(a if a is not None and a.size else None, b if a is not None and a.size else None, d if d is not None and d.size else None,
                      f if d is not None and d.size else None, n=n), h)
        out.append(h)
    return out


def _random_hierarchies():
    libc = ctypes.CDLL("libc.so.6")
    libc.srand(0)
    a0 = eigen_random(libc, 2, 4); d0 = eigen_random(libc, 2, 4)                      # HoQp_test.cpp:19-33 (TEST(HoQP, twoTask))
    hier = [[(a0, np.ones(2), d0, np.ones(2)), (np.ones((2, 4)), np.ones(2), d0, np.ones(2))]]
    rng = np.random.default_rng(3)
    for n in (6, 8, 12):
        for _ in range(4):
            t0 = (rng.normal(size=(3, n)), rng.normal(size=3), rng.normal(size=(2, n)), rng.normal(size=2) + 1.0)
            t1 = (rng.normal(size=(2, n)), rng.normal(size=2), rng.normal(size=(3, n)), rng.normal(size=3))
            t2 = (rng.normal(size=(4, n)), rng.normal(size=4), None, None)
            hier.append([t0, t1, t2])
    return hier


def _full_stack_hierarchies():
    """Three levels with inequality rows at every level, 30 + 30 + 20 of them: the stack reaches its 80-row capacity at level 2."""
    rng = np.random.default_rng(11)
    hier = []
    for n, ma in ((10, (4, 3, 4)), (10, (4, 3, 4)), (14, (3, 2, 4)), (14, (3, 2, 4))):
        hier.append([(rng.normal(size=(m, n)), rng.normal(size=m), rng.normal(size=(md, n)), rng.normal(size=md) + 1.0)
                     for m, md in zip(ma, (30, 30, 20))])
    return hier


def _check_hierarchies(hier, x, sl, st):
    """Device cascades against the oracle's; returns how many hierarchies leave no freedom (x itself unique)."""
    assert (st == 0).all(), st
    n_unique = 0
    for i, levels in enumerate(hier):
        chain = _oracle_chain(levels)
        n = chain[-1].x.size
        xo = chain[-1].solution()
        # what every level achieves (A_l x and the violated part of D_l x - f_l) is unique; x itself only when no freedom is left over
        # (otherwise the regulariser picks a point that depends on the null-space basis: FullPivLU kernel / SVD / Gauss-Jordan)
        for (a, b, d, f) in levels:
            assert np.abs(a @ x[i, :n] - a @ xo).max() < 1e-5 * max(1.0, np.abs(a @ xo).max()), i
            if d is not None:
                assert np.abs(np.maximum(d @ x[i, :n] - f, 0) - np.maximum(d @ xo - f, 0)).max() < 1e-5, i      # interior-point tolerance on an active row
        rank_left = chain[-1].stacked_z.shape[1]
        if rank_left == 0:
            n_unique += 1
            assert np.abs(x[i, :n] - xo).max() < 1e-5 * max(1.0, np.abs(xo).max()), i
        # strict priorities on the device solution itself
        a_top, b_top, d_top, f_top = levels[0]
        assert np.abs(a_top @ x[i, :n] - a_top @ chain[0].solution()).max() < 1e-6
        assert np.all(d_top @ x[i, :n] <= f_top + chain[0].slack + 1e-6)
        # each level's slack solution, stacked in level order
        off = 0
        for level, (a, b, d, f) in zip(chain, levels):
            md = 0 if d is None else d.shape[0]
            assert np.abs(sl[i, off:off + md] - level.slack).max(initial=0.0) < 1e-5, i
            off += md
        assert (sl[i, :off] > -1e-8).all() and np.abs(sl[i, off:]).max(initial=0.0) == 0.0
    return n_unique


def test_reference_unit_test_matrices_and_random_hierarchies(gpu_ctx):
    hier = _random_hierarchies()
    x, sl, st = gpu_ctx.hoqp_solve(hb.make_hoqp_problems(hier))
    assert _check_hierarchies(hier, x, sl, st) >= 4


def test_inequalities_at_every_level_fill_the_stack(gpu_ctx):
    hier = _full_stack_hierarchies()
    pbs = hb.make_hoqp_problems(hier)
    assert all(sum(p.md) == 80 for p in pbs)
    x, sl, st = gpu_ctx.hoqp_solve(pbs)
    assert _check_hierarchies(hier, x, sl, st) == 2


def test_device_call_without_slack_buffer(gpu_ctx):
    """hb_hoqp_solve_batch_dev with slack = NULL gives the bits of the call with a slack buffer."""
    import torch
    hier = _random_hierarchies() + _full_stack_hierarchies()
    pbs = hb.make_hoqp_problems(hier)
    B, lib = len(hier), gpu_ctx._lib
    d_pbs = torch.from_numpy(np.frombuffer(bytes(pbs), dtype=np.uint8).copy()).cuda()
    P = lambda t: ctypes.c_void_p(t.data_ptr())      # noqa: E731

    def run(with_slack):
        x = torch.full((B, hb.api.HB_HOQP_N), np.nan, dtype=torch.float64, device="cuda")
        st = torch.full((B,), -1, dtype=torch.int32, device="cuda")
        sl = torch.full((B, hb.api.HB_HOQP_MAX_STACKED), np.nan, dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        assert lib.hb_hoqp_solve_batch_dev(gpu_ctx._h, B, P(d_pbs), P(x), P(sl) if with_slack else None, P(st)) == 0
        gpu_ctx.sync()
        return x.cpu().numpy(), st.cpu().numpy(), sl.cpu().numpy()

    x1, st1, sl1 = run(True)
    x0, st0, _ = run(False)
    assert (st1 == 0).all() and np.isfinite(sl1).all()
    assert np.array_equal(x0.view(np.uint64), x1.view(np.uint64)) and np.array_equal(st0, st1)


def _wbc_cases(B, seed):
    from hunter_bipedal_control_b200 import scenarios as sc
    rng = np.random.default_rng(seed)
    mode = np.array([3, 2, 1, 3, 2, 1, 0, 3][:B], dtype=np.int32)
    x = np.tile(sc.INITIAL_STATE, (B, 1)) + rng.uniform(-.04, .04, (B, 22))
    u = np.zeros((B, 22))
    for i in range(B):
        fl = sc.mode_flags(int(mode[i]))
        for c in range(4):
            if fl[c]:
                u[i, 3 * c + 2] = sc.TOTAL_MASS * 9.81 / sum(fl)
        u[i, 12:] = rng.uniform(-.3, .3, 10)
    rbd = sc.consistent_rbd(x, rng, 0.01)
    return x, u, rbd, mode


def test_hierarchical_wbc_tasks_and_solution_vs_oracle(gpu_ctx, oracle):
    from oracle.hoqp import hierarchical_wbc
    B = 8
    x, u, rbd, mode = _wbc_cases(B, 4)
    pbs = gpu_ctx.hierarchical_wbc_tasks(x, u, rbd, mode)
    sol, st = gpu_ctx.hierarchical_wbc_solve(x, u, rbd, mode)
    assert (st == 0).all(), st
    for i in range(B):
        so, levels, tasks = hierarchical_wbc(x[i], u[i], rbd[i], int(mode[i]))
        dev = hb.hoqp_tasks(pbs[i])
        # same tasks: compare as sets of rows (the order of the rows inside a task is free)
        for (a, b, d, f), t in zip(dev, tasks):
            for M_dev, v_dev, M_o, v_o in ((a, b, t.a, t.b), (d, f, t.d, t.f)):
                assert M_dev.shape == M_o.shape, (i, M_dev.shape, M_o.shape)
                if M_o.size == 0:
                    continue
                rows_dev = np.hstack([M_dev, v_dev[:, None]]); rows_o = np.hstack([M_o, v_o[:, None]])
                for r in rows_o:
                    assert np.abs(rows_dev - r[None]).max(axis=1).min() < 1e-8 * max(1.0, np.abs(r).max()), i
        t0, t1, t2 = tasks
        s = sol[i]
        # level 0 (EoM, zero swing forces, no contact motion): the same least-squares optimum as the restatement. With a moving foot the
        # toe and heel "zero acceleration" rows are mutually inconsistent (centripetal term), so the residual is small but not zero.
        assert np.abs(t0.a @ s - t0.a @ levels[0].solution()).max() < 1e-5 * max(1.0, np.abs(t0.b).max())
        assert np.abs(t0.a[:16] @ s - t0.b[:16]).max() < 1e-4                              # the EoM rows themselves hold
        assert np.all(t0.d @ s <= t0.f + 1e-4)                                             # torque limits, friction pyramid
        assert np.abs(t1.a @ s - t1.a @ levels[1].solution()).max() < 1e-5                  # base task as good as the physics allows
        assert np.abs(t2.a @ s - t2.a @ so).max() < 1e-4 * max(1.0, np.abs(t2.a @ so).max())
        assert np.abs(s[28:] - so[28:]).max() < 1e-4 * max(1.0, np.abs(so[28:]).max())     # torques (north_star tolerance)


def test_hierarchical_wbc_mirror_class(gpu_ctx, oracle):
    x, u, rbd, mode = _wbc_cases(1, 9)
    w = hb.HierarchicalWbc(gpu_ctx)
    s = w.update(x[0], u[0], rbd[0], int(mode[0]), 0.002)
    assert s.shape == (38,) and np.isfinite(s).all() and np.abs(s[28:]).max() <= 60 + 1e-6
