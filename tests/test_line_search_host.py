"""The MPC line search's cases and the oracle's per-trial record, without a GPU: every case of linesearch_ref sits in the branch its name
gives with the margin the GPU test needs, the record agrees with the iteration's info, the oracle's trial cap stops the search like
hb_config.line_search_max_trials, and hb_create refuses a cap below one trial."""
import numpy as np
import pytest

import linesearch_ref as L

CAPS = (1, 2, 13, 14, 20)


@pytest.fixture(scope="module")
def cases(oracle):
    return {g: L.make_cases(oracle, g) for g in L.GRIDS}


@pytest.mark.parametrize("grid", tuple(L.GRIDS))
def test_cases_sit_in_their_named_branches_with_margin(grid, cases, oracle):
    """make_cases asserts each case's trials on the record; here the grid's cases also cover every branch accepting, every trial count
    and the rejected step."""
    got = {}
    for name, N, dt, *c, expected in cases[grid]:
        info, trials = L._record(oracle, N, dt, c)
        assert L.pattern(trials) == expected, name
        assert L.check_margins(trials, info) >= 1.0, name
        got[name] = trials
    accepted = {t[-1]["branch"] for t in got.values() if t[-1]["accepted"]}
    assert accepted == {"violation", "armijo", "filter"}
    counts = sorted(len(t) for t in got.values() if t[-1]["accepted"])
    assert set(range(1, L.MAX_TRIALS + 1)) <= set(counts)
    assert any(len(t) == L.MAX_TRIALS and not t[-1]["accepted"] for t in got.values())
    # mixed: trials rejected in one branch before another accepts; filter accepts on the merit alone and on the violation alone
    assert any(len({b for b, _ in L.pattern(t)}) > 1 and t[-1]["accepted"] for t in got.values())
    assert "filter/alpha1/merit-only" in got and "filter/alpha1/violation-only" in got
    if grid in L.DROP:
        assert L.pattern(got["armijo/backtracked/unloaded-heels"]) == [("armijo", False), ("armijo", True)]
        assert L.pattern(got["armijo/alpha1/between-factors"]) == [("armijo", True)]


@pytest.mark.parametrize("grid", tuple(L.GRIDS))
def test_trial_record_agrees_with_the_iteration_info(grid, cases, oracle):
    for name, N, dt, *c, expected in cases[grid]:
        x0, xr, sw, md, xt, ut = c
        xa, ua, info = oracle.mpc_iteration(N, dt, *c)
        xb, ub, info_r, trials = oracle.mpc_iteration(N, dt, *c, record=True)
        assert info == info_r and np.array_equal(xa, xb) and np.array_equal(ua, ub), name
        assert info["status"] == 0 and info["n_trials"] == len(trials), name
        last = trials[-1]
        assert [t["alpha"] for t in trials] == [0.5 ** j for j in range(len(trials))], name
        if last["accepted"]:
            assert (info["alpha"], info["merit1"], info["viol1"]) == (last["alpha"], last["merit"], last["viol"]), name
        else:
            assert (info["alpha"], info["merit1"], info["viol1"]) == (0.0, info["merit0"], info["viol0"]), name
            assert np.array_equal(xa[1:], xt[1:]) and np.array_equal(xa[0], x0) and np.array_equal(ua, ut), name
        for t in trials:      # the branch each trial took follows from armijo in the info as the kernel computes it
            assert L.decide(t, info) == (t["branch"], t["accepted"]), name


@pytest.mark.parametrize("grid", tuple(L.GRIDS))
def test_trial_cap_stops_the_search(grid, cases, oracle):
    """With a cap of k the oracle returns the uncapped answer when it needs k trials or fewer, and otherwise rejects after k trials."""
    for name, N, dt, *c, expected in cases[grid]:
        x0, xr, sw, md, xt, ut = c
        full = oracle.mpc_iteration(N, dt, *c)
        for k in CAPS:
            x, u, info, trials = oracle.mpc_iteration(N, dt, *c, max_trials=k, record=True)
            if full[2]["n_trials"] <= k:
                assert info == full[2] and np.array_equal(x, full[0]) and np.array_equal(u, full[1]), (name, k)
            else:
                assert info["n_trials"] == k and info["alpha"] == 0.0 and len(trials) == k, (name, k)
                assert L.pattern(trials) == expected[:k], (name, k)
                assert (info["merit1"], info["viol1"]) == (info["merit0"], info["viol0"]), (name, k)
                assert np.array_equal(x[1:], xt[1:]) and np.array_equal(x[0], x0) and np.array_equal(u, ut), (name, k)


def test_trial_cap_below_one_is_rejected_before_any_cuda_call():
    """hb_create checks line_search_max_trials >= 1 with the other settings, before it touches the device: a context whose line search
    runs no trial would report every solve as status 0 with alpha 0."""
    import hunter_bipedal_control_b200 as hb
    for k in (0, -1):
        with pytest.raises(hb.HunterB200Error, match=r"invalid argument \(-1\)"):
            hb.Context(horizon_N=8, max_batch=1, line_search_max_trials=k)
