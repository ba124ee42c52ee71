"""The episode tools without a GPU: every tool's command line, the harness's per-cell tally on hand-counted episodes, the JSON line's common
fields and sentences, and that no tool imports another tool."""
import ast
import glob
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest

import hunter_bipedal_control_b200 as hb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")
sys.path.insert(0, TOOLS)
import episode_harness as eh  # noqa: E402

EPISODE_TOOLS = ["bench_rollout", "record_episodes", "latency_sweep", "push_sweep", "plant_sweep", "terrain_sweep", "goal_sweep", "odometry_sweep",
                 "gain_sweep", "hardware_sweep", "gait_sweep"]


@pytest.mark.parametrize("tool", EPISODE_TOOLS)
def test_tool_parses_help(tool):
    out = subprocess.run([sys.executable, os.path.join(TOOLS, tool + ".py"), "--help"], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    assert out.stdout.startswith("usage: %s.py" % tool) and "--batch" in out.stdout and "--wbc" in out.stdout


def test_no_tool_imports_another_tool():
    tools = {os.path.basename(p)[:-3] for p in glob.glob(os.path.join(TOOLS, "*.py"))}
    for path in glob.glob(os.path.join(TOOLS, "*.py")):
        names = set()
        for node in ast.walk(ast.parse(open(path).read())):
            if isinstance(node, ast.Import):
                names |= {a.name.split(".")[0] for a in node.names}
            elif isinstance(node, ast.ImportFrom) and node.module:
                names.add(node.module.split(".")[0])
        assert names & tools <= {"episode_harness"}, (path, names & tools)


def stats(fail_tick, fail_reason, fallbacks):
    st = hb.rollout_stats(len(fail_tick))
    st["fail_tick"], st["fail_reason"], st["wbc_fallbacks"] = fail_tick, fail_reason, fallbacks
    return st


# eight robots on a 3 x 2 grid: robots 1 (height and orientation) and 3 (estop) fall, the others stay up
COL, ROW = np.array([0, 1, 2, 0, 1, 2, 0, 1]), np.array([0, 0, 0, 1, 1, 1, 0, 0])
F = hb.ROLLOUT_FAIL
ST = stats([-1, 300, -1, 20, -1, -1, -1, -1], [0, F["height"] | F["orientation"], 0, F["estop"], 0, 0, 0, 0], [2, 1, 0, 0, 0, 0, 0, 3])
VALUE = np.array([1.0, np.nan, 3.0, 9.0, 5.0, 7.0, 2.0, 4.0])


def test_tally_counts_cells_reasons_and_survivors_value():
    t = eh.Tally(3, 2)
    t.add(COL, ROW, ST, value=VALUE)
    assert t.total.tolist() == [[2, 2, 1], [1, 1, 1]] and t.up.tolist() == [[2, 1, 1], [0, 1, 1]]
    assert t.survival().tolist() == [[1.0, 0.5, 1.0], [0.0, 1.0, 1.0]]
    assert t.fallbacks.tolist() == [[2, 4, 0], [0, 0, 0]]
    assert t.mean() == [[1.5, 4.0, 3.0], [None, 5.0, 7.0]]
    assert t.reasons == {"estop": 1, "orientation": 1, "height": 1, "nonfinite": 0}
    assert t.largest(["a", "b", "c"]) == ["a", None]
    assert t.largest(["a", "b", "c"], threshold=0.5) == ["c", None]
    t.add(COL, ROW, ST, value=VALUE)                  # a second episode adds to every count
    assert t.total.tolist() == [[4, 4, 2], [2, 2, 2]] and t.survival().tolist() == [[1.0, 0.5, 1.0], [0.0, 1.0, 1.0]]
    assert t.mean() == [[1.5, 4.0, 3.0], [None, 5.0, 7.0]]
    assert t.reasons == {"estop": 2, "orientation": 2, "height": 2, "nonfinite": 0}


def test_tally_counts_only_the_masked_robots():
    t = eh.Tally(3, 2)
    t.add(COL, ROW, ST, counts=np.array([True, True, True, False, True, True, True, False]), value=VALUE)
    assert t.total.tolist() == [[2, 1, 1], [0, 1, 1]] and t.up.tolist() == [[2, 0, 1], [0, 1, 1]]
    assert t.survival().tolist() == [[1.0, 0.0, 1.0], [0.0, 1.0, 1.0]]
    assert t.fallbacks.tolist() == [[2, 1, 0], [0, 0, 0]]
    assert t.mean() == [[1.5, None, 3.0], [None, 5.0, 7.0]]
    assert t.reasons == {"estop": 0, "orientation": 1, "height": 1, "nonfinite": 0}
    assert t.largest([10, 20, 30]) == [10, 30]         # a cell without robots does not end the walk
    assert eh.keyed(["r0", "r1"], ["c0", "c1", "c2"], t.mean()) == {"r0": {"c0": 1.5, "c1": None, "c2": 3.0},
                                                                  "r1": {"c0": None, "c1": 5.0, "c2": 7.0}}


def test_report_fields_with_and_without_the_estimator():
    clocks = {"sm_mhz": [1980]}
    plain = eh.report(eh.parser().parse_args([]), clocks)
    assert set(plain) == {"n_gpus", "dtype", "data", "estimator", "wbc", "gpu", "clocks"}
    assert (plain["n_gpus"], plain["dtype"], plain["data"], plain["estimator"], plain["wbc"], plain["clocks"]) == (1, "f64", "synthetic", False,
                                                                                                                 "weighted", clocks)
    assert set(plain["gpu"]) == {"name", "power_limit_w"}
    args = eh.parser().parse_args(["--estimator", "--sensor-noise", "2", "--wbc", "hierarchical"])
    est = eh.report(args, clocks)
    assert set(est) == set(plain) | {"sensor_noise", "noise_seed"} and est["estimator"] is True and est["wbc"] == "hierarchical"
    assert est["sensor_noise"] == {k: 2 * v for k, v in eh.NOISE_SIGMAS.items()} and est["noise_seed"] == eh.SEED
    assert set(eh.report(args, clocks, estimator=False)) == {"n_gpus", "dtype", "data", "wbc", "gpu", "clocks"}


def test_workload_and_failure_sentences():
    h = SimpleNamespace(B=1024, ticks=750, prm=SimpleNamespace(period=0.002))
    assert eh.workload(h, "; 16 payload masses x 4 friction scales, 4 episodes") == (
        "1024 robots, 1.5 s simulated (750 ticks of 2 ms), trot at 0.3 m/s from t = 0.1 s, initial poses of "
        "scenarios.random_initial_states(seed 20240901), N=100 dt=10 ms; 16 payload masses x 4 friction scales, 4 episodes")
    h.ticks = 3250
    assert eh.workload(h, ", through the estimator", "trot with cmd_vel 0 from t = 0.1 s", 6.5, 2, "robots through the estimator") == (
        "1024 robots through the estimator, 6.50 s simulated (3250 ticks of 2 ms), trot with cmd_vel 0 from t = 0.1 s, initial poses of "
        "scenarios.random_initial_states(seed 20240901), N=100 dt=10 ms, through the estimator")
    assert eh.failure_checks() == "non-finite state, |roll| > pi/2, base z < 0.30 m, emergency stop"
    assert eh.failure_checks("base z above the terrain") == "non-finite state, |roll| > pi/2, base z above the terrain < 0.30 m, emergency stop"


def test_sweep_args_validates_the_common_arguments(monkeypatch):
    def parse(*argv, **kw):
        monkeypatch.setattr(sys, "argv", ["goal_sweep.py", *argv])
        return eh.sweep_args("goal_sweep.py", "timed", 32, **kw)

    assert parse("--batch", "64").repeats == 4
    for argv in (["--batch", "48"], ["--batch", "16"], ["--repeats", "0"], ["--sensor-noise", "1"], ["--estimator", "--sensor-noise", "-1"]):
        with pytest.raises(SystemExit, match="goal_sweep.py: --batch a multiple of 32, --repeats >= 1, --sensor-noise"):
            parse(*argv)
    with pytest.raises(SystemExit, match="--repeats >= 1, --settle >= 0, --sensor-noise"):
        parse("--batch", "64", valid=lambda a: False, needs="--settle >= 0, ")
