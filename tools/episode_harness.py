"""The closed-loop episode harness of the tools that run batched episodes: bench_rollout.py, record_episodes.py, latency_sweep.py and the
sweeps push_sweep.py, plant_sweep.py, terrain_sweep.py, goal_sweep.py, odometry_sweep.py, gain_sweep.py, hardware_sweep.py,
gait_sweep.py, bridge_sweep.py and teleop_sweep.py. It holds their shared command line, the workload (bench.py's configs[1] start poses trotting at 0.3 m/s on ground at
GROUND, failure below MIN_HEIGHT), one timed episode call, the robot -> cell assignment of the sweeps and their per-cell tally, the timed
alternation of a per-robot setting, its null setting and no setting, the timing of a grid in one call against one call per cell, and the
fields and sentences the tools' JSON lines share."""
import argparse
import ctypes as C
import os
import subprocess
import sys
import time
from collections import namedtuple

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import DT, HORIZON_N, SEED, ClockSampler  # noqa: E402

GROUND, MIN_HEIGHT = 0.02, 0.3
# sensor noise at --sensor-noise 1 (standard deviations): orientation [rad], gyro [rad/s], accelerometer [m/s^2], encoders [rad], [rad/s]
NOISE_SIGMAS = dict(orientation=0.005, angular_velocity=0.02, linear_acceleration=0.1, joint_position=0.001, joint_velocity=0.02)
PUSH_T, PUSH_DURATION = 0.5, 0.1                # [s]: the push of push_sweep.py and gain_sweep.py --push

# one episode: device time [ms], launches, final hb_rollout_stats, final rbd (B x 32), hb_estimation_stats when asked for, and the logs of
# the true and (in an estimated episode) estimated states (B x rows x 32) when asked for
Run = namedtuple("Run", "ms launches stats rbd est_stats log est_log", defaults=(None, None))


def gpu_identity(index):
    """Card name and power limit, read in the run that measures."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True,
                             text=True, timeout=10).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1])}
    except Exception:
        return {"name": None, "power_limit_w": None}


def parser(batch_help="robots per episode"):
    """The arguments every tool takes; the tool adds its own."""
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024, help=batch_help)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--estimator", action="store_true", help="run the episodes through the state estimator")
    ap.add_argument("--sensor-noise", type=float, default=0.0, metavar="SCALE", help="with --estimator: sensor noise, SCALE x NOISE_SIGMAS")
    ap.add_argument("--wbc", choices=("weighted", "hierarchical"), default="weighted", help="the controller's whole-body controller")
    return ap


def noise_ok(args):
    """Whether --sensor-noise is a scale >= 0, given only with --estimator."""
    return not (args.sensor_noise < 0 or (args.sensor_noise and not args.estimator))


def sweep_args(tool, timed_help, ncell, extra=None, repeats=4, timed=3, valid=lambda args: True, needs=""):
    """The command line of a sweep over ncell cells, validated: --repeats, --timed, the common arguments and what extra(parser) adds,
    which valid(args) checks and `needs` names in the message."""
    ap = parser("robots per episode (a multiple of %d)" % ncell)
    ap.add_argument("--repeats", type=int, default=repeats, help="episodes per grid (the robot -> cell assignment shifts between them)")
    ap.add_argument("--timed", type=int, default=timed, help=timed_help)
    if extra:
        extra(ap)
    args = ap.parse_args()
    if args.batch < ncell or args.batch % ncell or args.repeats < 1 or not noise_ok(args) or not valid(args):
        raise SystemExit("%s: --batch a multiple of %d, --repeats >= 1, %s--sensor-noise takes a scale >= 0 and needs --estimator"
                         % (tool, ncell, needs))
    return args


def cells(B, ncols, nrows, shift):
    """(column, row) of every robot's cell in an nrows x ncols grid: robot i takes cell (i + shift) mod (ncols nrows), row-major."""
    c = (np.arange(B) + shift) % (ncols * nrows)
    return c % ncols, c // ncols


def cell_members(B, ncols, nrows, shift):
    """The robots of every cell of cells(B, ncols, nrows, shift), row-major."""
    col, row = cells(B, ncols, nrows, shift)
    return [np.nonzero(row * ncols + col == k)[0] for k in range(ncols * nrows)]


class Tally:
    """Per-cell counts of a sweep's episodes over an nrows x ncols grid, as arrays indexed [row, column]: robots (total), robots still up at
    the end (up), WBC fallbacks and a per-robot value summed over the robots up; and per fail reason, the robots that fell with it."""

    def __init__(self, ncols, nrows):
        from hunter_bipedal_control_b200 import ROLLOUT_FAIL
        self.total, self.up, self.fallbacks = (np.zeros((nrows, ncols), dtype=int) for _ in range(3))
        self.value = np.zeros((nrows, ncols))
        self.fail_bits = ROLLOUT_FAIL
        self.reasons = {name: 0 for name in ROLLOUT_FAIL}

    def add(self, col, row, stats, counts=None, value=None):
        """One episode: robot i in cell (col[i], row[i]) ended with hb_rollout_stats stats[i]. counts: a mask of the robots that count
        (default all); value: a per-robot value, summed over the robots that count and are up."""
        counts = np.ones(len(stats), dtype=bool) if counts is None else counts
        ok = stats["fail_tick"] < 0
        at = (row[counts], col[counts])
        np.add.at(self.total, at, 1)
        np.add.at(self.up, at, ok[counts].astype(int))
        np.add.at(self.fallbacks, at, stats["wbc_fallbacks"][counts])
        if value is not None:
            np.add.at(self.value, at, np.where(ok, value, 0.0)[counts])
        for name, bit in self.fail_bits.items():
            self.reasons[name] += int(((stats["fail_reason"] & bit) != 0)[counts & ~ok].sum())

    def survival(self):
        """The fraction of each cell's robots up at the end (0 for a cell without robots)."""
        return self.up / np.maximum(self.total, 1)

    def mean(self):
        """The value's mean over each cell's robots up (None for a cell without them), as nested lists [row][column]."""
        return [[float(v / u) if u else None for v, u in zip(vs, us)] for vs, us in zip(self.value, self.up)]

    def largest(self, col_values, threshold=0.9):
        """Per row, the largest of col_values up to which every cell of the row keeps a survival >= threshold (None when the first
        cell does not)."""
        leading = np.cumprod(self.up >= threshold * self.total, axis=1).sum(axis=1)     # the row's first cells that keep it
        return [col_values[n - 1] if n else None for n in leading]


def keyed(row_keys, col_keys, table):
    """A [row][column] table of nested lists as {row key: {column key: value}}."""
    return {r: dict(zip(col_keys, line)) for r, line in zip(row_keys, table)}


def sensor_noise(args):
    """The estimator's sensor noise and its seed, as the JSON lines report them."""
    return {"sensor_noise": {k: args.sensor_noise * v for k, v in NOISE_SIGMAS.items()}, "noise_seed": SEED}


def report(args, clocks, estimator=True):
    """The fields every tool's JSON line shares: n_gpus, dtype, data, wbc, the card's name and power limit and the clocks sampled while
    timing. estimator: also whether the episodes ran through the estimator and, when they did, sensor_noise(args)."""
    line = {"n_gpus": 1, "dtype": "f64", "data": "synthetic", "wbc": args.wbc, "gpu": gpu_identity(args.device), "clocks": clocks}
    if estimator:
        line["estimator"] = bool(args.estimator)
        if args.estimator:
            line.update(sensor_noise(args))
    return line


def workload(h, detail, motion="trot at 0.3 m/s from t = 0.1 s", seconds=None, digits=1, robots="robots"):
    """The config.workload sentence of h's episodes: the robots, the simulated time (default h.ticks ticks) to `digits` decimals, the
    motion, the start poses and the MPC's N and dt, then detail."""
    seconds = h.ticks * h.prm.period if seconds is None else seconds
    return ("%d %s, %.*f s simulated (%d ticks of %.0f ms), %s, initial poses of scenarios.random_initial_states(seed %d), N=%d dt=%.0f ms%s"
            % (h.B, robots, digits, seconds, h.ticks, 1e3 * h.prm.period, motion, SEED, HORIZON_N, 1e3 * DT, detail))


def failure_checks(height="base z"):
    """The config.failure_checks sentence: what ends a robot's episode."""
    return "non-finite state, |roll| > pi/2, %s < %.2f m, emergency stop" % (height, MIN_HEIGHT)


class Episodes:
    """The tools' workload on one context: B robots from the randomised poses of bench.py's configs[1] (N, dt of configs[1]), each lowered
    until its lowest contact frame is 1 mm inside the ground at GROUND, trotting at 0.3 m/s from t = 0.1 s, failure below a base height of
    MIN_HEIGHT; the estimator's sensor noise is args.sensor_noise x NOISE_SIGMAS, seeded with SEED."""

    def __init__(self, tool, args, ticks):
        import torch
        import hunter_bipedal_control_b200 as hb
        from hunter_bipedal_control_b200 import scenarios as S
        if not torch.cuda.is_available():
            raise SystemExit("%s: no CUDA device visible; the product path has no CPU fallback" % tool)
        self.torch, self.hb, self.args, self.ticks = torch, hb, args, ticks
        self.dev = torch.device("cuda", args.device)
        torch.cuda.set_device(self.dev)
        self.B = B = args.batch
        self.ctx = hb.Context(horizon_N=HORIZON_N, dt=DT, max_batch=B, device=args.device)
        self.ctx.set_wbc_formulation(args.wbc)
        x0 = S.random_initial_states(B, SEED)
        self.rbd0 = S.consistent_rbd(x0)
        self.feet = self.ctx.contact_positions(x0).reshape(B, 4, 3)
        self.rbd0[:, 5] -= self.feet[:, :, 2].min(axis=1) - (GROUND - 0.001)
        self.prm = hb.default_rollout_params()
        self.prm.sim.ground_height = GROUND
        self.prm.min_base_height = MIN_HEIGHT
        self.cmds = hb.make_rollout_commands("trot", np.full(B, 0.1), [0.0], [[0.3, 0.0, 0.0, 0.0]])
        self.ep = hb.default_estimation_params()
        self.ep.noise.seed = SEED
        for k, v in NOISE_SIGMAS.items():
            setattr(self.ep.noise, k, args.sensor_noise * v)
        self.stream = torch.cuda.ExternalStream(self.ctx.stream_handle, device=self.dev)
        self.lib = hb.load_library()

    def episode(self, estimated=None, est_stats=False, rows=None, log_every=0, est_log=False):
        """One episode of self.ticks ticks from the start poses in one hb_rollout_batch_dev call, or hb_rollout_estimated_batch_dev when
        estimated (default: --estimator), with device events around the call. est_stats: also collect the estimation stats. rows: the
        robots of a smaller batch (default: all), each with its start pose, command and noise stream, as instances 0 .. len(rows) - 1.
        log_every: also log the true state every log_every ticks (0: no log); est_log: in an estimated episode, the estimated state too."""
        torch, hb, dev, ctx = self.torch, self.hb, self.dev, self.ctx
        rows = np.arange(self.B) if rows is None else np.asarray(rows)
        B = len(rows)
        cmds = self.cmds if B == self.B and (rows == np.arange(B)).all() else (hb.HbRolloutCommand * B)(*[self.cmds[i] for i in rows])
        estimated = self.args.estimator if estimated is None else estimated
        P = lambda t: None if t is None else C.c_void_p(t.data_ptr())      # noqa: E731
        d_rbd = torch.from_numpy(np.ascontiguousarray(self.rbd0[rows])).to(dev)
        d_act = torch.zeros(B * C.sizeof(hb.HbActuationState), dtype=torch.uint8, device=dev)
        d_estop = torch.zeros(B, dtype=torch.uint8, device=dev)
        d_st = torch.from_numpy(hb.rollout_stats(B).view(np.uint8).copy()).to(dev)
        d_es = d_log = d_est_log = None
        if log_every:
            d_log = torch.zeros(B * ((self.ticks + log_every - 1) // log_every) * 32, dtype=torch.float64, device=dev)
        self.prm.log_every = log_every
        if estimated:
            est = hb.estimation_states(B)
            for k, i in enumerate(rows):
                est[k].noise_stream = int(i)
            d_est = torch.from_numpy(np.frombuffer(bytes(est), dtype=np.uint8).copy()).to(dev)
            if est_stats:
                d_es = torch.from_numpy(hb.estimation_stats(B).view(np.uint8).copy()).to(dev)
            if log_every and est_log:
                d_est_log = torch.zeros_like(d_log)
        torch.cuda.synchronize(dev)
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        l0 = ctx.launch_count
        e0.record(self.stream)
        if estimated:
            rc = self.lib.hb_rollout_estimated_batch_dev(ctx._h, B, C.c_int64(0), self.ticks, C.byref(self.prm), C.byref(self.ep), cmds, P(d_rbd),
                                                         P(d_act), P(d_estop), P(d_st), P(d_est), P(d_es), P(d_log), P(d_est_log))
        else:
            rc = self.lib.hb_rollout_batch_dev(ctx._h, B, C.c_int64(0), self.ticks, C.byref(self.prm), cmds, P(d_rbd), P(d_act), P(d_estop), P(d_st),
                                               P(d_log))
        e1.record(self.stream)
        assert rc == 0, rc
        ctx.sync()
        log = lambda t: None if t is None else t.cpu().numpy().reshape(B, -1, 32)      # noqa: E731
        return Run(e0.elapsed_time(e1), ctx.launch_count - l0, d_st.cpu().numpy().view(hb.ROLLOUT_STATS_DTYPE), d_rbd.cpu().numpy(),
                   None if d_es is None else d_es.cpu().numpy().view(hb.ESTIMATION_STATS_DTYPE), log(d_log), log(d_est_log))

    def sweep(self, set_, settings, **kw):
        """A sweep's episodes: set_(settings(0)) and one warm-up episode, then for each of the --repeats assignment shifts r, set_(settings(r))
        and one episode; yields (r, the episode). kw: episode()'s arguments."""
        set_(settings(0))
        self.episode(**kw)
        for r in range(self.args.repeats):
            set_(settings(r))
            yield r, self.episode(**kw)

    def alternate(self, set_, settings, timed, launches=False):
        """Times a setting against its null setting and no setting: `timed` rounds (at least one), each setting the three of `settings`
        ((name, value) pairs in that order, the last value None) in turn with set_ and running one episode. Returns the episodes per name,
        the clocks sampled meanwhile and the timing entries: per name the median and range of the episode time, the first two names'
        excess over the third, the number of rounds, whether the three launched equally often, and whether the null setting gave the
        outcome (final stats and states) of no setting in every round; with launches, also each name's launches as launches_<name>."""
        names = [n for n, _ in settings]
        runs = {n: [] for n in names}
        sampler = ClockSampler(self.args.device); sampler.start()
        for _ in range(max(1, timed)):
            for n, value in settings:
                set_(value)
                runs[n].append(self.episode())
        clocks = sampler.stop()
        ms = {n: [r.ms for r in runs[n]] for n in names}
        timing = {}
        for n in names:
            timing["ms_per_episode_" + n] = float(np.median(ms[n]))
            timing["ms_per_episode_%s_range" % n] = [min(ms[n]), max(ms[n])]
        unset = names[2]
        for n in names[:2]:
            timing["%s_minus_%s_ms" % (n, unset)] = float(np.median(ms[n]) - np.median(ms[unset]))
        timing["%s_same_outcome_as_%s" % (names[1], unset)] = all(np.array_equal(a.stats, b.stats) and np.array_equal(a.rbd, b.rbd)
                                                                 for a, b in zip(runs[names[1]], runs[unset]))
        timing["episodes"] = len(runs[unset])
        timing["launches_equal"] = len({runs[n][-1].launches for n in names}) == 1
        if launches:
            timing.update({"launches_" + n: int(runs[n][-1].launches) for n in names})
        return runs, clocks, timing

    def one_call_against_per_cell_calls(self, set_, records, set_cell, restore, members, est_stats=False):
        """Times a grid as one episode call on its per-robot records against the way it runs without the setting, alternated over --timed
        rounds (at least one): set_(records) and one call, then set_(None) and one call per cell on its members (robot indices), each after
        set_cell(k) puts cell k's values into the call, and restore() after the last. Returns the timing entries: per way the median and
        range of the device time (summed over the calls) and of the host time to the last synchronise, the rounds, the launches of each
        way, and whether every cell's final stats and states (and estimation stats, with est_stats) are bitwise equal between the two."""
        times = {"one_call_ms": [], "one_call_wall_ms": [], "per_cell_calls_ms": [], "per_cell_calls_wall_ms": []}
        equal, rounds = True, max(1, self.args.timed)
        for _ in range(rounds):
            set_(records)
            t0 = time.perf_counter()
            one = self.episode(est_stats=est_stats)
            w1 = time.perf_counter() - t0
            set_(None)
            many, t0 = [], time.perf_counter()
            for k, m in enumerate(members):
                set_cell(k)
                many.append(self.episode(est_stats=est_stats, rows=m))
            wall = time.perf_counter() - t0
            restore()
            times["one_call_ms"].append(one.ms); times["one_call_wall_ms"].append(1e3 * w1)
            times["per_cell_calls_ms"].append(sum(r.ms for r in many)); times["per_cell_calls_wall_ms"].append(1e3 * wall)
            for m, r in zip(members, many):
                equal &= bool(np.array_equal(one.stats[m], r.stats) and np.array_equal(one.rbd[m], r.rbd)
                              and (not est_stats or np.array_equal(one.est_stats[m], r.est_stats)))
        timing = {k: float(np.median(v)) for k, v in times.items()}
        timing.update({k + "_range": [min(v), max(v)] for k, v in times.items()})
        timing.update(rounds=rounds, launches_one_call=int(one.launches), launches_per_cell_calls=int(sum(r.launches for r in many)),
                      cells_bitwise_equal=equal)
        return timing
