"""The closed-loop episode harness of tools/bench_rollout.py, push_sweep.py, plant_sweep.py and terrain_sweep.py: their shared command line,
the workload (bench.py's configs[1] start poses trotting at 0.3 m/s on ground at GROUND, failure below MIN_HEIGHT), one timed episode call,
the robot -> cell assignment of the sweeps, and the timed alternation of a per-robot setting, its null setting and no setting."""
import argparse
import ctypes as C
import os
import subprocess
import sys
from collections import namedtuple

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import DT, HORIZON_N, SEED, ClockSampler  # noqa: E402

GROUND, MIN_HEIGHT = 0.02, 0.3
# sensor noise at --sensor-noise 1 (standard deviations): orientation [rad], gyro [rad/s], accelerometer [m/s^2], encoders [rad], [rad/s]
NOISE_SIGMAS = dict(orientation=0.005, angular_velocity=0.02, linear_acceleration=0.1, joint_position=0.001, joint_velocity=0.02)

# one episode: device time [ms], launches, final hb_rollout_stats, final rbd (B x 32), hb_estimation_stats when asked for, and the log of
# the true states (B x rows x 32) when asked for
Run = namedtuple("Run", "ms launches stats rbd est_stats log", defaults=(None,))


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


def sweep_args(tool, timed_help, ncell, extra=None):
    """The command line of a sweep over ncell cells, validated: --repeats, --timed, the common arguments and what extra(parser) adds."""
    ap = parser("robots per episode (a multiple of %d)" % ncell)
    ap.add_argument("--repeats", type=int, default=4, help="episodes per grid (the robot -> cell assignment shifts between them)")
    ap.add_argument("--timed", type=int, default=3, help=timed_help)
    if extra:
        extra(ap)
    args = ap.parse_args()
    if args.batch < ncell or args.batch % ncell or args.repeats < 1 or args.sensor_noise < 0 or (args.sensor_noise and not args.estimator):
        raise SystemExit("%s: --batch a multiple of %d, --repeats >= 1, --sensor-noise takes a scale >= 0 and needs --estimator" % (tool, ncell))
    return args


def cells(B, ncols, nrows, shift):
    """(column, row) of every robot's cell in an nrows x ncols grid: robot i takes cell (i + shift) mod (ncols nrows), row-major."""
    c = (np.arange(B) + shift) % (ncols * nrows)
    return c % ncols, c // ncols


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

    def episode(self, estimated=None, est_stats=False, rows=None, log_every=0):
        """One episode of self.ticks ticks from the start poses in one hb_rollout_batch_dev call, or hb_rollout_estimated_batch_dev when
        estimated (default: --estimator), with device events around the call. est_stats: also collect the estimation stats. rows: the
        robots of a smaller batch (default: all), each with its start pose, command and noise stream, as instances 0 .. len(rows) - 1.
        log_every: also log the true state every log_every ticks (0: no log)."""
        torch, hb, dev, ctx = self.torch, self.hb, self.dev, self.ctx
        rows = np.arange(self.B) if rows is None else np.asarray(rows)
        B = len(rows)
        cmds = self.cmds if B == self.B and (rows == np.arange(B)).all() else (hb.HbRolloutCommand * B)(*[self.cmds[i] for i in rows])
        estimated = self.args.estimator if estimated is None else estimated
        P = lambda t: C.c_void_p(t.data_ptr())
        d_rbd = torch.from_numpy(np.ascontiguousarray(self.rbd0[rows])).to(dev)
        d_act = torch.zeros(B * C.sizeof(hb.HbActuationState), dtype=torch.uint8, device=dev)
        d_estop = torch.zeros(B, dtype=torch.uint8, device=dev)
        d_st = torch.from_numpy(hb.rollout_stats(B).view(np.uint8).copy()).to(dev)
        d_es = d_log = None
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
        torch.cuda.synchronize(dev)
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        l0 = ctx.launch_count
        e0.record(self.stream)
        if estimated:
            rc = self.lib.hb_rollout_estimated_batch_dev(ctx._h, B, C.c_int64(0), self.ticks, C.byref(self.prm), C.byref(self.ep), cmds, P(d_rbd),
                                                         P(d_act), P(d_estop), P(d_st), P(d_est), None if d_es is None else P(d_es),
                                                         None if d_log is None else P(d_log), None)
        else:
            rc = self.lib.hb_rollout_batch_dev(ctx._h, B, C.c_int64(0), self.ticks, C.byref(self.prm), cmds, P(d_rbd), P(d_act), P(d_estop), P(d_st),
                                               None if d_log is None else P(d_log))
        e1.record(self.stream)
        assert rc == 0, rc
        ctx.sync()
        return Run(e0.elapsed_time(e1), ctx.launch_count - l0, d_st.cpu().numpy().view(hb.ROLLOUT_STATS_DTYPE), d_rbd.cpu().numpy(),
                   None if d_es is None else d_es.cpu().numpy().view(hb.ESTIMATION_STATS_DTYPE),
                   None if d_log is None else d_log.cpu().numpy().reshape(B, -1, 32))

    def alternate(self, set_, settings, timed):
        """Times a setting against its null setting and no setting: `timed` rounds (at least one), each setting the three of `settings`
        ((name, value) pairs in that order, the last value None) in turn with set_ and running one episode. Returns the episodes per name,
        the clocks sampled meanwhile and the timing entries: per name the median and range of the episode time, the first two names'
        excess over the third, the number of rounds, whether the three launched equally often, and whether the null setting gave the
        outcome (final stats and states) of no setting in every round."""
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
        return runs, clocks, timing
