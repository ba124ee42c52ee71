#!/usr/bin/env python3
"""Terrain sweep of the closed-loop episodes (hb_rollout_set_terrains + hb_rollout_batch_dev): prints one JSON line.

  python tools/terrain_sweep.py [--repeats R] [--timed K] [--batch B] [--estimator [--sensor-noise SCALE]]

The workload of tools/bench_rollout.py (B robots, default 1024, trotting at 0.3 m/s from the randomised poses of bench.py's configs[1],
N = 100, dt = 10 ms, ground at 0.02 m, failure below a base height of 0.3 m, measured above the terrain), run for 1.5 s (750 ticks). Every
robot walks blind over a terrain of its own, which the planner, controllers and estimator are not told about: a 64 x 64 height field at
2.5 cm spacing centred on its start, with the ground at 0.02 m under the start pose and, across the robot's initial heading,
  - a step up or a step down of 0 to 15 cm (1 cm steps) whose edge lies 0.15 m ahead of the base origin, or
  - an incline or a decline of 0 to 15 degrees (1 degree steps) that starts 0.10 m ahead of it.
The height field is interpolated bilinearly between its samples, so a step is a ramp one cell (2.5 cm) wide; the plant has point
contacts only, so no foot meets the step's face. A robot whose foremost contact point starts less than 1.5 cells (3.75 cm, more than the
cell's diagonal) behind the edge or the ramp's start has them moved ahead to that distance, so that the ground under every start pose is
0.02 m exactly and the start states are those of bench_rollout (the randomised poses put the foremost contact point up to about 0.12 m
ahead of the base origin); the line reports how many robots that moves.

The 64 (kind, magnitude) cells share the batch, 1/64 of the robots each; episode r of R shifts the assignment by r, so every cell sees
R x B / 64 different start poses. Per cell: survival (the fraction of its robots still up at the end) and the mean horizontal base speed of
the survivors (their base displacement in the ground plane over the episode time). Per kind: the largest magnitude up to which every cell
keeps >= 90 % survival.

The line also times, in the same invocation, the terrain batch against the same batch on flat terrains at 0.02 m and with no terrain set,
alternately, with device events around the episode call, and reports the launch counts of the three (terrains add no launch), whether
flat and unset give the same outcome, and the card's name and power limit and the clocks sampled during the timed episodes.

--estimator runs everything through hb_rollout_estimated_batch_dev (controllers on the Kalman filter's estimate from simulated sensors,
noise = SCALE x episode_harness's NOISE_SIGMAS).

--height-maps tells the planner where the ground is (hb_plan_set_maps): each robot's height map is its terrain minus the flat ground of
0.02 m, so the planner plans on the terrain the plant stands on. The line then reports the blind and the mapped survival tables over the
same cells and start poses, each with its largest magnitude at >= 90 % per kind, and times mapped episodes against the same terrain
episodes with all-zero maps and blind (no map), alternately, with the launch counts of the three and whether zero maps gave the blind
outcome.

--estimator-maps (with --height-maps --estimator) also tells the Kalman filter where the ground is (hb_estimator_set_maps), with the same
maps, so that it measures each foot's height on the terrain instead of at z = 0. Planner maps and estimator maps are separate settings:
the line reports four tables over the same cells and start poses -- blind, planner maps only, estimator maps only, both -- and times
episodes with both maps against planner maps with all-zero estimator maps and planner maps only, alternately; the tool asserts that
all-zero estimator maps give the outcome of planner maps only bit for bit.

--mpc-maps (with --height-maps) also holds the MPC's stance feet on the ground (hb_mpc_set_maps), with the same maps: the stance-foot
constraint pulls each stance contact to 0.02 m above the map instead of z = 0.02. The line reports the tables above plus one with MPC maps
added to every map the run gives (planner + MPC maps; with --estimator-maps all three), and times episodes with MPC maps against the same
episodes with all-zero MPC maps and without MPC maps, alternately; the tool asserts that all-zero MPC maps give the outcome of no MPC maps
bit for bit.

--wbc-maps (with --height-maps) also tilts the WBC's friction pyramids on the ground (hb_wbc_set_maps), with the same maps: each stance
contact's pyramid is about the map's normal at the contact's measured position instead of the world z axis. The line reports the tables
above plus one, with_wbc_maps, with WBC maps added to every map the run gives, and times episodes with WBC maps against the same episodes
with all-zero WBC maps and without WBC maps, alternately; the tool asserts that all-zero WBC maps give the outcome of no WBC maps bit for
bit.

--mpc-cone-maps (with --height-maps) also stands the MPC's friction cones on the ground (hb_mpc_set_cone_maps), with the same maps: each
stance contact's cone bounds its force in the map's surface frame at its swing reference instead of about the world z axis. The line
reports the tables above plus one, with_cone_maps, with MPC cone maps added to every map the run gives, and times episodes with cone maps
against the same episodes with all-zero cone maps and without cone maps, alternately; the tool asserts that all-zero cone maps give the
outcome of no cone maps bit for bit.

--contact-detection (with --estimator) hands each robot's Kalman filter the contact flags of the momentum observer
(hb_rollout_set_contact_detection, default_contact_detection: task.info's threshold, fractions 0.75 and 0.25) instead of the schedule's.
The line reports four tables over the same cells and start poses -- blind, blind with detection, estimator maps (each robot's terrain
minus 0.02 m, hb_estimator_set_maps) and estimator maps with detection -- each with its largest magnitude at >= 90 % per kind and, per
kind and magnitude, the mean over the cell's robots of the estimation stats' largest base-height error and RMS base-velocity error. It
times episodes with detection against the same episodes with the setting made and cleared and without it, alternately; the tool asserts
that the cleared setting gives the outcome of none bit for bit.

--friction-scale S scales every robot's ground friction by S in every table (hb_rollout_set_plant_variations, friction_scale) and runs its
WBC with friction_coefficient S times the context's (task.info's) value (hb_rollout_set_controller_settings): the slope's direction
matters most to the friction pyramids where friction is short.
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from episode_harness import GROUND, Episodes, Tally, cells, failure_checks, keyed, report, sweep_args, workload  # noqa: E402

TICKS = 750
KINDS = ["step_up", "step_down", "incline", "decline"]
MAGNITUDES = list(range(16))                             # [cm] for steps, [deg] for slopes
GRID, SPACING = 64, 0.025
STEP_AHEAD, RAMP_AHEAD = 0.15, 0.10                      # [m] ahead of the base origin along the initial heading


def feature_distances(rbd0, feet):
    """Per robot, how far ahead of the base origin along the initial heading the step's edge and the ramp's start lie: STEP_AHEAD and
    RAMP_AHEAD, or 1.5 cells ahead of the foremost start contact point (feet, B x 4 x 3) when that is further."""
    front = ((feet[:, :, 0] - rbd0[:, 3, None]) * np.cos(rbd0[:, 0, None]) + (feet[:, :, 1] - rbd0[:, 4, None]) * np.sin(rbd0[:, 0, None])).max(axis=1)
    return np.maximum(STEP_AHEAD, front + 1.5 * SPACING), np.maximum(RAMP_AHEAD, front + 1.5 * SPACING)


def terrain_heights(rbd0, kind, magnitude, step_ahead, ramp_ahead):
    """(origin (B, 2), heights (B, GRID, GRID)) of one kind and magnitude per robot, centred on each start pose, with the step's edge and
    the ramp's start step_ahead / ramp_ahead (B,) ahead of the base origin."""
    origin = rbd0[:, 3:5] - 0.5 * (GRID - 1) * SPACING
    k = SPACING * np.arange(GRID)
    X = origin[:, 0, None, None] + k[None, None, :]
    Y = origin[:, 1, None, None] + k[None, :, None]
    d = (X - rbd0[:, 3, None, None]) * np.cos(rbd0[:, 0])[:, None, None] + (Y - rbd0[:, 4, None, None]) * np.sin(rbd0[:, 0])[:, None, None]
    m = np.asarray(magnitude, dtype=float)[:, None, None]
    kind = np.asarray(kind)[:, None, None]
    step = np.where(d >= step_ahead[:, None, None], 0.01 * m, 0.0)
    ramp = np.maximum(d - ramp_ahead[:, None, None], 0.0) * np.tan(np.radians(m))
    h = np.select([kind == "step_up", kind == "step_down", kind == "incline"], [step, -step, ramp], -ramp)
    return origin, GROUND + h


def height_map_sweep(h, args, grid):
    """--height-maps: the blind and the mapped sweep over the same cells, then mapped / zero-map / blind terrain episodes timed alternately;
    with --estimator-maps the four tables (blind, planner maps, estimator maps, both), then both / zero estimator maps / planner maps only.
    grid(shift) gives the (origin, heights) of the terrains of assignment shift."""
    hb, ctx, prm, B, rbd0 = h.hb, h.ctx, h.prm, h.B, h.rbd0
    T_episode = TICKS * prm.period

    def set_all(value):
        terrains, maps, est_maps, mpc_maps, wbc_maps, cone_maps = value
        ctx.set_terrains(terrains)
        ctx.set_height_maps(maps)
        ctx.set_estimator_maps(est_maps)
        ctx.set_mpc_maps(mpc_maps)
        ctx.set_wbc_maps(wbc_maps)
        ctx.set_mpc_cone_maps(cone_maps)

    def settings(shift, planner, estimator, mpc=False, wbc=False, cone=False):
        origin, heights = grid(shift)
        maps = hb.make_terrains(B, heights - GROUND, SPACING, origin)
        return (hb.make_terrains(B, heights, SPACING, origin), maps if planner else None, maps if estimator else None, maps if mpc else None,
                maps if wbc else None, maps if cone else None)

    tables = [("blind", False, False), ("mapped", True, False)]
    if args.estimator_maps:
        tables = [("blind", False, False), ("planner_maps", True, False), ("estimator_maps", False, True), ("both_maps", True, True)]
    tables = [t + (False, False, False) for t in tables]
    if args.mpc_maps:
        tables.append(("all_maps", True, True, True, False, False) if args.estimator_maps else ("planner_mpc_maps", True, False, True, False, False))
    if args.wbc_maps:
        tables.append(("with_wbc_maps", True, args.estimator_maps, args.mpc_maps, True, False))
    if args.mpc_cone_maps:
        tables.append(("with_cone_maps", True, args.estimator_maps, args.mpc_maps, args.wbc_maps, True))
    out, mk = {}, [str(m) for m in MAGNITUDES]
    for name, planner, estimator, mpc, wbc, cone in tables:
        tally = Tally(len(MAGNITUDES), len(KINDS))
        for r, run in h.sweep(set_all, lambda shift: settings(shift, planner, estimator, mpc, wbc, cone)):
            tally.add(*cells(B, len(MAGNITUDES), len(KINDS), r), run.stats, value=np.hypot(*(run.rbd[:, 3:5] - rbd0[:, 3:5]).T) / T_episode)
        out[name] = {"largest_magnitude_90pct": dict(zip(KINDS, tally.largest(MAGNITUDES))), "survival": keyed(KINDS, mk, tally.survival().tolist()),
                     "mean_speed_of_survivors_m_per_s": keyed(KINDS, mk, tally.mean()), "fail_reasons": tally.reasons}
    terrains, maps, _, _, _, _ = settings(0, True, True)
    origin, heights = grid(0)
    zero = hb.make_terrains(B, np.zeros_like(heights), SPACING, origin)
    est = maps if args.estimator_maps else None
    if args.mpc_cone_maps:
        mpc, wbc = (maps if args.mpc_maps else None), (maps if args.wbc_maps else None)
        _, clocks, timing = h.alternate(set_all, [("cone_maps", (terrains, maps, est, mpc, wbc, maps)),
                                                  ("zero_cone_maps", (terrains, maps, est, mpc, wbc, zero)),
                                                  ("no_cone_maps", (terrains, maps, est, mpc, wbc, None))], args.timed, launches=True)
        assert timing["zero_cone_maps_same_outcome_as_no_cone_maps"], "all-zero MPC cone maps changed the outcome of no cone maps"
    elif args.wbc_maps:
        mpc = maps if args.mpc_maps else None
        _, clocks, timing = h.alternate(set_all, [("wbc_maps", (terrains, maps, est, mpc, maps, None)), ("zero_wbc_maps", (terrains, maps, est, mpc, zero, None)),
                                                  ("no_wbc_maps", (terrains, maps, est, mpc, None, None))], args.timed, launches=True)
        assert timing["zero_wbc_maps_same_outcome_as_no_wbc_maps"], "all-zero WBC maps changed the outcome of no WBC maps"
    elif args.mpc_maps:
        _, clocks, timing = h.alternate(set_all, [("mpc_maps", (terrains, maps, est, maps, None, None)), ("zero_mpc_maps", (terrains, maps, est, zero, None, None)),
                                                  ("no_mpc_maps", (terrains, maps, est, None, None, None))], args.timed, launches=True)
        assert timing["zero_mpc_maps_same_outcome_as_no_mpc_maps"], "all-zero MPC maps changed the outcome of no MPC maps"
    elif args.estimator_maps:
        _, clocks, timing = h.alternate(set_all, [("both_maps", (terrains, maps, maps, None, None, None)),
                                                  ("zero_estimator_maps", (terrains, maps, zero, None, None, None)),
                                                  ("planner_maps", (terrains, maps, None, None, None, None))], args.timed, launches=True)
        assert timing["zero_estimator_maps_same_outcome_as_planner_maps"], "all-zero estimator maps changed the outcome of planner maps only"
    else:
        _, clocks, timing = h.alternate(set_all, [("mapped", (terrains, maps, None, None, None, None)), ("zero_maps", (terrains, zero, None, None, None, None)),
                                                  ("blind", (terrains, None, None, None, None, None))], args.timed, launches=True)
    set_all((None, None, None, None, None, None))
    return out, clocks, timing


def contact_detection_sweep(h, args, grid):
    """--contact-detection: blind, blind with detection, estimator maps and estimator maps with detection over the same cells, each with its
    estimation errors; then detection / cleared / unset episodes timed alternately."""
    hb, ctx, prm, B, rbd0 = h.hb, h.ctx, h.prm, h.B, h.rbd0
    records = hb.make_contact_detection_settings(B)
    mk = [str(m) for m in MAGNITUDES]

    def set_all(value):
        terrains, est_maps, detection = value
        ctx.set_terrains(terrains)
        ctx.set_estimator_maps(est_maps)
        if detection == "cleared":
            ctx.set_contact_detection(records)
            detection = None
        ctx.set_contact_detection(detection)

    def settings(shift, maps, detection):
        origin, heights = grid(shift)
        return hb.make_terrains(B, heights, SPACING, origin), hb.make_terrains(B, heights - GROUND, SPACING, origin) if maps else None, \
            records if detection else None

    out = {}
    for name, maps, detection in [("blind", False, False), ("blind_detection", False, True), ("estimator_maps", True, False),
                                  ("estimator_maps_detection", True, True)]:
        tally = Tally(len(MAGNITUDES), len(KINDS))
        height, vel = np.zeros((len(KINDS), len(MAGNITUDES))), np.zeros((len(KINDS), len(MAGNITUDES)))
        for r, run in h.sweep(set_all, lambda shift: settings(shift, maps, detection), est_stats=True):
            mi, ki = cells(B, len(MAGNITUDES), len(KINDS), r)
            tally.add(mi, ki, run.stats, value=np.hypot(*(run.rbd[:, 3:5] - rbd0[:, 3:5]).T) / (TICKS * prm.period))
            es = run.est_stats
            rms = np.sqrt(es["sum_sq_vel_err"] / np.maximum(es["count"], 1))
            np.add.at(height, (ki, mi), es["max_height_err"] / (args.repeats * B / (len(KINDS) * len(MAGNITUDES))))
            np.add.at(vel, (ki, mi), rms / (args.repeats * B / (len(KINDS) * len(MAGNITUDES))))
        out[name] = {"largest_magnitude_90pct": dict(zip(KINDS, tally.largest(MAGNITUDES))), "survival": keyed(KINDS, mk, tally.survival().tolist()),
                     "mean_max_height_err_m": keyed(KINDS, mk, height.tolist()), "mean_rms_vel_err_m_per_s": keyed(KINDS, mk, vel.tolist()),
                     "fail_reasons": tally.reasons}
    terrains, _, _ = settings(0, False, True)
    _, clocks, timing = h.alternate(set_all, [("detection", (terrains, None, records)), ("cleared", (terrains, None, "cleared")),
                                              ("no_detection", (terrains, None, None))], args.timed, launches=True)
    assert timing["cleared_same_outcome_as_no_detection"], "a cleared contact detection changed the outcome of none"
    set_all((None, None, None))
    return out, clocks, timing


def main():
    def extra(ap):
        ap.add_argument("--height-maps", action="store_true", help="also plan on maps of the terrains")
        ap.add_argument("--estimator-maps", action="store_true", help="with --height-maps --estimator: also give the Kalman filter the maps")
        ap.add_argument("--mpc-maps", action="store_true", help="with --height-maps: also hold the MPC's stance feet on the maps")
        ap.add_argument("--wbc-maps", action="store_true", help="with --height-maps: also tilt the WBC's friction pyramids on the maps")
        ap.add_argument("--mpc-cone-maps", action="store_true", help="with --height-maps: also stand the MPC's friction cones on the maps")
        ap.add_argument("--friction-scale", type=float, default=1.0, help="scale of every robot's ground friction and WBC friction coefficient")
        ap.add_argument("--contact-detection", action="store_true", help="with --estimator: also run the filter on detected contact flags")

    args = sweep_args("terrain_sweep.py", "timed terrain / flat / unset episode triples (with --height-maps: mapped / zero-map / blind)",
                      len(KINDS) * len(MAGNITUDES), extra=extra,
                      valid=lambda a: ((not a.estimator_maps or (a.height_maps and a.estimator)) and (not a.mpc_maps or a.height_maps)
                                       and (not a.wbc_maps or a.height_maps) and (not a.mpc_cone_maps or a.height_maps) and a.friction_scale > 0
                                       and (not a.contact_detection or (a.estimator and not a.height_maps))),
                      needs="--estimator-maps needs --height-maps --estimator, --mpc-maps needs --height-maps, "
                            "--wbc-maps needs --height-maps, --mpc-cone-maps needs --height-maps, --friction-scale takes a scale > 0, "
                            "--contact-detection needs --estimator and no --height-maps, ")
    h = Episodes("terrain_sweep.py", args, TICKS)
    hb, ctx, prm, B, rbd0 = h.hb, h.ctx, h.prm, h.B, h.rbd0
    step_ahead, ramp_ahead = feature_distances(rbd0, h.feet)
    T_episode = TICKS * prm.period
    if args.friction_scale != 1.0:         # short friction on both sides of the loop: the plant's ground and the WBC's pyramids
        ctx.set_plant_variations(hb.make_plant_variations(B, friction_scale=args.friction_scale))
        ctx.set_controller_settings(hb.make_controller_settings(B, wbc=ctx.wbc_settings(),
                                                                friction_coefficient=args.friction_scale * ctx.wbc_settings().friction_coefficient))

    def grid(shift):
        mi, ki = cells(B, len(MAGNITUDES), len(KINDS), shift)
        return terrain_heights(rbd0, np.array(KINDS)[ki], np.array(MAGNITUDES)[mi], step_ahead, ramp_ahead)

    if args.contact_detection:
        out, clocks, timing = contact_detection_sweep(h, args, grid)
        print(json.dumps({
            "metric": "contact detection: the highest step [cm] that >= 90 %% of the trotting robots cross within %.1f s through the estimator "
                      "when the Kalman filter's contact flags come from the momentum observer; %s tables per kind (steps in cm, slopes in "
                      "degrees)" % (T_episode, ", ".join(out)), "value": out["blind_detection"]["largest_magnitude_90pct"]["step_up"], "unit": "cm",
            **report(args, clocks), **out, "timing": timing,
            "config": {"workload": workload(h, "; %d kinds x %d magnitudes, %d episodes per table" % (len(KINDS), len(MAGNITUDES), args.repeats)),
                       "terrain": "%d x %d height field at %g m centred on the start, ground %g m under the start; steps with the edge %g m "
                                  "ahead (a ramp one cell wide), slopes starting %g m ahead, across the initial heading"
                                  % (GRID, GRID, SPACING, GROUND, STEP_AHEAD, RAMP_AHEAD),
                       "contact_detection": "default_contact_detection() for every robot: threshold 75 N, fractions 0.75 / 0.25, cutoff 250",
                       "estimator_maps": "each robot's terrain minus %g m (hb_estimator_set_maps)" % GROUND,
                       "survival": "robots still up at the end of the episode", "failure_checks": failure_checks("base z above the terrain")}}))
        return

    if args.height_maps:
        out, clocks, timing = height_map_sweep(h, args, grid)
        if args.mpc_cone_maps:
            metric = ("MPC cone maps: the highest step [cm] that >= 90 %% of the trotting robots cross within %.1f s%s when the planner%s%s%s "
                      "and the MPC's friction cones are told the terrain; %s tables per kind (steps in cm, slopes in degrees)"
                      % (T_episode, " through the estimator" if args.estimator else "", ", the Kalman filter" if args.estimator_maps else "",
                         ", the MPC's stance feet" if args.mpc_maps else "", ", the WBC" if args.wbc_maps else "", ", ".join(out)))
            value = out["with_cone_maps"]["largest_magnitude_90pct"]["step_up"]
        elif args.wbc_maps:
            metric = ("WBC maps: the highest step [cm] that >= 90 %% of the trotting robots cross within %.1f s%s when the planner%s%s and "
                      "the WBC are told the terrain; %s tables per kind (steps in cm, slopes in degrees)"
                      % (T_episode, " through the estimator" if args.estimator else "", ", the Kalman filter" if args.estimator_maps else "",
                         ", the MPC" if args.mpc_maps else "", ", ".join(out)))
            value = out["with_wbc_maps"]["largest_magnitude_90pct"]["step_up"]
        elif args.mpc_maps:
            last = "all_maps" if args.estimator_maps else "planner_mpc_maps"
            metric = ("MPC maps: the highest step [cm] that >= 90 %% of the trotting robots cross within %.1f s%s when the planner%s and the "
                      "MPC are told the terrain; %s tables per kind (steps in cm, slopes in degrees)"
                      % (T_episode, " through the estimator" if args.estimator else "", ", the Kalman filter" if args.estimator_maps else "",
                         ", ".join(out)))
            value = out[last]["largest_magnitude_90pct"]["step_up"]
        elif args.estimator_maps:
            metric = ("estimator maps: the highest step [cm] that >= 90 %% of the trotting robots cross within %.1f s through the estimator "
                      "when the planner and the Kalman filter are told the terrain; blind, planner-map, estimator-map and both-map tables per "
                      "kind (steps in cm, slopes in degrees)" % T_episode)
            value = out["both_maps"]["largest_magnitude_90pct"]["step_up"]
        else:
            metric = ("height maps: the highest step [cm] that >= 90 %% of the trotting robots cross within %.1f s when the planner is told "
                      "the terrain; blind and mapped tables per kind (steps in cm, slopes in degrees)" % T_episode)
            value = out["mapped"]["largest_magnitude_90pct"]["step_up"]
        print(json.dumps({
            "metric": metric, "value": value, "unit": "cm", **report(args, clocks), **out, "timing": timing,
            "config": {"workload": workload(h, "; %d kinds x %d magnitudes, %d episodes per table" % (len(KINDS), len(MAGNITUDES), args.repeats)),
                       "terrain": "%d x %d height field at %g m centred on the start, ground %g m under the start; steps with the edge %g m "
                                  "ahead (a ramp one cell wide), slopes starting %g m ahead, across the initial heading"
                                  % (GRID, GRID, SPACING, GROUND, STEP_AHEAD, RAMP_AHEAD),
                       "height_maps": "each robot's terrain minus %g m (hb_plan_set_maps%s%s); blind: no map"
                                      % (GROUND, ", and the same maps with hb_estimator_set_maps" if args.estimator_maps else "",
                                         ", and the same maps with hb_mpc_set_maps in the last table" if args.mpc_maps else "")
                                      + (", and the same maps with hb_wbc_set_maps in with_wbc_maps" if args.wbc_maps else "")
                                      + (", and the same maps with hb_mpc_set_cone_maps in with_cone_maps" if args.mpc_cone_maps else ""),
                       "friction_scale": args.friction_scale,
                       "survival": "robots still up at the end of the episode", "failure_checks": failure_checks("base z above the terrain")}}))
        return

    def terrains(shift):
        mi, ki = cells(B, len(MAGNITUDES), len(KINDS), shift)
        origin, h = terrain_heights(rbd0, np.array(KINDS)[ki], np.array(MAGNITUDES)[mi], step_ahead, ramp_ahead)
        return hb.make_terrains(B, h, SPACING, origin)

    tally = Tally(len(MAGNITUDES), len(KINDS))
    for r, run in h.sweep(ctx.set_terrains, terrains):
        tally.add(*cells(B, len(MAGNITUDES), len(KINDS), r), run.stats, value=np.hypot(*(run.rbd[:, 3:5] - rbd0[:, 3:5]).T) / T_episode)
    mk = [str(m) for m in MAGNITUDES]
    largest = dict(zip(KINDS, tally.largest(MAGNITUDES)))   # per kind: the largest magnitude up to which every cell keeps >= 90 % survival

    # terrain, flat-terrain and unset episodes alternate
    flat_origin, flat_h = terrain_heights(rbd0, np.full(B, "step_up"), np.zeros(B), step_ahead, ramp_ahead)
    flat = hb.make_terrains(B, flat_h, SPACING, flat_origin)
    runs, clocks, timing = h.alternate(ctx.set_terrains, [("terrain", terrains(0)), ("flat", flat), ("unset", None)], args.timed, launches=True)
    print(json.dumps({
        "metric": "terrain: the highest step [cm] that >= 90 %% of the trotting robots cross blind within %.1f s; per kind (steps in cm, "
                  "slopes in degrees) under largest_magnitude_90pct" % T_episode, "value": largest["step_up"], "unit": "cm",
        **report(args, clocks), "largest_magnitude_90pct": largest, "survival": keyed(KINDS, mk, tally.survival().tolist()),
        "mean_speed_of_survivors_m_per_s": keyed(KINDS, mk, tally.mean()), "fail_reasons": tally.reasons,
        "upright_fraction_unset": float((runs["unset"][-1].stats["fail_tick"] < 0).mean()), "timing": timing,
        "config": {"workload": workload(h, "; %d kinds x %d magnitudes, %d episodes" % (len(KINDS), len(MAGNITUDES), args.repeats)),
                   "terrain": "%d x %d height field at %g m centred on the start, ground %g m under the start; steps with the edge %g m "
                              "ahead (a ramp one cell wide), slopes starting %g m ahead, across the initial heading"
                              % (GRID, GRID, SPACING, GROUND, STEP_AHEAD, RAMP_AHEAD),
                   "robots_with_features_moved_ahead": {"step": int((step_ahead > STEP_AHEAD).sum()), "ramp": int((ramp_ahead > RAMP_AHEAD).sum()),
                                                        "max_step_ahead_m": float(step_ahead.max()), "max_ramp_ahead_m": float(ramp_ahead.max())},
                   "survival": "robots still up at the end of the episode",
                   "failure_checks": failure_checks("base z above the terrain")}}))


if __name__ == "__main__":
    main()
