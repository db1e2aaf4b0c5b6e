"""Closed-loop batched simulation on one GPU: the controller of qm_controllers (QMController) driving the plant step of this library, at the
reference's rates, entirely on device buffers of one CUDA stream (INTEGRATION.md §3).

Per simulated millisecond (Gazebo's default physics step, 1 kHz):
  every 10 ms (mpcDesiredFrequency 100, task.info)  target_trajectories_dev (cmd_vel) → mpc_solve_dev          (the MPC node + target publisher)
  every WBC period (default 2 ms)                     update_dev: observation → evaluatePolicy → WBC → control law (QMController::update)
  every 1 ms                                          hw_write_dev (QMHWSim::writeSim, 9 ms command delay of qm_gazebo/config/default.yaml)
                                                      → sim_step_dev (physics step + QMHWSim::readSim's contact flags)
Per-robot experiments (robustness sweeps): cmd_vel and gait may differ per robot, and the plant may vary per robot through the handle's robot
params (floor friction, end-effector and base payloads: Solver.sim_set_robot_params), heightfield terrain under the feet
(Solver.sim_set_terrain / sim_set_robot_terrain) and external pushes held over whole plant steps.  The
controller is not told about any of them unless the run sets its model payload (Solver.set_model_payload), e.g. to the plant's payload.
With payload_estimator set, an online estimate of each robot's end-effector payload (Solver.payload_est_*) runs beside the plant on what the
controller sees: it steps after every plant step and is committed to the model payload right before every MPC tick.
With state_estimator set, the controller no longer reads the plant's true state: after every plant step the IMU and encoders are read
(Solver.sim_read_sensors_dev) and a base state estimator (Solver.state_est_*) turns them and the contact flags into the measurement every consumer on
the controller side reads (the updates, the targets' end-effector state, the payload estimator).  The plant and the record keep the truth.
With attitude_filter set as well, an attitude filter (Solver.attitude_*) rewrites each reading's orientation and gyro columns before the estimator reads them.
With slip_detector set as well, a slip detector (Solver.slip_*) removes the stance feet that slide from the contact mask the estimator reads.
On terrain the estimator needs ground_map, its own map of the run's tile library (Solver.state_est_set_ground); the controller still sees no terrain.
With commands set, the gait is rolled on the device (Solver.gait_dev_*): each robot follows its own timeline of gait and cmd_vel commands, and a gait
step right before every target call writes the window GaitSchedule::getModeSchedule gives into the MPC problem's mode schedule rows.  The
timeline may also command the end effector (a goal pose published once and then held, or an ee_cmd_vel stream): the step then tells each robot's
target call which kind to take (DESIGN.md §4.8).
The start mirrors QMController::starting (QMController.cpp:98-126): the first observation from the measured state and one blocking solve before
the loop.  The clock starts at t >= 10 s, so the legs are torque controlled from the first tick (QMController.cpp:177-190).  Without commands the
mode schedule is tiled once on the host for the whole run.  No host synchronisation happens inside the loop; the per-MPC-tick record is the one host copy.
"""
import contextlib

import numpy as np

from . import _lib
from ._lib import EMAX, KMAX, NX, RBD, SENSORS, TARGET
from .interface import gait_schedule, gait_template_names

MPC_PERIOD_MS = 10         # mpcDesiredFrequency 100 (task.info)
HW_DELAY = 0.009           # gazebo/delay (qm_gazebo/config/default.yaml:2)
T_START = 10.0             # QMController::updateControlLaw drives the legs only once time > 10 s


def _schedules(gait, B, t_start, t_obs0, t_end):
    """Mode schedules of one gait name, or of a sequence of B names (tiled once per distinct name) → (event_times[B, EMAX], modes[B, EMAX+1], n_events[B])."""
    names = [gait] * B if isinstance(gait, str) else list(gait)
    if len(names) != B:
        raise ValueError("closed_loop.run: gait must be one name or a sequence of %d names, got %d" % (B, len(names)))
    tiles = {}
    for name in dict.fromkeys(names):
        ev, md, ne = gait_schedule(name, t_start, t_obs0, t_end) if name != "stance" else (np.zeros(EMAX), np.full(EMAX + 1, 15, dtype=np.int32), 0)
        if ne >= EMAX:
            raise ValueError("closed_loop.run: the %s schedule of %.2f s needs more than %d events" % (name, t_end - t_start, EMAX))
        tiles[name] = (ev, md, ne)
    return (np.array([tiles[n][0] for n in names]), np.array([tiles[n][1] for n in names], dtype=np.int32), np.array([tiles[n][2] for n in names], dtype=np.int32))


def run(solver, duration=1.0, gait="stance", cmd_vel=(0.0, 0.0, 0.0, 0.0), wbc_period_ms=2, xy_yaw=None, t_start=T_START, torch_device=None, sim_timer=None,
        friction_mu=None, payload=None, pushes=None, model_payload=None, terrain=None, payload_estimator=None, state_estimator=None, sensor_noise=None,
        attitude_filter=None, slip_detector=None, ground_map=None, commands=None, tuning=None, respawn=None, randomize=None, spawn=None, metrics=None,
        timeline=None, curriculum=None, ee_frame=None, ee_paths=None, ee_path_draw=None):
    """Run `duration` s of closed loop for all solver.batch robots.

    gait: a gait.info template name ("stance", "trot", ...), or a sequence of B names, started at t_start; cmd_vel: (vx, vy, vz, yaw rate) in the
    base frame, (4,) for every robot or [B, 4]; xy_yaw: [B, 3] initial base x, y, yaw (default zeros), each robot starts in qmb200_sim_standing_state.
    friction_mu: scalar or [B], payload: [B, 8] (_lib.PAYLOAD_LAYOUT): set as the handle's robot params for this run (None keeps the handle's own);
    the previous robot params are restored when run returns.  pushes: (t_on[B], duration[B], wrench[B, 12]) with t_on in seconds after the start
    and wrench in _lib.WRENCH_LAYOUT: robot b's wrench acts in every 1 ms plant step whose start lies in [t_on, t_on + duration).
    model_payload: the controller's model payload for this run (Solver.set_model_payload): None keeps the handle's own, "plant" copies this run's plant
    payload (zeros where the plant carries none), or an array [B, 8]; the previous model payload is restored when run returns.
    terrain: dict(tiles [T, ny, nx], cell, tile [B], origin [B, 2]) (qm_control_b200.terrain builds tiles): the plant's ground for this run
    (Solver.sim_set_terrain / sim_set_robot_terrain), each robot starting in the standing state on its own ground; the previous terrain is restored
    when run returns.  The controller does not see the terrain.
    payload_estimator: True, or a dict of qmb200_payload_est_params overrides (Solver.payload_est_set_params), runs the online payload estimate from the model
    payload in force (model_payload's value, or the handle's own): one step after every plant step with the same effort and measurement, one commit right
    before every MPC tick, so the targets, solve, updates and observation of one 10 ms window share one model.  Its status is OR-ed into the record's.
    The estimator is stopped and the previous model payload and estimator parameters restored when run returns.
    state_estimator: True, or a dict of qmb200_state_est_params overrides (Solver.state_est_set_params), closes the loop on estimated base states: after
    every plant step (1 ms step k) the sensors are read with sample = k (-1 for the reading of the start) and the estimator steps; update_dev, the
    targets' end-effector state and the payload estimator read its rbd_est.  It starts at the plant's start position.  Its status is OR-ed into the
    record's.  With terrain only together with ground_map: the estimator's foot-height rows assume the plane otherwise.
    sensor_noise: None (noise-free readings), "reference" (_lib.SENSOR_NOISE_REFERENCE, the IMU covariances of qm_gazebo/config/default.yaml) or a dict
    of qmb200_sensor_params overrides; only with state_estimator.  The estimator is stopped and the previous sensor and estimator parameters restored
    when run returns.
    attitude_filter: True, or a dict of qmb200_attitude_params overrides (Solver.attitude_set_params); only with state_estimator.  After every sensor
    reading (the start's included) an attitude filter step replaces the reading's quaternion and gyro with the filtered orientation and the
    bias-corrected rate, and the estimator steps on that.  Its status is OR-ed into the record's.  The filter is stopped and its previous parameters
    restored when run returns.
    slip_detector: True, or a dict of qmb200_slip_params overrides (Solver.slip_set_params); only with state_estimator.  After every sensor reading
    (and attitude filter step) a detector step turns the plant's contact mask into the mask of trusted stance feet, and the estimator steps on that
    mask.  Its status is OR-ed into the record's.  The detector is stopped and its previous parameters restored when run returns.
    ground_map: True, or dict(tile [B], origin [B, 2]); needs state_estimator and terrain.  The estimator's ground map for this run
    (Solver.state_est_set_ground), on this run's tile library: True gives it the run's own terrain rows (a perfect map), a dict rows of its own (a
    wrong tile, a shifted origin).  Its foot-height rows then follow the mapped ground under each foot.  The controller still does not see the terrain.
    The previous map is restored when run returns.
    commands: dict(t [B, C] in seconds after the start, gait [B, C] of template names or None, and optionally cmd_vel [B, C, 4], ee_goal [B, C, 7]
    (position, quaternion xyzw of unit norm, world frame) and ee_cmd_vel [B, C, 3] (end-effector velocity, world frame), each with NaN rows for none
    and at most one of the three per command): robot b's timeline, sorted per robot.  The run then loads every template of qm_gait.info (Solver.gait_dev_set_templates), starts each robot on
    stance until t_start and then its gait (Solver.gait_dev_reset), and right before every target call (the first, blocking solve included) a gait
    step applies the robot's commands due at t_obs (a gait is inserted at t_obs + T after phaseTransitionStanceTime of stance, as GaitReceiver
    does; a cmd_vel row replaces the robot's cmd_vel) and writes the window [t_obs - T, t_obs + 2T] into the MPC's mode schedule rows.  The host
    tiling and its limit of QMB200_EMAX events over the whole run do not apply.  Its status is OR-ed into the record's; the device schedule is
    stopped when run returns.  Each robot's target source starts on the cmd_vel stream; the last target command a step applies sets it
    (DESIGN.md §4.8): an ee_goal row is published once by that tick's target call (EEgoalPoseToTargetTrajectories, last_ee_target set) and then
    held (the robot's target is left as published), an ee_cmd_vel row switches the robot to the ee_cmd_vel stream (EeCmdVelToTargetTrajectories
    every tick), a cmd_vel row back to the cmd_vel stream.  For both end-effector commands the base target is the end-effector target minus
    (0.52, 0.09) in the world frame, as upstream computes it: meant for robots facing +x.  With commands every target call takes each robot's kind
    from its gait step (Solver.target_trajectories_dev with a per-robot kind).
    tuning: the controller's per-robot tuning rows for this run (Solver.set_robot_tuning): dict field of _lib.TUNING_LAYOUT -> scalar or [B] ([k] or [B, k]
    for the vector gains), fields not named at the handle's own values; friction_mu="plant" / wbc_friction="plant" take this run's plant friction
    (friction_mu's value, or the handle's robot params or plant params).  The previous rows are restored when run returns.
    respawn: True or dict(on_fall=True, hold=0.1, z_min=0.3, tilt_max=0.3, every=None) restarts single robots inside the loop (DESIGN.md §4.10).
    Right before the first solve the run saves its start image (Solver.robot_image_save and a device copy of the loop's own per-robot rows) and
    restores it for every robot, so the first episode starts through the same cold path as every later one.  At the end of every 10 ms window the
    fall detector (Solver.fall_detect_dev, z_min / tilt_max) runs on the plant's rbd; a robot respawns at the next window boundary, before the MPC
    tick, when on_fall and it has been fallen at the last hold / 10 ms window ends, or when every is set and its episode has lasted every seconds
    (hold and every: positive multiples of 10 ms).  A respawned robot returns to its start pose, its estimators' and gait schedule's start
    rows and a cold MPC, WBC and command FIFO, and lives on its own episode clock: its hw_write time, pushes (t_on counts from the episode's start),
    gait commands and mode schedule replay; only the sensor noise keeps the global sample index, so each episode draws new noise.  The image is freed
    when run returns.  at="here" (default "start") restarts a robot where it is (DESIGN.md §4.18): right before its restore the row that stands it on the
    ground point under its base with its heading (Solver.spawn_here_dev, on the plant's rbd), then the restore, then that row placed
    (Solver.spawn_place_dev) with the run's start origins in place of a spawn draw; with spawn episode 0 still draws.  Not with a curriculum spawn, a
    drawn spawn yaw, ee_goal / ee_cmd_vel commands or a ground_map dict.  on_request=True (a Session only; it may stand without on_fall and every) lets
    Session.respawn end robots' episodes.
    randomize: dict(seed=0, <field>=(lo, hi), ...) draws a new plant for every episode (DESIGN.md §4.11): fields of _lib.EPISODE_LAYOUT (the plant's
    friction_mu and payload columns, push_t_on and push_duration in s from the episode's start, the push wrench columns, cmd_vel_x / _y / _z and
    cmd_yaw_rate), each bound a scalar or [B]; fields not named stay at this run's values (friction_mu, payload, pushes and cmd_vel, else the handle's
    robot params or plant params, zero payload and no push).  The start state is read and the start image taken under those values; then every
    episode, the first included, draws its row on the device (Solver.episode_sample_dev) right before its first solve: the plant's friction and
    payload, its push rows and its cmd_vel.  Without respawn every robot draws episode 0 once.  model_payload="plant" also writes a drawn payload into
    the model payload (not together with payload_estimator), tuning friction_mu="plant" / wbc_friction="plant" a drawn friction into the tuning rows.
    The previous ranges, robot params, model payload and tuning rows are restored when run returns.
    spawn: dict(seed=0, tile=(lo, hi), dx=(lo, hi), dy=(lo, hi), yaw=(lo, hi)) starts every episode on new ground (DESIGN.md §4.12), each bound a scalar
    or [B]: the plant's tile (an integer of the run's library, -1 the plane), the offset (dx, dy) in m the robot stands further along it (world axes:
    the tile moves by -(dx, dy) under the robot, whose world x, y stay), and the base yaw in [-pi, pi].  Columns not named stay at this run's values
    (the robot's terrain row, no offset, xy_yaw's yaw, wrapped into [-pi, pi] where it lies outside).  tile, dx and dy need terrain; with
    ground_map=True the estimator's map follows the draw, and a ground_map dict cannot go with them; a yaw that is not fixed cannot go with ee_goal /
    ee_cmd_vel commands (their world-frame goals assume +x).  The start image is taken under the run's own pose; then every episode, the first included, draws its spawn on the device (Solver.spawn_sample_dev)
    right after its restore and its randomize draw and before its first solve: the plant's terrain row, the standing pose there, the measured state,
    the observation, the held end-effector target turned with the base and the estimators' reset rows.  Without respawn every robot spawns episode 0
    once.  The previous terrain rows and ground map are restored when run returns, and then the previous ranges, whose offsets count again from the
    origins of the restored robot terrain rows (the origins are read when ranges are set, and are not part of what spawn_get_ranges reports).
    sim_timer: optional callable(start: bool) wrapped around every sim_step_dev (tools/bench_closedloop.py brackets them with CUDA events).
    Returns dict(t[ticks], base[ticks, B, 6] = (x, y, z, yaw, pitch, roll), ee[ticks, B, 7] = (pos, quat xyzw), status[ticks, B] = OR of the WBC /
    safety, hw_write and plant status words since the previous record, contact[B] at the end, q[B, 24], v[B, 24] at the end; with payload_estimator also
    payload_est[ticks, B, 8] = the model payload rows committed at each record's MPC tick; with state_estimator also base_est[ticks, B, 6], the estimated base in
    the layout of base; with slip_detector also slip[ticks, B], the OR of the detector's slip masks over each record's 10 ms window; with commands also
    gait[ticks, B], the active template id after each record's gait step (an index of gait_templates), mode[ticks, B], the window's mode at that
    step's t_obs, gait_templates, the table's names, target_kind[ticks, B], the kind each robot's target call took at that record's MPC tick (0
    cmd_vel, 1 ee_cmd_vel, 2 goal published, -1 goal held), and ee_target[ticks, B, 7], the final-knot end-effector pose of the target in force after
    that call); with respawn also episode[ticks, B], each robot's episode index in that record's window (0 for the first), and fallen[ticks, B], the
    detector's flag at that window's end; with randomize also episode_params[B, E, 27], the row each robot drew for each episode e < E (E: the most
    episodes of any robot), NaN where a robot had no episode e; with spawn also spawn_params[B, E, 4], the spawn row of each such episode (once any
    restart placed a robot, with or without spawn, the device's record of every episode's row: drawn, placed, or the start's; NaN for a rejected place).
    metrics: True scores every episode on the device (DESIGN.md §4.13, Solver.metrics_step_dev / metrics_close_dev): after every plant step, once the
    step's status words are in the record's and the estimators have stepped, one sample of the plant's truth (its rbd, contact mask and the effort held
    over the step, the target in force, the robot's episode clock, the record's status word and, with state_estimator, the estimate) goes into each
    robot's accumulator.  A respawning robot's episode closes right before its restore (end 1 when the fall rule restarted it, 2 when every did), and
    every robot's open episode closes when the loop ends (end 0).  The samples only read the loop's tensors, so every other output is unchanged.
    Returns also episode_metrics[B, E, METRICS] in the columns of metrics_layout (_lib.METRICS_LAYOUT), E as for episode_params, NaN rows where a
    robot had no episode e.
    timeline: dict(seed=0, n, t_first=(lo, hi), gap=(lo, hi), p_gait=0, gaits=[names], weights=dict(none, cmd_vel, ee_cmd_vel, ee_goal), <box>=(lo, hi),
    ee_quat) draws a new command timeline of n slots for every episode (DESIGN.md §4.14), in place of commands: slot 0 at t_first s after the start, each
    later one gap s after the one before; each slot inserts a gait with probability p_gait, picked uniformly among gaits (qm_gait.info names: one list, or
    B lists), and carries one target command, none, cmd_vel, ee_cmd_vel or ee_goal, with probability proportional to its weight (missing weights are 0;
    default none=1).  The box columns are cmd_vel_x, cmd_vel_y, cmd_vel_z, cmd_yaw_rate (a column not named stays at the run's cmd_vel), ee_vx, ee_vy,
    ee_vz and ee_x, ee_y, ee_z (world frame; named when their kind's weight is positive), ee_quat the goal's quaternion xyzw [4] or [B, 4] (with ee_goal).
    Every bound, p_gait and weight is a scalar or [B].  The run rolls the gait on the device as with commands (gait is the start gait, the same record
    and outputs): it loads a placeholder timeline of width n and every episode, the first included, draws its slots on the device
    (Solver.timeline_sample_dev) right after its restore, its randomize draw and its spawn, before its first solve.  With randomize cmd_vel fields the
    episode's drawn cmd_vel applies from its start, and the timeline's cmd_vel slots replace it as they fall due.  ee_goal / ee_cmd_vel weights cannot
    go with a drawn spawn yaw.  The previous ranges are restored when run returns.  Returns also timeline_params[B, E, n, TIMELINE_CMD], the slots of
    each episode (_lib.TIMELINE_CMD_LAYOUT, t in s after the episode's start), E and the NaN rows as for episode_params.
    curriculum: dict(levels=L, start=0, up_after=1, down_after=1, when=[(column, op, threshold, role), ...], randomize=dict(<field>=(lo, hi)),
    spawn=dict(...), timeline=dict(<box>=(lo, hi), p_gait=..., weights=...)) gives every robot a level in [0, L) that moves with the outcomes of its
    episodes (DESIGN.md §4.15; needs respawn with every).  The run's own randomize / spawn / timeline specs are level 0; curriculum[kind] names the hard
    box of the last level (the columns it does not name are equal at both ends; a timeline's gaits and ee_quat must stay), and level l draws from the
    box fma(l / (L - 1), top - base, base) (Solver.curriculum_attach).  An episode fails when the fall rule ended it or a "fail" condition holds, and
    passes when every ended it and every "pass" condition holds (column of _lib.METRICS_LAYOUT, op ">=" or "<=", threshold a scalar or [B]; conditions
    need metrics=True); up_after passes in a row move a robot one level up, down_after fails one down.  At every respawn the update runs on the device
    after the metrics close and before the restore, so the next episode draws at the new level.  start, up_after and down_after are integers or [B]
    integers, every bound a scalar or [B].  The curriculum is cleared before the previous ranges are restored.  Returns also curriculum_level[ticks, B]
    (each robot's level in that record's window), episode_level[B, E] (-1 where a robot had no episode e), curriculum_state[B, CURRICULUM_STATE] at
    the end (_lib.CURRICULUM_STATE_LAYOUT), and each attached kind's *_params drawn at its episode's level.
    ee_frame: the frame each robot's end-effector targets are stated in for this run (Solver.set_ee_frame; DESIGN.md §4.19): "world" (the default; no
    rows are set, upstream's arithmetic), "heading" (every robot) or [B] of 0 (world) / 1 (heading).  A heading-frame robot holds its hand where it is
    relative to its body while it walks and turns, its ee_goal rows (commands, timeline, Session.command) are poses in its heading frame at the
    publishing tick (the timeline's ee_x / ee_y / ee_z box is in heading coordinates), and the base offset of its end-effector targets turns with its
    yaw.  The refusals of end-effector commands beside varying headings (a drawn spawn yaw, a restart "here" or on given rows) then apply to
    world-frame robots only.  The previous rows are restored when run returns.
    ee_paths: the end-effector path table for this run (Solver.set_ee_paths; DESIGN.md §4.20), a list of (t [n], pose [n, 7]): waypoint times in
    seconds after a path starts (t[0] > 0, strictly increasing, gaps >= time_horizon / 2, 1 <= n <= _lib.EE_PATH_MAX) and waypoint poses (position,
    quaternion xyzw of unit norm; in the heading frame at the path's start for a heading-frame robot).  commands ee_path [B, C] (path ids, -1: none) and
    Session.command(ee_path=[B]) start a path: the hand then follows the piecewise lerp / slerp from its pose at the start through the waypoints on
    their schedule, and holds the last one.  Path commands to world-frame robots share the refusals of ee_goal / ee_cmd_vel.  The previous table is
    restored when run returns; without ee_paths the loop makes exactly the calls it made before.
    ee_path_draw: dict(seed=0, n, tau_first=(lo, hi), gap=(lo, hi), x=(lo, hi), y=(lo, hi), z=(lo, hi), yaw=(lo, hi), quat) draws a new end-effector path
    of n waypoints for every episode (DESIGN.md §4.21): waypoint 0 at tau_first s after the episode's first MPC tick, each next one gap later (gap lo >=
    time_horizon / 2), each at a position drawn in the box x, y, z and oriented Rz(draw(yaw)) quat (yaw in [-pi, pi], quat xyzw of unit norm), stated in
    the path's frame as ee_paths' waypoints are.  Every bound is a scalar or [B].  It rolls the device gait schedule (as commands and timeline do, with
    or without them and with or without ee_paths): every episode, the first included, draws its path on the device last in its beginning, after its
    restore, its randomize draw, its spawn and its timeline draw (Solver.ee_path_sample_dev), into its own row of the path table, and the path starts on
    the episode's first MPC tick.  World-frame robots cannot go with a drawn spawn yaw or restarts "here".  The previous ranges are cleared when run
    returns, before the ee_paths table is restored.  Returns also ee_path_params[B, E, n, 8], the waypoints (tau in s after the episode's start,
    position, quaternion xyzw) of every episode's path (NaN where a robot had no episode e): each robot's own draw, so a robot a Session branched
    from robot s (restore with source) shows its draw while it follows s's path, row P + s; a curriculum may attach it as ee_path_draw=dict(<box>=(lo,
    hi)).  Without ee_path_draw the loop makes exactly the calls it made before."""
    if isinstance(respawn, dict) and _place_spec(respawn)["on_request"]:
        raise ValueError("closed_loop.run: respawn on_request needs a Session (nothing can request a restart inside run; Session.respawn does)")
    with Session(solver, duration, gait=gait, cmd_vel=cmd_vel, wbc_period_ms=wbc_period_ms, xy_yaw=xy_yaw, t_start=t_start, torch_device=torch_device,
                 sim_timer=sim_timer, friction_mu=friction_mu, payload=payload, pushes=pushes, model_payload=model_payload, terrain=terrain,
                 payload_estimator=payload_estimator, state_estimator=state_estimator, sensor_noise=sensor_noise, attitude_filter=attitude_filter,
                 slip_detector=slip_detector, ground_map=ground_map, commands=commands, tuning=tuning, respawn=respawn, randomize=randomize, spawn=spawn,
                 metrics=metrics, timeline=timeline, curriculum=curriculum, ee_frame=ee_frame, ee_paths=ee_paths, ee_path_draw=ee_path_draw) as s:
        rec = s.step(s.windows)
        end = s.finish()   # synchronises the session's stream
        out = {k: v if isinstance(v, np.ndarray) else v.cpu().numpy() for k, v in rec.items()}
        out.update(end)
        return out


RUN_DEFAULTS = dict(gait="stance", cmd_vel=(0.0, 0.0, 0.0, 0.0), wbc_period_ms=2, xy_yaw=None, t_start=T_START, torch_device=None, sim_timer=None, friction_mu=None,
                    payload=None, pushes=None, model_payload=None, terrain=None, payload_estimator=None, state_estimator=None, sensor_noise=None, attitude_filter=None,
                    slip_detector=None, ground_map=None, commands=None, tuning=None, respawn=None, randomize=None, spawn=None, metrics=None, timeline=None, curriculum=None,
                    ee_frame=None, ee_paths=None, ee_path_draw=None)


def _run_specs(solver, steer, o):
    """run's keywords o (RUN_DEFAULTS filled in) → the parsed specs; ValueError, before any solver call, when one is malformed.  steer: a run without
    commands or timeline still rolls the device gait schedule, on an empty timeline."""
    metrics, respawn, randomize, gait, commands, timeline, spawn, curriculum = (o[k] for k in ("metrics", "respawn", "randomize", "gait", "commands", "timeline", "spawn", "curriculum"))
    payload_estimator, state_estimator, sensor_noise, ground_map, terrain = (o[k] for k in ("payload_estimator", "state_estimator", "sensor_noise", "ground_map", "terrain"))
    attitude_filter, slip_detector, model_payload, tuning = (o[k] for k in ("attitude_filter", "slip_detector", "model_payload", "tuning"))
    ef = _ee_frame_spec(getattr(solver, "batch", None), o["ee_frame"])
    world = True if ef is None else ef == _lib.EE_FRAME_WORLD   # the robots whose end-effector targets assume they face +x
    ep = _ee_paths_spec(getattr(solver, "time_horizon", None), o["ee_paths"])
    pd = None if o["ee_path_draw"] is None else _ee_path_draw_spec(getattr(solver, "batch", None), getattr(solver, "time_horizon", None), o["ee_path_draw"])
    if metrics is not None and metrics is not True:
        raise ValueError("closed_loop.run: metrics must be None or True, got %r" % (metrics,))
    rs = None if respawn is None else dict(_respawn_spec(respawn), **_place_spec(respawn))
    rz = None if randomize is None else _randomize_spec(getattr(solver, "batch", None), randomize)
    if payload_estimator is not None and payload_estimator is not True and not isinstance(payload_estimator, dict):
        raise ValueError("closed_loop.run: payload_estimator must be None, True or a dict of estimator parameters, got %r" % (payload_estimator,))
    if state_estimator is not None and state_estimator is not True and not isinstance(state_estimator, dict):
        raise ValueError("closed_loop.run: state_estimator must be None, True or a dict of estimator parameters, got %r" % (state_estimator,))
    if sensor_noise is not None and sensor_noise != "reference" and not isinstance(sensor_noise, dict):
        raise ValueError("closed_loop.run: sensor_noise must be None, \"reference\" or a dict of sensor parameters, got %r" % (sensor_noise,))
    if sensor_noise is not None and state_estimator is None:
        raise ValueError("closed_loop.run: sensor_noise needs state_estimator (the controller reads the plant's true state otherwise)")
    if ground_map is not None and ground_map is not True and not isinstance(ground_map, dict):
        raise ValueError("closed_loop.run: ground_map must be None, True or dict(tile, origin), got %r" % (ground_map,))
    if ground_map is not None and (state_estimator is None or terrain is None):
        raise ValueError("closed_loop.run: ground_map needs state_estimator and terrain (it maps the run's tile library for the estimator)")
    if state_estimator is not None and terrain is not None and ground_map is None:
        raise ValueError("closed_loop.run: state_estimator on terrain needs ground_map (without one its foot-height rows assume the plane)")
    if attitude_filter is not None and attitude_filter is not True and not isinstance(attitude_filter, dict):
        raise ValueError("closed_loop.run: attitude_filter must be None, True or a dict of attitude filter parameters, got %r" % (attitude_filter,))
    if attitude_filter is not None and state_estimator is None:
        raise ValueError("closed_loop.run: attitude_filter needs state_estimator (it filters the sensor readings the estimator reads)")
    if slip_detector is not None and slip_detector is not True and not isinstance(slip_detector, dict):
        raise ValueError("closed_loop.run: slip_detector must be None, True or a dict of slip detector parameters, got %r" % (slip_detector,))
    if slip_detector is not None and state_estimator is None:
        raise ValueError("closed_loop.run: slip_detector needs state_estimator (it chooses the stance feet the estimator trusts)")
    gd = None if commands is None else _gait_commands(solver.batch, gait, commands, 0 if ep is None else len(ep))
    if (steer or pd is not None) and commands is None and timeline is None:   # an empty timeline: the session's commands are the schedule's only input
        gd = _gait_commands(solver.batch, gait, dict(t=np.zeros((solver.batch, 0)), gait=np.empty((solver.batch, 0), dtype=object)))
    tl = None if timeline is None else _timeline_spec(getattr(solver, "batch", None), gait, timeline, commands)
    if tl is not None:
        gd = tl["gd"]
    if pd is not None:
        gd = _with_paths(gd)
    tn = None if tuning is None else _tuning_spec(solver.batch, tuning)
    sp = None if spawn is None else _spawn_spec(getattr(solver, "batch", None), spawn, terrain, ground_map, gd, world)
    cu = None
    if curriculum is not None:
        cu = _curriculum_spec(getattr(solver, "batch", None), curriculum, rs, metrics is not None, gait,
                              dict(episode=randomize, spawn=spawn, timeline=timeline, ee_path=o["ee_path_draw"]), terrain, ground_map, gd, world,
                              getattr(solver, "time_horizon", None))
        if cu["gd"] is not None:   # a top box that weighs end-effector commands needs the placeholder timeline's end-effector rows
            gd = tl["gd"] = cu["gd"] if pd is None else _with_paths(cu["gd"])
    if rs is not None and rs["at"] == "here":
        yaw_drawn = sp is not None and "yaw" in sp["fields"] and np.any(sp["fields"]["yaw"][0] != sp["fields"]["yaw"][1])
        why = _here_refusal(yaw_drawn, gd, curriculum, ground_map, world)
        if why is not None:
            raise ValueError("closed_loop.run: respawn at=\"here\" cannot go with %s" % why)
    if rz is not None:   # the links: a drawn payload / friction also goes where the run told the controller the plant's
        drawn = set(rz["fields"]) | set(cu["tops"]["episode"]["fields"] if cu is not None and "episode" in cu["tops"] else ())
        if isinstance(model_payload, str) and model_payload == "plant" and drawn & set(_lib.PAYLOAD_LAYOUT):
            if payload_estimator is not None:
                raise ValueError("closed_loop.run: model_payload=\"plant\" with a randomized payload cannot run with payload_estimator (its commits own the model payload)")
            rz["link"] |= _lib.EPISODE_MODEL_PAYLOAD
        if tn is not None and "friction_mu" in drawn:
            rz["link"] |= (_lib.EPISODE_MPC_FRICTION if isinstance(tn.get("friction_mu"), str) else 0) | (_lib.EPISODE_WBC_FRICTION if isinstance(tn.get("wbc_friction"), str) else 0)
    return dict(rs=rs, rz=rz, gd=gd, tl=tl, tn=tn, sp=sp, cu=cu, ef=ef, world=world, ep=ep, pd=pd)


def _respawn_spec(respawn):
    """closed_loop.run's respawn → dict(on_fall, hold_windows, z_min, tilt_max, every_ms or None); ValueError when malformed (_place_spec reads at and
    on_request)"""
    spec = dict(on_fall=True, hold=0.1, z_min=0.3, tilt_max=0.3, every=None)
    place = _place_spec(respawn)
    if respawn is not True:
        if not isinstance(respawn, dict) or not set(respawn) <= set(spec) | set(place):
            raise ValueError("closed_loop.run: respawn must be None, True or dict(on_fall, hold, z_min, tilt_max, every, at, on_request), got %r" % (respawn,))
        spec.update({k: v for k, v in respawn.items() if k not in place})
    if not isinstance(spec["on_fall"], (bool, np.bool_)):
        raise ValueError("closed_loop.run: respawn on_fall must be True or False, got %r" % (spec["on_fall"],))

    def ms(name, v):
        try:
            x = np.nan if isinstance(v, (str, bool)) else float(v) * 1e3
        except (TypeError, ValueError):
            x = np.nan
        n = int(round(x)) if np.isfinite(x) else 0
        if not (n > 0 and n % MPC_PERIOD_MS == 0 and abs(x - n) < 1e-6):
            raise ValueError("closed_loop.run: respawn %s must be a positive multiple of %d ms, got %r" % (name, MPC_PERIOD_MS, v))
        return n
    hold = ms("hold", spec["hold"]); every = None if spec["every"] is None else ms("every", spec["every"])
    for name in ("z_min", "tilt_max"):
        if isinstance(spec[name], (bool, str)) or not np.isfinite(np.asarray(spec[name], dtype=np.float64)) or np.ndim(spec[name]) != 0:
            raise ValueError("closed_loop.run: respawn %s must be a finite number, got %r" % (name, spec[name]))
    if not float(spec["tilt_max"]) > 0.0:
        raise ValueError("closed_loop.run: respawn tilt_max must be > 0, got %r" % (spec["tilt_max"],))
    if not spec["on_fall"] and every is None and not place["on_request"]:
        raise ValueError("closed_loop.run: respawn needs on_fall, every or on_request (it would never restart a robot)")
    return dict(on_fall=bool(spec["on_fall"]), hold_windows=hold // MPC_PERIOD_MS, z_min=float(spec["z_min"]), tilt_max=float(spec["tilt_max"]), every_ms=every)


RESPAWN_AT = ("start", "here")   # respawn at: a restart returns to the start pose (or draws the spawn), or stands the robot where it is (DESIGN.md §4.18)


def _place_spec(respawn):
    """closed_loop.run's respawn → dict(at, on_request): where its restarts stand robots and whether a Session may request them; ValueError when malformed"""
    spec = dict(at="start", on_request=False)
    if isinstance(respawn, dict):
        spec.update({k: respawn[k] for k in spec if k in respawn})
    if not isinstance(spec["on_request"], (bool, np.bool_)):
        raise ValueError("closed_loop.run: respawn on_request must be True or False, got %r" % (spec["on_request"],))
    if not isinstance(spec["at"], str) or spec["at"] not in RESPAWN_AT:
        raise ValueError("closed_loop.run: respawn at must be \"start\" or \"here\", got %r" % (spec["at"],))
    return dict(at=spec["at"], on_request=bool(spec["on_request"]))


def _ee_names(goal_or_vel, path):
    """the end-effector commands a refusal names: "ee_goal / ee_cmd_vel", "ee_path" or both, or None for none"""
    names = (["ee_goal / ee_cmd_vel"] if goal_or_vel else []) + (["ee_path"] if path else [])
    return " / ".join(names) or None


def _ee_refused(gd, world, robots=True):
    """the end-effector commands of the parsed commands gd that go to world-frame robots (world: True or bool [B]) among robots (True or bool [B]),
    named for a refusal (_ee_names), or None"""
    if gd is None:
        return None
    m = gd["ee_robots"] & world & robots; path = gd.get("path_robots", False)
    return _ee_names(np.any(m & gd.get("goal_robots", gd["ee_robots"])), np.any(m & path))


def _here_refusal(sp_yaw_drawn, gd, curriculum, ground_map, world=True):
    """why a restart "here" (or on given spawn rows) cannot go with this run's specs, or None: the heading it keeps varies per robot.  world: True or
    bool [B], the world-frame robots (end-effector commands to heading-frame robots follow their heading)."""
    if curriculum is not None and "spawn" in curriculum:
        return "a curriculum attached to the spawn (its levels draw every spawn)"
    if sp_yaw_drawn:
        return "a drawn spawn yaw (the heading a restart keeps would not be the draw's)"
    names = _ee_refused(gd, world)
    if names is not None:
        return "%s commands to world-frame robots (their world-frame goals assume the robot faces +x)" % names
    if isinstance(ground_map, dict):
        return "a ground_map dict (the map would not follow the ground; ground_map=True does)"
    return None


def _ranges_spec(kind, layout, B, value):
    """closed_loop.run's randomize or spawn dict (kind names it) → (seed, fields: name -> (lo, hi) float arrays, scalar or [B]) for the columns of
    layout; ValueError when the seed or a field is malformed.  B None: the bounds' length is not checked."""
    seed = value.get("seed", 0)
    if isinstance(seed, (bool, np.bool_)) or not isinstance(seed, (int, np.integer)) or not 0 <= int(seed) < 1 << 64:
        raise ValueError("closed_loop.run: %s seed must be an integer in [0, 2^64), got %r" % (kind, seed))
    fields = {}
    for k, v in value.items():
        if k == "seed":
            continue
        if k not in layout:
            raise ValueError("closed_loop.run: unknown %s field %r (one of seed, %s)" % (kind, k, ", ".join(layout)))
        try:
            if isinstance(v, str) or len(v) != 2 or any(isinstance(a, str) for a in v):
                raise TypeError
            lo, hi = (np.asarray(a, dtype=np.float64) for a in v)
        except (TypeError, ValueError):
            raise ValueError("closed_loop.run: %s %s must be a pair (lo, hi) of numbers or [B] arrays, got %r" % (kind, k, v)) from None
        if any(a.ndim > 1 or (a.ndim == 1 and B is not None and a.shape != (B,)) for a in (lo, hi)) or (lo.ndim == hi.ndim == 1 and lo.shape != hi.shape):
            raise ValueError("closed_loop.run: %s %s bounds must be scalars or [%s], got shapes %s and %s" % (kind, k, "B" if B is None else B, lo.shape, hi.shape))
        with np.errstate(invalid="ignore", over="ignore"):
            if not (np.all(np.isfinite(lo)) and np.all(np.isfinite(hi)) and np.all(lo <= hi) and np.all(np.isfinite(hi - lo))):
                raise ValueError("closed_loop.run: %s %s bounds must be finite with lo <= hi, got %r" % (kind, k, v))
        fields[k] = (lo, hi)
    return int(seed), fields


def _randomize_spec(B, randomize):
    """closed_loop.run's randomize → dict(seed, fields: name -> (lo, hi) float arrays, scalar or [B], link=0); ValueError when malformed.  B None: the
    bounds' length is not checked."""
    if not isinstance(randomize, dict):
        raise ValueError("closed_loop.run: randomize must be None or dict(seed=..., <field>=(lo, hi), ...), got %r" % (randomize,))
    seed, fields = _ranges_spec("randomize", _lib.EPISODE_LAYOUT, B, randomize)
    for k, (lo, hi) in fields.items():
        if k == "friction_mu" and not np.all(lo > 0.0):
            raise ValueError("closed_loop.run: randomize friction_mu lo must be > 0")
        if k in ("m_ee", "m_base", "push_t_on", "push_duration") and not np.all(lo >= 0.0):
            raise ValueError("closed_loop.run: randomize %s lo must be >= 0" % k)
    return dict(seed=seed, fields=fields, link=0)


def _spawn_spec(B, spawn, terrain, ground_map, gd, world=True):
    """closed_loop.run's spawn (with its terrain, ground_map and parsed commands) → dict(seed, fields: name -> (lo, hi) float arrays, scalar or [B],
    link); ValueError when malformed.  B None: the bounds' length is not checked.  world: True or bool [B], the world-frame robots."""
    if not isinstance(spawn, dict):
        raise ValueError("closed_loop.run: spawn must be None or dict(seed=..., tile=(lo, hi), dx=(lo, hi), dy=(lo, hi), yaw=(lo, hi)), got %r" % (spawn,))
    seed, fields = _ranges_spec("spawn", _lib.SPAWN_LAYOUT, B, spawn)
    if "yaw" in fields and not (np.all(fields["yaw"][0] >= -np.pi) and np.all(fields["yaw"][1] <= np.pi)):
        raise ValueError("closed_loop.run: spawn yaw bounds must lie in [-pi, pi]")
    ground = set(fields) & {"tile", "dx", "dy"}
    if ground and terrain is None:
        raise ValueError("closed_loop.run: spawn %s needs terrain (it moves the plant's tile under the robot)" % ", ".join(sorted(ground)))
    if "tile" in fields:
        lo, hi = fields["tile"]; n = len(terrain["tiles"])
        if not (np.all(np.floor(lo) == lo) and np.all(np.floor(hi) == hi) and np.all(lo >= -1) and np.all(hi < n)):
            raise ValueError("closed_loop.run: spawn tile bounds must be integers in [-1, %d), the run's tile library" % n)
    if ground and isinstance(ground_map, dict):
        raise ValueError("closed_loop.run: a ground_map dict cannot go with a spawn that draws %s (the map would not follow the ground; ground_map=True does)"
                         % ", ".join(sorted(ground)))
    names = _ee_refused(gd, world, fields["yaw"][0] != fields["yaw"][1]) if "yaw" in fields else None
    if names is not None:
        raise ValueError("closed_loop.run: a drawn spawn yaw cannot go with %s commands to world-frame robots (their world-frame goals assume the robot "
                         "faces +x)" % names)
    return dict(seed=seed, fields=fields, link=_lib.SPAWN_GROUND_MAP if ground_map is True else 0)


@contextlib.contextmanager
def _ranges(solver, kind):
    """the ranges of solver's kind ("episode", "spawn", "timeline" or "ee_path") draws in force, set again on exit"""
    prev = getattr(solver, kind + "_get_ranges")()
    try:
        yield   # the session's start sets this run's ranges once it has read its fixed values
    finally:
        if prev is None:
            getattr(solver, kind + "_set_ranges")(None)
        else:
            getattr(solver, kind + "_set_ranges")(**prev)


def _box(layout, row, spec):
    """a box of ranges: every column fixed at the run's value, row [B, C], except the spec's fields, drawn within their bounds → lo, hi [B, C]"""
    col = {n: i for i, n in enumerate(layout)}
    lo = row.copy(); hi = row.copy()
    for k, (l, h) in spec["fields"].items():
        lo[:, col[k]] = l; hi[:, col[k]] = h
    return lo, hi


def _timeline_box(tl, cmd_vel, t_start):
    """the box of a parsed timeline spec: the fixed columns, the run's cmd_vel where not named, the named columns' bounds; times on the observation clock"""
    TL = {n: i for i, n in enumerate(_lib.TIMELINE_LAYOUT)}
    row = np.zeros((len(cmd_vel), _lib.TIMELINE)); row[:, TL["p_gait"]] = tl["p_gait"]; row[:, TL["gait_set"]] = tl["gait_set"]
    row[:, TL["w_none"]:TL["w_none"] + 4] = tl["weights"]; row[:, TL["cmd_vel_x"]:TL["cmd_vel_x"] + 4] = cmd_vel; row[:, TL["ee_qx"]:TL["ee_qx"] + 4] = tl["quat"]
    lo, hi = _box(_lib.TIMELINE_LAYOUT, row, tl)
    lo[:, TL["t_first"]] += t_start; hi[:, TL["t_first"]] += t_start
    return lo, hi


def _gait_commands(B, gait, commands, n_paths=0):
    """closed_loop.run's gait and commands → dict(names, gait [B] ids, t [B, C], tmpl [B, C] ids or -1, cmd_vel [B, C, 4], ee: {} or dict(ee_kind [B, C],
    ee_cmd [B, C, 7]) when the timeline has ee_goal / ee_cmd_vel / ee_path); ValueError when malformed.  n_paths: the run's ee_paths table size"""
    names = gait_template_names()
    ids = {n: i for i, n in enumerate(names)}
    start = [gait] * B if isinstance(gait, str) else list(gait)
    if len(start) != B:
        raise ValueError("closed_loop.run: gait must be one name or a sequence of %d names, got %d" % (B, len(start)))
    if not isinstance(commands, dict) or not {"t", "gait"} <= set(commands) or not set(commands) <= {"t", "gait", "cmd_vel", "ee_goal", "ee_cmd_vel", "ee_path"}:
        raise ValueError("closed_loop.run: commands must be dict(t, gait[, cmd_vel][, ee_goal][, ee_cmd_vel][, ee_path]), got %r" % (commands,))
    t = np.asarray(commands["t"], dtype=np.float64)
    if t.ndim != 2 or t.shape[0] != B:
        raise ValueError("closed_loop.run: commands t must have shape (%d, C), got %s" % (B, t.shape))
    C = t.shape[1]
    g = np.asarray(commands["gait"], dtype=object)
    vel = np.full((B, C, 4), np.nan) if commands.get("cmd_vel") is None else np.asarray(commands["cmd_vel"], dtype=np.float64)
    if g.shape != (B, C) or vel.shape != (B, C, 4):
        raise ValueError("closed_loop.run: commands gait must have shape (%d, %d) and cmd_vel (%d, %d, 4), got %s and %s" % (B, C, B, C, g.shape, vel.shape))
    unknown = sorted({str(n) for n in list(start) + [n for n in g.ravel() if n is not None] if n not in ids})
    if unknown:
        raise ValueError("closed_loop.run: unknown gait name(s) %s (qm_gait.info has %s)" % (", ".join(unknown), ", ".join(names)))
    if not np.all(np.isfinite(t)) or np.any(np.diff(t, axis=1) < 0):
        raise ValueError("closed_loop.run: commands t must be finite and sorted per robot")
    if np.any(np.isnan(vel).any(-1) != np.isnan(vel).all(-1)) or np.any(np.isinf(vel)):
        raise ValueError("closed_loop.run: each commands cmd_vel row must be finite or all NaN")
    tmpl = np.array([[-1 if n is None else ids[n] for n in row] for row in g], dtype=np.int32).reshape(B, C)
    ee = _ee_commands(B, C, commands, vel, n_paths)
    return dict(names=names, gait=np.array([ids[n] for n in start], dtype=np.int32), t=t, tmpl=tmpl, cmd_vel=vel, ee=ee,
                ee_robots=(ee["ee_kind"] >= 0).any(-1) if ee else np.zeros(B, dtype=bool),
                goal_robots=np.isin(ee["ee_kind"], (_lib.TARGET_EE_CMD_VEL, _lib.TARGET_EE_GOAL)).any(-1) if ee else np.zeros(B, dtype=bool),
                path_robots=(ee["ee_kind"] == _lib.TARGET_EE_PATH).any(-1) if ee else np.zeros(B, dtype=bool))


def _ee_commands(B, C, commands, vel, n_paths=0):
    """commands' ee_goal [B, C, 7] / ee_cmd_vel [B, C, 3] / ee_path [B, C] → {} when none is given, else dict(ee_kind [B, C], ee_cmd [B, C, 7]) for
    Solver.gait_dev_set_commands; ValueError when malformed.  n_paths: the run's ee_paths table size (ee_path ids lie in [-1, n_paths))"""
    if commands.get("ee_goal") is None and commands.get("ee_cmd_vel") is None and commands.get("ee_path") is None:
        return {}
    path = np.full((B, C), -1) if commands.get("ee_path") is None else np.asarray(commands["ee_path"])
    if path.shape != (B, C) or path.dtype.kind not in "iu" or np.any(path < -1):
        raise ValueError("closed_loop.run: commands ee_path must be integer path ids (-1: none) of shape (%d, %d), got %r" % (B, C, commands.get("ee_path")))
    if np.any(path >= n_paths):
        raise ValueError("closed_loop.run: commands ee_path ids must lie in [-1, %d), the run's ee_paths (ee_paths=[(t, pose), ...] sets them)" % n_paths)
    goal = np.full((B, C, 7), np.nan) if commands.get("ee_goal") is None else np.asarray(commands["ee_goal"], dtype=np.float64)
    eev = np.full((B, C, 3), np.nan) if commands.get("ee_cmd_vel") is None else np.asarray(commands["ee_cmd_vel"], dtype=np.float64)
    if goal.shape != (B, C, 7) or eev.shape != (B, C, 3):
        raise ValueError("closed_loop.run: commands ee_goal must have shape (%d, %d, 7) and ee_cmd_vel (%d, %d, 3), got %s and %s" % (B, C, B, C, goal.shape, eev.shape))
    for name, a in (("ee_goal", goal), ("ee_cmd_vel", eev)):
        if np.any(np.isnan(a).any(-1) != np.isnan(a).all(-1)) or np.any(np.isinf(a)):
            raise ValueError("closed_loop.run: each commands %s row must be finite or all NaN" % name)
    has_goal, has_eev, has_path = ~np.isnan(goal[..., 0]), ~np.isnan(eev[..., 0]), path >= 0
    if np.any(has_goal.astype(int) + has_eev + has_path + ~np.isnan(vel[..., 0]) > 1):
        raise ValueError("closed_loop.run: a command carries at most one of cmd_vel, ee_goal, ee_cmd_vel and ee_path")
    if np.any(np.abs(np.linalg.norm(goal[has_goal][:, 3:7], axis=-1) - 1.0) > 1e-9):
        raise ValueError("closed_loop.run: each commands ee_goal quaternion (xyzw) must have unit norm (within 1e-9)")
    kind = np.where(has_goal, _lib.TARGET_EE_GOAL, np.where(has_eev, _lib.TARGET_EE_CMD_VEL, np.where(has_path, _lib.TARGET_EE_PATH, -1))).astype(np.int32)
    cmd = np.where(has_goal[..., None], goal, 0.0); cmd[..., :3] = np.where(has_eev[..., None], eev, cmd[..., :3])
    cmd[..., 0] = np.where(has_path, path, cmd[..., 0])
    return dict(ee_kind=kind, ee_cmd=cmd)


TIMELINE_BOX = ("t_first", "gap", "cmd_vel_x", "cmd_vel_y", "cmd_vel_z", "cmd_yaw_rate", "ee_vx", "ee_vy", "ee_vz", "ee_x", "ee_y", "ee_z")
TIMELINE_KINDS = ("none", "cmd_vel", "ee_cmd_vel", "ee_goal")


def _timeline_spec(B, gait, timeline, commands):
    """closed_loop.run's gait and timeline → dict(seed, n, fields: name -> (lo, hi) float arrays, scalar or [B], p_gait, gait_set, weights [4] or [B, 4],
    quat [4] or [B, 4], gd: the placeholder timeline as _gait_commands gives it); ValueError when malformed.  B None: the lengths are not checked."""
    if commands is not None:
        raise ValueError("closed_loop.run: timeline and commands cannot go together (both set the device gait schedule's timeline)")
    if not isinstance(timeline, dict):
        raise ValueError("closed_loop.run: timeline must be None or dict(seed, n, t_first, gap, p_gait, gaits, weights, <field>=(lo, hi), ee_quat), got %r" % (timeline,))
    n = timeline.get("n")
    if isinstance(n, (bool, np.bool_)) or not isinstance(n, (int, np.integer)) or n < 1:
        raise ValueError("closed_loop.run: timeline n must be an integer >= 1, got %r" % (n,))
    seed, fields = _ranges_spec("timeline", TIMELINE_BOX, B, {k: v for k, v in timeline.items() if k not in ("n", "p_gait", "gaits", "weights", "ee_quat")})
    for k in ("t_first", "gap"):
        if k not in fields:
            raise ValueError("closed_loop.run: timeline needs %s=(lo, hi)" % k)
    if not np.all(fields["gap"][0] >= 0.0):
        raise ValueError("closed_loop.run: timeline gap lo must be >= 0")

    def per_robot(name, v, width=None):
        a = np.asarray(v, dtype=np.float64) if not isinstance(v, (str, bool, np.bool_)) else np.array(np.nan)
        ok = ((width,),) if width else ((),)
        if a.shape not in ok and not (a.ndim == (2 if width else 1) and (B is None or a.shape[0] == B) and (not width or a.shape[1] == width)):
            raise ValueError("closed_loop.run: timeline %s must be %s or [%s%s], got shape %s" % (name, "[%d]" % width if width else "a scalar", "B" if B is None else B,
                                                                                           ", %d" % width if width else "", a.shape))
        if not np.all(np.isfinite(a)):
            raise ValueError("closed_loop.run: timeline %s must be finite, got %r" % (name, v))
        return a
    p_gait = per_robot("p_gait", timeline.get("p_gait", 0.0))
    if not np.all((p_gait >= 0.0) & (p_gait <= 1.0)):
        raise ValueError("closed_loop.run: timeline p_gait must lie in [0, 1]")
    names = gait_template_names(); ids = {nm: i for i, nm in enumerate(names)}
    start = [gait] * (1 if B is None else B) if isinstance(gait, str) else list(gait)
    if B is not None and len(start) != B:
        raise ValueError("closed_loop.run: gait must be one name or a sequence of %d names, got %d" % (B, len(start)))
    gaits = timeline.get("gaits", [])
    sets = [gaits] if all(isinstance(g, str) for g in gaits) else list(gaits)
    if any(isinstance(g, str) or not all(isinstance(x, str) for x in g) for g in sets) or (len(sets) != 1 and B is not None and len(sets) != B):
        raise ValueError("closed_loop.run: timeline gaits must be one list of gait names or %s such lists, got %r" % ("B" if B is None else B, gaits))
    unknown = sorted({str(x) for x in start + [x for g in sets for x in g] if x not in ids})
    if unknown:
        raise ValueError("closed_loop.run: unknown gait name(s) %s (qm_gait.info has %s)" % (", ".join(unknown), ", ".join(names)))
    gait_set = np.array([float(sum(1 << ids[x] for x in set(g))) for g in sets]); gait_set = gait_set[0] if len(sets) == 1 else gait_set
    if np.any((p_gait > 0.0) & (gait_set == 0.0)):
        raise ValueError("closed_loop.run: timeline gaits must name at least one gait where p_gait > 0")
    w = timeline.get("weights", dict(none=1.0))
    if not isinstance(w, dict) or not set(w) <= set(TIMELINE_KINDS):
        raise ValueError("closed_loop.run: timeline weights must be dict(%s), got %r" % (", ".join(TIMELINE_KINDS), w))
    weights = np.stack(np.broadcast_arrays(*(per_robot("weight " + k, w.get(k, 0.0)) for k in TIMELINE_KINDS)), axis=-1)
    if np.any(weights < 0.0) or not np.all(weights.sum(-1) > 0.0):
        raise ValueError("closed_loop.run: timeline weights must be >= 0 with a positive sum")
    need = [(k, c) for k, cols in (("ee_cmd_vel", ("ee_vx", "ee_vy", "ee_vz")), ("ee_goal", ("ee_x", "ee_y", "ee_z"))) for c in cols
            if np.any(weights[..., TIMELINE_KINDS.index(k)] > 0.0) and c not in fields]
    if need:
        raise ValueError("closed_loop.run: timeline %s needs %s=(lo, hi) (its weight is positive)" % (need[0][0], need[0][1]))
    goal = np.any(weights[..., 3] > 0.0)
    if goal and timeline.get("ee_quat") is None:
        raise ValueError("closed_loop.run: timeline ee_goal needs ee_quat (its weight is positive)")
    quat = per_robot("ee_quat", timeline.get("ee_quat", (0.0, 0.0, 0.0, 1.0)), 4)
    if np.any(np.abs(np.linalg.norm(quat, axis=-1) - 1.0) > 1e-9):
        raise ValueError("closed_loop.run: timeline ee_quat (xyzw) must have unit norm (within 1e-9)")
    Bn = len(start)   # the placeholder timeline the sampler writes into: +inf times, no command
    ee = {} if not np.any(weights[..., 2:] > 0.0) else dict(ee_kind=np.full((Bn, n), -1, dtype=np.int32), ee_cmd=np.zeros((Bn, n, 7)))
    gd = dict(names=names, gait=np.array([ids[x] for x in start], dtype=np.int32), t=np.full((Bn, n), np.inf), tmpl=np.full((Bn, n), -1, dtype=np.int32),
              cmd_vel=np.full((Bn, n, 4), np.nan), ee=ee, ee_robots=np.any(weights[..., 2:] > 0.0, axis=-1))
    return dict(seed=seed, n=int(n), fields=fields, p_gait=p_gait, gait_set=gait_set, weights=weights, quat=quat, gd=gd)


EE_PATH_BOX = ("tau_first", "gap", "x", "y", "z", "yaw")


def _ee_path_draw_spec(B, T, spec):
    """closed_loop.run's ee_path_draw → dict(seed, n, fields: name -> (lo, hi) float arrays, scalar or [B], quat [4] or [B, 4]); ValueError when malformed
    (the library's rules: DESIGN.md §4.21).  B None: the lengths are not checked; T (the handle's time horizon) None: the T/2 gap rule is left to the
    library."""
    keys = ("seed", "n", "quat") + EE_PATH_BOX
    if not isinstance(spec, dict) or not set(spec) <= set(keys):
        raise ValueError("closed_loop.run: ee_path_draw must be None or dict(%s), got %r" % (", ".join(keys), spec))
    n = spec.get("n")
    if isinstance(n, (bool, np.bool_)) or not isinstance(n, (int, np.integer)) or not 1 <= n <= _lib.EE_PATH_MAX:
        raise ValueError("closed_loop.run: ee_path_draw n must be an integer in [1, %d], got %r" % (_lib.EE_PATH_MAX, n))
    seed, fields = _ranges_spec("ee_path_draw", EE_PATH_BOX, B, {k: v for k, v in spec.items() if k not in ("n", "quat")})
    missing = [k for k in EE_PATH_BOX if k not in fields and k != "yaw"]
    if missing:
        raise ValueError("closed_loop.run: ee_path_draw needs %s=(lo, hi)" % missing[0])
    if not np.all(fields["tau_first"][0] > 0.0):
        raise ValueError("closed_loop.run: ee_path_draw tau_first lo must be > 0 (seconds after the path starts)")
    if T is not None and not np.all(fields["gap"][0] >= 0.5 * T):
        raise ValueError("closed_loop.run: ee_path_draw gap lo must be >= time_horizon / 2 = %g s" % (0.5 * T))
    if "yaw" in fields and not (np.all(fields["yaw"][0] >= -np.pi) and np.all(fields["yaw"][1] <= np.pi)):
        raise ValueError("closed_loop.run: ee_path_draw yaw bounds must lie in [-pi, pi]")
    with np.errstate(over="ignore"):
        if not np.all(fields["tau_first"][1] + (n - 1) * fields["gap"][1] <= 1e300):
            raise ValueError("closed_loop.run: ee_path_draw tau_first hi + (n - 1) gap hi must be <= 1e300 s (every drawn time finite)")
    q = spec.get("quat")
    quat = np.array(np.nan) if q is None or isinstance(q, (str, bool, np.bool_)) else np.asarray(q, dtype=np.float64)
    if quat.shape != (4,) and not (quat.ndim == 2 and quat.shape[1] == 4 and (B is None or quat.shape[0] == B)):
        raise ValueError("closed_loop.run: ee_path_draw quat must be [4] or [%s, 4] (xyzw), got %r" % ("B" if B is None else B, q))
    if not np.all(np.isfinite(quat)) or np.any(np.abs(np.linalg.norm(quat, axis=-1) - 1.0) > 1e-9):
        raise ValueError("closed_loop.run: ee_path_draw quat (xyzw) must be finite with unit norm (within 1e-9)")
    return dict(seed=seed, n=int(n), fields=fields, quat=quat)


def _ee_path_box(pd, B):
    """the ranges lo, hi [B, EE_PATH_RANGES] of a parsed ee_path_draw spec: n_way and the quaternion fixed, the named columns' bounds (yaw 0 unless named)"""
    row = np.zeros((B, _lib.EE_PATH_RANGES)); row[:, 0] = pd["n"]; row[:, 7:11] = pd["quat"]
    return _box(_lib.EE_PATH_RANGES_LAYOUT, row, pd)


def _with_paths(gd):
    """the parsed commands gd with every robot commanded an end-effector path (a drawn path starts every episode), for the refusals"""
    B = len(gd["gait"])
    return dict(gd, ee_robots=np.ones(B, dtype=bool), goal_robots=gd.get("goal_robots", gd["ee_robots"]), path_robots=np.ones(B, dtype=bool))


CURRICULUM_KINDS = dict(randomize="episode", spawn="spawn", timeline="timeline", ee_path_draw="ee_path")   # a curriculum spec's key → the draw kind it attaches to


def _curriculum_spec(B, curriculum, rs, metrics, gait, base, terrain, ground_map, gd, world=True, T=None):
    """closed_loop.run's curriculum (with the run's respawn spec rs, whether metrics is on, its gait, base: the run's own randomize / spawn / timeline
    specs by kind, terrain, ground_map and parsed commands) → dict(levels, start, up_after, down_after (int arrays, scalar or [B]), conditions [(column,
    op, role)], thresholds [float arrays, scalar or [B]], tops: kind -> the parsed spec of its top box, gd: the placeholder timeline when the top box
    weighs end-effector commands and the base does not, else None); ValueError when malformed.  B None: the lengths are not checked; T: the handle's
    time horizon, for an ee_path_draw top box."""
    keys = ("levels", "start", "up_after", "down_after", "when") + tuple(CURRICULUM_KINDS)
    if not isinstance(curriculum, dict) or not set(curriculum) <= set(keys):
        raise ValueError("closed_loop.run: curriculum must be None or dict(%s), got %r" % (", ".join(keys), curriculum))
    if rs is None:
        raise ValueError("closed_loop.run: curriculum needs respawn (a level moves when an episode closes)")
    if rs["every_ms"] is None:
        raise ValueError("closed_loop.run: curriculum needs respawn every (without it no episode can pass)")

    def ints(name, v, lo, hi=None):
        a = np.asarray(v) if not isinstance(v, (str, bool, np.bool_)) else np.array(np.nan)
        if a.ndim > 1 or (a.ndim == 1 and B is not None and a.shape != (B,)) or a.dtype.kind not in "iuf" or not np.all(np.isfinite(a)) or np.any(np.floor(a) != a) \
                or np.any(a < lo) or (hi is not None and np.any(a >= hi)):
            raise ValueError("closed_loop.run: curriculum %s must be an integer in [%d, %s) or [%s] such integers, got %r"
                             % (name, lo, "inf" if hi is None else hi, "B" if B is None else B, v))
        return a.astype(np.int64)
    levels = curriculum.get("levels")
    if isinstance(levels, (bool, np.bool_)) or not isinstance(levels, (int, np.integer)) or levels < 2:
        raise ValueError("closed_loop.run: curriculum levels must be an integer >= 2, got %r" % (levels,))
    start = ints("start", curriculum.get("start", 0), 0, int(levels))
    up, down = (ints(k, curriculum.get(k, 1), 1, 1 << 31) for k in ("up_after", "down_after"))
    when = list(curriculum.get("when", []))
    if when and not metrics:
        raise ValueError("closed_loop.run: curriculum when needs metrics=True (its conditions read the closed episode's metrics row)")
    if len(when) > _lib.CURRICULUM_MAX_COND:
        raise ValueError("closed_loop.run: curriculum when takes at most %d conditions, got %d" % (_lib.CURRICULUM_MAX_COND, len(when)))
    conditions, thresholds = [], []
    for c in when:
        if isinstance(c, str) or len(c) != 4:
            raise ValueError("closed_loop.run: a curriculum condition must be (column, op, threshold, role), got %r" % (c,))
        col, op, thr, role = c
        if col not in _lib.METRICS_LAYOUT:
            raise ValueError("closed_loop.run: unknown curriculum column %r (one of %s)" % (col, ", ".join(_lib.METRICS_LAYOUT)))
        if op not in _lib.CURRICULUM_OPS or role not in _lib.CURRICULUM_ROLES:
            raise ValueError("closed_loop.run: a curriculum condition's op must be one of %s and its role one of %s, got %r and %r"
                             % (", ".join(_lib.CURRICULUM_OPS), ", ".join(_lib.CURRICULUM_ROLES), op, role))
        t = np.asarray(thr, dtype=np.float64) if not isinstance(thr, (str, bool, np.bool_)) else np.array(np.nan)
        if t.ndim > 1 or (t.ndim == 1 and B is not None and t.shape != (B,)) or not np.all(np.isfinite(t)):
            raise ValueError("closed_loop.run: curriculum threshold of %s must be a finite scalar or [%s], got %r" % (col, "B" if B is None else B, thr))
        conditions.append((col, op, role)); thresholds.append(t)
    tops, top_gd = {}, None
    for key in ("timeline", "randomize", "spawn", "ee_path_draw"):   # the timeline first: its end-effector weights decide what a drawn spawn yaw may go with
        if key not in curriculum:
            continue
        kind = CURRICULUM_KINDS[key]; top = curriculum[key]
        if base[kind] is None:
            raise ValueError("closed_loop.run: curriculum %s needs the run's own %s (its level 0)" % (key, key))
        if not isinstance(top, dict) or {"seed", "n"} & set(top):
            raise ValueError("closed_loop.run: curriculum %s must be a dict of the top box's fields (the run's %s gives the seed%s), got %r"
                             % (key, key, " and n" if key in ("timeline", "ee_path_draw") else "", top))
        spec = dict(base[kind], **top)
        if key == "randomize":
            tops[kind] = _randomize_spec(B, spec)
        elif key == "spawn":
            tops[kind] = _spawn_spec(B, spec, terrain, ground_map, top_gd or gd, world)
        elif key == "ee_path_draw":
            b, t = _ee_path_draw_spec(B, T, base[kind]), _ee_path_draw_spec(B, T, spec)
            if not np.array_equal(*np.broadcast_arrays(b["quat"], t["quat"])):
                raise ValueError("closed_loop.run: curriculum ee_path_draw quat must equal the run's (only the boxes move with the level)")
            tops[kind] = t
        else:
            b, t = _timeline_spec(B, gait, base[kind], None), _timeline_spec(B, gait, spec, None)
            for name, k in (("gaits (gait_set)", "gait_set"), ("ee_quat", "quat")):
                if not np.array_equal(np.broadcast_to(b[k], np.broadcast_shapes(np.shape(b[k]), np.shape(t[k]))), np.broadcast_to(t[k], np.broadcast_shapes(np.shape(b[k]), np.shape(t[k])))):
                    raise ValueError("closed_loop.run: curriculum timeline %s must equal the run's (only the boxes, p_gait and weights move with the level)" % name)
            tops[kind] = t
            top_gd = t["gd"] if t["gd"]["ee"] and not b["gd"]["ee"] else None
    if not tops:
        raise ValueError("closed_loop.run: curriculum needs at least one of %s (the boxes its level moves)" % ", ".join(CURRICULUM_KINDS))
    if top_gd is not None and base["spawn"] is not None:   # the run's own spawn, checked against the timeline its top box needs
        _spawn_spec(B, base["spawn"], terrain, ground_map, top_gd, world)
    return dict(levels=int(levels), start=start, up_after=up, down_after=down, conditions=conditions, thresholds=thresholds, tops=tops, gd=top_gd)


@contextlib.contextmanager
def _gait_dev(solver, gd):
    solver.gait_dev_set_templates(gd["names"])
    try:
        yield   # the session's start resets the schedule and loads the timeline once it knows the start time
    finally:
        solver.gait_dev_stop()


@contextlib.contextmanager
def _terrain(solver, terrain):
    prev_lib, prev_robot = solver.sim_get_terrain(), solver.sim_get_robot_terrain()
    try:
        solver.sim_set_robot_terrain(None)
        solver.sim_set_terrain(terrain["tiles"], terrain["cell"])
        solver.sim_set_robot_terrain(terrain["tile"], terrain["origin"])
        yield
    finally:
        solver.sim_set_robot_terrain(None)   # the previous library may have fewer tiles than this run's robots reference
        if prev_lib is None:
            solver.sim_set_terrain(None)
        else:
            solver.sim_set_terrain(**prev_lib)
        if prev_robot is not None:
            solver.sim_set_robot_terrain(**prev_robot)


@contextlib.contextmanager
def _ground_map(solver, rows):
    prev = solver.state_est_get_ground()   # entered after _terrain: the previous map has survived its library change
    try:
        solver.state_est_set_ground(rows["tile"], rows["origin"])
        yield
    finally:
        solver.state_est_set_ground(None)
        if prev is not None:
            solver.state_est_set_ground(**prev)


@contextlib.contextmanager
def _model_payload(solver, model_payload, payload):
    prev_model = solver.get_model_payload()
    try:
        if isinstance(model_payload, str):
            if model_payload != "plant":
                raise ValueError("closed_loop.run: model_payload must be None, \"plant\" or an array [%d, 8], got %r" % (solver.batch, model_payload))
            plant = payload if payload is not None else solver.sim_get_robot_params()["payload"]
            model_payload = np.zeros((solver.batch, 8)) if plant is None else plant
        solver.set_model_payload(model_payload)
        yield
    finally:
        solver.set_model_payload(prev_model)


def _tuning_spec(B, tuning):
    """closed_loop.run's tuning → dict field -> float array shaped as Solver.set_robot_tuning takes it, or "plant"; ValueError when malformed"""
    if not isinstance(tuning, dict):
        raise ValueError("closed_loop.run: tuning must be a dict of robot tuning fields, got %r" % (tuning,))
    out = {}
    for k, v in tuning.items():
        if k not in _lib.TUNING_LAYOUT:
            raise ValueError("closed_loop.run: unknown tuning field %r (one of %s)" % (k, ", ".join(_lib.TUNING_LAYOUT)))
        if isinstance(v, str):
            if v != "plant" or k not in ("friction_mu", "wbc_friction"):
                raise ValueError("closed_loop.run: tuning %s must be numbers%s, got %r" % (k, " or \"plant\"" if k in ("friction_mu", "wbc_friction") else "", v))
            out[k] = v; continue
        w = _lib.TUNING_LAYOUT[k][1]; a = np.asarray(v, dtype=np.float64)
        if a.shape not in ((), (B, w), (B,) if w == 1 else (w,)):
            raise ValueError("closed_loop.run: tuning %s must be a scalar, %s, got shape %s" % (k, "[%d]" % B if w == 1 else "[%d] or [%d, %d]" % (w, B, w), a.shape))
        if not np.all(np.isfinite(a)) or np.any(a <= 0.0 if k in ("friction_mu", "wbc_friction") else a < 0.0):
            raise ValueError("closed_loop.run: tuning %s must be finite and %s" % (k, "> 0" if k in ("friction_mu", "wbc_friction") else ">= 0"))
        out[k] = a
    return out


@contextlib.contextmanager
def _robot_tuning(solver, spec, friction_mu):
    prev = solver.get_robot_tuning()
    try:
        if any(isinstance(v, str) for v in spec.values()):
            plant = friction_mu if friction_mu is not None else solver.sim_get_robot_params()["friction_mu"]
            plant = solver.sim_get_params()["friction_mu"] if plant is None else plant
            spec = {k: (np.broadcast_to(np.asarray(plant, dtype=np.float64), (solver.batch,)) if isinstance(v, str) else v) for k, v in spec.items()}
        solver.set_robot_tuning(spec)
        yield
    finally:
        solver.set_robot_tuning(prev)


EE_FRAMES = ("world", "heading")   # closed_loop.run's ee_frame names, in _lib.EE_FRAME_* order


def _ee_frame_spec(B, ee_frame):
    """closed_loop.run's ee_frame → None ("world", the default: no rows are set) or int32 [B] rows for Solver.set_ee_frame; ValueError when malformed.
    B None: the rows' length is not checked."""
    if ee_frame is None or (isinstance(ee_frame, str) and ee_frame == "world"):
        return None
    if isinstance(ee_frame, str):
        if ee_frame not in EE_FRAMES:
            raise ValueError("closed_loop.run: ee_frame must be \"world\", \"heading\" or [B] of 0 (world) / 1 (heading), got %r" % (ee_frame,))
        return np.full(1 if B is None else B, _lib.EE_FRAME_HEADING, dtype=np.int32)
    a = np.asarray(ee_frame)
    if a.ndim != 1 or (B is not None and a.shape != (B,)) or a.dtype.kind not in "iub" or not np.all((a == 0) | (a == 1)):
        raise ValueError("closed_loop.run: ee_frame must be \"world\", \"heading\" or [%s] of 0 (world) / 1 (heading), got %r" % ("B" if B is None else B, ee_frame))
    return a.astype(np.int32)


def _ee_paths_spec(T, ee_paths):
    """closed_loop.run's ee_paths → None or a list of (t [n], pose [n, 7]) float arrays for Solver.set_ee_paths; ValueError when malformed (the
    library's rules: DESIGN.md §4.20).  T: the handle's time horizon (None: the T/2 gap rule is left to the library)."""
    if ee_paths is None:
        return None
    if isinstance(ee_paths, (str, dict)) or not hasattr(ee_paths, "__len__") or len(ee_paths) == 0:
        raise ValueError("closed_loop.run: ee_paths must be a non-empty list of (t [n], pose [n, 7]), got %r" % (ee_paths,))
    out = []
    for p, item in enumerate(ee_paths):
        try:
            t, pose = item
            t, pose = np.asarray(t, dtype=np.float64), np.asarray(pose, dtype=np.float64)
        except (TypeError, ValueError):
            raise ValueError("closed_loop.run: ee_paths[%d] must be a pair (t [n], pose [n, 7]) of numbers" % p) from None
        if t.ndim != 1 or pose.shape != (len(t), 7) or not 1 <= len(t) <= _lib.EE_PATH_MAX:
            raise ValueError("closed_loop.run: ee_paths[%d] must be (t [n], pose [n, 7]) with 1 <= n <= %d, got shapes %s and %s" % (p, _lib.EE_PATH_MAX, t.shape, pose.shape))
        if not (np.all(np.isfinite(t)) and np.all(np.isfinite(pose))):
            raise ValueError("closed_loop.run: ee_paths[%d] must be finite" % p)
        if not (t[0] > 0.0 and np.all(np.diff(t) > 0.0)):
            raise ValueError("closed_loop.run: ee_paths[%d] times must be > 0 and strictly increasing" % p)
        if T is not None and np.any(np.diff(t) < 0.5 * T):
            raise ValueError("closed_loop.run: ee_paths[%d] waypoints must lie at least time_horizon / 2 = %g s apart" % (p, 0.5 * T))
        if np.any(np.abs(np.linalg.norm(pose[:, 3:7], axis=-1) - 1.0) > 1e-9):
            raise ValueError("closed_loop.run: ee_paths[%d] quaternions (xyzw) must have unit norm (within 1e-9)" % p)
        out.append((t, pose))
    return out


@contextlib.contextmanager
def _ee_paths(solver, paths):
    prev = solver.get_ee_paths()
    try:
        solver.set_ee_paths(paths)
        yield
    finally:
        solver.set_ee_paths(prev)


@contextlib.contextmanager
def _ee_frame(solver, rows):
    prev = solver.get_ee_frame()
    try:
        solver.set_ee_frame(rows)
        yield
    finally:
        solver.set_ee_frame(prev)


@contextlib.contextmanager
def _payload_estimator(solver, params):
    prev_model, prev_params = solver.get_model_payload(), solver.payload_est_get_params()
    try:
        if isinstance(params, dict):
            solver.payload_est_set_params(**params)
        solver.payload_est_reset()
        yield
    finally:
        solver.payload_est_stop()
        solver.set_model_payload(prev_model)
        solver.payload_est_set_params(**prev_params)


@contextlib.contextmanager
def _state_estimator(solver, params, noise):
    prev_params, prev_noise = solver.state_est_get_params(), solver.sim_get_sensor_params()
    try:
        if isinstance(params, dict):
            solver.state_est_set_params(**params)
        if noise is not None:
            solver.sim_set_sensor_params(**(_lib.SENSOR_NOISE_REFERENCE if noise == "reference" else noise))
        yield   # the session's start resets the estimator once it knows the start position
    finally:
        solver.state_est_stop()
        solver.sim_set_sensor_params(**prev_noise)
        solver.state_est_set_params(**prev_params)


@contextlib.contextmanager
def _attitude_filter(solver, params):
    prev_params = solver.attitude_get_params()
    try:
        if isinstance(params, dict):
            solver.attitude_set_params(**params)
        yield   # the session's start resets the filter right before its first reading
    finally:
        solver.attitude_stop()
        solver.attitude_set_params(**prev_params)


@contextlib.contextmanager
def _slip_detector(solver, params):
    prev_params = solver.slip_get_params()
    try:
        if isinstance(params, dict):
            solver.slip_set_params(**params)
        yield   # the session's start resets the detector with the estimator
    finally:
        solver.slip_stop()
        solver.slip_set_params(**prev_params)


@contextlib.contextmanager
def _robot_params(solver, friction_mu, payload):
    prev = solver.sim_get_robot_params()
    solver.sim_set_robot_params(friction_mu=prev["friction_mu"] if friction_mu is None else friction_mu, payload=prev["payload"] if payload is None else payload)
    try:
        yield
    finally:
        solver.sim_set_robot_params(**prev)


def _metrics_episodes(ticks, rs):
    """the most episodes a run of `ticks` 10 ms windows can hold under the respawn spec rs (None: one): a robot respawns only at a window boundary
    after its episode has lasted at least hold windows (on the fall rule) or every (at the limit), whichever is shorter, and at least one window"""
    if rs is None:
        return 1
    if rs.get("on_request"):   # a request may restart a robot at every boundary
        return ticks
    shortest = min([rs["hold_windows"]] * rs["on_fall"] + ([rs["every_ms"] // MPC_PERIOD_MS] if rs["every_ms"] is not None else []))
    return (ticks - 1) // max(shortest, 1) + 1


def _gather(rows, src_rows, ok, idx=None):   # every robot b with ok[b] (bool [B]) takes row idx[b] (None: b) of each src_rows tensor into rows
    import torch
    for a, a0 in zip(rows, src_rows):
        a.copy_(torch.where(ok.view((ok.shape[0],) + (1,) * (a.dim() - 1)), a0 if idx is None else a0[idx], a))


class Snapshot:
    """Every robot of a Session at one window boundary (Session.snapshot; DESIGN.md §4.17): buf, the library's rows (uint8 device tensor), desc, what
    they hold (_lib.RobotStateDesc), rows, device clones of the loop's per-robot rows (Session.rows), k0 [B], each robot's clock origin then, and k, the
    plant step of the boundary (window = k / 10)."""

    def __init__(self, session, buf, desc, rows, k0, k):
        self.session, self.buf, self.desc, self.rows, self.k0, self.k = session, buf, desc, rows, k0, k

    @property
    def window(self):
        return self.k // MPC_PERIOD_MS

    @property
    def nbytes(self):
        """device bytes the snapshot holds: the library's rows and the loop's"""
        return self.buf.numel() + sum(a.numel() * a.element_size() for a in self.rows) + self.k0.numel() * 8


class Session:
    """A closed loop stepped window by window: run's loop, with its live state on the device between windows and per-robot commands from device tensors.

    Session(solver, duration, steer=False, **kw) takes run's keywords; duration fixes the capacities run computes from it (the host-tiled mode schedule's
    horizon, the metrics rows' episodes) and the most windows step may take.  steer=True rolls the device gait schedule on an empty timeline when neither
    commands nor timeline is given, so that command() can steer every robot.  Spec errors raise ValueError here, before any solver call.
    with Session(...) as s: entering sets run's per-run overrides in run's order, reads the start state, saves the start image, begins episode 0 and
    makes the blocking first solve (window 0's MPC tick); leaving restores the overrides in reverse.
    s.step(windows=1) advances that many 10 ms windows and returns their per-window records (run's per-window keys; t a numpy array, the rest device
    tensors [windows, B, ...]), enqueued on s.stream without a synchronisation: wait for s.stream before reading them on another stream.  The session
    keeps no record of earlier chunks.
    s.command(mask, gait=None, cmd_vel=None, ee_goal=None, ee_cmd_vel=None): one command for each masked robot, applied by its first MPC tick after the
    call (Solver.gait_dev_command_dev; DESIGN.md §4.16).
    s.state: the live device tensors (read-only: the loop writes them).  s.finish() closes the open episodes and returns run's end-of-run keys.
    snap = s.snapshot() and s.restore(snap, mask=None, source=None) rewind robots to a window boundary, or branch one robot's state onto others
    (DESIGN.md §4.17); not with respawn, randomize, spawn, timeline or curriculum.
    s.respawn(mask, end=2, at=None) restarts robots at the next boundary (respawn=dict(..., on_request=True); DESIGN.md §4.18).  Sensor noise is a pure function of (seed, robot, plant step k,
    channel): a rewound or branched robot draws fresh noise, so exact replay needs the noise off.
    run(solver, duration, **kw) is Session + one step(windows) + finish()."""

    def __init__(self, solver, duration=1.0, steer=False, **kw):
        unknown = sorted(set(kw) - set(RUN_DEFAULTS))
        if unknown:
            raise TypeError("closed_loop.Session: unknown keyword argument(s) %s" % ", ".join(unknown))
        self.solver, self.duration = solver, duration
        self._o = dict(RUN_DEFAULTS, **kw)
        self._spec = _run_specs(solver, steer, self._o)
        sp, cu = self._spec["sp"], self._spec["cu"]
        spawns = [x for x in (sp, cu["tops"].get("spawn") if cu is not None else None) if x is not None]
        self._yaw_drawn = any("yaw" in x["fields"] and np.any(x["fields"]["yaw"][0] != x["fields"]["yaw"][1]) for x in spawns)
        rs = self._spec["rs"]
        # restarts may place robots on rows of their own: "here", or a request's (DESIGN.md §4.18); the heading then varies as with a drawn yaw
        self._placing = rs is not None and (rs["at"] == "here" or rs["on_request"])
        self._heading_varies = self._yaw_drawn or (rs is not None and rs["at"] == "here")
        self._ee_commanded = set(); self._place_due = rs is not None and rs["at"] == "here"   # whether the next boundary places robots
        self._scope = None; self._open = False; self._finished = False

    # ------------------------------------------------------------------------------------------------------------------------------------ scopes
    def __enter__(self):
        solver, o, p = self.solver, self._o, self._spec
        sp, tn, rz, tl, cu, gd, rs = p["sp"], p["tn"], p["rz"], p["tl"], p["cu"], p["gd"], p["rs"]
        # set in this order, restored in reverse: the estimator starts from the model payload in force, and "plant" reads this run's payload or the handle's
        scope = self._scope = contextlib.ExitStack()
        try:
            if sp is not None:   # restored last: the earlier ranges are set again on the earlier library and robot terrain rows, which give their origins
                scope.enter_context(_ranges(solver, "spawn"))
            if o["terrain"] is not None:
                scope.enter_context(_terrain(solver, o["terrain"]))
            if o["ground_map"] is not None:
                scope.enter_context(_ground_map(solver, o["terrain"] if o["ground_map"] is True else o["ground_map"]))
            if o["model_payload"] is not None:
                scope.enter_context(_model_payload(solver, o["model_payload"], o["payload"]))
            if tn is not None:
                scope.enter_context(_robot_tuning(solver, tn, o["friction_mu"]))
            if p["ef"] is not None:
                scope.enter_context(_ee_frame(solver, p["ef"]))
            if p["ep"] is not None:
                scope.enter_context(_ee_paths(solver, p["ep"]))
            if o["payload_estimator"] is not None:
                scope.enter_context(_payload_estimator(solver, o["payload_estimator"]))
            if o["state_estimator"] is not None:
                scope.enter_context(_state_estimator(solver, o["state_estimator"], o["sensor_noise"]))
            if o["attitude_filter"] is not None:
                scope.enter_context(_attitude_filter(solver, o["attitude_filter"]))
            if o["slip_detector"] is not None:
                scope.enter_context(_slip_detector(solver, o["slip_detector"]))
            if o["friction_mu"] is not None or o["payload"] is not None or rz is not None:
                scope.enter_context(_robot_params(solver, o["friction_mu"], o["payload"]))
            if rz is not None:
                scope.enter_context(_ranges(solver, "episode"))
            if tl is not None:
                scope.enter_context(_ranges(solver, "timeline"))
            if p["pd"] is not None:   # cleared before the ee_paths scope restores the table, which the library refuses while ranges are set
                scope.enter_context(_ranges(solver, "ee_path"))
            if cu is not None:   # cleared first: the ranges go back to their base boxes, then the scopes above restore what they found
                scope.callback(solver.curriculum_set)
            if gd is not None:
                scope.enter_context(_gait_dev(solver, gd))
            if rs is not None:
                scope.callback(solver.robot_image_clear)
            self._start()
        except BaseException:
            scope.__exit__(None, None, None)   # a failed start restores what it had set, as run's scope did
            raise
        self._open = True
        return self

    def __exit__(self, *exc):
        self._open = False
        return self._scope.__exit__(*exc)

    # ------------------------------------------------------------------------------------------------------------------------------------ start
    def _start(self):
        """everything run does before its loop: the fixed values, the ranges, the start state, the start image, episode 0 and the blocking first solve"""
        import torch
        solver, o, p = self.solver, self._o, self._spec
        rs, rz, sp, tl, cu, gd = p["rs"], p["rz"], p["sp"], p["tl"], p["cu"], p["gd"]
        est, se, att, sl, mt = (o[k] is not None for k in ("payload_estimator", "state_estimator", "attitude_filter", "slip_detector", "metrics"))
        gait, cmd_vel, wbc_period_ms, t_start, pushes = o["gait"], o["cmd_vel"], o["wbc_period_ms"], o["t_start"], o["pushes"]
        B = solver.batch; dev = self.device = torch.device(o["torch_device"] or "cuda:%d" % solver._cfg.device)
        n_ms = int(round(self.duration * 1e3)); assert n_ms > 0 and n_ms % MPC_PERIOD_MS == 0, "duration must be a multiple of 10 ms"
        assert MPC_PERIOD_MS % wbc_period_ms == 0, "the WBC period must divide the MPC period"
        cmd_vel = np.asarray(cmd_vel, dtype=np.float64)
        if cmd_vel.shape not in ((4,), (B, 4)):
            raise ValueError("closed_loop.run: cmd_vel must have shape (4,) or (%d, 4), got %s" % (B, cmd_vel.shape))
        if pushes is not None:
            t_on, t_dur, wrench = (np.asarray(a, dtype=np.float64) for a in pushes)
            if t_on.shape != (B,) or t_dur.shape != (B,) or wrench.shape != (B, 12):
                raise ValueError("closed_loop.run: pushes must be (t_on[%d], duration[%d], wrench[%d, 12])" % (B, B, B))
        tops = {} if cu is None else dict(cu["tops"])   # each attached kind's top box, built from this run's values as its base box is
        if rz is not None:   # the ranges: this run's values (entered after _robot_params: the handle's robot params are this run's plant), the named fields' bounds
            EP = {n: i for i, n in enumerate(_lib.EPISODE_LAYOUT)}
            rp = solver.sim_get_robot_params()
            row = np.zeros((B, _lib.EPISODE))
            row[:, EP["friction_mu"]] = solver.sim_get_params()["friction_mu"] if rp["friction_mu"] is None else rp["friction_mu"]
            if rp["payload"] is not None:
                row[:, EP["m_ee"]:EP["m_ee"] + 8] = rp["payload"]
            if pushes is not None:
                row[:, EP["push_t_on"]] = t_on; row[:, EP["push_duration"]] = t_dur; row[:, EP["f_base_x"]:EP["f_base_x"] + 12] = wrench
            row[:, EP["cmd_vel_x"]:EP["cmd_vel_x"] + 4] = cmd_vel
            lo, hi = _box(_lib.EPISODE_LAYOUT, row, rz); solver.episode_set_ranges(lo, hi, rz["seed"])
            if "episode" in tops:
                tops["episode"] = _box(_lib.EPISODE_LAYOUT, row, tops["episode"]); hi = np.maximum(hi, tops["episode"][1])
            if pushes is None and np.any(hi[:, EP["push_duration"]] > 0.0):   # the draws overwrite these rows before the first solve
                t_on, t_dur, wrench = np.zeros(B), np.zeros(B), np.zeros((B, 12)); pushes = (t_on, t_dur, wrench)
        xy_yaw = o["xy_yaw"]
        xy = np.zeros((B, 3)) if xy_yaw is None else np.asarray(xy_yaw, dtype=np.float64).reshape(B, 3)
        if sp is not None:   # the ranges: this run's values (entered after _terrain: the robot terrain rows are this run's), the named columns' bounds
            SP = {n: i for i, n in enumerate(_lib.SPAWN_LAYOUT)}
            rt = solver.sim_get_robot_terrain()
            yaw = xy[:, 2]; yaw = np.where(np.abs(yaw) <= np.pi, yaw, np.remainder(yaw + np.pi, 2.0 * np.pi) - np.pi)   # the same heading within [-pi, pi]
            row = np.zeros((B, _lib.SPAWN)); row[:, SP["tile"]] = -1.0 if rt is None else rt["tile"]; row[:, SP["yaw"]] = yaw
            solver.spawn_set_ranges(*_box(_lib.SPAWN_LAYOUT, row, sp), sp["seed"])
            if "spawn" in tops:
                tops["spawn"] = _box(_lib.SPAWN_LAYOUT, row, tops["spawn"])
        if tl is not None:
            cmd_b = np.broadcast_to(cmd_vel, (B, 4))
            solver.timeline_set_ranges(tl["n"], *_timeline_box(tl, cmd_b, t_start), tl["seed"])
            if "timeline" in tops:
                tops["timeline"] = _timeline_box(tops["timeline"], cmd_b, t_start)
        if p["pd"] is not None:
            solver.ee_path_set_ranges(*_ee_path_box(p["pd"], B), p["pd"]["seed"])
            if "ee_path" in tops:
                tops["ee_path"] = _ee_path_box(tops["ee_path"], B)
        if cu is not None:   # the levels start at the run's start levels; each kind's ranges set above are its level 0
            rows = np.zeros((B, _lib.CURRICULUM))
            rows[:, 0] = cu["start"]; rows[:, 1] = cu["up_after"]; rows[:, 2] = cu["down_after"]
            for i, thr in enumerate(cu["thresholds"]):
                rows[:, 3 + i] = thr
            solver.curriculum_set(cu["levels"], rows, cu["conditions"])
            for kind, (lo, hi) in tops.items():
                solver.curriculum_attach(kind, lo, hi)
        stream = self.stream = torch.cuda.Stream(device=dev); s = self._s = stream.cuda_stream
        f64 = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=dev)
        i32 = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.int32), device=dev)
        self.B, self.windows, self.t_start, self._wbc, self._n_ms, self._k = B, n_ms // MPC_PERIOD_MS, t_start, wbc_period_ms, n_ms, 0
        self._est, self._se, self._att, self._sl, self._mt, self._tops = est, se, att, sl, mt, tops

        # ---- plant state, the first measurement, the controller's members (host → device once) ----
        q0, v0 = solver.sim_standing_state(xy)
        t_obs0 = t_start - wbc_period_ms * 1e-3   # observation clock of `starting`; the first update brings it to t_start, the plant's clock
        if gd is None:
            ev, md, ne = _schedules(gait, B, t_start, t_obs0, t_start + self.duration + solver.time_horizon + 1.0)
        else:   # the first gait step writes the rows
            ev, md, ne = np.zeros((B, EMAX)), np.full((B, EMAX + 1), 15, dtype=np.int32), np.zeros(B, dtype=np.int32)
        with torch.cuda.stream(stream):
            q = self.q = f64(q0); v = self.v = f64(v0); rbd = self.rbd = torch.zeros((B, RBD), dtype=torch.float64, device=dev)
            contact = self.contact = torch.zeros(B, dtype=torch.int32, device=dev)
            self.sim_st = torch.zeros_like(contact); self.hw_st = torch.zeros_like(contact); self.ctl_st = torch.zeros_like(contact)
            self.acc_st = torch.zeros_like(contact)
            self.effort = torch.zeros((B, 18), dtype=torch.float64, device=dev); self.jpos = torch.zeros_like(self.effort); self.jvel = torch.zeros_like(self.effort)
            if se:   # the controller's measurement: the estimator's rbd_est in place of the plant's rbd
                v_prev = self.v_prev = torch.zeros_like(v); sensors = self.sensors = torch.zeros((B, SENSORS), dtype=torch.float64, device=dev)
                rbd_est = self.rbd_est = torch.zeros_like(rbd)
                self.se_st = torch.zeros_like(contact); v_prev.copy_(v)
                if att:
                    self.at_st = torch.zeros_like(contact)
                if sl:   # the estimator reads the trusted stance mask in place of the plant's contact mask
                    stance = self.stance = torch.zeros_like(contact); self.slip = torch.zeros_like(contact); self.sl_st = torch.zeros_like(contact)
                    self.slip_acc = torch.zeros_like(contact)
        stream.synchronize()
        solver.sim_step_dev(1e-6, self.effort, q, v, rbd, contact, self.sim_st, s)   # a 1 us physics step with zero effort reads the first measured state
        meas = rbd
        if se:
            solver.sim_read_sensors_dev(1e-6, -1, q, v, v_prev, sensors, s)
            stream.synchronize()
            solver.state_est_reset(q0[:, 0:3])
            if att:
                solver.attitude_reset()
                solver.attitude_step_dev(1e-6, sensors, self.at_st, s)   # the first call after the reset takes the reading
            self.se_contact = contact
            if sl:
                solver.slip_reset()
                solver.slip_step_dev(1e-6, sensors, contact, stance, self.slip, self.sl_st, s)   # passes the contact mask through: the estimator has had no call yet
                self.se_contact = stance
            solver.state_est_step_dev(1e-6, sensors, self.se_contact, rbd_est, self.se_st, s)   # the first call after the reset places the feet
            meas = rbd_est
        self.meas = meas
        stream.synchronize()
        rbd_h = rbd.cpu().numpy()
        x_obs0 = solver.centroidal_state_from_rbd(meas.cpu().numpy())
        self._start_out = dict(start_base=np.c_[q0[:, 0:3], q0[:, 3:6]], start_ee=rbd_h[:, 48:55])
        with torch.cuda.stream(stream):
            t_obs = self.t_obs = f64(np.full(B, t_obs0)); x_obs = self.x_obs = f64(x_obs0)
            self.joint_cmd = torch.zeros((B, 18, 5), dtype=torch.float64, device=dev); self.arm_pos = torch.zeros((B, 6), dtype=torch.float64, device=dev)
            self.last_time = f64(np.full(B, t_obs0))
            self.cmd54 = torch.zeros((B, 54), dtype=torch.float64, device=dev)
            cmd7 = self.cmd7 = torch.zeros((B, 7), dtype=torch.float64, device=dev); cmd7[:, :4] = f64(cmd_vel[None, :4] if cmd_vel.ndim == 1 else cmd_vel)
            self.last_ee = f64(solver.initial_ee_target()); self.ee_state = torch.zeros((B, 7), dtype=torch.float64, device=dev)
            prob = self.prob = dict(t0=t_obs, x0=x_obs, n_events=i32(ne), event_times=f64(ev), modes=i32(md),
                                    n_target=torch.zeros(B, dtype=torch.int32, device=dev), target_times=torch.zeros((B, KMAX), dtype=torch.float64, device=dev),
                                    target_states=torch.zeros((B, KMAX, TARGET), dtype=torch.float64, device=dev))
            self.period = f64(np.full(B, wbc_period_ms * 1e-3)); self.hw_period = f64(np.full(B, 1e-3)); self.hw_time = torch.zeros(B, dtype=torch.float64, device=dev)
            ticks = self.windows
            if est:   # the model payload rows committed at the current window's MPC tick
                self.est_st = torch.zeros_like(contact); self.tick_pl = torch.zeros((B, 8), dtype=torch.float64, device=dev)
            if gd is not None:   # the current window's gait step: active template, mode, target kind
                self.gait_st = torch.zeros_like(contact); self.tick_gait = torch.zeros_like(contact); self.tick_mode = torch.zeros_like(contact)
                self.tick_kind = torch.zeros_like(contact)
                self.cmd_st = torch.zeros_like(contact); self.cmd_acc = torch.zeros_like(contact); self._commanded = False
            push = self.push = None
            if pushes is not None:   # robot b is pushed in plant step k (start k ms after the start) when t_on <= k ms < t_on + duration
                push = self.push = dict(on=f64(t_on * 1e3 - 1e-6), off=f64((t_on + t_dur) * 1e3 - 1e-6), wrench=f64(wrench),
                                        zero=torch.zeros((B, 12), dtype=torch.float64, device=dev), now=torch.zeros((B, 12), dtype=torch.float64, device=dev))
        stream.synchronize()
        if gd is not None:
            solver.gait_dev_reset(gd["gait"], np.full(B, t_start))
            solver.gait_dev_set_commands(t_start + gd["t"], gd["tmpl"], gd["cmd_vel"], **gd["ee"])
        solver.hw_set_delay(HW_DELAY)

        # the loop's per-robot rows: own, the rows a respawn returns to the start image, then the rows a snapshot holds as well (self.rows, completed once
        # the accumulator exists): the push rows, the metrics accumulator, the pending commands' status, the current window's MPC tick rows and its
        # status accumulators (a snapshot of window 0 is taken after that window's tick)
        self.own = [q, v, rbd, contact, t_obs, x_obs, self.joint_cmd, self.arm_pos, self.last_time, self.cmd54, cmd7, self.last_ee, prob["n_events"],
                    prob["event_times"], prob["modes"], prob["n_target"], prob["target_times"], prob["target_states"]] + \
                   ([v_prev, sensors, rbd_est] if se else []) + ([stance] if sl else [])
        self.path_state = None
        if p["ep"] is not None or p["pd"] is not None:   # each robot's end-effector path row (index -1: none), the target call's in-out row beside last_ee
            with torch.cuda.stream(stream):
                self.path_state = torch.zeros((B, _lib.EE_PATH_STATE), dtype=torch.float64, device=dev); self.path_state[:, 0] = -1.0
            self.own.append(self.path_state)
        self.k0 = None   # each robot's clock origin (plant step): with respawn, or once a restore has happened; the global k otherwise
        if rs is not None:   # the start image: the library's rows and the loop's own, then one restore of every robot through the cold path of every later one
            solver.robot_image_save()
            with torch.cuda.stream(stream):
                self.start = [a.clone() for a in self.own]
                self.k0 = torch.zeros(B, dtype=torch.int64, device=dev); self.dk = torch.zeros_like(self.k0)   # each robot's episode start (plant step), and k - k0
                episode = self.episode = torch.zeros(B, dtype=torch.int32, device=dev); self.fall_count = torch.zeros_like(episode)
                self.fallen = torch.zeros_like(episode); self.due = torch.ones_like(episode)
                if mt or cu is not None:   # the fall part of due: why a closed episode ended
                    self.due_fall = torch.zeros_like(episode); self.mt_end = torch.zeros_like(episode)
                if cu is not None:   # each robot's level, and the level of each episode it began
                    self.cu_level = i32(np.broadcast_to(cu["start"], (B,)))
                    self.ep_level = torch.full((B, _metrics_episodes(ticks, rs)), -1, dtype=torch.int32, device=dev); self._level_begun(self.due)
            solver.robot_image_restore_dev(self.due, s)
        if mt:   # every robot's open episode (zeros: open and empty) and its closed rows
            with torch.cuda.stream(stream):
                self.mt_acc = torch.zeros((B, _lib.METRICS_ACC), dtype=torch.float64, device=dev)
                self.mt_out = torch.full((B, _metrics_episodes(ticks, rs), _lib.METRICS), np.nan, dtype=torch.float64, device=dev)
        self.rows = self.own + ([push["on"], push["off"], push["wrench"]] if push is not None else []) + ([self.mt_acc] if mt else []) + \
            ([self.cmd_acc, self.tick_gait, self.tick_mode, self.tick_kind] if gd is not None else []) + ([self.tick_pl] if est else []) + \
            [self.acc_st] + ([self.slip_acc] if sl else [])
        with torch.cuda.stream(stream):
            self.restore_st = torch.zeros(B, dtype=torch.int32, device=dev)   # a restore's status (ST_RESTORE for an invalid source)

        if self._placing:   # the rows restarts place robots on, counted from the run's start origins, and every episode's spawn row on the device
            rt = solver.sim_get_robot_terrain(); self.sp_rows = None
            yaw = xy[:, 2]; yaw = np.where(np.abs(yaw) <= np.pi, yaw, np.remainder(yaw + np.pi, 2.0 * np.pi) - np.pi)
            start_row = np.zeros((B, _lib.SPAWN)); start_row[:, 0] = -1.0 if rt is None else rt["tile"]; start_row[:, 3] = yaw
            with torch.cuda.stream(stream):
                self.sp_origin = f64(np.zeros((B, 2)) if rt is None else rt["origin"]); self.start_row = f64(start_row)
                self.pl_rows = torch.zeros((B, _lib.SPAWN), dtype=torch.float64, device=dev); self.pl_st = torch.zeros_like(contact)
                self.sp_rec = torch.full((B, _metrics_episodes(ticks, rs), _lib.SPAWN), np.nan, dtype=torch.float64, device=dev)
                self.pl_any = torch.zeros(1, dtype=torch.int32, device=dev)
                self._at_default = 1 if rs["at"] == "here" else 0   # each robot's next restart: 0 start (or the spawn's draw), 1 here, 2 a request's row
                self.at_mode = torch.full((B,), self._at_default, dtype=torch.int32, device=dev)
                if rs["on_request"]:
                    self.req = torch.zeros_like(contact); self.req_end = torch.full_like(contact, 2); self.req_rows = torch.zeros_like(self.pl_rows)
            self._place_link = p["sp"]["link"] if sp is not None else (_lib.SPAWN_GROUND_MAP if o["ground_map"] is True else 0)

        if rz is not None or sp is not None or tl is not None or p["pd"] is not None:   # every robot's first episode begins right before the first solve (after the restore of the start image)
            with torch.cuda.stream(stream):
                self.ep_rows = torch.zeros((B, _lib.EPISODE), dtype=torch.float64, device=dev) if rz is not None else None
                self.sp_rows = torch.zeros((B, _lib.SPAWN), dtype=torch.float64, device=dev) if sp is not None else None
                self.tl_rows = torch.zeros((B, tl["n"], _lib.TIMELINE_CMD), dtype=torch.float64, device=dev) if tl is not None else None
                self.pd_rows = torch.zeros((B, _lib.EE_PATH_MAX, 8), dtype=torch.float64, device=dev) if p["pd"] is not None else None
                if rs is None:
                    self._begin(torch.ones(B, dtype=torch.int32, device=dev), torch.zeros(B, dtype=torch.int32, device=dev))
                else:
                    self._begin(self.due, self.episode)
        if self._placing:
            with torch.cuda.stream(stream):
                self._record_spawn(self.due, None)
                if rs["on_request"]:   # the start restored every robot; from here on due holds the robots that restart at the next boundary
                    self.due.zero_()

        with torch.cuda.stream(stream):
            self._mpc_tick(); stream.synchronize()          # QMController::starting: one blocking solve before the loop

    # ------------------------------------------------------------------------------------------------------------------------------------ the loop's parts
    def _mpc_tick(self):
        solver, s, gd, prob = self.solver, self._s, self._spec["gd"], self.prob
        if self._est:
            solver.payload_est_commit_dev(s); solver.get_model_payload_dev(self.tick_pl, s)
        self.ee_state.copy_(self.meas[:, 48:55])
        if gd is None:
            solver.target_trajectories_dev(0, self.cmd7, self.t_obs, self.x_obs, self.ee_state, self.last_ee, prob["n_target"], prob["target_times"], prob["target_states"], s)
        else:   # the step's target kinds go straight to the target call, and stay in the record
            solver.gait_dev_step_dev(self.t_obs, prob, self.cmd7, self.tick_gait, self.tick_mode, self.gait_st, s, target_kind=self.tick_kind)
            self.acc_st.bitwise_or_(self.gait_st)
            if self._commanded:   # the status of the commands this step applied goes into the window it opens
                self.acc_st.bitwise_or_(self.cmd_acc); self.cmd_acc.zero_(); self._commanded = False
            solver.target_trajectories_dev(self.tick_kind, self.cmd7, self.t_obs, self.x_obs, self.ee_state, self.last_ee, prob["n_target"], prob["target_times"],
                                           prob["target_states"], s, **({} if self.path_state is None else dict(path_state=self.path_state)))
        solver.mpc_solve_dev(prob, s)

    def _respawn(self, k):   # the robots due restart at window boundary k: their episode closes, their level moves, then the library's rows, the loop's, their new plant
        solver, s, cu, due, rs = self.solver, self._s, self._spec["cu"], self.due, self._spec["rs"]
        if self._mt or cu is not None:
            self.mt_end.copy_(self.due_fall).neg_().add_(2)   # 1: the fall rule, 2: every
            if rs["on_request"]:   # a request's end, where the fall rule did not end the episode
                self.mt_end.copy_(self.mt_end.where(self.due_fall.bool() | ~self.req.bool(), self.req_end))
        if self._mt:
            solver.metrics_close_dev(due, self.mt_end, self.episode, self.mt_acc, self.mt_out, self.acc_st, s)
        if cu is not None:   # reads the row the close just wrote; writes the ranges the draws of _begin() read
            solver.curriculum_update_dev(due, self.mt_end, self.episode, self.mt_out if self._mt else None, self.cu_level, self.acc_st, s)
        placed = None
        if self._place_due:   # the rows of the robots placed here, read from the plant before the restore: here, then a request's own rows
            m = due.bool()
            here = (m & (self.at_mode == 1)).to(due.dtype); placed = (m & (self.at_mode >= 1)).to(due.dtype)
            solver.spawn_here_dev(here, self.rbd, self.start[0], self.sp_origin, self.pl_rows, s)
            if rs["on_request"]:
                _gather([self.pl_rows], [self.req_rows], m & (self.at_mode == 2))
        solver.robot_image_restore_dev(due, s)
        m = due.bool()
        _gather(self.own + [self.k0], self.start + [k], m)   # their rows return to the start, their clock origin to k
        self.episode.add_(due); self.fall_count.masked_fill_(m, 0)
        if cu is not None:
            self._level_begun(due)
        self._begin(due, self.episode, placed)
        if self._placing:
            self._record_spawn(due, placed)
            self.at_mode.fill_(self._at_default)
            self._place_due = rs["at"] == "here"
            if rs["on_request"]:
                self.req.zero_()

    def _level_begun(self, mask):   # the masked robots begin their episode at their current level
        import torch
        rows = torch.arange(self.B, device=self.device); e = self.episode.long()
        self.ep_level[rows, e] = torch.where(mask.bool(), self.cu_level, self.ep_level[rows, e])

    def _begin(self, mask, idx, placed=None):   # the masked robots begin episode idx: their plant's draw, their spawn or place, their command timeline, their path
        p, solver, s = self._spec, self.solver, self._s
        if p["rz"] is not None:
            self._draw(mask, idx)
        if p["sp"] is not None:   # new ground under them, their start state there
            drawn = mask if placed is None else (mask.bool() & ~placed.bool()).to(mask.dtype)
            solver.spawn_sample_dev(drawn, idx, self.sp_rows, self.q, self.v, self.rbd, self.contact, self.x_obs, self.last_ee, self.rbd_est if self._se else None,
                                    p["sp"]["link"], s)
        if placed is not None:   # the placed robots stand on their rows; a rejected row leaves the robot at its restored start and goes into the window's status
            solver.spawn_place_dev(placed, self.pl_rows, self.sp_origin, self.q, self.v, self.rbd, self.contact, self.x_obs, self.last_ee,
                                   self.rbd_est if self._se else None, self.pl_st, self._place_link, s)
            self.acc_st.bitwise_or_(self.pl_st)
        if p["tl"] is not None:
            solver.timeline_sample_dev(mask, idx, self.tl_rows, s)
        if p["pd"] is not None:   # last: its pending start is applied after the timeline's rows due on the first tick (the restore dropped any pending command)
            solver.ee_path_sample_dev(mask, idx, self.pd_rows, s)

    def _record_spawn(self, mask, placed):   # the masked robots' new episode's spawn row: placed, drawn, or the start's; NaN where a place was rejected
        import torch
        row = self.start_row if self.sp_rows is None else self.sp_rows
        if placed is not None:
            ok = placed.bool() & (self.pl_st == 0)
            row = torch.where(ok[:, None], self.pl_rows, torch.where(placed.bool()[:, None], torch.full_like(row, np.nan), row))
            self.pl_any.bitwise_or_(ok.any().to(torch.int32))
        b = torch.arange(self.B, device=self.device); e = self.episode.long()
        self.sp_rec[b, e] = torch.where(mask.bool()[:, None], row, self.sp_rec[b, e])

    def _draw(self, mask, idx):   # the masked robots draw episode idx: the plant rows on the device, then the loop's cmd_vel and push rows from the drawn row
        ep_rows, push = self.ep_rows, self.push
        self.solver.episode_sample_dev(mask, idx, ep_rows, self._spec["rz"]["link"], self._s)
        m = mask.bool()
        _gather([self.cmd7[:, :4]], [ep_rows[:, 23:27]], m)
        if push is not None:
            on = ep_rows[:, 9] * 1e3 - 1e-6; off = (ep_rows[:, 9] + ep_rows[:, 10]) * 1e3 - 1e-6
            _gather([push["on"], push["off"], push["wrench"]], [on, off, ep_rows[:, 11:23]], m)

    # ------------------------------------------------------------------------------------------------------------------------------------ public
    def step(self, windows=1):
        """Advance `windows` 10 ms windows → their records: t [windows] (numpy, the window ends), and device tensors base [windows, B, 6], ee, status
        and the optional records of run, row i for the session's window (done + i).  Enqueued on self.stream; no synchronisation."""
        import torch
        if not self._open or self._finished:
            raise ValueError("closed_loop.Session.step: the session is not open (enter it with `with`; finish() ends it)")
        if isinstance(windows, (bool, np.bool_)) or not isinstance(windows, (int, np.integer)) or windows < 1:
            raise ValueError("closed_loop.Session.step: windows must be an integer >= 1, got %r" % (windows,))
        i0 = self._k // MPC_PERIOD_MS
        if i0 + windows > self.windows:
            raise ValueError("closed_loop.Session.step: %d windows past window %d exceed the session's %d (its duration, %g s)" % (windows, i0, self.windows, self.duration))
        solver, s, p, B, dev = self.solver, self._s, self._spec, self.B, self.device
        rs, cu, gd, se, sl, est, mt, att = p["rs"], p["cu"], p["gd"], self._se, self._sl, self._est, self._mt, self._att
        q, v, rbd, contact, acc_st, push, sim_timer = self.q, self.v, self.rbd, self.contact, self.acc_st, self.push, self._o["sim_timer"]
        n = windows
        with torch.cuda.stream(self.stream):
            rec = dict(t=self.t_start + np.arange(i0 + 1, i0 + n + 1) * MPC_PERIOD_MS * 1e-3, base=torch.zeros((n, B, 6), dtype=torch.float64, device=dev),
                       ee=torch.zeros((n, B, 7), dtype=torch.float64, device=dev), status=torch.zeros((n, B), dtype=torch.int32, device=dev))
            if est:   # row i: the rows of window i's MPC tick
                rec["payload_est"] = torch.zeros((n, B, 8), dtype=torch.float64, device=dev)
            if se:
                rec["base_est"] = torch.zeros((n, B, 6), dtype=torch.float64, device=dev)
            if sl:
                rec["slip"] = torch.zeros((n, B), dtype=torch.int32, device=dev)
            if gd is not None:
                for key in ("gait", "mode", "target_kind"):
                    rec[key] = torch.zeros((n, B), dtype=torch.int32, device=dev)
                rec["ee_target"] = torch.zeros((n, B, 7), dtype=torch.float64, device=dev)
            if rs is not None:
                rec["episode"] = torch.zeros((n, B), dtype=torch.int32, device=dev); rec["fallen"] = torch.zeros_like(rec["episode"])
                if cu is not None:
                    rec["curriculum_level"] = torch.zeros_like(rec["episode"])
            for k in range(self._k, self._k + n * MPC_PERIOD_MS):
                if k % MPC_PERIOD_MS == 0 and k > 0:
                    if rs is not None:
                        self._respawn(k)
                    self._mpc_tick()
                if k % self._wbc == 0:
                    solver.update_dev(self.meas, self.period, self.t_obs, self.x_obs, self.joint_cmd, self.arm_pos, self.last_time, self.cmd54, self.ctl_st, s)
                    acc_st.bitwise_or_(self.ctl_st)
                if self.k0 is None:
                    self.hw_time.fill_(self.t_start + k * 1e-3)
                else:   # the robot's episode clock
                    torch.sub(self.k0, k, out=self.dk).neg_(); self.hw_time.copy_(self.dk).mul_(1e-3).add_(self.t_start)
                self.jpos.copy_(q[:, 6:]); self.jvel.copy_(v[:, 6:])
                solver.hw_write_dev(self.hw_time, self.hw_period, self.joint_cmd, self.jpos, self.jvel, self.effort, self.hw_st, s)
                if se:
                    self.v_prev.copy_(v)
                if sim_timer:
                    sim_timer(True)
                if push is not None:
                    kk = k if self.k0 is None else self.dk   # plant steps since the episode's start
                    torch.where(((push["on"] <= kk) & (push["off"] > kk))[:, None], push["wrench"], push["zero"], out=push["now"])
                solver.sim_step_dev(1e-3, self.effort, q, v, rbd, contact, self.sim_st, s, wrench=None if push is None else push["now"])
                if sim_timer:
                    sim_timer(False)
                acc_st.bitwise_or_(self.hw_st).bitwise_or_(self.sim_st)
                if se:
                    solver.sim_read_sensors_dev(1e-3, k, q, v, self.v_prev, self.sensors, s)
                    if att:
                        solver.attitude_step_dev(1e-3, self.sensors, self.at_st, s)
                        acc_st.bitwise_or_(self.at_st)
                    if sl:
                        solver.slip_step_dev(1e-3, self.sensors, contact, self.stance, self.slip, self.sl_st, s)
                        acc_st.bitwise_or_(self.sl_st); self.slip_acc.bitwise_or_(self.slip)
                    solver.state_est_step_dev(1e-3, self.sensors, self.se_contact, self.rbd_est, self.se_st, s)
                    acc_st.bitwise_or_(self.se_st)
                if est:
                    solver.payload_est_step_dev(1e-3, self.effort, self.meas, self.est_st, s)
                    acc_st.bitwise_or_(self.est_st)
                if mt:   # the plant's truth after the step, on the robot's episode clock, with the window's status so far
                    solver.metrics_step_dev(1e-3, rbd, contact, self.effort, self.cmd7, self.prob["n_target"], self.prob["target_times"], self.prob["target_states"],
                                            self.hw_time, acc_st, self.mt_acc, kind=None if gd is None else self.tick_kind, rbd_est=self.rbd_est if se else None, stream=s)
                if (k + 1) % MPC_PERIOD_MS == 0:
                    i = (k + 1) // MPC_PERIOD_MS - 1 - i0
                    rec["base"][i, :, 0:3] = rbd[:, 3:6]; rec["base"][i, :, 3:6] = rbd[:, 0:3]; rec["ee"][i] = rbd[:, 48:55]; rec["status"][i] = acc_st; acc_st.zero_()
                    if est:
                        rec["payload_est"][i] = self.tick_pl
                    if se:
                        rec["base_est"][i, :, 0:3] = self.rbd_est[:, 3:6]; rec["base_est"][i, :, 3:6] = self.rbd_est[:, 0:3]
                    if sl:
                        rec["slip"][i] = self.slip_acc; self.slip_acc.zero_()
                    if gd is not None:   # the window's gait step and the target in force after its target call
                        rec["gait"][i] = self.tick_gait; rec["mode"][i] = self.tick_mode; rec["target_kind"][i] = self.tick_kind
                        rec["ee_target"][i] = self.prob["target_states"][:, 1, 30:37]
                    if rs is not None:
                        solver.fall_detect_dev(rbd, self.fall_count, self.fallen, rs["z_min"], rs["tilt_max"], s)
                        rec["episode"][i] = self.episode; rec["fallen"][i] = self.fallen
                        if cu is not None:
                            rec["curriculum_level"][i] = self.cu_level
                        d = self.fall_count >= rs["hold_windows"] if rs["on_fall"] else torch.zeros_like(self.fallen, dtype=torch.bool)
                        if mt or cu is not None:
                            self.due_fall.copy_(d)
                        if rs["every_ms"] is not None:
                            d |= (k + 1 - self.k0) >= rs["every_ms"]
                        if rs["on_request"]:
                            d |= self.req.bool()
                        self.due.copy_(d)
        self._k += n * MPC_PERIOD_MS
        return rec

    def command(self, mask, gait=None, cmd_vel=None, ee_goal=None, ee_cmd_vel=None, ee_path=None):
        """One command for each robot with mask [B] set, from device tensors (host arrays are copied): gait [B] template ids (an index of
        self.gait_templates, -1: none), cmd_vel [B, 4], ee_goal [B, 7] (position, quaternion xyzw of unit norm, world frame) and ee_cmd_vel [B, 3], NaN
        rows meaning none; a row carries at most one of cmd_vel, ee_goal and ee_cmd_vel.  The rows take the semantics of a commands timeline row due at
        the robot's first MPC tick after this call: the tick at the start of the next step (before the first step, the one that opens window 1).  A
        later command before that tick replaces an earlier one; a robot that respawns at that boundary drops it.  A rejected row (checked on the device
        with the timeline's rules) is not applied and sets _lib.ST_COMMAND in that window's record status.  Enqueued on self.stream after the work
        the caller's current stream holds (the tensors may come from it), no synchronisation.  ValueError without the device gait schedule (steer, commands or timeline), on wrong shapes, and for end-effector commands in
        a session that draws spawn yaws.  ee_path [B]: integer path ids of the session's ee_paths (-1: none), which start that path (DESIGN.md §4.20);
        ValueError without ee_paths."""
        import torch
        if self._spec["gd"] is None:
            raise ValueError("closed_loop.Session.command: needs the device gait schedule (steer=True, commands or timeline)")
        B = getattr(self.solver, "batch", None)
        for name, a, shape in (("mask", mask, (B,)), ("gait", gait, (B,)), ("cmd_vel", cmd_vel, (B, 4)), ("ee_goal", ee_goal, (B, 7)), ("ee_cmd_vel", ee_cmd_vel, (B, 3)),
                               ("ee_path", ee_path, (B,))):
            if a is not None and tuple(np.shape(a)) != shape:
                raise ValueError("closed_loop.Session.command: %s must have shape %s, got %s" % (name, shape, tuple(np.shape(a))))
        if ee_path is not None and self._spec["ep"] is None:
            raise ValueError("closed_loop.Session.command: ee_path needs the session's ee_paths")
        if ee_path is not None and (ee_path.dtype.is_floating_point or ee_path.dtype == torch.bool if isinstance(ee_path, torch.Tensor) else np.asarray(ee_path).dtype.kind not in "iu"):
            raise ValueError("closed_loop.Session.command: ee_path must hold integer path ids (-1: none), got %r" % (ee_path,))
        names = _ee_names(ee_goal is not None or ee_cmd_vel is not None, ee_path is not None)
        ee_world = self._ee_to_world(mask, names is not None)
        if self._heading_varies and ee_world:
            raise ValueError("closed_loop.Session.command: %s to world-frame robots cannot go with a drawn spawn yaw or a restart \"here\" "
                             "(their world-frame goals assume the robot faces +x)" % names)
        if not self._open or self._finished:
            raise ValueError("closed_loop.Session.command: the session is not open (enter it with `with`; finish() ends it)")
        self._wait_caller()
        put = self._put
        with torch.cuda.stream(self.stream):
            m = put(mask, torch.int32, (B,), 0); tmpl = put(gait, torch.int32, (B,), -1); vel = put(cmd_vel, torch.float64, (B, 4), np.nan)
            goal = put(ee_goal, torch.float64, (B, 7), np.nan); eev = put(ee_cmd_vel, torch.float64, (B, 3), np.nan)
            has_goal, has_eev = ~torch.isnan(goal).all(-1), ~torch.isnan(eev).all(-1)   # a partly NaN row is a command the check rejects
            kind = torch.where(has_goal, _lib.TARGET_EE_GOAL, torch.where(has_eev, _lib.TARGET_EE_CMD_VEL, -1))
            ee = torch.where(has_goal[:, None], goal, 0.0); ee[:, :3] = torch.where(has_eev[:, None], eev, ee[:, :3])
            n_ee = has_goal.int() + has_eev.int()
            if ee_path is not None:   # a path id below -1 is a path index the check rejects
                path = put(ee_path, torch.float64, (B,), -1.0); has_path = path != -1.0
                kind = torch.where(has_path, _lib.TARGET_EE_PATH, kind); ee[:, 0] = torch.where(has_path, path, ee[:, 0]); n_ee = n_ee + has_path.int()
            kind = torch.where(n_ee > 1, -2, kind).to(torch.int32)   # more than one: a kind the check rejects
            self.solver.gait_dev_command_dev(m, tmpl, vel, kind, ee, self.cmd_st, self._s)
            self.cmd_acc.bitwise_or_(self.cmd_st)
        self._commanded = True
        if ee_world:
            self._ee_commanded.add(names)

    def respawn(self, mask, end=2, at=None):
        """Restart each robot with mask [B] set at the next window boundary, before its MPC tick, through run's respawn path (DESIGN.md §4.18); needs
        respawn=dict(..., on_request=True).  end: why its episode ended, 1 (failure) or 2 (ended alive), a scalar or [B]: the metrics row's end and the
        curriculum's fail / pass (the fall rule's 1 wins where it also restarts the robot).  at: None (the respawn spec's at), "start", "here", or [B, 4]
        spawn rows (_lib.SPAWN_LAYOUT) counted from the run's start origins; a row the device rejects leaves the robot at its restored start pose and
        sets _lib.ST_SPAWN in the record of the window the next tick opens.  A later request before the boundary replaces an earlier one; state["due"]
        shows the merged mask.  mask and rows as command takes them (device tensors, enqueued on self.stream after the caller's current stream, no
        synchronisation); an end tensor's values are checked on the host.  ValueError, before any write, on wrong shapes or values, without on_request,
        and for "here" or rows where run refuses at="here"."""
        import torch
        rs, B = self._spec["rs"], getattr(self.solver, "batch", None)
        if rs is None or not rs["on_request"]:
            raise ValueError("closed_loop.Session.respawn: needs respawn=dict(..., on_request=True)")
        if tuple(np.shape(mask)) != (B,):
            raise ValueError("closed_loop.Session.respawn: mask must have shape (%s,), got %s" % (B, tuple(np.shape(mask))))
        if isinstance(end, (bool, np.bool_)) or tuple(np.shape(end)) not in ((), (B,)):
            raise ValueError("closed_loop.Session.respawn: end must be 1 or 2, a scalar or [%s], got %r" % (B, end))
        e = end.detach().cpu().numpy() if isinstance(end, torch.Tensor) else np.asarray(end)
        if e.dtype.kind not in "iuf" or not np.all(np.isin(e, (1, 2))):
            raise ValueError("closed_loop.Session.respawn: end must be 1 (failure) or 2 (ended alive), got %r" % (end,))
        rows = None
        if at is None:
            code = 1 if rs["at"] == "here" else 0
        elif isinstance(at, str):
            if at not in RESPAWN_AT:
                raise ValueError("closed_loop.Session.respawn: at must be None, \"start\", \"here\" or [%s, 4] spawn rows, got %r" % (B, at))
            code = RESPAWN_AT.index(at)
        else:
            if tuple(np.shape(at)) != (B, _lib.SPAWN):
                raise ValueError("closed_loop.Session.respawn: at rows must have shape (%s, %d), got %s" % (B, _lib.SPAWN, tuple(np.shape(at))))
            code, rows = 2, at
        if code:
            why = _here_refusal(False, self._spec["gd"], self._o["curriculum"], self._o["ground_map"], self._spec["world"])
            if why is None and self._ee_commanded:
                names = _ee_names(any("ee_goal" in n for n in self._ee_commanded), any("ee_path" in n for n in self._ee_commanded))
                why = "%s commands to world-frame robots (their world-frame goals assume the robot faces +x)" % names
            if why is not None:
                raise ValueError("closed_loop.Session.respawn: a restart \"here\" or on given rows cannot go with %s" % why)
        if not self._open or self._finished:
            raise ValueError("closed_loop.Session.respawn: the session is not open (enter it with `with`; finish() ends it)")
        self._wait_caller()
        with torch.cuda.stream(self.stream):
            m = self._put(mask, torch.int32, (B,), 0).bool()
            self.due.bitwise_or_(m.to(self.due.dtype)); self.req.bitwise_or_(m.to(self.req.dtype))
            self.req_end.copy_(torch.where(m, torch.as_tensor(np.broadcast_to(e, (B,)).astype(np.int32), device=self.device), self.req_end))
            self.at_mode.masked_fill_(m, code)
            if rows is not None:
                _gather([self.req_rows], [self._put(rows, torch.float64, (B, _lib.SPAWN), 0.0)], m)
        if code:
            self._place_due = True; self._heading_varies = True

    def _ee_to_world(self, mask, ee):
        """whether a command with end-effector rows (ee) to the robots of mask [B] reaches a world-frame robot: any masked one (read on the host)
        when the session sets frame rows, every command with end-effector rows when it does not"""
        world = self._spec["world"]
        if not ee or world is True:
            return ee
        m = mask.detach().cpu().numpy() if hasattr(mask, "detach") else np.asarray(mask)
        return bool(np.any((m != 0) & world))

    def _wait_caller(self):   # rows the caller wrote on its own stream are complete before the session's stream reads them
        import torch
        if self.device.type == "cuda":
            self.stream.wait_stream(torch.cuda.current_stream(self.device))

    def _put(self, a, dtype, shape, fill):   # a caller's rows (device tensor, host array or None: fill) as a tensor the session's stream may read
        import torch
        dev = self.device
        if a is None:
            return torch.full(shape, fill, dtype=dtype, device=dev)
        if isinstance(a, torch.Tensor):
            t = a.to(device=dev, dtype=dtype).contiguous()
            if t.is_cuda:   # the caller may free it before the session's stream has read it: its memory waits for that stream
                t.record_stream(self.stream)
            return t
        return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64 if dtype == torch.float64 else np.int32), device=dev)

    def _branchable(self, who):   # ValueError where snapshots do not apply: finish() rebuilds per-episode rows from (robot, episode)
        used = [k for k, key in (("respawn", "rs"), ("randomize", "rz"), ("spawn", "sp"), ("timeline", "tl"), ("curriculum", "cu")) if self._spec[key] is not None]
        if used:
            raise ValueError("closed_loop.Session.%s: snapshots cannot go with %s (a branched robot would break the per-episode rows finish() rebuilds "
                             "from robot and episode)" % (who, ", ".join(used)))
        if not self._open or self._finished:
            raise ValueError("closed_loop.Session.%s: the session is not open (enter it with `with`; finish() ends it)" % who)

    def snapshot(self):
        """A Snapshot of every robot at the current window boundary: the library's rows (Solver.robot_state_save_dev) and device clones of the loop's
        per-robot rows.  Enqueued on self.stream, no synchronisation.  ValueError with respawn, randomize, spawn, timeline or curriculum."""
        import torch
        self._branchable("snapshot")
        with torch.cuda.stream(self.stream):
            buf = torch.empty(self.B * self.solver.robot_state_bytes(), dtype=torch.uint8, device=self.device)
            desc = self.solver.robot_state_save_dev(buf, self._s)
            rows = [a.clone() for a in self.rows]
            k0 = self.k0.clone() if self.k0 is not None else torch.zeros(self.B, dtype=torch.int64, device=self.device)
        return Snapshot(self, buf, desc, rows, k0, self._k)

    def restore(self, snap, mask=None, source=None):
        """Each robot b with mask[b] set (device tensor [B], as command takes; None: every robot) takes robot source[b]'s rows of snap (int32 [B]; None:
        its own): the library's and the loop's, and its clock, so that it resumes where the source was when snap was taken.  Applied in stream order at
        the current window boundary, before the next MPC tick.  A source outside [0, B) leaves the robot untouched and OR-s _lib.ST_RESTORE into the
        record of the window that tick opens.  Enqueued on self.stream after the caller's current stream, no synchronisation.  ValueError, before any
        write, for a snapshot of another or a finished session, one the library refuses (a component reset, stopped or re-allocated since, a settings
        array set or cleared since), one taken at window 0 (after the first MPC tick) restored at a later boundary or the reverse, and as snapshot()."""
        import torch
        from ._lib import QmbError
        self._branchable("restore")
        B = self.B
        if not isinstance(snap, Snapshot) or snap.session is not self:
            raise ValueError("closed_loop.Session.restore: the snapshot belongs to another session")
        if (snap.k == 0) != (self._k == 0):
            raise ValueError("closed_loop.Session.restore: a snapshot of window 0 (taken after the first MPC tick) restores only at window 0, and a later one "
                             "only at a later boundary (before its MPC tick)")
        for name, a in (("mask", mask), ("source", source)):
            if a is not None and tuple(np.shape(a)) != (B,):
                raise ValueError("closed_loop.Session.restore: %s must have shape (%d,), got %s" % (name, B, tuple(np.shape(a))))
        self._wait_caller()
        with torch.cuda.stream(self.stream):
            m = self._put(mask, torch.int32, (B,), 1); src = None if source is None else self._put(source, torch.int32, (B,), 0)
            try:
                self.solver.robot_state_load_dev(snap.buf, snap.desc, m, src, self.restore_st, self._s)
            except QmbError as e:
                raise ValueError("closed_loop.Session.restore: the library refuses the snapshot: %s" % e) from None
            ok = m.bool() if src is None else m.bool() & (src >= 0) & (src < B)
            if self.k0 is None:   # from now on every robot runs on its own clock; k0 = 0 gives the global one
                self.k0 = torch.zeros(B, dtype=torch.int64, device=self.device); self.dk = torch.zeros_like(self.k0)
            idx = None if src is None else src.long().clamp(0, B - 1)
            _gather(self.rows + [self.k0], snap.rows + [self._k - (snap.k - snap.k0)], ok, idx)   # the rows, and the source's clock shifted to now
            self.acc_st.bitwise_or_(self.restore_st)
        if self._spec["gd"] is not None:   # the restored robots' pending commands' status goes into the window the tick opens
            self._commanded = True

    @property
    def gait_templates(self):
        """the device gait schedule's template names (a template id is its index), or None without it"""
        gd = self._spec["gd"]
        return None if gd is None else list(gd["names"])

    @property
    def state(self):
        """The live device tensors at the current window boundary (the loop writes them: read, do not write): q, v [B, 24] and rbd [B, 55] (the plant's
        truth), meas (what the controller reads: rbd, or the estimator's rbd_est), x_obs, t_obs, contact, cmd [B, 7] (the target front-end's command),
        and with respawn episode, fallen and due (the robots that respawn at the next boundary, requests merged), with curriculum level; None where not running.  clock
        [B]: each robot's episode time in s, computed on self.stream at this call."""
        import torch
        rs, cu = self._spec["rs"], self._spec["cu"]
        with torch.cuda.stream(self.stream):
            clock = (self._k - self.k0).to(torch.float64) * 1e-3 if self.k0 is not None else torch.full((self.B,), self._k * 1e-3, dtype=torch.float64, device=self.device)
        return dict(q=self.q, v=self.v, rbd=self.rbd, meas=self.meas, x_obs=self.x_obs, t_obs=self.t_obs, contact=self.contact, cmd=self.cmd7,
                    episode=self.episode if rs is not None else None, fallen=self.fallen if rs is not None else None, due=self.due if rs is not None else None,
                    level=self.cu_level if cu is not None else None, clock=clock)

    def finish(self):
        """Close every robot's open episode (end 0) and return run's end-of-run keys as numpy arrays, from the device state: contact, q, v, start_base,
        start_ee, and as run gives them gait_templates, episode_level, curriculum_state, episode_params, spawn_params, timeline_params, ee_path_params,
        episode_metrics and metrics_layout.  Synchronises self.stream; the session takes no more steps."""
        import torch
        if not self._open or self._finished:
            raise ValueError("closed_loop.Session.finish: the session is not open (enter it with `with`; finish() ends it)")
        self._finished = True
        solver, p, B = self.solver, self._spec, self.B
        rs, rz, sp, tl, cu, gd = p["rs"], p["rz"], p["sp"], p["tl"], p["cu"], p["gd"]
        if self._mt:   # the run's end closes every robot's open episode
            with torch.cuda.stream(self.stream):
                ones = torch.ones(B, dtype=torch.int32, device=self.device)
                solver.metrics_close_dev(ones, torch.zeros_like(ones), self.episode if rs is not None else torch.zeros_like(ones), self.mt_acc, self.mt_out, self.acc_st, self._s)
        self.stream.synchronize()
        out = dict(contact=self.contact.cpu().numpy(), q=self.q.cpu().numpy(), v=self.v.cpu().numpy(), **self._start_out)
        if gd is not None:
            out["gait_templates"] = list(gd["names"])
        last = self.episode.cpu().numpy() if rs is not None else np.zeros(B, dtype=np.int32)   # a robot's episodes are 0 .. last[b]
        had = np.arange(int(last.max()) + 1)[None, :] <= last[:, None]
        if cu is not None:   # a robot's level is constant over an episode: it moves at the respawn that starts the next
            el = self.ep_level[:, :had.shape[1]].cpu().numpy()
            out.update(episode_level=el, curriculum_state=solver.curriculum_get())
        if rz is not None or sp is not None or tl is not None:   # rebuilt on the host: the samplers' rows are pure functions of (ranges, seed, robot, episode[, level])
            rb, re_ = np.nonzero(had)
            for kind, spec, shape in (("episode", rz, (_lib.EPISODE,)), ("spawn", sp, (_lib.SPAWN,)), ("timeline", tl, (0 if tl is None else tl["n"], _lib.TIMELINE_CMD))):
                if spec is not None:
                    rows = solver.curriculum_draw(kind, rb, re_, el[rb, re_]) if kind in self._tops else getattr(solver, kind + "_draw")(rb, re_)
                    out[kind + "_params"] = np.full(had.shape + shape, np.nan); out[kind + "_params"][rb, re_] = rows
            if tl is not None:   # on the episode's clock: exact for drawn times in [t_start / 2, 2 t_start]
                out["timeline_params"][..., 0] -= self.t_start
        if p["pd"] is not None:   # tau counts from the path's start, the episode's first MPC tick
            rb, re_ = np.nonzero(had)
            _, way = solver.curriculum_draw("ee_path", rb, re_, el[rb, re_]) if "ee_path" in self._tops else solver.ee_path_draw(rb, re_)
            out["ee_path_params"] = np.full(had.shape + (p["pd"]["n"], 8), np.nan); out["ee_path_params"][rb, re_] = way[:, :p["pd"]["n"]]
        if self._placing and int(self.pl_any.item()):   # placed rows are not draws: the device record holds every episode's row
            out["spawn_params"] = self.sp_rec[:, :had.shape[1]].cpu().numpy()
        if self._mt:   # trimmed to the most episodes of any robot
            out.update(episode_metrics=self.mt_out[:, :had.shape[1]].cpu().numpy(), metrics_layout=_lib.METRICS_LAYOUT)
        return out
