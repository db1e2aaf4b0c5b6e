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
        attitude_filter=None, slip_detector=None, ground_map=None, commands=None, tuning=None, respawn=None, randomize=None, spawn=None):
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
    when run returns.
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
    episodes of any robot), NaN where a robot had no episode e; with spawn also spawn_params[B, E, 4], the spawn row of each such episode."""
    rs = None if respawn is None else _respawn_spec(respawn)
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
    gd = None if commands is None else _gait_commands(solver.batch, gait, commands)
    tn = None if tuning is None else _tuning_spec(solver.batch, tuning)
    sp = None if spawn is None else _spawn_spec(getattr(solver, "batch", None), spawn, terrain, ground_map, gd)
    if rz is not None:   # the links: a drawn payload / friction also goes where the run told the controller the plant's
        if isinstance(model_payload, str) and model_payload == "plant" and set(rz["fields"]) & set(_lib.PAYLOAD_LAYOUT):
            if payload_estimator is not None:
                raise ValueError("closed_loop.run: model_payload=\"plant\" with a randomized payload cannot run with payload_estimator (its commits own the model payload)")
            rz["link"] |= _lib.EPISODE_MODEL_PAYLOAD
        if tn is not None and "friction_mu" in rz["fields"]:
            rz["link"] |= (_lib.EPISODE_MPC_FRICTION if isinstance(tn.get("friction_mu"), str) else 0) | (_lib.EPISODE_WBC_FRICTION if isinstance(tn.get("wbc_friction"), str) else 0)
    # set in this order, restored in reverse: the estimator starts from the model payload in force, and "plant" reads this run's payload or the handle's
    with contextlib.ExitStack() as scope:
        if sp is not None:   # restored last: the earlier ranges are set again on the earlier library and robot terrain rows, which give their origins
            scope.enter_context(_ranges(solver, "spawn"))
        if terrain is not None:
            scope.enter_context(_terrain(solver, terrain))
        if ground_map is not None:
            scope.enter_context(_ground_map(solver, terrain if ground_map is True else ground_map))
        if model_payload is not None:
            scope.enter_context(_model_payload(solver, model_payload, payload))
        if tn is not None:
            scope.enter_context(_robot_tuning(solver, tn, friction_mu))
        if payload_estimator is not None:
            scope.enter_context(_payload_estimator(solver, payload_estimator))
        if state_estimator is not None:
            scope.enter_context(_state_estimator(solver, state_estimator, sensor_noise))
        if attitude_filter is not None:
            scope.enter_context(_attitude_filter(solver, attitude_filter))
        if slip_detector is not None:
            scope.enter_context(_slip_detector(solver, slip_detector))
        if friction_mu is not None or payload is not None or rz is not None:
            scope.enter_context(_robot_params(solver, friction_mu, payload))
        if rz is not None:
            scope.enter_context(_ranges(solver, "episode"))
        if gd is not None:
            scope.enter_context(_gait_dev(solver, gd))
        if rs is not None:
            scope.callback(solver.robot_image_clear)
        return _run(solver, duration=duration, gait=gait, cmd_vel=cmd_vel, wbc_period_ms=wbc_period_ms, xy_yaw=xy_yaw, t_start=t_start,
                    torch_device=torch_device, sim_timer=sim_timer, pushes=pushes, est=payload_estimator is not None, se=state_estimator is not None,
                    att=attitude_filter is not None, sl=slip_detector is not None, gd=gd, rs=rs, rz=rz, sp=sp)


def _respawn_spec(respawn):
    """closed_loop.run's respawn → dict(on_fall, hold_windows, z_min, tilt_max, every_ms or None); ValueError when malformed"""
    spec = dict(on_fall=True, hold=0.1, z_min=0.3, tilt_max=0.3, every=None)
    if respawn is not True:
        if not isinstance(respawn, dict) or not set(respawn) <= set(spec):
            raise ValueError("closed_loop.run: respawn must be None, True or dict(on_fall, hold, z_min, tilt_max, every), got %r" % (respawn,))
        spec.update(respawn)
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
    if not spec["on_fall"] and every is None:
        raise ValueError("closed_loop.run: respawn needs on_fall or every (it would never restart a robot)")
    return dict(on_fall=bool(spec["on_fall"]), hold_windows=hold // MPC_PERIOD_MS, z_min=float(spec["z_min"]), tilt_max=float(spec["tilt_max"]), every_ms=every)


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


def _spawn_spec(B, spawn, terrain, ground_map, gd):
    """closed_loop.run's spawn (with its terrain, ground_map and parsed commands) → dict(seed, fields: name -> (lo, hi) float arrays, scalar or [B],
    link); ValueError when malformed.  B None: the bounds' length is not checked."""
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
    if "yaw" in fields and gd is not None and gd["ee"] and np.any(fields["yaw"][0] != fields["yaw"][1]):
        raise ValueError("closed_loop.run: a drawn spawn yaw cannot go with ee_goal / ee_cmd_vel commands (their world-frame goals assume the robot faces +x)")
    return dict(seed=seed, fields=fields, link=_lib.SPAWN_GROUND_MAP if ground_map is True else 0)


@contextlib.contextmanager
def _ranges(solver, kind):
    """the ranges of solver's kind ("episode" or "spawn") draws in force, set again on exit"""
    prev = getattr(solver, kind + "_get_ranges")()
    try:
        yield   # _run sets this run's ranges once it has read its fixed values
    finally:
        if prev is None:
            getattr(solver, kind + "_set_ranges")(None)
        else:
            getattr(solver, kind + "_set_ranges")(**prev)


def _set_ranges(solver, kind, layout, row, spec):
    """sets the run's ranges of solver's kind draws: every column fixed at the run's value, row [B, C], except the spec's fields, drawn within their
    bounds → hi [B, C]"""
    col = {n: i for i, n in enumerate(layout)}
    lo = row.copy(); hi = row.copy()
    for k, (l, h) in spec["fields"].items():
        lo[:, col[k]] = l; hi[:, col[k]] = h
    getattr(solver, kind + "_set_ranges")(lo, hi, spec["seed"])
    return hi


def _gait_commands(B, gait, commands):
    """closed_loop.run's gait and commands → dict(names, gait [B] ids, t [B, C], tmpl [B, C] ids or -1, cmd_vel [B, C, 4], ee: {} or dict(ee_kind [B, C],
    ee_cmd [B, C, 7]) when the timeline has ee_goal / ee_cmd_vel); ValueError when malformed"""
    names = gait_template_names()
    ids = {n: i for i, n in enumerate(names)}
    start = [gait] * B if isinstance(gait, str) else list(gait)
    if len(start) != B:
        raise ValueError("closed_loop.run: gait must be one name or a sequence of %d names, got %d" % (B, len(start)))
    if not isinstance(commands, dict) or not {"t", "gait"} <= set(commands) or not set(commands) <= {"t", "gait", "cmd_vel", "ee_goal", "ee_cmd_vel"}:
        raise ValueError("closed_loop.run: commands must be dict(t, gait[, cmd_vel][, ee_goal][, ee_cmd_vel]), got %r" % (commands,))
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
    return dict(names=names, gait=np.array([ids[n] for n in start], dtype=np.int32), t=t, tmpl=tmpl, cmd_vel=vel, ee=_ee_commands(B, C, commands, vel))


def _ee_commands(B, C, commands, vel):
    """commands' ee_goal [B, C, 7] / ee_cmd_vel [B, C, 3] → {} when neither is given, else dict(ee_kind [B, C], ee_cmd [B, C, 7]) for
    Solver.gait_dev_set_commands; ValueError when malformed"""
    if commands.get("ee_goal") is None and commands.get("ee_cmd_vel") is None:
        return {}
    goal = np.full((B, C, 7), np.nan) if commands.get("ee_goal") is None else np.asarray(commands["ee_goal"], dtype=np.float64)
    eev = np.full((B, C, 3), np.nan) if commands.get("ee_cmd_vel") is None else np.asarray(commands["ee_cmd_vel"], dtype=np.float64)
    if goal.shape != (B, C, 7) or eev.shape != (B, C, 3):
        raise ValueError("closed_loop.run: commands ee_goal must have shape (%d, %d, 7) and ee_cmd_vel (%d, %d, 3), got %s and %s" % (B, C, B, C, goal.shape, eev.shape))
    for name, a in (("ee_goal", goal), ("ee_cmd_vel", eev)):
        if np.any(np.isnan(a).any(-1) != np.isnan(a).all(-1)) or np.any(np.isinf(a)):
            raise ValueError("closed_loop.run: each commands %s row must be finite or all NaN" % name)
    has_goal, has_eev = ~np.isnan(goal[..., 0]), ~np.isnan(eev[..., 0])
    if np.any(has_goal.astype(int) + has_eev + ~np.isnan(vel[..., 0]) > 1):
        raise ValueError("closed_loop.run: a command carries at most one of cmd_vel, ee_goal and ee_cmd_vel")
    if np.any(np.abs(np.linalg.norm(goal[has_goal][:, 3:7], axis=-1) - 1.0) > 1e-9):
        raise ValueError("closed_loop.run: each commands ee_goal quaternion (xyzw) must have unit norm (within 1e-9)")
    kind = np.where(has_goal, _lib.TARGET_EE_GOAL, np.where(has_eev, _lib.TARGET_EE_CMD_VEL, -1)).astype(np.int32)
    cmd = np.where(has_goal[..., None], goal, 0.0); cmd[..., :3] = np.where(has_eev[..., None], eev, cmd[..., :3])
    return dict(ee_kind=kind, ee_cmd=cmd)


@contextlib.contextmanager
def _gait_dev(solver, gd):
    solver.gait_dev_set_templates(gd["names"])
    try:
        yield   # _run resets the schedule and loads the timeline once it knows the start time
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
        yield   # _run resets the estimator once it knows the start position
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
        yield   # _run resets the filter right before its first reading
    finally:
        solver.attitude_stop()
        solver.attitude_set_params(**prev_params)


@contextlib.contextmanager
def _slip_detector(solver, params):
    prev_params = solver.slip_get_params()
    try:
        if isinstance(params, dict):
            solver.slip_set_params(**params)
        yield   # _run resets the detector with the estimator
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


def _run(solver, duration, gait, cmd_vel, wbc_period_ms, xy_yaw, t_start, torch_device, sim_timer, pushes, est=False, se=False, att=False, sl=False, gd=None,
         rs=None, rz=None, sp=None):
    import torch
    B = solver.batch; dev = torch.device(torch_device or "cuda:%d" % solver._cfg.device)
    n_ms = int(round(duration * 1e3)); assert n_ms > 0 and n_ms % MPC_PERIOD_MS == 0, "duration must be a multiple of 10 ms"
    assert MPC_PERIOD_MS % wbc_period_ms == 0, "the WBC period must divide the MPC period"
    cmd_vel = np.asarray(cmd_vel, dtype=np.float64)
    if cmd_vel.shape not in ((4,), (B, 4)):
        raise ValueError("closed_loop.run: cmd_vel must have shape (4,) or (%d, 4), got %s" % (B, cmd_vel.shape))
    if pushes is not None:
        t_on, t_dur, wrench = (np.asarray(a, dtype=np.float64) for a in pushes)
        if t_on.shape != (B,) or t_dur.shape != (B,) or wrench.shape != (B, 12):
            raise ValueError("closed_loop.run: pushes must be (t_on[%d], duration[%d], wrench[%d, 12])" % (B, B, B))
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
        hi = _set_ranges(solver, "episode", _lib.EPISODE_LAYOUT, row, rz)
        if pushes is None and np.any(hi[:, EP["push_duration"]] > 0.0):   # the draws overwrite these rows before the first solve
            t_on, t_dur, wrench = np.zeros(B), np.zeros(B), np.zeros((B, 12)); pushes = (t_on, t_dur, wrench)
    xy = np.zeros((B, 3)) if xy_yaw is None else np.asarray(xy_yaw, dtype=np.float64).reshape(B, 3)
    if sp is not None:   # the ranges: this run's values (entered after _terrain: the robot terrain rows are this run's), the named columns' bounds
        SP = {n: i for i, n in enumerate(_lib.SPAWN_LAYOUT)}
        rt = solver.sim_get_robot_terrain()
        yaw = xy[:, 2]; yaw = np.where(np.abs(yaw) <= np.pi, yaw, np.remainder(yaw + np.pi, 2.0 * np.pi) - np.pi)   # the same heading within [-pi, pi]
        row = np.zeros((B, _lib.SPAWN)); row[:, SP["tile"]] = -1.0 if rt is None else rt["tile"]; row[:, SP["yaw"]] = yaw
        _set_ranges(solver, "spawn", _lib.SPAWN_LAYOUT, row, sp)
    stream = torch.cuda.Stream(device=dev); s = stream.cuda_stream
    f64 = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=dev)
    i32 = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.int32), device=dev)

    # ---- plant state, the first measurement, the controller's members (host → device once) ----
    q0, v0 = solver.sim_standing_state(xy)
    t_obs0 = t_start - wbc_period_ms * 1e-3   # observation clock of `starting`; the first update brings it to t_start, the plant's clock
    if gd is None:
        ev, md, ne = _schedules(gait, B, t_start, t_obs0, t_start + duration + solver.time_horizon + 1.0)
    else:   # the first gait step writes the rows
        ev, md, ne = np.zeros((B, EMAX)), np.full((B, EMAX + 1), 15, dtype=np.int32), np.zeros(B, dtype=np.int32)
    with torch.cuda.stream(stream):
        q = f64(q0); v = f64(v0); rbd = torch.zeros((B, RBD), dtype=torch.float64, device=dev)
        contact = torch.zeros(B, dtype=torch.int32, device=dev); sim_st = torch.zeros_like(contact); hw_st = torch.zeros_like(contact); ctl_st = torch.zeros_like(contact)
        acc_st = torch.zeros_like(contact)
        effort = torch.zeros((B, 18), dtype=torch.float64, device=dev); jpos = torch.zeros_like(effort); jvel = torch.zeros_like(effort)
        if se:   # the controller's measurement: the estimator's rbd_est in place of the plant's rbd
            v_prev = torch.zeros_like(v); sensors = torch.zeros((B, SENSORS), dtype=torch.float64, device=dev); rbd_est = torch.zeros_like(rbd)
            se_st = torch.zeros_like(contact); v_prev.copy_(v)
            if att:
                at_st = torch.zeros_like(contact)
            if sl:   # the estimator reads the trusted stance mask in place of the plant's contact mask
                stance = torch.zeros_like(contact); slip = torch.zeros_like(contact); sl_st = torch.zeros_like(contact); slip_acc = torch.zeros_like(contact)
    stream.synchronize()
    solver.sim_step_dev(1e-6, effort, q, v, rbd, contact, sim_st, s)   # a 1 us physics step with zero effort reads the first measured state
    meas = rbd
    if se:
        solver.sim_read_sensors_dev(1e-6, -1, q, v, v_prev, sensors, s)
        stream.synchronize()
        solver.state_est_reset(q0[:, 0:3])
        if att:
            solver.attitude_reset()
            solver.attitude_step_dev(1e-6, sensors, at_st, s)   # the first call after the reset takes the reading
        se_contact = contact
        if sl:
            solver.slip_reset()
            solver.slip_step_dev(1e-6, sensors, contact, stance, slip, sl_st, s)   # passes the contact mask through: the estimator has had no call yet
            se_contact = stance
        solver.state_est_step_dev(1e-6, sensors, se_contact, rbd_est, se_st, s)   # the first call after the reset places the feet
        meas = rbd_est
    stream.synchronize()
    rbd_h = rbd.cpu().numpy()
    x_obs0 = solver.centroidal_state_from_rbd(meas.cpu().numpy())
    with torch.cuda.stream(stream):
        t_obs = f64(np.full(B, t_obs0)); x_obs = f64(x_obs0)
        joint_cmd = torch.zeros((B, 18, 5), dtype=torch.float64, device=dev); arm_pos = torch.zeros((B, 6), dtype=torch.float64, device=dev); last_time = f64(np.full(B, t_obs0))
        cmd54 = torch.zeros((B, 54), dtype=torch.float64, device=dev)
        cmd7 = torch.zeros((B, 7), dtype=torch.float64, device=dev); cmd7[:, :4] = f64(cmd_vel[None, :4] if cmd_vel.ndim == 1 else cmd_vel)
        last_ee = f64(solver.initial_ee_target()); ee_state = torch.zeros((B, 7), dtype=torch.float64, device=dev)
        prob = dict(t0=t_obs, x0=x_obs, n_events=i32(ne), event_times=f64(ev), modes=i32(md),
                    n_target=torch.zeros(B, dtype=torch.int32, device=dev), target_times=torch.zeros((B, KMAX), dtype=torch.float64, device=dev),
                    target_states=torch.zeros((B, KMAX, TARGET), dtype=torch.float64, device=dev))
        period = f64(np.full(B, wbc_period_ms * 1e-3)); hw_period = f64(np.full(B, 1e-3)); hw_time = torch.zeros(B, dtype=torch.float64, device=dev)
        ticks = n_ms // MPC_PERIOD_MS
        rec_base = torch.zeros((ticks, B, 6), dtype=torch.float64, device=dev); rec_ee = torch.zeros((ticks, B, 7), dtype=torch.float64, device=dev)
        rec_st = torch.zeros((ticks, B), dtype=torch.int32, device=dev)
        if est:
            est_st = torch.zeros_like(contact); rec_pl = torch.zeros((ticks, B, 8), dtype=torch.float64, device=dev)   # row i: the rows of window i's MPC tick
        if se:
            rec_base_est = torch.zeros((ticks, B, 6), dtype=torch.float64, device=dev)
        if sl:
            rec_slip = torch.zeros((ticks, B), dtype=torch.int32, device=dev)
        if gd is not None:
            gait_st = torch.zeros_like(contact); rec_gait = torch.zeros((ticks, B), dtype=torch.int32, device=dev); rec_mode = torch.zeros_like(rec_gait)
            rec_kind = torch.zeros_like(rec_gait); rec_ee_target = torch.zeros((ticks, B, 7), dtype=torch.float64, device=dev)
        push = None
        if pushes is not None:   # robot b is pushed in plant step k (start k ms after the start) when t_on <= k ms < t_on + duration
            push = dict(on=f64(t_on * 1e3 - 1e-6), off=f64((t_on + t_dur) * 1e3 - 1e-6), wrench=f64(wrench), zero=torch.zeros((B, 12), dtype=torch.float64, device=dev),
                        now=torch.zeros((B, 12), dtype=torch.float64, device=dev))
    stream.synchronize()
    if gd is not None:
        solver.gait_dev_reset(gd["gait"], np.full(B, t_start))
        solver.gait_dev_set_commands(t_start + gd["t"], gd["tmpl"], gd["cmd_vel"], **gd["ee"])
    solver.hw_set_delay(HW_DELAY)

    def mpc_tick(i):
        if est:
            solver.payload_est_commit_dev(s); solver.get_model_payload_dev(rec_pl[i], s)
        ee_state.copy_(meas[:, 48:55])
        if gd is None:
            solver.target_trajectories_dev(0, cmd7, t_obs, x_obs, ee_state, last_ee, prob["n_target"], prob["target_times"], prob["target_states"], s)
        else:   # the step's target kinds go straight to the target call, and stay in the record
            kind = rec_kind[i]
            solver.gait_dev_step_dev(t_obs, prob, cmd7, rec_gait[i], rec_mode[i], gait_st, s, target_kind=kind)
            acc_st.bitwise_or_(gait_st)
            solver.target_trajectories_dev(kind, cmd7, t_obs, x_obs, ee_state, last_ee, prob["n_target"], prob["target_times"], prob["target_states"], s)
            rec_ee_target[i] = prob["target_states"][:, 1, 30:37]
        solver.mpc_solve_dev(prob, s)

    if rs is not None:   # the start image: the library's rows and the loop's own, then one restore of every robot through the cold path of every later one
        own = [q, v, rbd, contact, t_obs, x_obs, joint_cmd, arm_pos, last_time, cmd54, cmd7, last_ee, prob["n_events"], prob["event_times"], prob["modes"],
               prob["n_target"], prob["target_times"], prob["target_states"]] + ([v_prev, sensors, rbd_est] if se else []) + ([stance] if sl else [])
        solver.robot_image_save()
        with torch.cuda.stream(stream):
            start = [a.clone() for a in own]
            k0 = torch.zeros(B, dtype=torch.int64, device=dev); dk = torch.zeros_like(k0)   # each robot's episode start (plant step), and k - k0
            episode = torch.zeros(B, dtype=torch.int32, device=dev); fall_count = torch.zeros_like(episode); fallen = torch.zeros_like(episode)
            due = torch.ones_like(episode); rec_episode = torch.zeros((ticks, B), dtype=torch.int32, device=dev); rec_fallen = torch.zeros_like(rec_episode)
        solver.robot_image_restore_dev(due, s)

    def respawn(k):   # the robots due restart at window boundary k: the library's rows, then the loop's, then their new plant
        solver.robot_image_restore_dev(due, s)
        m = due.bool()
        for a, a0 in zip(own, start):
            a.copy_(torch.where(m.view((B,) + (1,) * (a.dim() - 1)), a0, a))
        k0.copy_(torch.where(m, k, k0)); episode.add_(due); fall_count.masked_fill_(m, 0)
        begin(due, episode)

    def begin(mask, idx):   # the masked robots begin episode idx: their plant's draw, then their spawn
        if rz is not None:
            draw(mask, idx)
        if sp is not None:
            stand(mask, idx)

    def draw(mask, idx):   # the masked robots draw episode idx: the plant rows on the device, then the loop's cmd_vel and push rows from the drawn row
        solver.episode_sample_dev(mask, idx, ep_rows, rz["link"], s)
        m = mask.bool()
        cmd7[:, :4] = torch.where(m[:, None], ep_rows[:, 23:27], cmd7[:, :4])
        if push is not None:
            on = ep_rows[:, 9] * 1e3 - 1e-6; off = (ep_rows[:, 9] + ep_rows[:, 10]) * 1e3 - 1e-6
            push["on"].copy_(torch.where(m, on, push["on"])); push["off"].copy_(torch.where(m, off, push["off"]))
            push["wrench"].copy_(torch.where(m[:, None], ep_rows[:, 11:23], push["wrench"]))

    def stand(mask, idx):   # the masked robots spawn episode idx: new ground under them, their start state there
        solver.spawn_sample_dev(mask, idx, sp_rows, q, v, rbd, contact, x_obs, last_ee, rbd_est if se else None, sp["link"], s)

    if rz is not None or sp is not None:   # every robot's first episode begins right before the first solve (after the restore of the start image)
        with torch.cuda.stream(stream):
            ep_rows = torch.zeros((B, _lib.EPISODE), dtype=torch.float64, device=dev) if rz is not None else None
            sp_rows = torch.zeros((B, _lib.SPAWN), dtype=torch.float64, device=dev) if sp is not None else None
            if rs is None:
                begin(torch.ones(B, dtype=torch.int32, device=dev), torch.zeros(B, dtype=torch.int32, device=dev))
            else:
                begin(due, episode)

    with torch.cuda.stream(stream):
        mpc_tick(0); stream.synchronize()          # QMController::starting: one blocking solve before the loop
        for k in range(n_ms):
            if k % MPC_PERIOD_MS == 0 and k > 0:
                if rs is not None:
                    respawn(k)
                mpc_tick(k // MPC_PERIOD_MS)
            if k % wbc_period_ms == 0:
                solver.update_dev(meas, period, t_obs, x_obs, joint_cmd, arm_pos, last_time, cmd54, ctl_st, s)
                acc_st.bitwise_or_(ctl_st)
            if rs is None:
                hw_time.fill_(t_start + k * 1e-3)
            else:   # the robot's episode clock
                torch.sub(k0, k, out=dk).neg_(); hw_time.copy_(dk).mul_(1e-3).add_(t_start)
            jpos.copy_(q[:, 6:]); jvel.copy_(v[:, 6:])
            solver.hw_write_dev(hw_time, hw_period, joint_cmd, jpos, jvel, effort, hw_st, s)
            if se:
                v_prev.copy_(v)
            if sim_timer:
                sim_timer(True)
            if push is not None:
                kk = k if rs is None else dk   # plant steps since the episode's start
                torch.where(((push["on"] <= kk) & (push["off"] > kk))[:, None], push["wrench"], push["zero"], out=push["now"])
            solver.sim_step_dev(1e-3, effort, q, v, rbd, contact, sim_st, s, wrench=None if push is None else push["now"])
            if sim_timer:
                sim_timer(False)
            acc_st.bitwise_or_(hw_st).bitwise_or_(sim_st)
            if se:
                solver.sim_read_sensors_dev(1e-3, k, q, v, v_prev, sensors, s)
                if att:
                    solver.attitude_step_dev(1e-3, sensors, at_st, s)
                    acc_st.bitwise_or_(at_st)
                if sl:
                    solver.slip_step_dev(1e-3, sensors, contact, stance, slip, sl_st, s)
                    acc_st.bitwise_or_(sl_st); slip_acc.bitwise_or_(slip)
                solver.state_est_step_dev(1e-3, sensors, se_contact, rbd_est, se_st, s)
                acc_st.bitwise_or_(se_st)
            if est:
                solver.payload_est_step_dev(1e-3, effort, meas, est_st, s)
                acc_st.bitwise_or_(est_st)
            if (k + 1) % MPC_PERIOD_MS == 0:
                i = (k + 1) // MPC_PERIOD_MS - 1
                rec_base[i, :, 0:3] = rbd[:, 3:6]; rec_base[i, :, 3:6] = rbd[:, 0:3]; rec_ee[i] = rbd[:, 48:55]; rec_st[i] = acc_st; acc_st.zero_()
                if se:
                    rec_base_est[i, :, 0:3] = rbd_est[:, 3:6]; rec_base_est[i, :, 3:6] = rbd_est[:, 0:3]
                if sl:
                    rec_slip[i] = slip_acc; slip_acc.zero_()
                if rs is not None:
                    solver.fall_detect_dev(rbd, fall_count, fallen, rs["z_min"], rs["tilt_max"], s)
                    rec_episode[i] = episode; rec_fallen[i] = fallen
                    d = fall_count >= rs["hold_windows"] if rs["on_fall"] else torch.zeros_like(fallen, dtype=torch.bool)
                    if rs["every_ms"] is not None:
                        d |= (k + 1 - k0) >= rs["every_ms"]
                    due.copy_(d)
    stream.synchronize()
    t = t_start + np.arange(1, ticks + 1) * MPC_PERIOD_MS * 1e-3
    out = dict(t=t, base=rec_base.cpu().numpy(), ee=rec_ee.cpu().numpy(), status=rec_st.cpu().numpy(), contact=contact.cpu().numpy(), q=q.cpu().numpy(), v=v.cpu().numpy(),
               start_base=np.c_[q0[:, 0:3], q0[:, 3:6]], start_ee=rbd_h[:, 48:55])
    if est:
        out["payload_est"] = rec_pl.cpu().numpy()
    if se:
        out["base_est"] = rec_base_est.cpu().numpy()
    if sl:
        out["slip"] = rec_slip.cpu().numpy()
    if gd is not None:
        out.update(gait=rec_gait.cpu().numpy(), mode=rec_mode.cpu().numpy(), gait_templates=list(gd["names"]), target_kind=rec_kind.cpu().numpy(),
                   ee_target=rec_ee_target.cpu().numpy())
    if rs is not None:
        out.update(episode=rec_episode.cpu().numpy(), fallen=rec_fallen.cpu().numpy())
    if rz is not None or sp is not None:   # rebuilt on the host from the episode record: the samplers' rows are pure functions of (ranges, seed, robot, episode)
        ep = out["episode"] if rs is not None else np.zeros((ticks, B), dtype=np.int32)
        had = np.zeros((B, int(ep.max()) + 1), dtype=bool); had[np.broadcast_to(np.arange(B), ep.shape), ep] = True
        rb, re_ = np.nonzero(had)
        for kind, spec, width in (("episode", rz, _lib.EPISODE), ("spawn", sp, _lib.SPAWN)):
            if spec is not None:
                out[kind + "_params"] = np.full(had.shape + (width,), np.nan); out[kind + "_params"][rb, re_] = getattr(solver, kind + "_draw")(rb, re_)
    return out
