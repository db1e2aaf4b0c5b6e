"""Closed-loop benchmark on one GPU (qm_control_b200.closed_loop): the controller at the reference's rates driving this library's plant step.

Default: 8192 robots, trot at cmd_vel 0.3 m/s, 1 s simulated after a warm-up run of the same length.  Prints one JSON line with the wall time per
simulated second, the plant step's device time per call (CUDA events) and its share of the loop, and quality lines (base distance, end-effector
deviation from the initial pose, as percentiles over the robots) of this project's compliant-contact plant.  Writes nothing to disk.

    python tools/bench_closedloop.py [--batch 8192] [--duration 1.0] [--gait trot] [--vx 0.3] [--vary | --terrain] [--state-estimator [--sensor-noise reference] [--attitude-filter] [--slip-detector]]
                                     [--gait-commands] [--ee-goals]
    python tools/bench_closedloop.py --respawn [--randomize | --spawn | --timeline | --curriculum] [--batch 8192] [--duration 1.0] [--gait trot] [--vx 0.3]

--vary runs a per-robot robustness sweep on the same loop: robot b carries an end-effector payload of 0-2 kg (5 bins), stands on a floor with
mu 0.15-1.0 (5 bins) and takes a lateral (+y) base push of 0-180 N for 0.1 s from 0.4 s (4 bins), every combination equally often.  The JSON line
gains "vary": the quality per condition bin of each axis (fallen robots, base distance, end-effector deviation).  The controller is not told about
any of it, unless --model-payload plant sets the controller's model payload to the plant's (closed_loop.run(model_payload="plant")): the timed run
and the bins are then those of the told controller, and "vary" gains "payload_kg_not_told", the payload bins of the same sweep with the controller
not told, from one more (untimed) run.

--model-payload estimate runs the online payload estimator in the loop (closed_loop.run(payload_estimator=True)): the timed run and the bins are then those
of the estimating controller; "vary" gains "payload_kg_not_told" as above and, per payload bin, the p50 / max of |m_hat - m| at the end; the JSON line
gains "payload_est": the estimator's device time per call at this batch (CUDA events, alternated with blocks of plant steps).

--terrain runs the loop on heightfield terrain (qm_control_b200.terrain): robot b's tile rises beyond 0.35 m ahead of its start, as a ramp of 0/5/10/15
degrees and steps of 0/3/6/9 cm rise every 0.3 m on it, every combination equally often; the controller does not see the terrain.  The JSON line gains
"terrain": fallen robots (height above the ground under the base <= 0.3 m or |roll|, |pitch| >= 0.3 rad or non-finite) and base distance per bin of
each axis, and the plant step's device time at this batch with and without terrain (CUDA events, the two alternated in one process, from one standing
state).

--state-estimator closes the loop on the base state estimate (closed_loop.run(state_estimator=True)): the controller reads what the IMU, the encoders
and the contact flags give, with --sensor-noise reference the IMU noise of qm_gazebo/config/default.yaml.  The timed run and the quality lines are then
those of the estimating controller.  The JSON line gains "state_est": the device time per call of the sensor reading and the estimator step together at
this batch (CUDA events, alternated with blocks of plant steps); percentiles over the robots of |z_hat - z| and |v_hat - v| (over the run and at the
end) and of the xy drift at the end (taken in the warm-up run, which is the timed run's twin); and the quality lines of a ground-truth run of the same
sweep (one more untimed run in the same process).  Each of these runs starts from a cold MPC and WBC state (Solver.mpc_reset, wbc_set_input_last).
The error percentiles include the wrapped zyx orientation error of rbd_est against the plant (the largest of the three angles).
With --terrain the estimator runs on a perfect ground map (closed_loop.run(ground_map=True)), and "terrain" gains "state_est": per ramp and step bin
the fallen robots of the estimate arm and of the true-state arm and |z_hat - z| p50 / p95 over the run, and the estimator step's device time at this
batch with the map and without it (CUDA events, alternated).

--attitude-filter (with --state-estimator) runs the attitude filter between the sensors and the estimator (closed_loop.run(attitude_filter=True)): the
timed run and the quality lines are then those of the filtered chain.  The JSON line gains "attitude": the filter's device time per call at this batch
(CUDA events, alternated with blocks of plant steps), and the fallen count and quality lines of the same sweep on the estimate without the filter (one
more untimed run in the same process).

--slip-detector (with --state-estimator) runs the slip detector before every estimator step (closed_loop.run(slip_detector=True)): the timed run and the
quality lines are then those of the chain with the detector.  The JSON line gains "slip": the detector's device time per call at this batch (CUDA
events, alternated with blocks of plant steps); the robots with any foot flagged; and, for the warm-up run (the timed run's twin) and for one more
untimed run of the same sweep without the detector, the fallen robots, the xy drift of the estimate at the end (p50 / p95) and |v_hat - v| over the run
from the error watch.  With --vary these come per friction bin as well.

--gait-commands adds the device gait schedule (closed_loop.run(commands=...)).  The JSON line gains "gait_commands": the wall time per simulated second
of the same run with a timeline that changes nothing (every robot re-sends its cmd_vel at 0.3 s), timed after the sweep below in the same process; the
device time per call of the gait step and of the MPC solve in that run (CUDA events around each call); and a switch sweep of 4 s: every robot stands,
trots at cmd_vel from 0.5 s and switches at 2 s to one of stance, standing_trot, flying_trot, pace, static_walk, dynamic_walk and amble (equally
often), with the fallen robots and the OR of the status bits per pair.

--ee-goals commands the end effector on the device command timeline (closed_loop.run(commands=dict(..., ee_goal=...))).  The JSON line gains "ee_goals":
a reach sweep of 5 s in which every robot starts at yaw 0 on the grid, trots, is given one goal at 0.2 s (an offset from its start pose of dx -0.1..0.4 m,
dz -0.1..0.1 m and a rotation of 0-20 deg about a fixed axis, every combination equally often) and is commanded to stance at 2.5 s, with per bin of each
axis the end-effector position and orientation errors at the end (p50 / p95), the fallen robots and the OR of the status bits; the device time per call
of the per-robot target call and of the scalar one on the same rows (CUDA events, alternated blocks); and the wall time per simulated second of a run
of --duration with the goals, with a timeline that changes nothing, and without commands (the timed run above).  --ee-tuning adds "ee_tuning_sweep": the
same reach sweep once more with per-robot tuning rows (closed_loop.run(tuning=...)) over the MPC's end-effector weights x 0.5 / 1 / 2 / 4, the WBC's
end-effector gains x 0.5 / 1 / 2 and kd_arm_wbc 0.5 / 2, every goal bin in every tuning cell alike, with the errors per bin and per cell.

--model-friction plant (with --vary) tells the MPC friction cone and the WBC friction pyramid each robot's floor friction (closed_loop.run(tuning=...)),
and runs the same sweep untold as well; both arms start from a cold MPC and WBC state.

--respawn measures episode rates instead (closed_loop.run(respawn=...)): trot at --vx on the state estimate with the reference IMU noise and no attitude
filter, robots restarted after 0.1 s fallen.  It prints one JSON line "respawn" with, from one 5 s run, the episodes per robot, the falls per
robot-second and the fraction of episodes that fall within their first second, for first and later episodes apart, over the episodes that start at
least 1 s before the run's end (with binomial standard deviations);
the wall time per simulated second of --duration runs with and without respawn, alternated in one process; and the device time per call of the fall
detector and the image restore against the plant step (CUDA events, alternated blocks).

--respawn --randomize draws a new plant for every episode (closed_loop.run(randomize=...)): floor friction in [0.15, 1.0], end-effector payload in
[0, 2] kg and a base push of (f_x, f_y) in [-180, 180] N each for 0.1 s from t_on in [0.2, 0.5] s of the episode.  It prints one JSON line "randomize"
with, from one 5 s run, the episodes per robot and the fraction of episodes that fall within their first second per friction bin x push-magnitude bin
(episodes that start at least 1 s before the run's end); the wall time per simulated second of --duration runs with and without randomize (both with
respawn), alternated in one process; and the device time per call of the sampler against the image restore (CUDA events, alternated blocks).

--respawn --curriculum gives every robot a level stepped from its episodes' outcomes (closed_loop.run(curriculum=...)).  It prints one JSON line
"curriculum" with the update's device time against the plant step (CUDA events, alternated blocks); the wall time per simulated second of --duration
runs with respawn and --randomize's plant in both arms, without and with a curriculum on the push bounds, alternated in one process; and an up-down
staircase on the base push (12 levels from 0 to 255 N, one up after an episode that lasted 1 s, one down after a fall) per friction bin on the state
estimate, beside the 50 % crossing of the fall fraction of a run with the push drawn uniformly over the same range, the same robots and duration.

--respawn --spawn starts every episode on new ground (closed_loop.run(spawn=...)) on a library of flat ground, a 10 deg ramp, 6 cm stairs and rough
ground (2 cm), each flat within 0.35 m of its centre: the tile U{0..3}, dx U[-0.5, 0] m (the flat zone before the first edge, so the controller's
absolute base-height target is met at the start), dy U[-0.2, 0.2] m and the yaw U[-pi, pi]; the estimator's ground map follows the draw.  It prints
one JSON line "spawn" with, from one 5 s run, the fraction of episodes that fall within their first second per tile x 45 deg heading bin (episodes that
start at least 1 s before the run's end); the same bins from a control run of 5 s without spawn, each robot's heading drawn once into xy_yaw on the
flat tile; the wall time per simulated second of --duration runs without spawn, with spawn ranges fixed at the run's values and with the draws (all
with respawn on the library), alternated in one process; and the device time per call of the spawn sampler against the plant step (CUDA events,
alternated blocks).

--snapshot times robot-state snapshots (closed_loop.Session.snapshot / restore) with every component running (payload and state estimators, attitude
filter, slip detector, terrain with a ground map, per-robot friction, payload, model payload and tuning rows, a commands timeline with a gait switch and
an end-effector goal, metrics).  It prints one JSON line "snapshot" with the held blocks, the library's and the session's bytes per robot, the device
time per save and per load of every robot from a permuted source (CUDA events, alternated blocks) with the copy bandwidth they reach (bytes read and
written) beside the H100's 3.35 TB/s, and the wall time per simulated second of a session stepped one window at a time without a restore and with a
snapshot and a branch of every robot every window, alternated; the card's name and power limit are read in the same process.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from qm_control_b200 import _lib   # noqa: E402  (the tree's package, as above)


def card():
    """GPU name and power limit as nvidia-smi reports them (read-only query); None where unavailable."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")[:2]]
        return name, limit
    except Exception:
        return None, None


def plant_step_times(solver, ter, xy_yaw, reps=7, calls=20):
    """Device time per 1 ms plant step (4 substeps) of the whole batch, with the sweep's terrain and without any, alternated `reps` times: each block of
    `calls` steps starts from the same terrain standing state with zero effort, timed with CUDA events → median ms per call of each."""
    import torch
    B = solver.batch; dev = torch.device("cuda", 0); s = torch.cuda.Stream(device=dev)   # a stream of its own: the legacy stream's handle 0 would select the handle's stream
    solver.sim_set_terrain(ter["tiles"], ter["cell"]); solver.sim_set_robot_terrain(ter["tile"], ter["origin"])
    q0, v0 = solver.sim_standing_state(xy_yaw)
    q0t = torch.as_tensor(q0, device=dev); v0t = torch.as_tensor(v0, device=dev); q = q0t.clone(); v = v0t.clone()
    eff = torch.zeros((B, 18), dtype=torch.float64, device=dev); rbd = torch.zeros((B, 55), dtype=torch.float64, device=dev)
    contact = torch.zeros(B, dtype=torch.int32, device=dev); st = torch.zeros_like(contact)
    times = {"terrain": [], "flat": []}
    try:
        for rep in range(reps + 1):   # the first round warms up
            for mode in ("terrain", "flat"):
                if mode == "terrain":
                    solver.sim_set_robot_terrain(ter["tile"], ter["origin"])
                else:
                    solver.sim_set_robot_terrain(None)
                q.copy_(q0t); v.copy_(v0t); torch.cuda.synchronize(dev)   # every block starts from the same state
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(s)
                for _ in range(calls):
                    solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)
                b.record(s); torch.cuda.synchronize(dev)
                if rep:
                    times[mode].append(a.elapsed_time(b) / calls)
    finally:
        solver.sim_set_terrain(None)
    return {"label": "device time per 1 ms plant step of %d robots, median of %d alternated blocks of %d calls" % (B, reps, calls),
            "ms_per_call_terrain": float(np.median(times["terrain"])), "ms_per_call_flat": float(np.median(times["flat"])),
            "spread_terrain": [float(min(times["terrain"])), float(max(times["terrain"]))], "spread_flat": [float(min(times["flat"])), float(max(times["flat"]))]}


def est_step_times(solver, xy_yaw, reps=7, calls=20):
    """Device time per payload-estimator call and per 1 ms plant step of the whole batch, alternated `reps` times in blocks of `calls` from one standing
    state (CUDA events) → median ms per call of each."""
    import torch
    B = solver.batch; dev = torch.device("cuda", 0); s = torch.cuda.Stream(device=dev)
    q0, v0 = solver.sim_standing_state(xy_yaw)
    q = torch.as_tensor(q0, device=dev); v = torch.as_tensor(v0, device=dev)
    eff = torch.zeros((B, 18), dtype=torch.float64, device=dev); rbd = torch.zeros((B, 55), dtype=torch.float64, device=dev)
    contact = torch.zeros(B, dtype=torch.int32, device=dev); st = torch.zeros_like(contact)
    prev = solver.get_model_payload(); solver.payload_est_reset(np.zeros((B, 8)))
    solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)
    times = {"estimator": [], "plant": []}
    try:
        for rep in range(reps + 1):   # the first round warms up
            for mode in ("estimator", "plant"):
                torch.cuda.synchronize(dev)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(s)
                for _ in range(calls):
                    if mode == "estimator":
                        solver.payload_est_step_dev(1e-3, eff, rbd, st, s.cuda_stream)
                    else:
                        solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)
                b.record(s); torch.cuda.synchronize(dev)
                if rep:
                    times[mode].append(a.elapsed_time(b) / calls)
    finally:
        solver.payload_est_stop(); solver.set_model_payload(prev)
    return {"label": "device time per payload-estimator call and per 1 ms plant step of %d robots, median of %d alternated blocks of %d calls" % (B, reps, calls),
            "ms_per_call": float(np.median(times["estimator"])), "ms_per_plant_step": float(np.median(times["plant"])),
            "spread": [float(min(times["estimator"])), float(max(times["estimator"]))]}


def state_est_times(solver, xy_yaw, reps=7, calls=20):
    """Device time per sensor reading + estimator step and per 1 ms plant step of the whole batch, alternated `reps` times in blocks of `calls` from one
    standing state (CUDA events) → median ms per call of each."""
    import torch
    B = solver.batch; dev = torch.device("cuda", 0); s = torch.cuda.Stream(device=dev)
    q0, v0 = solver.sim_standing_state(xy_yaw)
    q = torch.as_tensor(q0, device=dev); v = torch.as_tensor(v0, device=dev); v_prev = v.clone()
    eff = torch.zeros((B, 18), dtype=torch.float64, device=dev); rbd = torch.zeros((B, 55), dtype=torch.float64, device=dev); rbd_est = torch.zeros_like(rbd)
    sensors = torch.zeros((B, 46), dtype=torch.float64, device=dev); contact = torch.zeros(B, dtype=torch.int32, device=dev); st = torch.zeros_like(contact)
    solver.state_est_reset(q0[:, 0:3])
    solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)
    times = {"estimator": [], "plant": []}
    try:
        for rep in range(reps + 1):   # the first round warms up
            for mode in ("estimator", "plant"):
                torch.cuda.synchronize(dev)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(s)
                for k in range(calls):
                    if mode == "estimator":
                        solver.sim_read_sensors_dev(1e-3, k, q, v, v_prev, sensors, s.cuda_stream)
                        solver.state_est_step_dev(1e-3, sensors, contact, rbd_est, st, s.cuda_stream)
                    else:
                        solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)
                b.record(s); torch.cuda.synchronize(dev)
                if rep:
                    times[mode].append(a.elapsed_time(b) / calls)
    finally:
        solver.state_est_stop()
    return {"label": "device time per sensor reading + estimator step and per 1 ms plant step of %d robots, median of %d alternated blocks of %d calls" % (B, reps, calls),
            "ms_per_call": float(np.median(times["estimator"])), "ms_per_plant_step": float(np.median(times["plant"])),
            "spread": [float(min(times["estimator"])), float(max(times["estimator"]))]}


def ground_map_times(solver, ter, xy_yaw, reps=7, calls=20):
    """Device time per estimator step of the whole batch with the sweep's terrain as the estimator's ground map and without a map, alternated `reps`
    times in blocks of `calls` from one terrain standing state past the estimator's first call (CUDA events) → median ms per call of each."""
    import torch
    B = solver.batch; dev = torch.device("cuda", 0); s = torch.cuda.Stream(device=dev)
    solver.sim_set_terrain(ter["tiles"], ter["cell"]); solver.sim_set_robot_terrain(ter["tile"], ter["origin"])
    q0, v0 = solver.sim_standing_state(xy_yaw)
    q = torch.as_tensor(q0, device=dev); v = torch.as_tensor(v0, device=dev)
    eff = torch.zeros((B, 18), dtype=torch.float64, device=dev); rbd = torch.zeros((B, 55), dtype=torch.float64, device=dev); rbd_est = torch.zeros_like(rbd)
    sensors = torch.zeros((B, 46), dtype=torch.float64, device=dev); contact = torch.zeros(B, dtype=torch.int32, device=dev); st = torch.zeros_like(contact)
    solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)
    solver.sim_read_sensors_dev(1e-3, 0, q, v, v, sensors, s.cuda_stream); torch.cuda.synchronize(dev)
    solver.state_est_reset(q0[:, 0:3]); solver.state_est_step_dev(1e-3, sensors, contact, rbd_est, st, s.cuda_stream)   # past the first call
    times = {"map": [], "plane": []}
    try:
        for rep in range(reps + 1):   # the first round warms up
            for mode in ("map", "plane"):
                if mode == "map":
                    solver.state_est_set_ground(ter["tile"], ter["origin"])
                else:
                    solver.state_est_set_ground(None)
                torch.cuda.synchronize(dev)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(s)
                for _ in range(calls):
                    solver.state_est_step_dev(1e-3, sensors, contact, rbd_est, st, s.cuda_stream)
                b.record(s); torch.cuda.synchronize(dev)
                if rep:
                    times[mode].append(a.elapsed_time(b) / calls)
    finally:
        solver.state_est_stop(); solver.sim_set_terrain(None)
    return {"label": "device time per estimator step of %d robots with the ground map and without, median of %d alternated blocks of %d calls" % (B, reps, calls),
            "ms_per_call_map": float(np.median(times["map"])), "ms_per_call_plane": float(np.median(times["plane"])),
            "spread_map": [float(min(times["map"])), float(max(times["map"]))], "spread_plane": [float(min(times["plane"])), float(max(times["plane"]))]}


def attitude_times(solver, xy_yaw, reps=7, calls=20):
    """Device time per attitude filter call and per 1 ms plant step of the whole batch, alternated `reps` times in blocks of `calls` from one standing
    state (CUDA events) → median ms per call of each."""
    import torch
    B = solver.batch; dev = torch.device("cuda", 0); s = torch.cuda.Stream(device=dev)
    q0, v0 = solver.sim_standing_state(xy_yaw)
    q = torch.as_tensor(q0, device=dev); v = torch.as_tensor(v0, device=dev)
    eff = torch.zeros((B, 18), dtype=torch.float64, device=dev); rbd = torch.zeros((B, 55), dtype=torch.float64, device=dev)
    sensors = torch.zeros((B, 46), dtype=torch.float64, device=dev); contact = torch.zeros(B, dtype=torch.int32, device=dev); st = torch.zeros_like(contact)
    solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)
    solver.sim_read_sensors_dev(1e-3, 0, q, v, v, sensors, s.cuda_stream); torch.cuda.synchronize(dev)
    solver.attitude_reset(); solver.attitude_step_dev(1e-3, sensors, st, s.cuda_stream)   # past the first call, which only takes the reading
    times = {"attitude": [], "plant": []}
    try:
        for rep in range(reps + 1):   # the first round warms up
            for mode in ("attitude", "plant"):
                torch.cuda.synchronize(dev)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(s)
                for _ in range(calls):
                    if mode == "attitude":
                        solver.attitude_step_dev(1e-3, sensors, st, s.cuda_stream)
                    else:
                        solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)
                b.record(s); torch.cuda.synchronize(dev)
                if rep:
                    times[mode].append(a.elapsed_time(b) / calls)
    finally:
        solver.attitude_stop()
    return {"label": "device time per attitude filter call and per 1 ms plant step of %d robots, median of %d alternated blocks of %d calls" % (B, reps, calls),
            "ms_per_call": float(np.median(times["attitude"])), "ms_per_plant_step": float(np.median(times["plant"])),
            "spread": [float(min(times["attitude"])), float(max(times["attitude"]))]}


def slip_times(solver, xy_yaw, reps=7, calls=20):
    """Device time per slip detector call and per 1 ms plant step of the whole batch, alternated `reps` times in blocks of `calls` from one standing
    state past the estimator's first call (CUDA events) → median ms per call of each."""
    import torch
    B = solver.batch; dev = torch.device("cuda", 0); s = torch.cuda.Stream(device=dev)
    q0, v0 = solver.sim_standing_state(xy_yaw)
    q = torch.as_tensor(q0, device=dev); v = torch.as_tensor(v0, device=dev)
    eff = torch.zeros((B, 18), dtype=torch.float64, device=dev); rbd = torch.zeros((B, 55), dtype=torch.float64, device=dev); rbd_est = torch.zeros_like(rbd)
    sensors = torch.zeros((B, 46), dtype=torch.float64, device=dev); contact = torch.zeros(B, dtype=torch.int32, device=dev); st = torch.zeros_like(contact)
    stance, slip = torch.zeros_like(contact), torch.zeros_like(contact)
    solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)
    solver.sim_read_sensors_dev(1e-3, 0, q, v, v, sensors, s.cuda_stream); torch.cuda.synchronize(dev)
    solver.state_est_reset(q0[:, 0:3]); solver.slip_reset()
    solver.state_est_step_dev(1e-3, sensors, contact, rbd_est, st, s.cuda_stream)   # past the estimator's first call, before which the mask passes through
    times = {"slip": [], "plant": []}
    try:
        for rep in range(reps + 1):   # the first round warms up
            for mode in ("slip", "plant"):
                torch.cuda.synchronize(dev)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(s)
                for _ in range(calls):
                    if mode == "slip":
                        solver.slip_step_dev(1e-3, sensors, contact, stance, slip, st, s.cuda_stream)
                    else:
                        solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)
                b.record(s); torch.cuda.synchronize(dev)
                if rep:
                    times[mode].append(a.elapsed_time(b) / calls)
    finally:
        solver.slip_stop(); solver.state_est_stop()
    return {"label": "device time per slip detector call and per 1 ms plant step of %d robots, median of %d alternated blocks of %d calls" % (B, reps, calls),
            "ms_per_call": float(np.median(times["slip"])), "ms_per_plant_step": float(np.median(times["plant"])),
            "spread": [float(min(times["slip"])), float(max(times["slip"]))]}


def gait_commands(solver, closed_loop, B, sim_s, cmd, xy, kw, upright):
    """The switch sweep (which also warms the commands path up), then the timed run with a timeline that changes nothing, its gait step and MPC solve
    bracketed with CUDA events."""
    import torch
    targets = ("stance", "standing_trot", "flying_trot", "pace", "static_walk", "dynamic_walk", "amble"); pair = np.arange(B) % len(targets)
    sweep = dict(t=np.tile([0.5, 2.0], (B, 1)), gait=np.array([["trot", targets[p]] for p in pair], dtype=object), cmd_vel=np.tile([cmd, [np.nan] * 4], (B, 1, 1)))
    sw = closed_loop.run(solver, duration=4.0, gait="stance", cmd_vel=(0.0, 0.0, 0.0, 0.0), xy_yaw=xy, commands=sweep, **kw)
    up, bits = upright(sw), np.bitwise_or.reduce(sw["status"], axis=0)
    pairs = [{"pair": "stance -> trot -> " + g, "robots": int(np.sum(pair == i)), "fallen": int(np.sum(~up[pair == i])),
              "status_bits_or": int(np.bitwise_or.reduce(bits[pair == i]))} for i, g in enumerate(targets)]
    ev = {"gait_dev_step_dev": [], "mpc_solve_dev": []}

    def bracket(name):
        orig = getattr(solver, name)

        def call(*a, **k):
            e = [torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)]; s = torch.cuda.ExternalStream(a[-1]) if isinstance(a[-1], int) else None
            e[0].record(s); orig(*a, **k); e[1].record(s); ev[name].append(e)
        setattr(solver, name, call)
    for n in ev:
        bracket(n)
    try:
        noop = dict(t=np.full((B, 1), 0.3), gait=np.full((B, 1), None, dtype=object), cmd_vel=np.tile(cmd, (B, 1, 1)))
        torch.cuda.synchronize(); t0 = time.perf_counter()
        closed_loop.run(solver, duration=sim_s, gait="trot", cmd_vel=cmd, xy_yaw=xy, commands=noop, **kw)
        torch.cuda.synchronize(); wall = time.perf_counter() - t0
    finally:
        for n in ev:
            delattr(solver, n)
    ms = {n: float(np.median([a.elapsed_time(b) for a, b in e])) for n, e in ev.items()}
    return {"label": "timed: the run with commands that change nothing, after the sweep; per-call device times are medians over that run's calls",
            "wall_s_per_sim_s": wall / sim_s, "gait_step_ms_per_call": ms["gait_dev_step_dev"], "mpc_solve_ms_per_call": ms["mpc_solve_dev"],
            "switch_sweep": {"label": "4 s: stance, trot at cmd_vel from 0.5 s, the target gait from 2 s (each command takes effect 1 s later)", "pairs": pairs}}


def target_call_times(solver, reps=7, calls=50):
    """Device time per target call of the whole batch: the scalar entry point (kind 0 for every robot) and the per-robot one with the same kinds and
    with kinds 0 / 1 / 2 / -1 mixed, alternated `reps` times in blocks of `calls` on one set of rows (CUDA events) → median ms per call of each."""
    import torch
    B = solver.batch; dev = torch.device("cuda", 0); s = torch.cuda.Stream(device=dev); rng = np.random.default_rng(0)
    f64 = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=dev)
    cmd = np.zeros((B, 7)); cmd[:, :3] = [0.6, 0.1, 0.45]; cmd[:, 3:] = [0.5, -0.5, 0.5, -0.5]
    x = np.zeros((B, 30)); x[:, 8] = 0.45; ee = np.tile([0.52, 0.09, 0.44, 0.5, -0.5, 0.5, -0.5], (B, 1))
    rows = [f64(cmd), f64(np.full(B, 10.0)), f64(x), f64(ee), f64(ee), torch.zeros(B, dtype=torch.int32, device=dev), torch.zeros((B, 4), dtype=torch.float64, device=dev),
            torch.zeros((B, 4, 37), dtype=torch.float64, device=dev)]
    kinds = {"scalar": 0, "per_robot": torch.zeros(B, dtype=torch.int32, device=dev),
             "per_robot_mixed": torch.as_tensor(rng.integers(-1, 3, B).astype(np.int32), device=dev)}
    times = {k: [] for k in kinds}
    for rep in range(reps + 1):   # the first round warms up
        for name, kind in kinds.items():
            torch.cuda.synchronize(dev)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(s)
            for _ in range(calls):
                solver.target_trajectories_dev(kind, *rows, s.cuda_stream)
            b.record(s); torch.cuda.synchronize(dev)
            if rep:
                times[name].append(a.elapsed_time(b) / calls)
    return {"label": "device time per target call of %d robots, median of %d alternated blocks of %d calls" % (B, reps, calls),
            **{"ms_per_call_" + k: float(np.median(v)) for k, v in times.items()}, "spread_per_robot": [float(min(times["per_robot"])), float(max(times["per_robot"]))]}


def ee_paths_main(args, duration=4.0, t_first=0.5, gap=0.75):
    """End-effector paths (DESIGN.md §4.20): the target call of the whole batch without path robots (kinds 0 / 1 / 2 / -1 mixed, the per-robot call)
    and with every robot following a path (the path call), alternated blocks of CUDA events, medians; then every robot standing in the heading frame
    traces a 10 cm square (4 waypoints gap s apart from t_first, from the standing hand's pose at t_first, read from a first run of t_first s): the
    hand's position error against p(t) between the first and the last waypoint and at the end (the final waypoint held), p50 / p95, and the wall
    seconds per simulated second of the same loop with and without the path."""
    import time
    import torch
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    B = args.batch; solver = q.Solver(batch=B, device=0); dev = torch.device("cuda", 0); st = torch.cuda.Stream(device=dev); rng = np.random.default_rng(0)
    f64 = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=dev)
    xy = np.c_[np.arange(B) * 2.0, np.zeros(B), np.zeros(B)]
    r = closed_loop.run(solver, duration=t_first, gait="stance", xy_yaw=xy, ee_frame="heading")
    hand = np.r_[r["ee"][-1, 0, :2] - r["base"][-1, 0, :2], r["ee"][-1, 0, 2:7]]   # robot 0's standing hand relative to its base (yaw 0)
    corners = hand[:3] + np.array([[0.1, 0, 0], [0.1, 0.1, 0], [0, 0.1, 0], [0, 0, 0]])
    tau = gap * np.arange(1, 5); paths = [(tau, np.c_[corners, np.tile(hand[3:7], (4, 1))])]
    solver.set_ee_paths(paths)
    cmd = np.zeros((B, 7)); cmd[:, :3] = [0.6, 0.1, 0.45]; cmd[:, 3:] = [0.5, -0.5, 0.5, -0.5]
    x = np.zeros((B, 30)); x[:, 8] = 0.45; x[:, 9] = rng.uniform(-np.pi, np.pi, B); ee = np.tile([0.52, 0.09, 0.44, 0.5, -0.5, 0.5, -0.5], (B, 1))
    ps = np.zeros((B, _lib.EE_PATH_STATE)); ps[:, 1] = 10.0 - rng.uniform(0.0, 3.0, B); ps[:, 4] = x[:, 9]; ps[:, 5:] = ee
    rows = [f64(cmd), f64(np.full(B, 10.0)), f64(x), f64(ee), f64(ee), torch.zeros(B, dtype=torch.int32, device=dev), torch.zeros((B, 4), dtype=torch.float64, device=dev),
            torch.zeros((B, 4, 37), dtype=torch.float64, device=dev)]
    settings = {"no_path_robots": (torch.as_tensor(rng.integers(-1, 3, B).astype(np.int32), device=dev), None),
                "every_robot_following": (torch.full((B,), _lib.TARGET_EE_PATH_FOLLOW, dtype=torch.int32, device=dev), f64(ps))}
    times = {k: [] for k in settings}; reps, calls = 7, 50
    for rep in range(reps + 1):   # the first round warms up
        for name, (kind, path_state) in settings.items():
            kw = {} if path_state is None else dict(path_state=path_state)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(st)
            for _ in range(calls):
                solver.target_trajectories_dev(kind, *rows, st.cuda_stream, **kw)
            b.record(st); torch.cuda.synchronize(dev)
            if rep:
                times[name].append(a.elapsed_time(b) / calls)
    solver.set_ee_paths(None)
    out = {"card": card(), "target_call": {"label": "device ms per target call of %d robots, median of %d alternated blocks of %d calls" % (B, reps, calls),
                                           **{k: float(np.median(v)) for k, v in times.items()}}}
    wall = {}
    for name, kw in (("without_path", dict(steer=True)),
                     ("with_path", dict(ee_paths=paths, commands=dict(t=np.full((B, 1), t_first), gait=[[None]] * B, ee_path=np.zeros((B, 1), dtype=np.int64))))):
        solver.mpc_reset(); solver.wbc_set_input_last(None)
        with closed_loop.Session(solver, duration, gait="stance", xy_yaw=xy, ee_frame="heading", **kw) as ss:
            torch.cuda.synchronize(dev); t0 = time.perf_counter()
            rec = ss.step(ss.windows); ss.stream.synchronize(); wall[name] = (time.perf_counter() - t0) / duration
            rec = {k: (v if isinstance(v, np.ndarray) else v.cpu().numpy()) for k, v in rec.items()}
            p = ss.path_state.cpu().numpy() if ss.path_state is not None else None
            ss.finish()
    t = rec["t"]; ref = np.zeros((len(t), B, 3))
    for c in range(3):
        ref[..., c] = np.interp(t[:, None] - p[None, :, 1], tau, paths[0][1][:, c])
    cs, sn = np.cos(p[:, 4]), np.sin(p[:, 4])
    world = np.stack([cs * ref[..., 0] - sn * ref[..., 1] + p[:, 2], sn * ref[..., 0] + cs * ref[..., 1] + p[:, 3], ref[..., 2]], -1)
    err = np.linalg.norm(rec["ee"][..., :3] - world, axis=-1) * 1e3
    along = (t[:, None] >= p[None, :, 1] + tau[0]) & (t[:, None] <= p[None, :, 1] + tau[-1])
    base = rec["base"]; up = np.all(np.isfinite(base), axis=(0, 2)) & (np.min(base[:, :, 2], axis=0) > 0.3)
    out["square"] = {"robots": B, "frame": "heading", "side_m": 0.1, "gap_s": gap, "fallen": int(np.sum(~up)), "status_robots": int(np.sum(np.any(rec["status"] != 0, axis=0))),
                     "along_path_mm_p50_p95": [float(v) for v in np.percentile(err[along], [50, 95])],
                     "final_waypoint_mm_p50_p95": [float(v) for v in np.percentile(err[-1], [50, 95])],
                     "wall_s_per_sim_s": wall}
    print(json.dumps(out))


def ee_path_draw_main(args, track_s=4.0, box=0.05):
    """Per-episode end-effector paths (DESIGN.md §4.21): the sampler's device time for one draw of every robot against one 1 ms plant step of the batch
    (alternated blocks of CUDA events, medians); the wall seconds per simulated second of --duration respawning runs of --gait at --vx (respawn after
    0.1 s fallen or 1 s) with and without a heading-frame path draw per episode, alternated twice after a warm-up pair; and 256 standing heading robots on
    drawn 4-waypoint paths in a +-box m box about the standing hand: the hand's position error against p(t) from the first to the last waypoint, p50 / p95."""
    import torch
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    if not torch.cuda.is_available():
        raise SystemExit("bench_closedloop.py: no CUDA device — the product path has no CPU fallback")
    dev = torch.device("cuda", 0); B = args.batch; solver = q.Solver(batch=B, device=0); st = torch.cuda.Stream(device=dev)
    xy = np.zeros((B, 3)); xy[:, 0] = 2.0 * (np.arange(B) % 64); xy[:, 1] = 2.0 * (np.arange(B) // 64)
    r = closed_loop.run(solver, duration=0.5, gait="stance", xy_yaw=xy, ee_frame="heading")
    hand = np.r_[r["ee"][-1, 0, :2] - r["base"][-1, 0, :2], r["ee"][-1, 0, 2:7]]   # robot 0's standing hand relative to its base (yaw 0)
    spec = dict(seed=1, n=4, tau_first=(0.5, 0.6), gap=(0.6, 0.8), yaw=(-0.3, 0.3), quat=hand[3:7], **{c: (hand[i] - box, hand[i] + box) for i, c in enumerate("xyz")})
    # per call: the sampler on a running device gait schedule, and the plant step
    pd = closed_loop._ee_path_draw_spec(B, solver.time_horizon, spec)
    solver.gait_dev_set_templates(closed_loop.gait_template_names()); solver.gait_dev_reset(np.zeros(B, dtype=np.int32), np.full(B, 10.0))
    solver.ee_path_set_ranges(*closed_loop._ee_path_box(pd, B), 1)
    q0, v0 = solver.sim_standing_state(xy); qq = torch.as_tensor(q0, device=dev); vv = torch.as_tensor(v0, device=dev)
    eff = torch.zeros((B, 18), dtype=torch.float64, device=dev); rbd = torch.zeros((B, 55), dtype=torch.float64, device=dev)
    contact = torch.zeros(B, dtype=torch.int32, device=dev); sst = torch.zeros_like(contact)
    every = torch.ones_like(contact); episode = torch.zeros_like(contact); rows = torch.zeros((B, _lib.EE_PATH_MAX, 8), dtype=torch.float64, device=dev)
    calls_of = {"ee_path_sample": lambda: (episode.add_(1), solver.ee_path_sample_dev(every, episode, rows, st.cuda_stream)),
                "plant": lambda: solver.sim_step_dev(1e-3, eff, qq, vv, rbd, contact, sst, st.cuda_stream)}
    times = {k: [] for k in calls_of}; reps, calls = 7, 20
    with torch.cuda.stream(st):
        for rep in range(reps + 1):   # the first round warms up
            for mode, call in calls_of.items():
                torch.cuda.synchronize(dev)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(st)
                for _ in range(calls):
                    call()
                b.record(st); torch.cuda.synchronize(dev)
                if rep:
                    times[mode].append(a.elapsed_time(b) / calls)
    solver.ee_path_set_ranges(None); solver.gait_dev_stop()
    per_call = {"label": "device time per call on %d robots (every robot drawing 4 waypoints), median of %d alternated blocks of %d calls" % (B, reps, calls),
                **{"ms_per_%s" % k: float(np.median(v)) for k, v in times.items()}, "spread_ee_path_sample": [float(min(times["ee_path_sample"])), float(max(times["ee_path_sample"]))]}
    # wall time of a respawning trot with and without the draws
    kw = dict(gait=args.gait, cmd_vel=np.array([args.vx, 0.0, 0.0, 0.0]), xy_yaw=xy, ee_frame="heading", respawn=dict(hold=0.1, every=1.0))
    wall = {"without_draw": [], "with_draw": []}
    for rep in range(3):   # the first round warms up
        for name, extra in (("without_draw", {}), ("with_draw", dict(ee_path_draw=spec))):
            solver.mpc_reset(); solver.wbc_set_input_last(None); torch.cuda.synchronize(dev); t0 = time.perf_counter()
            closed_loop.run(solver, duration=args.duration, **kw, **extra); torch.cuda.synchronize(dev)
            if rep:
                wall[name].append((time.perf_counter() - t0) / args.duration)
    # tracking: 256 standing heading robots on drawn paths
    n = min(B, 256); s2 = q.Solver(batch=n, device=0); xy2 = xy[:n]
    with closed_loop.Session(s2, track_s, gait="stance", xy_yaw=xy2, ee_frame="heading", ee_path_draw=spec) as ss:
        rec = ss.step(ss.windows); ss.stream.synchronize(); p = ss.path_state.cpu().numpy(); end = ss.finish()
    rec = {k: (v if isinstance(v, np.ndarray) else v.cpu().numpy()) for k, v in rec.items()}
    way = end["ee_path_params"][:, 0]; t = rec["t"]; ref = np.zeros((len(t), n, 3))
    for b in range(n):
        for c in range(3):
            ref[:, b, c] = np.interp(t - p[b, 1], way[b, :, 0], way[b, :, 1 + c])
    cs, sn = np.cos(p[:, 4]), np.sin(p[:, 4])
    world = np.stack([cs * ref[..., 0] - sn * ref[..., 1] + p[:, 2], sn * ref[..., 0] + cs * ref[..., 1] + p[:, 3], ref[..., 2]], -1)
    err = np.linalg.norm(rec["ee"][..., :3] - world, axis=-1) * 1e3
    along = (t[:, None] >= p[None, :, 1] + way[None, :, 0, 0]) & (t[:, None] <= p[None, :, 1] + way[None, :, -1, 0])
    base = rec["base"]; up = np.all(np.isfinite(base), axis=(0, 2)) & (np.min(base[:, :, 2], axis=0) > 0.3)
    name, limit = card()
    print(json.dumps({"metric": "ee_path_draw", "gpu": name, "power_limit": limit, "batch": B, "per_call": per_call,
                      "wall_s_per_sim_s": {"label": "%s at %.2f m/s, heading frame, respawn after 0.1 s fallen or 1 s, runs of %.1f s, two alternated pairs after a "
                                                    "warm-up pair" % (args.gait, args.vx, args.duration), **wall},
                      "tracking": {"robots": n, "frame": "heading", "box_m": box, "waypoints": 4, "fallen": int(np.sum(~up)),
                                   "status_robots": int(np.sum(np.any(rec["status"] != 0, axis=0))),
                                   "along_path_mm_p50_p95": [float(v) for v in np.percentile(err[along], [50, 95])]}}))


def ee_frame_main(args, sweep_s=4.0):
    """End-effector targets in the heading frame (DESIGN.md §4.19): the target call of the whole batch (kinds 0 / 1 / 2 / -1 mixed) with no frame rows,
    all-world rows and all-heading rows, alternated blocks of CUDA events, medians; then the turning sweep (start yaws over [-pi, pi], yaw rates
    +-0.5 / +-1 rad/s, trot 0.3 m/s, sweep_s s) in both frames: fallen robots and QMB200_ST_OVERFLOW per frame and yaw rate."""
    import torch
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    B = args.batch; solver = q.Solver(batch=B, device=0); dev = torch.device("cuda", 0); st = torch.cuda.Stream(device=dev); rng = np.random.default_rng(0)
    f64 = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=dev)
    cmd = np.zeros((B, 7)); cmd[:, :3] = [0.6, 0.1, 0.45]; cmd[:, 3:] = [0.5, -0.5, 0.5, -0.5]
    x = np.zeros((B, 30)); x[:, 8] = 0.45; x[:, 9] = rng.uniform(-np.pi, np.pi, B); ee = np.tile([0.52, 0.09, 0.44, 0.5, -0.5, 0.5, -0.5], (B, 1))
    rows = [f64(cmd), f64(np.full(B, 10.0)), f64(x), f64(ee), f64(ee), torch.zeros(B, dtype=torch.int32, device=dev), torch.zeros((B, 4), dtype=torch.float64, device=dev),
            torch.zeros((B, 4, 37), dtype=torch.float64, device=dev)]
    kind = torch.as_tensor(rng.integers(-1, 3, B).astype(np.int32), device=dev)
    settings = {"no_rows": None, "world_rows": np.zeros(B, dtype=np.int32), "heading_rows": np.ones(B, dtype=np.int32)}
    times = {k: [] for k in settings}; reps, calls = 7, 50
    for rep in range(reps + 1):   # the first round warms up
        for name, frame in settings.items():
            solver.set_ee_frame(frame); torch.cuda.synchronize(dev)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(st)
            for _ in range(calls):
                solver.target_trajectories_dev(kind, *rows, st.cuda_stream)
            b.record(st); torch.cuda.synchronize(dev)
            if rep:
                times[name].append(a.elapsed_time(b) / calls)
    solver.set_ee_frame(None)
    out = {"card": card(), "target_call": {"label": "device ms per target call of %d robots (kinds mixed), median of %d alternated blocks of %d calls" % (B, reps, calls),
                                           **{k: float(np.median(v)) for k, v in times.items()}}}
    rates = np.array([-1.0, -0.5, 0.5, 1.0])[np.arange(B) % 4]
    xy = np.c_[np.arange(B) * 3.0, np.zeros(B), -np.pi + 2 * np.pi * np.arange(B) / B]
    cmd_vel = np.c_[np.full(B, 0.3), np.zeros(B), np.zeros(B), rates]
    for frame in ("world", "heading"):
        solver.mpc_reset(); solver.wbc_set_input_last(None)
        r = closed_loop.run(solver, duration=sweep_s, gait="trot", cmd_vel=cmd_vel, xy_yaw=xy, ee_frame=frame)
        base = r["base"]; up = np.all(np.isfinite(base), axis=(0, 2)) & (np.min(base[:, :, 2], axis=0) > 0.3)
        stw = np.bitwise_or.reduce(r["status"], axis=0); ovf = (stw & _lib.ST_OVERFLOW) != 0
        out["turning_" + frame] = {str(w): {"robots": int(np.sum(rates == w)), "fallen": int(np.sum(~up & (rates == w))), "overflow": int(np.sum(ovf & (rates == w)))}
                                   for w in (-1.0, -0.5, 0.5, 1.0)}
    print(json.dumps(out))


def ee_goals(solver, closed_loop, B, sim_s, xy, upright, tuning=False):
    """The reach sweep, the target call times, then the runs of sim_s with the goals and with a timeline that changes nothing (wall time).  With tuning
    also the reach sweep again under per-robot tuning rows (ee_tuning_sweep)."""
    import torch
    b = np.arange(B); bins = dict(dx_m=np.array([-0.1, 0.0, 0.1, 0.2, 0.3, 0.4]), dz_m=np.array([-0.1, 0.0, 0.1]), rot_deg=np.array([0.0, 10.0, 20.0]))
    idx = dict(dx_m=b % 6, dz_m=(b // 6) % 3, rot_deg=(b // 18) % 3)
    ee0 = closed_loop.run(solver, duration=0.01, gait="stance", xy_yaw=xy)["start_ee"]
    goal = ee0.copy(); goal[:, 0] += bins["dx_m"][idx["dx_m"]]; goal[:, 2] += bins["dz_m"][idx["dz_m"]]
    half = np.radians(bins["rot_deg"][idx["rot_deg"]]) / 2; axis = np.array([1.0, 1.0, 1.0]) / np.sqrt(3.0)
    rq = np.c_[np.outer(np.sin(half), axis), np.cos(half)]; qx, qy, qz, qw = ee0[:, 3:].T; rx, ry, rz, rw = rq.T   # goal orientation: rq * start's
    goal[:, 3:] = np.c_[rw * qx + rx * qw + ry * qz - rz * qy, rw * qy - rx * qz + ry * qw + rz * qx, rw * qz + rx * qy - ry * qx + rz * qw, rw * qw - rx * qx - ry * qy - rz * qz]
    goal[:, 3:] /= np.linalg.norm(goal[:, 3:], axis=1, keepdims=True)
    sweep = dict(t=np.tile([0.2, 2.5], (B, 1)), gait=np.tile(np.array([None, "stance"], dtype=object), (B, 1)), ee_goal=np.stack([goal, np.full((B, 7), np.nan)], 1))
    solver.mpc_reset(); solver.wbc_set_input_last(None)
    r = closed_loop.run(solver, duration=5.0, gait="trot", xy_yaw=xy, commands=sweep)
    pe = np.linalg.norm(r["ee"][-1, :, :3] - goal[:, :3], axis=1)
    oe = np.degrees(2.0 * np.arccos(np.clip(np.abs(np.sum(r["ee"][-1, :, 3:] * goal[:, 3:], axis=1)), 0.0, 1.0)))
    up, bits = upright(r), np.bitwise_or.reduce(r["status"], axis=0)
    pct = lambda a: [float(np.percentile(a, 50)), float(np.percentile(a, 95))]
    sweep_bins = {axis: [{"value": float(val), "robots": int(np.sum(idx[axis] == i)), "fallen": int(np.sum(~up[idx[axis] == i])),
                          "pos_err_m_p50_p95": pct(pe[idx[axis] == i]), "ori_err_deg_p50_p95": pct(oe[idx[axis] == i]),
                          "status_bits_or": int(np.bitwise_or.reduce(bits[idx[axis] == i]))} for i, val in enumerate(bins[axis])] for axis in bins}
    walls = {}
    for name, cmds in (("with_goals", dict(t=np.full((B, 1), 0.2), gait=np.full((B, 1), None, dtype=object), ee_goal=goal[:, None])),
                       ("timeline_that_changes_nothing", dict(t=np.full((B, 1), 0.2), gait=np.full((B, 1), None, dtype=object)))):
        solver.mpc_reset(); solver.wbc_set_input_last(None)
        torch.cuda.synchronize(); t0 = time.perf_counter()
        closed_loop.run(solver, duration=sim_s, gait="stance", xy_yaw=xy, commands=cmds)
        torch.cuda.synchronize(); walls[name] = (time.perf_counter() - t0) / sim_s
    return {"reach_sweep": {"label": "5 s: trot from the start at yaw 0, one goal at 0.2 s (offset from the start pose), stance commanded at 2.5 s (in force from 3.5 s); "
                                     "errors of the end effector against the goal at the end; fallen = min base z <= 0.3 m or |roll|, |pitch| >= 0.3 rad or non-finite",
                            "bins": sweep_bins, "fallen": int(np.sum(~up)), "pos_err_m_p50_p95": pct(pe), "ori_err_deg_p50_p95": pct(oe)},
            **({"ee_tuning_sweep": ee_tuning_sweep(solver, closed_loop, B, xy, upright, sweep, goal, idx["dz_m"], idx["rot_deg"])} if tuning else {}),
            "target_call": target_call_times(solver),
            "wall_s_per_sim_s": {"label": "stance runs of %.2f s from a cold MPC / WBC state" % sim_s, **walls}}


def ee_tuning_sweep(solver, closed_loop, B, xy, upright, sweep, goal, dz_bin, rot_bin):
    """The reach sweep of ee_goals again, each robot with its own tuning row: the MPC's end-effector weights (mu_ee_pos / ori and the final ones, scaled
    together), the WBC's end-effector gains (kp / kd of ee_linear and ee_angular, scaled together) and the control law's kd_arm_wbc.  The tuning index is
    b // 54, so every tuning bin holds every goal bin of ee_goals (period 54) alike.  Errors at the end per bin of each axis and per cell."""
    b = np.arange(B); h = solver.get_handle_tuning(); L = _lib.TUNING_LAYOUT
    bins = dict(mu_ee_scale=np.array([0.5, 1.0, 2.0, 4.0]), wbc_ee_gain_scale=np.array([0.5, 1.0, 2.0]), kd_arm_wbc=np.array([0.5, 2.0]))
    cell = (b // 54) % 24; idx = dict(mu_ee_scale=cell % 4, wbc_ee_gain_scale=(cell // 4) % 3, kd_arm_wbc=cell // 12)
    rows = np.repeat(h[None], B, axis=0)
    for k in ("mu_ee_pos", "mu_ee_ori", "mu_final_ee_pos", "mu_final_ee_ori"):
        rows[:, L[k][0]] *= bins["mu_ee_scale"][idx["mu_ee_scale"]]
    for k in ("kp_ee_linear", "kd_ee_linear", "kp_ee_angular", "kd_ee_angular"):
        off, w = L[k]; rows[:, off:off + w] *= bins["wbc_ee_gain_scale"][idx["wbc_ee_gain_scale"]][:, None]
    rows[:, L["kd_arm_wbc"][0]] = bins["kd_arm_wbc"][idx["kd_arm_wbc"]]
    solver.mpc_reset(); solver.wbc_set_input_last(None)
    r = closed_loop.run(solver, duration=5.0, gait="trot", xy_yaw=xy, commands=sweep,
                        tuning={k: rows[:, off] if w == 1 else rows[:, off:off + w] for k, (off, w) in L.items()})
    pe = np.linalg.norm(r["ee"][-1, :, :3] - goal[:, :3], axis=1)
    oe = np.degrees(2.0 * np.arccos(np.clip(np.abs(np.sum(r["ee"][-1, :, 3:] * goal[:, 3:], axis=1)), 0.0, 1.0)))
    up = upright(r); pct = lambda a: [float(np.percentile(a, 50)), float(np.percentile(a, 95))]
    def stats(m):
        return {"robots": int(np.sum(m)), "fallen": int(np.sum(~up[m])), "pos_err_m_p50_p95": pct(pe[m]), "ori_err_deg_p50_p95": pct(oe[m])}
    hard = (dz_bin == 2) | (rot_bin == 2)   # the goals the untuned sweep misses most: 10 cm up or turned 20 degrees
    return {"label": "the reach sweep of ee_goals with per-robot tuning rows; scales multiply the handle's values (scale 1 and kd_arm_wbc 0.5 = the handle's own); "
                     "hard_goals = dz +0.1 m or 20 degrees",
            "bins": {axis: [{"value": float(v), **stats(idx[axis] == i), "hard_goals": stats((idx[axis] == i) & hard)} for i, v in enumerate(bins[axis])] for axis in bins},
            "cells": [{"mu_ee_scale": float(bins["mu_ee_scale"][c % 4]), "wbc_ee_gain_scale": float(bins["wbc_ee_gain_scale"][(c // 4) % 3]),
                       "kd_arm_wbc": float(bins["kd_arm_wbc"][c // 12]), **stats(cell == c), "hard_goals": stats((cell == c) & hard)} for c in range(24)],
            "fallen": int(np.sum(~up))}


def respawn_times(solver, xy_yaw, reps=7, calls=20):
    """Device time per fall detector call, per image restore (every robot masked, and none) and per 1 ms plant step of the whole batch, alternated
    `reps` times in blocks of `calls` from one standing state, with the state estimator running and imaged (CUDA events) → median ms per call of each."""
    import torch
    B = solver.batch; dev = torch.device("cuda", 0); s = torch.cuda.Stream(device=dev)
    q0, v0 = solver.sim_standing_state(xy_yaw)
    q = torch.as_tensor(q0, device=dev); v = torch.as_tensor(v0, device=dev)
    eff = torch.zeros((B, 18), dtype=torch.float64, device=dev); rbd = torch.zeros((B, 55), dtype=torch.float64, device=dev)
    contact = torch.zeros(B, dtype=torch.int32, device=dev); st = torch.zeros_like(contact); count = torch.zeros_like(contact); fallen = torch.zeros_like(contact)
    every, none = torch.ones_like(contact), torch.zeros_like(contact)
    solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream); torch.cuda.synchronize(dev)
    solver.hw_set_delay(0.009); solver.state_est_reset(q0[:, 0:3]); solver.robot_image_save()
    calls_of = {"fall_detect": lambda: solver.fall_detect_dev(rbd, count, fallen, 0.3, 0.3, s.cuda_stream),
                "restore_all": lambda: solver.robot_image_restore_dev(every, s.cuda_stream), "restore_none": lambda: solver.robot_image_restore_dev(none, s.cuda_stream),
                "plant": lambda: solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)}
    times = {k: [] for k in calls_of}
    try:
        for rep in range(reps + 1):   # the first round warms up
            for mode, call in calls_of.items():
                torch.cuda.synchronize(dev)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(s)
                for _ in range(calls):
                    call()
                b.record(s); torch.cuda.synchronize(dev)
                if rep:
                    times[mode].append(a.elapsed_time(b) / calls)
    finally:
        solver.robot_image_clear(); solver.state_est_stop()
    return {"label": "device time per call on %d robots, median of %d alternated blocks of %d calls; the image holds the state estimator's rows" % (B, reps, calls),
            **{"ms_per_%s" % k: float(np.median(v)) for k, v in times.items()}, "spread_restore_all": [float(min(times["restore_all"])), float(max(times["restore_all"]))]}


def respawn_rates(r, ep_s=1.0):
    """Episode statistics of a closed_loop.run(respawn=...) result: episodes per robot, falls per robot-second and, for first and later episodes apart,
    the fraction of episodes that fall within their first ep_s seconds.  Only episodes that start at least ep_s before the run's end count, fallen or
    not: an episode that starts later is cut off by the run whatever its outcome, and counting it only when it falls would bias the later episodes'
    fraction upwards (first episodes all start at 0)."""
    ep, fl = r["episode"], r["fallen"].astype(bool); ticks, B = ep.shape; w = int(round(ep_s * 100))
    falls = 0; first = [0, 0]; later = [0, 0]
    for b in range(B):
        for e in range(int(ep[-1, b]) + 1):
            rows = np.flatnonzero(ep[:, b] == e); f = fl[rows, b]
            falls += int(f.any())
            if rows[0] + w <= ticks:   # its first ep_s seconds lie inside the run
                box = first if e == 0 else later; box[0] += int(f[:w].any()); box[1] += 1
    frac = lambda a: {"fell": a[0], "episodes": a[1], "fraction": a[0] / a[1] if a[1] else None,
                      "binomial_sd": float(np.sqrt(a[0] / a[1] * (1 - a[0] / a[1]) / a[1])) if a[1] else None}
    return {"episodes_per_robot": float(np.mean(ep[-1] + 1)), "falls_per_robot_s": falls / (B * ticks * 0.01), "falls": falls,
            "fell_within_%gs_first_episodes" % ep_s: frac(first), "fell_within_%gs_later_episodes" % ep_s: frac(later)}


RANDOMIZE = dict(seed=0, friction_mu=(0.15, 1.0), m_ee=(0.0, 2.0), push_t_on=(0.2, 0.5), push_duration=(0.1, 0.1), f_base_x=(-180.0, 180.0), f_base_y=(-180.0, 180.0))
MU_BINS, PUSH_BINS = [0.15, 0.3, 0.45, 0.6, 0.8, 1.0], [0.0, 60.0, 120.0, 180.0, 255.0]


def episode_times(solver, xy_yaw, reps=7, calls=20):
    """Device time per sampler call (every robot masked, and none) and per image restore of every robot, alternated `reps` times in blocks of `calls`
    (CUDA events), with RANDOMIZE's ranges and the state estimator running and imaged → median ms per call of each."""
    import torch
    B = solver.batch; dev = torch.device("cuda", 0); s = torch.cuda.Stream(device=dev)
    q0, _ = solver.sim_standing_state(xy_yaw)
    EP = {n: i for i, n in enumerate(_lib.EPISODE_LAYOUT)}; lo = np.zeros((B, _lib.EPISODE)); lo[:, EP["friction_mu"]] = 0.6; hi = lo.copy()
    for k, v in RANDOMIZE.items():
        if k != "seed":
            lo[:, EP[k]], hi[:, EP[k]] = v
    every = torch.ones(B, dtype=torch.int32, device=dev); none = torch.zeros_like(every); ep = torch.zeros_like(every)
    rows = torch.zeros((B, _lib.EPISODE), dtype=torch.float64, device=dev)
    prev = solver.sim_get_robot_params()
    solver.hw_set_delay(0.009); solver.state_est_reset(q0[:, 0:3]); solver.robot_image_save(); solver.episode_set_ranges(lo, hi, 0)
    calls_of = {"sample_all": lambda: solver.episode_sample_dev(every, ep, rows, 0, s.cuda_stream), "sample_none": lambda: solver.episode_sample_dev(none, ep, rows, 0, s.cuda_stream),
                "restore_all": lambda: solver.robot_image_restore_dev(every, s.cuda_stream)}
    times = {k: [] for k in calls_of}
    try:
        for rep in range(reps + 1):   # the first round warms up
            for mode, call in calls_of.items():
                torch.cuda.synchronize(dev)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(s)
                for _ in range(calls):
                    call()
                b.record(s); torch.cuda.synchronize(dev)
                if rep:
                    times[mode].append(a.elapsed_time(b) / calls)
    finally:
        solver.episode_set_ranges(None); solver.sim_set_robot_params(**prev); solver.robot_image_clear(); solver.state_est_stop()
    return {"label": "device time per call on %d robots, median of %d alternated blocks of %d calls; the image holds the state estimator's rows" % (B, reps, calls),
            **{"ms_per_%s" % k: float(np.median(v)) for k, v in times.items()}, "spread_sample_all": [float(min(times["sample_all"])), float(max(times["sample_all"]))]}


def randomize_falls(r, ep_s=1.0):
    """Per friction bin x push-magnitude bin of a closed_loop.run(respawn=..., randomize=RANDOMIZE) result: the episodes that start at least ep_s before
    the run's end and how many of them fall within their first ep_s seconds"""
    ep, fl, P = r["episode"], r["fallen"].astype(bool), r["episode_params"]; ticks, B = ep.shape; w = int(round(ep_s * 100))
    EP = {n: i for i, n in enumerate(_lib.EPISODE_LAYOUT)}
    fell = np.zeros((len(MU_BINS) - 1, len(PUSH_BINS) - 1), dtype=int); n = np.zeros_like(fell)
    for b in range(B):
        for e in range(int(ep[-1, b]) + 1):
            rows = np.flatnonzero(ep[:, b] == e)
            if rows[0] + w > ticks:
                continue
            mu = P[b, e, EP["friction_mu"]]; f = np.hypot(P[b, e, EP["f_base_x"]], P[b, e, EP["f_base_y"]])
            i = min(np.searchsorted(MU_BINS, mu, side="right") - 1, len(MU_BINS) - 2); j = min(np.searchsorted(PUSH_BINS, f, side="right") - 1, len(PUSH_BINS) - 2)
            n[i, j] += 1; fell[i, j] += int(fl[rows[:w], b].any())
    return {"mu_bins": MU_BINS, "push_bins_N": PUSH_BINS, "episodes": n.tolist(), "fell": fell.tolist(),
            "fraction": np.where(n > 0, fell / np.maximum(n, 1), np.nan).round(4).tolist(), "total_episodes": int(n.sum()), "total_fell": int(fell.sum())}


def randomize_main(args, solver, kw, xy, timed, episode_run_s=5.0):
    """--respawn --randomize: the same loop with RANDOMIZE drawn per episode.  One run of episode_run_s for the falls per bin; the wall time per
    simulated second of --duration runs with and without randomize (both with respawn), alternated twice after one warm-up run of each; the sampler's
    per-call device time."""
    wall = {False: [], True: []}
    for rep in range(3):   # the first round warms up
        for rnd in (False, True):
            _, w = timed(True, args.duration, randomize=RANDOMIZE if rnd else None)
            if rep:
                wall[rnd].append(w)
    r, _ = timed(True, episode_run_s, randomize=RANDOMIZE)
    name, limit = card()
    print(json.dumps({"metric": "randomize", "gpu": name, "power_limit": limit, "batch": solver.batch,
                      "config": "%s at %.2f m/s on the state estimate, reference IMU noise, no attitude filter; respawn after 0.1 s fallen; per episode: friction_mu "
                                "U[0.15, 1.0], m_ee U[0, 2] kg, base push f_x, f_y U[-180, 180] N for 0.1 s from t_on U[0.2, 0.5] s" % (args.gait, args.vx),
                      "simulated_s": episode_run_s, "episodes_per_robot": float(np.mean(r["episode"][-1] + 1)),
                      "fell_within_1s": randomize_falls(r),
                      "wall_s_per_sim_s": {"label": "runs of %.1f s with respawn, two alternated pairs after a warm-up pair" % args.duration,
                                           "without_randomize": wall[False], "with_randomize": wall[True]},
                      "per_call": episode_times(solver, xy)}))


SPAWN_TILES = ("flat", "ramp_10deg", "stairs_6cm", "rough_2cm")
SPAWN = dict(seed=0, tile=(0, 3), dx=(-0.5, 0.0), dy=(-0.2, 0.2), yaw=(-np.pi, np.pi))


def spawn_terrain(xy):
    """the --spawn library and every robot's run row: tile 0 (flat) centred under its start"""
    from qm_control_b200 import terrain as T
    tiles = np.stack([T.flat(), T.ramp(10.0, start=0.35), T.stairs(0.06, 0.25, start=0.35), T.rough(0.02, seed=1, flat_radius=0.35)])
    return dict(tiles=tiles, cell=T.CELL, tile=np.zeros(len(xy), dtype=np.int32), origin=T.centred_origin(xy[:, :2]))


def spawn_times(solver, ter, xy_yaw, reps=7, calls=20):
    """Device time per spawn call (every robot masked, and none) on SPAWN's ranges with the state estimator, attitude filter and slip detector running
    and the ground-map link, against the plant step on the same library, alternated `reps` times in blocks of `calls` (CUDA events) → median ms per call"""
    import torch
    B = solver.batch; dev = torch.device("cuda", 0); s = torch.cuda.Stream(device=dev)
    solver.sim_set_terrain(ter["tiles"], ter["cell"]); solver.sim_set_robot_terrain(ter["tile"], ter["origin"]); solver.state_est_set_ground(ter["tile"], ter["origin"])
    q0, v0 = solver.sim_standing_state(xy_yaw)
    solver.state_est_reset(q0[:, 0:3]); solver.attitude_reset(); solver.slip_reset()
    lo = np.zeros((B, _lib.SPAWN)); hi = np.zeros((B, _lib.SPAWN))
    for i, k in enumerate(_lib.SPAWN_LAYOUT):
        lo[:, i], hi[:, i] = SPAWN[k]
    solver.spawn_set_ranges(lo, hi, 0)
    f64 = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=dev)
    q0t = f64(q0); q = q0t.clone(); v = f64(v0); rbd = torch.zeros((B, 55), dtype=torch.float64, device=dev); x_obs = torch.zeros((B, 30), dtype=torch.float64, device=dev)
    last_ee = f64(solver.initial_ee_target()); rbd_est = torch.zeros_like(rbd); rows = torch.zeros((B, _lib.SPAWN), dtype=torch.float64, device=dev)
    contact = torch.zeros(B, dtype=torch.int32, device=dev); st = torch.zeros_like(contact); eff = torch.zeros((B, 18), dtype=torch.float64, device=dev)
    every = torch.ones(B, dtype=torch.int32, device=dev); none = torch.zeros_like(every); ep = torch.arange(B, dtype=torch.int32, device=dev)
    spawn = lambda m: solver.spawn_sample_dev(m, ep, rows, q, v, rbd, contact, x_obs, last_ee, rbd_est, _lib.SPAWN_GROUND_MAP, s.cuda_stream)
    calls_of = {"spawn_all": lambda: spawn(every), "spawn_none": lambda: spawn(none),
                "plant_step": lambda: solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)}
    times = {k: [] for k in calls_of}
    try:
        for rep in range(reps + 1):   # the first round warms up
            for mode, call in calls_of.items():
                q.copy_(q0t); v.zero_(); torch.cuda.synchronize(dev)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(s)
                for _ in range(calls):
                    call()
                b.record(s); torch.cuda.synchronize(dev)
                if rep:
                    times[mode].append(a.elapsed_time(b) / calls)
    finally:
        solver.spawn_set_ranges(None); solver.state_est_set_ground(None); solver.sim_set_robot_terrain(None); solver.sim_set_terrain(None)
        solver.slip_stop(); solver.attitude_stop(); solver.state_est_stop()
    return {"label": "device time per call on %d robots, median of %d alternated blocks of %d calls; estimator, attitude filter, slip detector and ground-map "
                     "link on, plant step on the same library" % (B, reps, calls),
            **{"ms_per_%s" % k: float(np.median(v)) for k, v in times.items()}, "spread_spawn_all": [float(min(times["spawn_all"])), float(max(times["spawn_all"]))]}


def spawn_falls(r, ep_s=1.0, P=None):
    """Per tile x 45 deg heading bin of a closed_loop.run(respawn=..., spawn=SPAWN) result: the episodes that start at least ep_s before the run's end and
    how many of them fall within their first ep_s seconds.  P [B, E, 4]: the spawn rows to bin by (default the run's spawn_params)"""
    ep, fl = r["episode"], r["fallen"].astype(bool); P = r["spawn_params"] if P is None else P; ticks, B = ep.shape; w = int(round(ep_s * 100))
    edges = np.linspace(-np.pi, np.pi, 9)
    fell = np.zeros((len(SPAWN_TILES), 8), dtype=int); n = np.zeros_like(fell)
    for b in range(B):
        for e in range(int(ep[-1, b]) + 1):
            rows = np.flatnonzero(ep[:, b] == e)
            if rows[0] + w > ticks:
                continue
            i = int(P[b, e, 0]); j = min(np.searchsorted(edges, P[b, e, 3], side="right") - 1, 7)
            n[i, j] += 1; fell[i, j] += int(fl[rows[:w], b].any())
    return {"tiles": list(SPAWN_TILES), "heading_bins_deg": np.degrees(edges).round(1).tolist(), "episodes": n.tolist(), "fell": fell.tolist(),
            "fraction": np.where(n > 0, fell / np.maximum(n, 1), np.nan).round(4).tolist(), "total_episodes": int(n.sum()), "total_fell": int(fell.sum())}


def spawn_main(args, solver, kw, xy, timed, episode_run_s=5.0):
    """--respawn --spawn: the same loop on the --spawn library with SPAWN drawn per episode.  One run of episode_run_s for the falls per bin; the wall
    time per simulated second of --duration runs with and without spawns (both with respawn and the library), alternated twice after one warm-up run
    of each; the spawn call's per-call device time against the plant step."""
    ter = spawn_terrain(xy); kw.update(terrain=ter, ground_map=True)
    arms = {"without_spawn": None, "spawn_fixed_at_the_runs_values": dict(seed=0), "with_spawn": SPAWN}
    wall = {k: [] for k in arms}
    for rep in range(3):   # the first round warms up
        for name, sp in arms.items():
            _, w = timed(True, args.duration, spawn=sp)
            if rep:
                wall[name].append(w)
    r, _ = timed(True, episode_run_s, spawn=SPAWN)
    # the control: no spawn, each robot's heading built by hand into xy_yaw (drawn once, kept by every respawn), on the flat tile
    yaw = np.random.default_rng(0).uniform(-np.pi, np.pi, solver.batch); kw_xy = kw["xy_yaw"]; kw["xy_yaw"] = np.c_[xy[:, :2], yaw]
    try:
        rc, _ = timed(True, episode_run_s)
    finally:
        kw["xy_yaw"] = kw_xy
    E = int(rc["episode"].max()) + 1; Pc = np.zeros((solver.batch, E, _lib.SPAWN)); Pc[:, :, 3] = yaw[:, None]
    name, limit = card()
    print(json.dumps({"metric": "spawn", "gpu": name, "power_limit": limit, "batch": solver.batch, "ee_frame": kw.get("ee_frame", "world"),
                      "config": "%s at %.2f m/s on the state estimate with the ground map, reference IMU noise, no attitude filter; respawn after 0.1 s fallen; "
                                "per episode: tile U{flat, 10 deg ramp, 6 cm stairs, 2 cm rough}, dx U[-0.5, 0] m, dy U[-0.2, 0.2] m, yaw U[-pi, pi]" % (args.gait, args.vx),
                      "simulated_s": episode_run_s, "episodes_per_robot": float(np.mean(r["episode"][-1] + 1)),
                      "fell_within_1s": spawn_falls(r),
                      "control_fell_within_1s": {"label": "no spawn: the same run on the flat tile with each robot's heading drawn once into xy_yaw",
                                                 "episodes_per_robot": float(np.mean(rc["episode"][-1] + 1)), **spawn_falls(rc, P=Pc)},
                      "wall_s_per_sim_s": {"label": "runs of %.1f s with respawn on the library, the three arms alternated twice after a warm-up round; the fixed "
                                                    "arm runs the spawn path at the run's own values (flat tile, yaw 0)" % args.duration, **wall},
                      "per_call": spawn_times(solver, ter, xy)}))


def respawn_main(args, episode_run_s=5.0):
    """--respawn: trot at --vx on the estimate from the reference IMU noise without the attitude filter, robots restarted after 0.1 s fallen.  One
    run of episode_run_s for the rates; the wall time per simulated second of --duration runs with and without respawn, alternated twice after one
    warm-up run of each; the per-call device times."""
    import torch
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    if not torch.cuda.is_available():
        raise SystemExit("bench_closedloop.py: no CUDA device — the product path has no CPU fallback")
    dev = torch.device("cuda", 0); B = args.batch; cmd = (args.vx, 0.0, 0.0, 0.0)
    solver = q.Solver(batch=B, device=0)
    xy = np.zeros((B, 3)); xy[:, 0] = 2.0 * (np.arange(B) % 64); xy[:, 1] = 2.0 * (np.arange(B) // 64)
    kw = dict(gait=args.gait, cmd_vel=cmd, xy_yaw=xy, state_estimator=True, sensor_noise="reference")
    if args.ee_frame:   # every robot's end-effector target in its heading frame (DESIGN.md §4.19)
        kw["ee_frame"] = "heading"

    def timed(respawn, duration, randomize=None, spawn=None):
        solver.mpc_reset(); solver.wbc_set_input_last(None); torch.cuda.synchronize(dev); t0 = time.perf_counter()
        r = closed_loop.run(solver, duration=duration, **kw, **({"respawn": dict(hold=0.1)} if respawn else {}), **({"randomize": randomize} if randomize else {}),
                            **({"spawn": spawn} if spawn else {}))
        torch.cuda.synchronize(dev)
        return r, (time.perf_counter() - t0) / duration
    if args.randomize:
        return randomize_main(args, solver, kw, xy, timed)
    if args.spawn:
        return spawn_main(args, solver, kw, xy, timed)
    wall = {False: [], True: []}
    for rep in range(3):   # the first round warms up
        for respawn in (False, True):
            _, w = timed(respawn, args.duration)
            if rep:
                wall[respawn].append(w)
    r, _ = timed(True, episode_run_s)
    name, limit = card()
    print(json.dumps({"metric": "respawn", "gpu": name, "power_limit": limit, "batch": B,
                      "config": "%s at %.2f m/s on the state estimate, reference IMU noise, no attitude filter; respawn after 0.1 s fallen (min base height above "
                                "the ground <= 0.3 m or |roll|, |pitch| >= 0.3 rad or non-finite)" % (args.gait, args.vx),
                      "rates": {"simulated_s": episode_run_s, **respawn_rates(r)},
                      "wall_s_per_sim_s": {"label": "runs of %.1f s, two alternated pairs after a warm-up pair" % args.duration,
                                           "without_respawn": wall[False], "with_respawn": wall[True]},
                      "per_call": respawn_times(solver, xy)}))


def place_times(solver, reps=7, calls=20):
    """Device time per spawn_here_dev + spawn_place_dev of every robot (the rows of a restart "here") and per 1 ms plant step of the whole batch, on
    robot terrain rows of a stairs tile, alternated `reps` times in blocks of `calls` (CUDA events) → median ms per call of each."""
    import torch
    from qm_control_b200 import terrain as T
    B = solver.batch; dev = torch.device("cuda", 0); s = torch.cuda.Stream(device=dev)
    solver.sim_set_terrain(np.stack([T.stairs(0.05, 0.3)]), T.CELL); origin = T.centred_origin(np.zeros((B, 2))); solver.sim_set_robot_terrain(np.zeros(B), origin)
    q0, v0 = solver.sim_standing_state(np.zeros((B, 3)))
    f64 = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=dev)
    q, v, q_start, o = f64(q0), f64(v0), f64(q0), f64(origin)
    eff = torch.zeros((B, 18), dtype=torch.float64, device=dev); rbd = torch.zeros((B, 55), dtype=torch.float64, device=dev)
    contact = torch.zeros(B, dtype=torch.int32, device=dev); st = torch.zeros_like(contact); every = torch.ones_like(contact); pst = torch.zeros_like(contact)
    x_obs = torch.zeros((B, 30), dtype=torch.float64, device=dev); last_ee = f64(solver.initial_ee_target()); rows = torch.zeros((B, 4), dtype=torch.float64, device=dev)
    solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream); torch.cuda.synchronize(dev)

    def here_place():
        solver.spawn_here_dev(every, rbd, q_start, o, rows, s.cuda_stream)
        solver.spawn_place_dev(every, rows, o, q, v, rbd, contact, x_obs, last_ee, None, pst, 0, s.cuda_stream)
    calls_of = {"here_place_all": here_place, "plant": lambda: solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)}
    times = {k: [] for k in calls_of}
    try:
        for rep in range(reps + 1):   # the first round warms up
            for mode, call in calls_of.items():
                torch.cuda.synchronize(dev)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(s)
                for _ in range(calls):
                    call()
                b.record(s); torch.cuda.synchronize(dev)
                if rep:
                    times[mode].append(a.elapsed_time(b) / calls)
    finally:
        solver.sim_set_robot_terrain(None); solver.sim_set_terrain(None)
    return {"label": "device time per call on %d robots, median of %d alternated blocks of %d calls" % (B, reps, calls), **{"ms_per_%s" % k: float(np.median(v)) for k, v in times.items()}}


def at_here_main(args, course_s=6.0):
    """--respawn --at-here: trot at --vx over a stairs tile with the fall rule (0.1 s fallen), restarts at the start against restarts "here".  The wall
    time per simulated second of --duration runs of each, alternated twice after one warm-up run of each; a course run of course_s each, the farthest
    point along the tile (tile x) each robot's base reached; the device time of here + place against a plant step."""
    import torch
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop, terrain as T
    if not torch.cuda.is_available():
        raise SystemExit("bench_closedloop.py: no CUDA device — the product path has no CPU fallback")
    dev = torch.device("cuda", 0); B = args.batch
    solver = q.Solver(batch=B, device=0)
    origin = T.centred_origin(np.zeros((B, 2)))
    ter = dict(tiles=np.stack([T.stairs(0.05, 0.3)]), cell=T.CELL, tile=np.zeros(B), origin=origin)
    kw = dict(gait=args.gait, cmd_vel=(args.vx, 0.0, 0.0, 0.0), terrain=ter)

    def timed(at, duration):
        solver.mpc_reset(); solver.wbc_set_input_last(None); torch.cuda.synchronize(dev); t0 = time.perf_counter()
        r = closed_loop.run(solver, duration=duration, **kw, respawn=dict(hold=0.1, at=at))
        torch.cuda.synchronize(dev)
        return r, (time.perf_counter() - t0) / duration
    wall = {"start": [], "here": []}
    for rep in range(3):   # the first round warms up
        for at in wall:
            _, w = timed(at, args.duration)
            if rep:
                wall[at].append(w)
    course = {}
    for at in wall:
        r, _ = timed(at, course_s)
        ep = r["episode"]; sp = r.get("spawn_params")
        dx = np.zeros(ep.shape) if sp is None else np.take_along_axis(np.nan_to_num(sp[:, :, 1]), ep.T.astype(np.int64), axis=1).T
        tile_x = r["base"][:, :, 0] - (origin[None, :, 0] - dx)   # the base's x in its tile's frame, window by window
        reach = tile_x.max(axis=0)
        course[at] = {"median_m": float(np.median(reach)), "p90_m": float(np.percentile(reach, 90)), "max_m": float(reach.max()),
                      "restarts_per_robot": float(ep[-1].mean())}
    name, limit = card()
    print(json.dumps({"metric": "respawn_at_here", "gpu": name, "power_limit": limit, "batch": B,
                      "config": "%s at %.2f m/s over a stairs tile (rise 0.05 m, run 0.3 m from 0.35 m), respawn after 0.1 s fallen" % (args.gait, args.vx),
                      "wall_s_per_sim_s": {"label": "runs of %.1f s, two alternated pairs after a warm-up pair" % args.duration, **wall},
                      "course": {"simulated_s": course_s, "label": "farthest tile x of the base per robot (m), over the run", **course},
                      "per_call": place_times(solver)}))


def metrics_times(solver, xy_yaw, reps=7, calls=20):
    """Device time per metrics sample (metrics_step_dev), per close of every robot (metrics_close_dev) and per 1 ms plant step of the whole batch,
    alternated `reps` times in blocks of `calls` from one standing state with a cmd_vel target (CUDA events) → median ms per call of each."""
    import torch
    B = solver.batch; dev = torch.device("cuda", 0); s = torch.cuda.Stream(device=dev)
    q0, v0 = solver.sim_standing_state(xy_yaw)
    q = torch.as_tensor(q0, device=dev); v = torch.as_tensor(v0, device=dev)
    eff = torch.zeros((B, 18), dtype=torch.float64, device=dev); rbd = torch.zeros((B, 55), dtype=torch.float64, device=dev)
    contact = torch.zeros(B, dtype=torch.int32, device=dev); st = torch.zeros_like(contact)
    solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream); torch.cuda.synchronize(dev)
    x = torch.as_tensor(solver.centroidal_state_from_rbd(rbd.cpu().numpy()), device=dev); t_obs = torch.full((B,), 10.0, dtype=torch.float64, device=dev)
    cmd = torch.zeros((B, 7), dtype=torch.float64, device=dev); cmd[:, 0] = 0.3; last_ee = torch.as_tensor(solver.initial_ee_target(), device=dev)
    n_target = torch.zeros(B, dtype=torch.int32, device=dev); tt = torch.zeros((B, _lib.KMAX), dtype=torch.float64, device=dev)
    ts = torch.zeros((B, _lib.KMAX, _lib.TARGET), dtype=torch.float64, device=dev)
    solver.target_trajectories_dev(0, cmd, t_obs, x, rbd[:, 48:55].contiguous(), last_ee, n_target, tt, ts, s.cuda_stream)
    acc = torch.zeros((B, _lib.METRICS_ACC), dtype=torch.float64, device=dev); out = torch.zeros((B, 1, _lib.METRICS), dtype=torch.float64, device=dev)
    every, zero = torch.ones_like(contact), torch.zeros_like(contact)
    calls_of = {"metrics_step": lambda: solver.metrics_step_dev(1e-3, rbd, contact, eff, cmd, n_target, tt, ts, t_obs, st, acc, stream=s.cuda_stream),
                "metrics_close_all": lambda: solver.metrics_close_dev(every, zero, zero, acc, out, st, s.cuda_stream),
                "plant": lambda: solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)}
    times = {k: [] for k in calls_of}
    for rep in range(reps + 1):   # the first round warms up
        for mode, call in calls_of.items():
            torch.cuda.synchronize(dev)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(s)
            for _ in range(calls):
                call()
            b.record(s); torch.cuda.synchronize(dev)
            if rep:
                times[mode].append(a.elapsed_time(b) / calls)
    return {"label": "device time per call on %d robots, median of %d alternated blocks of %d calls" % (B, reps, calls),
            **{"ms_per_%s" % k: float(np.median(v)) for k, v in times.items()}, "spread_metrics_step": [float(min(times["metrics_step"])), float(max(times["metrics_step"]))]}


def metrics_main(args, episode_run_s=3.0):
    """--metrics: the wall time per simulated second of --duration runs of --gait at --vx on the plant's truth with and without metrics, alternated three
    times after one warm-up run of each; the per-call device times; and the medians of every column over the complete episodes (closed by a respawn) of
    an episode_run_s run on the state estimate with the reference IMU noise, respawn (0.1 s fallen, or 1 s) and RANDOMIZE's plant per episode."""
    import torch
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    if not torch.cuda.is_available():
        raise SystemExit("bench_closedloop.py: no CUDA device — the product path has no CPU fallback")
    dev = torch.device("cuda", 0); B = args.batch
    solver = q.Solver(batch=B, device=0)
    xy = np.zeros((B, 3)); xy[:, 0] = 2.0 * (np.arange(B) % 64); xy[:, 1] = 2.0 * (np.arange(B) // 64)
    kw = dict(gait=args.gait, cmd_vel=(args.vx, 0.0, 0.0, 0.0), xy_yaw=xy)

    def timed(duration, **extra):
        solver.mpc_reset(); solver.wbc_set_input_last(None); torch.cuda.synchronize(dev); t0 = time.perf_counter()
        r = closed_loop.run(solver, duration=duration, **kw, **extra)
        torch.cuda.synchronize(dev)
        return r, (time.perf_counter() - t0) / duration
    wall = {"without_metrics": [], "with_metrics": []}
    for rep in range(4):   # the first round warms up
        for name, extra in (("without_metrics", {}), ("with_metrics", dict(metrics=True))):
            _, w = timed(args.duration, **extra)
            if rep:
                wall[name].append(w)
    r, _ = timed(episode_run_s, metrics=True, state_estimator=True, sensor_noise="reference", respawn=dict(hold=0.1, every=1.0), randomize=RANDOMIZE)
    M = r["episode_metrics"]; done = M[..., 1] > 0
    name, limit = card()
    print(json.dumps({"metric": "metrics", "gpu": name, "power_limit": limit, "batch": B,
                      "wall_s_per_sim_s": {"label": "%s at %.2f m/s on the plant's truth, runs of %.1f s, three alternated pairs after a warm-up pair"
                                                    % (args.gait, args.vx, args.duration), **wall},
                      "per_call": metrics_times(solver, xy),
                      "episodes": {"label": "%s at %.2f m/s on the state estimate, reference IMU noise; respawn after 0.1 s fallen or 1 s; RANDOMIZE per episode; "
                                            "%.1f s; medians over the episodes a respawn closed" % (args.gait, args.vx, episode_run_s),
                                   "complete": int(done.sum()), "fell": int(np.sum(M[..., 1] == 1)),
                                   "median": {c: float(np.nanmedian(M[..., i][done])) for i, c in enumerate(r["metrics_layout"]) if c not in ("end", "status")}}}))


# A gait slot due at t takes effect at the first MPC tick at or after t, plus the time horizon (GaitReceiver's insertion time) and the transition stance:
# with the 1 s horizon the first switch starts 1.0-1.4 s into an episode, so the episodes of the per-transition run last TIMELINE_EPISODE_S
TIMELINE = dict(seed=1, n=3, t_first=(0.0, 0.3), gap=(0.8, 1.2), p_gait=0.5, gaits=["trot", "pace", "static_walk", "standing_trot"],
                weights=dict(none=1.0, cmd_vel=1.0), cmd_vel_x=(-0.2, 0.6), cmd_yaw_rate=(-0.3, 0.3))
TIMELINE_EPISODE_S = 3.0


def timeline_times(solver, reps=7, calls=20):
    """Device time per timeline draw of every robot (timeline_sample_dev, TIMELINE's ranges on a loaded placeholder timeline) and per 1 ms plant step of
    the whole batch, alternated `reps` times in blocks of `calls` (CUDA events) → median ms per call of each."""
    import torch
    from qm_control_b200 import closed_loop
    B = solver.batch; dev = torch.device("cuda", 0); s = torch.cuda.Stream(device=dev); n = TIMELINE["n"]
    xy = np.zeros((B, 3)); xy[:, 0] = 2.0 * (np.arange(B) % 64); xy[:, 1] = 2.0 * (np.arange(B) // 64)
    q0, v0 = solver.sim_standing_state(xy); q = torch.as_tensor(q0, device=dev); v = torch.as_tensor(v0, device=dev)
    eff = torch.zeros((B, 18), dtype=torch.float64, device=dev); rbd = torch.zeros((B, 55), dtype=torch.float64, device=dev)
    contact = torch.zeros(B, dtype=torch.int32, device=dev); st = torch.zeros_like(contact)
    tl = closed_loop._timeline_spec(B, "trot", TIMELINE, None); gd = tl["gd"]
    solver.gait_dev_set_templates(gd["names"]); solver.gait_dev_reset(gd["gait"], np.full(B, 10.0)); solver.gait_dev_set_commands(gd["t"], gd["tmpl"], gd["cmd_vel"])
    TL = {c: i for i, c in enumerate(_lib.TIMELINE_LAYOUT)}
    lo = np.zeros((B, _lib.TIMELINE)); lo[:, TL["p_gait"]] = tl["p_gait"]; lo[:, TL["gait_set"]] = tl["gait_set"]; lo[:, 4:8] = tl["weights"]; lo[:, TL["ee_qw"]] = 1.0
    hi = lo.copy()
    for c, (l, h) in tl["fields"].items():
        lo[:, TL[c]] = l; hi[:, TL[c]] = h
    solver.timeline_set_ranges(n, lo, hi, 1)
    every = torch.ones_like(contact); episode = torch.zeros_like(contact); rows = torch.zeros((B, n, _lib.TIMELINE_CMD), dtype=torch.float64, device=dev)
    calls_of = {"timeline_sample": lambda: (episode.add_(1), solver.timeline_sample_dev(every, episode, rows, s.cuda_stream)),
                "plant": lambda: solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)}
    times = {k: [] for k in calls_of}
    with torch.cuda.stream(s):
        for rep in range(reps + 1):   # the first round warms up
            for mode, call in calls_of.items():
                torch.cuda.synchronize(dev)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(s)
                for _ in range(calls):
                    call()
                b.record(s); torch.cuda.synchronize(dev)
                if rep:
                    times[mode].append(a.elapsed_time(b) / calls)
    solver.timeline_set_ranges(None); solver.gait_dev_stop()
    return {"label": "device time per call on %d robots (every robot drawing %d slots), median of %d alternated blocks of %d calls" % (B, n, reps, calls),
            **{"ms_per_%s" % k: float(np.median(v)) for k, v in times.items()},
            "spread_timeline_sample": [float(min(times["timeline_sample"])), float(max(times["timeline_sample"]))]}


def stance_time(solver):
    """phaseTransitionStanceTime of the solver's task file, the stance a gait insertion puts before the new gait (0.4 s where the file has none)"""
    import re
    m = re.search(r"phaseTransitionStanceTime\s+([-+0-9.eE]+)", open(solver.interface.taskFile).read())
    return float(m.group(1)) if m else 0.4


def timeline_bins(r, start_gait, cmd_vel, horizon, stance, wbc_period=0.002):
    """Each episode scored by metrics, classed by its first gait switch that takes effect inside it (start gait → drawn gait) and by |delta cmd_vel|
    (planar) of its first cmd_vel slot that takes effect inside it → per class: episodes, fall rate, median vel_err_rms (over the whole episode) and the
    median time the episode ran after the switch or step.  A slot due at t (s after the episode's start) is applied by the first MPC tick at or after t
    (ticks at -wbc_period + 10 ms k); a cmd_vel row takes effect there, a gait at that tick + horizon + the transition stance (an upper bound: no stance
    is inserted where the schedule already stands there)."""
    M, P, names = r["episode_metrics"], r["timeline_params"], r["gait_templates"]
    ok = ~np.isnan(M[..., 0]); by_gait, by_dv = {}, {}
    for b, e in zip(*np.nonzero(ok)):
        dur = M[b, e, 0]; tick = np.ceil(np.round((P[b, e, :, 0] + wbc_period) / 0.01, 9)) * 0.01 - wbc_period
        g = P[b, e, :, 1]; v = P[b, e, :, 2:4]; t_gait = tick + horizon + stance
        gi = np.nonzero((g >= 0) & (t_gait < dur))[0]; vi = np.nonzero(~np.isnan(v[:, 0]) & (tick < dur))[0]
        key_g = "%s -> %s" % (start_gait, names[int(g[gi[0]])]) if len(gi) else "no switch in the episode"
        dv = np.hypot(*(v[vi[0]] - cmd_vel[:2])) if len(vi) else None
        key_v = "no step in the episode" if dv is None else "[%.1f, %.1f)" % (np.floor(dv / 0.2) * 0.2, np.floor(dv / 0.2) * 0.2 + 0.2)
        for d, k, t0 in ((by_gait, key_g, t_gait[gi[0]] if len(gi) else np.nan), (by_dv, key_v, tick[vi[0]] if len(vi) else np.nan)):
            d.setdefault(k, []).append((M[b, e, 1] == 1, M[b, e, 7], dur - t0))

    def stats(d):
        return {k: {"episodes": len(x), "fall_rate": float(np.mean([f for f, _, _ in x])), "median_vel_err_rms": float(np.nanmedian([m for _, m, _ in x])),
                    "median_s_after": None if np.all(np.isnan([a for _, _, a in x])) else float(np.nanmedian([a for _, _, a in x]))}
                for k, x in sorted(d.items())}
    return {"transition": stats(by_gait), "abs_dcmd_vel": stats(by_dv)}


def timeline_main(args, episode_run_s=6.0):
    """--respawn --timeline: the sampler's per-call device time; the wall time per simulated second of --duration respawning runs of --gait at --vx on the
    plant's truth with and without TIMELINE, alternated twice after one warm-up pair; and episodes, fall rate and median velocity error per gait
    transition and per |delta cmd_vel| bin (timeline_bins) of an episode_run_s run with respawn (0.1 s fallen, or TIMELINE_EPISODE_S), TIMELINE and
    metrics."""
    import torch
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    if not torch.cuda.is_available():
        raise SystemExit("bench_closedloop.py: no CUDA device — the product path has no CPU fallback")
    dev = torch.device("cuda", 0); B = args.batch
    solver = q.Solver(batch=B, device=0)
    xy = np.zeros((B, 3)); xy[:, 0] = 2.0 * (np.arange(B) % 64); xy[:, 1] = 2.0 * (np.arange(B) // 64)
    cmd = np.array([args.vx, 0.0, 0.0, 0.0]); kw = dict(gait=args.gait, cmd_vel=cmd, xy_yaw=xy)

    def timed(duration, respawn=dict(hold=0.1, every=1.0), **extra):
        solver.mpc_reset(); solver.wbc_set_input_last(None); torch.cuda.synchronize(dev); t0 = time.perf_counter()
        r = closed_loop.run(solver, duration=duration, respawn=respawn, **kw, **extra)
        torch.cuda.synchronize(dev)
        return r, (time.perf_counter() - t0) / duration
    per_call = timeline_times(solver)
    wall = {"without_timeline": [], "with_timeline": []}
    for rep in range(3):   # the first round warms up
        for name, extra in (("without_timeline", {}), ("with_timeline", dict(timeline=TIMELINE))):
            _, w = timed(args.duration, **extra)
            if rep:
                wall[name].append(w)
    r, _ = timed(episode_run_s, metrics=True, timeline=TIMELINE, respawn=dict(hold=0.1, every=TIMELINE_EPISODE_S))
    name, limit = card()
    print(json.dumps({"metric": "timeline", "gpu": name, "power_limit": limit, "batch": B,
                      "per_call": per_call,
                      "wall_s_per_sim_s": {"label": "%s at %.2f m/s on the plant's truth, respawn after 0.1 s fallen or 1 s, runs of %.1f s, two alternated pairs "
                                                    "after a warm-up pair" % (args.gait, args.vx, args.duration), **wall},
                      "episodes": {"label": "%.1f s, respawn after 0.1 s fallen or %.1f s, TIMELINE per episode, metrics; classed by the first gait switch and the "
                                            "first cmd_vel step that take effect inside the episode (horizon %.2f s, transition stance %.2f s)"
                                            % (episode_run_s, TIMELINE_EPISODE_S, solver.time_horizon, stance_time(solver)),
                                   "count": int(np.sum(~np.isnan(r["episode_metrics"][..., 0]))),
                                   **timeline_bins(r, args.gait, cmd, solver.time_horizon, stance_time(solver))}}))


def watch_state_est(solver):
    """Wrap the solver's plant and estimator steps so that each estimator call updates per-robot maxima of |z_hat - z|, |v_hat - v| and the wrapped zyx
    error (the largest of the three angles) on the device (no synchronisation) → (box, unwrap); box["max"] [B, 3], box["last"] [B, 3] after the run."""
    import torch
    orig_sim, orig_est = solver.sim_step_dev, solver.state_est_step_dev; box = {}

    def sim(duration, effort, q, v, rbd, contact, status, stream=None, wrench=None):
        box["rbd"] = rbd; orig_sim(duration, effort, q, v, rbd, contact, status, stream, wrench=wrench)

    def est(dt, sensors, contact, rbd_est, status, stream=None):
        orig_est(dt, sensors, contact, rbd_est, status, stream)
        with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
            e = torch.stack([(rbd_est[:, 5] - box["rbd"][:, 5]).abs(), (rbd_est[:, 27:30] - box["rbd"][:, 27:30]).norm(dim=1),
                             torch.remainder(rbd_est[:, 0:3] - box["rbd"][:, 0:3] + np.pi, 2 * np.pi).sub_(np.pi).abs().amax(dim=1)], 1)
            box["last"] = e; box["max"] = e if "max" not in box else torch.maximum(box["max"], e)

    def unwrap():
        del solver.sim_step_dev, solver.state_est_step_dev
    solver.sim_step_dev, solver.state_est_step_dev = sim, est
    return box, unwrap


# --respawn --curriculum: an up-down staircase (one level up after an episode that lasted `every`, one down after a fall) on the base push along +x, from
# 0 N at level 0 to 255 N at level CURRICULUM_LEVELS - 1, starting half way, each robot on a fixed friction of one MU_BINS bin (the bins of
# --randomize's sweep, on the same state estimate); pushes for 0.1 s from 0.2-0.5 s
CURRICULUM_LEVELS, CURRICULUM_PUSH, CURRICULUM_MU_BINS = 12, 255.0, MU_BINS
CURRICULUM_RUN_S, CURRICULUM_EVERY_S = 12.0, 1.0


def curriculum_times(solver, reps=7, calls=20):
    """Device time per curriculum update of every robot (curriculum_update_dev, one pass condition on a metrics row, the episode ranges attached) and per
    1 ms plant step of the whole batch, alternated `reps` times in blocks of `calls` (CUDA events) → median ms per call of each."""
    import torch
    B = solver.batch; dev = torch.device("cuda", 0); s = torch.cuda.Stream(device=dev)
    xy = np.zeros((B, 3)); xy[:, 0] = 2.0 * (np.arange(B) % 64); xy[:, 1] = 2.0 * (np.arange(B) // 64)
    q0, v0 = solver.sim_standing_state(xy); q = torch.as_tensor(q0, device=dev); v = torch.as_tensor(v0, device=dev)
    eff = torch.zeros((B, 18), dtype=torch.float64, device=dev); rbd = torch.zeros((B, 55), dtype=torch.float64, device=dev)
    contact = torch.zeros(B, dtype=torch.int32, device=dev); st = torch.zeros_like(contact)
    lo = np.zeros((B, _lib.EPISODE)); lo[:, 0] = 0.7; hi = lo.copy(); hi[:, 11:13] = 180.0; lo[:, 11:13] = -180.0
    solver.episode_set_ranges(lo, hi, 1)
    rows = np.zeros((B, _lib.CURRICULUM)); rows[:, 1:3] = 1.0; rows[:, 3] = 0.2
    solver.curriculum_set(CURRICULUM_LEVELS, rows, [("distance", ">=", "pass")]); solver.curriculum_attach("episode", lo * 1.4, hi * 1.4)
    every = torch.ones_like(contact); end = torch.full_like(contact, 2); ep = torch.zeros_like(contact); level = torch.zeros_like(contact)
    out = torch.rand((B, 1, _lib.METRICS), dtype=torch.float64, device=dev)
    calls_of = {"curriculum_update": lambda: solver.curriculum_update_dev(every, end, ep, out, level, st, s.cuda_stream),
                "plant": lambda: solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)}
    times = {k: [] for k in calls_of}
    for rep in range(reps + 1):   # the first round warms up
        for mode, call in calls_of.items():
            torch.cuda.synchronize(dev)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(s)
            for _ in range(calls):
                call()
            b.record(s); torch.cuda.synchronize(dev)
            if rep:
                times[mode].append(a.elapsed_time(b) / calls)
    solver.curriculum_set(None); solver.episode_set_ranges(None)
    return {"label": "device time per call on %d robots, median of %d alternated blocks of %d calls" % (B, reps, calls),
            **{"ms_per_%s" % k: float(np.median(v)) for k, v in times.items()},
            "spread_curriculum_update": [float(min(times["curriculum_update"])), float(max(times["curriculum_update"]))]}


def curriculum_main(args):
    """--respawn --curriculum: the update's per-call device time; the wall time per simulated second of --duration runs of --gait at --vx on the plant's
    truth with respawn and RANDOMIZE in both arms, without and with a curriculum on RANDOMIZE's push bounds, alternated twice after a warm-up pair; and
    the push each friction bin survives, estimated two ways from runs of CURRICULUM_RUN_S with respawn (0.1 s fallen, or CURRICULUM_EVERY_S): the
    staircase's threshold (each robot's mean level over the second half of its episodes) against the 50 % crossing of the fall fraction over the push
    of a run with the push drawn uniformly from the staircase's range, the same robots and episode budget."""
    import torch
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    if not torch.cuda.is_available():
        raise SystemExit("bench_closedloop.py: no CUDA device — the product path has no CPU fallback")
    dev = torch.device("cuda", 0); B = args.batch
    solver = q.Solver(batch=B, device=0)
    xy = np.zeros((B, 3)); xy[:, 0] = 2.0 * (np.arange(B) % 64); xy[:, 1] = 2.0 * (np.arange(B) // 64)
    kw = dict(gait=args.gait, cmd_vel=(args.vx, 0.0, 0.0, 0.0), xy_yaw=xy)

    def timed(duration, **extra):
        solver.mpc_reset(); solver.wbc_set_input_last(None); torch.cuda.synchronize(dev); t0 = time.perf_counter()
        r = closed_loop.run(solver, duration=duration, **kw, **extra)
        torch.cuda.synchronize(dev)
        return r, (time.perf_counter() - t0) / duration
    per_call = curriculum_times(solver)
    respawn = dict(hold=0.1, every=CURRICULUM_EVERY_S)
    wall = {"without_curriculum": [], "with_curriculum": []}
    arms = (("without_curriculum", {}), ("with_curriculum", dict(curriculum=dict(levels=CURRICULUM_LEVELS, randomize=dict(f_base_x=(-255.0, 255.0), f_base_y=(-255.0, 255.0))))))
    for rep in range(3):   # the first round warms up
        for name, extra in arms:
            _, w = timed(args.duration, respawn=respawn, randomize=RANDOMIZE, **extra)
            if rep:
                wall[name].append(w)
    # runs of CURRICULUM_RUN_S roll the gait on the device (a command timeline that changes nothing): the host-tiled schedule holds about 5 s of trot
    kw["commands"] = dict(t=np.full((B, 1), 0.2), gait=np.full((B, 1), None, dtype=object))
    bins = np.array(CURRICULUM_MU_BINS); mu_bin = np.arange(B) % (len(bins) - 1)
    mu = bins[mu_bin] + (bins[mu_bin + 1] - bins[mu_bin]) * ((np.arange(B) // (len(bins) - 1)) % 16 + 0.5) / 16.0
    base = dict(seed=0, friction_mu=(mu, mu), push_t_on=(0.2, 0.5), push_duration=(0.1, 0.1))
    est = dict(state_estimator=True, sensor_noise="reference")
    stair, _ = timed(CURRICULUM_RUN_S, respawn=respawn, randomize=base, **est,
                     curriculum=dict(levels=CURRICULUM_LEVELS, start=CURRICULUM_LEVELS // 2, randomize=dict(f_base_x=(CURRICULUM_PUSH, CURRICULUM_PUSH))))
    flat, _ = timed(CURRICULUM_RUN_S, respawn=respawn, randomize=dict(base, f_base_x=(0.0, CURRICULUM_PUSH)), metrics=True, **est)
    el = stair["episode_level"]; n_ep = (el >= 0).sum(1)
    second = np.array([el[b, n_ep[b] // 2:n_ep[b]].mean() for b in range(B)])
    thr = second * CURRICULUM_PUSH / (CURRICULUM_LEVELS - 1)
    push_bins = np.linspace(0.0, CURRICULUM_PUSH, 9)
    P, M = flat["episode_params"], flat["episode_metrics"]; ok = M[..., 1] > 0; fell = M[..., 1] == 1   # the episodes a respawn closed; those the fall rule did
    out = {}
    for i in range(len(bins) - 1):
        rob = mu_bin == i; sel = ok & rob[:, None]; f = P[..., 11][sel]; y = fell[sel]
        frac = [float(np.mean(y[(f >= a) & (f < c)])) if np.any((f >= a) & (f < c)) else None for a, c in zip(push_bins[:-1], push_bins[1:])]
        centres = (push_bins[:-1] + push_bins[1:]) / 2; crossing = None
        for j in range(len(frac) - 1):
            if frac[j] is not None and frac[j + 1] is not None and frac[j] < 0.5 <= frac[j + 1]:
                crossing = float(centres[j] + (0.5 - frac[j]) / (frac[j + 1] - frac[j]) * (centres[j + 1] - centres[j])); break
        out["mu_%.2f-%.2f" % (bins[i], bins[i + 1])] = {
            "staircase_threshold_N": {"mean": float(thr[rob].mean()), "median": float(np.median(thr[rob])), "robots": int(rob.sum())},
            "saturated": {"bottom": float(np.mean(second[rob] == 0)), "top": float(np.mean(second[rob] == CURRICULUM_LEVELS - 1))},
            "uniform_50pct_crossing_N": crossing, "uniform_fall_fraction_per_push_bin": frac, "uniform_episodes": int(sel.sum())}
    name, limit = card()
    print(json.dumps({"metric": "curriculum", "gpu": name, "power_limit": limit, "batch": B,
                      "per_call": per_call,
                      "wall_s_per_sim_s": {"label": "%s at %.2f m/s on the plant's truth, respawn after 0.1 s fallen or %.1f s, RANDOMIZE per episode; runs of %.1f s, "
                                                    "two alternated pairs after a warm-up pair; the curriculum arm moves RANDOMIZE's push bounds to +-255 N over %d levels"
                                                    % (args.gait, args.vx, CURRICULUM_EVERY_S, args.duration, CURRICULUM_LEVELS), **wall},
                      "staircase": {"label": "%s at %.2f m/s on the state estimate with the reference IMU noise, the gait rolled on the device, %.1f s, respawn after 0.1 s fallen or %.1f s; push f_base_x for 0.1 s from "
                                             "0.2-0.5 s; staircase 0-%.0f N over %d levels, up after an episode that lasted, down after a fall, from level 6; "
                                             "uniform: f_base_x U[0, %.0f] N, fall fraction per push bin of %.0f N over the episodes a respawn closed"
                                             % (args.gait, args.vx, CURRICULUM_RUN_S, CURRICULUM_EVERY_S, CURRICULUM_PUSH, CURRICULUM_LEVELS, CURRICULUM_PUSH,
                                                push_bins[1]),
                                    "episodes": {"staircase": int(n_ep.sum()), "uniform": int(ok.sum())}, "per_mu_bin": out}}))


def heading_controller(state, goal, vx=0.25, gain=2.0, rate_max=0.6):
    """a torch heading controller on a session's live tensors: cmd_vel = (vx, 0, 0, clamp(gain * wrap(goal - yaw))) from the plant's yaw q[:, 3]"""
    import torch
    err = torch.remainder(goal - state["q"][:, 3] + np.pi, 2.0 * np.pi) - np.pi
    vel = torch.zeros((len(goal), 4), dtype=torch.float64, device=goal.device)
    vel[:, 0] = vx; vel[:, 3] = torch.clamp(gain * err, -rate_max, rate_max)
    return vel


def command_times(solver, reps=7, calls=50):
    """Device time per qmb200_gait_dev_command_dev on every robot (a cmd_vel row each) and per 1 ms plant step of the whole batch, alternated `reps`
    times in blocks of `calls` (CUDA events) → median ms per call of each."""
    import torch
    B = solver.batch; dev = torch.device("cuda", 0); s = torch.cuda.Stream(device=dev)
    solver.gait_dev_set_templates(); solver.gait_dev_reset(np.zeros(B, dtype=np.int32), np.full(B, 10.0))
    xy = np.zeros((B, 3)); xy[:, 0] = 2.0 * (np.arange(B) % 64); xy[:, 1] = 2.0 * (np.arange(B) // 64)
    q0, v0 = solver.sim_standing_state(xy); q = torch.as_tensor(q0, device=dev); v = torch.as_tensor(v0, device=dev)
    eff = torch.zeros((B, 18), dtype=torch.float64, device=dev); rbd = torch.zeros((B, 55), dtype=torch.float64, device=dev)
    contact = torch.zeros(B, dtype=torch.int32, device=dev); st = torch.zeros_like(contact)
    ones = torch.ones_like(contact); tmpl = torch.full_like(contact, -1); kind = torch.full_like(contact, -1)
    vel = torch.full((B, 4), 0.2, dtype=torch.float64, device=dev); ee = torch.zeros((B, 7), dtype=torch.float64, device=dev)
    calls_of = {"command": lambda: solver.gait_dev_command_dev(ones, tmpl, vel, kind, ee, st, s.cuda_stream),
                "plant": lambda: solver.sim_step_dev(1e-3, eff, q, v, rbd, contact, st, s.cuda_stream)}
    times = {k: [] for k in calls_of}
    for rep in range(reps + 1):   # the first round warms up
        for mode, call in calls_of.items():
            torch.cuda.synchronize(dev)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(s)
            for _ in range(calls):
                call()
            b.record(s); torch.cuda.synchronize(dev)
            if rep:
                times[mode].append(a.elapsed_time(b) / calls)
    solver.gait_dev_stop()
    return {"label": "device time per call on %d robots, median of %d alternated blocks of %d calls" % (B, reps, calls),
            **{"ms_per_%s" % k: float(np.median(v)) for k, v in times.items()},
            "spread_command": [float(min(times["command"])), float(max(times["command"]))]}


def session_main(args, reps=2):
    """Wall time per simulated second of closed_loop.run against a Session stepped one 10 ms window at a time, without commands and with one heading
    command per window from a torch controller on the session's stream (alternated, best of reps), and the command kernel's time."""
    import torch
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    if not torch.cuda.is_available():
        raise SystemExit("bench_closedloop.py: no CUDA device — the product path has no CPU fallback")
    B = args.batch; sim_s = args.duration; solver = q.Solver(batch=B, device=0)
    xy = np.zeros((B, 3)); xy[:, 0] = 2.0 * (np.arange(B) % 64); xy[:, 1] = 2.0 * (np.arange(B) // 64)
    kw = dict(gait=args.gait, cmd_vel=(args.vx, 0.0, 0.0, 0.0), xy_yaw=xy)
    goal_h = np.random.default_rng(0).uniform(-1.0, 1.0, B)

    def stepped(commanded, duration):
        with closed_loop.Session(solver, duration, steer=commanded, **kw) as ss:
            with torch.cuda.stream(ss.stream):
                goal = torch.as_tensor(goal_h, device=ss.device); ones = torch.ones(B, dtype=torch.int32, device=ss.device)
            for _ in range(ss.windows):
                if commanded:
                    with torch.cuda.stream(ss.stream):
                        ss.command(ones, cmd_vel=heading_controller(ss.state, goal))
                ss.step(1)
            return ss.finish()
    modes = {"run": lambda d: closed_loop.run(solver, duration=d, **kw), "session": lambda d: stepped(False, d), "session_commands": lambda d: stepped(True, d)}
    for f in modes.values():   # warm-up: every shape of the timed runs
        f(0.05)
    wall = {k: [] for k in modes}; end = None
    for _ in range(reps):
        for k, f in modes.items():
            torch.cuda.synchronize(); t0 = time.perf_counter(); r = f(sim_s); torch.cuda.synchronize(); wall[k].append((time.perf_counter() - t0) / sim_s)
            end = r if k == "session_commands" else end
    err = np.abs(np.remainder(goal_h - end["q"][:, 3] + np.pi, 2 * np.pi) - np.pi)
    name, limit = card()
    print(json.dumps({"metric": "session", "gpu": name, "power_limit": limit, "batch": B, "gait": args.gait, "sim_s": sim_s,
                      "wall_s_per_sim_s": {k: float(min(v)) for k, v in wall.items()}, "wall_s_per_sim_s_all": wall,
                      "heading_error_rad": dict(max=float(err.max()), mean=float(err.mean()), start_max=float(np.abs(goal_h).max())),
                      "times": command_times(solver)}))



def snapshot_main(args, reps=7, calls=10, sim_reps=2):
    """Robot-state snapshots (DESIGN.md §4.17) with every component running and a commands timeline: bytes per robot, device time per save and per
    load of every robot from a permuted source (CUDA events, alternated blocks of `calls`, median of reps) with the copy bandwidth (bytes read +
    written) against the H100's 3.35 TB/s, and wall time per simulated second of a Session stepped one window at a time without a restore and with a
    snapshot and a branch of every robot every window (alternated, best of sim_reps)."""
    import torch
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    from qm_control_b200 import terrain as TR
    if not torch.cuda.is_available():
        raise SystemExit("bench_closedloop.py: no CUDA device — the product path has no CPU fallback")
    B = args.batch; sim_s = args.duration; solver = q.Solver(batch=B, device=0); rng = np.random.default_rng(0)
    xy = np.zeros((B, 3)); xy[:, 0] = 2.0 * (np.arange(B) % 64); xy[:, 1] = 2.0 * (np.arange(B) // 64)
    ter = dict(tiles=np.stack([TR.ramp(5.0), TR.rough(0.01, seed=3)]), cell=TR.CELL, tile=(np.arange(B) % 3 - 1).astype(np.int32), origin=TR.centred_origin(xy[:, :2]))
    t = np.tile([0.2, 0.5], (B, 1)); goal = np.full((B, 2, 7), np.nan); goal[:, 1] = [0.55, 0.0, 0.45, 0.0, 0.0, 0.0, 1.0]
    commands = dict(t=t, gait=[["pace", None]] * B, cmd_vel=np.full((B, 2, 4), np.nan), ee_goal=goal)
    kw = dict(gait=args.gait, cmd_vel=(args.vx, 0.0, 0.0, 0.0), xy_yaw=xy, terrain=ter, friction_mu=rng.uniform(0.5, 0.9, B), payload=np.c_[rng.uniform(0, 0.5, B), np.zeros((B, 7))],
              model_payload="plant", tuning=dict(kp_swing=rng.uniform(300.0, 400.0, B)), payload_estimator=True, state_estimator=True, attitude_filter=True,
              slip_detector=True, ground_map=True, commands=commands, metrics=True)
    perm = torch.as_tensor(rng.permutation(B).astype(np.int32), device="cuda:0")

    def stepped(branch, duration):
        with closed_loop.Session(solver, duration, **kw) as ss:
            for _ in range(ss.windows):
                if branch:
                    ss.restore(ss.snapshot(), source=perm)
                ss.step(1)
            return ss.finish()

    with closed_loop.Session(solver, 0.05, **kw) as ss:
        ss.step(2); st = ss._s; per_robot = solver.robot_state_bytes()
        snap = ss.snapshot(); loop_bytes = snap.nbytes - B * per_robot
        blocks = [n for i, n in enumerate(_lib.ROBOT_STATE_BLOCKS) if (snap.desc.blocks >> i) & 1]
        buf = torch.empty(B * per_robot, dtype=torch.uint8, device=ss.device); ones = torch.ones(B, dtype=torch.int32, device=ss.device)
        calls_of = {"save": lambda: solver.robot_state_save_dev(buf, st), "load": lambda: solver.robot_state_load_dev(snap.buf, snap.desc, ones, perm, None, st)}
        times = {k: [] for k in calls_of}
        for rep in range(reps + 1):   # the first round warms up
            for mode, call in calls_of.items():
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True); a.record(ss.stream)
                for _ in range(calls):
                    call()
                b.record(ss.stream); torch.cuda.synchronize()
                if rep:
                    times[mode].append(a.elapsed_time(b) / calls)
        ss.finish()
    name, limit = card()   # read in the same call as the timings
    modes = {"no_restore": lambda d: stepped(False, d), "branch_every_window": lambda d: stepped(True, d)}
    for f in modes.values():   # warm-up: every shape of the timed runs
        f(0.03)
    wall = {k: [] for k in modes}
    for _ in range(sim_reps):
        for k, f in modes.items():
            torch.cuda.synchronize(); t0 = time.perf_counter(); f(sim_s); torch.cuda.synchronize(); wall[k].append((time.perf_counter() - t0) / sim_s)
    moved = 2.0 * B * per_robot   # every robot's rows read once and written once
    print(json.dumps({"metric": "snapshot", "gpu": name, "power_limit": limit, "batch": B, "gait": args.gait, "sim_s": sim_s, "blocks": blocks,
                      "library_bytes_per_robot": per_robot, "loop_bytes_per_robot": loop_bytes / B, "snapshot_bytes": snap.nbytes,
                      "label": "device time per call on %d robots, median of %d alternated blocks of %d calls" % (B, reps, calls),
                      **{"ms_per_%s" % k: float(np.median(v)) for k, v in times.items()}, "ms_all": times,
                      **{"tb_per_s_%s" % k: moved / (float(np.median(v)) * 1e-3) / 1e12 for k, v in times.items()}, "hbm_tb_per_s_datasheet": 3.35,
                      "wall_s_per_sim_s": {k: float(min(v)) for k, v in wall.items()}, "wall_s_per_sim_s_all": wall}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8192); ap.add_argument("--duration", type=float, default=1.0)
    ap.add_argument("--gait", default="trot"); ap.add_argument("--vx", type=float, default=0.3)
    ap.add_argument("--vary", action="store_true", help="per-robot sweep of EE payload, floor friction and a lateral base push")
    ap.add_argument("--model-payload", choices=["plant", "estimate"],
                    help="plant: tell the controller the plant's payload (its model payload, Solver.set_model_payload); estimate: run the online payload estimator")
    ap.add_argument("--model-friction", choices=["plant"], help="with --vary: tell the MPC friction cone and the WBC friction pyramid each robot's floor friction (robot tuning rows)")
    ap.add_argument("--terrain", action="store_true", help="per-robot sweep of ramp angle and step rise under the feet")
    ap.add_argument("--state-estimator", action="store_true", help="the controller reads the base state estimate from the IMU, encoders and contact flags")
    ap.add_argument("--sensor-noise", choices=["reference"], help="with --state-estimator: the IMU noise of qm_gazebo/config/default.yaml")
    ap.add_argument("--attitude-filter", action="store_true", help="with --state-estimator: filter the IMU orientation before the estimator reads it")
    ap.add_argument("--slip-detector", action="store_true", help="with --state-estimator: keep slipping stance feet out of the estimate")
    ap.add_argument("--gait-commands", action="store_true", help="time the device gait schedule in the loop and run a gait switch sweep")
    ap.add_argument("--ee-goals", action="store_true", help="end-effector goals on the device command timeline: a reach sweep and the target call's time")
    ap.add_argument("--ee-tuning", action="store_true", help="with --ee-goals: the reach sweep again with per-robot end-effector weights, WBC end-effector gains and kd_arm_wbc")
    ap.add_argument("--respawn", action="store_true", help="restart robots that fell (hold 0.1 s) on the reference IMU noise without the attitude filter: episode rates")
    ap.add_argument("--randomize", action="store_true", help="with --respawn: a new plant per episode (friction, payload, push): falls per friction x push bin")
    ap.add_argument("--spawn", action="store_true", help="with --respawn: new ground per episode (tile, offset, yaw): falls per tile x heading bin")
    ap.add_argument("--at-here", action="store_true", help="with --respawn: restarts where robots fell against restarts at the start on a stairs tile: "
                                                            "wall time, distance along the tile, here + place device time")
    ap.add_argument("--metrics", action="store_true", help="per-episode metrics: wall time with and without them, per-call times, column medians of a respawn run")
    ap.add_argument("--timeline", action="store_true", help="with --respawn: a new command timeline per episode (gait switches, cmd_vel steps): sampler time, "
                                                            "wall time, falls and velocity error per transition")
    ap.add_argument("--curriculum", action="store_true", help="with --respawn: per-robot levels stepped from each episode's outcome: update time, wall time, "
                                                              "an up-down staircase on the push against a uniform sweep")
    ap.add_argument("--snapshot", action="store_true", help="robot-state snapshots with every component running: bytes per robot, save and load times, and a "
                    "session branching every robot every window against one without restores")
    ap.add_argument("--session", action="store_true", help="closed_loop.run against a Session stepped one window at a time, without commands and with a "
                                                           "torch heading controller's command every window: wall time per simulated second, the command kernel's time")
    ap.add_argument("--ee-paths", action="store_true", help="end-effector paths: the target call's time with and without path robots, and a 10 cm square "
                    "traced by every robot standing: hand error along the path and at the final waypoint, wall time with and without the path")
    ap.add_argument("--ee-frame", action="store_true", help="end-effector targets in the heading frame: the target call's time with no, all-world and all-heading "
                                                            "frame rows, and a turning sweep over start yaws and yaw rates in both frames; with --respawn: "
                                                            "that run with every robot's targets in its heading frame")
    ap.add_argument("--ee-path-draw", action="store_true", help="per-episode end-effector paths: the sampler's time against the plant step, a respawning run "
                    "with and without draws, and the hand error against drawn 4-waypoint paths of 256 standing robots")
    args = ap.parse_args()
    if args.ee_path_draw:
        return ee_path_draw_main(args)
    if args.ee_frame and not args.respawn:
        return ee_frame_main(args)
    if args.ee_paths:
        return ee_paths_main(args)
    if args.session:
        return session_main(args)
    if args.snapshot:
        return snapshot_main(args)
    if args.curriculum and not args.respawn:
        ap.error("--curriculum needs --respawn")
    if args.curriculum:
        return curriculum_main(args)
    if args.metrics:
        return metrics_main(args)
    if args.timeline and not args.respawn:
        ap.error("--timeline needs --respawn")
    if args.timeline:
        return timeline_main(args)
    if args.randomize and not args.respawn:
        ap.error("--randomize needs --respawn")
    if args.spawn and not args.respawn:
        ap.error("--spawn needs --respawn")
    if args.at_here and not args.respawn:
        ap.error("--at-here needs --respawn")
    if args.at_here:
        return at_here_main(args)
    if args.respawn:
        return respawn_main(args)
    if args.ee_tuning and not args.ee_goals:
        ap.error("--ee-tuning needs --ee-goals")
    if args.model_friction and not args.vary:
        ap.error("--model-friction needs --vary")
    if args.vary and args.terrain:
        ap.error("--vary and --terrain are separate sweeps")
    if args.sensor_noise and not args.state_estimator:
        ap.error("--sensor-noise needs --state-estimator")
    if args.attitude_filter and not args.state_estimator:
        ap.error("--attitude-filter needs --state-estimator")
    if args.slip_detector and not args.state_estimator:
        ap.error("--slip-detector needs --state-estimator")
    import torch
    import qm_control_b200 as q
    from qm_control_b200 import closed_loop
    if not torch.cuda.is_available():
        raise SystemExit("bench_closedloop.py: no CUDA device — the product path has no CPU fallback")
    dev = torch.device("cuda", 0); B = args.batch; sim_s = args.duration; cmd = (args.vx, 0.0, 0.0, 0.0)
    solver = q.Solver(batch=B, device=0)
    xy = np.zeros((B, 3)); xy[:, 0] = 2.0 * (np.arange(B) % 64); xy[:, 1] = 2.0 * (np.arange(B) // 64)   # robots do not interact; spread for readability only
    kw = {}
    if args.vary:
        b = np.arange(B); bins = dict(payload_kg=np.linspace(0.0, 2.0, 5), mu=np.linspace(0.15, 1.0, 5), push_N=np.array([0.0, 60.0, 120.0, 180.0]))
        idx = dict(payload_kg=b % 5, mu=(b // 5) % 5, push_N=(b // 25) % 4)
        pl = np.zeros((B, 8)); pl[:, 0] = bins["payload_kg"][idx["payload_kg"]]
        w = np.zeros((B, 12)); w[:, 1] = bins["push_N"][idx["push_N"]]
        kw = dict(payload=pl, friction_mu=bins["mu"][idx["mu"]], pushes=(np.full(B, 0.4), np.full(B, 0.1), w))
    if args.terrain:
        from qm_control_b200 import terrain as T
        b = np.arange(B); bins = dict(ramp_deg=np.array([0.0, 5.0, 10.0, 15.0]), step_rise_m=np.array([0.0, 0.03, 0.06, 0.09]))
        idx = dict(ramp_deg=b % 4, step_rise_m=(b // 4) % 4)
        tiles = np.stack([T.ramp(a, start=0.35) + T.stairs(r, 0.3, start=0.35) for a in bins["ramp_deg"] for r in bins["step_rise_m"]])
        ter = dict(tiles=tiles, cell=T.CELL, tile=idx["ramp_deg"] * 4 + idx["step_rise_m"], origin=T.centred_origin(xy[:, :2]))
        kw = dict(terrain=ter)
    told = {"plant": dict(model_payload="plant"), "estimate": dict(payload_estimator=True), None: {}}[args.model_payload]
    if args.model_friction:
        told = dict(told, tuning=dict(friction_mu="plant", wbc_friction="plant"))
    se = dict(state_estimator=True, sensor_noise=args.sensor_noise, **({"attitude_filter": True} if args.attitude_filter else {}),
              **({"slip_detector": True} if args.slip_detector else {}), **({"ground_map": True} if args.terrain else {})) if args.state_estimator else {}
    def fresh():
        """with --state-estimator or --model-friction every run starts from a cold MPC and WBC state: a run whose robots fell leaves warm starts the next run
        must not inherit"""
        if args.state_estimator or args.model_friction:
            solver.mpc_reset(); solver.wbc_set_input_last(None)
    if args.state_estimator:
        box, unwrap = watch_state_est(solver)
    try:
        fresh()
        warm = closed_loop.run(solver, duration=sim_s, gait=args.gait, cmd_vel=cmd, xy_yaw=xy, **kw, **told, **se)   # warm-up run of the same length
    finally:
        if args.state_estimator:
            unwrap()
    pairs = []

    def sim_timer(start):
        if start:
            pairs.append([torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)]); pairs[-1][0].record()
        else:
            pairs[-1][1].record()
    fresh(); torch.cuda.synchronize(dev); t0 = time.perf_counter()
    r = closed_loop.run(solver, duration=sim_s, gait=args.gait, cmd_vel=cmd, xy_yaw=xy, sim_timer=sim_timer, **kw, **told, **se)
    torch.cuda.synchronize(dev); wall = time.perf_counter() - t0
    sim_ms = float(np.sum([a.elapsed_time(b) for a, b in pairs])); per_call = sim_ms / len(pairs)
    pct = lambda a: {"p50": float(np.percentile(a, 50)), "p95": float(np.percentile(a, 95)), "max": float(np.max(a))}

    def quality(r):
        dist = np.linalg.norm(r["base"][-1, :, :2] - r["start_base"][:, :2], axis=1)
        dpos = np.max(np.linalg.norm(r["ee"][:, :, :3] - r["start_ee"][None, :, :3], axis=2), axis=0) * 1e3
        dot = np.clip(np.abs(np.sum(r["ee"][:, :, 3:] * r["start_ee"][None, :, 3:], axis=2)), 0.0, 1.0); dang = np.max(np.degrees(2.0 * np.arccos(dot)), axis=0)
        return dist, dpos, dang

    def vary_bins(r, axis):
        dist, dpos, dang = quality(r); base = r["base"]; ground = 0.0
        if args.terrain:   # height above the ground under the base
            ground = T.height(ter["tiles"], ter["cell"], ter["tile"][None], ter["origin"][None], base[:, :, :2])
        fallen = ~(np.all(np.isfinite(base), axis=(0, 2)) & (np.min(base[:, :, 2] - ground, axis=0) > 0.3) & (np.max(np.abs(base[:, :, 4:6]), axis=(0, 2)) < 0.3))
        return [{"value": float(val), "robots": int(np.sum(idx[axis] == i)), "fallen": int(np.sum(fallen[idx[axis] == i])),
                 "base_distance_m_p50": float(np.percentile(dist[idx[axis] == i], 50)),
                 **({"base_distance_m": pct(dist[idx[axis] == i])} if args.terrain else
                    {"ee_max_pos_dev_mm": pct(dpos[idx[axis] == i]), "ee_max_ori_dev_deg_p50": float(np.percentile(dang[idx[axis] == i], 50))})}
                for i, val in enumerate(bins[axis])]
    def upright(r):
        base = r["base"]
        return np.all(np.isfinite(base), axis=(0, 2)) & (np.min(base[:, :, 2], axis=0) > 0.3) & (np.max(np.abs(base[:, :, 4:6]), axis=(0, 2)) < 0.3)
    dist, dpos, dang = quality(r)
    name, limit = card()
    extra = {}
    if args.vary:
        extra["vary"] = {"label": "per-robot sweep; fallen = min base z <= 0.3 m or |roll|, |pitch| >= 0.3 rad or non-finite", "push": "lateral +y base force for 0.1 s from 0.4 s",
                         "bins": {axis: vary_bins(r, axis) for axis in bins}}
        if args.model_payload == "estimate":
            err = np.abs(r["payload_est"][-1, :, 0] - kw["payload"][:, 0])
            extra["vary"]["payload_estimate_error_kg"] = [{"value": float(val), "p50": float(np.percentile(err[idx["payload_kg"] == i], 50)), "max": float(np.max(err[idx["payload_kg"] == i]))}
                                                          for i, val in enumerate(bins["payload_kg"])]
        if args.model_payload:
            extra["vary"]["model_payload"] = {"plant": "the controller is told the plant's payload (bins)", "estimate": "the controller runs the online payload estimate (bins)"}[
                args.model_payload] + "; payload_kg_not_told: the same sweep, controller not told"
            extra["vary"]["payload_kg_not_told"] = vary_bins(closed_loop.run(solver, duration=sim_s, gait=args.gait, cmd_vel=cmd, xy_yaw=xy, **kw), "payload_kg")
        if args.model_friction:
            extra["vary"]["model_friction"] = "the MPC cone and the WBC pyramid are told the plant's floor friction (bins); mu_not_told: the same sweep, controller not told; both arms from a cold MPC and WBC state"
            fresh(); extra["vary"]["mu_not_told"] = vary_bins(closed_loop.run(solver, duration=sim_s, gait=args.gait, cmd_vel=cmd, xy_yaw=xy, **kw), "mu")
    if args.terrain:
        extra["terrain"] = {"label": "per-robot sweep, controller blind to the terrain; fallen = height above the ground under the base <= 0.3 m or |roll|, |pitch| >= 0.3 rad "
                                     "or non-finite", "tiles": "ground z = 0 up to 0.35 m ahead of the start, then a ramp (deg) with steps (rise m, run 0.3 m) on it",
                            "bins": {axis: vary_bins(r, axis) for axis in bins}, "plant_step": plant_step_times(solver, ter, xy)}
    if args.model_payload == "estimate":
        extra["payload_est"] = {**est_step_times(solver, xy), "gpu": name, "power_limit": limit}
    if args.state_estimator:
        mx, last = box["max"].cpu().numpy(), box["last"].cpu().numpy()
        drift = np.linalg.norm(warm["base_est"][-1, :, 0:2] - warm["base"][-1, :, 0:2], axis=1)
        fresh(); truth = closed_loop.run(solver, duration=sim_s, gait=args.gait, cmd_vel=cmd, xy_yaw=xy, **kw, **told)
        t_dist, t_dpos, t_dang = quality(truth)
        extra["state_est"] = {**state_est_times(solver, xy), "gpu": name, "power_limit": limit, "sensor_noise": args.sensor_noise or "none",
                              "errors": {"label": "over the robots, from the warm-up run (the timed run's twin)", "z_abs_m_over_run": pct(mx[:, 0]), "z_abs_m_at_end": pct(last[:, 0]),
                                         "v_abs_m_s_over_run": pct(mx[:, 1]), "v_abs_m_s_at_end": pct(last[:, 1]), "xy_drift_m_at_end": pct(drift),
                                         "zyx_abs_rad_over_run": pct(mx[:, 2]), "zyx_abs_rad_at_end": pct(last[:, 2])},
                              "fallen": int(np.sum(~upright(r))), "fallen_warmup": int(np.sum(~upright(warm))), "ground_truth": {"label": "the same sweep, controller reading the plant's true state", "fallen": int(np.sum(~upright(truth))),
                                                                                    "base_distance_m": pct(t_dist), "ee_max_pos_dev_mm": pct(t_dpos), "ee_max_ori_dev_deg": pct(t_dang),
                                                                                    "robots_with_status_bits": int(np.count_nonzero(np.bitwise_or.reduce(truth["status"], axis=0)))}}
        if args.terrain:
            def fallen(run):
                base = run["base"]; ground = T.height(ter["tiles"], ter["cell"], ter["tile"][None], ter["origin"][None], base[:, :, :2])
                return ~(np.all(np.isfinite(base), axis=(0, 2)) & (np.min(base[:, :, 2] - ground, axis=0) > 0.3) & (np.max(np.abs(base[:, :, 4:6]), axis=(0, 2)) < 0.3))
            f_est, f_truth = fallen(warm), fallen(truth)
            extra["terrain"]["state_est"] = {
                "label": "per bin: the estimate arm (the warm-up run, the timed run's twin, the estimator on a perfect ground map) and the true-state arm of the "
                         "same sweep; |z_hat - z| over the run from the error watch", **ground_map_times(solver, ter, xy), "gpu": name, "power_limit": limit,
                "bins": {axis: [{"value": float(val), "robots": int(np.sum(idx[axis] == i)), "fallen_estimate": int(np.sum(f_est[idx[axis] == i])),
                                 "fallen_truth": int(np.sum(f_truth[idx[axis] == i])), "z_abs_m_over_run_p50": float(np.percentile(mx[idx[axis] == i, 0], 50)),
                                 "z_abs_m_over_run_p95": float(np.percentile(mx[idx[axis] == i, 0], 95))} for i, val in enumerate(bins[axis])] for axis in bins}}
        if args.attitude_filter:
            fresh(); raw = closed_loop.run(solver, duration=sim_s, gait=args.gait, cmd_vel=cmd, xy_yaw=xy, **kw, **told, state_estimator=True, sensor_noise=args.sensor_noise,
                                           **({"ground_map": True} if args.terrain else {}))
            n_dist, n_dpos, n_dang = quality(raw)
            extra["attitude"] = {**attitude_times(solver, xy), "gpu": name, "power_limit": limit,
                                 "without_filter": {"label": "the same sweep on the estimate, without the attitude filter", "fallen": int(np.sum(~upright(raw))),
                                                    "base_distance_m": pct(n_dist), "ee_max_pos_dev_mm": pct(n_dpos), "ee_max_ori_dev_deg": pct(n_dang),
                                                    "robots_with_status_bits": int(np.count_nonzero(np.bitwise_or.reduce(raw["status"], axis=0)))}}
        if args.slip_detector:
            box2, unwrap2 = watch_state_est(solver)
            try:
                fresh(); nodet = closed_loop.run(solver, duration=sim_s, gait=args.gait, cmd_vel=cmd, xy_yaw=xy, **kw, **told, **{k: v for k, v in se.items() if k != "slip_detector"})
            finally:
                unwrap2()
            arms = {"with_detector": (warm, mx[:, 1]), "without_detector": (nodet, box2["max"].cpu().numpy()[:, 1])}

            def slip_arm(run, verr, sel):
                d = np.linalg.norm(run["base_est"][-1, sel, 0:2] - run["base"][-1, sel, 0:2], axis=1)
                return {"robots": int(np.sum(sel)), "fallen": int(np.sum(~upright(run)[sel])), "xy_drift_m_at_end_p50": float(np.percentile(d, 50)),
                        "xy_drift_m_at_end_p95": float(np.percentile(d, 95)), "v_abs_m_s_over_run_p50": float(np.percentile(verr[sel], 50)),
                        "v_abs_m_s_over_run_p95": float(np.percentile(verr[sel], 95)),
                        **({"robots_flagged": int(np.sum(run["slip"].any(axis=0)[sel]))} if "slip" in run else {})}
            every = np.ones(B, dtype=bool)
            extra["slip"] = {**slip_times(solver, xy), "gpu": name, "power_limit": limit, "robots_flagged_timed_run": int(np.sum(r["slip"].any(axis=0))),
                             "label": "with_detector: the warm-up run (the timed run's twin); without_detector: the same sweep without the detector, in the same process",
                             **{tag: slip_arm(run, verr, every) for tag, (run, verr) in arms.items()}}
            if args.vary:
                extra["slip"]["mu_bins"] = [{"mu": float(val), **{tag: slip_arm(run, verr, idx["mu"] == i) for tag, (run, verr) in arms.items()}}
                                            for i, val in enumerate(bins["mu"])]
    if args.gait_commands:
        extra["gait_commands"] = {**gait_commands(solver, closed_loop, B, sim_s, cmd, xy, kw, upright), "gpu": name, "power_limit": limit,
                                  "wall_s_per_sim_s_without_commands": wall / sim_s}
    if args.ee_goals:
        extra["ee_goals"] = {**ee_goals(solver, closed_loop, B, sim_s, xy, upright, tuning=args.ee_tuning), "gpu": name, "power_limit": limit, "wall_s_per_sim_s_without_commands": wall / sim_s}
    print(json.dumps({"metric": "robot_sim_seconds_per_s", "value": B * sim_s / wall, "unit": "robot-simulated-seconds per wall-clock second", "n_gpus": 1,
                      "wall_s_per_sim_s": wall / sim_s, "gpu": name, "power_limit": limit, "dtype": "f64", "data": "synthetic",
                      "plant": {"ms_per_call": per_call, "calls": len(pairs), "share_of_loop": sim_ms * 1e-3 / wall},
                      "quality": {"label": "this project's compliant-contact plant, not Gazebo/ODE: not comparable to README.md:116", "base_distance_m": pct(dist),
                                  "ee_max_pos_dev_mm": pct(dpos), "ee_max_ori_dev_deg": pct(dang),
                                  "robots_with_status_bits": int(np.count_nonzero(np.bitwise_or.reduce(r["status"], axis=0))),
                                  "min_base_height_m": float(np.min(r["base"][:, :, 2])), "max_abs_roll_pitch_rad": float(np.max(np.abs(r["base"][:, :, 4:6])))},
                      "config": {"workload": "closed loop: %s, cmd_vel %.2f m/s, MPC 100 Hz / WBC 500 Hz / plant 1 kHz (4 substeps), 9 ms command delay" % (args.gait, args.vx),
                                 "batch": B, "simulated_s": sim_s, "warmup": "one run of the same length", **({"model_payload": args.model_payload} if args.model_payload else {}),
                                 **({"state_estimator": True, "sensor_noise": args.sensor_noise or "none", "attitude_filter": args.attitude_filter,
                                     "slip_detector": args.slip_detector} if args.state_estimator else {})},
                      **extra}))


if __name__ == "__main__":
    main()
