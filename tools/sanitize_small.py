"""Tiny end-to-end run for compute-sanitizer (memcheck / racecheck / initcheck): every kernel of the library once, 5 robots (mixed gaits); then the
per-episode spawn sampler inside a few respawned windows of closed_loop.run on terrain, with the ground-map link and the estimator, attitude filter and
slip detector rows live."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import qm_control_b200 as q  # noqa: E402
from qm_control_b200 import synthetic  # noqa: E402

B = 5
ctrl = q.QMController(batch=B, dt=0.015); s = ctrl.solver
prob, wbc = synthetic.make_batch(np.arange(B), config=5)
ctrl.starting(wbc["rbd"], time=12.0)
for tick in range(2):
    p = dict(prob); p["t0"] = ctrl.t_obs.copy(); p["x0"] = ctrl.x_obs.copy()
    nt, tt, ts = ctrl.targetTrajectories(0, np.tile([0.2, 0.0, 0.0, 0.1], (B, 1)))
    cmd, status = s.tick(p, p["t0"] + 0.002, wbc["rbd"], wbc["period"])
    cmd2, status2 = ctrl.update(wbc["rbd"], 0.002)
    eff, st = s.hw_write(ctrl.t_obs, np.full(B, 0.002), ctrl.joint_cmd, wbc["rbd"][:, 6:24], wbc["rbd"][:, 30:48])
# solver variants (IPM thresholds; DDP: rollout kernels) and the multi-GPU pack path on one rank
import torch  # noqa: E402
for name in ("ipm", "ddp", "sqp"):
    s.mpc_set_solver(name); out = s.mpc_solve(prob)
dev = torch.device("cuda", 0); cmd_d = torch.from_numpy(cmd).to(dev); all_d = torch.zeros((B, 18), dtype=torch.float64, device=dev)
perm = s.gait_bin_permutation(prob); s.allgather_torque(cmd_d, all_d, torch.from_numpy(perm).to(dev)); torch.cuda.synchronize()
s1 = q.Solver(batch=B, dt=0.015, wbc_variant=1); c1, st1 = s1.tick(prob, prob["t0"] + 0.002, wbc["rbd"], wbc["period"])
# per-episode spawns (DESIGN.md §4.12): 50 ms with a respawn every 20 ms, so the sampler runs at the start and at two window boundaries
from qm_control_b200 import closed_loop, terrain as T  # noqa: E402
s2 = q.Solver(batch=B); xy = np.c_[3.0 * np.arange(B), np.zeros(B), np.zeros(B)]
ter = dict(tiles=np.stack([T.flat(), T.stairs(0.06, 0.25)]), cell=T.CELL, tile=np.arange(B) % 3 - 1, origin=T.centred_origin(xy[:, :2]))
r = closed_loop.run(s2, duration=0.05, gait="trot", xy_yaw=xy, terrain=ter, state_estimator=True, attitude_filter=True, slip_detector=True, ground_map=True,
                    respawn=dict(on_fall=False, every=0.02), spawn=dict(seed=1, tile=(-1, 1), dx=(-0.2, 0.0), dy=(-0.1, 0.1), yaw=(-np.pi, np.pi)))
print("sanitize_small ok", status, status2, out["status"], st1, "spawn episodes", r["episode"][-1], "rows", r["spawn_params"].shape)
