"""Tiny run for compute-sanitizer memcheck at the node limit: one robot of five needs more nodes than the handle holds (a trot with 40 ms phases needs
102 at dt 0.015), through qmb200_mpc_solve, qmb200_mpc_solve_dev and qmb200_tick.  The overflowing robot must carry QMB200_ST_OVERFLOW and no kernel may
touch memory past nmax:  compute-sanitizer --tool memcheck python tools/sanitize_overflow.py"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import qm_control_b200 as q  # noqa: E402
from qm_control_b200 import synthetic  # noqa: E402

B, F, T0 = 5, 2, 12.0
prob, wbc = synthetic.make_batch(np.arange(B), config=4)
ev = [T0 - 0.02 + 0.04 * i for i in range(30)]; md = [15] + [9 if i % 2 == 0 else 6 for i in range(29)] + [15]
prob["event_times"][F] = 0.0; prob["event_times"][F, :30] = ev; prob["modes"][F] = 15; prob["modes"][F, :31] = md; prob["n_events"][F] = 30
import torch  # noqa: E402
dev = torch.device("cuda", 0); keys = ("t0", "x0", "n_events", "event_times", "modes", "n_target", "target_times", "target_states")
for max_nodes in (0, 101):                                                   # the default handle (88 nodes) and one node short
    s = q.Solver(batch=B, dt=0.015, max_nodes=max_nodes)
    out = s.mpc_solve(prob)
    s.mpc_reset(); s.mpc_solve_dev({k: torch.from_numpy(np.ascontiguousarray(prob[k])).to(dev) for k in keys}); torch.cuda.synchronize(); sol = s.mpc_get_solution()
    s.mpc_reset(); cmd, st = s.tick(prob, prob["t0"] + 0.002, wbc["rbd"], wbc["period"])
    assert out["status"][F] & 2 and sol["status"][F] & 2 and (st[F] >> 8) & 2, (out["status"], sol["status"], st)
    print("nmax %d: status solve %s dev %s tick %s" % (s.nmax, out["status"].tolist(), sol["status"].tolist(), [hex(int(v)) for v in st]))
print("sanitize_overflow ok")
