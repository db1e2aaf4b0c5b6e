"""Cost of per-robot controller tuning rows on the flagship tick (bench.py's workload: 8192 robots, trot, horizon 1 s, dt 0.01, one chain).

Times qmb200_tick_dev on one handle without rows, with neutral rows (the handle's own values) and with distinct rows on every robot, alternating the
three in rounds so that drift of the shared card hits all of them alike.  Prints one JSON line with ms per tick per arm, the card and its power limit.

  python tools/bench_tuning.py [--batch 8192] [--rounds 5] [--ticks 10]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def distinct_rows(handle_row, n, seed=5):
    """n distinct rows: row 0 is the handle's own, the others scale every field by a factor of its own in [0.5, 1.5]"""
    rows = np.repeat(np.asarray(handle_row, dtype=np.float64)[None], n, axis=0)
    rows[1:] *= np.random.default_rng(seed).uniform(0.5, 1.5, rows[1:].shape)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8192); ap.add_argument("--rounds", type=int, default=5); ap.add_argument("--ticks", type=int, default=10)
    args = ap.parse_args()
    import torch
    import bench
    import qm_control_b200 as q
    from qm_control_b200 import _lib
    if not torch.cuda.is_available():
        raise SystemExit("bench_tuning.py: no CUDA device — the product path has no CPU fallback")
    dev = torch.device("cuda", 0); side = torch.cuda.Stream(dev); stream = side.cuda_stream   # as bench.py: the ticks run on a side stream
    loop = bench.TickLoop(q, torch, dev, 0, stream, args.batch, np.arange(args.batch), bench.CONFIG, 1, 0)
    s = loop.solver; B = args.batch; h = s.get_handle_tuning()
    as_dict = lambda r: {k: r[:, off] if w == 1 else r[:, off:off + w] for k, (off, w) in _lib.TUNING_LAYOUT.items()}
    arms = {"none": None, "neutral_rows": as_dict(np.repeat(h[None], B, axis=0)), "distinct_rows": as_dict(np.repeat(distinct_rows(h, 8), B // 8 + 1, axis=0)[:B])}
    ms = {k: [] for k in arms}
    for name, t in arms.items():   # warm-up of every arm
        s.set_robot_tuning(t); [loop.step() for _ in range(3)]; torch.cuda.synchronize(dev)
    for _ in range(args.rounds):
        for name, t in arms.items():
            s.set_robot_tuning(t); loop.step(); torch.cuda.synchronize(dev); t0 = time.perf_counter()
            for _ in range(args.ticks):
                loop.step()
            torch.cuda.synchronize(dev); ms[name].append((time.perf_counter() - t0) * 1e3 / args.ticks)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"batch": B, "ticks_per_round": args.ticks, "card": card, "ms_per_tick": ms, "median_ms": {k: float(np.median(v)) for k, v in ms.items()}}))


if __name__ == "__main__":
    main()
