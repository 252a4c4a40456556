"""Aviary steps per second of a batch of several vehicle kinds (``BatchedAviary(drone_type=[...])``, one launch per step)
against three single-kind batches, one per kind, over the same drones, stepped back to back (three launches per step).
CUDA events around each ``step(n_steps)`` with the library's Philox motor noise, after warm-up; the median of ``--reps``.

Sizes: n = 3 (the reference's examples/core/08_mixed_drones.py), 3 x 1 024 and 3 x 21 845 (~65 536), a third of each kind,
with the kinds grouped (all QuadX, then all fixed-wing, then all rockets) and interleaved drone by drone.  One JSON line per
(size, layout):

    python tools/bench_mixed_kinds.py [--n-steps 1] [--reps 50] [--warmup 10]

Nothing is written to the tree."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

KINDS = ("quadx", "fixedwing", "rocket")


def time_steps(avs, n_steps, reps, warmup):
    for _ in range(warmup):
        for av in avs:
            av.step(n_steps)
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        for av in avs:
            av.step(n_steps)
        b.record()
    torch.cuda.synchronize()
    ms = sorted(a.elapsed_time(b) for a, b in ev)
    return ms[len(ms) // 2]


def setpoints(kinds, start):
    """hover-ish commands: QuadX mode 7 holding its start, fixed-wing mode 0 at 0.8 throttle, rockets ignited at 0.6"""
    sp = np.zeros((len(kinds), 7), dtype=np.float32)
    for i, k in enumerate(kinds):
        if k == "quadx":
            sp[i, :4] = [start[i, 0], start[i, 1], 0.0, start[i, 2]]
        elif k == "fixedwing":
            sp[i, :4] = [0.0, 0.0, 0.0, 0.8]
        else:
            sp[i] = [0.0, 0.0, 0.0, 1.0, 0.6, 0.0, 0.0]
    return sp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-steps", type=int, default=1)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    from pyflyt_b200.core.aviary import BatchedAviary

    dev = torch.device("cuda", 0)
    prop = torch.cuda.get_device_properties(dev)
    try:  # read-only query: the power limit is part of the number
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    rng = np.random.default_rng(0)
    for per_kind in (1, 1024, 21845):
        n = 3 * per_kind
        for layout in ("grouped", "interleaved"):
            kinds = [KINDS[i // per_kind] for i in range(n)] if layout == "grouped" else [KINDS[i % 3] for i in range(n)]
            ks = np.array(kinds)
            start = np.column_stack([rng.uniform(-5, 5, n), rng.uniform(-5, 5, n), rng.uniform(200, 300, n)]).astype(np.float32)
            orn = np.zeros((n, 3), dtype=np.float32)
            orn[ks == "rocket", 0] = np.pi / 2
            modes = [7 if k == "quadx" else 0 for k in kinds]
            sp = setpoints(kinds, start)
            mixed = BatchedAviary(start, orn, drone_type=kinds, seed=0, device=dev)
            mixed.set_mode(modes)
            mixed.set_all_setpoints(sp)
            singles = []
            for k in KINDS:  # the same drones, one batch per kind
                m = ks == k
                av = BatchedAviary(start[m], orn[m], drone_type=k, seed=0, device=dev)
                av.set_mode(7 if k == "quadx" else 0)
                av.set_all_setpoints(torch.as_tensor(sp[m][:, : av.setpoint_dim]))
                singles.append(av)
            ms_mixed = time_steps([mixed], args.n_steps, args.reps, args.warmup)
            ms_single = time_steps(singles, args.n_steps, args.reps, args.warmup)
            print(json.dumps({"drones": n, "layout": layout, "n_steps": args.n_steps, "gpu": prop.name, "power_limit_w,sm_max_mhz": q,
                              "mixed_ms": ms_mixed, "three_single_kind_ms": ms_single,
                              "mixed_aviary_steps_per_s": args.n_steps / (ms_mixed * 1e-3),
                              "three_single_kind_aviary_steps_per_s": args.n_steps / (ms_single * 1e-3),
                              "speedup_of_one_launch": ms_single / ms_mixed}), flush=True)
            del mixed, singles


if __name__ == "__main__":
    main()
