"""Aviary-level drone-steps/s with one flight mode per drone (``BatchedAviary.set_mode(list)``).  A CUDA-event pair around each
``step(n_steps)`` with the library's Philox motor noise, after warm-up.  One JSON line per layout:

    uniform_m<M>   every drone in mode M (the single-mode kernels), M = -1 .. 7
    tile           modes -1 .. 7 cycled per 32-drone tile (every warp flies one mode)
    interleaved    modes -1 .. 7 cycled lane by lane (every warp flies all nine)
    random         modes drawn at random per drone
    tile_k2        the tile layout on a cf2x / primitive_drone model set (models alternate per tile as well)
    fw_uniform_m<M> / fw_interleaved   fixed-wing, modes -1 / 0, at --fw-drones

    python tools/bench_mixed_modes.py [--drones 65536] [--fw-drones 16384] [--n-steps 10] [--reps 20] [--warmup 5]

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


def time_steps(av, n_steps, reps, warmup, dev):
    for _ in range(warmup):
        av.step(n_steps)
    torch.cuda.synchronize(dev)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        av.step(n_steps)
        b.record()
    torch.cuda.synchronize(dev)
    ms = sorted(a.elapsed_time(b) for a, b in ev)
    return ms[len(ms) // 2]  # median launch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--drones", type=int, default=65536)
    ap.add_argument("--fw-drones", type=int, default=16384)
    ap.add_argument("--n-steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
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

    def run(name, kind, n, opts, modes):
        start = np.column_stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(40, 60, n)]).astype(np.float32)
        av = BatchedAviary(start, np.zeros((n, 3), dtype=np.float32), drone_type=kind, drone_options=opts, seed=0, device=dev)
        av.set_mode(modes if isinstance(modes, int) else modes.tolist())
        if kind == "quadx":  # hover-ish commands that every mode accepts: thrust / pwm / height near the start
            sp = np.column_stack([np.zeros((n, 3)), np.full(n, 0.4)])
            held = np.isin(np.broadcast_to(modes, (n,)), (2, 3, 4, 7))
            sp[held, 3] = start[held, 2]
            sp[np.broadcast_to(modes, (n,)) == 7, :2] = start[np.broadcast_to(modes, (n,)) == 7, :2]
        else:
            sp = np.column_stack([np.zeros((n, 3)), np.full(n, 0.6), np.zeros((n, 2))])
        av.set_all_setpoints(torch.as_tensor(sp, dtype=torch.float32, device=dev))
        ms = time_steps(av, args.n_steps, args.reps, args.warmup, dev)
        print(json.dumps({"layout": name, "kind": kind, "drones": n, "models": len(av.models), "n_steps": args.n_steps, "gpu": prop.name,
                          "power_limit_w,sm_max_mhz": q, "ms_per_launch": ms, "drone_steps_per_s": n * args.n_steps / (ms * 1e-3)}), flush=True)
        del av

    n = args.drones
    i = np.arange(n)
    cf2x = dict(drone_model="cf2x")
    for m in range(-1, 8):
        run(f"uniform_m{m}", "quadx", n, cf2x, m)
    run("tile", "quadx", n, cf2x, -1 + (i // 32) % 9)
    run("interleaved", "quadx", n, cf2x, -1 + i % 9)
    run("random", "quadx", n, cf2x, rng.integers(-1, 8, n))
    k2 = [cf2x if (j // 32) % 2 == 0 else dict(drone_model="primitive_drone") for j in range(n)]
    run("tile_k2", "quadx", n, k2, -1 + (i // 32) % 9)
    nf = args.fw_drones
    for m in (-1, 0):
        run(f"fw_uniform_m{m}", "fixedwing", nf, None, m)
    run("fw_interleaved", "fixedwing", nf, None, np.arange(nf) % 2 - 1)


if __name__ == "__main__":
    main()
